// One frame of the online tracker's bookkeeping as ONE cooperative routine (a single CTA on the device).
//
// Follows src/trackformer/models/tracker.py:266-548 decision by decision, in the reference's order:
//   prune inactive tracks (270-273)  ->  established tracks + re-identification queries (329-373)  ->  track NMS
//   (388-406)  ->  new detections above the score threshold (425-436)  ->  public-detection gating (122-164)  ->
//   ReID by embedding distance + Hungarian matching or by greedy centre distance (166-264)  ->  new tracks (470-492)  ->
//   detection NMS with established tracks at +inf (494-515)  ->  results (533-545)  ->  inactive counters, reid_sim_only.
// All box arithmetic is fp32 with separately rounded products and sums (no FMA contraction), i.e. the values the
// reference's torch / numpy ops produce; the assignment problem is solved in double precision like scipy.
//
// The same source is compiled twice: by nvcc into track_step.cu's kernel, and by g++ (one "thread") into the test-only
// host build that tests/test_track_step_cpu.py replays the reference-recorded sequences through; host_device.h holds
// the only difference between the two.
#pragma once

#include <math.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "host_device.h"
#include "lsa_core.h"

namespace tfb200_track {

constexpr int kMaxRows = 2048;          // tracks + object queries of one frame
constexpr int kThreads = 256;

struct Shared {
  int act[kMaxRows];                    // work-table rows of the active tracks, list order
  int inact[kMaxRows];                  // ... of the inactive tracks
  int tmp[kMaxRows];
  int flag[kMaxRows];
  int na, ni, nin, nd, err, track_num, num_reids, nres, nquery_next;
};

struct Box { float x0, y0, x1, y1; };

HD_FN float ts_clampf(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }

// boxes[i] of this frame: the detector's pixel box, clipped to the image unless the model allows overflow
// (tracker.py:323-327, torchvision clip_boxes_to_image)
HD_FN Box ts_row_box(const TfbTrackStepArgs& a, int i) {
  const float* r = a.rows + size_t(i) * 6;
  Box b{r[2], r[3], r[4], r[5]};
  if (!a.overflow_boxes) {
    const float w = float(a.img_w), h = float(a.img_h);
    b.x0 = ts_clampf(b.x0, 0.f, w); b.x1 = ts_clampf(b.x1, 0.f, w);
    b.y0 = ts_clampf(b.y0, 0.f, h); b.y1 = ts_clampf(b.y1, 0.f, h);
  }
  return b;
}
HD_FN Box ts_load(const float* p, int r) { return Box{p[4 * r], p[4 * r + 1], p[4 * r + 2], p[4 * r + 3]}; }
HD_FN void ts_store(float* p, int r, const Box& b) { p[4 * r] = b.x0; p[4 * r + 1] = b.y0; p[4 * r + 2] = b.x1; p[4 * r + 3] = b.y1; }
HD_FN float ts_area(const Box& b) { return hd_fmul(hd_fsub(b.x1, b.x0), hd_fsub(b.y1, b.y0)); }
HD_FN float ts_cx(const Box& b) { return hd_fmul(hd_fadd(b.x0, b.x1), 0.5f); }     // (x0 + x1) / 2, exact either way
HD_FN float ts_cy(const Box& b) { return hd_fmul(hd_fadd(b.y0, b.y1), 0.5f); }

// torchvision box_iou / nms arithmetic: inter / (area_a + area_b - inter)
HD_FN float ts_iou(const Box& a, float area_a, const Box& b, float area_b) {
  float w = hd_fsub(fminf(a.x1, b.x1), fmaxf(a.x0, b.x0));
  float h = hd_fsub(fminf(a.y1, b.y1), fmaxf(a.y0, b.y0));
  w = w < 0.f ? 0.f : w;
  h = h < 0.f ? 0.f : h;
  const float inter = hd_fmul(w, h);
  return hd_fdiv(inter, hd_fsub(hd_fadd(area_a, area_b), inter));
}

// has_positive_area and within the patience window (tracker.py:171-174, 270-273)
HD_FN bool ts_alive(const TfbTrackState& s, int r, double patience) {
  const Box b = ts_load(s.pos, r);
  return b.x1 > b.x0 && b.y1 > b.y0 && double(s.count_inactive[r]) <= patience;
}

// ------------------------------------------------------------------------------------------------------------ NMS
// Greedy NMS over list[0..n) (torchvision.ops.nms semantics: descending score, stable; suppress IoU > thr), scores of
// rows that are not `fresh` replaced by +inf when fresh_only (tracker.py:503).  Survivors stay in list order; returns
// through sh.tmp / *n_out (thread 0).  Whole CTA.
HD_FN void ts_nms(const TfbTrackStepArgs& a, Shared& sh, int* list, int& n_ref, float thr, bool fresh_only, const int* fresh,
                  float* f_sc, float* f_area, float* f_box, int* order, int* dead) {
  const int n = n_ref;
  const TfbTrackState& S = a.in;
  for (int k = HD_TID; k < n; k += HD_NT) {
    const int r = list[k];
    const Box b = ts_load(S.pos, r);
    ts_store(f_box, k, b);
    f_area[k] = ts_area(b);
    f_sc[k] = (fresh_only && !fresh[r]) ? INFINITY : S.score[r];
    dead[k] = 0;
  }
  HD_SYNC();
  for (int k = HD_TID; k < n; k += HD_NT) {
    const float s = f_sc[k];
    int rank = 0;
    for (int m = 0; m < n; ++m) {
      const float t = f_sc[m];
      rank += (t > s) || (t == s && m < k);
    }
    order[rank] = k;
  }
  HD_SYNC();
  for (int p = 0; p < n; ++p) {
    const int i = order[p];
    if (dead[i]) continue;                                   // uniform: written before the last barrier
    const Box bi = ts_load(f_box, i);
    const float ai = f_area[i];
    for (int q = p + 1 + HD_TID; q < n; q += HD_NT) {
      const int j = order[q];
      if (dead[j]) continue;
      if (ts_iou(bi, ai, ts_load(f_box, j), f_area[j]) > thr) dead[j] = 1;
    }
    HD_SYNC();
  }
  HD_SYNC();
  if (HD_TID == 0) {
    int m = 0;
    for (int k = 0; k < n; ++k)
      if (!dead[k]) list[m++] = list[k];
    n_ref = m;
  }
  HD_SYNC();
}

// --------------------------------------------------------------------------------------- rectangular assignment
// scipy.optimize.linear_sum_assignment of dist[nr0][ld] (nc0 columns used), run by ONE warp; a tall problem is solved
// transposed.  rowmatch[r] = column assigned to row r, or -1 (only when nr0 > nc0, or for non-finite distances).
HD_FN void ts_lsa_warp(const float* dist, int ld, int nr0, int nc0, double* dws, int* iws, int* rowmatch) {
  namespace lsa = tfb200_lsa;
  const bool tr = nr0 > nc0;
  const int nr = tr ? nc0 : nr0, nc = tr ? nr0 : nc0;
  const lsa::Cols C{dws, dws + nc, iws, iws + nc, reinterpret_cast<uint8_t*>(iws + 2 * nc)};
  const lsa::Rows R{dws + 2 * nc, iws + 3 * nc, iws + 3 * nc + nr};
  for (int r = HD_LANE; r < nr0; r += HD_NLANES) rowmatch[r] = -1;
  lsa::Warp::Scratch scratch;
  const lsa::Strided cost{dist, tr ? 1 : size_t(ld), tr ? size_t(ld) : 1};
  if (lsa::solve<lsa::Warp>(nr, nc, cost, R, C, scratch))
    for (int r = HD_LANE; r < nr; r += HD_NLANES) rowmatch[tr ? R.col4row[r] : r] = tr ? r : R.col4row[r];
  HD_SYNCWARP();
}

// ---------------------------------------------------------------------------------------------------- the step
HD_FN void ts_step(const TfbTrackStepArgs& a, Shared& sh) {
  const int tid = HD_TID, nt = HD_NT;
  const TfbTrackState& S = a.in;
  const int cap = a.capacity, nq = a.nq, nqy = a.n_query;
  int* hs_src = a.iscratch;                 // [cap] row -> index into hs_embeds whose embedding the track takes, or -1
  int* order = hs_src + cap;                // [cap]
  int* dead = order + cap;                  // [cap]
  int* dl = dead + cap;                     // [cap] detections: object-query indices
  int* dsel = dl + cap;                     // [cap] per detection flags
  int* fresh = dsel + cap;                  // [cap] per row: track started this frame
  int* rowmatch = fresh + cap;              // [cap]
  int* lsa_i = rowmatch + cap;              // [5 * cap]
  float* f_sc = a.fscratch;                 // [cap]
  float* f_area = f_sc + cap;               // [cap]
  float* f_box = f_area + cap;              // [4 * cap]
  float* f_mat = f_box + 4 * cap;           // [cap * max(nq, n_public)] distance / IoU matrix

  // ---- A. start of the step: prune the inactive list (tracker.py:270-273); check the caller's query count
  if (tid == 0) {
    const int na = S.header[0], ni = S.header[1];
    sh.track_num = S.header[2];
    sh.num_reids = S.header[3];
    sh.err = 0;
    if (na < 0 || ni < 0 || nq < 0 || cap > kMaxRows || na + ni + nq > cap) sh.err = 2;
    else {
      for (int i = 0; i < na; ++i) sh.act[i] = i;
      int k = 0;
      for (int i = 0; i < ni; ++i)
        if (ts_alive(S, na + i, a.inactive_patience)) sh.inact[k++] = na + i;
      sh.na = na; sh.ni = k; sh.nin = na + ni;
      if (na + k != nqy) sh.err = 1;
    }
  }
  HD_SYNC();
  if (sh.err) {
    if (tid == 0) {
      for (int k = 0; k < 8; ++k) a.result[k] = 0;
      a.result[5] = sh.err;
      a.out.header[5] = sh.err;
    }
    return;
  }
  const int nin = sh.nin;
  const int na0 = sh.na;
  for (int r = tid; r < nin + nq; r += nt) { hs_src[r] = -1; fresh[r] = 0; }
  HD_SYNC();

  // ---- B/C. established tracks and re-identification queries (tracker.py:300-303, 329-386)
  if (nqy > 0) {
    for (int i = tid; i < nqy; i += nt) {
      const bool is_active = i < na0;
      const int r = is_active ? sh.act[i] : sh.inact[i - na0];
      if (is_active) ts_store(S.anchor, r, ts_load(S.pos, r));             // last_pos.append(pos.clone())
      const float score = a.rows[size_t(i) * 6], label = a.rows[size_t(i) * 6 + 1];
      const bool person = label == 0.f;
      int f;
      if (is_active) {
        if (score > a.track_obj_score_thresh && person) {
          S.score[r] = score;
          ts_store(S.pos, r, ts_row_box(a, i));
          hs_src[r] = i;
          S.count_termination[r] = 0;
          f = 1;
        } else {
          const int c = S.count_termination[r] + 1;
          S.count_termination[r] = c;
          f = c >= a.steps_termination ? 2 : 0;
        }
      } else {
        f = 0;
        if (score > a.reid_score_thresh && person) {
          S.score[r] = score;
          ts_store(S.pos, r, ts_row_box(a, i));
          hs_src[r] = i;
          f = 1;
        }
      }
      sh.flag[i] = f;
    }
    HD_SYNC();
    if (tid == 0) {
      int na = 0, ni = 0;
      for (int i = 0; i < na0; ++i)
        if (sh.flag[i] != 2) sh.tmp[na++] = sh.act[i];
      for (int i = na0; i < nqy; ++i)
        if (sh.flag[i]) { sh.tmp[na++] = sh.inact[i - na0]; ++sh.num_reids; }
      for (int i = na0; i < nqy; ++i)
        if (!sh.flag[i]) sh.inact[ni++] = sh.inact[i - na0];              // in place: ni <= i - na0
      for (int i = 0; i < na0; ++i)
        if (sh.flag[i] == 2) {                                              // tracks_to_inactive (tracker.py:86-91)
          const int r = sh.act[i];
          ts_store(S.pos, r, ts_load(S.anchor, r));
          sh.inact[ni++] = r;
        }
      for (int i = 0; i < na; ++i) sh.act[i] = sh.tmp[i];
      sh.na = na; sh.ni = ni;
    }
    HD_SYNC();
    if (a.track_nms_on && sh.na > 0)
      ts_nms(a, sh, sh.act, sh.na, a.track_nms_thresh, false, fresh, f_sc, f_area, f_box, order, dead);
  }

  // ---- E. new detections (tracker.py:408-436)
  for (int j = tid; j < nq; j += nt) {
    const float* r = a.rows + size_t(nqy + j) * 6;
    sh.flag[j] = r[0] > a.detection_obj_score_thresh && r[1] == 0.f;
  }
  HD_SYNC();
  if (tid == 0) {
    int nd = 0;
    for (int j = 0; j < nq; ++j)
      if (sh.flag[j]) dl[nd++] = j;
    sh.nd = nd;
  }
  HD_SYNC();

  // ---- F. public-detection gating (tracker.py:122-164)
  if (a.public_mode != 0) {
    const int nd = sh.nd, np = a.public_dets ? a.n_public : 0;
    HD_SYNC();                                  // every thread has read sh.nd before thread 0 rewrites it below
    if (nd > 0 && np > 0) {
      for (int e = tid; e < nd * np; e += nt) {
        const int i = e / np, j = e % np;
        const Box b = ts_row_box(a, nqy + dl[i]);
        const Box p = ts_load(a.public_dets, j);
        float m;
        if (a.public_mode == 1) {
          const float dx = hd_fsub(ts_cx(b), ts_cx(p)), dy = hd_fsub(ts_cy(b), ts_cy(p));
          m = hd_fadd(hd_fmul(dx, dx), hd_fmul(dy, dy));
        } else {
          m = ts_iou(b, ts_area(b), p, ts_area(p));
        }
        f_mat[e] = m;
      }
      for (int i = tid; i < nd; i += nt) dsel[i] = 0;
      HD_SYNC();
      if (tid == 0) {
        for (int j = 0; j < np; ++j) {
          int best = 0;
          float bv = f_mat[j];
          if (a.public_mode == 1) {
            for (int i = 1; i < nd; ++i) {                                  // numpy argmin: first minimum
              const float v = f_mat[i * np + j];
              if (v < bv) { bv = v; best = i; }
            }
            if (bv < ts_area(ts_row_box(a, nqy + dl[best]))) {
              for (int k = 0; k < np; ++k) f_mat[best * np + k] = 1e18f;
              dsel[best] = 1;
            }
          } else {
            for (int i = 1; i < nd && !(bv != bv); ++i) {                   // numpy argmax: first maximum, NaN first
              const float v = f_mat[i * np + j];
              if (v > bv || v != v) { bv = v; best = i; }
            }
            if (bv >= 0.5f) {
              for (int k = 0; k < np; ++k) f_mat[best * np + k] = 0.f;
              dsel[best] = 1;
            }
          }
        }
        int m = 0;
        for (int i = 0; i < nd; ++i)
          if (dsel[i]) dl[m++] = dl[i];
        sh.nd = m;
      }
    } else if (tid == 0) {
      sh.nd = 0;
    }
    HD_SYNC();
  }

  // ---- G. ReID of inactive tracks with the remaining detections (tracker.py:166-264)
  if (tid == 0) {
    int k = 0;
    for (int i = 0; i < sh.ni; ++i)
      if (ts_alive(S, sh.inact[i], a.inactive_patience)) sh.inact[k++] = sh.inact[i];
    sh.ni = k;
  }
  for (int i = tid; i < sh.nd; i += nt) dsel[i] = 1;                         // 1 = still free for a new track
  HD_SYNC();
  if (sh.ni > 0 && sh.nd > 0) {
    const int ni = sh.ni, nd = sh.nd;
    if (a.reid_greedy_matching) {
      for (int e = tid; e < ni * nd; e += nt) {
        const int r = e / nd, c = e % nd;
        const Box t = ts_load(S.pos, sh.inact[r]);
        const Box d = ts_row_box(a, nqy + dl[c]);
        const float dx = hd_fsub(ts_cx(t), ts_cx(d)), dy = hd_fsub(ts_cy(t), ts_cy(d));
        const float dist = hd_fadd(hd_fmul(dx, dx), hd_fmul(dy, dy));
        const float track_size = hd_fmul(hd_fsub(t.x1, t.x0), hd_fsub(t.y1, t.y0));
        const float item_size = hd_fmul(hd_fsub(d.x1, d.x0), hd_fsub(d.y1, d.y0));
        f_mat[e] = (dist > track_size || dist > item_size) ? 1e18f : dist;
      }
      HD_SYNC();
      if (tid == 0) {
        for (int r = 0; r < ni; ++r) {
          int best = 0;
          float bv = f_mat[r * nd];
          for (int c = 1; c < nd; ++c) {
            const float v = f_mat[r * nd + c];
            if (v < bv) { bv = v; best = c; }
          }
          rowmatch[r] = -1;
          if (bv < 1e16f) {
            for (int k = 0; k < ni; ++k) f_mat[k * nd + best] = 1e18f;
            rowmatch[r] = best;
          }
        }
      }
    } else {
      // F.pairwise_distance(track embedding, detection embedding): || x1 - x2 + 1e-6 ||_2
      for (int e = tid; e < ni * nd; e += nt) {
        const int r = e / nd, c = e % nd;
        const float* x1 = S.bank + size_t(sh.inact[r]) * a.hidden;
        const float* x2 = a.hs_embeds + size_t(nqy + dl[c]) * a.hidden;
        double acc = 0.0;
        for (int h = 0; h < a.hidden; ++h) {
          const float d = hd_fadd(hd_fsub(x1[h], x2[h]), 1e-6f);
          acc += double(d) * double(d);
        }
        f_mat[e] = float(sqrt(acc));
      }
      HD_SYNC();
      if (tid < 32) ts_lsa_warp(f_mat, nd, ni, nd, a.dscratch, lsa_i, rowmatch);
    }
    HD_SYNC();
    if (tid == 0) {
      int k = 0;
      for (int r = 0; r < ni; ++r) {
        const int c = rowmatch[r];
        const int row = sh.inact[r];
        bool revive = false;
        if (c >= 0) revive = a.reid_greedy_matching ? (0.0 <= a.reid_sim_threshold)
                                                     : (f_mat[r * nd + c] <= float(a.reid_sim_threshold));
        if (revive) {
          const int qi = nqy + dl[c];
          const Box b = ts_row_box(a, qi);
          S.count_inactive[row] = 0;
          ts_store(S.pos, row, b);
          ts_store(S.anchor, row, b);                                        // reset_last_pos
          S.score[row] = a.rows[size_t(qi) * 6];
          hs_src[row] = qi;
          dsel[c] = 0;
          sh.act[sh.na++] = row;
          ++sh.num_reids;
        } else {
          sh.inact[k++] = row;
        }
      }
      sh.ni = k;
    }
    HD_SYNC();
  }

  // ---- H. new tracks (tracker.py:470-492)
  if (tid == 0) {
    int created = 0;
    for (int c = 0; c < sh.nd; ++c) {
      if (!dsel[c]) continue;
      const int j = dl[c], row = nin + j, qi = nqy + j;
      const Box b = ts_row_box(a, qi);
      S.ids[row] = sh.track_num + created;
      ts_store(S.pos, row, b);
      ts_store(S.anchor, row, b);
      S.score[row] = a.rows[size_t(qi) * 6];
      S.obj_ind[row] = j;
      S.count_inactive[row] = 0;
      S.count_termination[row] = 0;
      hs_src[row] = qi;
      fresh[row] = 1;
      sh.act[sh.na++] = row;
      ++created;
    }
    sh.track_num += created;
  }
  HD_SYNC();

  // ---- I. NMS between new and established tracks (tracker.py:494-515)
  if (a.detection_nms_on && sh.na > 0)
    ts_nms(a, sh, sh.act, sh.na, a.detection_nms_thresh, true, fresh, f_sc, f_area, f_box, order, dead);

  // ---- J. results of this frame (tracker.py:533-545)
  const int nres = sh.na;
  for (int k = tid; k < nres; k += nt) {
    const int r = sh.act[k];
    Box b = ts_load(S.pos, r);
    if (!a.overflow_boxes) {
      const float w = float(a.img_w), h = float(a.img_h);
      b.x0 = ts_clampf(b.x0, 0.f, w); b.x1 = ts_clampf(b.x1, 0.f, w);
      b.y0 = ts_clampf(b.y0, 0.f, h); b.y1 = ts_clampf(b.y1, 0.f, h);
    }
    int32_t* o = a.result + 8 + 8 * k;
    float* of = reinterpret_cast<float*>(o);
    o[0] = S.ids[r];
    o[1] = S.obj_ind[r];
    of[2] = S.score[r];
    of[3] = b.x0; of[4] = b.y0; of[5] = b.x1; of[6] = b.y1;
    o[7] = hs_src[r];                     // query row of this frame's embedding (and mask), or -1
  }
  HD_SYNC();
  if (tid == 0) {
    for (int i = 0; i < sh.ni; ++i) S.count_inactive[sh.inact[i]] += 1;     // tracker.py:541-542
    if (a.reid_sim_only) {                                                  // tracker.py:547-548
      for (int k = 0; k < sh.na; ++k) {
        const int r = sh.act[k];
        ts_store(S.pos, r, ts_load(S.anchor, r));
        sh.inact[sh.ni++] = r;
      }
      sh.na = 0;
    }
    // queries of the next frame: active tracks, then the inactive ones the next step's pruning keeps
    int m = 0;
    for (int k = 0; k < sh.na; ++k) sh.tmp[m++] = sh.act[k];
    for (int i = 0; i < sh.ni; ++i)
      if (ts_alive(S, sh.inact[i], a.inactive_patience)) sh.tmp[m++] = sh.inact[i];
    sh.nquery_next = m;
    const int hdr[8] = {sh.na, sh.ni, sh.track_num, sh.num_reids, m, 0, nres, 0};
    for (int k = 0; k < 8; ++k) { a.out.header[k] = hdr[k]; a.result[k] = hdr[k]; }
  }
  HD_SYNC();

  // ---- K. new state in list order, embeddings of this frame scattered into the bank, next frame's queries
  const int na = sh.na, nall = sh.na + sh.ni, hid = a.hidden;
  const TfbTrackState& O = a.out;
  for (int e = tid; e < nall; e += nt) {
    const int r = e < na ? sh.act[e] : sh.inact[e - na];
    O.ids[e] = S.ids[r];
    ts_store(O.pos, e, ts_load(S.pos, r));
    ts_store(O.anchor, e, ts_load(S.anchor, r));
    O.score[e] = S.score[r];
    O.obj_ind[e] = S.obj_ind[r];
    O.count_inactive[e] = S.count_inactive[r];
    O.count_termination[e] = S.count_termination[r];
  }
  for (int e = tid; e < nall * hid; e += nt) {
    const int k = e / hid, h = e % hid;
    const int r = k < na ? sh.act[k] : sh.inact[k - na];
    const int src = hs_src[r];
    O.bank[e] = src >= 0 ? a.hs_embeds[size_t(src) * hid + h] : S.bank[size_t(r) * hid + h];
  }
  const int nnext = sh.nquery_next;
  const float fw = float(a.img_w), fh = float(a.img_h);
  for (int k = tid; k < nnext; k += nt) {
    const Box b = ts_load(S.pos, sh.tmp[k]);
    a.q_boxes[4 * k] = hd_fdiv(ts_cx(b), fw);
    a.q_boxes[4 * k + 1] = hd_fdiv(ts_cy(b), fh);
    a.q_boxes[4 * k + 2] = hd_fdiv(hd_fsub(b.x1, b.x0), fw);
    a.q_boxes[4 * k + 3] = hd_fdiv(hd_fsub(b.y1, b.y0), fh);
  }
  for (int e = tid; e < nnext * hid; e += nt) {
    const int k = e / hid, h = e % hid;
    const int r = sh.tmp[k];
    const int src = hs_src[r];
    a.q_embeds[e] = src >= 0 ? a.hs_embeds[size_t(src) * hid + h] : S.bank[size_t(r) * hid + h];
  }
}

}  // namespace tfb200_track
