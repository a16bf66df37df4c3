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
// host build that tests/test_track_step_cpu.py replays the reference-recorded sequences through.  The TS_* macros are
// the only difference between the two.
#pragma once

#include <float.h>
#include <math.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"

#if defined(__CUDACC__)
#define TS_FN __device__ inline
#define TS_SYNC() __syncthreads()
#define TS_SYNCWARP() __syncwarp()
#define TS_TID (int(threadIdx.x))
#define TS_NT (int(blockDim.x))
#define TS_LANE (int(threadIdx.x) & 31)
#define TS_NLANES 32
#define ts_mul(a, b) __fmul_rn((a), (b))
#define ts_add(a, b) __fadd_rn((a), (b))
#define ts_sub(a, b) __fsub_rn((a), (b))
#define ts_div(a, b) __fdiv_rn((a), (b))
#else
#define TS_FN static inline
#define TS_SYNC() ((void)0)
#define TS_SYNCWARP() ((void)0)
#define TS_TID 0
#define TS_NT 1
#define TS_LANE 0
#define TS_NLANES 1
#define ts_mul(a, b) ((a) * (b))        // the host build is compiled with -ffp-contract=off
#define ts_add(a, b) ((a) + (b))
#define ts_sub(a, b) ((a) - (b))
#define ts_div(a, b) ((a) / (b))
#endif

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

TS_FN float ts_clampf(float v, float lo, float hi) { return v < lo ? lo : (v > hi ? hi : v); }

// boxes[i] of this frame: the detector's pixel box, clipped to the image unless the model allows overflow
// (tracker.py:323-327, torchvision clip_boxes_to_image)
TS_FN Box ts_row_box(const TfbTrackStepArgs& a, int i) {
  const float* r = a.rows + size_t(i) * 6;
  Box b{r[2], r[3], r[4], r[5]};
  if (!a.overflow_boxes) {
    const float w = float(a.img_w), h = float(a.img_h);
    b.x0 = ts_clampf(b.x0, 0.f, w); b.x1 = ts_clampf(b.x1, 0.f, w);
    b.y0 = ts_clampf(b.y0, 0.f, h); b.y1 = ts_clampf(b.y1, 0.f, h);
  }
  return b;
}
TS_FN Box ts_load(const float* p, int r) { return Box{p[4 * r], p[4 * r + 1], p[4 * r + 2], p[4 * r + 3]}; }
TS_FN void ts_store(float* p, int r, const Box& b) { p[4 * r] = b.x0; p[4 * r + 1] = b.y0; p[4 * r + 2] = b.x1; p[4 * r + 3] = b.y1; }
TS_FN float ts_area(const Box& b) { return ts_mul(ts_sub(b.x1, b.x0), ts_sub(b.y1, b.y0)); }
TS_FN float ts_cx(const Box& b) { return ts_mul(ts_add(b.x0, b.x1), 0.5f); }     // (x0 + x1) / 2, exact either way
TS_FN float ts_cy(const Box& b) { return ts_mul(ts_add(b.y0, b.y1), 0.5f); }

// torchvision box_iou / nms arithmetic: inter / (area_a + area_b - inter)
TS_FN float ts_iou(const Box& a, float area_a, const Box& b, float area_b) {
  float w = ts_sub(fminf(a.x1, b.x1), fmaxf(a.x0, b.x0));
  float h = ts_sub(fminf(a.y1, b.y1), fmaxf(a.y0, b.y0));
  w = w < 0.f ? 0.f : w;
  h = h < 0.f ? 0.f : h;
  const float inter = ts_mul(w, h);
  return ts_div(inter, ts_sub(ts_add(area_a, area_b), inter));
}

// has_positive_area and within the patience window (tracker.py:171-174, 270-273)
TS_FN bool ts_alive(const TfbTrackState& s, int r, double patience) {
  const Box b = ts_load(s.pos, r);
  return b.x1 > b.x0 && b.y1 > b.y0 && double(s.count_inactive[r]) <= patience;
}

// ------------------------------------------------------------------------------------------------------------ NMS
// Greedy NMS over list[0..n) (torchvision.ops.nms semantics: descending score, stable; suppress IoU > thr), scores of
// rows that are not `fresh` replaced by +inf when fresh_only (tracker.py:503).  Survivors stay in list order; returns
// through sh.tmp / *n_out (thread 0).  Whole CTA.
TS_FN void ts_nms(const TfbTrackStepArgs& a, Shared& sh, int* list, int& n_ref, float thr, bool fresh_only, const int* fresh,
                  float* f_sc, float* f_area, float* f_box, int* order, int* dead) {
  const int n = n_ref;
  const TfbTrackState& S = a.in;
  for (int k = TS_TID; k < n; k += TS_NT) {
    const int r = list[k];
    const Box b = ts_load(S.pos, r);
    ts_store(f_box, k, b);
    f_area[k] = ts_area(b);
    f_sc[k] = (fresh_only && !fresh[r]) ? INFINITY : S.score[r];
    dead[k] = 0;
  }
  TS_SYNC();
  for (int k = TS_TID; k < n; k += TS_NT) {
    const float s = f_sc[k];
    int rank = 0;
    for (int m = 0; m < n; ++m) {
      const float t = f_sc[m];
      rank += (t > s) || (t == s && m < k);
    }
    order[rank] = k;
  }
  TS_SYNC();
  for (int p = 0; p < n; ++p) {
    const int i = order[p];
    if (dead[i]) continue;                                   // uniform: written before the last barrier
    const Box bi = ts_load(f_box, i);
    const float ai = f_area[i];
    for (int q = p + 1 + TS_TID; q < n; q += TS_NT) {
      const int j = order[q];
      if (dead[j]) continue;
      if (ts_iou(bi, ai, ts_load(f_box, j), f_area[j]) > thr) dead[j] = 1;
    }
    TS_SYNC();
  }
  TS_SYNC();
  if (TS_TID == 0) {
    int m = 0;
    for (int k = 0; k < n; ++k)
      if (!dead[k]) list[m++] = list[k];
    n_ref = m;
  }
  TS_SYNC();
}

// --------------------------------------------------------------------------------------- rectangular assignment
struct MinKey { double val; int tie; int idx; };
TS_FN bool ts_better(const MinKey& x, const MinKey& y) {
  if (x.val != y.val) return x.val < y.val;
  if (x.tie != y.tie) return x.tie < y.tie;
  return x.idx < y.idx;
}
TS_FN MinKey ts_warp_min(MinKey k) {
#if defined(__CUDACC__)
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    MinKey other;
    other.val = __shfl_xor_sync(0xffffffffu, k.val, o);
    other.tie = __shfl_xor_sync(0xffffffffu, k.tie, o);
    other.idx = __shfl_xor_sync(0xffffffffu, k.idx, o);
    if (ts_better(other, k)) k = other;
  }
#endif
  return k;
}

// scipy.optimize.linear_sum_assignment of dist[nr0][ld] (nc0 columns used) by shortest augmenting paths with duals in
// double precision; run by ONE warp.  rowmatch[r] = column assigned to row r, or -1 (only when nr0 > nc0).
TS_FN void ts_lsa_warp(const float* dist, int ld, int nr0, int nc0, double* dws, int* iws, int* rowmatch) {
  const bool transposed = nr0 > nc0;
  const int nr = transposed ? nc0 : nr0, nc = transposed ? nr0 : nc0;
  double* shortest = dws;
  double* v = shortest + nc;
  double* u = v + nc;
  int* path = iws;
  int* row4col = path + nc;
  int* in_sc = row4col + nc;
  int* col4row = in_sc + nc;
  int* visited = col4row + nr;
  const int lane = TS_LANE;
  for (int j = lane; j < nc; j += TS_NLANES) { v[j] = 0.0; row4col[j] = -1; }
  for (int i = lane; i < nr; i += TS_NLANES) { u[i] = 0.0; col4row[i] = -1; }
  for (int r = lane; r < nr0; r += TS_NLANES) rowmatch[r] = -1;
  TS_SYNCWARP();
  bool fail = false;
  for (int cur = 0; cur < nr && !fail; ++cur) {
    for (int j = lane; j < nc; j += TS_NLANES) { shortest[j] = DBL_MAX; path[j] = -1; in_sc[j] = 0; }
    TS_SYNCWARP();
    int i = cur, sink = -1, nvis = 0;
    double min_val = 0.0;
    while (sink == -1) {
      if (lane == 0) visited[nvis] = i;
      ++nvis;
      const double ui = u[i];
      MinKey best{DBL_MAX, 1, INT32_MAX};
      for (int j = lane; j < nc; j += TS_NLANES) {
        if (in_sc[j]) continue;
        const double c = double(transposed ? dist[size_t(j) * ld + i] : dist[size_t(i) * ld + j]);
        const double r = min_val + c - ui - v[j];
        if (r < shortest[j]) { shortest[j] = r; path[j] = i; }
        const MinKey cand{shortest[j], row4col[j] == -1 ? 0 : 1, j};
        if (ts_better(cand, best)) best = cand;
      }
      best = ts_warp_min(best);
      if (best.idx == INT32_MAX || best.val == DBL_MAX) { fail = true; break; }     // non-finite costs
      min_val = best.val;
      if (lane == 0) in_sc[best.idx] = 1;
      TS_SYNCWARP();
      if (row4col[best.idx] == -1) sink = best.idx;
      else i = row4col[best.idx];
    }
    if (fail) break;
    for (int t = lane; t < nvis; t += TS_NLANES) {
      const int r = visited[t];
      if (r == cur) u[r] += min_val;
      else u[r] += min_val - shortest[col4row[r]];
    }
    for (int j = lane; j < nc; j += TS_NLANES)
      if (in_sc[j]) v[j] -= min_val - shortest[j];
    TS_SYNCWARP();
    if (lane == 0) {
      int j = sink;
      while (true) {
        const int r = path[j];
        row4col[j] = r;
        const int prev = col4row[r];
        col4row[r] = j;
        j = prev;
        if (r == cur) break;
      }
    }
    TS_SYNCWARP();
  }
  if (!fail) {
    for (int r = lane; r < nr; r += TS_NLANES) {
      if (transposed) rowmatch[col4row[r]] = r;
      else rowmatch[r] = col4row[r];
    }
  }
  TS_SYNCWARP();
}

// ---------------------------------------------------------------------------------------------------- the step
TS_FN void ts_step(const TfbTrackStepArgs& a, Shared& sh) {
  const int tid = TS_TID, nt = TS_NT;
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
  TS_SYNC();
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
  TS_SYNC();

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
    TS_SYNC();
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
    TS_SYNC();
    if (a.track_nms_on && sh.na > 0)
      ts_nms(a, sh, sh.act, sh.na, a.track_nms_thresh, false, fresh, f_sc, f_area, f_box, order, dead);
  }

  // ---- E. new detections (tracker.py:408-436)
  for (int j = tid; j < nq; j += nt) {
    const float* r = a.rows + size_t(nqy + j) * 6;
    sh.flag[j] = r[0] > a.detection_obj_score_thresh && r[1] == 0.f;
  }
  TS_SYNC();
  if (tid == 0) {
    int nd = 0;
    for (int j = 0; j < nq; ++j)
      if (sh.flag[j]) dl[nd++] = j;
    sh.nd = nd;
  }
  TS_SYNC();

  // ---- F. public-detection gating (tracker.py:122-164)
  if (a.public_mode != 0) {
    const int nd = sh.nd, np = a.public_dets ? a.n_public : 0;
    TS_SYNC();                                  // every thread has read sh.nd before thread 0 rewrites it below
    if (nd > 0 && np > 0) {
      for (int e = tid; e < nd * np; e += nt) {
        const int i = e / np, j = e % np;
        const Box b = ts_row_box(a, nqy + dl[i]);
        const Box p = ts_load(a.public_dets, j);
        float m;
        if (a.public_mode == 1) {
          const float dx = ts_sub(ts_cx(b), ts_cx(p)), dy = ts_sub(ts_cy(b), ts_cy(p));
          m = ts_add(ts_mul(dx, dx), ts_mul(dy, dy));
        } else {
          m = ts_iou(b, ts_area(b), p, ts_area(p));
        }
        f_mat[e] = m;
      }
      for (int i = tid; i < nd; i += nt) dsel[i] = 0;
      TS_SYNC();
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
    TS_SYNC();
  }

  // ---- G. ReID of inactive tracks with the remaining detections (tracker.py:166-264)
  if (tid == 0) {
    int k = 0;
    for (int i = 0; i < sh.ni; ++i)
      if (ts_alive(S, sh.inact[i], a.inactive_patience)) sh.inact[k++] = sh.inact[i];
    sh.ni = k;
  }
  for (int i = tid; i < sh.nd; i += nt) dsel[i] = 1;                         // 1 = still free for a new track
  TS_SYNC();
  if (sh.ni > 0 && sh.nd > 0) {
    const int ni = sh.ni, nd = sh.nd;
    if (a.reid_greedy_matching) {
      for (int e = tid; e < ni * nd; e += nt) {
        const int r = e / nd, c = e % nd;
        const Box t = ts_load(S.pos, sh.inact[r]);
        const Box d = ts_row_box(a, nqy + dl[c]);
        const float dx = ts_sub(ts_cx(t), ts_cx(d)), dy = ts_sub(ts_cy(t), ts_cy(d));
        const float dist = ts_add(ts_mul(dx, dx), ts_mul(dy, dy));
        const float track_size = ts_mul(ts_sub(t.x1, t.x0), ts_sub(t.y1, t.y0));
        const float item_size = ts_mul(ts_sub(d.x1, d.x0), ts_sub(d.y1, d.y0));
        f_mat[e] = (dist > track_size || dist > item_size) ? 1e18f : dist;
      }
      TS_SYNC();
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
          const float d = ts_add(ts_sub(x1[h], x2[h]), 1e-6f);
          acc += double(d) * double(d);
        }
        f_mat[e] = float(sqrt(acc));
      }
      TS_SYNC();
      if (tid < 32) ts_lsa_warp(f_mat, nd, ni, nd, a.dscratch, lsa_i, rowmatch);
    }
    TS_SYNC();
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
    TS_SYNC();
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
  TS_SYNC();

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
  TS_SYNC();
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
  TS_SYNC();

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
    a.q_boxes[4 * k] = ts_div(ts_cx(b), fw);
    a.q_boxes[4 * k + 1] = ts_div(ts_cy(b), fh);
    a.q_boxes[4 * k + 2] = ts_div(ts_sub(b.x1, b.x0), fw);
    a.q_boxes[4 * k + 3] = ts_div(ts_sub(b.y1, b.y0), fh);
  }
  for (int e = tid; e < nnext * hid; e += nt) {
    const int k = e / hid, h = e % hid;
    const int r = sh.tmp[k];
    const int src = hs_src[r];
    a.q_embeds[e] = src >= 0 ? a.hs_embeds[size_t(src) * hid + h] : S.bank[size_t(r) * hid + h];
  }
}

}  // namespace tfb200_track
