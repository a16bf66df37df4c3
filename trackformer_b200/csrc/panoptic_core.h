// Panoptic segmentation: the reference's PostProcessPanoptic (src/trackformer/models/detr_segmentation.py:256-388)
// and panopticapi's pq_compute, written once as cooperative routines:
//
//   pp_classes  (one thread per query row)        fp32 softmax over the class logits: first maximal class and its
//                                                 probability (the host derives the kept queries from them)
//   pp_label    (one CTA per image x pixel block) per processed pixel: bilinear sample of every surviving kept query's
//                                                 padded stride-4 logits, first query of maximal fp32 softmax, the
//                                                 stuff representative on a dedup pass; writes the processed-size
//                                                 label map and adds rows_mapped(y) * cols_mapped(x) -- the pixel's
//                                                 weight under Pillow's nearest resize -- to its label's target area
//   pp_final    (one CTA per image x pixel block) the int32 target-size map: survivor position of the nearest source
//   pq_count    (one CTA per image x pixel block) raw 24-bit ids -> dense segment index (sorted per-image id tables),
//                                                 integer (GT class) x (prediction class) intersection counts
//   pq_match    (one CTA per image)               panopticapi's match / FN / FP rules -> per-(image, category) tp, fp,
//                                                 fn and the fp64 IoU sum in ascending GT id order; error records
//   pq_reduce   (one thread per category)         sum of the per-image records over images in the given order
//
// nvcc compiles them into csrc/panoptic.cu's kernels, g++ (one "thread") into the test-only host build
// tests/host_build/panoptic_host.cpp (-ffp-contract=off).  Counts are integers and every floating-point sum runs in a
// fixed order, so results repeat bit for bit.
#pragma once

#include <limits.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "host_device.h"
#include "interp_index.h"

namespace tfb200_panoptic {

using tfb200_interp::Lin;
using tfb200_interp::bilinear_at;
using tfb200_interp::linear_src;

constexpr int kThreads = 256;
constexpr int kBlockPixels = 4096;                     // pixels of one CTA of the pixel passes
constexpr int kMaxKept = TFB200_PANOPTIC_MAX_KEPT;     // kept queries of one image
constexpr int kMaxSeg = TFB200_PANOPTIC_MAX_SEGMENTS;  // listed segments of one image, per side
constexpr int kMaxCat = TFB200_PANOPTIC_MAX_CATEGORIES;
constexpr int kSharedCells = 8192;                     // intersection cells counted in shared memory

// ---- post-processing -------------------------------------------------------------------------------------------
// per-image row of the geometry table (int64 [B][kPpFields], built on the host)
enum {
  kPpH, kPpW,            // processed size
  kPpHt, kPpWt,          // target size
  kPpKeptOff, kPpK,      // kept queries: rows kept_off .. kept_off + K of the kept tables
  kPpMapOff,             // processed label map: [H][W] at map_off
  kPpRowOff, kPpColOff,  // Pillow nearest source of each target row / column: [Ht] / [Wt] at row_off / col_off
  kPpRcntOff, kPpCcntOff,// number of target rows / columns mapped to each processed row / column: [H] / [W]
  kPpOutOff,             // target-size map: [Ht][Wt] at out_off
  kPpActive, kPpDedup,   // this round labels the image; stuff duplicates take their first kept query
  kPpFields
};

struct PpParams {
  int B, Q, C, h, w;                 // batch, queries, classes (last = no object), stride-4 mask size
  float threshold;
  const float* logits;               // [B][Q][C]
  const float* masks;                // [B][Q][h][w]
  const int64_t* img;                // [B][kPpFields]
  int32_t* cls;                      // [B * Q] out: first maximal class
  float* score;                      // [B * Q] out: its probability
  uint8_t* keep;                     // [B * Q] out
  const int32_t* kept_q;             // [kept] query index
  const int32_t* kept_alive;         // [kept] 1: survives the small-segment filter so far
  const int32_t* kept_rep;           // [kept] stuff representative (kept index) on a dedup pass
  const int32_t* kept_pos;           // [kept] position among the survivors
  const int32_t* idx;                // Pillow row / column sources and mapped counts
  int32_t* map;                      // processed label maps (kept index)
  unsigned long long* area;          // [kept] target-size area of each kept query
  int32_t* out;                      // target-size maps (survivor position)
};

HD_FN void pp_classes(const PpParams& p, int64_t row) {
  if (row >= int64_t(p.B) * p.Q) return;
  const float* x = p.logits + row * p.C;
  float m = x[0];
  for (int c = 1; c < p.C; ++c) m = x[c] > m ? x[c] : m;
  float s = 0.f;
  for (int c = 0; c < p.C; ++c) s = hd_fadd(s, expf(hd_fsub(x[c], m)));
  float best = -1.f;
  int arg = 0;
  for (int c = 0; c < p.C; ++c) {
    const float v = hd_fdiv(expf(hd_fsub(x[c], m)), s);
    if (v > best) { best = v; arg = c; }
  }
  p.cls[row] = arg;
  p.score[row] = best;
  p.keep[row] = uint8_t(arg != p.C - 1 && best > p.threshold);
}

// one CTA: pixels blk * kBlockPixels .. of image b; hist has kMaxKept entries (shared memory on the device)
HD_FN void pp_label(const PpParams& p, int b, int blk, unsigned long long* hist) {
  const int64_t* g = p.img + int64_t(b) * kPpFields;
  const int H = int(g[kPpH]), W = int(g[kPpW]), K = int(g[kPpK]);
  const int64_t npix = int64_t(H) * W, first = int64_t(blk) * kBlockPixels;
  if (!g[kPpActive] || first >= npix) return;
  const int64_t ko = g[kPpKeptOff];
  const int32_t* q = p.kept_q + ko;
  const int32_t* alive = p.kept_alive + ko;
  const int32_t* rep = p.kept_rep + ko;
  const int32_t* rcnt = p.idx + g[kPpRcntOff];
  const int32_t* ccnt = p.idx + g[kPpCcntOff];
  int32_t* map = p.map + g[kPpMapOff];
  const bool dedup = g[kPpDedup] != 0;
  const int64_t plane = int64_t(p.h) * p.w;
  const float* mb = p.masks + int64_t(b) * p.Q * plane;
  for (int k = HD_TID; k < K; k += HD_NT) hist[k] = 0ull;
  HD_SYNC();
  const int64_t last = first + kBlockPixels < npix ? first + kBlockPixels : npix;
  for (int64_t i = first + HD_TID; i < last; i += HD_NT) {
    const int y = int(i / W), x = int(i - int64_t(y) * W);
    const Lin ly = linear_src(y, p.h, H), lx = linear_src(x, p.w, W);
    // max and its first position, then the sum of expf(x - max), then the ties of the rounded probabilities
    float m = -INFINITY;
    int arg = -1;
    for (int k = 0; k < K; ++k) {
      if (!alive[k]) continue;
      const float v = bilinear_at(mb + q[k] * plane, p.w, ly, lx);
      if (arg < 0 || v > m) { m = v; arg = k; }
    }
    if (arg < 0) continue;                               // no survivor: the host leaves the image inactive
    float s = 0.f;
    int cand = arg;
    for (int k = 0; k < K; ++k) {
      if (!alive[k]) continue;
      const float e = expf(hd_fsub(bilinear_at(mb + q[k] * plane, p.w, ly, lx), m));
      s = hd_fadd(s, e);
      if (k < cand && e > 0.99999f) cand = k;           // p_k can round equal to 1 / s only if e_k > 1 - 2^-20
    }
    const float top = hd_fdiv(1.f, s);
    for (int k = cand; k < arg; ++k) {
      if (!alive[k]) continue;
      const float e = expf(hd_fsub(bilinear_at(mb + q[k] * plane, p.w, ly, lx), m));
      if (hd_fdiv(e, s) == top) { arg = k; break; }
    }
    const int lab = dedup ? rep[arg] : arg;
    map[i] = lab;
    const unsigned long long wgt = (unsigned long long)rcnt[y] * (unsigned long long)ccnt[x];
    if (wgt) hd_atomic_add(hist + lab, wgt);
  }
  HD_SYNC();
  for (int k = HD_TID; k < K; k += HD_NT)
    if (hist[k]) hd_atomic_add(p.area + ko + k, hist[k]);
}

HD_FN void pp_final(const PpParams& p, int b, int blk) {
  const int64_t* g = p.img + int64_t(b) * kPpFields;
  const int W = int(g[kPpW]), Ht = int(g[kPpHt]), Wt = int(g[kPpWt]), K = int(g[kPpK]);
  const int64_t npix = int64_t(Ht) * Wt, first = int64_t(blk) * kBlockPixels;
  if (first >= npix) return;
  const int64_t ko = g[kPpKeptOff];
  int any = 0;
  for (int k = 0; k < K; ++k) any |= p.kept_alive[ko + k];
  const int32_t* rows = p.idx + g[kPpRowOff];
  const int32_t* cols = p.idx + g[kPpColOff];
  const int32_t* map = p.map + g[kPpMapOff];
  int32_t* out = p.out + g[kPpOutOff];
  const int64_t last = first + kBlockPixels < npix ? first + kBlockPixels : npix;
  for (int64_t i = first + HD_TID; i < last; i += HD_NT) {
    const int y = int(i / Wt), x = int(i - int64_t(y) * Wt);
    out[i] = any ? p.kept_pos[ko + map[int64_t(rows[y]) * W + cols[x]]] : 0;
  }
}

// ---- PQ ----------------------------------------------------------------------------------------------------------
// per-image row of the update table (int64 [B][kPqFields])
enum {
  kPqPix,                // pixels
  kPqGtMap, kPqPredMap,  // element offsets of the raw-id maps (int32)
  kPqGtOff, kPqG,        // GT segments: sorted ids, category index, crowd, JSON area, JSON position at gt_off
  kPqVoidRow,            // dense GT row of raw id 0 (G when 0 is not listed)
  kPqPredOff, kPqP,      // prediction segments: sorted ids and category index at pred_off
  kPqCellOff,            // intersection counts [G + 2][P + 1] at cell_off
  kPqStatRow,            // row of the per-image records
  kPqFields
};
// error record of an image (int64 [3]): smallest id in the prediction PNG but not its JSON (or LLONG_MAX); smallest id
// present with an unknown category (or LLONG_MAX); number of JSON ids absent from the PNG
enum { kErrUnlisted, kErrCategory, kErrMissing, kErrFields };

struct PqParams {
  int B, Kc;
  const int64_t* img;                // [B][kPqFields]
  const int32_t* maps;               // raw 24-bit ids (both sides)
  const int32_t* gt_id;              // sorted per image
  const int32_t* gt_cat;             // category index (-1: not among the categories)
  const int32_t* gt_crowd;
  const double* gt_area;             // the JSON area
  const int32_t* gt_json;            // position in the image's segments_info
  const int32_t* pred_id;            // sorted per image
  const int32_t* pred_cat;           // category index (-1: unknown)
  int* cells;                        // intersection counts
  int64_t* pred_area;                // [pred rows] out: pixel count of each listed prediction segment
  int32_t* stat_i;                   // [rows][Kc][3] out: tp, fp, fn
  double* stat_iou;                  // [rows][Kc] out
  long long* err;                    // [rows][kErrFields] out
};

HD_FN int pq_find(const int32_t* ids, int n, int32_t v) {
  int lo = 0, hi = n;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (ids[mid] < v) lo = mid + 1; else hi = mid;
  }
  return lo < n && ids[lo] == v ? lo : -1;
}

// one CTA: pixels blk * kBlockPixels .. of image b; sh has kSharedCells entries (shared memory on the device)
HD_FN void pq_count(const PqParams& p, int b, int blk, int* sh) {
  const int64_t* g = p.img + int64_t(b) * kPqFields;
  const int64_t npix = g[kPqPix], first = int64_t(blk) * kBlockPixels;
  if (first >= npix) return;
  const int G = int(g[kPqG]), P = int(g[kPqP]), void_row = int(g[kPqVoidRow]);
  const int ncell = (G + 2) * (P + 1);
  const bool in_sh = ncell <= kSharedCells;
  int* cells = p.cells + g[kPqCellOff];
  int* acc = in_sh ? sh : cells;
  const int32_t* gid = p.gt_id + g[kPqGtOff];
  const int32_t* pid = p.pred_id + g[kPqPredOff];
  const int32_t* gm = p.maps + g[kPqGtMap];
  const int32_t* pm = p.maps + g[kPqPredMap];
  long long* err = p.err + g[kPqStatRow] * kErrFields;
  if (in_sh) {
    for (int c = HD_TID; c < ncell; c += HD_NT) sh[c] = 0;
    HD_SYNC();
  }
  const int64_t last = first + kBlockPixels < npix ? first + kBlockPixels : npix;
  for (int64_t i = first + HD_TID; i < last; i += HD_NT) {
    const int32_t gv = gm[i], pv = pm[i];
    int gr = pq_find(gid, G, gv);
    if (gr < 0) gr = gv == 0 ? void_row : G + 1;        // VOID, or an id the JSON does not list
    int pc = pq_find(pid, P, pv);
    if (pc < 0) {
      if (pv != 0) { hd_atomic_min(err + kErrUnlisted, (long long)pv); continue; }
      pc = P;                                            // VOID
    }
    hd_atomic_add(acc + gr * (P + 1) + pc, 1);
  }
  if (in_sh) {
    HD_SYNC();
    for (int c = HD_TID; c < ncell; c += HD_NT)
      if (sh[c]) hd_atomic_add(cells + c, sh[c]);
  }
}

struct MatchShared {
  int match[kMaxSeg];                // GT segment -> matched prediction, or -1
  double iou[kMaxSeg];
  int pmatched[kMaxSeg];
  int crowd_of[kMaxCat];             // category -> crowd GT segment (last in JSON order), or -1
};

HD_FN void pq_match(const PqParams& p, int b, MatchShared& sh) {
  const int64_t* g = p.img + int64_t(b) * kPqFields;
  const int G = int(g[kPqG]), P = int(g[kPqP]), void_row = int(g[kPqVoidRow]);
  const int64_t go = g[kPqGtOff], po = g[kPqPredOff], row = g[kPqStatRow];
  const int* cells = p.cells + g[kPqCellOff];
  const int32_t* gcat = p.gt_cat + go;
  const int32_t* gcrowd = p.gt_crowd + go;
  const double* garea = p.gt_area + go;
  const int32_t* gjson = p.gt_json + go;
  const int32_t* pid = p.pred_id + po;
  const int32_t* pcat = p.pred_cat + po;
  int64_t* parea = p.pred_area + po;
  long long* err = p.err + row * kErrFields;
  int32_t* st = p.stat_i + row * p.Kc * 3;
  double* siou = p.stat_iou + row * p.Kc;
  const int stride = P + 1;
  for (int k = HD_TID; k < p.Kc; k += HD_NT) {
    st[3 * k] = st[3 * k + 1] = st[3 * k + 2] = 0;
    siou[k] = 0.0;
    sh.crowd_of[k] = -1;
  }
  for (int j = HD_TID; j < P; j += HD_NT) {
    int64_t a = 0;
    for (int r = 0; r < G + 2; ++r) a += cells[r * stride + j];
    parea[j] = a;
    sh.pmatched[j] = 0;
  }
  HD_SYNC();
  if (HD_TID == 0) {                                     // the image's errors, as panopticapi meets them
    long long cat_err = LLONG_MAX, missing = 0;
    for (int j = 0; j < P; ++j) {
      if (parea[j] == 0) ++missing;
      else if (pcat[j] < 0 && pid[j] < cat_err) cat_err = pid[j];
    }
    err[kErrCategory] = cat_err;
    err[kErrMissing] = missing;
  }
  for (int r = HD_TID; r < G; r += HD_NT) {
    sh.match[r] = -1;
    sh.iou[r] = 0.0;
    if (gcrowd[r]) continue;
    const int64_t void_inter_row = int64_t(void_row) * stride;
    for (int j = 0; j < P; ++j) {
      const int inter = cells[r * stride + j];
      if (inter == 0 || pcat[j] != gcat[r]) continue;
      const double uni = hd_dsub(hd_dsub(hd_dadd(double(parea[j]), garea[r]), double(inter)),
                                 double(cells[void_inter_row + j]));
      const double iou = hd_ddiv(double(inter), uni);
      if (iou > 0.5) { sh.match[r] = j; sh.iou[r] = iou; }
    }
  }
  HD_SYNC();
  if (HD_TID == 0) {
    for (int r = 0; r < G; ++r) {                        // ascending GT id: the order of np.unique's pair keys
      const int c = gcat[r];
      if (sh.match[r] >= 0) {
        sh.pmatched[sh.match[r]] = 1;
        if (c >= 0) { st[3 * c] += 1; siou[c] = hd_dadd(siou[c], sh.iou[r]); }
      } else if (gcrowd[r]) {
        if (c >= 0 && (sh.crowd_of[c] < 0 || gjson[sh.crowd_of[c]] < gjson[r])) sh.crowd_of[c] = r;
      } else if (c >= 0) {
        st[3 * c + 2] += 1;
      }
    }
    for (int j = 0; j < P; ++j) {
      const int c = pcat[j];
      if (sh.pmatched[j] || c < 0 || parea[j] == 0) continue;
      int64_t inter = cells[int64_t(void_row) * stride + j];
      if (sh.crowd_of[c] >= 0) inter += cells[int64_t(sh.crowd_of[c]) * stride + j];
      if (hd_ddiv(double(inter), double(parea[j])) > 0.5) continue;
      st[3 * c + 1] += 1;
    }
  }
}

// category k: sums over the records rows[0 .. n) in that order; out [Kc][4] tp, fp, fn, iou.  err_out[0] is the first
// i whose record has an error (or n)
HD_FN void pq_reduce(const int32_t* stat_i, const double* stat_iou, const long long* err, const int64_t* rows,
                     int64_t n, int Kc, int k, double* out, int64_t* err_out) {
  if (k < Kc) {
    int64_t tp = 0, fp = 0, fn = 0;
    double iou = 0.0;
    for (int64_t i = 0; i < n; ++i) {
      const int64_t r = rows[i];
      tp += stat_i[(r * Kc + k) * 3];
      fp += stat_i[(r * Kc + k) * 3 + 1];
      fn += stat_i[(r * Kc + k) * 3 + 2];
      iou = hd_dadd(iou, stat_iou[r * Kc + k]);
    }
    out[4 * k] = double(tp);
    out[4 * k + 1] = double(fp);
    out[4 * k + 2] = double(fn);
    out[4 * k + 3] = iou;
  } else if (k == Kc) {
    int64_t first = n;
    for (int64_t i = 0; i < n; ++i) {
      const long long* e = err + rows[i] * kErrFields;
      if (e[kErrUnlisted] != LLONG_MAX || e[kErrCategory] != LLONG_MAX || e[kErrMissing] != 0) { first = i; break; }
    }
    err_out[0] = first;
  }
}

}  // namespace tfb200_panoptic
