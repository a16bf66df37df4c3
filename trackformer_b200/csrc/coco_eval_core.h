// COCO box / mask AP (what pycocotools 2.0's COCOeval computes for the reference's CocoEvaluator,
// src/trackformer/datasets/coco_eval.py), written once as cooperative routines:
//
//   ce_rank      (one CTA per image)            category index of each detection, its stable score rank within
//                                               (image, category), the sort key, and the detections ordered by
//                                               (category, rank); ranks >= max_det are not evaluated
//   ce_pack_dt   (one CTA per image x detection) segm: the mask (> 0.5) bit-packed, its pixel count and tight box
//   ce_decode_gt (one CTA per image x GT)        segm: the ground truth's runs of ones set into a bit plane
//   ce_iou       (one CTA per image x detection) fp64 IoU against the image's ground truths of the same category
//   ce_match     (one CTA per image)            evaluateImg: one thread per (category, area range, IoU threshold),
//                                               sequential over detections and ground truths; a 2-bit state per
//                                               (detection, area range, threshold)
//   ce_acc       (one CTA per category x area x maxDet x threshold)  accumulate over the score-sorted detections
//
// nvcc compiles them into csrc/coco_eval.cu's kernels, g++ (one "thread") into the test-only host build
// tests/host_build/coco_eval_host.cpp.  All IoU arithmetic is fp64 with separately rounded operations (no
// contraction; the host build is compiled with -ffp-contract=off), as pycocotools' C routines compute it.
//
// Bit planes are column-major like COCO RLE: word (wy, x) = bits[wy * W + x] holds rows 32 wy .. 32 wy + 31 of
// column x, bit i = row 32 wy + i.
#pragma once

#include <limits.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "host_device.h"

namespace tfb200_coco {

constexpr int kThreads = 256;
constexpr int kMaxDets = TFB200_COCO_MAX_DETS;       // detections of one image in one update
constexpr int kMaxGt = TFB200_COCO_MAX_GT;           // ground truths of one image x category
constexpr int kMaxThr = 16;                          // IoU thresholds (2 state bits each in a 32-bit word)
constexpr int kMaxArea = 8;                          // area ranges
constexpr int kMaxRec = 1024;                        // recall thresholds
constexpr int kMaxMaxDets = 8;                       // maxDets entries

// per-image row of the update table (int64 [B][kImgFields], built on the host)
enum { kGtImg, kDetBegin, kDetCount, kH, kW, kMaskPtr, kIouOff, kDbitsOff, kGbitsOff, kGtmOff, kImgFields };
// detection states (2 bits per IoU threshold)
enum { kFp = 0, kTp = 1, kIgnored = 2 };
// status bits of an update
enum { kErrScore = 1 };

struct MatchParams {
  int B, K, A, T, max_det, segm;
  const int64_t* img;                // [B][kImgFields]
  const float* boxes;                // [N][4] x0, y0, x1, y1 (box evaluation)
  const float* scores;               // [N]
  const int64_t* labels;             // [N]; category id = label + 1
  const int64_t* cat_ids;            // [K] ascending
  const int64_t* gt_off;             // [GT images + 1] annotation rows of each image, sorted by category index
  const int32_t* gt_k;               // category index
  const double* gt_box;              // [4] x, y, w, h
  const double* gt_area;             // the annotation's area
  const uint8_t* gt_crowd;
  const int64_t* gt_id;
  const int64_t* gt_run_off;         // segm: [annotations + 1] into gt_runs
  const uint32_t* gt_runs;           // segm: [runs][2] column-major start, length of each run of ones
  const int32_t* gt_bbox;            // segm: [4] x0, y0, x1, y1 inclusive tight box (x0 > x1: empty)
  const int64_t* gt_px;              // segm: pixel count
  const double* area_rng;            // [A][2]
  const double* iou_thr;             // [T] min(threshold, 1 - 1e-10)
  uint64_t* key;                     // [N] out: (category index << 32) | descending-score bits; K << 32: not evaluated
  int32_t* rank;                     // [N] out
  uint32_t* state;                   // [N][A] out
  int32_t* status;                   // [1] out, or-ed
  // workspace
  int32_t* dk;                       // [N] category index or -1
  int32_t* dord;                     // [N] per image: detections by (category, rank); -1 past the valid ones
  double* iou;                       // per image [n_det][n_gt]
  uint32_t* dbits;                   // segm: per image [n_det][plane]
  uint32_t* gbits;                   // segm: per image [n_gt][plane]
  int32_t* dbox;                     // segm: [N][4]
  int64_t* dpx;                      // segm: [N]
  uint8_t* gtm;                      // per image [A * T][n_gt] matched flags
};

struct AccParams {
  int K, A, T, R, M, n_kept;
  int64_t n_rec, n;                  // records over all updates; kept detections
  const uint64_t* key;               // [n_rec]
  const int32_t* rank;               // [n_rec]
  const uint32_t* state;             // [n_rec][A]
  const int64_t* kept;               // [n_kept][3] record begin, destination begin, count (image-id order)
  const int64_t* npig;               // [K][A]
  const double* rec_thr;             // [R]
  const int32_t* max_dets;           // [M]
  const int32_t* status_in;          // [1]
  double* precision;                 // [T][R][K][A][M]
  double* recall;                    // [T][K][A][M]
  double* scores;                    // [T][R][K][A][M]
  double* status_out;                // [1]
  // workspace
  uint64_t* key_in; uint64_t* key_out; int64_t* val_in; int64_t* val_out;
};

// ---- scores ----
// Ascending in the result = descending in the score; -0 and +0 tie.
HD_FN uint32_t ce_desc_bits(float s) {
  uint32_t u = hd_float_bits(s + 0.0f);
  u = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ~u;
}
HD_FN float ce_desc_score(uint32_t d) {
  uint32_t u = ~d;
  u = (u & 0x80000000u) ? (u & 0x7fffffffu) : ~u;
  return hd_bits_float(u);
}
HD_FN bool ce_finite(float s) { return (hd_float_bits(s) & 0x7f800000u) != 0x7f800000u; }

HD_FN int ce_cat_index(const int64_t* cat_ids, int K, int64_t cat) {
  int lo = 0, hi = K;
  while (lo < hi) {
    const int mid = (lo + hi) >> 1;
    if (cat_ids[mid] < cat) lo = mid + 1; else hi = mid;
  }
  return (lo < K && cat_ids[lo] == cat) ? lo : -1;
}

// The image's ground-truth rows [b, e) of category k (rows are sorted by category index).
HD_FN void ce_gt_range(const MatchParams& p, int64_t gi, int k, int64_t& b, int64_t& e) {
  int64_t lo = p.gt_off[gi], hi = p.gt_off[gi + 1];
  int64_t l = lo, h = hi;
  while (l < h) { const int64_t m = (l + h) >> 1; if (p.gt_k[m] < k) l = m + 1; else h = m; }
  b = l; h = hi;
  while (l < h) { const int64_t m = (l + h) >> 1; if (p.gt_k[m] <= k) l = m + 1; else h = m; }
  e = l;
}

// ---- pycocotools maskApi.c bbIou: [x, y, w, h] in fp64, separately rounded ----
HD_FN double ce_bb_iou(const double* d, const double* g, bool crowd) {
  const double da = hd_dmul(d[2], d[3]), ga = hd_dmul(g[2], g[3]);
  const double dx1 = hd_dadd(d[2], d[0]), gx1 = hd_dadd(g[2], g[0]);
  const double w = hd_dsub(dx1 < gx1 ? dx1 : gx1, d[0] > g[0] ? d[0] : g[0]);
  if (!(w > 0.0)) return 0.0;
  const double dy1 = hd_dadd(d[3], d[1]), gy1 = hd_dadd(g[3], g[1]);
  const double h = hd_dsub(dy1 < gy1 ? dy1 : gy1, d[1] > g[1] ? d[1] : g[1]);
  if (!(h > 0.0)) return 0.0;
  const double i = hd_dmul(w, h);
  const double u = crowd ? da : hd_dsub(hd_dadd(da, ga), i);
  return hd_ddiv(i, u);
}

// The detection box as convert_to_xywh makes it: w = x1 - x0 in float32, then widened.
HD_FN void ce_dt_xywh(const float* b, double* o) {
  o[0] = double(b[0]); o[1] = double(b[1]);
  o[2] = double(float(b[2] - b[0])); o[3] = double(float(b[3] - b[1]));
}

// ---- 1. category, rank, key, order (one CTA per image) ----
HD_FN void ce_rank(const MatchParams& p, int b) {
  const int64_t* im = p.img + int64_t(b) * kImgFields;
  const int64_t d0 = im[kDetBegin];
  const int n = int(im[kDetCount]);
  for (int j = HD_TID; j < n; j += HD_NT) {
    const float s = p.scores[d0 + j];
    int k = ce_cat_index(p.cat_ids, p.K, p.labels[d0 + j] + 1);
    if (!ce_finite(s)) {
      k = -1;
      hd_atomic_or(reinterpret_cast<uint32_t*>(p.status), kErrScore);
    }
    p.dk[d0 + j] = k;
    p.dord[d0 + j] = -1;
    for (int a = 0; a < p.A; ++a) p.state[(d0 + j) * p.A + a] = 0;
  }
  HD_SYNC();
  for (int j = HD_TID; j < n; j += HD_NT) {
    const int k = p.dk[d0 + j];
    int r = INT32_MAX;
    if (k >= 0) {
      const float s = p.scores[d0 + j] + 0.0f;
      int below = 0;
      r = 0;
      for (int i = 0; i < n; ++i) {
        const int ki = p.dk[d0 + i];
        if (ki < 0) continue;
        if (ki < k) ++below;
        else if (ki == k && i != j) {
          const float si = p.scores[d0 + i] + 0.0f;
          if (si > s || (si == s && i < j)) ++r;
        }
      }
      p.dord[d0 + below + r] = j;
    }
    p.rank[d0 + j] = r;
    p.key[d0 + j] = (k >= 0 && r < p.max_det) ? (uint64_t(k) << 32) | ce_desc_bits(p.scores[d0 + j])
                                              : uint64_t(p.K) << 32;
  }
}

HD_FN bool ce_evaluated(const MatchParams& p, int64_t row) { return (p.key[row] >> 32) < uint64_t(p.K); }

// ---- 2. segm: pack one detection's mask (one CTA per image x detection) ----
struct PackShared { long long px; int x0, y0, x1, y1; };

HD_FN void ce_pack_dt(const MatchParams& p, int b, int j, PackShared& sh) {
  const int64_t* im = p.img + int64_t(b) * kImgFields;
  if (j >= im[kDetCount]) return;
  const int64_t row = im[kDetBegin] + j;
  if (!ce_evaluated(p, row)) return;
  const int H = int(im[kH]), W = int(im[kW]), Hw = (H + 31) >> 5;
  const int64_t plane = int64_t(Hw) * W;
  const uint8_t* m = reinterpret_cast<const uint8_t*>(im[kMaskPtr]) + int64_t(j) * H * W;
  uint32_t* bits = p.dbits + im[kDbitsOff] + int64_t(j) * plane;
  if (HD_TID == 0) { sh.px = 0; sh.x0 = INT_MAX; sh.y0 = INT_MAX; sh.x1 = -1; sh.y1 = -1; }
  HD_SYNC();
  long long px = 0;
  int x0 = INT_MAX, y0 = INT_MAX, x1 = -1, y1 = -1;
  for (int64_t w = HD_TID; w < plane; w += HD_NT) {
    const int x = int(w % W), wy = int(w / W);
    const int rows = H - 32 * wy < 32 ? H - 32 * wy : 32;
    uint32_t v = 0;
    for (int i = 0; i < rows; ++i) v |= uint32_t(m[int64_t(32 * wy + i) * W + x] != 0) << i;
    bits[w] = v;
    if (v) {
      px += hd_popc(v);
      x0 = x < x0 ? x : x0; x1 = x > x1 ? x : x1;
      const int ya = 32 * wy + hd_ctz(v), yb = 32 * wy + 31 - hd_clz(v);
      y0 = ya < y0 ? ya : y0; y1 = yb > y1 ? yb : y1;
    }
  }
  hd_atomic_add(&sh.px, px);
  hd_atomic_min(&sh.x0, x0); hd_atomic_min(&sh.y0, y0); hd_atomic_max(&sh.x1, x1); hd_atomic_max(&sh.y1, y1);
  HD_SYNC();
  if (HD_TID == 0) {
    p.dpx[row] = sh.px;
    int32_t* bx = p.dbox + row * 4;
    bx[0] = sh.x0; bx[1] = sh.y0; bx[2] = sh.x1; bx[3] = sh.y1;
  }
}

// ---- 3. segm: one ground truth's runs into its bit plane (zeroed before; one CTA per image x GT) ----
HD_FN void ce_decode_gt(const MatchParams& p, int b, int g) {
  const int64_t* im = p.img + int64_t(b) * kImgFields;
  const int64_t gi = im[kGtImg], gb = p.gt_off[gi];
  if (g >= p.gt_off[gi + 1] - gb) return;
  const int64_t row = gb + g;
  const int H = int(im[kH]), W = int(im[kW]), Hw = (H + 31) >> 5;
  uint32_t* bits = p.gbits + im[kGbitsOff] + int64_t(g) * Hw * W;
  for (int64_t r = p.gt_run_off[row] + HD_TID; r < p.gt_run_off[row + 1]; r += HD_NT) {
    int64_t t = p.gt_runs[2 * r], len = p.gt_runs[2 * r + 1];
    while (len > 0) {
      const int x = int(t / H), y = int(t % H);
      const int cnt = int(len < H - y ? len : H - y);
      for (int wy = y >> 5; wy <= (y + cnt - 1) >> 5; ++wy) {
        const int lo = y > 32 * wy ? y - 32 * wy : 0;
        const int hi = y + cnt - 32 * wy < 32 ? y + cnt - 32 * wy : 32;       // exclusive
        const uint32_t mk = (hi == 32 ? 0xffffffffu : ((1u << hi) - 1u)) & ~((1u << lo) - 1u);
        hd_atomic_or(bits + int64_t(wy) * W + x, mk);
      }
      t += cnt; len -= cnt;
    }
  }
}

// ---- 4. IoU of one detection against the image's ground truths of its category ----
struct IouShared { long long inter; };

HD_FN void ce_iou(const MatchParams& p, int b, int j, IouShared& sh) {
  const int64_t* im = p.img + int64_t(b) * kImgFields;
  if (j >= im[kDetCount]) return;
  const int64_t row = im[kDetBegin] + j;
  if (!ce_evaluated(p, row)) return;
  const int64_t gi = im[kGtImg], gbase = p.gt_off[gi], ng = p.gt_off[gi + 1] - gbase;
  int64_t g0, g1;
  ce_gt_range(p, gi, p.dk[row], g0, g1);
  double* out = p.iou + im[kIouOff] + int64_t(j) * ng - gbase;
  if (!p.segm) {
    double d[4];
    ce_dt_xywh(p.boxes + row * 4, d);
    for (int64_t g = g0 + HD_TID; g < g1; g += HD_NT) out[g] = ce_bb_iou(d, p.gt_box + g * 4, p.gt_crowd[g] != 0);
    return;
  }
  const int H = int(im[kH]), W = int(im[kW]), Hw = (H + 31) >> 5;
  const int64_t plane = int64_t(Hw) * W;
  const uint32_t* db = p.dbits + im[kDbitsOff] + int64_t(j) * plane;
  const int32_t* bx = p.dbox + row * 4;
  for (int64_t g = g0; g < g1; ++g) {
    const int32_t* gx = p.gt_bbox + g * 4;
    const int x0 = bx[0] > gx[0] ? bx[0] : gx[0], x1 = bx[2] < gx[2] ? bx[2] : gx[2];
    const int y0 = bx[1] > gx[1] ? bx[1] : gx[1], y1 = bx[3] < gx[3] ? bx[3] : gx[3];
    if (x0 > x1 || y0 > y1) {                       // disjoint boxes (or an empty mask): IoU 0
      if (HD_TID == 0) out[g] = 0.0;
      continue;
    }
    const uint32_t* gbits = p.gbits + im[kGbitsOff] + (g - gbase) * plane;
    const int nx = x1 - x0 + 1, w0 = y0 >> 5, nw = (y1 >> 5) - w0 + 1;
    if (HD_TID == 0) sh.inter = 0;
    HD_SYNC();
    long long c = 0;
    for (int q = HD_TID; q < nx * nw; q += HD_NT) {
      const int64_t w = int64_t(w0 + q / nx) * W + x0 + q % nx;
      c += hd_popc(db[w] & gbits[w]);
    }
    hd_atomic_add(&sh.inter, c);
    HD_SYNC();
    if (HD_TID == 0) {
      const long long i = sh.inter;
      const long long u = p.gt_crowd[g] ? p.dpx[row] : p.dpx[row] + p.gt_px[g] - i;
      out[g] = i == 0 ? 0.0 : hd_ddiv(double(i), double(u));
    }
    HD_SYNC();
  }
}

// ---- 5. evaluateImg (one CTA per image; gtm zeroed before) ----
HD_FN bool ce_outside(double v, const double* rng) { return v < rng[0] || v > rng[1]; }

HD_FN void ce_match(const MatchParams& p, int b) {
  const int64_t* im = p.img + int64_t(b) * kImgFields;
  const int64_t d0 = im[kDetBegin];
  const int n = int(im[kDetCount]);
  const int64_t gi = im[kGtImg], gbase = p.gt_off[gi], ng = p.gt_off[gi + 1] - gbase;
  const int AT = p.A * p.T;
  for (int64_t task = HD_TID; task < int64_t(n) * AT; task += HD_NT) {
    const int pos = int(task / AT), a = int(task % AT) / p.T, t = int(task % p.T);
    const int j0 = p.dord[d0 + pos];
    if (j0 < 0) continue;
    const int k = p.dk[d0 + j0];
    if (pos > 0 && p.dk[d0 + p.dord[d0 + pos - 1]] == k) continue;    // not the first of its category
    int D = 0;
    while (pos + D < n && D < p.max_det && p.dord[d0 + pos + D] >= 0 && p.dk[d0 + p.dord[d0 + pos + D]] == k) ++D;
    int64_t g0, g1;
    ce_gt_range(p, gi, k, g0, g1);
    const double* rng = p.area_rng + 2 * a;
    uint8_t* gtm = p.gtm + im[kGtmOff] + int64_t(a * p.T + t) * ng - gbase;
    for (int d = 0; d < D; ++d) {
      const int j = p.dord[d0 + pos + d];
      const int64_t row = d0 + j;
      const double* iou = p.iou + im[kIouOff] + int64_t(j) * ng - gbase;
      double thr = p.iou_thr[t];
      int64_t m = -1;
      int m_ig = 0;
      for (int pass = 0; pass < 2; ++pass) {          // stable order: non-ignored ground truths first
        bool stop = false;
        for (int64_t g = g0; g < g1; ++g) {
          const bool crowd = p.gt_crowd[g] != 0;
          const int ig = (crowd || ce_outside(p.gt_area[g], rng)) ? 1 : 0;
          if (ig != pass) continue;
          if (gtm[g] && !crowd) continue;
          if (m >= 0 && m_ig == 0 && ig == 1) { stop = true; break; }
          if (iou[g] < thr) continue;
          thr = iou[g]; m = g; m_ig = ig;
        }
        if (stop) break;
      }
      double area;
      if (p.segm) {
        area = double(p.dpx[row]);
      } else {
        const float* bx = p.boxes + row * 4;
        area = hd_dmul(double(float(bx[2] - bx[0])), double(float(bx[3] - bx[1])));
      }
      uint32_t st;
      if (m >= 0) {
        gtm[m] = 1;
        // accumulate tests the matched annotation id for truth: a match to id 0 is not a true positive
        st = m_ig ? kIgnored : p.gt_id[m] != 0 ? kTp : ce_outside(area, rng) ? kIgnored : kFp;
      } else {
        st = ce_outside(area, rng) ? kIgnored : kFp;
      }
      hd_atomic_or(p.state + row * p.A + a, st << (2 * t));
    }
  }
}

// ---- 6. accumulate ----
// kept images' keys, in image-id order, with their record index as the sort value (one CTA per kept image)
HD_FN void ce_gather(const AccParams& p, int i) {
  const int64_t* kp = p.kept + int64_t(i) * 3;
  for (int64_t q = HD_TID; q < kp[2]; q += HD_NT) {
    p.key_in[kp[1] + q] = p.key[kp[0] + q];
    p.val_in[kp[1] + q] = kp[0] + q;
  }
}

HD_FN int64_t ce_lower(const uint64_t* a, int64_t n, uint64_t v) {
  int64_t lo = 0, hi = n;
  while (lo < hi) { const int64_t m = (lo + hi) >> 1; if (a[m] < v) lo = m + 1; else hi = m; }
  return lo;
}

struct AccShared {
  long long part_tp[kThreads], part_fp[kThreads], part_n[kThreads];
  unsigned long long best[kMaxRec];               // per recall index: max precision (bits of a double >= 0)
  double ss[kMaxRec];
  long long tq[kMaxRec];                          // least tp count with tp / npig >= recThrs[r]
};

// One (k, a, m, t): the score-sorted detections of category k with rank < maxDets[m] (accumulate's concatenation,
// sorted stably).  pr[i] is counted towards q[r] for every r whose recall threshold tp[i] reaches, so the envelope
// max_{i' >= i_r} pr[i'] is a maximum over recall indices; scores[r] is the score at i_r, the detection that makes
// tp reach tq[r] (the first detection when tq[r] = 0).
HD_FN void ce_acc(const AccParams& p, int cta, AccShared& sh) {
  const int t = cta % p.T, m = (cta / p.T) % p.M, a = (cta / (p.T * p.M)) % p.A, k = cta / (p.T * p.M * p.A);
  const int R = p.R, K = p.K, A = p.A, M = p.M;
  const int64_t npig = p.npig[k * A + a];
  auto at5 = [&](int r) { return ((((int64_t(t) * R + r) * K + k) * A + a) * M + m); };
  const int64_t at4 = ((int64_t(t) * K + k) * A + a) * M + m;
  if (npig == 0) {
    for (int r = HD_TID; r < R; r += HD_NT) { p.precision[at5(r)] = -1.0; p.scores[at5(r)] = -1.0; }
    if (HD_TID == 0) p.recall[at4] = -1.0;
    return;
  }
  const int64_t sb = ce_lower(p.key_out, p.n, uint64_t(k) << 32), se = ce_lower(p.key_out, p.n, uint64_t(k + 1) << 32);
  const int maxd = p.max_dets[m];
  const double dn = double(npig);
  for (int r = HD_TID; r < R; r += HD_NT) {
    long long lo = 0, hi = npig;                  // rc = x / npig is monotone in x and reaches 1 at npig
    while (lo < hi) { const long long x = (lo + hi) >> 1; if (hd_ddiv(double(x), dn) >= p.rec_thr[r]) hi = x; else lo = x + 1; }
    sh.tq[r] = lo;
    sh.best[r] = 0;
    sh.ss[r] = 0.0;
  }
  const int64_t len = se - sb, per = (len + HD_NT - 1) / HD_NT;
  const int64_t cb = sb + (per * HD_TID < len ? per * HD_TID : len), ce = sb + (per * (HD_TID + 1) < len ? per * (HD_TID + 1) : len);
  long long ltp = 0, lfp = 0, ln = 0;
  for (int64_t i = cb; i < ce; ++i) {
    const int64_t src = p.val_out[i];
    if (p.rank[src] >= maxd) continue;
    ++ln;
    const uint32_t st = (p.state[src * A + a] >> (2 * t)) & 3u;
    ltp += st == kTp; lfp += st == kFp;
  }
  sh.part_tp[HD_TID] = ltp; sh.part_fp[HD_TID] = lfp; sh.part_n[HD_TID] = ln;
  HD_SYNC();
  long long tp = 0, fp = 0, nb = 0, tp_all = 0, n_all = 0;
  for (int q = 0; q < HD_NT; ++q) {
    if (q < HD_TID) { tp += sh.part_tp[q]; fp += sh.part_fp[q]; nb += sh.part_n[q]; }
    tp_all += sh.part_tp[q]; n_all += sh.part_n[q];
  }
  const double eps = 2.220446049250313e-16;       // np.spacing(1)
  for (int64_t i = cb; i < ce; ++i) {
    const int64_t src = p.val_out[i];
    if (p.rank[src] >= maxd) continue;
    const uint32_t st = (p.state[src * A + a] >> (2 * t)) & 3u;
    const bool first = nb == 0;
    tp += st == kTp; fp += st == kFp; ++nb;
    const double dtp = double(tp);
    const double pr = hd_ddiv(dtp, hd_dadd(hd_dadd(double(fp), dtp), eps));
    int lo = 0, hi = R;                           // recall indices reached: tq[r] <= tp, r < lo
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (sh.tq[mid] <= tp) lo = mid + 1; else hi = mid; }
    if (lo > 0) {
      union { double d; unsigned long long u; } c; c.d = pr;
      hd_atomic_max(&sh.best[lo - 1], c.u);
    }
    if (st == kTp || first) {
      const double sc = double(ce_desc_score(uint32_t(p.key_out[i])));
      if (st == kTp)
        for (int r = lo - 1; r >= 0 && sh.tq[r] == tp; --r) sh.ss[r] = sc;
      if (first)
        for (int r = 0; r < R && sh.tq[r] == 0; ++r) sh.ss[r] = sc;
    }
  }
  HD_SYNC();
  if (HD_TID == 0) {
    double run = 0.0;
    for (int r = R - 1; r >= 0; --r) {
      union { double d; unsigned long long u; } c; c.u = sh.best[r];
      run = c.d > run ? c.d : run;
      const bool reached = n_all > 0 && sh.tq[r] <= tp_all;
      p.precision[at5(r)] = reached ? run : 0.0;
      p.scores[at5(r)] = reached ? sh.ss[r] : 0.0;
    }
    p.recall[at4] = n_all > 0 ? hd_ddiv(double(tp_all), dn) : 0.0;
  }
}

// Argument ranges of the C entries: 0 or TFB200_E_SHAPE.
static inline int ce_check_match(int B, int64_t N, int K, int A, int T, int max_det) {
  if (B <= 0 || N < 0 || K <= 0 || A <= 0 || A > kMaxArea || T <= 0 || T > kMaxThr || max_det <= 0 ||
      max_det > kMaxDets || N > INT32_MAX)
    return TFB200_E_SHAPE;
  return 0;
}
static inline int ce_check_acc(int K, int A, int T, int R, int M, int n_kept, int64_t n_rec, int64_t n) {
  if (K <= 0 || A <= 0 || A > kMaxArea || T <= 0 || T > kMaxThr || R <= 0 || R > kMaxRec || M <= 0 ||
      M > kMaxMaxDets || n_kept < 0 || n_rec < 0 || n < 0 || n > n_rec)
    return TFB200_E_SHAPE;
  if (int64_t(K) * A * M * T > INT32_MAX) return TFB200_E_SHAPE;
  return 0;
}

}  // namespace tfb200_coco
