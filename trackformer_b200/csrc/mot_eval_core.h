// MOTChallenge CLEAR-MOT and identity metrics (what motmetrics 1.2.0 computes for the reference's get_mot_accum /
// evaluate_mot_accums, src/trackformer/util/track_utils.py:354-417), written once as cooperative routines:
//
//   me_init_seq   (one CTA per sequence)  zero the sequence's state and counters (the tp matrices: a memset)
//   me_pairs_frame(one CTA per frame)     fp64 IoU of every object x hypothesis pair; count, or write the valid ones
//                                         (d = 1 - IoU <= 0.5) in row-major order and count tp(o, h)
//   me_scan       (one CTA)               frame pair offsets; a pair buffer that is too small flags every sequence
//   me_clear_seq  (one CTA per sequence)  MOTAccumulator.update frame by frame: re-establish, then a maximum-
//                                         cardinality / minimum-cost assignment per connected component of the
//                                         residual valid pairs (one thread per component), MISS / FP, FM, MT / ML
//   me_id_label   (one CTA per sequence)  connected components of the tp graph (GT ids x track ids)
//   me_id_comp    (one CTA per component) exact integer maximum-weight matching of tp; IDTP
//
// nvcc compiles them into csrc/mot_eval.cu's kernels, g++ (one "thread") into the test-only host build
// tests/host_build/mot_eval_host.cpp.  All box arithmetic is fp64 with separately rounded operations (no contraction;
// the host build is compiled with -ffp-contract=off), as numpy computes motmetrics' iou_matrix.
#pragma once

#include <float.h>
#include <limits.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include <initializer_list>
#include <type_traits>

#include "../../include/tfb200_fused.h"
#include "host_device.h"
#include "lsa_core.h"

namespace tfb200_mot {

namespace lsa = tfb200_lsa;

constexpr int kThreads = 256;
constexpr int kMaxClearSide = 64;        // rows / columns of one residual component of a frame's assignment
constexpr int kMaxIdSmall = 8192;        // the smaller side (GT ids or track ids) of one identity component
constexpr int kMaxIdLarge = 65536;       // its larger side

// per-sequence descriptor (int64 [S][kSeqFields], built on the host)
enum { kFrameBegin, kFrameEnd, kGtBegin, kGtCount, kTrkBegin, kTrkCount, kTpBegin, kSeqFields = 8 };

// per-sequence output slots (8 bytes each; kSumD holds a double)
enum {
  kStatus, kPairs, kMatches, kSwitches, kMisses, kFalsePos, kFrag, kMostly, kPartly, kLost, kIdtp,
  kClearRows, kClearCols, kIdRows, kIdCols, kSumD, kOutSlots = 16
};
// status bits
enum { kErrPairCapacity = 1, kErrFrameSize = 2, kErrClearComponent = 4, kErrIdComponent = 8 };


struct Params {
  int S, F, max_obj, max_hyp;
  int64_t pair_cap;
  const int64_t* seq;                              // [S][kSeqFields]
  const int32_t* fobj;                             // [F + 1] object rows of frame f: fobj[f] .. fobj[f + 1]
  const int32_t* fhyp;                             // [F + 1] hypothesis rows
  const int32_t* obj_id;                           // [n_obj] dense GT id within the sequence
  const float* obj_box;                            // [n_obj][4] x, y, w, h
  const int32_t* hyp_id;                           // [n_hyp] dense track id within the sequence
  const float* hyp_box;                            // [n_hyp][4]
  int64_t* out;                                    // [S][kOutSlots]
  // workspace
  int32_t* fcount;                                 // [F] valid pairs per frame
  int64_t* foff;                                   // [F + 1]
  int32_t* pair_o; int32_t* pair_h; double* pair_d;   // [pair_cap] global object row, global hypothesis row, d
  int32_t* tp;                                     // sequence s: [n_gt][n_trk] from seq[kTpBegin]
  int32_t* m; int32_t* present; int32_t* tracked; int32_t* fstate;   // [sum n_gt], from seq[kGtBegin]
  int32_t* hslot;                                  // [sum n_trk]: frame-local row of the track this frame, or -1
  int32_t* idlabel;                                // [sum n_gt + sum n_trk], from seq[kGtBegin] + seq[kTrkBegin]
  // identity components: per root GT id its member counts and list offsets within the sequence; then one slot per
  // GT id and per track for the member lists and the assignment's vectors (components are disjoint)
  int32_t *id_nr, *id_nc, *id_or, *id_oc;          // [sum n_gt]
  int32_t *g_list; lsa::Cols g_lsa;                                    // [sum n_gt]
  int32_t *t_list; lsa::Cols t_lsa;                                    // [sum n_trk]
  // frame scratch: [S][max_obj] per object, [S][max_hyp] per hypothesis
  lsa::Cols o_lsa;
  double* o_dev;
  int32_t *o_label, *o_list, *o_cand, *o_rb, *o_re, *o_ca, *o_cb, *o_oa, *o_ob, *o_state;
  uint8_t* o_mask;
  lsa::Cols h_lsa;
  int32_t *h_label, *h_list, *h_win;
  uint8_t* h_mask;
};

// Argument ranges shared by the C entries: 0 or TFB200_E_SHAPE.
static inline int me_check(int S, int F, int64_t n_gt, int64_t n_trk, int64_t tp_cells, int max_obj, int max_hyp,
                           int64_t pair_cap) {
  if (S <= 0 || F < 0 || n_gt < 0 || n_trk < 0 || tp_cells < 0 || max_obj < 0 || max_hyp < 0 || pair_cap < 0)
    return TFB200_E_SHAPE;
  if (n_gt + n_trk > INT32_MAX || int64_t(max_obj) * max_hyp > INT32_MAX) return TFB200_E_SHAPE;
  return 0;
}

// Carves the workspace (ws may be NULL to size it).  Returns the bytes needed; every array is 256-byte aligned.
static inline size_t me_carve(Params& p, char* ws, int S, int F, int64_t n_gt, int64_t n_trk, int64_t tp_cells,
                              int max_obj, int max_hyp, int64_t pair_cap) {
  size_t o = 0;
  auto take = [&](auto*& ptr, size_t n) {
    ptr = reinterpret_cast<std::remove_reference_t<decltype(ptr)>>(reinterpret_cast<uintptr_t>(ws) + o);
    o += (n * sizeof(*ptr) + 255) & ~size_t(255);
  };
  // the assignment state of a side that can be either the rows or the columns of a problem (see me_lsa_state)
  auto take_lsa = [&](lsa::Cols& c, size_t n) {
    take(c.shortest, n); take(c.v, n); take(c.path, n); take(c.row4col, n); take(c.in_sc, n);
  };
  const size_t so = size_t(S) * size_t(max_obj), sh = size_t(S) * size_t(max_hyp);
  take(p.fcount, size_t(F));
  take(p.foff, size_t(F) + 1);
  take(p.pair_o, size_t(pair_cap));
  take(p.pair_h, size_t(pair_cap));
  take(p.pair_d, size_t(pair_cap));
  take(p.tp, size_t(tp_cells));
  for (int32_t** a : {&p.m, &p.present, &p.tracked, &p.fstate}) take(*a, size_t(n_gt));
  take(p.hslot, size_t(n_trk));
  take(p.idlabel, size_t(n_gt + n_trk));
  for (int32_t** a : {&p.id_nr, &p.id_nc, &p.id_or, &p.id_oc, &p.g_list}) take(*a, size_t(n_gt));
  take_lsa(p.g_lsa, size_t(n_gt));
  take(p.t_list, size_t(n_trk));
  take_lsa(p.t_lsa, size_t(n_trk));
  take_lsa(p.o_lsa, so);
  take(p.o_dev, so);
  for (int32_t** a : {&p.o_label, &p.o_list, &p.o_cand, &p.o_rb, &p.o_re, &p.o_ca, &p.o_cb, &p.o_oa, &p.o_ob,
                      &p.o_state})
    take(*a, so);
  take(p.o_mask, so);
  take_lsa(p.h_lsa, sh);
  for (int32_t** a : {&p.h_label, &p.h_list, &p.h_win}) take(*a, sh);
  take(p.h_mask, sh);
  return o;
}

// Shared state of one CTA (a plain struct in the host build).
struct Shared {
  int64_t part[kThreads];
  double dpart[kThreads];
  int64_t base;
  int changed, err;
  int n_match, n_switch, n_miss, n_fp, n_frag, n_mt, n_pt, n_ml, max_rows, max_cols;
  lsa::Cta<kThreads>::Scratch lsa;
};


// ---- distances (motmetrics.distances.iou_matrix on float32 x, y, w, h promoted to float64) ----
HD_FN double me_max0(double v) { return v > 0.0 ? v : (v == v ? 0.0 : v); }     // np.maximum(v, 0), NaN kept
HD_FN double me_dist(const float* a, const float* b) {
  const double ax0 = a[0], ay0 = a[1], ax1 = hd_dadd(ax0, double(a[2])), ay1 = hd_dadd(ay0, double(a[3]));
  const double bx0 = b[0], by0 = b[1], bx1 = hd_dadd(bx0, double(b[2])), by1 = hd_dadd(by0, double(b[3]));
  const double ix = me_max0(hd_dsub(ax1 < bx1 ? ax1 : bx1, ax0 > bx0 ? ax0 : bx0));
  const double iy = me_max0(hd_dsub(ay1 < by1 ? ay1 : by1, ay0 > by0 ? ay0 : by0));
  const double inter = hd_dmul(ix, iy);
  const double area_a = hd_dmul(me_max0(hd_dsub(ax1, ax0)), me_max0(hd_dsub(ay1, ay0)));
  const double area_b = hd_dmul(me_max0(hd_dsub(bx1, bx0)), me_max0(hd_dsub(by1, by0)));
  const double uni = hd_dsub(hd_dadd(area_a, area_b), inter);
  const double iou = inter == 0.0 ? 0.0 : hd_ddiv(inter, uni);
  return hd_dsub(1.0, iou);
}
HD_FN bool me_valid(double d) { return d <= 0.5; }       // max_iou = 0.5; NaN is invalid

// ---- ordered block scan: thread t owns the contiguous chunk [b, e) of n items, in index order ----
HD_FN void me_chunk(int64_t n, int64_t& b, int64_t& e) {
  const int64_t per = (n + HD_NT - 1) / HD_NT;
  b = per * HD_TID < n ? per * HD_TID : n;
  e = b + per < n ? b + per : n;
}
// exclusive base of this thread's chunk from every thread's chunk total v; sh.base = the total
HD_FN int64_t me_scan_parts(Shared& sh, int64_t v) {
  HD_SYNC();
  sh.part[HD_TID] = v;
  HD_SYNC();
  if (HD_TID == 0) {
    int64_t run = 0;
    for (int t = 0; t < HD_NT; ++t) { const int64_t x = sh.part[t]; sh.part[t] = run; run += x; }
    sh.base = run;
  }
  HD_SYNC();
  const int64_t r = sh.part[HD_TID];
  HD_SYNC();
  return r;
}
// sum of v over the threads in thread order (a fixed order: bit-reproducible run to run)
HD_FN double me_sum_ordered(Shared& sh, double v) {
  HD_SYNC();
  sh.dpart[HD_TID] = v;
  HD_SYNC();
  double s = 0.0;
  for (int t = 0; t < HD_NT; ++t) s += sh.dpart[t];
  HD_SYNC();
  return s;
}

// ---- rectangular assignment: every member of the smaller side to a distinct member of the larger side ----
// Either side of a component can be the rows, so each is carved with a column's arrays: side a (from offset ao) gives
// the rows, which take its dual, assignment and path arrays as their dual, assignment and visited list, and side b
// (from offset bo) the columns.
HD_FN void me_lsa_state(const lsa::Cols& a, int64_t ao, const lsa::Cols& b, int64_t bo, lsa::Rows& R,
                        lsa::Cols& C) {
  R = lsa::Rows{a.v + ao, a.row4col + ao, a.path + ao};
  C = lsa::Cols{b.shortest + bo, b.v + bo, b.path + bo, b.row4col + bo, b.in_sc + bo};
}

// the sequence whose range of `field` (kFrameBegin or kGtBegin) holds v; sequences are stored in order
HD_FN int me_seq_of(const Params& P, int field, int64_t v) {
  int lo = 0, hi = P.S - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (P.seq[int64_t(mid) * kSeqFields + field] <= v) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- per sequence: zero the state ----
HD_FN void me_init_seq(const Params& P, int s) {
  const int64_t* q = P.seq + int64_t(s) * kSeqFields;
  const int64_t gb = q[kGtBegin], G = q[kGtCount], tb = q[kTrkBegin], H = q[kTrkCount];
  for (int k = HD_TID; k < kOutSlots; k += HD_NT) P.out[int64_t(s) * kOutSlots + k] = 0;
  for (int64_t g = HD_TID; g < G; g += HD_NT) {
    P.m[gb + g] = -1; P.present[gb + g] = 0; P.tracked[gb + g] = 0; P.fstate[gb + g] = 0;
  }
  for (int64_t h = HD_TID; h < H; h += HD_NT) P.hslot[tb + h] = -1;
  int32_t* lab = P.idlabel + gb + tb;
  for (int64_t n = HD_TID; n < G + H; n += HD_NT) lab[n] = int32_t(n);
  for (int64_t g = HD_TID; g < G; g += HD_NT) { P.id_nr[gb + g] = 0; P.id_nc[gb + g] = 0; }
}

// ---- per frame: valid pairs ----
template <bool kWrite>
HD_FN void me_pairs_frame(const Params& P, int f, Shared& sh) {
  if (kWrite && P.foff[P.F] > P.pair_cap) return;
  const int ob = P.fobj[f], no = P.fobj[f + 1] - ob, hb = P.fhyp[f], nh = P.fhyp[f + 1] - hb;
  int64_t b, e;
  me_chunk(int64_t(no) * nh, b, e);
  int64_t cnt = 0;
  for (int64_t k = b; k < e; ++k)
    cnt += me_valid(me_dist(P.obj_box + 4 * (ob + k / nh), P.hyp_box + 4 * (hb + k % nh)));
  int64_t at = me_scan_parts(sh, cnt);
  if (!kWrite) {
    if (HD_TID == 0) P.fcount[f] = int32_t(sh.base);
    return;
  }
  at += P.foff[f];
  const int64_t* q = P.seq + int64_t(me_seq_of(P, kFrameBegin, f)) * kSeqFields;
  int32_t* tp = P.tp + q[kTpBegin];
  const int64_t H = q[kTrkCount];
  for (int64_t k = b; k < e; ++k) {
    const int o = ob + int(k / nh), h = hb + int(k % nh);
    const double d = me_dist(P.obj_box + 4 * o, P.hyp_box + 4 * h);
    if (!me_valid(d)) continue;
    P.pair_o[at] = o; P.pair_h[at] = h; P.pair_d[at] = d;
    ++at;
    hd_atomic_add(tp + int64_t(P.obj_id[o]) * H + P.hyp_id[h], 1);
  }
}

// ---- one CTA: frame offsets; flags every sequence when the pair buffer is too small ----
HD_FN void me_scan(const Params& P, Shared& sh) {
  int64_t b, e;
  me_chunk(P.F, b, e);
  int64_t v = 0;
  for (int64_t f = b; f < e; ++f) v += P.fcount[f];
  int64_t at = me_scan_parts(sh, v);
  for (int64_t f = b; f < e; ++f) { P.foff[f] = at; at += P.fcount[f]; }
  if (HD_TID == 0) P.foff[P.F] = sh.base;
  HD_SYNC();
  for (int s = HD_TID; s < P.S; s += HD_NT) {
    const int64_t* q = P.seq + int64_t(s) * kSeqFields;
    int64_t* out = P.out + int64_t(s) * kOutSlots;
    out[kPairs] = P.foff[q[kFrameEnd]] - P.foff[q[kFrameBegin]];
    if (sh.base > P.pair_cap) out[kStatus] |= kErrPairCapacity;
  }
}

// pair index of (frame-local object o, global hypothesis row h) in o's row of the frame's pairs, or -1
HD_FN int64_t me_find(const Params& P, const int32_t* rb, const int32_t* re, int64_t pb, int o, int h) {
  int64_t lo = pb + rb[o], hi = pb + re[o];
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (P.pair_h[mid] < h) lo = mid + 1; else hi = mid;
  }
  return lo < pb + re[o] && P.pair_h[lo] == h ? lo : -1;
}

struct ClearCost {
  const Params* P; const int32_t *rows, *cols, *rb, *re; int64_t pb; int hb; bool tr; double big;
  HD_FN double operator()(int r, int c) const {
    const int o = tr ? cols[c] : rows[r], h = tr ? rows[r] : cols[c];
    const int64_t k = me_find(*P, rb, re, pb, o, hb + h);
    return k >= 0 ? P->pair_d[k] : big;
  }
};

// ---- per sequence: MOTAccumulator.update over the frames, then the per-GT-id counts ----
HD_FN void me_clear_seq(const Params& P, int s, Shared& sh) {
  const int64_t* q = P.seq + int64_t(s) * kSeqFields;
  int64_t* out = P.out + int64_t(s) * kOutSlots;
  if (out[kStatus] & kErrPairCapacity) return;
  const int64_t gb = q[kGtBegin], G = q[kGtCount], tb = q[kTrkBegin];
  const int64_t so = int64_t(s) * P.max_obj, sq = int64_t(s) * P.max_hyp;
  double* odev = P.o_dev + so;
  int32_t *olab = P.o_label + so, *olist = P.o_list + so;
  int32_t *ocand = P.o_cand + so, *orb = P.o_rb + so, *ore = P.o_re + so, *oca = P.o_ca + so, *ocb = P.o_cb + so;
  int32_t *ooa = P.o_oa + so, *oob = P.o_ob + so, *ostate = P.o_state + so;
  uint8_t* omask = P.o_mask + so;
  int32_t *hlab = P.h_label + sq, *hlist = P.h_list + sq, *hwin = P.h_win + sq;
  uint8_t* hmask = P.h_mask + sq;
  if (HD_TID == 0) {
    sh.err = 0; sh.n_match = sh.n_switch = sh.n_miss = sh.n_fp = sh.n_frag = sh.n_mt = sh.n_pt = sh.n_ml = 0;
    sh.max_rows = sh.max_cols = 0;
  }
  double sumd = 0.0;
  for (int64_t f = q[kFrameBegin]; f < q[kFrameEnd]; ++f) {
    const int ob = P.fobj[f], no = P.fobj[f + 1] - ob, hb = P.fhyp[f], nh = P.fhyp[f + 1] - hb;
    const int64_t pb = P.foff[f], np = P.foff[f + 1] - pb;
    if (no > P.max_obj || nh > P.max_hyp) {
      if (HD_TID == 0) out[kStatus] |= kErrFrameSize;
      return;
    }
    for (int o = HD_TID; o < no; o += HD_NT) {
      omask[o] = 0; odev[o] = 0.0; ostate[o] = 0; orb[o] = ore[o] = 0; olab[o] = o; ocand[o] = -1;
    }
    for (int h = HD_TID; h < nh; h += HD_NT) {
      hmask[h] = 0; hwin[h] = INT_MAX; hlab[h] = no + h; P.hslot[tb + P.hyp_id[hb + h]] = h;
    }
    HD_SYNC();
    for (int64_t k = HD_TID; k < np; k += HD_NT) {          // pairs are row-major: each object's row is contiguous
      const int32_t o = P.pair_o[pb + k];
      if (k == 0 || P.pair_o[pb + k - 1] != o) orb[o - ob] = int32_t(k);
      if (k == np - 1 || P.pair_o[pb + k + 1] != o) ore[o - ob] = int32_t(k + 1);
    }
    HD_SYNC();
    if (np > 0) {
      // re-establish: object o keeps its previous partner if present and valid; the first object in order wins it
      for (int o = HD_TID; o < no; o += HD_NT) {
        const int32_t p = P.m[gb + P.obj_id[ob + o]];
        if (p < 0) continue;
        const int32_t j = P.hslot[tb + p];
        if (j >= 0 && me_find(P, orb, ore, pb, o, hb + j) >= 0) { ocand[o] = j; hd_atomic_min(hwin + j, o); }
      }
      HD_SYNC();
      for (int o = HD_TID; o < no; o += HD_NT) {
        const int j = ocand[o];
        if (j < 0 || hwin[j] != o) continue;
        omask[o] = 1; hmask[j] = 1; ostate[o] = 1;
        odev[o] = P.pair_d[me_find(P, orb, ore, pb, o, hb + j)];
      }
      HD_SYNC();
      // connected components of the residual valid pairs: every node ends labelled with its component's least node
      for (;;) {
        if (HD_TID == 0) sh.changed = 0;
        HD_SYNC();
        for (int64_t k = HD_TID; k < np; k += HD_NT) {
          const int o = P.pair_o[pb + k] - ob, h = P.pair_h[pb + k] - hb;
          if (omask[o] || hmask[h]) continue;
          const int la = olab[o], lb = hlab[h];
          if (la != lb) {
            const int mn = la < lb ? la : lb;
            hd_atomic_min(olab + o, mn); hd_atomic_min(hlab + h, mn);
            sh.changed = 1;
          }
        }
        HD_SYNC();
        for (int x = HD_TID; x < no + nh; x += HD_NT) {
          int32_t* lx = x < no ? olab + x : hlab + (x - no);
          const int l = *lx, ll = l < no ? olab[l] : hlab[l - no];
          if (ll < l) hd_atomic_min(lx, ll);
        }
        HD_SYNC();
        const int again = sh.changed;
        HD_SYNC();
        if (!again) break;
      }
      // a component with an edge holds an object, so its label is an object: size it from its root
      for (int o = HD_TID; o < no; o += HD_NT) {
        int a = 0, b = 0;
        if (!omask[o] && olab[o] == o) {
          for (int x = 0; x < no; ++x) a += !omask[x] && olab[x] == o;
          for (int y = 0; y < nh; ++y) b += !hmask[y] && hlab[y] == o;
        }
        oca[o] = b > 0 ? a : 0; ocb[o] = b;
      }
      HD_SYNC();                                            // written with a thread stride, read by chunk below
      int64_t cb0, ce0;
      me_chunk(no, cb0, ce0);
      int64_t va = 0, vb = 0;
      for (int64_t o = cb0; o < ce0; ++o) { va += oca[o]; vb += ocb[o]; }
      int64_t xa = me_scan_parts(sh, va), xb = me_scan_parts(sh, vb);
      for (int64_t o = cb0; o < ce0; ++o) { ooa[o] = int32_t(xa); oob[o] = int32_t(xb); xa += oca[o]; xb += ocb[o]; }
      HD_SYNC();
      for (int o = HD_TID; o < no; o += HD_NT) {
        const int a = oca[o], b = ocb[o];
        if (b == 0) continue;
        hd_atomic_max(&sh.max_rows, a); hd_atomic_max(&sh.max_cols, b);
        if (a > kMaxClearSide || b > kMaxClearSide) { sh.err = 1; continue; }
        int32_t *rl = olist + ooa[o], *cl = hlist + oob[o];
        for (int x = 0, n = 0; x < no; ++x) if (!omask[x] && olab[x] == o) rl[n++] = x;
        for (int y = 0, n = 0; y < nh; ++y) if (!hmask[y] && hlab[y] == o) cl[n++] = y;
        const bool tr = a > b;
        const int r = tr ? b : a;
        lsa::Rows R;
        lsa::Cols C;
        if (tr) me_lsa_state(P.h_lsa, sq + oob[o], P.o_lsa, so + ooa[o], R, C);
        else me_lsa_state(P.o_lsa, so + ooa[o], P.h_lsa, sq + oob[o], R, C);
        // motmetrics' add_expensive_edges: an invalid pair costs more than any two valid matchings differ by
        const ClearCost cost{&P, tr ? cl : rl, tr ? rl : cl, orb, ore, pb, hb, tr, 2.0 * r * (0.5 + 1.0) + 1.0};
        lsa::Thread::Scratch scratch;
        lsa::solve<lsa::Thread>(r, tr ? a : b, cost, R, C, scratch);     // finite costs: always feasible
        for (int i = 0; i < r; ++i) {
          const int x = tr ? rl[R.col4row[i]] : rl[i], y = tr ? cl[i] : cl[R.col4row[i]];
          const int64_t k = me_find(P, orb, ore, pb, x, hb + y);
          if (k < 0) continue;                              // an expensive edge: not a match
          const int gi = int(gb + P.obj_id[ob + x]), hid = P.hyp_id[hb + y], prev = P.m[gi];
          ostate[x] = prev >= 0 && prev != hid ? 2 : 1;
          P.m[gi] = hid;
          odev[x] = P.pair_d[k];
          omask[x] = 1; hmask[y] = 1;
        }
      }
      HD_SYNC();
      if (sh.err) {
        if (HD_TID == 0) {
          out[kStatus] |= kErrClearComponent;
          out[kClearRows] = sh.max_rows;
          out[kClearCols] = sh.max_cols;
        }
        return;
      }
    }
    // events: MATCH / SWITCH / MISS per object, FP per unmatched hypothesis
    for (int o = HD_TID; o < no; o += HD_NT) {
      const int gi = int(gb + P.obj_id[ob + o]), st = ostate[o];
      int fs = P.fstate[gi];                              // bit 0: tracked before; bit 1: missed since then
      ++P.present[gi];
      if (st) {
        ++P.tracked[gi];
        hd_atomic_add(st == 2 ? &sh.n_switch : &sh.n_match, 1);
        if (fs & 2) hd_atomic_add(&sh.n_frag, 1);
        fs = 1;
      } else {
        hd_atomic_add(&sh.n_miss, 1);
        if (fs & 1) fs |= 2;
      }
      P.fstate[gi] = fs;
    }
    for (int h = HD_TID; h < nh; h += HD_NT) {
      if (!hmask[h]) hd_atomic_add(&sh.n_fp, 1);
      P.hslot[tb + P.hyp_id[hb + h]] = -1;
    }
    int64_t db, de;
    me_chunk(no, db, de);
    double part = 0.0;
    for (int64_t o = db; o < de; ++o) part += odev[o];
    sumd += me_sum_ordered(sh, part);
  }
  for (int64_t g = HD_TID; g < G; g += HD_NT) {
    const int64_t pr = P.present[gb + g], tr = P.tracked[gb + g];
    if (pr == 0) continue;
    if (5 * tr >= 4 * pr) hd_atomic_add(&sh.n_mt, 1);          // tracked ratio >= 0.8
    else if (5 * tr < pr) hd_atomic_add(&sh.n_ml, 1);          // < 0.2
    else hd_atomic_add(&sh.n_pt, 1);
  }
  HD_SYNC();
  if (HD_TID == 0) {
    out[kMatches] = sh.n_match; out[kSwitches] = sh.n_switch; out[kMisses] = sh.n_miss; out[kFalsePos] = sh.n_fp;
    out[kFrag] = sh.n_frag; out[kMostly] = sh.n_mt; out[kPartly] = sh.n_pt; out[kLost] = sh.n_ml;
    out[kClearRows] = sh.max_rows; out[kClearCols] = sh.max_cols;
    double* sd = reinterpret_cast<double*>(out + kSumD);
    *sd = sumd;
  }
}

// ---- per sequence: connected components of the tp graph (nodes: GT ids, then track ids) ----
HD_FN void me_id_label(const Params& P, int s, Shared& sh) {
  const int64_t* q = P.seq + int64_t(s) * kSeqFields;
  if (P.out[int64_t(s) * kOutSlots + kStatus] & kErrPairCapacity) return;
  const int64_t G = q[kGtCount], H = q[kTrkCount];
  int32_t* lab = P.idlabel + q[kGtBegin] + q[kTrkBegin];
  const int64_t pb = P.foff[q[kFrameBegin]], pe = P.foff[q[kFrameEnd]];
  for (;;) {
    if (HD_TID == 0) sh.changed = 0;
    HD_SYNC();
    for (int64_t k = pb + HD_TID; k < pe; k += HD_NT) {
      const int64_t a = P.obj_id[P.pair_o[k]], b = G + P.hyp_id[P.pair_h[k]];
      const int la = lab[a], lb = lab[b];
      if (la != lb) {
        const int mn = la < lb ? la : lb;
        hd_atomic_min(lab + a, mn); hd_atomic_min(lab + b, mn);
        sh.changed = 1;
      }
    }
    HD_SYNC();
    for (int64_t x = HD_TID; x < G + H; x += HD_NT) {
      const int l = lab[x], ll = lab[l];
      if (ll < l) hd_atomic_min(lab + x, ll);
    }
    HD_SYNC();
    const int again = sh.changed;
    HD_SYNC();
    if (!again) break;
  }
  // members per component root (a GT id: every edge has one) and the offsets of its member lists
  int32_t *nr = P.id_nr + q[kGtBegin], *nc = P.id_nc + q[kGtBegin];
  for (int64_t x = HD_TID; x < G + H; x += HD_NT) {
    const int l = lab[x];
    if (l < G) hd_atomic_add(x < G ? nr + l : nc + l, 1);
  }
  HD_SYNC();
  int64_t b, e;
  me_chunk(G, b, e);
  int64_t vr = 0, vc = 0;
  for (int64_t g = b; g < e; ++g) { vr += nr[g]; vc += nc[g]; }
  int64_t xr = me_scan_parts(sh, vr), xc = me_scan_parts(sh, vc);
  int32_t *orr = P.id_or + q[kGtBegin], *occ = P.id_oc + q[kGtBegin];
  for (int64_t g = b; g < e; ++g) { orr[g] = int32_t(xr); occ[g] = int32_t(xc); xr += nr[g]; xc += nc[g]; }
}

// ordered compaction of the nodes [0, n) labelled root into list; returns their count (nothing written above cap)
HD_FN int me_gather(const int32_t* lab, int64_t n, int root, int32_t* list, int cap, Shared& sh) {
  int64_t b, e;
  me_chunk(n, b, e);
  int64_t c = 0;
  for (int64_t x = b; x < e; ++x) c += lab[x] == root;
  int64_t at = me_scan_parts(sh, c);
  const int64_t total = sh.base;
  if (total <= cap)
    for (int64_t x = b; x < e; ++x)
      if (lab[x] == root) list[at++] = int32_t(x);
  HD_SYNC();
  return int(total);
}

struct IdCost {
  const int32_t* tp; const int32_t *rows, *cols; int64_t H; bool tr;
  HD_FN double operator()(int r, int c) const {
    const int64_t g = tr ? cols[c] : rows[r], h = tr ? rows[r] : cols[c];
    return -double(tp[g * H + h]);
  }
};

// ---- per GT id k (global index): if it roots a component of the tp graph, its maximum-weight matching ----
HD_FN void me_id_comp(const Params& P, int64_t k, Shared& sh) {
  const int s = me_seq_of(P, kGtBegin, k);
  const int64_t* q = P.seq + int64_t(s) * kSeqFields;
  int64_t* out = P.out + int64_t(s) * kOutSlots;
  if (out[kStatus] & kErrPairCapacity) return;
  const int64_t G = q[kGtCount], H = q[kTrkCount], g = k - q[kGtBegin];
  const int64_t gb = q[kGtBegin], tb = q[kTrkBegin];
  const int32_t* lab = P.idlabel + gb + tb;
  const int a = P.id_nr[gb + g], b = P.id_nc[gb + g];
  if (lab[g] != g || b == 0) return;                      // not a root, or a GT id no track ever covered
  if (HD_TID == 0) { hd_atomic_max(out + kIdRows, a); hd_atomic_max(out + kIdCols, b); }
  if ((a < b ? a : b) > kMaxIdSmall || (a < b ? b : a) > kMaxIdLarge) {
    if (HD_TID == 0) hd_atomic_or(out + kStatus, kErrIdComponent);
    return;
  }
  const int64_t orr = gb + P.id_or[gb + g], occ = tb + P.id_oc[gb + g];
  me_gather(lab, G, int(g), P.g_list + orr, a, sh);
  me_gather(lab + G, H, int(g), P.t_list + occ, b, sh);
  const bool tr = a > b;
  lsa::Rows R;
  lsa::Cols C;
  if (tr) me_lsa_state(P.t_lsa, occ, P.g_lsa, orr, R, C);
  else me_lsa_state(P.g_lsa, orr, P.t_lsa, occ, R, C);
  const IdCost cost{P.tp + q[kTpBegin], tr ? P.t_list + occ : P.g_list + orr, tr ? P.g_list + orr : P.t_list + occ,
                    H, tr};
  lsa::solve<lsa::Cta<kThreads>>(tr ? b : a, tr ? a : b, cost, R, C, sh.lsa);     // finite costs: always feasible
  if (HD_TID == 0) {
    int64_t idtp = 0;
    for (int r = 0; r < (tr ? b : a); ++r) idtp -= int64_t(cost(r, R.col4row[r]));
    hd_atomic_add(out + kIdtp, idtp);
  }
}

}  // namespace tfb200_mot
