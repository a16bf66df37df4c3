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

#if defined(__CUDACC__)
#define ME_FN __device__ inline
#define ME_MFN __device__ inline
#define ME_SYNC() __syncthreads()
#define ME_TID (int(threadIdx.x))
#define ME_NT (int(blockDim.x))
#define me_atomic_min(p, v) atomicMin((p), (v))
#define me_atomic_add(p, v) atomicAdd((p), (v))
#define me_atomic_max(p, v) atomicMax((p), (v))
__device__ inline void me_add64(int64_t* p, int64_t v) {
  atomicAdd(reinterpret_cast<unsigned long long*>(p), static_cast<unsigned long long>(v));
}
__device__ inline void me_max64(int64_t* p, int64_t v) { atomicMax(reinterpret_cast<long long*>(p), (long long)v); }
__device__ inline void me_or64(int64_t* p, int64_t v) {
  atomicOr(reinterpret_cast<unsigned long long*>(p), static_cast<unsigned long long>(v));
}
#define me_add(a, b) __dadd_rn((a), (b))
#define me_sub(a, b) __dsub_rn((a), (b))
#define me_mul(a, b) __dmul_rn((a), (b))
#define me_div(a, b) __ddiv_rn((a), (b))
#else
#define ME_FN static inline
#define ME_MFN inline
#define ME_SYNC() ((void)0)
#define ME_TID 0
#define ME_NT 1
template <class T> static inline T me_atomic_min(T* p, T v) { T o = *p; if (v < o) *p = v; return o; }
template <class T> static inline T me_atomic_add(T* p, T v) { T o = *p; *p = o + v; return o; }
template <class T> static inline T me_atomic_max(T* p, T v) { T o = *p; if (v > o) *p = v; return o; }
static inline void me_add64(int64_t* p, int64_t v) { *p += v; }
static inline void me_max64(int64_t* p, int64_t v) { if (v > *p) *p = v; }
static inline void me_or64(int64_t* p, int64_t v) { *p |= v; }
#define me_add(a, b) ((a) + (b))
#define me_sub(a, b) ((a) - (b))
#define me_mul(a, b) ((a) * (b))
#define me_div(a, b) ((a) / (b))
#endif

namespace tfb200_mot {

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


// One side (rows or columns) of an assignment problem, indexed by the component's compact position.
struct LsaSide {
  double* dual; double* shortest; int32_t* path; int32_t* mate; uint8_t* flag;
};

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
  int32_t *g_list, *g_path, *g_mate; double *g_dual, *g_short; uint8_t* g_flag;   // [sum n_gt]
  int32_t *t_list, *t_path, *t_mate; double *t_dual, *t_short; uint8_t* t_flag;   // [sum n_trk]
  // frame scratch: [S][max_obj] per object, [S][max_hyp] per hypothesis
  double *o_dual, *o_short, *o_dev;
  int32_t *o_path, *o_mate, *o_label, *o_list, *o_cand, *o_rb, *o_re, *o_ca, *o_cb, *o_oa, *o_ob, *o_state;
  uint8_t *o_flag, *o_mask;
  double *h_dual, *h_short;
  int32_t *h_path, *h_mate, *h_label, *h_list, *h_win;
  uint8_t *h_flag, *h_mask;
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
  for (int32_t** a : {&p.id_nr, &p.id_nc, &p.id_or, &p.id_oc, &p.g_list, &p.g_path, &p.g_mate}) take(*a, size_t(n_gt));
  for (double** a : {&p.g_dual, &p.g_short}) take(*a, size_t(n_gt));
  take(p.g_flag, size_t(n_gt));
  for (int32_t** a : {&p.t_list, &p.t_path, &p.t_mate}) take(*a, size_t(n_trk));
  for (double** a : {&p.t_dual, &p.t_short}) take(*a, size_t(n_trk));
  take(p.t_flag, size_t(n_trk));
  for (double** a : {&p.o_dual, &p.o_short, &p.o_dev}) take(*a, so);
  for (int32_t** a : {&p.o_path, &p.o_mate, &p.o_label, &p.o_list, &p.o_cand, &p.o_rb, &p.o_re, &p.o_ca, &p.o_cb,
                      &p.o_oa, &p.o_ob, &p.o_state})
    take(*a, so);
  for (uint8_t** a : {&p.o_flag, &p.o_mask}) take(*a, so);
  for (double** a : {&p.h_dual, &p.h_short}) take(*a, sh);
  for (int32_t** a : {&p.h_path, &p.h_mate, &p.h_label, &p.h_list, &p.h_win}) take(*a, sh);
  for (uint8_t** a : {&p.h_flag, &p.h_mask}) take(*a, sh);
  return o;
}

// Shared state of one CTA (a plain struct in the host build).
struct Shared {
  int64_t part[kThreads];
  double dpart[kThreads];
  double red_v[kThreads];
  int red_b[kThreads], red_k[kThreads];
  int64_t base;
  double ctl_min;
  int ctl_i, ctl_sink, changed, err;
  int n_match, n_switch, n_miss, n_fp, n_frag, n_mt, n_pt, n_ml, max_rows, max_cols;
};


// ---- distances (motmetrics.distances.iou_matrix on float32 x, y, w, h promoted to float64) ----
ME_FN double me_max0(double v) { return v > 0.0 ? v : (v == v ? 0.0 : v); }     // np.maximum(v, 0), NaN kept
ME_FN double me_dist(const float* a, const float* b) {
  const double ax0 = a[0], ay0 = a[1], ax1 = me_add(ax0, double(a[2])), ay1 = me_add(ay0, double(a[3]));
  const double bx0 = b[0], by0 = b[1], bx1 = me_add(bx0, double(b[2])), by1 = me_add(by0, double(b[3]));
  const double ix = me_max0(me_sub(ax1 < bx1 ? ax1 : bx1, ax0 > bx0 ? ax0 : bx0));
  const double iy = me_max0(me_sub(ay1 < by1 ? ay1 : by1, ay0 > by0 ? ay0 : by0));
  const double inter = me_mul(ix, iy);
  const double area_a = me_mul(me_max0(me_sub(ax1, ax0)), me_max0(me_sub(ay1, ay0)));
  const double area_b = me_mul(me_max0(me_sub(bx1, bx0)), me_max0(me_sub(by1, by0)));
  const double uni = me_sub(me_add(area_a, area_b), inter);
  const double iou = inter == 0.0 ? 0.0 : me_div(inter, uni);
  return me_sub(1.0, iou);
}
ME_FN bool me_valid(double d) { return d <= 0.5; }       // max_iou = 0.5; NaN is invalid

// ---- ordered block scan: thread t owns the contiguous chunk [b, e) of n items, in index order ----
ME_FN void me_chunk(int64_t n, int64_t& b, int64_t& e) {
  const int64_t per = (n + ME_NT - 1) / ME_NT;
  b = per * ME_TID < n ? per * ME_TID : n;
  e = b + per < n ? b + per : n;
}
// exclusive base of this thread's chunk from every thread's chunk total v; sh.base = the total
ME_FN int64_t me_scan_parts(Shared& sh, int64_t v) {
  ME_SYNC();
  sh.part[ME_TID] = v;
  ME_SYNC();
  if (ME_TID == 0) {
    int64_t run = 0;
    for (int t = 0; t < ME_NT; ++t) { const int64_t x = sh.part[t]; sh.part[t] = run; run += x; }
    sh.base = run;
  }
  ME_SYNC();
  const int64_t r = sh.part[ME_TID];
  ME_SYNC();
  return r;
}
// sum of v over the threads in thread order (a fixed order: bit-reproducible run to run)
ME_FN double me_sum_ordered(Shared& sh, double v) {
  ME_SYNC();
  sh.dpart[ME_TID] = v;
  ME_SYNC();
  double s = 0.0;
  for (int t = 0; t < ME_NT; ++t) s += sh.dpart[t];
  ME_SYNC();
  return s;
}

// ---- rectangular assignment: every one of a rows to a distinct column of b >= a, minimum total cost ----
// The shortest augmenting path method scipy.optimize.linear_sum_assignment uses (Crouse 2016), with every cost
// finite.  kTeam: the CTA shares the column scans; otherwise the calling thread solves it alone.  Among equal reduced
// costs the scan prefers an unmatched column, then the lower index.
ME_FN bool me_better(double v, int busy, int k, double lv, int lb, int lk) {
  return v < lv || (v == lv && (busy < lb || (busy == lb && k < lk)));
}

template <bool kTeam, class Cost>
ME_FN void me_lsa(int a, int b, const Cost& cost, const LsaSide& R, const LsaSide& C, Shared& sh) {
  const int t0 = kTeam ? ME_TID : 0, nt = kTeam ? ME_NT : 1;
  for (int r = t0; r < a; r += nt) { R.dual[r] = 0.0; R.mate[r] = -1; }
  for (int c = t0; c < b; c += nt) { C.dual[c] = 0.0; C.mate[c] = -1; }
  for (int cur = 0; cur < a; ++cur) {
    for (int r = t0; r < a; r += nt) R.flag[r] = 0;
    for (int c = t0; c < b; c += nt) { C.flag[c] = 0; C.shortest[c] = INFINITY; }
    if (kTeam) ME_SYNC();
    double minv = 0.0;
    int i = cur, sink = -1;
    while (sink < 0) {
      if (t0 == 0) R.flag[i] = 1;
      const double ui = R.dual[i];
      double lo = INFINITY;
      int lb = 2, lk = INT_MAX;
      for (int c = t0; c < b; c += nt) {
        if (C.flag[c]) continue;
        const double r = minv + cost(i, c) - ui - C.dual[c];
        if (r < C.shortest[c]) { C.path[c] = i; C.shortest[c] = r; }
        const int busy = C.mate[c] >= 0;
        if (me_better(C.shortest[c], busy, c, lo, lb, lk)) { lo = C.shortest[c]; lb = busy; lk = c; }
      }
      if (kTeam) {
#if defined(__CUDACC__)
        for (int sh_off = 16; sh_off > 0; sh_off >>= 1) {          // warp argmin, then one entry per warp
          const double v = __shfl_xor_sync(0xffffffffu, lo, sh_off);
          const int bb = __shfl_xor_sync(0xffffffffu, lb, sh_off), kk = __shfl_xor_sync(0xffffffffu, lk, sh_off);
          if (me_better(v, bb, kk, lo, lb, lk)) { lo = v; lb = bb; lk = kk; }
        }
        const int slot = t0 >> 5, n_slots = (nt + 31) >> 5;
        if ((t0 & 31) == 0) { sh.red_v[slot] = lo; sh.red_b[slot] = lb; sh.red_k[slot] = lk; }
#else
        const int slot = t0, n_slots = nt;
        sh.red_v[slot] = lo; sh.red_b[slot] = lb; sh.red_k[slot] = lk;
#endif
        ME_SYNC();
        if (t0 == 0) {
          for (int t = 1; t < n_slots; ++t)
            if (me_better(sh.red_v[t], sh.red_b[t], sh.red_k[t], lo, lb, lk)) {
              lo = sh.red_v[t]; lb = sh.red_b[t]; lk = sh.red_k[t];
            }
          C.flag[lk] = 1;
          sh.ctl_min = lo;
          sh.ctl_sink = C.mate[lk] < 0 ? lk : -1;
          sh.ctl_i = C.mate[lk];
        }
        ME_SYNC();
        minv = sh.ctl_min; sink = sh.ctl_sink; i = sh.ctl_i;
      } else {
        C.flag[lk] = 1;
        minv = lo;
        if (C.mate[lk] < 0) sink = lk; else i = C.mate[lk];
      }
    }
    for (int r = t0; r < a; r += nt)
      if (R.flag[r] && r != cur) R.dual[r] += minv - C.shortest[R.mate[r]];
    for (int c = t0; c < b; c += nt)
      if (C.flag[c]) C.dual[c] -= minv - C.shortest[c];
    if (kTeam) ME_SYNC();
    if (t0 == 0) {
      R.dual[cur] += minv;
      for (int j = sink;;) {
        const int r = C.path[j];
        C.mate[j] = r;
        const int next = R.mate[r];
        R.mate[r] = j;
        j = next;
        if (r == cur) break;
      }
    }
    if (kTeam) ME_SYNC();
  }
}

// the sequence whose range of `field` (kFrameBegin or kGtBegin) holds v; sequences are stored in order
ME_FN int me_seq_of(const Params& P, int field, int64_t v) {
  int lo = 0, hi = P.S - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (P.seq[int64_t(mid) * kSeqFields + field] <= v) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- per sequence: zero the state ----
ME_FN void me_init_seq(const Params& P, int s) {
  const int64_t* q = P.seq + int64_t(s) * kSeqFields;
  const int64_t gb = q[kGtBegin], G = q[kGtCount], tb = q[kTrkBegin], H = q[kTrkCount];
  for (int k = ME_TID; k < kOutSlots; k += ME_NT) P.out[int64_t(s) * kOutSlots + k] = 0;
  for (int64_t g = ME_TID; g < G; g += ME_NT) {
    P.m[gb + g] = -1; P.present[gb + g] = 0; P.tracked[gb + g] = 0; P.fstate[gb + g] = 0;
  }
  for (int64_t h = ME_TID; h < H; h += ME_NT) P.hslot[tb + h] = -1;
  int32_t* lab = P.idlabel + gb + tb;
  for (int64_t n = ME_TID; n < G + H; n += ME_NT) lab[n] = int32_t(n);
  for (int64_t g = ME_TID; g < G; g += ME_NT) { P.id_nr[gb + g] = 0; P.id_nc[gb + g] = 0; }
}

// ---- per frame: valid pairs ----
template <bool kWrite>
ME_FN void me_pairs_frame(const Params& P, int f, Shared& sh) {
  if (kWrite && P.foff[P.F] > P.pair_cap) return;
  const int ob = P.fobj[f], no = P.fobj[f + 1] - ob, hb = P.fhyp[f], nh = P.fhyp[f + 1] - hb;
  int64_t b, e;
  me_chunk(int64_t(no) * nh, b, e);
  int64_t cnt = 0;
  for (int64_t k = b; k < e; ++k)
    cnt += me_valid(me_dist(P.obj_box + 4 * (ob + k / nh), P.hyp_box + 4 * (hb + k % nh)));
  int64_t at = me_scan_parts(sh, cnt);
  if (!kWrite) {
    if (ME_TID == 0) P.fcount[f] = int32_t(sh.base);
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
    me_atomic_add(tp + int64_t(P.obj_id[o]) * H + P.hyp_id[h], 1);
  }
}

// ---- one CTA: frame offsets; flags every sequence when the pair buffer is too small ----
ME_FN void me_scan(const Params& P, Shared& sh) {
  int64_t b, e;
  me_chunk(P.F, b, e);
  int64_t v = 0;
  for (int64_t f = b; f < e; ++f) v += P.fcount[f];
  int64_t at = me_scan_parts(sh, v);
  for (int64_t f = b; f < e; ++f) { P.foff[f] = at; at += P.fcount[f]; }
  if (ME_TID == 0) P.foff[P.F] = sh.base;
  ME_SYNC();
  for (int s = ME_TID; s < P.S; s += ME_NT) {
    const int64_t* q = P.seq + int64_t(s) * kSeqFields;
    int64_t* out = P.out + int64_t(s) * kOutSlots;
    out[kPairs] = P.foff[q[kFrameEnd]] - P.foff[q[kFrameBegin]];
    if (sh.base > P.pair_cap) out[kStatus] |= kErrPairCapacity;
  }
}

// pair index of (frame-local object o, global hypothesis row h) in o's row of the frame's pairs, or -1
ME_FN int64_t me_find(const Params& P, const int32_t* rb, const int32_t* re, int64_t pb, int o, int h) {
  int64_t lo = pb + rb[o], hi = pb + re[o];
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (P.pair_h[mid] < h) lo = mid + 1; else hi = mid;
  }
  return lo < pb + re[o] && P.pair_h[lo] == h ? lo : -1;
}

struct ClearCost {
  const Params* P; const int32_t *rows, *cols, *rb, *re; int64_t pb; int hb; bool tr; double big;
  ME_MFN double operator()(int r, int c) const {
    const int o = tr ? cols[c] : rows[r], h = tr ? rows[r] : cols[c];
    const int64_t k = me_find(*P, rb, re, pb, o, hb + h);
    return k >= 0 ? P->pair_d[k] : big;
  }
};

// ---- per sequence: MOTAccumulator.update over the frames, then the per-GT-id counts ----
ME_FN void me_clear_seq(const Params& P, int s, Shared& sh) {
  const int64_t* q = P.seq + int64_t(s) * kSeqFields;
  int64_t* out = P.out + int64_t(s) * kOutSlots;
  if (out[kStatus] & kErrPairCapacity) return;
  const int64_t gb = q[kGtBegin], G = q[kGtCount], tb = q[kTrkBegin];
  const int64_t so = int64_t(s) * P.max_obj, sq = int64_t(s) * P.max_hyp;
  double* odual = P.o_dual + so; double* oshort = P.o_short + so; double* odev = P.o_dev + so;
  int32_t *opath = P.o_path + so, *omate = P.o_mate + so, *olab = P.o_label + so, *olist = P.o_list + so;
  int32_t *ocand = P.o_cand + so, *orb = P.o_rb + so, *ore = P.o_re + so, *oca = P.o_ca + so, *ocb = P.o_cb + so;
  int32_t *ooa = P.o_oa + so, *oob = P.o_ob + so, *ostate = P.o_state + so;
  uint8_t *oflag = P.o_flag + so, *omask = P.o_mask + so;
  double* hdual = P.h_dual + sq; double* hshort = P.h_short + sq;
  int32_t *hpath = P.h_path + sq, *hmate = P.h_mate + sq, *hlab = P.h_label + sq, *hlist = P.h_list + sq;
  int32_t* hwin = P.h_win + sq;
  uint8_t *hflag = P.h_flag + sq, *hmask = P.h_mask + sq;
  if (ME_TID == 0) {
    sh.err = 0; sh.n_match = sh.n_switch = sh.n_miss = sh.n_fp = sh.n_frag = sh.n_mt = sh.n_pt = sh.n_ml = 0;
    sh.max_rows = sh.max_cols = 0;
  }
  double sumd = 0.0;
  for (int64_t f = q[kFrameBegin]; f < q[kFrameEnd]; ++f) {
    const int ob = P.fobj[f], no = P.fobj[f + 1] - ob, hb = P.fhyp[f], nh = P.fhyp[f + 1] - hb;
    const int64_t pb = P.foff[f], np = P.foff[f + 1] - pb;
    if (no > P.max_obj || nh > P.max_hyp) {
      if (ME_TID == 0) out[kStatus] |= kErrFrameSize;
      return;
    }
    for (int o = ME_TID; o < no; o += ME_NT) {
      omask[o] = 0; odev[o] = 0.0; ostate[o] = 0; orb[o] = ore[o] = 0; olab[o] = o; ocand[o] = -1;
    }
    for (int h = ME_TID; h < nh; h += ME_NT) {
      hmask[h] = 0; hwin[h] = INT_MAX; hlab[h] = no + h; P.hslot[tb + P.hyp_id[hb + h]] = h;
    }
    ME_SYNC();
    for (int64_t k = ME_TID; k < np; k += ME_NT) {          // pairs are row-major: each object's row is contiguous
      const int32_t o = P.pair_o[pb + k];
      if (k == 0 || P.pair_o[pb + k - 1] != o) orb[o - ob] = int32_t(k);
      if (k == np - 1 || P.pair_o[pb + k + 1] != o) ore[o - ob] = int32_t(k + 1);
    }
    ME_SYNC();
    if (np > 0) {
      // re-establish: object o keeps its previous partner if present and valid; the first object in order wins it
      for (int o = ME_TID; o < no; o += ME_NT) {
        const int32_t p = P.m[gb + P.obj_id[ob + o]];
        if (p < 0) continue;
        const int32_t j = P.hslot[tb + p];
        if (j >= 0 && me_find(P, orb, ore, pb, o, hb + j) >= 0) { ocand[o] = j; me_atomic_min(hwin + j, o); }
      }
      ME_SYNC();
      for (int o = ME_TID; o < no; o += ME_NT) {
        const int j = ocand[o];
        if (j < 0 || hwin[j] != o) continue;
        omask[o] = 1; hmask[j] = 1; ostate[o] = 1;
        odev[o] = P.pair_d[me_find(P, orb, ore, pb, o, hb + j)];
      }
      ME_SYNC();
      // connected components of the residual valid pairs: every node ends labelled with its component's least node
      for (;;) {
        if (ME_TID == 0) sh.changed = 0;
        ME_SYNC();
        for (int64_t k = ME_TID; k < np; k += ME_NT) {
          const int o = P.pair_o[pb + k] - ob, h = P.pair_h[pb + k] - hb;
          if (omask[o] || hmask[h]) continue;
          const int la = olab[o], lb = hlab[h];
          if (la != lb) {
            const int mn = la < lb ? la : lb;
            me_atomic_min(olab + o, mn); me_atomic_min(hlab + h, mn);
            sh.changed = 1;
          }
        }
        ME_SYNC();
        for (int x = ME_TID; x < no + nh; x += ME_NT) {
          int32_t* lx = x < no ? olab + x : hlab + (x - no);
          const int l = *lx, ll = l < no ? olab[l] : hlab[l - no];
          if (ll < l) me_atomic_min(lx, ll);
        }
        ME_SYNC();
        const int again = sh.changed;
        ME_SYNC();
        if (!again) break;
      }
      // a component with an edge holds an object, so its label is an object: size it from its root
      for (int o = ME_TID; o < no; o += ME_NT) {
        int a = 0, b = 0;
        if (!omask[o] && olab[o] == o) {
          for (int x = 0; x < no; ++x) a += !omask[x] && olab[x] == o;
          for (int y = 0; y < nh; ++y) b += !hmask[y] && hlab[y] == o;
        }
        oca[o] = b > 0 ? a : 0; ocb[o] = b;
      }
      ME_SYNC();                                            // written with a thread stride, read by chunk below
      int64_t cb0, ce0;
      me_chunk(no, cb0, ce0);
      int64_t va = 0, vb = 0;
      for (int64_t o = cb0; o < ce0; ++o) { va += oca[o]; vb += ocb[o]; }
      int64_t xa = me_scan_parts(sh, va), xb = me_scan_parts(sh, vb);
      for (int64_t o = cb0; o < ce0; ++o) { ooa[o] = int32_t(xa); oob[o] = int32_t(xb); xa += oca[o]; xb += ocb[o]; }
      ME_SYNC();
      for (int o = ME_TID; o < no; o += ME_NT) {
        const int a = oca[o], b = ocb[o];
        if (b == 0) continue;
        me_atomic_max(&sh.max_rows, a); me_atomic_max(&sh.max_cols, b);
        if (a > kMaxClearSide || b > kMaxClearSide) { sh.err = 1; continue; }
        int32_t *rl = olist + ooa[o], *cl = hlist + oob[o];
        for (int x = 0, n = 0; x < no; ++x) if (!omask[x] && olab[x] == o) rl[n++] = x;
        for (int y = 0, n = 0; y < nh; ++y) if (!hmask[y] && hlab[y] == o) cl[n++] = y;
        const LsaSide os{odual + ooa[o], oshort + ooa[o], opath + ooa[o], omate + ooa[o], oflag + ooa[o]};
        const LsaSide hs{hdual + oob[o], hshort + oob[o], hpath + oob[o], hmate + oob[o], hflag + oob[o]};
        const bool tr = a > b;
        const int r = tr ? b : a;
        // motmetrics' add_expensive_edges: an invalid pair costs more than any two valid matchings differ by
        const ClearCost cost{&P, tr ? cl : rl, tr ? rl : cl, orb, ore, pb, hb, tr, 2.0 * r * (0.5 + 1.0) + 1.0};
        me_lsa<false>(r, tr ? a : b, cost, tr ? hs : os, tr ? os : hs, sh);
        for (int i = 0; i < r; ++i) {
          const int x = tr ? rl[hs.mate[i]] : rl[i], y = tr ? cl[i] : cl[os.mate[i]];
          const int64_t k = me_find(P, orb, ore, pb, x, hb + y);
          if (k < 0) continue;                              // an expensive edge: not a match
          const int gi = int(gb + P.obj_id[ob + x]), hid = P.hyp_id[hb + y], prev = P.m[gi];
          ostate[x] = prev >= 0 && prev != hid ? 2 : 1;
          P.m[gi] = hid;
          odev[x] = P.pair_d[k];
          omask[x] = 1; hmask[y] = 1;
        }
      }
      ME_SYNC();
      if (sh.err) {
        if (ME_TID == 0) {
          out[kStatus] |= kErrClearComponent;
          out[kClearRows] = sh.max_rows;
          out[kClearCols] = sh.max_cols;
        }
        return;
      }
    }
    // events: MATCH / SWITCH / MISS per object, FP per unmatched hypothesis
    for (int o = ME_TID; o < no; o += ME_NT) {
      const int gi = int(gb + P.obj_id[ob + o]), st = ostate[o];
      int fs = P.fstate[gi];                              // bit 0: tracked before; bit 1: missed since then
      ++P.present[gi];
      if (st) {
        ++P.tracked[gi];
        me_atomic_add(st == 2 ? &sh.n_switch : &sh.n_match, 1);
        if (fs & 2) me_atomic_add(&sh.n_frag, 1);
        fs = 1;
      } else {
        me_atomic_add(&sh.n_miss, 1);
        if (fs & 1) fs |= 2;
      }
      P.fstate[gi] = fs;
    }
    for (int h = ME_TID; h < nh; h += ME_NT) {
      if (!hmask[h]) me_atomic_add(&sh.n_fp, 1);
      P.hslot[tb + P.hyp_id[hb + h]] = -1;
    }
    int64_t db, de;
    me_chunk(no, db, de);
    double part = 0.0;
    for (int64_t o = db; o < de; ++o) part += odev[o];
    sumd += me_sum_ordered(sh, part);
  }
  for (int64_t g = ME_TID; g < G; g += ME_NT) {
    const int64_t pr = P.present[gb + g], tr = P.tracked[gb + g];
    if (pr == 0) continue;
    if (5 * tr >= 4 * pr) me_atomic_add(&sh.n_mt, 1);          // tracked ratio >= 0.8
    else if (5 * tr < pr) me_atomic_add(&sh.n_ml, 1);          // < 0.2
    else me_atomic_add(&sh.n_pt, 1);
  }
  ME_SYNC();
  if (ME_TID == 0) {
    out[kMatches] = sh.n_match; out[kSwitches] = sh.n_switch; out[kMisses] = sh.n_miss; out[kFalsePos] = sh.n_fp;
    out[kFrag] = sh.n_frag; out[kMostly] = sh.n_mt; out[kPartly] = sh.n_pt; out[kLost] = sh.n_ml;
    out[kClearRows] = sh.max_rows; out[kClearCols] = sh.max_cols;
    double* sd = reinterpret_cast<double*>(out + kSumD);
    *sd = sumd;
  }
}

// ---- per sequence: connected components of the tp graph (nodes: GT ids, then track ids) ----
ME_FN void me_id_label(const Params& P, int s, Shared& sh) {
  const int64_t* q = P.seq + int64_t(s) * kSeqFields;
  if (P.out[int64_t(s) * kOutSlots + kStatus] & kErrPairCapacity) return;
  const int64_t G = q[kGtCount], H = q[kTrkCount];
  int32_t* lab = P.idlabel + q[kGtBegin] + q[kTrkBegin];
  const int64_t pb = P.foff[q[kFrameBegin]], pe = P.foff[q[kFrameEnd]];
  for (;;) {
    if (ME_TID == 0) sh.changed = 0;
    ME_SYNC();
    for (int64_t k = pb + ME_TID; k < pe; k += ME_NT) {
      const int64_t a = P.obj_id[P.pair_o[k]], b = G + P.hyp_id[P.pair_h[k]];
      const int la = lab[a], lb = lab[b];
      if (la != lb) {
        const int mn = la < lb ? la : lb;
        me_atomic_min(lab + a, mn); me_atomic_min(lab + b, mn);
        sh.changed = 1;
      }
    }
    ME_SYNC();
    for (int64_t x = ME_TID; x < G + H; x += ME_NT) {
      const int l = lab[x], ll = lab[l];
      if (ll < l) me_atomic_min(lab + x, ll);
    }
    ME_SYNC();
    const int again = sh.changed;
    ME_SYNC();
    if (!again) break;
  }
  // members per component root (a GT id: every edge has one) and the offsets of its member lists
  int32_t *nr = P.id_nr + q[kGtBegin], *nc = P.id_nc + q[kGtBegin];
  for (int64_t x = ME_TID; x < G + H; x += ME_NT) {
    const int l = lab[x];
    if (l < G) me_atomic_add(x < G ? nr + l : nc + l, 1);
  }
  ME_SYNC();
  int64_t b, e;
  me_chunk(G, b, e);
  int64_t vr = 0, vc = 0;
  for (int64_t g = b; g < e; ++g) { vr += nr[g]; vc += nc[g]; }
  int64_t xr = me_scan_parts(sh, vr), xc = me_scan_parts(sh, vc);
  int32_t *orr = P.id_or + q[kGtBegin], *occ = P.id_oc + q[kGtBegin];
  for (int64_t g = b; g < e; ++g) { orr[g] = int32_t(xr); occ[g] = int32_t(xc); xr += nr[g]; xc += nc[g]; }
}

// ordered compaction of the nodes [0, n) labelled root into list; returns their count (nothing written above cap)
ME_FN int me_gather(const int32_t* lab, int64_t n, int root, int32_t* list, int cap, Shared& sh) {
  int64_t b, e;
  me_chunk(n, b, e);
  int64_t c = 0;
  for (int64_t x = b; x < e; ++x) c += lab[x] == root;
  int64_t at = me_scan_parts(sh, c);
  const int64_t total = sh.base;
  if (total <= cap)
    for (int64_t x = b; x < e; ++x)
      if (lab[x] == root) list[at++] = int32_t(x);
  ME_SYNC();
  return int(total);
}

struct IdCost {
  const int32_t* tp; const int32_t *rows, *cols; int64_t H; bool tr;
  ME_MFN double operator()(int r, int c) const {
    const int64_t g = tr ? cols[c] : rows[r], h = tr ? rows[r] : cols[c];
    return -double(tp[g * H + h]);
  }
};

// ---- per GT id k (global index): if it roots a component of the tp graph, its maximum-weight matching ----
ME_FN void me_id_comp(const Params& P, int64_t k, Shared& sh) {
  const int s = me_seq_of(P, kGtBegin, k);
  const int64_t* q = P.seq + int64_t(s) * kSeqFields;
  int64_t* out = P.out + int64_t(s) * kOutSlots;
  if (out[kStatus] & kErrPairCapacity) return;
  const int64_t G = q[kGtCount], H = q[kTrkCount], g = k - q[kGtBegin];
  const int64_t gb = q[kGtBegin], tb = q[kTrkBegin];
  const int32_t* lab = P.idlabel + gb + tb;
  const int a = P.id_nr[gb + g], b = P.id_nc[gb + g];
  if (lab[g] != g || b == 0) return;                      // not a root, or a GT id no track ever covered
  if (ME_TID == 0) { me_max64(out + kIdRows, a); me_max64(out + kIdCols, b); }
  if ((a < b ? a : b) > kMaxIdSmall || (a < b ? b : a) > kMaxIdLarge) {
    if (ME_TID == 0) me_or64(out + kStatus, kErrIdComponent);
    return;
  }
  const int64_t orr = gb + P.id_or[gb + g], occ = tb + P.id_oc[gb + g];
  me_gather(lab, G, int(g), P.g_list + orr, a, sh);
  me_gather(lab + G, H, int(g), P.t_list + occ, b, sh);
  const LsaSide gs{P.g_dual + orr, P.g_short + orr, P.g_path + orr, P.g_mate + orr, P.g_flag + orr};
  const LsaSide ts{P.t_dual + occ, P.t_short + occ, P.t_path + occ, P.t_mate + occ, P.t_flag + occ};
  const bool tr = a > b;
  const LsaSide &rs = tr ? ts : gs, &cs = tr ? gs : ts;
  const IdCost cost{P.tp + q[kTpBegin], tr ? P.t_list + occ : P.g_list + orr, tr ? P.g_list + orr : P.t_list + occ,
                    H, tr};
  me_lsa<true>(tr ? b : a, tr ? a : b, cost, rs, cs, sh);
  if (ME_TID == 0) {
    int64_t idtp = 0;
    for (int r = 0; r < (tr ? b : a); ++r) idtp -= int64_t(cost(r, rs.mate[r]));
    me_add64(out + kIdtp, idtp);
  }
}

}  // namespace tfb200_mot
