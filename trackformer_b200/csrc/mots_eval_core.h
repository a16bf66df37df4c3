// MOTS metrics (sMOTSA, MOTSA, MOTSP and the CLEAR-MOT / identity counts) from the masks' COCO RLE strings, written
// once as routines that feed the pairs of mot_eval_core.h:
//
//   ms_init_seq   (one CTA per sequence)   me_init_seq, plus this file's per-sequence slots
//   ms_decode     (one thread per mask)    validate a counts string (mots.decode_counts is the specification) and
//                                          count its foreground intervals; then write them, [start, end) of the
//                                          column-major pixel index
//   ms_scan_masks (one CTA)                interval offsets per mask, and the two segments of every frame (GT and
//                                          ignore masks; hypotheses) that the caller sorts by interval start
//   ms_gather     (one thread per sorted interval)  end and GT row of each sorted interval; neighbours that overlap
//                                          are masks of one side that overlap: an error
//   ms_intersect  (one thread per hypothesis interval)  binary search in the frame's sorted GT-side intervals and add
//                                          every overlap to the frame's [GT rows + ignore][hypotheses] counts
//   ms_frame      (one CTA per frame)      candidates (inter > 0, 2 inter >= union) and the ignore rule; count, or
//                                          write the kept hypotheses and the valid pairs row-major with their tp
//   ms_scan       (one CTA)                me_scan, and the kept hypotheses' frame offsets
//
// after which mot_eval_core.h's me_clear_seq / me_id_label / me_id_comp run unchanged.  Work scales with intervals,
// not pixels; every count is an exact integer and d = 1 - inter / union is one fp64 division and one subtraction.
// nvcc compiles them into csrc/mots_eval.cu's kernels (the sort: CUB), g++ (one "thread", std::stable_sort) into the
// test-only host build tests/host_build/mots_eval_host.cpp.
#pragma once

#include "mot_eval_core.h"

namespace tfb200_mots {

using namespace tfb200_mot;

constexpr int64_t kMaxPixels = int64_t(1) << 28;     // H x W of a mask: interval ends fit int32
constexpr int kMaxValueChars = 7;                    // 35 bits: any count difference of a mask under kMaxPixels

// per-mask table (int32 [n_masks][kMaskFields])
enum { kMaskFrame, kMaskId, kMaskH, kMaskW, kMaskFields = 4 };
// frame table (int32 [3 F + 1]): frame f's GT masks are rows fm[3f] .., ignore masks fm[3f + 1] .., hypotheses
// fm[3f + 2] .. fm[3f + 3]
enum { kSideGt, kSideIgnore, kSideHyp };

// per-sequence slots after mot_eval's [S][kOutSlots] (8 bytes each)
enum {
  kMsStatus, kMsGtDets, kMsKept, kMsRemoved, kMsIntervals, kMsIntersecting,
  kMsFirstFrame,                                       // kMsFirstFrame + b: first frame (sequence-local) of error bit b
  kMsSlots = kMsFirstFrame + 5
};
// status bits (kMsStatus)
enum { kMsErrOverlapGt = 1, kMsErrOverlapHyp = 2, kMsErrSize = 4, kMsErrRle = 8, kMsErrCapacity = 16 };

struct MsParams {
  Params core;                                       // seq, fobj, obj_id, out and the pair / tp workspace;
                                                     // fhyp and hyp_id point into this workspace
  int n_masks;
  int64_t icap, cells;
  const int32_t* seq_hw;                             // [S][2] H, W of the sequence
  const int32_t* fm;                                 // [3 F + 1]
  const int64_t* fcell;                              // [F + 1] frame f's counts: fcell[f] .., (GT rows + 1) x hyps
  const int32_t* mask;                               // [n_masks][kMaskFields]
  const int64_t* str_off;                            // [n_masks + 1]
  const uint8_t* chars;
  int64_t* xout;                                     // [S][kMsSlots]
  // workspace
  int32_t *icount, *area, *ioff;                     // [n_masks], [n_masks], [n_masks + 1]
  int32_t *keep;                                     // [n_masks]: 1 kept hypothesis, then its frame-local rank
  int32_t *segoff;                                   // [2 F + 1]
  int32_t *istart, *iend;                            // [icap] intervals in mask order
  int32_t *sstart, *sidx, *gs_end, *gs_row;          // [icap] sorted within each segment: start, source, end, row
  int32_t *ival;                                     // = gs_end: each interval's own index, the sort's values (read
                                                     // by the sort only, before ms_gather writes gs_end)
  int32_t *cell;                                     // [cells]
  int32_t *fcount_kept, *fhyp, *hyp_id;              // [F], [F + 1], [n_masks]
};

// Argument ranges: 0 or TFB200_E_SHAPE.
static inline int ms_check(int S, int F, int n_masks, int64_t n_gt, int64_t n_trk, int64_t tp_cells, int max_obj,
                           int max_hyp, int64_t pair_cap, int64_t icap, int64_t cells) {
  if (int rc = me_check(S, F, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap)) return rc;
  if (n_masks < 0 || icap < 0 || icap > INT32_MAX || cells < 0 || F > (INT32_MAX - 1) / 3) return TFB200_E_SHAPE;
  return 0;
}

// Carves the workspace after the core's (ws may be NULL to size it); returns the bytes of both.  `sort_bytes` is
// appended for the caller's segmented sort and returned in sort_at.
static inline size_t ms_carve(MsParams& p, char* ws, int S, int F, int n_masks, int64_t n_gt, int64_t n_trk,
                              int64_t tp_cells, int max_obj, int max_hyp, int64_t pair_cap, int64_t icap,
                              int64_t cells, size_t sort_bytes, size_t* sort_at) {
  size_t o = me_carve(p.core, ws, S, F, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap);
  auto take = [&](auto*& ptr, size_t n) {
    ptr = reinterpret_cast<std::remove_reference_t<decltype(ptr)>>(reinterpret_cast<uintptr_t>(ws) + o);
    o += (n * sizeof(*ptr) + 255) & ~size_t(255);
  };
  const size_t n = size_t(n_masks), ic = size_t(icap);
  for (int32_t** a : {&p.icount, &p.area, &p.keep, &p.hyp_id}) take(*a, n);
  take(p.ioff, n + 1);
  take(p.segoff, 2 * size_t(F) + 1);
  for (int32_t** a : {&p.istart, &p.iend, &p.sstart, &p.sidx, &p.gs_end, &p.gs_row}) take(*a, ic);
  p.ival = p.gs_end;
  take(p.cell, size_t(cells));
  take(p.fcount_kept, size_t(F));
  take(p.fhyp, size_t(F) + 1);
  *sort_at = o;
  return o + ((sort_bytes + 255) & ~size_t(255));
}

ME_FN void ms_min64(int64_t* p, int64_t v) {
#if defined(__CUDACC__)
  atomicMin(reinterpret_cast<long long*>(p), (long long)v);
#else
  if (v < *p) *p = v;
#endif
}

// error `bit` in frame f (global): the status bit and the first such frame of f's sequence
ME_FN void ms_flag(const MsParams& P, int64_t f, int bit) {
  const int s = me_seq_of(P.core, kFrameBegin, f);
  int64_t* x = P.xout + int64_t(s) * kMsSlots;
  me_or64(x + kMsStatus, bit);
  int b = 0;
  while ((1 << b) != bit) ++b;
  ms_min64(x + kMsFirstFrame + b, f - P.core.seq[int64_t(s) * kSeqFields + kFrameBegin]);
}

ME_FN int ms_side(const MsParams& P, int f, int m) {
  return m >= P.fm[3 * f + 2] ? kSideHyp : m >= P.fm[3 * f + 1] ? kSideIgnore : kSideGt;
}

// ---- per sequence ----
ME_FN void ms_init_seq(const MsParams& P, int s) {
  me_init_seq(P.core, s);
  int64_t* x = P.xout + int64_t(s) * kMsSlots;
  for (int k = ME_TID; k < kMsSlots; k += ME_NT) x[k] = k >= kMsFirstFrame ? INT64_MAX : 0;
}

// ---- per mask m: decode its counts string.  Count pass: icount / area (0 for a bad mask, with the error flagged);
// write pass: the intervals at ioff[m] .. ioff[m + 1] ----
template <bool kWrite>
ME_FN void ms_decode(const MsParams& P, int m) {
  const int32_t* mi = P.mask + int64_t(m) * kMaskFields;
  const int f = mi[kMaskFrame];
  int64_t at = 0, lim = 0;
  if (kWrite) {
    at = P.ioff[m]; lim = P.ioff[m + 1];
    if (at == lim) return;
  } else {
    P.icount[m] = 0; P.area[m] = 0;
    const int s = me_seq_of(P.core, kFrameBegin, f);
    const int64_t H = mi[kMaskH], W = mi[kMaskW];
    if (H != P.seq_hw[2 * s] || W != P.seq_hw[2 * s + 1] || H < 0 || W < 0 || H * W >= kMaxPixels) {
      ms_flag(P, f, kMsErrSize);
      return;
    }
  }
  const int64_t n = int64_t(mi[kMaskH]) * mi[kMaskW];
  const uint8_t* c = P.chars + P.str_off[m];
  const int64_t len = P.str_off[m + 1] - P.str_off[m];
  int64_t pos = 0, c1 = 0, c2 = 0, nint = 0, area = 0;
  bool bad = len == 0;
  for (int64_t j = 0, i = 0; j < len && !bad; ++i) {
    int64_t x = 0;
    int k = 0, v = 0;
    do {
      if (j >= len || k >= kMaxValueChars) { bad = true; break; }
      v = int(c[j++]) - 48;
      if (v < 0 || v > 63) { bad = true; break; }
      x |= int64_t(v & 0x1F) << (5 * k);
      ++k;
    } while (v & 0x20);
    if (bad) break;
    if (v & 0x10) x |= -(int64_t(1) << (5 * k));      // sign bit of the last group
    const int64_t cnt = i > 2 ? x + c2 : x;           // deltas against the count two back
    if (cnt < 0 || cnt > n - pos) { bad = true; break; }
    if ((i & 1) && cnt > 0) {
      if (kWrite) {
        if (at < lim) {
          P.istart[at] = int32_t(pos); P.iend[at] = int32_t(pos + cnt); P.ival[at] = int32_t(at);
          ++at;
        }
      } else {
        ++nint; area += cnt;
      }
    }
    pos += cnt; c2 = c1; c1 = cnt;
  }
  if (kWrite) return;
  if (bad || pos != n) {
    ms_flag(P, f, kMsErrRle);
    return;
  }
  P.icount[m] = int32_t(nint); P.area[m] = int32_t(area);
}

// ---- one CTA: interval offsets (all zero, capacity flagged everywhere, when they pass icap) and frame segments ----
ME_FN void ms_scan_masks(const MsParams& P, Shared& sh) {
  int64_t b, e;
  me_chunk(P.n_masks, b, e);
  int64_t v = 0;
  for (int64_t m = b; m < e; ++m) v += P.icount[m];
  int64_t at = me_scan_parts(sh, v);
  const bool over = sh.base > P.icap;
  for (int64_t m = b; m < e; ++m) { P.ioff[m] = over ? 0 : int32_t(at); at += P.icount[m]; }
  if (ME_TID == 0) P.ioff[P.n_masks] = over ? 0 : int32_t(sh.base);
  ME_SYNC();
  const int F = P.core.F;
  for (int f = ME_TID; f < F; f += ME_NT) {
    P.segoff[2 * f] = P.ioff[P.fm[3 * f]];
    P.segoff[2 * f + 1] = P.ioff[P.fm[3 * f + 2]];
  }
  if (ME_TID == 0) P.segoff[2 * F] = P.ioff[P.fm[3 * F]];
  for (int s = ME_TID; s < P.core.S; s += ME_NT) {
    const int64_t* q = P.core.seq + int64_t(s) * kSeqFields;
    int64_t* x = P.xout + int64_t(s) * kMsSlots;
    x[kMsIntervals] = P.ioff[P.fm[3 * q[kFrameEnd]]] - P.ioff[P.fm[3 * q[kFrameBegin]]];
    if (over) x[kMsStatus] |= kMsErrCapacity;
  }
}

// the mask holding interval k < ioff[n_masks]: the last m with ioff[m] <= k (empty masks share the next offset)
ME_FN int ms_mask_of(const MsParams& P, int64_t k) {
  int lo = 0, hi = P.n_masks - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (P.ioff[mid] <= k) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// ---- per sorted interval k: its end and GT row (the frame's GT count for an ignore mask); overlap with the previous
// interval of its segment ----
ME_FN void ms_gather(const MsParams& P, int64_t k) {
  if (k >= P.ioff[P.n_masks]) return;
  const int src = P.sidx[k], m = ms_mask_of(P, src), f = P.mask[int64_t(m) * kMaskFields + kMaskFrame];
  const int side = ms_side(P, f, m);
  P.gs_end[k] = P.iend[src];
  P.gs_row[k] = side == kSideGt ? m - P.fm[3 * f] : P.fm[3 * f + 1] - P.fm[3 * f];
  const int64_t sb = P.segoff[2 * f + (side == kSideHyp)];
  if (k > sb && P.sstart[k] < P.iend[P.sidx[k - 1]])
    ms_flag(P, f, side == kSideHyp ? kMsErrOverlapHyp : kMsErrOverlapGt);
}

// ---- per interval k (mask order): a hypothesis interval's overlaps with the frame's GT-side intervals ----
ME_FN void ms_intersect(const MsParams& P, int64_t k) {
  if (k >= P.ioff[P.n_masks]) return;
  const int m = ms_mask_of(P, k), f = P.mask[int64_t(m) * kMaskFields + kMaskFrame];
  if (ms_side(P, f, m) != kSideHyp) return;
  const int32_t s0 = P.istart[k], e0 = P.iend[k];
  int64_t lo = P.segoff[2 * f], hi = P.segoff[2 * f + 1];
  const int64_t end = hi;
  while (lo < hi) {                                  // first GT-side interval ending after s0 (ends ascend: disjoint)
    const int64_t mid = (lo + hi) >> 1;
    if (P.gs_end[mid] <= s0) lo = mid + 1; else hi = mid;
  }
  const int nh = P.fm[3 * f + 3] - P.fm[3 * f + 2], h = m - P.fm[3 * f + 2];
  int32_t* cell = P.cell + P.fcell[f];
  for (int64_t j = lo; j < end && P.sstart[j] < e0; ++j) {
    const int32_t a = P.sstart[j] > s0 ? P.sstart[j] : s0, b = P.gs_end[j] < e0 ? P.gs_end[j] : e0;
    if (b > a) me_atomic_add(cell + int64_t(P.gs_row[j]) * nh + h, b - a);
  }
}

// candidate pair: exact IoU >= 0.5 with a non-empty intersection
ME_FN bool ms_cand(int64_t inter, int64_t uni) { return inter > 0 && 2 * inter >= uni; }

// ---- per frame: candidates and the ignore rule.  Count pass: keep flags, fcount (valid pairs), kept hypotheses and
// the sequence's counters; write pass: kept hypotheses' track ids at their compacted rows, the valid pairs (object,
// then kept hypothesis) with d, and tp ----
template <bool kWrite>
ME_FN void ms_frame(const MsParams& P, int f, Shared& sh) {
  const Params& C = P.core;
  if (kWrite && C.foff[C.F] > C.pair_cap) return;
  const int gb = P.fm[3 * f], no = P.fm[3 * f + 1] - gb, hb = P.fm[3 * f + 2], nh = P.fm[3 * f + 3] - hb;
  const int32_t* cell = P.cell + P.fcell[f];
  const int32_t *ga = P.area + gb, *ha = P.area + hb;
  if (!kWrite) {
    int64_t kept = 0, inters = 0;
    for (int h = ME_TID; h < nh; h += ME_NT) {
      bool cand = false;
      for (int o = 0; o < no; ++o) {
        const int64_t in = cell[int64_t(o) * nh + h];
        inters += in > 0;
        cand |= ms_cand(in, int64_t(ga[o]) + ha[h] - in);
      }
      const int64_t ign = cell[int64_t(no) * nh + h];
      const int k = cand || !(2 * ign > ha[h]);
      P.keep[hb + h] = k;
      kept += k;
    }
    int64_t b, e;
    me_chunk(int64_t(no) * nh, b, e);
    int64_t cnt = 0;
    for (int64_t k = b; k < e; ++k) {
      const int64_t in = cell[k];
      cnt += ms_cand(in, int64_t(ga[k / nh]) + ha[k % nh] - in);
    }
    me_scan_parts(sh, cnt);
    const int64_t pairs = sh.base;
    me_scan_parts(sh, kept);
    const int64_t nk = sh.base;
    me_scan_parts(sh, inters);
    if (ME_TID == 0) {
      C.fcount[f] = int32_t(pairs);
      P.fcount_kept[f] = int32_t(nk);
      int64_t* x = P.xout + int64_t(me_seq_of(C, kFrameBegin, f)) * kMsSlots;
      me_add64(x + kMsGtDets, no);
      me_add64(x + kMsKept, nk);
      me_add64(x + kMsRemoved, nh - nk);
      me_add64(x + kMsIntersecting, sh.base);
    }
    return;
  }
  // kept hypotheses in order: rank within the frame, track id at the compacted row
  int64_t b, e;
  me_chunk(nh, b, e);
  int64_t v = 0;
  for (int64_t h = b; h < e; ++h) v += P.keep[hb + h];
  int64_t r = me_scan_parts(sh, v);
  for (int64_t h = b; h < e; ++h) {
    if (!P.keep[hb + h]) continue;
    P.keep[hb + h] = int32_t(1 + r);
    P.hyp_id[P.fhyp[f] + r] = P.mask[int64_t(hb + h) * kMaskFields + kMaskId];
    ++r;
  }
  ME_SYNC();
  me_chunk(int64_t(no) * nh, b, e);
  int64_t cnt = 0;
  for (int64_t k = b; k < e; ++k) {
    const int64_t in = cell[k];
    cnt += ms_cand(in, int64_t(ga[k / nh]) + ha[k % nh] - in);
  }
  int64_t at = me_scan_parts(sh, cnt) + C.foff[f];
  const int64_t* q = C.seq + int64_t(me_seq_of(C, kFrameBegin, f)) * kSeqFields;
  int32_t* tp = C.tp + q[kTpBegin];
  const int64_t H = q[kTrkCount];
  for (int64_t k = b; k < e; ++k) {
    const int o = int(k / nh), h = int(k % nh);
    const int64_t in = cell[k], uni = int64_t(ga[o]) + ha[h] - in;
    if (!ms_cand(in, uni)) continue;
    const int row = P.fhyp[f] + P.keep[hb + h] - 1;
    C.pair_o[at] = C.fobj[f] + o; C.pair_h[at] = row;
    C.pair_d[at] = me_sub(1.0, me_div(double(in), double(uni)));
    ++at;
    me_atomic_add(tp + int64_t(C.obj_id[C.fobj[f] + o]) * H + P.hyp_id[row], 1);
  }
}

// ---- one CTA: the pairs' frame offsets (me_scan) and the kept hypotheses' ----
ME_FN void ms_scan(const MsParams& P, Shared& sh) {
  me_scan(P.core, sh);
  int64_t b, e;
  me_chunk(P.core.F, b, e);
  int64_t v = 0;
  for (int64_t f = b; f < e; ++f) v += P.fcount_kept[f];
  int64_t at = me_scan_parts(sh, v);
  for (int64_t f = b; f < e; ++f) { P.fhyp[f] = int32_t(at); at += P.fcount_kept[f]; }
  if (ME_TID == 0) P.fhyp[P.core.F] = int32_t(sh.base);
  ME_SYNC();
}

}  // namespace tfb200_mots
