// TEST-ONLY host build of the MOTS evaluation: the very routines csrc/mots_eval.cu's kernels are compiled from
// (trackformer_b200/csrc/mots_eval_core.h, feeding mot_eval_core.h), each CTA run in turn by one "thread" and the
// segmented sort done by std::stable_sort, so the CPU suite can compare the device algorithm with the oracle of
// tests/mots_eval_reference.py.  Built by tests/test_mots_eval_cpu.py; never shipped, never loaded by the package.
// Same arguments as tfb200_mots_eval, host memory, no stream.
#include <string.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "../../trackformer_b200/csrc/mots_eval_core.h"

using namespace tfb200_mots;

extern "C" size_t tfb200_mots_eval_host_workspace_bytes(int S, int F, int n_masks, int64_t n_gt, int64_t n_trk,
                                                        int64_t tp_cells, int max_obj, int max_hyp, int64_t pair_cap,
                                                        int64_t interval_cap, int64_t cells) {
  if (ms_check(S, F, n_masks, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap, interval_cap, cells)) return 0;
  MsParams p{};
  size_t at = 0;
  return ms_carve(p, nullptr, S, F, n_masks, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap, interval_cap, cells,
                  0, &at);
}

// ms_decode alone on one string of an H x W mask: returns the interval count (-1 for a bad string) and writes up to
// cap intervals [start, end) to iv
extern "C" int64_t tfb200_mots_decode_host(const uint8_t* chars, int64_t len, int H, int W, int32_t* iv, int64_t cap) {
  const int64_t seq[kSeqFields] = {0, 1, 0, 0, 0, 0, 0, 0};
  const int32_t hw[2] = {H, W}, mask[kMaskFields] = {0, 0, H, W};
  const int64_t str_off[2] = {0, len};
  int64_t xout[kMsSlots] = {};
  std::vector<int32_t> start(size_t(cap) + 1), end(size_t(cap) + 1), iv_idx(size_t(cap) + 1);
  int32_t icount = 0, area = 0, ioff[2] = {0, 0};
  MsParams p{};
  p.core.S = 1; p.core.F = 1; p.core.seq = seq;
  p.n_masks = 1; p.seq_hw = hw; p.mask = mask; p.str_off = str_off; p.chars = chars; p.xout = xout;
  p.icount = &icount; p.area = &area; p.ioff = ioff;
  p.istart = start.data(); p.iend = end.data(); p.ival = iv_idx.data();
  ms_decode<false>(p, 0);
  if (xout[kMsStatus]) return -1;
  ioff[1] = icount < cap ? icount : int32_t(cap);
  ms_decode<true>(p, 0);
  for (int32_t k = 0; k < ioff[1]; ++k) { iv[2 * k] = start[k]; iv[2 * k + 1] = end[k]; }
  return icount;
}

extern "C" int tfb200_mots_eval_host(const int64_t* seq, const int32_t* seq_hw, const int32_t* frame_mask,
                                     const int64_t* frame_cell, const int32_t* frame_obj, const int32_t* obj_id,
                                     const int32_t* mask, const int64_t* str_off, const uint8_t* chars, int S, int F,
                                     int n_masks, int64_t n_gt, int64_t n_trk, int64_t tp_cells, int max_obj,
                                     int max_hyp, int64_t pair_cap, int64_t interval_cap, int64_t cells,
                                     void* workspace, size_t workspace_bytes, int64_t* out) {
  if (int rc = ms_check(S, F, n_masks, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap, interval_cap, cells))
    return rc;
  MsParams p{};
  size_t sort_at = 0;
  if (workspace_bytes < ms_carve(p, static_cast<char*>(workspace), S, F, n_masks, n_gt, n_trk, tp_cells, max_obj,
                                 max_hyp, pair_cap, interval_cap, cells, 0, &sort_at))
    return TFB200_E_SHAPE;
  Params& c = p.core;
  c.S = S; c.F = F; c.max_obj = max_obj; c.max_hyp = max_hyp; c.pair_cap = pair_cap;
  c.seq = seq; c.fobj = frame_obj; c.obj_id = obj_id; c.fhyp = p.fhyp; c.hyp_id = p.hyp_id; c.out = out;
  p.n_masks = n_masks; p.icap = interval_cap; p.cells = cells;
  p.seq_hw = seq_hw; p.fm = frame_mask; p.fcell = frame_cell; p.mask = mask; p.str_off = str_off; p.chars = chars;
  p.xout = out + int64_t(S) * kOutSlots;
  static Shared sh;
  memset(c.tp, 0, size_t(tp_cells) * 4);
  memset(p.cell, 0, size_t(cells) * 4);
  for (int s = 0; s < S; ++s) ms_init_seq(p, s);
  for (int m = 0; m < n_masks; ++m) ms_decode<false>(p, m);
  ms_scan_masks(p, sh);
  for (int m = 0; m < n_masks; ++m) ms_decode<true>(p, m);
  const int64_t n = p.ioff[n_masks];
  std::vector<int32_t> idx(size_t(n), 0);
  for (int k = 0; k < 2 * F; ++k) {                 // each frame side by interval start
    std::iota(idx.begin() + p.segoff[k], idx.begin() + p.segoff[k + 1], p.segoff[k]);
    std::stable_sort(idx.begin() + p.segoff[k], idx.begin() + p.segoff[k + 1],
                     [&](int32_t a, int32_t b) { return p.istart[a] < p.istart[b]; });
  }
  for (int64_t k = 0; k < n; ++k) { p.sidx[k] = idx[size_t(k)]; p.sstart[k] = p.istart[idx[size_t(k)]]; }
  for (int64_t k = 0; k < n; ++k) ms_gather(p, k);
  for (int64_t k = 0; k < n; ++k) ms_intersect(p, k);
  for (int f = 0; f < F; ++f) ms_frame<false>(p, f, sh);
  ms_scan(p, sh);
  for (int f = 0; f < F; ++f) ms_frame<true>(p, f, sh);
  for (int s = 0; s < S; ++s) me_clear_seq(c, s, sh);
  for (int s = 0; s < S; ++s) me_id_label(c, s, sh);
  for (int64_t k = 0; k < n_gt; ++k) me_id_comp(c, k, sh);
  return 0;
}
