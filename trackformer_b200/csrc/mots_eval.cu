// MOTS metrics of many sequences on the device (sm_90a): the routines of mots_eval_core.h as two memsets (the tp
// matrices, the frames' intersection counts) and these launches -- state init, string count pass, interval offsets,
// string write pass, CUB's segmented sort of every frame side by interval start, sorted gather + overlap check,
// intersection, frame count pass, frame scan, frame write pass -- then mot_eval_core.h's CLEAR-MOT pass, tp-graph
// components and identity matching.  Nothing is read back here: the caller copies `out` once.
#include <cuda_runtime.h>

#include <cub/device/device_segmented_sort.cuh>

#include "launch_counter.h"
#include "mots_eval_core.h"

namespace {

using namespace tfb200_mots;

__global__ void __launch_bounds__(kThreads) ms_init_kernel(const __grid_constant__ MsParams p) {
  ms_init_seq(p, int(blockIdx.x));
}

template <bool kWrite>
__global__ void __launch_bounds__(kThreads) ms_decode_kernel(const __grid_constant__ MsParams p) {
  const int64_t m = int64_t(blockIdx.x) * kThreads + threadIdx.x;
  if (m < p.n_masks) ms_decode<kWrite>(p, int(m));
}

__global__ void __launch_bounds__(kThreads) ms_scan_masks_kernel(const __grid_constant__ MsParams p) {
  __shared__ Shared sh;
  ms_scan_masks(p, sh);
}

__global__ void __launch_bounds__(kThreads) ms_gather_kernel(const __grid_constant__ MsParams p) {
  ms_gather(p, int64_t(blockIdx.x) * kThreads + threadIdx.x);
}

__global__ void __launch_bounds__(kThreads) ms_intersect_kernel(const __grid_constant__ MsParams p) {
  ms_intersect(p, int64_t(blockIdx.x) * kThreads + threadIdx.x);
}

template <bool kWrite>
__global__ void __launch_bounds__(kThreads) ms_frame_kernel(const __grid_constant__ MsParams p) {
  __shared__ Shared sh;
  ms_frame<kWrite>(p, int(blockIdx.x), sh);
}

__global__ void __launch_bounds__(kThreads) ms_scan_kernel(const __grid_constant__ MsParams p) {
  __shared__ Shared sh;
  ms_scan(p, sh);
}

__global__ void __launch_bounds__(kThreads) ms_clear_kernel(const __grid_constant__ MsParams p) {
  __shared__ Shared sh;
  me_clear_seq(p.core, int(blockIdx.x), sh);
}

__global__ void __launch_bounds__(kThreads) ms_id_label_kernel(const __grid_constant__ MsParams p) {
  __shared__ Shared sh;
  me_id_label(p.core, int(blockIdx.x), sh);
}

__global__ void __launch_bounds__(kThreads) ms_id_comp_kernel(const __grid_constant__ MsParams p) {
  __shared__ Shared sh;
  me_id_comp(p.core, int64_t(blockIdx.x), sh);
}

size_t sort_bytes(int F, int64_t icap) {
  if (F == 0 || icap == 0) return 0;
  size_t bytes = 0;
  if (cub::DeviceSegmentedSort::SortPairs(nullptr, bytes, static_cast<const int32_t*>(nullptr),
                                          static_cast<int32_t*>(nullptr), static_cast<const int32_t*>(nullptr),
                                          static_cast<int32_t*>(nullptr), int(icap), 2 * F,
                                          static_cast<const int32_t*>(nullptr), static_cast<const int32_t*>(nullptr)))
    return 0;
  return bytes ? bytes : 1;
}

unsigned blocks(int64_t n) { return unsigned((n + kThreads - 1) / kThreads); }

}  // namespace

extern "C" size_t tfb200_mots_eval_workspace_bytes(int S, int F, int n_masks, int64_t n_gt, int64_t n_trk,
                                                   int64_t tp_cells, int max_obj, int max_hyp, int64_t pair_cap,
                                                   int64_t interval_cap, int64_t cells) {
  if (ms_check(S, F, n_masks, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap, interval_cap, cells)) return 0;
  MsParams p{};
  size_t at = 0;
  return ms_carve(p, nullptr, S, F, n_masks, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap, interval_cap, cells,
                  sort_bytes(F, interval_cap), &at);
}

extern "C" int tfb200_mots_eval(const int64_t* seq, const int32_t* seq_hw, const int32_t* frame_mask,
                                const int64_t* frame_cell, const int32_t* frame_obj, const int32_t* obj_id,
                                const int32_t* mask, const int64_t* str_off, const uint8_t* chars, int S, int F,
                                int n_masks, int64_t n_gt, int64_t n_trk, int64_t tp_cells, int max_obj, int max_hyp,
                                int64_t pair_cap, int64_t interval_cap, int64_t cells, void* workspace,
                                size_t workspace_bytes, int64_t* out, void* stream) {
  if (!seq || !seq_hw || !frame_mask || !frame_cell || !frame_obj || !obj_id || !mask || !str_off || !chars ||
      !workspace || !out)
    return TFB200_E_NULLPTR;
  if (int rc = ms_check(S, F, n_masks, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap, interval_cap, cells))
    return rc;
  MsParams p{};
  size_t sort_at = 0;
  const size_t sbytes = sort_bytes(F, interval_cap);
  if (workspace_bytes < ms_carve(p, static_cast<char*>(workspace), S, F, n_masks, n_gt, n_trk, tp_cells, max_obj,
                                 max_hyp, pair_cap, interval_cap, cells, sbytes, &sort_at))
    return TFB200_E_SHAPE;
  Params& c = p.core;
  c.S = S; c.F = F; c.max_obj = max_obj; c.max_hyp = max_hyp; c.pair_cap = pair_cap;
  c.seq = seq; c.fobj = frame_obj; c.obj_id = obj_id; c.fhyp = p.fhyp; c.hyp_id = p.hyp_id; c.out = out;
  p.n_masks = n_masks; p.icap = interval_cap; p.cells = cells;
  p.seq_hw = seq_hw; p.fm = frame_mask; p.fcell = frame_cell; p.mask = mask; p.str_off = str_off; p.chars = chars;
  p.xout = out + int64_t(S) * kOutSlots;
  const cudaStream_t s = cudaStream_t(stream);
  if (tp_cells > 0)
    if (cudaError_t e = cudaMemsetAsync(c.tp, 0, size_t(tp_cells) * 4, s)) return int(e);
  if (cells > 0)
    if (cudaError_t e = cudaMemsetAsync(p.cell, 0, size_t(cells) * 4, s)) return int(e);
  int launches = 7;
  ms_init_kernel<<<S, kThreads, 0, s>>>(p);
  if (n_masks > 0) {
    ms_decode_kernel<false><<<blocks(n_masks), kThreads, 0, s>>>(p);
    ++launches;
  }
  ms_scan_masks_kernel<<<1, kThreads, 0, s>>>(p);
  if (n_masks > 0 && interval_cap > 0) {
    ms_decode_kernel<true><<<blocks(n_masks), kThreads, 0, s>>>(p);
    size_t tb = sbytes;
    if (cudaError_t e = cub::DeviceSegmentedSort::SortPairs(static_cast<char*>(workspace) + sort_at, tb, p.istart,
                                                            p.sstart, p.ival, p.sidx, int(interval_cap), 2 * F,
                                                            p.segoff, p.segoff + 1, s))
      return int(e);
    ms_gather_kernel<<<blocks(interval_cap), kThreads, 0, s>>>(p);
    ms_intersect_kernel<<<blocks(interval_cap), kThreads, 0, s>>>(p);
    launches += 4;
  }
  if (F > 0) {
    ms_frame_kernel<false><<<F, kThreads, 0, s>>>(p);
    ms_scan_kernel<<<1, kThreads, 0, s>>>(p);
    ms_frame_kernel<true><<<F, kThreads, 0, s>>>(p);
  } else {
    ms_scan_kernel<<<1, kThreads, 0, s>>>(p);
    launches -= 2;
  }
  ms_clear_kernel<<<S, kThreads, 0, s>>>(p);
  ms_id_label_kernel<<<S, kThreads, 0, s>>>(p);
  if (n_gt > 0) {
    ms_id_comp_kernel<<<unsigned(n_gt), kThreads, 0, s>>>(p);
    ++launches;
  }
  msda_b200_count_launches(launches);
  return int(cudaGetLastError());
}
