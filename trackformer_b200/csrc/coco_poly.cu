// COCO polygon segmentations as mask runs on the device (sm_90a): the routines of coco_poly_core.h as these launches.
//   count: sizes init, edge points (checks, point totals), edge toggle counts, CUB's scan of the toggle offsets, sizes
//          finish.  The caller reads sizes back: the toggle count sizes the second call's buffers.
//   runs:  edge toggle writes, annotation segments, CUB's segmented sort of every annotation's toggles, union sweep
//          counts, CUB's scan of the run offsets, union sweep writes.
//   rle:   one thread per compressed counts string.
//   masks: one thread per output byte.
// Nothing is read back here.
#include <cuda_runtime.h>

#include <cub/block/block_reduce.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_segmented_sort.cuh>

#include "coco_poly_core.h"
#include "launch_counter.h"

namespace {

using namespace tfb200_poly;

__global__ void __launch_bounds__(1) cp_init_kernel(int64_t* sizes, int n_ann, int32_t* toggle_off) {
  sizes[kSzPoints] = 0; sizes[kSzToggles] = 0; sizes[kSzStatus] = 0;
  sizes[kSzBadFinite] = n_ann; sizes[kSzBadRange] = n_ann;
  toggle_off[0] = 0;
}

__global__ void __launch_bounds__(kThreads) cp_points_kernel(const __grid_constant__ PolyParams P,
                                                             int64_t* ann_points, int64_t* sizes) {
  using Reduce = cub::BlockReduce<long long, kThreads>;
  __shared__ typename Reduce::TempStorage tmp;
  const int64_t e = int64_t(blockIdx.x) * kThreads + threadIdx.x;
  long long n = 0;
  if (e < P.n_edges) {
    int bad = 0, a = 0;
    n = cp_edge_points(P, e, &bad, &a);
    if (bad) {
      atomicOr(reinterpret_cast<unsigned long long*>(sizes + kSzStatus), (unsigned long long)bad);
      if (bad & 1) atomicMin(reinterpret_cast<long long*>(sizes + kSzBadFinite), (long long)a);
      if (bad & 2) atomicMin(reinterpret_cast<long long*>(sizes + kSzBadRange), (long long)a);
    }
    if (n) atomicAdd(reinterpret_cast<unsigned long long*>(ann_points + a), (unsigned long long)n);
  }
  const long long total = Reduce(tmp).Sum(n);
  if (threadIdx.x == 0 && total)
    atomicAdd(reinterpret_cast<unsigned long long*>(sizes + kSzPoints), (unsigned long long)total);
}

template <bool kWrite>
__global__ void __launch_bounds__(kThreads) cp_toggles_kernel(const __grid_constant__ PolyParams P, int32_t* count,
                                                              const int32_t* toggle_off, const int64_t* sizes,
                                                              uint32_t* key, int32_t* val) {
  const int64_t e = int64_t(blockIdx.x) * kThreads + threadIdx.x;
  if (e >= P.n_edges) return;
  if (kWrite) {
    cp_edge_toggles<true>(P, e, toggle_off[e], key, val);
  } else {
    const bool ok = sizes[kSzStatus] == 0 && sizes[kSzPoints] <= INT32_MAX;
    count[e] = ok ? int32_t(cp_edge_toggles<false>(P, e, 0, nullptr, nullptr)) : 0;
  }
}

__global__ void __launch_bounds__(1) cp_finish_kernel(int64_t n_edges, const int32_t* toggle_off, int64_t* sizes) {
  if (sizes[kSzPoints] > INT32_MAX) sizes[kSzStatus] |= 4;
  sizes[kSzToggles] = sizes[kSzStatus] ? 0 : toggle_off[n_edges];
}

__global__ void __launch_bounds__(kThreads) cp_segments_kernel(const __grid_constant__ PolyParams P,
                                                               const int32_t* toggle_off, int32_t* seg) {
  const int a = int(blockIdx.x) * kThreads + threadIdx.x;
  if (a <= P.n_ann) seg[a] = toggle_off[P.part_off[P.ann_part[a]]];
}

template <bool kWrite>
__global__ void __launch_bounds__(kThreads) cp_sweep_kernel(const __grid_constant__ PolyParams P, const int32_t* seg,
                                                            const uint32_t* key, const int32_t* val, uint8_t* par,
                                                            int64_t* nrun, const int64_t* run_off, uint32_t* runs) {
  const int a = int(blockIdx.x) * kThreads + threadIdx.x;
  if (a >= P.n_ann) return;
  if (kWrite) cp_sweep<true>(P, a, seg, key, val, par, runs + 2 * run_off[a]);
  else nrun[a] = cp_sweep<false>(P, a, seg, key, val, par, nullptr);
}

__global__ void __launch_bounds__(kThreads) cp_rle_kernel(const uint8_t* chars, const int64_t* str_off,
                                                          const int64_t* cap_off, int n, int64_t hw, int64_t* bounds,
                                                          uint32_t* runs, int64_t* first_bad) {
  const int k = int(blockIdx.x) * kThreads + threadIdx.x;
  if (k >= n) return;
  const uint8_t* c = chars + str_off[k];
  const int64_t len = str_off[k + 1] - str_off[k], at = cap_off[k];
  const int64_t m = cp_rle_decode<false>(c, len, hw, nullptr);
  if (m < 0) atomicMin(reinterpret_cast<long long*>(first_bad), (long long)k);
  else cp_rle_decode<true>(c, len, hw, runs + 2 * at);
  bounds[2 * k] = at;
  bounds[2 * k + 1] = at + (m < 0 ? 0 : m);
}

__global__ void __launch_bounds__(kThreads) cp_masks_kernel(const int32_t* src, int64_t total, int H, int W,
                                                            const int64_t* poly_run_off, const uint32_t* poly_runs,
                                                            const int64_t* rle_bounds, const uint32_t* rle_runs,
                                                            uint8_t* out) {
  for (int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x; i < total; i += int64_t(gridDim.x) * kThreads) {
    const int64_t plane = int64_t(H) * W, m = i / plane, r = i - m * plane;
    const int s = src[m];
    const uint32_t* run = s >= 0 ? poly_runs : rle_runs;
    const int64_t b = s >= 0 ? poly_run_off[s] : rle_bounds[2 * (-1 - s)];
    const int64_t e = s >= 0 ? poly_run_off[s + 1] : rle_bounds[2 * (-1 - s) + 1];
    out[i] = cp_mask_pixel(run, b, e, H, r / W, r % W);
  }
}

unsigned blocks(int64_t n) { return unsigned((n + kThreads - 1) / kThreads); }

size_t align(size_t n) { return (n + 255) & ~size_t(255); }

size_t count_scan_bytes(int64_t n_edges) {
  size_t bytes = 0;
  if (cub::DeviceScan::InclusiveSum(nullptr, bytes, static_cast<const int32_t*>(nullptr),
                                    static_cast<int32_t*>(nullptr), int(n_edges)))
    return 0;
  return bytes ? bytes : 1;
}

size_t runs_temp_bytes(int n_ann, int64_t n_toggles) {
  size_t sort = 0, scan = 0;
  if (n_toggles > 0 &&
      cub::DeviceSegmentedSort::SortPairs(nullptr, sort, static_cast<const uint32_t*>(nullptr),
                                          static_cast<uint32_t*>(nullptr), static_cast<const int32_t*>(nullptr),
                                          static_cast<int32_t*>(nullptr), int(n_toggles), n_ann,
                                          static_cast<const int32_t*>(nullptr), static_cast<const int32_t*>(nullptr)))
    return 0;
  if (cub::DeviceScan::InclusiveSum(nullptr, scan, static_cast<const int64_t*>(nullptr),
                                    static_cast<int64_t*>(nullptr), n_ann))
    return 0;
  const size_t b = sort > scan ? sort : scan;
  return b ? b : 1;
}

// the runs workspace: key, key_out, val, val_out [n_toggles], seg [n_ann + 1], par [n_parts], nrun [n_ann], temp
struct RunsWs {
  uint32_t *key, *key_out;
  int32_t *val, *val_out, *seg;
  uint8_t* par;
  int64_t* nrun;
  void* temp;
  size_t temp_bytes, total;
};

RunsWs carve_runs(char* ws, int n_parts, int n_ann, int64_t n_toggles) {
  RunsWs r{};
  size_t o = 0;
  auto take = [&](auto*& ptr, size_t n) {
    ptr = reinterpret_cast<std::remove_reference_t<decltype(ptr)>>(ws + o);
    o += align(n * sizeof(*ptr));
  };
  const size_t t = size_t(n_toggles);
  take(r.key, t); take(r.key_out, t); take(r.val, t); take(r.val_out, t);
  take(r.seg, size_t(n_ann) + 1);
  take(r.par, size_t(n_parts));
  take(r.nrun, size_t(n_ann));
  r.temp_bytes = runs_temp_bytes(n_ann, n_toggles);
  r.temp = ws + o;
  r.total = o + align(r.temp_bytes);
  return r;
}

PolyParams params(const double* xy, const int64_t* part_off, const int32_t* part_ann, const int64_t* ann_part,
                  const int32_t* ann_hw, int n_parts, int n_ann, int64_t n_edges) {
  PolyParams P{};
  P.xy = xy; P.part_off = part_off; P.part_ann = part_ann; P.ann_part = ann_part; P.ann_hw = ann_hw;
  P.n_parts = n_parts; P.n_ann = n_ann; P.n_edges = n_edges;
  return P;
}

}  // namespace

extern "C" size_t tfb200_coco_poly_count_workspace_bytes(int n_parts, int n_ann, int64_t n_edges) {
  if (cp_check(n_parts, n_ann, n_edges)) return 0;
  return align(size_t(n_edges) * 4) + align(count_scan_bytes(n_edges));
}

extern "C" int tfb200_coco_poly_count(const double* xy, const int64_t* part_off, const int32_t* part_ann,
                                      const int64_t* ann_part, const int32_t* ann_hw, int n_parts, int n_ann,
                                      int64_t n_edges, void* workspace, size_t workspace_bytes, int32_t* toggle_off,
                                      int64_t* ann_points, int64_t* sizes, void* stream) {
  if (!xy || !part_off || !part_ann || !ann_part || !ann_hw || !workspace || !toggle_off || !ann_points || !sizes)
    return TFB200_E_NULLPTR;
  if (int rc = cp_check(n_parts, n_ann, n_edges)) return rc;
  if (workspace_bytes < tfb200_coco_poly_count_workspace_bytes(n_parts, n_ann, n_edges)) return TFB200_E_SHAPE;
  const PolyParams P = params(xy, part_off, part_ann, ann_part, ann_hw, n_parts, n_ann, n_edges);
  const cudaStream_t s = cudaStream_t(stream);
  int32_t* count = static_cast<int32_t*>(workspace);
  void* temp = static_cast<char*>(workspace) + align(size_t(n_edges) * 4);
  if (n_ann > 0)
    if (cudaError_t e = cudaMemsetAsync(ann_points, 0, size_t(n_ann) * 8, s)) return int(e);
  cp_init_kernel<<<1, 1, 0, s>>>(sizes, n_ann, toggle_off);
  int launches = 2;
  if (n_edges > 0) {
    cp_points_kernel<<<blocks(n_edges), kThreads, 0, s>>>(P, ann_points, sizes);
    cp_toggles_kernel<false><<<blocks(n_edges), kThreads, 0, s>>>(P, count, toggle_off, sizes, nullptr, nullptr);
    size_t tb = count_scan_bytes(n_edges);
    if (cudaError_t e = cub::DeviceScan::InclusiveSum(temp, tb, count, toggle_off + 1, int(n_edges), s)) return int(e);
    launches += 3;
  }
  cp_finish_kernel<<<1, 1, 0, s>>>(n_edges, toggle_off, sizes);
  msda_b200_count_launches(launches);
  return int(cudaGetLastError());
}

extern "C" size_t tfb200_coco_poly_runs_workspace_bytes(int n_parts, int n_ann, int64_t n_toggles) {
  if (cp_check(n_parts, n_ann, 0) || n_toggles < 0 || n_toggles > INT32_MAX) return 0;
  return carve_runs(nullptr, n_parts, n_ann, n_toggles).total;
}

extern "C" int tfb200_coco_poly_runs(const double* xy, const int64_t* part_off, const int32_t* part_ann,
                                     const int64_t* ann_part, const int32_t* ann_hw, int n_parts, int n_ann,
                                     int64_t n_edges, const int32_t* toggle_off, int64_t n_toggles, void* workspace,
                                     size_t workspace_bytes, int64_t* run_off, uint32_t* runs, void* stream) {
  if (!xy || !part_off || !part_ann || !ann_part || !ann_hw || !toggle_off || !workspace || !run_off || !runs)
    return TFB200_E_NULLPTR;
  if (int rc = cp_check(n_parts, n_ann, n_edges)) return rc;
  if (n_toggles < 0 || n_toggles > INT32_MAX) return TFB200_E_SHAPE;
  const RunsWs W = carve_runs(static_cast<char*>(workspace), n_parts, n_ann, n_toggles);
  if (workspace_bytes < W.total) return TFB200_E_SHAPE;
  const PolyParams P = params(xy, part_off, part_ann, ann_part, ann_hw, n_parts, n_ann, n_edges);
  const cudaStream_t s = cudaStream_t(stream);
  if (cudaError_t e = cudaMemsetAsync(run_off, 0, 8, s)) return int(e);
  if (n_ann == 0) return int(cudaGetLastError());
  int launches = 5;
  if (n_toggles > 0) {
    cp_toggles_kernel<true><<<blocks(n_edges), kThreads, 0, s>>>(P, nullptr, toggle_off, nullptr, W.key, W.val);
    ++launches;
  }
  cp_segments_kernel<<<blocks(int64_t(n_ann) + 1), kThreads, 0, s>>>(P, toggle_off, W.seg);
  if (n_parts > 0)
    if (cudaError_t e = cudaMemsetAsync(W.par, 0, size_t(n_parts), s)) return int(e);
  if (n_toggles > 0) {
    size_t tb = W.temp_bytes;
    if (cudaError_t e = cub::DeviceSegmentedSort::SortPairs(W.temp, tb, W.key, W.key_out, W.val, W.val_out,
                                                            int(n_toggles), n_ann, W.seg, W.seg + 1, s))
      return int(e);
    ++launches;
  }
  cp_sweep_kernel<false><<<blocks(n_ann), kThreads, 0, s>>>(P, W.seg, W.key_out, W.val_out, W.par, W.nrun, nullptr,
                                                            nullptr);
  size_t tb = W.temp_bytes;
  if (cudaError_t e = cub::DeviceScan::InclusiveSum(W.temp, tb, W.nrun, run_off + 1, n_ann, s)) return int(e);
  if (n_parts > 0)
    if (cudaError_t e = cudaMemsetAsync(W.par, 0, size_t(n_parts), s)) return int(e);
  cp_sweep_kernel<true><<<blocks(n_ann), kThreads, 0, s>>>(P, W.seg, W.key_out, W.val_out, W.par, nullptr, run_off,
                                                           runs);
  msda_b200_count_launches(launches);
  return int(cudaGetLastError());
}

extern "C" int tfb200_coco_rle_runs(const uint8_t* chars, const int64_t* str_off, const int64_t* run_cap_off, int n,
                                    int h, int w, int64_t* bounds, uint32_t* runs, int64_t* first_bad, void* stream) {
  if (!chars || !str_off || !run_cap_off || !bounds || !runs || !first_bad) return TFB200_E_NULLPTR;
  if (n < 0 || h < 0 || w < 0 || int64_t(h) * w > INT32_MAX) return TFB200_E_SHAPE;
  if (n == 0) return 0;
  cp_rle_kernel<<<blocks(n), kThreads, 0, cudaStream_t(stream)>>>(chars, str_off, run_cap_off, n, int64_t(h) * w,
                                                                  bounds, runs, first_bad);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_coco_masks_u8(const int32_t* src, int N, int H, int W, const int64_t* poly_run_off,
                                    const uint32_t* poly_runs, const int64_t* rle_bounds, const uint32_t* rle_runs,
                                    uint8_t* out, void* stream) {
  if (!src || !poly_run_off || !poly_runs || !rle_bounds || !rle_runs || !out) return TFB200_E_NULLPTR;
  if (N < 0 || H < 0 || W < 0 || int64_t(H) * W > INT32_MAX) return TFB200_E_SHAPE;
  const int64_t total = int64_t(N) * H * W;
  if (total == 0) return 0;
  const int64_t nb = (total + kThreads - 1) / kThreads;
  cp_masks_kernel<<<unsigned(nb < 65536 * 16 ? nb : 65536 * 16), kThreads, 0, cudaStream_t(stream)>>>(
      src, total, H, W, poly_run_off, poly_runs, rle_bounds, rle_runs, out);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}
