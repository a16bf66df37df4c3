// COCO box / mask AP on the device (sm_90a): the routines of coco_eval_core.h.  tfb200_coco_match_f32 ranks, (for
// segm) packs and decodes the masks, computes the IoUs and runs evaluateImg for the images of one update;
// tfb200_coco_accumulate_f32 gathers the kept images' detections in image-id order, sorts them stably by
// (category, descending score) with CUB's radix sort and runs accumulate.  Nothing is read back here.
#include <cuda_runtime.h>

#include <type_traits>

#include <cub/device/device_radix_sort.cuh>

#include "coco_eval_core.h"
#include "launch_counter.h"

namespace {

using namespace tfb200_coco;

__global__ void __launch_bounds__(kThreads) ce_rank_kernel(const __grid_constant__ MatchParams p) {
  ce_rank(p, int(blockIdx.x));
}

__global__ void __launch_bounds__(kThreads) ce_pack_kernel(const __grid_constant__ MatchParams p) {
  __shared__ PackShared sh;
  ce_pack_dt(p, int(blockIdx.x), int(blockIdx.y), sh);
}

__global__ void __launch_bounds__(kThreads) ce_decode_kernel(const __grid_constant__ MatchParams p) {
  ce_decode_gt(p, int(blockIdx.x), int(blockIdx.y));
}

__global__ void __launch_bounds__(kThreads) ce_iou_kernel(const __grid_constant__ MatchParams p) {
  __shared__ IouShared sh;
  ce_iou(p, int(blockIdx.x), int(blockIdx.y), sh);
}

__global__ void __launch_bounds__(kThreads) ce_match_kernel(const __grid_constant__ MatchParams p) {
  ce_match(p, int(blockIdx.x));
}

__global__ void __launch_bounds__(kThreads) ce_gather_kernel(const __grid_constant__ AccParams p) {
  ce_gather(p, int(blockIdx.x));
}

__global__ void __launch_bounds__(kThreads) ce_acc_kernel(const __grid_constant__ AccParams p) {
  __shared__ AccShared sh;
  ce_acc(p, int(blockIdx.x), sh);
}

__global__ void ce_status_kernel(const __grid_constant__ AccParams p) { p.status_out[0] = double(p.status_in[0]); }

size_t match_carve(MatchParams& p, char* ws, int64_t N, int64_t iou_cells, int64_t dbit_words, int64_t gbit_words,
                   int64_t gtm_bytes) {
  size_t o = 0;
  auto take = [&](auto*& ptr, size_t n) {
    ptr = reinterpret_cast<std::remove_reference_t<decltype(ptr)>>(reinterpret_cast<uintptr_t>(ws) + o);
    o += (n * sizeof(*ptr) + 255) & ~size_t(255);
  };
  take(p.dk, size_t(N));
  take(p.dord, size_t(N));
  take(p.iou, size_t(iou_cells));
  take(p.dbits, size_t(dbit_words));
  take(p.gbits, size_t(gbit_words));
  take(p.dbox, size_t(N) * 4);
  take(p.dpx, size_t(N));
  take(p.gtm, size_t(gtm_bytes));
  return o;
}

size_t acc_carve(AccParams& p, char* ws, int64_t n, size_t* sort_bytes_out, void** sort_ws) {
  size_t o = 0;
  auto take = [&](auto*& ptr, size_t cnt) {
    ptr = reinterpret_cast<std::remove_reference_t<decltype(ptr)>>(reinterpret_cast<uintptr_t>(ws) + o);
    o += (cnt * sizeof(*ptr) + 255) & ~size_t(255);
  };
  take(p.key_in, size_t(n));
  take(p.key_out, size_t(n));
  take(p.val_in, size_t(n));
  take(p.val_out, size_t(n));
  size_t sort_bytes = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, sort_bytes, p.key_in, p.key_out, p.val_in, p.val_out, int(n > 0 ? n : 1));
  *sort_bytes_out = sort_bytes;
  *sort_ws = reinterpret_cast<void*>(reinterpret_cast<uintptr_t>(ws) + o);
  return o + ((sort_bytes + 255) & ~size_t(255));
}

bool match_sizes_ok(int64_t N, int64_t iou_cells, int64_t dbit_words, int64_t gbit_words, int64_t gtm_bytes) {
  return N >= 0 && iou_cells >= 0 && dbit_words >= 0 && gbit_words >= 0 && gtm_bytes >= 0;
}

}  // namespace

extern "C" size_t tfb200_coco_match_workspace_bytes(int64_t N, int64_t iou_cells, int64_t dbit_words,
                                                    int64_t gbit_words, int64_t gtm_bytes) {
  if (!match_sizes_ok(N, iou_cells, dbit_words, gbit_words, gtm_bytes) || N > INT32_MAX) return 0;
  MatchParams p{};
  return match_carve(p, nullptr, N, iou_cells, dbit_words, gbit_words, gtm_bytes);
}

extern "C" int tfb200_coco_match_f32(const int64_t* img, int B, int max_n, int max_g, const float* boxes,
                                     const float* scores, const int64_t* labels, int64_t N, const int64_t* cat_ids,
                                     int K, const int64_t* gt_off, const int32_t* gt_k, const double* gt_box,
                                     const double* gt_area, const uint8_t* gt_crowd, const int64_t* gt_id,
                                     const int64_t* gt_run_off, const uint32_t* gt_runs, const int32_t* gt_bbox,
                                     const int64_t* gt_px, const double* area_rng, int A, const double* iou_thr, int T,
                                     int max_det, int segm, int64_t iou_cells, int64_t dbit_words, int64_t gbit_words,
                                     int64_t gtm_bytes, void* workspace, size_t workspace_bytes, uint64_t* key,
                                     int32_t* rank, uint32_t* state, int32_t* status, void* stream) {
  if (!img || !scores || !labels || !cat_ids || !gt_off || !gt_k || !gt_area || !gt_crowd || !gt_id || !area_rng ||
      !iou_thr || !workspace || !key || !rank || !state || !status)
    return TFB200_E_NULLPTR;
  if (segm ? (!gt_run_off || !gt_runs || !gt_bbox || !gt_px) : (!boxes || !gt_box)) return TFB200_E_NULLPTR;
  if (int rc = ce_check_match(B, N, K, A, T, max_det)) return rc;
  if (max_n < 0 || max_n > kMaxDets || max_g < 0 || !match_sizes_ok(N, iou_cells, dbit_words, gbit_words, gtm_bytes))
    return TFB200_E_SHAPE;
  MatchParams p{};
  if (workspace_bytes < match_carve(p, static_cast<char*>(workspace), N, iou_cells, dbit_words, gbit_words, gtm_bytes))
    return TFB200_E_SHAPE;
  p.B = B; p.K = K; p.A = A; p.T = T; p.max_det = max_det; p.segm = segm;
  p.img = img; p.boxes = boxes; p.scores = scores; p.labels = labels; p.cat_ids = cat_ids;
  p.gt_off = gt_off; p.gt_k = gt_k; p.gt_box = gt_box; p.gt_area = gt_area; p.gt_crowd = gt_crowd; p.gt_id = gt_id;
  p.gt_run_off = gt_run_off; p.gt_runs = gt_runs; p.gt_bbox = gt_bbox; p.gt_px = gt_px;
  p.area_rng = area_rng; p.iou_thr = iou_thr; p.key = key; p.rank = rank; p.state = state; p.status = status;
  const cudaStream_t s = cudaStream_t(stream);
  if (gtm_bytes > 0)
    if (cudaError_t e = cudaMemsetAsync(p.gtm, 0, size_t(gtm_bytes), s)) return int(e);
  int launches = 2;
  ce_rank_kernel<<<B, kThreads, 0, s>>>(p);
  if (max_n > 0) {
    if (segm) {
      if (gbit_words > 0)
        if (cudaError_t e = cudaMemsetAsync(p.gbits, 0, size_t(gbit_words) * 4, s)) return int(e);
      ce_pack_kernel<<<dim3(B, max_n), kThreads, 0, s>>>(p);
      ++launches;
      if (max_g > 0) {
        ce_decode_kernel<<<dim3(B, max_g), kThreads, 0, s>>>(p);
        ++launches;
      }
    }
    ce_iou_kernel<<<dim3(B, max_n), kThreads, 0, s>>>(p);
    ++launches;
  }
  ce_match_kernel<<<B, kThreads, 0, s>>>(p);
  msda_b200_count_launches(launches);
  return int(cudaGetLastError());
}

extern "C" size_t tfb200_coco_accumulate_workspace_bytes(int64_t n) {
  if (n < 0 || n > INT32_MAX) return 0;
  AccParams p{};
  size_t sort_bytes;
  void* sort_ws;
  return acc_carve(p, nullptr, n, &sort_bytes, &sort_ws);
}

extern "C" int tfb200_coco_accumulate_f32(const uint64_t* key, const int32_t* rank, const uint32_t* state,
                                          int64_t n_rec, const int64_t* kept, int n_kept, int64_t n,
                                          const int64_t* npig, const double* rec_thr, const int32_t* max_dets,
                                          const int32_t* status, int K, int A, int T, int R, int M, void* workspace,
                                          size_t workspace_bytes, double* precision, double* recall, double* scores,
                                          double* status_out, void* stream) {
  if (!kept || !npig || !rec_thr || !max_dets || !status || !workspace || !precision || !recall || !scores ||
      !status_out)
    return TFB200_E_NULLPTR;
  if (n_rec > 0 && (!key || !rank || !state)) return TFB200_E_NULLPTR;
  if (int rc = ce_check_acc(K, A, T, R, M, n_kept, n_rec, n)) return rc;
  if (n > INT32_MAX) return TFB200_E_SHAPE;
  AccParams p{};
  size_t sort_bytes;
  void* sort_ws;
  if (workspace_bytes < acc_carve(p, static_cast<char*>(workspace), n, &sort_bytes, &sort_ws)) return TFB200_E_SHAPE;
  p.K = K; p.A = A; p.T = T; p.R = R; p.M = M; p.n_kept = n_kept; p.n_rec = n_rec; p.n = n;
  p.key = key; p.rank = rank; p.state = state; p.kept = kept; p.npig = npig; p.rec_thr = rec_thr;
  p.max_dets = max_dets; p.status_in = status; p.precision = precision; p.recall = recall; p.scores = scores;
  p.status_out = status_out;
  const cudaStream_t s = cudaStream_t(stream);
  int launches = 2;
  if (n_kept > 0) {
    ce_gather_kernel<<<n_kept, kThreads, 0, s>>>(p);
    ++launches;
  }
  if (n > 0) {
    int end_bit = 33;                                    // category index K (not evaluated) must fit
    while ((uint64_t(1) << (end_bit - 32)) <= uint64_t(K)) ++end_bit;
    if (cudaError_t e = cub::DeviceRadixSort::SortPairs(sort_ws, sort_bytes, p.key_in, p.key_out, p.val_in, p.val_out,
                                                         int(n), 0, end_bit, s))
      return int(e);
  }
  ce_acc_kernel<<<K * A * M * T, kThreads, 0, s>>>(p);
  ce_status_kernel<<<1, 1, 0, s>>>(p);
  msda_b200_count_launches(launches);
  return int(cudaGetLastError());
}
