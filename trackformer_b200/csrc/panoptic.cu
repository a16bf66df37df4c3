// Panoptic post-processing and PQ scoring on the device (sm_90a): the routines of panoptic_core.h, one kernel each.
// Nothing is read back here; the caller's host code reads the kept flags, the per-round areas and the reduced sums.
#include <cuda_runtime.h>

#include "launch_counter.h"
#include "panoptic_core.h"

namespace {

using namespace tfb200_panoptic;

__global__ void __launch_bounds__(kThreads) pp_classes_kernel(const __grid_constant__ PpParams p) {
  pp_classes(p, int64_t(blockIdx.x) * kThreads + threadIdx.x);
}

__global__ void __launch_bounds__(kThreads) pp_label_kernel(const __grid_constant__ PpParams p) {
  __shared__ unsigned long long hist[kMaxKept];
  pp_label(p, int(blockIdx.y), int(blockIdx.x), hist);
}

__global__ void __launch_bounds__(kThreads) pp_final_kernel(const __grid_constant__ PpParams p) {
  pp_final(p, int(blockIdx.y), int(blockIdx.x));
}

__global__ void __launch_bounds__(kThreads) pq_count_kernel(const __grid_constant__ PqParams p) {
  __shared__ int sh[kSharedCells];
  pq_count(p, int(blockIdx.y), int(blockIdx.x), sh);
}

__global__ void __launch_bounds__(kThreads) pq_match_kernel(const __grid_constant__ PqParams p) {
  __shared__ MatchShared sh;
  pq_match(p, int(blockIdx.x), sh);
}

__global__ void __launch_bounds__(kThreads) pq_reduce_kernel(const int32_t* stat_i, const double* stat_iou,
                                                             const long long* err, const int64_t* rows, int64_t n,
                                                             int Kc, double* out, int64_t* err_out) {
  pq_reduce(stat_i, stat_iou, err, rows, n, Kc, int(blockIdx.x) * kThreads + int(threadIdx.x), out, err_out);
}

bool grid_ok(int B, int blocks) { return B > 0 && B <= 65535 && blocks > 0; }

}  // namespace

extern "C" int tfb200_panoptic_classes_f32(const float* logits, int B, int Q, int C, float threshold, int32_t* cls,
                                           float* score, uint8_t* keep, void* stream) {
  if (!logits || !cls || !score || !keep) return TFB200_E_NULLPTR;
  if (B <= 0 || Q <= 0 || C < 2) return TFB200_E_SHAPE;
  PpParams p{};
  p.B = B; p.Q = Q; p.C = C; p.threshold = threshold;
  p.logits = logits; p.cls = cls; p.score = score; p.keep = keep;
  const int64_t rows = int64_t(B) * Q;
  pp_classes_kernel<<<unsigned((rows + kThreads - 1) / kThreads), kThreads, 0, cudaStream_t(stream)>>>(p);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_panoptic_label_f32(const float* masks, int B, int Q, int h, int w, const int64_t* img,
                                         int max_kept, const int32_t* kept_q, const int32_t* kept_alive,
                                         const int32_t* kept_rep, const int32_t* idx, int32_t* map,
                                         unsigned long long* area, int blocks, void* stream) {
  if (!masks || !img || !kept_q || !kept_alive || !kept_rep || !idx || !map || !area) return TFB200_E_NULLPTR;
  if (!grid_ok(B, blocks) || Q <= 0 || h <= 0 || w <= 0 || max_kept < 0 || max_kept > kMaxKept) return TFB200_E_SHAPE;
  PpParams p{};
  p.B = B; p.Q = Q; p.h = h; p.w = w;
  p.masks = masks; p.img = img; p.kept_q = kept_q; p.kept_alive = kept_alive; p.kept_rep = kept_rep; p.idx = idx;
  p.map = map; p.area = area;
  pp_label_kernel<<<dim3(blocks, B), kThreads, 0, cudaStream_t(stream)>>>(p);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_panoptic_final_f32(const int64_t* img, int B, const int32_t* kept_alive, const int32_t* kept_pos,
                                         const int32_t* idx, const int32_t* map, int32_t* out, int blocks,
                                         void* stream) {
  if (!img || !kept_alive || !kept_pos || !idx || !map || !out) return TFB200_E_NULLPTR;
  if (!grid_ok(B, blocks)) return TFB200_E_SHAPE;
  PpParams p{};
  p.B = B; p.img = img; p.kept_alive = kept_alive; p.kept_pos = kept_pos; p.idx = idx;
  p.map = const_cast<int32_t*>(map);                   // read only by pp_final
  p.out = out;
  pp_final_kernel<<<dim3(blocks, B), kThreads, 0, cudaStream_t(stream)>>>(p);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_pq_update(const int64_t* img, int B, int Kc, int max_seg, const int32_t* maps,
                                const int32_t* gt_id, const int32_t* gt_cat, const int32_t* gt_crowd,
                                const double* gt_area, const int32_t* gt_json, const int32_t* pred_id,
                                const int32_t* pred_cat, int* cells, int64_t n_cells, int64_t* pred_area,
                                int32_t* stat_i, double* stat_iou, long long* err, int blocks, void* stream) {
  if (!img || !maps || !gt_id || !gt_cat || !gt_crowd || !gt_area || !gt_json || !pred_id || !pred_cat || !cells ||
      !pred_area || !stat_i || !stat_iou || !err)
    return TFB200_E_NULLPTR;
  if (!grid_ok(B, blocks) || Kc <= 0 || Kc > kMaxCat || max_seg < 0 || max_seg > kMaxSeg || n_cells <= 0)
    return TFB200_E_SHAPE;
  PqParams p{};
  p.B = B; p.Kc = Kc; p.img = img; p.maps = maps; p.gt_id = gt_id; p.gt_cat = gt_cat; p.gt_crowd = gt_crowd;
  p.gt_area = gt_area; p.gt_json = gt_json; p.pred_id = pred_id; p.pred_cat = pred_cat; p.cells = cells;
  p.pred_area = pred_area; p.stat_i = stat_i; p.stat_iou = stat_iou; p.err = err;
  const cudaStream_t s = cudaStream_t(stream);
  if (cudaError_t e = cudaMemsetAsync(cells, 0, size_t(n_cells) * sizeof(int), s)) return int(e);
  pq_count_kernel<<<dim3(blocks, B), kThreads, 0, s>>>(p);
  pq_match_kernel<<<B, kThreads, 0, s>>>(p);
  msda_b200_count_launches(2);
  return int(cudaGetLastError());
}

extern "C" int tfb200_pq_reduce(const int32_t* stat_i, const double* stat_iou, const long long* err,
                                const int64_t* rows, int64_t n, int Kc, double* out, int64_t* err_out, void* stream) {
  if (!stat_i || !stat_iou || !err || !rows || !out || !err_out) return TFB200_E_NULLPTR;
  if (n < 0 || Kc <= 0 || Kc > kMaxCat) return TFB200_E_SHAPE;
  pq_reduce_kernel<<<(Kc + kThreads) / kThreads, kThreads, 0, cudaStream_t(stream)>>>(stat_i, stat_iou, err, rows, n,
                                                                                       Kc, out, err_out);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}
