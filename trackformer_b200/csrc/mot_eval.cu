// MOTChallenge CLEAR-MOT and identity metrics of many sequences on the device (sm_90a): the routines of
// mot_eval_core.h as a memset of the tp matrices and seven launches -- state init, pair count, frame scan, pair write
// + tp, the CLEAR-MOT pass (one CTA per sequence), the tp-graph components (one CTA per sequence) and the identity
// matching (one CTA per GT id, which returns at once unless the id roots a component).  Nothing is read back here: the caller copies `out` once.
#include <cuda_runtime.h>

#include "launch_counter.h"
#include "mot_eval_core.h"

namespace {

using namespace tfb200_mot;

__global__ void __launch_bounds__(kThreads) me_init_kernel(const __grid_constant__ Params p) {
  me_init_seq(p, int(blockIdx.x));
}

template <bool kWrite>
__global__ void __launch_bounds__(kThreads) me_pairs_kernel(const __grid_constant__ Params p) {
  __shared__ Shared sh;
  me_pairs_frame<kWrite>(p, int(blockIdx.x), sh);
}

__global__ void __launch_bounds__(kThreads) me_scan_kernel(const __grid_constant__ Params p) {
  __shared__ Shared sh;
  me_scan(p, sh);
}

__global__ void __launch_bounds__(kThreads) me_clear_kernel(const __grid_constant__ Params p) {
  __shared__ Shared sh;
  me_clear_seq(p, int(blockIdx.x), sh);
}

__global__ void __launch_bounds__(kThreads) me_id_label_kernel(const __grid_constant__ Params p) {
  __shared__ Shared sh;
  me_id_label(p, int(blockIdx.x), sh);
}

__global__ void __launch_bounds__(kThreads) me_id_comp_kernel(const __grid_constant__ Params p) {
  __shared__ Shared sh;
  me_id_comp(p, int64_t(blockIdx.x), sh);
}

}  // namespace

extern "C" size_t tfb200_mot_eval_workspace_bytes(int S, int F, int64_t n_gt, int64_t n_trk, int64_t tp_cells,
                                                  int max_obj, int max_hyp, int64_t pair_cap) {
  if (me_check(S, F, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap)) return 0;
  Params p{};
  return me_carve(p, nullptr, S, F, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap);
}

extern "C" int tfb200_mot_eval_f32(const int64_t* seq, const int32_t* frame_obj, const int32_t* frame_hyp,
                                   const int32_t* obj_id, const float* obj_box, const int32_t* hyp_id,
                                   const float* hyp_box, int S, int F, int64_t n_gt, int64_t n_trk, int64_t tp_cells,
                                   int max_obj, int max_hyp, int64_t pair_cap, void* workspace,
                                   size_t workspace_bytes, int64_t* out, void* stream) {
  if (!seq || !frame_obj || !frame_hyp || !obj_id || !obj_box || !hyp_id || !hyp_box || !workspace || !out)
    return TFB200_E_NULLPTR;
  if (int rc = me_check(S, F, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap)) return rc;
  Params p{};
  if (workspace_bytes < me_carve(p, static_cast<char*>(workspace), S, F, n_gt, n_trk, tp_cells, max_obj, max_hyp,
                                 pair_cap))
    return TFB200_E_SHAPE;
  p.S = S; p.F = F; p.max_obj = max_obj; p.max_hyp = max_hyp; p.pair_cap = pair_cap;
  p.seq = seq; p.fobj = frame_obj; p.fhyp = frame_hyp; p.obj_id = obj_id; p.obj_box = obj_box; p.hyp_id = hyp_id;
  p.hyp_box = hyp_box; p.out = out;
  const cudaStream_t s = cudaStream_t(stream);
  if (tp_cells > 0)
    if (cudaError_t e = cudaMemsetAsync(p.tp, 0, size_t(tp_cells) * 4, s)) return int(e);
  me_init_kernel<<<S, kThreads, 0, s>>>(p);
  int launches = 4;
  if (F > 0) {
    me_pairs_kernel<false><<<F, kThreads, 0, s>>>(p);
    me_scan_kernel<<<1, kThreads, 0, s>>>(p);
    me_pairs_kernel<true><<<F, kThreads, 0, s>>>(p);
    launches += 2;
  } else {
    me_scan_kernel<<<1, kThreads, 0, s>>>(p);
  }
  me_clear_kernel<<<S, kThreads, 0, s>>>(p);
  me_id_label_kernel<<<S, kThreads, 0, s>>>(p);
  if (n_gt > 0) {
    me_id_comp_kernel<<<unsigned(n_gt), kThreads, 0, s>>>(p);
    ++launches;
  }
  msda_b200_count_launches(launches);
  return int(cudaGetLastError());
}
