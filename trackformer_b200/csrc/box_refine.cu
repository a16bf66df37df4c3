// boxes = sigmoid(delta + inverse_sigmoid(reference)) in one launch per direction (sm_90a).
//
// The reference refines its reference boxes after every decoder layer and again in the detection heads with a chain
// of ~8 PyTorch ops per call -- clamp(0,1), clamp(min=eps), 1-x, clamp(min=eps), div, log, add, sigmoid
// (src/trackformer/util/misc.py:515-519, models/deformable_transformer.py:412-422, models/deformable_detr.py:229-248)
// -- plus ~12 more in the backward; on [N, 300..800, 4] tensors every one of them is a launch-bound ~2 us kernel.
// Same arithmetic here, including the gradient gates of the three clamps (torch passes the gradient where
// min <= x <= max).  `ref_dim` = 2: only the first two of the four components get the reference added
// (2-d reference points, deformable_detr.py:240-242).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "launch_counter.h"

namespace {

__global__ void __launch_bounds__(256)
refine_boxes_fwd_kernel(const float* __restrict__ delta, const float* __restrict__ ref, float* __restrict__ out,
                        int64_t n, int ref_dim, float eps) {
  const int64_t i = int64_t(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n) return;
  const int c = int(i & 3);
  float z = delta[i];
  if (c < ref_dim) {
    const float x0 = fminf(fmaxf(ref[(i >> 2) * ref_dim + c], 0.f), 1.f);
    const float x1 = fmaxf(x0, eps), x2 = fmaxf(1.f - x0, eps);
    z += logf(x1 / x2);
  }
  out[i] = 1.f / (1.f + expf(-z));
}

__global__ void __launch_bounds__(256)
refine_boxes_bwd_kernel(const float* __restrict__ grad_out, const float* __restrict__ out, const float* __restrict__ ref,
                        float* __restrict__ grad_delta, float* __restrict__ grad_ref, int64_t n, int ref_dim, float eps) {
  const int64_t i = int64_t(blockIdx.x) * 256 + threadIdx.x;
  if (i >= n) return;
  const int c = int(i & 3);
  const float y = out[i];
  const float gz = grad_out[i] * y * (1.f - y);
  grad_delta[i] = gz;
  if (grad_ref != nullptr && c < ref_dim) {
    const float x = ref[(i >> 2) * ref_dim + c];
    float g = 0.f;
    if (x >= 0.f && x <= 1.f) {                                   // clamp(0, 1)
      const float x1 = fmaxf(x, eps), x2 = fmaxf(1.f - x, eps);
      g = (x >= eps ? 1.f / x1 : 0.f) + ((1.f - x) >= eps ? 1.f / x2 : 0.f);
    }
    grad_ref[(i >> 2) * ref_dim + c] = gz * g;
  }
}

}  // namespace

extern "C" int tfb200_refine_boxes_fwd_f32(const float* delta, const float* ref, float* out, int64_t rows, int ref_dim,
                                           float eps, void* stream) {
  if (!delta || !ref || !out) return TFB200_E_NULLPTR;
  if (rows < 0 || (ref_dim != 2 && ref_dim != 4)) return TFB200_E_SHAPE;
  if (rows == 0) return 0;
  const int64_t n = rows * 4;
  refine_boxes_fwd_kernel<<<unsigned((n + 255) / 256), 256, 0, cudaStream_t(stream)>>>(delta, ref, out, n, ref_dim, eps);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_refine_boxes_bwd_f32(const float* grad_out, const float* out, const float* ref, float* grad_delta,
                                           float* grad_ref, int64_t rows, int ref_dim, float eps, void* stream) {
  if (!grad_out || !out || !ref || !grad_delta) return TFB200_E_NULLPTR;
  if (rows < 0 || (ref_dim != 2 && ref_dim != 4)) return TFB200_E_SHAPE;
  if (rows == 0) return 0;
  const int64_t n = rows * 4;
  refine_boxes_bwd_kernel<<<unsigned((n + 255) / 256), 256, 0, cudaStream_t(stream)>>>(grad_out, out, ref, grad_delta,
                                                                                      grad_ref, n, ref_dim, eps);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}
