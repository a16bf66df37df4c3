// Gradient clipping + AdamW over one flat fp32 parameter range in a single pass (sm_90a).
//
// The reference step ends with clip_grad_norm_ and torch.optim.AdamW over ~600 parameter tensors
// (src/trackformer/engine.py:147-151, src/train.py:118-119).  With every parameter, gradient and moment living in
// flat buffers (train_step.py) the whole update of one learning-rate group is ONE streaming kernel:
// 4 reads + 3 writes of 4 bytes per parameter, nothing else -- the clip coefficient is read from the device-side
// gradient norm, so the scaled gradient is never written back.
//   g   = grad * min(1, max_norm / (norm + 1e-6))            (clip_grad_norm_)
//   p  -= lr * wd * p                                          (decoupled weight decay)
//   m   = m + (1 - b1) (g - m);   v = b2 v + (1 - b2) g g
//   p  -= (lr / (1 - b1^t)) * m / (sqrt(v) / sqrt(1 - b2^t) + eps)
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "launch_counter.h"

namespace {

struct AdamArgs {
  float lr, beta1, beta2, eps, weight_decay, step_size, inv_bc2_sqrt, max_norm;
};

__device__ __forceinline__ void adam_one(float& p, float g, float& m, float& v, float clip, const AdamArgs& a) {
  g *= clip;
  p -= a.lr * a.weight_decay * p;
  m += (1.f - a.beta1) * (g - m);
  v = a.beta2 * v + (1.f - a.beta2) * g * g;
  p -= a.step_size * m / (sqrtf(v) * a.inv_bc2_sqrt + a.eps);
}

__global__ void __launch_bounds__(256)
flat_adamw_kernel(float* __restrict__ param, const float* __restrict__ grad, float* __restrict__ exp_avg,
                  float* __restrict__ exp_avg_sq, int64_t n, const float* __restrict__ grad_norm, AdamArgs a) {
  float clip = 1.f;
  if (grad_norm != nullptr) clip = fminf(1.f, a.max_norm / (__ldg(grad_norm) + 1e-6f));
  const int64_t npk = n >> 2;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < npk; i += stride) {
    float4 p = reinterpret_cast<float4*>(param)[i];
    const float4 g = __ldcs(reinterpret_cast<const float4*>(grad) + i);     // streamed: not needed again this step
    float4 m = reinterpret_cast<float4*>(exp_avg)[i];
    float4 v = reinterpret_cast<float4*>(exp_avg_sq)[i];
    adam_one(p.x, g.x, m.x, v.x, clip, a);
    adam_one(p.y, g.y, m.y, v.y, clip, a);
    adam_one(p.z, g.z, m.z, v.z, clip, a);
    adam_one(p.w, g.w, m.w, v.w, clip, a);
    reinterpret_cast<float4*>(param)[i] = p;
    reinterpret_cast<float4*>(exp_avg)[i] = m;
    reinterpret_cast<float4*>(exp_avg_sq)[i] = v;
  }
  if (blockIdx.x == 0 && threadIdx.x < (n & 3)) {                            // tail
    const int64_t i = (npk << 2) + threadIdx.x;
    adam_one(param[i], grad[i], exp_avg[i], exp_avg_sq[i], clip, a);
  }
}

}  // namespace

extern "C" int tfb200_flat_adamw_f32(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                                     const float* grad_norm_dev, float max_norm, float lr, float beta1, float beta2,
                                     float eps, float weight_decay, int64_t step, void* stream) {
  if (!param || !grad || !exp_avg || !exp_avg_sq) return TFB200_E_NULLPTR;
  if (n < 0 || step < 1) return TFB200_E_SHAPE;
  if ((reinterpret_cast<uintptr_t>(param) | reinterpret_cast<uintptr_t>(grad) | reinterpret_cast<uintptr_t>(exp_avg) |
       reinterpret_cast<uintptr_t>(exp_avg_sq)) & 15) return TFB200_E_SHAPE;
  if (n == 0) return 0;
  const double bc1 = 1.0 - pow(double(beta1), double(step));
  const double bc2 = 1.0 - pow(double(beta2), double(step));
  AdamArgs a{lr, beta1, beta2, eps, weight_decay, float(double(lr) / bc1), float(1.0 / sqrt(bc2)), max_norm};
  const int64_t npk = n >> 2;
  int64_t ctas = (npk + 255) / 256;
  if (ctas > 132 * 8) ctas = 132 * 8;            // grid-stride over 8 CTAs per SM
  if (ctas < 1) ctas = 1;
  flat_adamw_kernel<<<unsigned(ctas), 256, 0, cudaStream_t(stream)>>>(param, grad, exp_avg, exp_avg_sq, n,
                                                                      grad_norm_dev, a);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}
