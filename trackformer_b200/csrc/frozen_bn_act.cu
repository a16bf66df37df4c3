// Frozen batch-norm + (residual add) + ReLU for NHWC activations in one pass (sm_90a).
//
// The reference backbone (torchvision ResNet-50 with FrozenBatchNorm2d, src/trackformer/models/backbone.py:19-55,
// 98-100) runs  y = relu(x * scale[c] + shift[c] [+ identity])  as 2-3 separate elementwise passes after every one of
// its 53 convolutions; at 3x800x1333 that is ~209 M activations per pass.  Here it is one streaming kernel per
// convolution output (read x [+ identity], write y) and one for the backward (read dy and y, write dx [+ d_identity]);
// the ReLU mask is recovered from the saved output (y > 0), nothing else is stored.  The batch-norm is frozen, so
// there are no parameter gradients.  Layout: channels-last, C % 4 == 0, 16-byte aligned -> float4 along C.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "launch_counter.h"

namespace {

constexpr int kThreads = 256;
constexpr int kMaxCtas = 132 * 8;

template <bool RELU, bool RES>
__global__ void __launch_bounds__(kThreads)
frozen_bn_act_fwd_kernel(const float4* __restrict__ x, const float4* __restrict__ res, const float4* __restrict__ scale,
                         const float4* __restrict__ shift, float4* __restrict__ y, int64_t npacks, int cpacks) {
  const int64_t stride = int64_t(gridDim.x) * kThreads;
  for (int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x; i < npacks; i += stride) {
    const int c = int(i % cpacks);
    const float4 v = __ldcs(x + i);                       // streamed: the convolution output is dead after this
    const float4 s = __ldg(scale + c), b = __ldg(shift + c);
    float4 o = make_float4(fmaf(v.x, s.x, b.x), fmaf(v.y, s.y, b.y), fmaf(v.z, s.z, b.z), fmaf(v.w, s.w, b.w));
    if (RES) {
      const float4 r = __ldg(res + i);
      o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
    }
    if (RELU) {
      o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f);
    }
    y[i] = o;
  }
}

template <bool RELU, bool RES>
__global__ void __launch_bounds__(kThreads)
frozen_bn_act_bwd_kernel(const float4* __restrict__ dy, const float4* __restrict__ y, const float4* __restrict__ scale,
                         float4* __restrict__ dx, float4* __restrict__ dres, int64_t npacks, int cpacks) {
  const int64_t stride = int64_t(gridDim.x) * kThreads;
  for (int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x; i < npacks; i += stride) {
    const int c = int(i % cpacks);
    float4 g = __ldcs(dy + i);
    if (RELU) {
      const float4 o = __ldg(y + i);
      g.x = o.x > 0.f ? g.x : 0.f; g.y = o.y > 0.f ? g.y : 0.f;
      g.z = o.z > 0.f ? g.z : 0.f; g.w = o.w > 0.f ? g.w : 0.f;
    }
    if (RES) dres[i] = g;
    if (dx != nullptr) {
      const float4 s = __ldg(scale + c);
      dx[i] = make_float4(g.x * s.x, g.y * s.y, g.z * s.z, g.w * s.w);
    }
  }
}

// Stem of the trunk in one pass: y = maxpool3x3/s2/p1(relu(x * scale + shift)) (torchvision resnet: bn1 -> relu ->
// maxpool; reference backbone.py:70-78).  Forward only -- the stem is frozen (backbone.py:64-68), nothing upstream needs
// a gradient.  Thread = output pixel x 4 channels; padding contributes nothing (max over the in-bounds taps, like
// PyTorch's -inf padding).
__global__ void __launch_bounds__(kThreads)
frozen_bn_relu_maxpool_kernel(const float4* __restrict__ x, const float4* __restrict__ scale, const float4* __restrict__ shift,
                              float4* __restrict__ y, int N, int H, int W, int Ho, int Wo, int cpacks) {
  const int64_t total = int64_t(N) * Ho * Wo * cpacks;
  const int64_t stride = int64_t(gridDim.x) * kThreads;
  for (int64_t i = int64_t(blockIdx.x) * kThreads + threadIdx.x; i < total; i += stride) {
    const int c = int(i % cpacks);
    int64_t p = i / cpacks;
    const int xo = int(p % Wo); p /= Wo;
    const int yo = int(p % Ho);
    const int n = int(p / Ho);
    const float4 s = __ldg(scale + c), b = __ldg(shift + c);
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f);                 // relu(.) >= 0 and every window has an in-bounds tap
#pragma unroll
    for (int dy = -1; dy <= 1; ++dy) {
      const int yi = 2 * yo + dy;
      if (yi < 0 || yi >= H) continue;
#pragma unroll
      for (int dx = -1; dx <= 1; ++dx) {
        const int xi = 2 * xo + dx;
        if (xi < 0 || xi >= W) continue;
        const float4 v = __ldg(x + ((int64_t(n) * H + yi) * W + xi) * cpacks + c);
        m.x = fmaxf(m.x, fmaf(v.x, s.x, b.x)); m.y = fmaxf(m.y, fmaf(v.y, s.y, b.y));
        m.z = fmaxf(m.z, fmaf(v.z, s.z, b.z)); m.w = fmaxf(m.w, fmaf(v.w, s.w, b.w));
      }
    }
    y[i] = m;
  }
}

inline bool misaligned(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) != 0; }

inline unsigned grid_for(int64_t npacks) {
  int64_t ctas = (npacks + kThreads - 1) / kThreads;
  return unsigned(ctas < 1 ? 1 : (ctas > kMaxCtas ? kMaxCtas : ctas));
}

}  // namespace

extern "C" {

int tfb200_frozen_bn_act_fwd_f32(const float* x, const float* residual, const float* scale, const float* shift,
                                 float* y, int64_t pixels, int C, int relu, void* stream) {
  if (!x || !scale || !shift || !y) return TFB200_E_NULLPTR;
  if (pixels < 0 || C <= 0 || C % 4 != 0) return TFB200_E_SHAPE;
  if (misaligned(x) || misaligned(y) || misaligned(scale) || misaligned(shift) || (residual && misaligned(residual)))
    return TFB200_E_SHAPE;
  if (pixels == 0) return 0;
  const int cpacks = C / 4;
  const int64_t npacks = pixels * cpacks;
  cudaStream_t st = cudaStream_t(stream);
#define TFB200_BN_FWD(R, S)                                                                                     \
  frozen_bn_act_fwd_kernel<R, S><<<grid_for(npacks), kThreads, 0, st>>>(                                          \
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(residual),                              \
      reinterpret_cast<const float4*>(scale), reinterpret_cast<const float4*>(shift), reinterpret_cast<float4*>(y), \
      npacks, cpacks)
  if (relu && residual) TFB200_BN_FWD(true, true);
  else if (relu) TFB200_BN_FWD(true, false);
  else if (residual) TFB200_BN_FWD(false, true);
  else TFB200_BN_FWD(false, false);
#undef TFB200_BN_FWD
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

int tfb200_frozen_bn_act_bwd_f32(const float* dy, const float* y, const float* scale, float* dx, float* dresidual,
                                 int64_t pixels, int C, int relu, void* stream) {
  if (!dy || !scale || (relu && !y) || (!dx && !dresidual)) return TFB200_E_NULLPTR;
  if (pixels < 0 || C <= 0 || C % 4 != 0) return TFB200_E_SHAPE;
  if (misaligned(dy) || misaligned(scale) || (y && misaligned(y)) || (dx && misaligned(dx)) ||
      (dresidual && misaligned(dresidual)))
    return TFB200_E_SHAPE;
  if (pixels == 0) return 0;
  const int cpacks = C / 4;
  const int64_t npacks = pixels * cpacks;
  cudaStream_t st = cudaStream_t(stream);
#define TFB200_BN_BWD(R, S)                                                                                  \
  frozen_bn_act_bwd_kernel<R, S><<<grid_for(npacks), kThreads, 0, st>>>(                                       \
      reinterpret_cast<const float4*>(dy), reinterpret_cast<const float4*>(y),                                 \
      reinterpret_cast<const float4*>(scale), reinterpret_cast<float4*>(dx), reinterpret_cast<float4*>(dresidual), \
      npacks, cpacks)
  if (relu && dresidual) TFB200_BN_BWD(true, true);
  else if (relu) TFB200_BN_BWD(true, false);
  else if (dresidual) TFB200_BN_BWD(false, true);
  else TFB200_BN_BWD(false, false);
#undef TFB200_BN_BWD
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}


int tfb200_frozen_bn_relu_maxpool_f32(const float* x, const float* scale, const float* shift, float* y, int N, int H, int W,
                                      int C, void* stream) {
  if (!x || !scale || !shift || !y) return TFB200_E_NULLPTR;
  if (N < 1 || H < 1 || W < 1 || C <= 0 || C % 4 != 0) return TFB200_E_SHAPE;
  if (misaligned(x) || misaligned(y) || misaligned(scale) || misaligned(shift)) return TFB200_E_SHAPE;
  const int Ho = (H + 2 - 3) / 2 + 1, Wo = (W + 2 - 3) / 2 + 1;
  const int64_t total = int64_t(N) * Ho * Wo * (C / 4);
  frozen_bn_relu_maxpool_kernel<<<grid_for(total), kThreads, 0, cudaStream_t(stream)>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<const float4*>(scale), reinterpret_cast<const float4*>(shift),
      reinterpret_cast<float4*>(y), N, H, W, Ho, Wo, C / 4);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}
}  // extern "C"
