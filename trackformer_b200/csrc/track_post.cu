// Detection post-processing for the online tracker in one launch (sm_90a).
//
// The reference turns the decoder outputs into per-query detections with a chain of ~8 PyTorch ops
// (src/trackformer/models/deformable_detr.py:286-334: sigmoid, max over classes, cxcywh -> xyxy, scale by the image
// size) and the tracker then reads scores, labels and boxes back track by track (src/trackformer/models/tracker.py:
// 306-330, 520-527: several .cpu() synchronisations per track per frame).  Here one kernel writes everything the
// tracker's bookkeeping needs into one packed row per query, so a frame costs one launch and one device->host copy:
//   packed[n][q] = { score, label (exact in fp32), x0, y0, x1, y1 }   boxes in pixels of the original image, unclipped
//   labels[n][q] = label as int64 (for the reference-shaped result dict)
// One warp per query: lanes stride the class axis, the arg-max keeps the FIRST maximal class like torch.max.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "launch_counter.h"

namespace {

// kSoftmax = false: sigmoid scores over all C classes (DeformablePostProcess, focal loss);
// kSoftmax = true:  softmax over the C logits (the last one is "no object"), best of the first C - 1 (PostProcess)
template <bool kSoftmax>
__global__ void __launch_bounds__(256)
detect_postprocess_kernel(const float* __restrict__ logits, const float* __restrict__ boxes,
                          const int64_t* __restrict__ sizes, float* __restrict__ packed, int64_t* __restrict__ labels,
                          int N, int Q, int C) {
  const int lane = threadIdx.x & 31;
  const int64_t row = int64_t(blockIdx.x) * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= int64_t(N) * Q) return;
  const float* lg = logits + row * C;
  float best = -1.f;          // sigmoid / softmax scores are >= 0
  int arg = 0x7fffffff;
  if (kSoftmax) {
    float mx = -INFINITY;
    for (int c = lane; c < C; c += 32) mx = fmaxf(mx, __ldg(lg + c));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int c = lane; c < C; c += 32) sum += expf(__ldg(lg + c) - mx);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    const float inv = 1.f / sum;
    for (int c = lane; c < C - 1; c += 32) {
      const float s = expf(__ldg(lg + c) - mx) * inv;
      if (s > best) { best = s; arg = c; }
    }
  } else {
    for (int c = lane; c < C; c += 32) {
      const float s = 1.f / (1.f + expf(-__ldg(lg + c)));
      if (s > best) { best = s; arg = c; }     // strict: the smallest class index wins inside a lane
    }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, o);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, o);
    if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
  }
  if (lane == 0) {
    const int n = int(row / Q);
    const float img_h = float(sizes[2 * n]), img_w = float(sizes[2 * n + 1]);
    const float4 b = __ldg(reinterpret_cast<const float4*>(boxes) + row);   // cx, cy, w, h
    float* out = packed + row * 6;
    out[0] = best;
    out[1] = float(arg);
    out[2] = (b.x - 0.5f * b.z) * img_w;
    out[3] = (b.y - 0.5f * b.w) * img_h;
    out[4] = (b.x + 0.5f * b.z) * img_w;
    out[5] = (b.y + 0.5f * b.w) * img_h;
    if (labels != nullptr) labels[row] = arg;
  }
}

}  // namespace

extern "C" int tfb200_detect_postprocess_f32(const float* logits, const float* boxes, const int64_t* sizes_hw,
                                             float* packed, int64_t* labels, int N, int Q, int C, void* stream) {
  if (!logits || !boxes || !sizes_hw || !packed) return TFB200_E_NULLPTR;
  if (N < 0 || Q < 0 || C <= 0) return TFB200_E_SHAPE;
  if (N == 0 || Q == 0) return 0;
  const int64_t rows = int64_t(N) * Q;
  const int grid = int((rows + 7) / 8);
  detect_postprocess_kernel<false><<<grid, 256, 0, cudaStream_t(stream)>>>(logits, boxes, sizes_hw, packed, labels, N, Q, C);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_detect_postprocess_softmax_f32(const float* logits, const float* boxes, const int64_t* sizes_hw,
                                                     float* packed, int64_t* labels, int N, int Q, int C, void* stream) {
  if (!logits || !boxes || !sizes_hw || !packed) return TFB200_E_NULLPTR;
  if (N < 0 || Q < 0 || C < 2) return TFB200_E_SHAPE;
  if (N == 0 || Q == 0) return 0;
  const int64_t rows = int64_t(N) * Q;
  const int grid = int((rows + 7) / 8);
  detect_postprocess_kernel<true><<<grid, 256, 0, cudaStream_t(stream)>>>(logits, boxes, sizes_hw, packed, labels, N, Q, C);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}
