// Two-stage Deformable DETR on sm_90a: the encoder proposals and the top-k query selection of
// src/trackformer/models/deformable_transformer.py:77-122, 180-194 (routines in two_stage_core.h).
//
//   tfb200_two_stage_proposals_f32  one launch: proposal logits + valid flags of every token, and the masked memory copy
//   tfb200_two_stage_mask_rows_f32  one launch: rows of [B*S][C] times the valid flag (masked memory of a memoised dense
//                                   geometry; the gradient of the masking)
//   tfb200_two_stage_select_f32     one launch, one CTA per image: top-k by class-0 logit, gathered boxes, reference
//                                   points and sine embedding; k is static, nothing is read back (graph-capturable)
#include <cuda_runtime.h>

#include "two_stage_core.h"
#include "launch_counter.h"

using namespace tfb200_two_stage;

namespace {

constexpr int kPropThreads = 256;          // tokens per CTA

__global__ void __launch_bounds__(kPropThreads) two_stage_proposals_kernel(ProposalParams p) {
  __shared__ int vw[kMaxLevels], vh[kMaxLevels];
  __shared__ uint8_t ok[kPropThreads];
  const int b = blockIdx.y, s0 = blockIdx.x * kPropThreads;
  ts_valid_counts(p, b, vw, vh);
  const int s = s0 + threadIdx.x;
  if (s < p.S) ok[threadIdx.x] = ts_proposal(p, b, s, vw, vh);
  if (p.memory == nullptr) return;
  __syncthreads();
  const int rows = min(kPropThreads, p.S - s0), c4 = p.C / 4;
  const float4* src = reinterpret_cast<const float4*>(p.memory + (size_t(b) * p.S + s0) * p.C);
  float4* dst = reinterpret_cast<float4*>(p.masked + (size_t(b) * p.S + s0) * p.C);
  for (int e = threadIdx.x; e < rows * c4; e += kPropThreads) {
    const float4 v = src[e];
    dst[e] = ok[e / c4] ? v : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

__global__ void two_stage_mask_rows_kernel(const float4* __restrict__ x, const uint8_t* __restrict__ valid,
                                           float4* __restrict__ y, int64_t n4, int c4) {
  for (int64_t e = blockIdx.x * int64_t(blockDim.x) + threadIdx.x; e < n4; e += int64_t(gridDim.x) * blockDim.x)
    y[e] = valid[e / c4] ? x[e] : make_float4(0.f, 0.f, 0.f, 0.f);
}

__global__ void __launch_bounds__(kSelThreads) two_stage_select_kernel(SelectParams p) {
  __shared__ SelectShared sh;
  ts_select(p, blockIdx.x, sh);
  ts_select_outputs(p, blockIdx.x, sh);
}

}  // namespace

extern "C" {

int tfb200_two_stage_proposals_f32(const uint8_t* mask, const float* memory, float* masked, float* prop,
                                   uint8_t* valid, int B, int S, int L, int C, const int* hw, void* stream) {
  if (!prop || !valid || !hw || (memory && !masked)) return TFB200_E_NULLPTR;
  if (int rc = ts_check_proposals(B, S, L, memory ? C : 0, hw)) return rc;
  if (B > 65535) return TFB200_E_SHAPE;
  if (memory && ((reinterpret_cast<uintptr_t>(memory) | reinterpret_cast<uintptr_t>(masked)) & 15u)) return TFB200_E_SHAPE;
  ProposalParams p{};
  p.B = B; p.S = S; p.L = L; p.C = memory ? C : 0;
  ts_levels(p, hw);
  p.mask = mask; p.memory = memory; p.masked = masked; p.prop = prop; p.valid = valid;
  two_stage_proposals_kernel<<<dim3(unsigned((S + kPropThreads - 1) / kPropThreads), unsigned(B)), kPropThreads, 0,
                               cudaStream_t(stream)>>>(p);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

int tfb200_two_stage_mask_rows_f32(const float* x, const uint8_t* valid, float* y, int64_t rows, int C, void* stream) {
  if (!x || !valid || !y) return TFB200_E_NULLPTR;
  if (rows < 0 || C <= 0 || C % 4 != 0) return TFB200_E_SHAPE;
  if ((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 15u) return TFB200_E_SHAPE;
  const int64_t n4 = rows * (C / 4);
  if (n4 == 0) return 0;
  const int64_t blocks = (n4 + 255) / 256;
  two_stage_mask_rows_kernel<<<unsigned(blocks < 4096 ? blocks : 4096), 256, 0, cudaStream_t(stream)>>>(
      reinterpret_cast<const float4*>(x), valid, reinterpret_cast<float4*>(y), n4, C / 4);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

int tfb200_two_stage_select_f32(const float* logits, const float* unact, const float* dim_t, uint32_t* keys,
                                int64_t* index, float* boxes, float* ref, float* embed, int B, int S, int C, int k,
                                void* stream) {
  if (!logits || !unact || !dim_t || !keys || !index || !boxes || !ref || !embed) return TFB200_E_NULLPTR;
  if (int rc = ts_check_select(B, S, C, k)) return rc;
  SelectParams p{};
  p.B = B; p.S = S; p.C = C; p.k = k;
  p.logits = logits; p.unact = unact; p.dim_t = dim_t; p.keys = keys;
  p.index = index; p.boxes = boxes; p.ref = ref; p.embed = embed;
  two_stage_select_kernel<<<unsigned(B), kSelThreads, 0, cudaStream_t(stream)>>>(p);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

}  // extern "C"
