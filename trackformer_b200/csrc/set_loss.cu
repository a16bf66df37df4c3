// SetCriterion on the device in three launches (sm_90a): matching cost, loss values + unit gradients, backward.
//
// The reference evaluates the Hungarian cost matrix and the focal / L1 / GIoU losses of the six decoder layers as
// chains of small PyTorch ops (src/trackformer/models/matcher.py:60-100, models/detr.py:213-328, util/misc.py:540-571,
// util/box_ops.py:24-61): ~25 kernels for the cost, ~70 for the losses and ~100 more in their autograd backward, every
// one of them launch-bound on [6, N, 300, 91] / [6, 20, 4] tensors.  Same arithmetic here:
//
//   match_cost      cost[r][t] = w_bbox * |b_r - g_t|_1 + w_class * (pos - neg)(sigmoid(logit[r][label_t])) - w_giou * GIoU
//   set_loss_rows   one warp per (layer, image, query) row: sigmoid focal loss of the row against its matched label
//                   (none = all zeros), its gradient, the row's arg-max (cardinality / class error); the matched rows also
//                   get the L1 and GIoU terms of their pair and the gradients of both with respect to the box
//   set_loss_final  one CTA per layer: fixed-order sums -> loss_ce / loss_bbox / loss_giou / cardinality_error (+ the
//                   class error of the last layer), all divided by the device-resident normaliser num_boxes
//   set_loss_bwd    grad_logits / grad_boxes from the three incoming gradient vectors [layers]
// Gradient formulas verified against autograd (fp64); torch's min / max / clamp subgradient
// conventions are kept (ties are measure-zero).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "launch_counter.h"

namespace {

struct Box { float x0, y0, x1, y1; };
__device__ __forceinline__ Box to_xyxy(const float4 b) {
  return Box{b.x - 0.5f * b.z, b.y - 0.5f * b.w, b.x + 0.5f * b.z, b.y + 0.5f * b.w};
}

__device__ __forceinline__ float giou_value(const Box a, const Box g) {
  const float area_a = (a.x1 - a.x0) * (a.y1 - a.y0), area_g = (g.x1 - g.x0) * (g.y1 - g.y0);
  const float iw = fmaxf(fminf(a.x1, g.x1) - fmaxf(a.x0, g.x0), 0.f), ih = fmaxf(fminf(a.y1, g.y1) - fmaxf(a.y0, g.y0), 0.f);
  const float inter = iw * ih, uni = area_a + area_g - inter;
  const float hw = fmaxf(fmaxf(a.x1, g.x1) - fminf(a.x0, g.x0), 0.f), hh = fmaxf(fmaxf(a.y1, g.y1) - fminf(a.y0, g.y0), 0.f);
  const float hull = hw * hh;
  return inter / uni - (hull - uni) / hull;
}

__device__ __forceinline__ float sigmoidf_(float x) { return 1.f / (1.f + expf(-x)); }

// ---- matching cost (focal class cost; matcher.py:60-75) ------------------------------------------------------------
__global__ void __launch_bounds__(256)
match_cost_kernel(const float* __restrict__ logits, const float* __restrict__ boxes, const int64_t* __restrict__ tgt_ids,
                  const float* __restrict__ tgt_boxes, float* __restrict__ cost, int64_t R, int C, int T, float w_class,
                  float w_bbox, float w_giou, float alpha, float gamma) {
  const int64_t i = int64_t(blockIdx.x) * 256 + threadIdx.x;
  if (i >= R * T) return;
  const int64_t r = i / T;
  const int t = int(i - r * T);
  const float p = sigmoidf_(__ldg(logits + r * C + __ldg(tgt_ids + t)));
  const float neg = (1.f - alpha) * powf(p, gamma) * (-logf(1.f - p + 1e-8f));
  const float pos = alpha * powf(1.f - p, gamma) * (-logf(p + 1e-8f));
  const float4 b = __ldg(reinterpret_cast<const float4*>(boxes) + r);
  const float4 g = __ldg(reinterpret_cast<const float4*>(tgt_boxes) + t);
  const float l1 = fabsf(b.x - g.x) + fabsf(b.y - g.y) + fabsf(b.z - g.z) + fabsf(b.w - g.w);
  cost[i] = w_bbox * l1 + w_class * (pos - neg) + w_giou * (-giou_value(to_xyxy(b), to_xyxy(g)));
}

// ---- per-row loss terms and unit gradients ---------------------------------------------------------------------------
// rows r = (k * B + b) * Q + q.  src / tgt [K][T]: columns off[b]..off[b+1]-1 are image b's (query, global box) pairs.
__global__ void __launch_bounds__(256)
set_loss_rows_kernel(const float* __restrict__ logits, const float* __restrict__ boxes, const int64_t* __restrict__ src,
                     const int64_t* __restrict__ tgt, const int64_t* __restrict__ tgt_ids,
                     const float* __restrict__ tgt_boxes, const int* __restrict__ off, float* __restrict__ unit_logits,
                     float* __restrict__ unit_l1, float* __restrict__ unit_giou, float* __restrict__ row_loss,
                     int* __restrict__ row_flags, float* __restrict__ pair_l1, float* __restrict__ pair_giou, int K,
                     int B, int Q, int C, int T, float alpha, float gamma) {
  const int lane = threadIdx.x & 31;
  const int64_t r = int64_t(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= int64_t(K) * B * Q) return;                               // warp-uniform
  const int q = int(r % Q), b = int((r / Q) % B), k = int(r / (int64_t(Q) * B));

  // which pair (if any) has this query as its source
  int hit = -1;
  for (int t = __ldg(off + b) + lane; t < __ldg(off + b + 1); t += 32)
    if (__ldg(src + int64_t(k) * T + t) == q) hit = t;
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) hit = max(hit, __shfl_xor_sync(0xffffffffu, hit, s));
  int64_t gidx = -1;
  int label = -1;
  if (hit >= 0) {
    gidx = __ldg(tgt + int64_t(k) * T + hit);
    label = int(__ldg(tgt_ids + gidx));
  }

  // sigmoid focal loss of the row (util/misc.py:540-571) and d/dlogit; arg-max with torch's first-maximum rule
  float sum = 0.f, best = -INFINITY;
  int arg = 0x7fffffff;
  for (int c = lane; c < C; c += 32) {
    const float x = __ldg(logits + r * C + c);
    const float t1 = (c == label) ? 1.f : 0.f;
    const float p = sigmoidf_(x);
    const float ce = fmaxf(x, 0.f) - x * t1 + log1pf(expf(-fabsf(x)));
    const float qt = 1.f - (p * t1 + (1.f - p) * (1.f - t1));
    const float at = alpha >= 0.f ? alpha * t1 + (1.f - alpha) * (1.f - t1) : 1.f;
    const float mod = gamma == 2.f ? qt * qt : powf(qt, gamma);
    const float modm1 = gamma == 2.f ? qt : powf(qt, gamma - 1.f);
    const float dpt = (2.f * t1 - 1.f) * p * (1.f - p);
    sum += at * mod * ce;
    unit_logits[r * C + c] = at * (-gamma * modm1 * dpt * ce + mod * (p - t1));
    if (x > best) { best = x; arg = c; }
  }
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    sum += __shfl_xor_sync(0xffffffffu, sum, s);
    const float ob = __shfl_xor_sync(0xffffffffu, best, s);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, s);
    if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
  }
  if (lane != 0) return;
  row_loss[r] = sum;
  row_flags[r] = (arg != C - 1 ? 1 : 0) | ((hit >= 0 && arg == label) ? 2 : 0);

  float4 u1 = make_float4(0.f, 0.f, 0.f, 0.f), ug = u1;
  if (hit >= 0) {
    const float4 bb = __ldg(reinterpret_cast<const float4*>(boxes) + r);
    const float4 gg = __ldg(reinterpret_cast<const float4*>(tgt_boxes) + gidx);
    // L1 (detr.py:302-304): sum |b - g|, gradient sign(b - g)
    pair_l1[int64_t(k) * T + hit] = fabsf(bb.x - gg.x) + fabsf(bb.y - gg.y) + fabsf(bb.z - gg.z) + fabsf(bb.w - gg.w);
    u1 = make_float4(float((bb.x > gg.x) - (bb.x < gg.x)), float((bb.y > gg.y) - (bb.y < gg.y)),
                     float((bb.z > gg.z) - (bb.z < gg.z)), float((bb.w > gg.w) - (bb.w < gg.w)));
    // 1 - GIoU (util/box_ops.py:24-61) and its gradient with respect to (cx, cy, w, h)
    const Box a = to_xyxy(bb), g = to_xyxy(gg);
    const float aw = a.x1 - a.x0, ah = a.y1 - a.y0;
    const float area_a = aw * ah, area_g = (g.x1 - g.x0) * (g.y1 - g.y0);
    const float iwr = fminf(a.x1, g.x1) - fmaxf(a.x0, g.x0), ihr = fminf(a.y1, g.y1) - fmaxf(a.y0, g.y0);
    const float iw = fmaxf(iwr, 0.f), ih = fmaxf(ihr, 0.f);
    const float inter = iw * ih, uni = area_a + area_g - inter;
    const float hwr = fmaxf(a.x1, g.x1) - fminf(a.x0, g.x0), hhr = fmaxf(a.y1, g.y1) - fminf(a.y0, g.y0);
    const float hw = fmaxf(hwr, 0.f), hh = fmaxf(hhr, 0.f);
    const float hull = hw * hh;
    pair_giou[int64_t(k) * T + hit] = 1.f - (inter / uni - (hull - uni) / hull);
    const float giw = iwr >= 0.f ? 1.f : 0.f, gih = ihr >= 0.f ? 1.f : 0.f;
    const float ghw = hwr >= 0.f ? 1.f : 0.f, ghh = hhr >= 0.f ? 1.f : 0.f;
    // partial derivatives with respect to (x0, y0, x1, y1) of the predicted box
    const float d_iw[4] = {a.x0 > g.x0 ? -giw : 0.f, 0.f, a.x1 < g.x1 ? giw : 0.f, 0.f};
    const float d_ih[4] = {0.f, a.y0 > g.y0 ? -gih : 0.f, 0.f, a.y1 < g.y1 ? gih : 0.f};
    const float d_hw[4] = {a.x0 < g.x0 ? -ghw : 0.f, 0.f, a.x1 > g.x1 ? ghw : 0.f, 0.f};
    const float d_hh[4] = {0.f, a.y0 < g.y0 ? -ghh : 0.f, 0.f, a.y1 > g.y1 ? ghh : 0.f};
    const float d_area[4] = {-ah, -aw, ah, aw};
    float dg[4];
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float d_inter = d_iw[c] * ih + iw * d_ih[c];
      const float d_uni = d_area[c] - d_inter;
      const float d_hull = d_hw[c] * hh + hw * d_hh[c];
      dg[c] = (d_inter * uni - inter * d_uni) / (uni * uni) + (d_uni * hull - uni * d_hull) / (hull * hull);
    }
    ug = make_float4(-(dg[0] + dg[2]), -(dg[1] + dg[3]), -0.5f * (dg[2] - dg[0]), -0.5f * (dg[3] - dg[1]));
  }
  reinterpret_cast<float4*>(unit_l1)[r] = u1;
  reinterpret_cast<float4*>(unit_giou)[r] = ug;
}

// ---- per-layer totals: one CTA per layer, fixed summation order ------------------------------------------------------
__device__ float block_sum(float v, float* sh) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
  __syncthreads();
  if (lane == 0) sh[w] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < int(blockDim.x >> 5); ++i) t += sh[i];
  return t;
}

__global__ void __launch_bounds__(256)
set_loss_final_kernel(const float* __restrict__ row_loss, const int* __restrict__ row_flags,
                      const float* __restrict__ pair_l1, const float* __restrict__ pair_giou,
                      const float* __restrict__ n_gt, const float* __restrict__ num_boxes, float* __restrict__ out,
                      int K, int B, int Q, int T) {
  __shared__ float sh[8];
  const int k = blockIdx.x;
  const float nb = __ldg(num_boxes);
  float ce = 0.f, l1 = 0.f, gi = 0.f, hits = 0.f;
  for (int i = threadIdx.x; i < B * Q; i += blockDim.x) {
    ce += row_loss[int64_t(k) * B * Q + i];
    hits += (row_flags[int64_t(k) * B * Q + i] & 2) ? 1.f : 0.f;
  }
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    l1 += pair_l1[int64_t(k) * T + t];
    gi += pair_giou[int64_t(k) * T + t];
  }
  ce = block_sum(ce, sh);
  l1 = block_sum(l1, sh);
  gi = block_sum(gi, sh);
  hits = block_sum(hits, sh);
  float card = 0.f;
  for (int b = 0; b < B; ++b) {
    float n = 0.f;
    for (int i = threadIdx.x; i < Q; i += blockDim.x) n += (row_flags[(int64_t(k) * B + b) * Q + i] & 1) ? 1.f : 0.f;
    n = block_sum(n, sh);
    card += fabsf(n - __ldg(n_gt + b));
  }
  if (threadIdx.x == 0) {
    out[0 * K + k] = ce / nb;                 // loss_ce   (= focal.mean(1).sum() / num_boxes * Q, detr.py:265-272)
    out[1 * K + k] = l1 / nb;                 // loss_bbox
    out[2 * K + k] = gi / nb;                 // loss_giou
    out[3 * K + k] = card / float(B);         // cardinality_error
    out[4 * K + k] = 100.f - 100.f * hits / float(T > 0 ? T : 1);      // class_error (meaningful for the last layer)
  }
}

// ---- backward ----------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
set_loss_bwd_kernel(const float* __restrict__ unit_logits, const float* __restrict__ unit_l1,
                    const float* __restrict__ unit_giou, const float* __restrict__ g_ce, const float* __restrict__ g_l1,
                    const float* __restrict__ g_giou, const float* __restrict__ num_boxes, float* __restrict__ grad_logits,
                    float* __restrict__ grad_boxes, int64_t rows_per_layer, int C, int64_t R) {
  const int64_t i = int64_t(blockIdx.x) * 256 + threadIdx.x;
  const float inv = 1.f / __ldg(num_boxes);
  if (i < R * C) {
    const int k = int((i / C) / rows_per_layer);
    grad_logits[i] = unit_logits[i] * (__ldg(g_ce + k) * inv);
  }
  if (i < R * 4) {
    const int k = int((i >> 2) / rows_per_layer);
    grad_boxes[i] = (unit_l1[i] * __ldg(g_l1 + k) + unit_giou[i] * __ldg(g_giou + k)) * inv;
  }
}

}  // namespace

extern "C" int tfb200_match_cost_f32(const float* logits, const float* boxes, const int64_t* tgt_ids,
                                     const float* tgt_boxes, float* cost, int64_t R, int C, int T, float w_class,
                                     float w_bbox, float w_giou, float alpha, float gamma, void* stream) {
  if (!logits || !boxes || !tgt_ids || !tgt_boxes || !cost) return TFB200_E_NULLPTR;
  if (R < 0 || C <= 0 || T <= 0) return TFB200_E_SHAPE;
  if (R == 0) return 0;
  const int64_t n = R * T;
  match_cost_kernel<<<unsigned((n + 255) / 256), 256, 0, cudaStream_t(stream)>>>(logits, boxes, tgt_ids, tgt_boxes, cost, R, C,
                                                                                T, w_class, w_bbox, w_giou, alpha, gamma);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_set_loss_fwd_f32(const float* logits, const float* boxes, const int64_t* src, const int64_t* tgt,
                                       const int64_t* tgt_ids, const float* tgt_boxes, const int* offsets,
                                       const float* n_gt, const float* num_boxes, float* unit_logits, float* unit_l1,
                                       float* unit_giou, float* row_loss, int* row_flags, float* pair_l1, float* pair_giou,
                                       float* out5k, int K, int B, int Q, int C, int T, float alpha, float gamma,
                                       void* stream) {
  if (!logits || !boxes || !src || !tgt || !tgt_ids || !tgt_boxes || !offsets || !n_gt || !num_boxes || !unit_logits ||
      !unit_l1 || !unit_giou || !row_loss || !row_flags || !pair_l1 || !pair_giou || !out5k)
    return TFB200_E_NULLPTR;
  if (K <= 0 || B <= 0 || Q <= 0 || C <= 0 || T <= 0) return TFB200_E_SHAPE;
  cudaStream_t st = cudaStream_t(stream);
  const int64_t R = int64_t(K) * B * Q;
  set_loss_rows_kernel<<<unsigned((R + 7) / 8), 256, 0, st>>>(logits, boxes, src, tgt, tgt_ids, tgt_boxes, offsets,
                                                              unit_logits, unit_l1, unit_giou, row_loss, row_flags, pair_l1,
                                                              pair_giou, K, B, Q, C, T, alpha, gamma);
  set_loss_final_kernel<<<K, 256, 0, st>>>(row_loss, row_flags, pair_l1, pair_giou, n_gt, num_boxes, out5k, K, B, Q, T);
  msda_b200_count_launches(2);
  return int(cudaGetLastError());
}

extern "C" int tfb200_set_loss_bwd_f32(const float* unit_logits, const float* unit_l1, const float* unit_giou,
                                       const float* g_ce, const float* g_l1, const float* g_giou, const float* num_boxes,
                                       float* grad_logits, float* grad_boxes, int K, int B, int Q, int C, void* stream) {
  if (!unit_logits || !unit_l1 || !unit_giou || !g_ce || !g_l1 || !g_giou || !num_boxes || !grad_logits || !grad_boxes)
    return TFB200_E_NULLPTR;
  if (K <= 0 || B <= 0 || Q <= 0 || C <= 0) return TFB200_E_SHAPE;
  const int64_t R = int64_t(K) * B * Q;
  const int64_t n = R * (C > 4 ? C : 4);
  set_loss_bwd_kernel<<<unsigned((n + 255) / 256), 256, 0, cudaStream_t(stream)>>>(
      unit_logits, unit_l1, unit_giou, g_ce, g_l1, g_giou, num_boxes, grad_logits, grad_boxes, int64_t(B) * Q, C, R);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}
