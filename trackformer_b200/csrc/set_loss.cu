// SetCriterion on the device in three launches (sm_90a): matching cost, loss values + unit gradients, backward.
//
// The reference evaluates the Hungarian cost matrix and the class / L1 / GIoU losses of the six decoder layers as
// chains of small PyTorch ops (src/trackformer/models/matcher.py:60-100, models/detr.py:172-328, util/misc.py:540-571,
// util/box_ops.py:24-61): ~25 kernels for the cost, ~70 for the losses and ~100 more in their autograd backward, every
// one of them launch-bound on [6, N, 300, 91] / [6, 20, 4] tensors.  Same arithmetic here:
//
//   match_cost      cost[r][t] = w_bbox * |b_r - g_t|_1 + w_class * class_cost(r, label_t) - w_giou * GIoU
//                   (match_cost_track: the same, with track queries pinned to their identity's box, matcher.py:112-128)
//   set_loss_rows   one warp per (layer, image, query) row: the class loss of the row against its matched label, its
//                   gradient, the row's arg-max (cardinality / class error); the matched rows also get the L1 and GIoU
//                   terms of their pair and the gradients of both with respect to the box; rows outside the optional
//                   validity mask (filler track queries) contribute nothing and get zero gradients
//   set_loss_final  one CTA per layer: fixed-order sums -> loss_ce / loss_bbox / loss_giou / cardinality_error (+ the
//                   class error of the last layer); box terms divided by the device-resident normaliser num_boxes
//   set_loss_bwd    grad_logits / grad_boxes from the three incoming gradient vectors [layers]
//
// The classifier is a compile-time policy of these kernels; everything else (box terms, pair lookup, arg-max, per-layer
// sums, filler masking) is shared:
//   FocalCls    sigmoid focal loss over C classes (focal_loss: true, matcher.py:70-75, detr.py:213-240);
//               loss_ce = sum of the rows' focal terms / num_boxes
//   SoftmaxCls  weighted cross-entropy over C = classes + 1 ("no object" last; focal_loss: false, matcher.py:77,
//               detr.py:172-211): cost -softmax(logit_r)[label_t] from one log-sum-exp per row; loss_ce[k] =
//               sum_r w_r ce_r / sum_r w_r (empty_weight: 1 for a matched row, eos_coef for no-object; a false-positive
//               track query keeps no-object but its ce is scaled by 1 / eos_coef and counts 1 in the normaliser)
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

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) v += __shfl_xor_sync(0xffffffffu, v, s);
  return v;
}

// arg-max over a warp with torch's first-maximum rule
__device__ __forceinline__ void warp_argmax(float& best, int& arg) {
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) {
    const float ob = __shfl_xor_sync(0xffffffffu, best, s);
    const int oa = __shfl_xor_sync(0xffffffffu, arg, s);
    if (ob > best || (ob == best && oa < arg)) { best = ob; arg = oa; }
  }
}

// ---- classifier policies ---------------------------------------------------------------------------------------------
// row_stats   (kRowStats only) per-row statistic the matching cost needs, computed once per row by a warp
// cost        class cost of row r against class `label`
// row_terms   one warp: the row's class loss (lane 0), its normaliser weight, its arg-max, and the unit gradient
//             d(loss row) / d(logit) written for every class
struct FocalCls {
  float alpha, gamma;
  static constexpr bool kRowStats = false;         // the cost needs nothing beyond the entry itself
  static constexpr bool kLayerNorm = false;        // loss_ce is normalised by num_boxes

  // matcher.py:60-75
  __device__ __forceinline__ float cost(const float* __restrict__ logits, int64_t r, int C, int label, float2) const {
    const float p = sigmoidf_(__ldg(logits + r * C + label));
    const float neg = (1.f - alpha) * powf(p, gamma) * (-logf(1.f - p + 1e-8f));
    const float pos = alpha * powf(1.f - p, gamma) * (-logf(p + 1e-8f));
    return pos - neg;
  }

  // sigmoid focal loss of the row (util/misc.py:540-571) against its label (-1: none = all zeros)
  __device__ __forceinline__ void row_terms(const float* __restrict__ x, float* __restrict__ unit, int C, int label,
                                            int lane, int /*pin*/, float& loss, float& norm, int& arg) const {
    float sum = 0.f, best = -INFINITY;
    arg = 0x7fffffff;
    for (int c = lane; c < C; c += 32) {
      const float v = __ldg(x + c);
      const float t1 = (c == label) ? 1.f : 0.f;
      const float p = sigmoidf_(v);
      const float ce = fmaxf(v, 0.f) - v * t1 + log1pf(expf(-fabsf(v)));
      const float qt = 1.f - (p * t1 + (1.f - p) * (1.f - t1));
      const float at = alpha >= 0.f ? alpha * t1 + (1.f - alpha) * (1.f - t1) : 1.f;
      const float mod = gamma == 2.f ? qt * qt : powf(qt, gamma);
      const float modm1 = gamma == 2.f ? qt : powf(qt, gamma - 1.f);
      const float dpt = (2.f * t1 - 1.f) * p * (1.f - p);
      sum += at * mod * ce;
      unit[c] = at * (-gamma * modm1 * dpt * ce + mod * (p - t1));
      if (v > best) { best = v; arg = c; }
    }
    loss = warp_sum(sum);
    warp_argmax(best, arg);
    norm = 0.f;
  }
};

struct SoftmaxCls {
  float eos_coef;
  int fp_full_weight;                              // false-positive track queries (pin -2) keep their full weight

  static constexpr bool kRowStats = true;          // (max, sum exp(x - max)) of the row
  static constexpr bool kLayerNorm = true;         // loss_ce[k] is normalised by the layer's weight sum

  __device__ __forceinline__ float2 row_stats(const float* __restrict__ x, int C, int lane) const {
    float m = -INFINITY;
    for (int c = lane; c < C; c += 32) m = fmaxf(m, __ldg(x + c));
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
    float e = 0.f;
    for (int c = lane; c < C; c += 32) e += expf(__ldg(x + c) - m);
    return make_float2(m, warp_sum(e));
  }

  // matcher.py:77: -softmax(logit_r)[label]
  __device__ __forceinline__ float cost(const float* __restrict__ logits, int64_t r, int C, int label,
                                        float2 st) const {
    return -(expf(__ldg(logits + r * C + label) - st.x) / st.y);
  }

  // weighted cross-entropy of the row (detr.py:185-204): target = label, or no-object (C - 1) when unmatched
  __device__ __forceinline__ void row_terms(const float* __restrict__ x, float* __restrict__ unit, int C, int label,
                                            int lane, int pin, float& loss, float& norm, int& arg) const {
    float best = -INFINITY;
    arg = 0x7fffffff;
    for (int c = lane; c < C; c += 32) {
      const float v = __ldg(x + c);
      if (v > best) { best = v; arg = c; }
    }
    warp_argmax(best, arg);                        // best = row maximum on every lane
    float e = 0.f;
    for (int c = lane; c < C; c += 32) e += expf(__ldg(x + c) - best);
    e = warp_sum(e);
    const int y = label >= 0 ? label : C - 1;
    const bool fal_pos = label < 0 && fp_full_weight && pin == -2;
    const float w = label >= 0 ? 1.f : eos_coef;                     // empty_weight[y]
    const float wn = fal_pos ? w * (1.f / eos_coef) : w;             // ce[fp] *= 1 / eos_coef
    norm = fal_pos ? 1.f : w;                                        // target class 0 for the normaliser
    const float inv = 1.f / e;
    for (int c = lane; c < C; c += 32) {
      const float p = expf(__ldg(x + c) - best) * inv;
      unit[c] = wn * (p - (c == y ? 1.f : 0.f));
    }
    loss = wn * ((best - __ldg(x + y)) + logf(e));
  }
};

// ---- matching cost ------------------------------------------------------------------------------------------------------
__device__ __forceinline__ float pair_cost(const float* __restrict__ boxes, const float* __restrict__ tgt_boxes,
                                           int64_t r, int t, float cls, float w_class, float w_bbox, float w_giou) {
  const float4 b = __ldg(reinterpret_cast<const float4*>(boxes) + r);
  const float4 g = __ldg(reinterpret_cast<const float4*>(tgt_boxes) + t);
  const float l1 = fabsf(b.x - g.x) + fabsf(b.y - g.y) + fabsf(b.z - g.z) + fabsf(b.w - g.w);
  return w_bbox * l1 + w_class * cls + w_giou * (-giou_value(to_xyxy(b), to_xyxy(g)));
}

// one thread per (row, box): the classifiers whose cost needs no per-row statistic
__global__ void __launch_bounds__(256)
match_cost_kernel(const float* __restrict__ logits, const float* __restrict__ boxes, const int64_t* __restrict__ tgt_ids,
                  const float* __restrict__ tgt_boxes, float* __restrict__ cost, int64_t R, int C, int T, float w_class,
                  float w_bbox, float w_giou, FocalCls cls) {
  const int64_t i = int64_t(blockIdx.x) * 256 + threadIdx.x;
  if (i >= R * T) return;
  const int64_t r = i / T;
  const int t = int(i - r * T);
  cost[i] = pair_cost(boxes, tgt_boxes, r, t, cls.cost(logits, r, C, int(__ldg(tgt_ids + t)), float2()), w_class,
                      w_bbox, w_giou);
}

// The cost by blocks of kTrackRows rows of one (layer, image), optionally with the track-query rewrite of
// matcher.py:112-128 applied in the same pass.  row_pin [B*Q] (shared by all layers; nullptr: every row free): -1 free
// row; c in [0, T) row pinned to global box c (its row becomes +inf except -1 at c, and column c becomes +inf for every
// other row of the image); any other value excluded row (all +inf: false-positive or filler track query).  With a pin
// the CTA first marks the image's pinned columns in shared memory; with a per-row statistic (softmax) it is computed
// once per row, a warp per row, before the (row, box) entries.
constexpr int kTrackRows = 16;

template <class Cls>
__global__ void __launch_bounds__(256)
match_cost_rows_kernel(const float* __restrict__ logits, const float* __restrict__ boxes,
                       const int64_t* __restrict__ tgt_ids, const float* __restrict__ tgt_boxes,
                       const int* __restrict__ row_pin, float* __restrict__ cost, int B, int Q, int C, int T,
                       float w_class, float w_bbox, float w_giou, Cls cls) {
  extern __shared__ unsigned char col_pinned[];                      // [T] (with row_pin)
  __shared__ float2 stats[kTrackRows];
  const int chunks = (Q + kTrackRows - 1) / kTrackRows;
  const int chunk = int(blockIdx.x % unsigned(chunks));
  const int64_t kb = blockIdx.x / unsigned(chunks);                  // layer * B + image
  const int b = int(kb % B);
  const int* pin_b = row_pin != nullptr ? row_pin + int64_t(b) * Q : nullptr;
  if (pin_b != nullptr) {
    for (int t = threadIdx.x; t < T; t += blockDim.x) col_pinned[t] = 0;
    __syncthreads();
    for (int q = threadIdx.x; q < Q; q += blockDim.x) {
      const int p = __ldg(pin_b + q);
      if (p >= 0 && p < T) col_pinned[p] = 1;
    }
  }
  const int q0 = chunk * kTrackRows;
  const int rows = min(kTrackRows, Q - q0);
  if constexpr (Cls::kRowStats) {
    const int lane = threadIdx.x & 31;
    for (int j = threadIdx.x >> 5; j < rows; j += blockDim.x >> 5) {
      const float2 st = cls.row_stats(logits + (kb * Q + q0 + j) * C, C, lane);
      if (lane == 0) stats[j] = st;
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < rows * T; i += blockDim.x) {
    const int j = i / T, t = i % T;
    const int q = q0 + j;
    const int64_t r = kb * Q + q;
    const int pin = pin_b != nullptr ? __ldg(pin_b + q) : -1;
    float v;
    if (pin >= 0 && pin < T) v = t == pin ? -1.f : INFINITY;
    else if (pin != -1 || (pin_b != nullptr && col_pinned[t])) v = INFINITY;
    else v = pair_cost(boxes, tgt_boxes, r, t, cls.cost(logits, r, C, int(__ldg(tgt_ids + t)), stats[j]), w_class,
                       w_bbox, w_giou);
    cost[r * T + t] = v;
  }
}

// ---- per-row loss terms and unit gradients ---------------------------------------------------------------------------
// rows r = (k * B + b) * Q + q.  src / tgt [K][T]: columns off[b]..off[b+1]-1 are image b's (query, global box) pairs.
// row_pin [B*Q] (optional) is passed to the classifier (false-positive track queries); row_norm [R] receives the
// classifier's normaliser weight of each row (classifiers with a per-layer normaliser only).
template <class Cls>
__global__ void __launch_bounds__(256)
set_loss_rows_kernel(const float* __restrict__ logits, const float* __restrict__ boxes, const int64_t* __restrict__ src,
                     const int64_t* __restrict__ tgt, const int64_t* __restrict__ tgt_ids,
                     const float* __restrict__ tgt_boxes, const int* __restrict__ off,
                     const uint8_t* __restrict__ row_valid, const int* __restrict__ row_pin,
                     float* __restrict__ unit_logits, float* __restrict__ unit_l1, float* __restrict__ unit_giou,
                     float* __restrict__ row_loss, float* __restrict__ row_norm, int* __restrict__ row_flags,
                     float* __restrict__ pair_l1, float* __restrict__ pair_giou, int K, int B, int Q, int C, int T,
                     Cls cls) {
  const int lane = threadIdx.x & 31;
  const int64_t r = int64_t(blockIdx.x) * 8 + (threadIdx.x >> 5);
  if (r >= int64_t(K) * B * Q) return;                               // warp-uniform
  const int q = int(r % Q), b = int((r / Q) % B), k = int(r / (int64_t(Q) * B));
  if (row_valid != nullptr && !__ldg(row_valid + int64_t(b) * Q + q)) {
    // masked row (filler track query): no loss, no cardinality count, zero unit gradients, no pair terms
    for (int c = lane; c < C; c += 32) unit_logits[r * C + c] = 0.f;
    if (lane == 0) {
      row_loss[r] = 0.f;
      if constexpr (Cls::kLayerNorm) row_norm[r] = 0.f;
      row_flags[r] = 0;
      reinterpret_cast<float4*>(unit_l1)[r] = make_float4(0.f, 0.f, 0.f, 0.f);
      reinterpret_cast<float4*>(unit_giou)[r] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
    return;                                                          // warp-uniform
  }

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

  // class loss of the row and d/dlogit; arg-max with torch's first-maximum rule
  const int pin = row_pin != nullptr ? __ldg(row_pin + int64_t(b) * Q + q) : -1;
  float loss, norm;
  int arg;
  cls.row_terms(logits + r * C, unit_logits + r * C, C, label, lane, pin, loss, norm, arg);
  if (lane != 0) return;
  row_loss[r] = loss;
  if constexpr (Cls::kLayerNorm) row_norm[r] = norm;
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

// kLayerNorm: loss_ce[k] is divided by the layer's sum of row_norm, which is also written to out[5][k]
template <bool kLayerNorm>
__global__ void __launch_bounds__(256)
set_loss_final_kernel(const float* __restrict__ row_loss, const float* __restrict__ row_norm,
                      const int* __restrict__ row_flags, const float* __restrict__ pair_l1,
                      const float* __restrict__ pair_giou, const float* __restrict__ n_gt,
                      const float* __restrict__ num_boxes, float* __restrict__ out, int K, int B, int Q, int T) {
  __shared__ float sh[8];
  const int k = blockIdx.x;
  const float nb = __ldg(num_boxes);
  float ce = 0.f, l1 = 0.f, gi = 0.f, hits = 0.f, wsum = 0.f;
  for (int i = threadIdx.x; i < B * Q; i += blockDim.x) {
    ce += row_loss[int64_t(k) * B * Q + i];
    if constexpr (kLayerNorm) wsum += row_norm[int64_t(k) * B * Q + i];
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
  if constexpr (kLayerNorm) wsum = block_sum(wsum, sh);
  float card = 0.f;
  for (int b = 0; b < B; ++b) {
    float n = 0.f;
    for (int i = threadIdx.x; i < Q; i += blockDim.x) n += (row_flags[(int64_t(k) * B + b) * Q + i] & 1) ? 1.f : 0.f;
    n = block_sum(n, sh);
    card += fabsf(n - __ldg(n_gt + b));
  }
  if (threadIdx.x == 0) {
    // loss_ce: focal.mean(1).sum() / num_boxes * Q (detr.py:265-272), or sum w_r ce_r / sum w_r (detr.py:204)
    out[0 * K + k] = kLayerNorm ? ce / wsum : ce / nb;
    out[1 * K + k] = l1 / nb;                 // loss_bbox
    out[2 * K + k] = gi / nb;                 // loss_giou
    out[3 * K + k] = card / float(B);         // cardinality_error
    out[4 * K + k] = 100.f - 100.f * hits / float(T > 0 ? T : 1);      // class_error (meaningful for the last layer)
    if constexpr (kLayerNorm) out[5 * K + k] = wsum;                   // the class-loss normaliser (backward)
  }
}

// ---- backward ----------------------------------------------------------------------------------------------------------
// ce_norm[k * ce_stride]: the class-loss normaliser of layer k (stride 0: the scalar num_boxes)
__global__ void __launch_bounds__(256)
set_loss_bwd_kernel(const float* __restrict__ unit_logits, const float* __restrict__ unit_l1,
                    const float* __restrict__ unit_giou, const float* __restrict__ g_ce, const float* __restrict__ g_l1,
                    const float* __restrict__ g_giou, const float* __restrict__ num_boxes,
                    const float* __restrict__ ce_norm, int ce_stride, float* __restrict__ grad_logits,
                    float* __restrict__ grad_boxes, int64_t rows_per_layer, int C, int64_t R) {
  const int64_t i = int64_t(blockIdx.x) * 256 + threadIdx.x;
  const float inv = 1.f / __ldg(num_boxes);
  if (i < R * C) {
    const int k = int((i / C) / rows_per_layer);
    grad_logits[i] = unit_logits[i] * (__ldg(g_ce + k) * (1.f / __ldg(ce_norm + int64_t(k) * ce_stride)));
  }
  if (i < R * 4) {
    const int k = int((i >> 2) / rows_per_layer);
    grad_boxes[i] = (unit_l1[i] * __ldg(g_l1 + k) + unit_giou[i] * __ldg(g_giou + k)) * inv;
  }
}

template <class Cls>
int match_cost_rows(const float* logits, const float* boxes, const int64_t* tgt_ids, const float* tgt_boxes,
                    const int* row_pin, float* cost, int K, int B, int Q, int C, int T, float w_class, float w_bbox,
                    float w_giou, Cls cls, void* stream) {
  const int chunks = (Q + kTrackRows - 1) / kTrackRows;
  const int64_t grid = int64_t(K) * B * chunks;
  if (grid > 0x7fffffff) return TFB200_E_SHAPE;
  match_cost_rows_kernel<Cls><<<unsigned(grid), 256, row_pin != nullptr ? size_t(T) : 0, cudaStream_t(stream)>>>(
      logits, boxes, tgt_ids, tgt_boxes, row_pin, cost, B, Q, C, T, w_class, w_bbox, w_giou, cls);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

}  // namespace

extern "C" int tfb200_match_cost_f32(const float* logits, const float* boxes, const int64_t* tgt_ids,
                                     const float* tgt_boxes, float* cost, int64_t R, int C, int T, float w_class,
                                     float w_bbox, float w_giou, float alpha, float gamma, void* stream) {
  if (!logits || !boxes || !tgt_ids || !tgt_boxes || !cost) return TFB200_E_NULLPTR;
  if (R < 0 || C <= 0 || T <= 0) return TFB200_E_SHAPE;
  if (R == 0) return 0;
  const int64_t n = R * T;
  match_cost_kernel<<<unsigned((n + 255) / 256), 256, 0, cudaStream_t(stream)>>>(
      logits, boxes, tgt_ids, tgt_boxes, cost, R, C, T, w_class, w_bbox, w_giou, FocalCls{alpha, gamma});
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_match_cost_track_f32(const float* logits, const float* boxes, const int64_t* tgt_ids,
                                           const float* tgt_boxes, const int* row_pin, float* cost, int K, int B, int Q,
                                           int C, int T, float w_class, float w_bbox, float w_giou, float alpha,
                                           float gamma, void* stream) {
  if (!logits || !boxes || !tgt_ids || !tgt_boxes || !row_pin || !cost) return TFB200_E_NULLPTR;
  if (K < 0 || B <= 0 || Q <= 0 || C <= 0 || T <= 0 || T > 48 * 1024) return TFB200_E_SHAPE;
  if (K == 0) return 0;
  return match_cost_rows(logits, boxes, tgt_ids, tgt_boxes, row_pin, cost, K, B, Q, C, T, w_class, w_bbox, w_giou,
                         FocalCls{alpha, gamma}, stream);
}

extern "C" int tfb200_match_cost_softmax_f32(const float* logits, const float* boxes, const int64_t* tgt_ids,
                                             const float* tgt_boxes, float* cost, int64_t R, int C, int T,
                                             float w_class, float w_bbox, float w_giou, void* stream) {
  if (!logits || !boxes || !tgt_ids || !tgt_boxes || !cost) return TFB200_E_NULLPTR;
  if (R < 0 || R > 0x7fffffff || C <= 1 || T <= 0) return TFB200_E_SHAPE;
  if (R == 0) return 0;
  return match_cost_rows(logits, boxes, tgt_ids, tgt_boxes, nullptr, cost, 1, 1, int(R), C, T, w_class, w_bbox, w_giou,
                         SoftmaxCls{1.f, 0}, stream);
}

extern "C" int tfb200_match_cost_track_softmax_f32(const float* logits, const float* boxes, const int64_t* tgt_ids,
                                                   const float* tgt_boxes, const int* row_pin, float* cost, int K,
                                                   int B, int Q, int C, int T, float w_class, float w_bbox,
                                                   float w_giou, void* stream) {
  if (!logits || !boxes || !tgt_ids || !tgt_boxes || !row_pin || !cost) return TFB200_E_NULLPTR;
  if (K < 0 || B <= 0 || Q <= 0 || C <= 1 || T <= 0 || T > 48 * 1024) return TFB200_E_SHAPE;
  if (K == 0) return 0;
  return match_cost_rows(logits, boxes, tgt_ids, tgt_boxes, row_pin, cost, K, B, Q, C, T, w_class, w_bbox, w_giou,
                         SoftmaxCls{1.f, 0}, stream);
}

namespace {
template <class Cls>
int set_loss_fwd(const float* logits, const float* boxes, const int64_t* src, const int64_t* tgt, const int64_t* tgt_ids,
                 const float* tgt_boxes, const int* offsets, const float* n_gt, const float* num_boxes,
                 const uint8_t* row_valid, const int* row_pin, float* unit_logits, float* unit_l1, float* unit_giou,
                 float* row_loss, float* row_norm, int* row_flags, float* pair_l1, float* pair_giou, float* out,
                 int K, int B, int Q, int C, int T, Cls cls, void* stream) {
  if (!logits || !boxes || !src || !tgt || !tgt_ids || !tgt_boxes || !offsets || !n_gt || !num_boxes || !unit_logits ||
      !unit_l1 || !unit_giou || !row_loss || !row_flags || !pair_l1 || !pair_giou || !out ||
      (Cls::kLayerNorm && !row_norm))
    return TFB200_E_NULLPTR;
  if (K <= 0 || B <= 0 || Q <= 0 || C <= 0 || T <= 0) return TFB200_E_SHAPE;
  cudaStream_t st = cudaStream_t(stream);
  const int64_t R = int64_t(K) * B * Q;
  set_loss_rows_kernel<Cls><<<unsigned((R + 7) / 8), 256, 0, st>>>(
      logits, boxes, src, tgt, tgt_ids, tgt_boxes, offsets, row_valid, row_pin, unit_logits, unit_l1, unit_giou,
      row_loss, row_norm, row_flags, pair_l1, pair_giou, K, B, Q, C, T, cls);
  set_loss_final_kernel<Cls::kLayerNorm><<<K, 256, 0, st>>>(row_loss, row_norm, row_flags, pair_l1, pair_giou, n_gt,
                                                            num_boxes, out, K, B, Q, T);
  msda_b200_count_launches(2);
  return int(cudaGetLastError());
}

int set_loss_bwd(const float* unit_logits, const float* unit_l1, const float* unit_giou, const float* g_ce,
                 const float* g_l1, const float* g_giou, const float* num_boxes, const float* ce_norm, int ce_stride,
                 float* grad_logits, float* grad_boxes, int K, int B, int Q, int C, void* stream) {
  const int64_t R = int64_t(K) * B * Q;
  const int64_t n = R * (C > 4 ? C : 4);
  set_loss_bwd_kernel<<<unsigned((n + 255) / 256), 256, 0, cudaStream_t(stream)>>>(
      unit_logits, unit_l1, unit_giou, g_ce, g_l1, g_giou, num_boxes, ce_norm, ce_stride, grad_logits, grad_boxes,
      int64_t(B) * Q, C, R);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}
}  // namespace

extern "C" int tfb200_set_loss_fwd_f32(const float* logits, const float* boxes, const int64_t* src, const int64_t* tgt,
                                       const int64_t* tgt_ids, const float* tgt_boxes, const int* offsets,
                                       const float* n_gt, const float* num_boxes, float* unit_logits, float* unit_l1,
                                       float* unit_giou, float* row_loss, int* row_flags, float* pair_l1, float* pair_giou,
                                       float* out5k, int K, int B, int Q, int C, int T, float alpha, float gamma,
                                       void* stream) {
  return set_loss_fwd(logits, boxes, src, tgt, tgt_ids, tgt_boxes, offsets, n_gt, num_boxes, nullptr, nullptr,
                      unit_logits, unit_l1, unit_giou, row_loss, nullptr, row_flags, pair_l1, pair_giou, out5k, K, B, Q,
                      C, T, FocalCls{alpha, gamma}, stream);
}

extern "C" int tfb200_set_loss_fwd_masked_f32(const float* logits, const float* boxes, const int64_t* src,
                                              const int64_t* tgt, const int64_t* tgt_ids, const float* tgt_boxes,
                                              const int* offsets, const float* n_gt, const float* num_boxes,
                                              const uint8_t* row_valid, float* unit_logits, float* unit_l1,
                                              float* unit_giou, float* row_loss, int* row_flags, float* pair_l1,
                                              float* pair_giou, float* out5k, int K, int B, int Q, int C, int T,
                                              float alpha, float gamma, void* stream) {
  if (!row_valid) return TFB200_E_NULLPTR;
  return set_loss_fwd(logits, boxes, src, tgt, tgt_ids, tgt_boxes, offsets, n_gt, num_boxes, row_valid, nullptr,
                      unit_logits, unit_l1, unit_giou, row_loss, nullptr, row_flags, pair_l1, pair_giou, out5k, K, B, Q,
                      C, T, FocalCls{alpha, gamma}, stream);
}

extern "C" int tfb200_set_loss_fwd_softmax_f32(const float* logits, const float* boxes, const int64_t* src,
                                               const int64_t* tgt, const int64_t* tgt_ids, const float* tgt_boxes,
                                               const int* offsets, const float* n_gt, const float* num_boxes,
                                               const uint8_t* row_valid, const int* row_pin, float* unit_logits,
                                               float* unit_l1, float* unit_giou, float* row_loss, float* row_norm,
                                               int* row_flags, float* pair_l1, float* pair_giou, float* out6k, int K,
                                               int B, int Q, int C, int T, float eos_coef, void* stream) {
  if (C <= 1 || !(eos_coef > 0.f)) return TFB200_E_SHAPE;
  return set_loss_fwd(logits, boxes, src, tgt, tgt_ids, tgt_boxes, offsets, n_gt, num_boxes, row_valid, row_pin,
                      unit_logits, unit_l1, unit_giou, row_loss, row_norm, row_flags, pair_l1, pair_giou, out6k, K, B,
                      Q, C, T, SoftmaxCls{eos_coef, row_pin != nullptr ? 1 : 0}, stream);
}

extern "C" int tfb200_set_loss_bwd_f32(const float* unit_logits, const float* unit_l1, const float* unit_giou,
                                       const float* g_ce, const float* g_l1, const float* g_giou, const float* num_boxes,
                                       float* grad_logits, float* grad_boxes, int K, int B, int Q, int C, void* stream) {
  if (!unit_logits || !unit_l1 || !unit_giou || !g_ce || !g_l1 || !g_giou || !num_boxes || !grad_logits || !grad_boxes)
    return TFB200_E_NULLPTR;
  if (K <= 0 || B <= 0 || Q <= 0 || C <= 0) return TFB200_E_SHAPE;
  return set_loss_bwd(unit_logits, unit_l1, unit_giou, g_ce, g_l1, g_giou, num_boxes, num_boxes, 0, grad_logits,
                      grad_boxes, K, B, Q, C, stream);
}

extern "C" int tfb200_set_loss_bwd_softmax_f32(const float* unit_logits, const float* unit_l1, const float* unit_giou,
                                               const float* g_ce, const float* g_l1, const float* g_giou,
                                               const float* num_boxes, const float* ce_norm, float* grad_logits,
                                               float* grad_boxes, int K, int B, int Q, int C, void* stream) {
  if (!unit_logits || !unit_l1 || !unit_giou || !g_ce || !g_l1 || !g_giou || !num_boxes || !ce_norm || !grad_logits ||
      !grad_boxes)
    return TFB200_E_NULLPTR;
  if (K <= 0 || B <= 0 || Q <= 0 || C <= 1) return TFB200_E_SHAPE;
  return set_loss_bwd(unit_logits, unit_l1, unit_giou, g_ce, g_l1, g_giou, num_boxes, ce_norm, 1, grad_logits,
                      grad_boxes, K, B, Q, C, stream);
}
