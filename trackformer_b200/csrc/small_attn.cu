// Dense self-attention over a few hundred queries (the decoder's query self-attention: 300 object queries, up to 800 with
// track queries; 8 heads x 32 channels) -- forward and backward, fp32, attention-weight dropout with the mask-free hash
// RNG of the other fused kernels.
//
// Replaces the core of nn.MultiheadAttention in the decoder layer (reference: models/deformable_transformer.py:342,
// 366-368: q = k = tgt + query_pos, v = tgt, dropout 0.1 on the attention weights).  PyTorch serves that call with its
// "memory-efficient" kernel (an sm80 fp32 kernel sized for far longer sequences); the problem is tiny (11.5 MFLOP per head), so three SIMT kernels with online softmax do:
//   forward        warp = query, lane = key inside a 32-key tile; output lane = channel
//   backward dq    warp = query (recomputes the probabilities from the saved log-sum-exp), also writes D = dO . O
//   backward dk/dv warp = key, lane = query inside a 32-query tile -- no atomics, fixed summation order
// Layout: q / k / v / out are [L, B, H, 32] VIEWS (channel stride 1, head stride 32, arbitrary sequence and batch
// strides), so the packed in-projection output is consumed in place.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "launch_counter.h"

namespace {

constexpr int kD = 32;          // channels per head
constexpr int kWarps = 8;       // queries (keys) per CTA
constexpr int kTile = 32;       // keys (queries) per shared-memory tile
constexpr int kPitch = kD + 1;  // odd pitch: lane = row reads are conflict-free

__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}
__device__ __forceinline__ bool keep_elem(uint64_t seed, uint64_t idx, uint32_t keep_thresh) {
  const uint32_t h = mix32(uint32_t(idx) ^ mix32(uint32_t(idx >> 32) + uint32_t(seed)) ^ uint32_t(seed >> 32) * 0x9e3779b9u);
  return h < keep_thresh;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct Strides {
  int64_t q_l, q_b, k_l, k_b, v_l, v_b, o_l, o_b;   // elements between consecutive sequence positions / batch entries
};

// stage rows [t0, t0 + 32) of a [L, B, H, 32] view into a [32][33] tile (zero beyond L)
__device__ __forceinline__ void stage_tile(float (*tile)[kPitch], const float* base, int64_t ld, int t0, int L) {
  for (int i = threadIdx.x; i < kTile * (kD / 4); i += kWarps * 32) {
    const int r = i >> 3, c = (i & 7) * 4;
    float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
    if (t0 + r < L) x = __ldg(reinterpret_cast<const float4*>(base + int64_t(t0 + r) * ld + c));
    tile[r][c] = x.x; tile[r][c + 1] = x.y; tile[r][c + 2] = x.z; tile[r][c + 3] = x.w;
  }
}

// ---------------------------------------------------------------------------------------------- forward
__global__ void __launch_bounds__(kWarps * 32)
small_attn_fwd_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                      const uint8_t* __restrict__ key_pad, const int64_t* __restrict__ seed_ptr, float* __restrict__ out,
                      float* __restrict__ lse, int B, int H, int L, float scale, float inv_keep, uint32_t keep_thresh,
                      Strides st) {
  __shared__ float sk[kTile][kPitch], sv[kTile][kPitch];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
  const int qi = blockIdx.x * kWarps + w;
  const bool active = qi < L;
  const uint64_t seed = seed_ptr ? uint64_t(__ldg(seed_ptr)) : 0;
  float qr[kD];
  {
    const float* qp = q + int64_t(active ? qi : 0) * st.q_l + int64_t(b) * st.q_b + h * kD;
#pragma unroll
    for (int c = 0; c < kD; c += 4) {
      const float4 x = __ldg(reinterpret_cast<const float4*>(qp + c));
      qr[c] = x.x * scale; qr[c + 1] = x.y * scale; qr[c + 2] = x.z * scale; qr[c + 3] = x.w * scale;
    }
  }
  const float* kb = k + int64_t(b) * st.k_b + h * kD;
  const float* vb = v + int64_t(b) * st.v_b + h * kD;
  float m = -INFINITY, l = 0.f, o = 0.f;                        // running max, running sum, output channel `lane`
  for (int t0 = 0; t0 < L; t0 += kTile) {
    __syncthreads();
    stage_tile(sk, kb, st.k_l, t0, L);
    stage_tile(sv, vb, st.v_l, t0, L);
    __syncthreads();
    const int key = t0 + lane;
    float s = -INFINITY;
    if (key < L && !(key_pad && key_pad[int64_t(b) * L + key])) {
      s = 0.f;
#pragma unroll
      for (int c = 0; c < kD; ++c) s = fmaf(qr[c], sk[lane][c], s);
    }
    const float m_new = fmaxf(m, warp_max(s));
    if (m_new == -INFINITY) continue;                            // every key so far is masked (warp-uniform)
    const float p = (s == -INFINITY) ? 0.f : __expf(s - m_new);
    const float corr = (m == -INFINITY) ? 0.f : __expf(m - m_new);
    l = l * corr + warp_sum(p);
    float pd = p;
    if (seed_ptr) pd = keep_elem(seed, (uint64_t(bh) * L + uint64_t(active ? qi : 0)) * L + key, keep_thresh) ? p * inv_keep : 0.f;
    o *= corr;
#pragma unroll
    for (int j = 0; j < kTile; ++j) o = fmaf(__shfl_sync(0xffffffffu, pd, j), sv[j][lane], o);
    m = m_new;
  }
  if (active) {
    const float inv = l > 0.f ? 1.f / l : 0.f;                    // fully masked row -> zeros (PyTorch would give NaN)
    out[int64_t(qi) * st.o_l + int64_t(b) * st.o_b + h * kD + lane] = o * inv;
    if (lane == 0) lse[int64_t(bh) * L + qi] = l > 0.f ? m + __logf(l) : INFINITY;
  }
}

// ---------------------------------------------------------------------------------------------- backward: dq (+ D)
__global__ void __launch_bounds__(kWarps * 32)
small_attn_bwd_dq_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                         const uint8_t* __restrict__ key_pad, const int64_t* __restrict__ seed_ptr,
                         const float* __restrict__ out, const float* __restrict__ lse, const float* __restrict__ dout,
                         float* __restrict__ dq, float* __restrict__ delta, int B, int H, int L, float scale, float inv_keep,
                         uint32_t keep_thresh, Strides st, int64_t do_l, int64_t do_b, int64_t dq_l, int64_t dq_b) {
  __shared__ float sk[kTile][kPitch], sv[kTile][kPitch];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
  const int qi = blockIdx.x * kWarps + w;
  const bool active = qi < L;
  const int qs = active ? qi : 0;
  const uint64_t seed = seed_ptr ? uint64_t(__ldg(seed_ptr)) : 0;
  float qr[kD], gr[kD];
  {
    const float* qp = q + int64_t(qs) * st.q_l + int64_t(b) * st.q_b + h * kD;
    const float* gp = dout + int64_t(qs) * do_l + int64_t(b) * do_b + h * kD;
#pragma unroll
    for (int c = 0; c < kD; c += 4) {
      const float4 x = __ldg(reinterpret_cast<const float4*>(qp + c));
      const float4 g = __ldg(reinterpret_cast<const float4*>(gp + c));
      qr[c] = x.x * scale; qr[c + 1] = x.y * scale; qr[c + 2] = x.z * scale; qr[c + 3] = x.w * scale;
      gr[c] = g.x; gr[c + 1] = g.y; gr[c + 2] = g.z; gr[c + 3] = g.w;
    }
  }
  const float dl = warp_sum(gr[lane] * __ldg(out + int64_t(qs) * st.o_l + int64_t(b) * st.o_b + h * kD + lane));   // D = dO . O
  const float ls = lse[int64_t(bh) * L + qs];
  const float* kb = k + int64_t(b) * st.k_b + h * kD;
  const float* vb = v + int64_t(b) * st.v_b + h * kD;
  float acc = 0.f;                                                // dq channel `lane`
  for (int t0 = 0; t0 < L; t0 += kTile) {
    __syncthreads();
    stage_tile(sk, kb, st.k_l, t0, L);
    stage_tile(sv, vb, st.v_l, t0, L);
    __syncthreads();
    const int key = t0 + lane;
    float ds = 0.f;
    if (key < L && ls != INFINITY && !(key_pad && key_pad[int64_t(b) * L + key])) {
      float s = 0.f, t = 0.f;
#pragma unroll
      for (int c = 0; c < kD; ++c) {
        s = fmaf(qr[c], sk[lane][c], s);
        t = fmaf(gr[c], sv[lane][c], t);
      }
      const float p = __expf(s - ls);
      float u = t;
      if (seed_ptr) u = keep_elem(seed, (uint64_t(bh) * L + uint64_t(qs)) * L + key, keep_thresh) ? t * inv_keep : 0.f;
      ds = p * (u - dl);
    }
#pragma unroll
    for (int j = 0; j < kTile; ++j) acc = fmaf(__shfl_sync(0xffffffffu, ds, j), sk[j][lane], acc);
  }
  if (active) {
    dq[int64_t(qi) * dq_l + int64_t(b) * dq_b + h * kD + lane] = acc * scale;
    if (lane == 0) delta[int64_t(bh) * L + qi] = dl;
  }
}

// ---------------------------------------------------------------------------------------------- backward: dk, dv
__global__ void __launch_bounds__(kWarps * 32)
small_attn_bwd_dkv_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                          const uint8_t* __restrict__ key_pad, const int64_t* __restrict__ seed_ptr,
                          const float* __restrict__ lse, const float* __restrict__ delta, const float* __restrict__ dout,
                          float* __restrict__ dk, float* __restrict__ dv, int B, int H, int L, float scale, float inv_keep,
                          uint32_t keep_thresh, Strides st, int64_t do_l, int64_t do_b, int64_t dk_l, int64_t dk_b,
                          int64_t dv_l, int64_t dv_b) {
  __shared__ float sq[kTile][kPitch], sg[kTile][kPitch];
  __shared__ float s_lse[kTile], s_dl[kTile];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
  const int ki = blockIdx.x * kWarps + w;
  const bool active = ki < L;
  const int ks = active ? ki : 0;
  const bool masked = !active || (key_pad && key_pad[int64_t(b) * L + ks]);
  const uint64_t seed = seed_ptr ? uint64_t(__ldg(seed_ptr)) : 0;
  float kr[kD], vr[kD];
  {
    const float* kp = k + int64_t(ks) * st.k_l + int64_t(b) * st.k_b + h * kD;
    const float* vp = v + int64_t(ks) * st.v_l + int64_t(b) * st.v_b + h * kD;
#pragma unroll
    for (int c = 0; c < kD; c += 4) {
      const float4 x = __ldg(reinterpret_cast<const float4*>(kp + c));
      const float4 y = __ldg(reinterpret_cast<const float4*>(vp + c));
      kr[c] = x.x * scale; kr[c + 1] = x.y * scale; kr[c + 2] = x.z * scale; kr[c + 3] = x.w * scale;
      vr[c] = y.x; vr[c + 1] = y.y; vr[c + 2] = y.z; vr[c + 3] = y.w;
    }
  }
  const float* qb = q + int64_t(b) * st.q_b + h * kD;
  const float* gb = dout + int64_t(b) * do_b + h * kD;
  float ak = 0.f, av = 0.f;                                       // dk / dv channel `lane`
  for (int t0 = 0; t0 < L; t0 += kTile) {
    __syncthreads();
    stage_tile(sq, qb, st.q_l, t0, L);
    stage_tile(sg, gb, do_l, t0, L);
    if (threadIdx.x < kTile) {
      const int qi = t0 + threadIdx.x;
      s_lse[threadIdx.x] = qi < L ? lse[int64_t(bh) * L + qi] : INFINITY;
      s_dl[threadIdx.x] = qi < L ? delta[int64_t(bh) * L + qi] : 0.f;
    }
    __syncthreads();
    const int qi = t0 + lane;
    float ds = 0.f, a = 0.f;
    const float ls = s_lse[lane];
    if (!masked && qi < L && ls != INFINITY) {
      float s = 0.f, t = 0.f;
#pragma unroll
      for (int c = 0; c < kD; ++c) {
        s = fmaf(kr[c], sq[lane][c], s);
        t = fmaf(vr[c], sg[lane][c], t);
      }
      const float p = __expf(s - ls);
      float u = t;
      a = p;
      if (seed_ptr) {
        const bool keep = keep_elem(seed, (uint64_t(bh) * L + uint64_t(qi)) * L + ks, keep_thresh);
        u = keep ? t * inv_keep : 0.f;
        a = keep ? p * inv_keep : 0.f;
      }
      ds = p * (u - s_dl[lane]);
    }
#pragma unroll
    for (int j = 0; j < kTile; ++j) {
      ak = fmaf(__shfl_sync(0xffffffffu, ds, j), sq[j][lane], ak);
      av = fmaf(__shfl_sync(0xffffffffu, a, j), sg[j][lane], av);
    }
  }
  if (active) {
    dk[int64_t(ki) * dk_l + int64_t(b) * dk_b + h * kD + lane] = ak * scale;
    dv[int64_t(ki) * dv_l + int64_t(b) * dv_b + h * kD + lane] = av;
  }
}

uint32_t keep_threshold(float keep_prob) {
  const double t = double(keep_prob) * 4294967296.0;
  return t >= 4294967295.0 ? 0xFFFFFFFFu : uint32_t(t);
}

}  // namespace

extern "C" int tfb200_small_attn_fwd_f32(const float* q, const float* k, const float* v, const uint8_t* key_pad,
                                         const int64_t* seed_dev, float* out, float* lse, int B, int H, int L,
                                         const int64_t* strides8, float scale, float keep_prob, void* stream) {
  if (!q || !k || !v || !out || !lse || !strides8) return TFB200_E_NULLPTR;
  if (B < 1 || H < 1 || L < 1 || keep_prob <= 0.f || keep_prob > 1.f) return TFB200_E_SHAPE;
  Strides st{strides8[0], strides8[1], strides8[2], strides8[3], strides8[4], strides8[5], strides8[6], strides8[7]};
  const dim3 grid((L + kWarps - 1) / kWarps, B * H);
  small_attn_fwd_kernel<<<grid, kWarps * 32, 0, cudaStream_t(stream)>>>(q, k, v, key_pad, seed_dev, out, lse, B, H, L, scale,
                                                                       1.f / keep_prob, keep_threshold(keep_prob), st);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_small_attn_bwd_f32(const float* q, const float* k, const float* v, const uint8_t* key_pad,
                                         const int64_t* seed_dev, const float* out, const float* lse, const float* dout,
                                         float* dq, float* dk, float* dv, float* delta_ws, int B, int H, int L,
                                         const int64_t* strides16, float scale, float keep_prob, void* stream) {
  if (!q || !k || !v || !out || !lse || !dout || !dq || !dk || !dv || !delta_ws || !strides16) return TFB200_E_NULLPTR;
  if (B < 1 || H < 1 || L < 1 || keep_prob <= 0.f || keep_prob > 1.f) return TFB200_E_SHAPE;
  const int64_t* s = strides16;
  Strides st{s[0], s[1], s[2], s[3], s[4], s[5], s[6], s[7]};
  const dim3 grid((L + kWarps - 1) / kWarps, B * H);
  cudaStream_t cs = cudaStream_t(stream);
  const float inv_keep = 1.f / keep_prob;
  const uint32_t th = keep_threshold(keep_prob);
  small_attn_bwd_dq_kernel<<<grid, kWarps * 32, 0, cs>>>(q, k, v, key_pad, seed_dev, out, lse, dout, dq, delta_ws, B, H, L, scale,
                                                        inv_keep, th, st, s[8], s[9], s[10], s[11]);
  small_attn_bwd_dkv_kernel<<<grid, kWarps * 32, 0, cs>>>(q, k, v, key_pad, seed_dev, lse, delta_ws, dout, dk, dv, B, H, L, scale,
                                                         inv_keep, th, st, s[8], s[9], s[12], s[13], s[14], s[15]);
  msda_b200_count_launches(2);
  return int(cudaGetLastError());
}
