// Dense multi-head attention over long key sequences (vanilla DETR: encoder self-attention over every stride-32 token,
// ~1050 at 800x1333 and ~4200 with DC5; decoder cross-attention from 100 + track queries onto those tokens), 32 channels
// per head -- forward and backward, fp32 in and out, attention-weight dropout with the mask-free hash RNG of
// small_attn.cu / fused_norm.cu.
//
// Replaces the core of the three nn.MultiheadAttention calls of the reference's vanilla transformer
// (models/transformer.py: encoder self-attention, decoder self- and cross-attention).  Flash-style:
//   forward        CTA = 64 queries of one (image, head), warp = 16 queries; 64-key tiles of K / V double-buffered in
//                  shared memory with cp.async; online softmax in fp32; the log-sum-exp is saved for the backward
//   backward D     D = rowsum(dO o O), one warp per row
//   backward dq    CTA = 64 queries, loops over key tiles (recomputes P from the saved log-sum-exp)
//   backward dk/dv CTA = 64 keys, loops over query tiles -- no atomics, fixed summation order: bitwise reproducible
// Both products of every pass run on tensor cores (mma.sync m16n8k8 TF32, fp32 accumulation) as split-TF32: each fp32
// operand x = hi + lo with hi = tf32(x), lo = tf32(x - hi), and a*b = ah*bh + ah*bl + al*bh, which carries ~21 mantissa
// bits -- fp32-level agreement, where plain TF32 (10 bits) would not meet it.
//
// Layout: q / out / dout / dq are [Lq, B, H, 32] views, k / v / dk / dv [Lk, B, H, 32] views (channel stride 1, head
// stride 32, arbitrary sequence and batch strides that are multiples of 4, 16-byte aligned base), so the packed
// in-projection output is consumed in place.  key_pad [B][Lk] (nonzero = ignore that key) may be any pattern.  A query
// whose keys are all masked gets a zero output and lse = +inf, as in small_attn.cu.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "dropout_hash.cuh"
#include "launch_counter.h"

namespace {

using tfb200::keep_elem;        // keyed by the logical element index ((b * H + h) * Lq + q) * Lk + k
using tfb200::keep_threshold;

constexpr int kD = 32;              // channels per head
constexpr int kWarps = 4;           // 16 rows (queries or keys) per warp
constexpr int kRows = 16 * kWarps;  // rows per CTA
constexpr int kTile = 64;           // keys (queries) per staged tile
constexpr int kPitch = kD + 4;      // 144-byte rows: 16-byte aligned for cp.async, conflict-free fragment reads

__device__ __forceinline__ uint32_t to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return r;
}
struct Split {
  uint32_t hi, lo;
};
__device__ __forceinline__ Split split(float x) {
  const uint32_t h = to_tf32(x);
  return {h, to_tf32(x - __uint_as_float(h))};
}

__device__ __forceinline__ void mma_tf32(float (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint32_t b0,
                                         uint32_t b1) {
  asm volatile("mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
               : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
// d += a b for one 16x8 A fragment (a[i] in the m16n8k8 register order) and one 8x8 B fragment, split-TF32
__device__ __forceinline__ void mma3(float (&d)[4], const Split (&a)[4], Split b0, Split b1) {
  mma_tf32(d, a[0].lo, a[1].lo, a[2].lo, a[3].lo, b0.hi, b1.hi);   // small terms first
  mma_tf32(d, a[0].hi, a[1].hi, a[2].hi, a[3].hi, b0.lo, b1.lo);
  mma_tf32(d, a[0].hi, a[1].hi, a[2].hi, a[3].hi, b0.hi, b1.hi);
}

__device__ __forceinline__ void cp_async16(float* smem, const float* gmem, bool valid) {
  const uint32_t s = uint32_t(__cvta_generic_to_shared(smem));
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(valid ? 16 : 0));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
__device__ __forceinline__ void cp_async_wait_1() { asm volatile("cp.async.wait_group 1;\n" ::); }

// stage rows [t0, t0 + 64) of a [L, B, H, 32] view (base already at (b, h)) into a [64][kPitch] tile, zeros beyond L
__device__ __forceinline__ void stage_rows(float (*tile)[kPitch], const float* base, int64_t ld, int t0, int L) {
#pragma unroll
  for (int i = threadIdx.x; i < kTile * (kD / 4); i += kWarps * 32) {
    const int r = i >> 3, c = (i & 7) * 4;
    const bool ok = t0 + r < L;
    cp_async16(&tile[r][c], base + int64_t(ok ? t0 + r : 0) * ld + c, ok);
  }
}

// A fragments (split) of 16 rows x 32 channels of a [L, B, H, 32] view, times `mul`; rows >= L read as zero.
// a[ks][i]: ks = channel block of 8, i in the m16n8k8 A order {(g, t), (g+8, t), (g, t+4), (g+8, t+4)}.
__device__ __forceinline__ void load_a_rows(Split (&a)[4][4], const float* base, int64_t ld, int r0, int L, float mul) {
  const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int r = r0 + g + 8 * hr;
    const float* p = base + int64_t(r < L ? r : 0) * ld;
#pragma unroll
    for (int ks = 0; ks < 4; ++ks) {
      const float x0 = r < L ? __ldg(p + 8 * ks + t) * mul : 0.f;
      const float x1 = r < L ? __ldg(p + 8 * ks + t + 4) * mul : 0.f;
      a[ks][hr] = split(x0);
      a[ks][hr + 2] = split(x1);
    }
  }
}

struct Strides {
  int64_t q_l, q_b, k_l, k_b, v_l, v_b, o_l, o_b;   // elements between consecutive sequence positions / batch entries
};

// ---------------------------------------------------------------------------------------------- forward
__global__ void __launch_bounds__(kWarps * 32)
dense_attn_fwd_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                      const uint8_t* __restrict__ key_pad, const int64_t* __restrict__ seed_ptr, float* __restrict__ out,
                      float* __restrict__ lse, int H, int Lq, int Lk, float scale, float inv_keep, uint32_t keep_thresh,
                      Strides st) {
  __shared__ __align__(16) float sk[2][kTile][kPitch];
  __shared__ __align__(16) float sv[2][kTile][kPitch];
  __shared__ uint8_t sm[2][kTile];                                 // 1 = key masked (padding or beyond Lk)
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
  const int r0 = blockIdx.x * kRows + w * 16;
  const uint64_t seed = seed_ptr ? uint64_t(__ldg(seed_ptr)) : 0;
  const float* kb = k + int64_t(b) * st.k_b + h * kD;
  const float* vb = v + int64_t(b) * st.v_b + h * kD;
  const uint8_t* pad = key_pad ? key_pad + int64_t(b) * Lk : nullptr;
  auto stage = [&](int buf, int t0) {
    stage_rows(sk[buf], kb, st.k_l, t0, Lk);
    stage_rows(sv[buf], vb, st.v_l, t0, Lk);
    if (threadIdx.x < kTile) {
      const int key = t0 + threadIdx.x;
      sm[buf][threadIdx.x] = key >= Lk || (pad && pad[key]);
    }
    cp_async_commit();
  };
  stage(0, 0);

  Split qa[4][4];
  load_a_rows(qa, q + int64_t(b) * st.q_b + h * kD, st.q_l, r0, Lq, scale);
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f};         // rows g, g + 8: running max, partial running sum
  float o[4][4] = {};                                              // output channels 8j + {2t, 2t+1}, rows {g, g+8}
  const uint64_t row_idx[2] = {uint64_t(bh) * Lq + uint64_t(r0 + g), uint64_t(bh) * Lq + uint64_t(r0 + g + 8)};

  const int n_tiles = (Lk + kTile - 1) / kTile;
  for (int it = 0; it < n_tiles; ++it) {
    const int buf = it & 1, t0 = it * kTile;
    if (it + 1 < n_tiles) stage(buf ^ 1, t0 + kTile);
    else cp_async_commit();                                        // empty group keeps the wait count uniform
    cp_async_wait_1();
    __syncthreads();

    float s[8][4];
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
      s[nt][0] = s[nt][1] = s[nt][2] = s[nt][3] = 0.f;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks)
        mma3(s[nt], qa[ks], split(sk[buf][8 * nt + g][8 * ks + t]), split(sk[buf][8 * nt + g][8 * ks + t + 4]));
    }
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (sm[buf][8 * nt + 2 * t + (e & 1)]) s[nt][e] = -INFINITY;
        mx[e >> 1] = fmaxf(mx[e >> 1], s[nt][e]);
      }
    }
    float corr[2];
#pragma unroll
    for (int hr = 0; hr < 2; ++hr) {
      mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 1));
      mx[hr] = fmaxf(mx[hr], __shfl_xor_sync(0xffffffffu, mx[hr], 2));
      const float m_new = fmaxf(m[hr], mx[hr]);
      corr[hr] = (m[hr] == -INFINITY) ? 0.f : __expf(m[hr] - m_new);
      m[hr] = m_new;
      l[hr] *= corr[hr];
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      o[j][0] *= corr[0]; o[j][1] *= corr[0]; o[j][2] *= corr[1]; o[j][3] *= corr[1];
    }
#pragma unroll
    for (int nt = 0; nt < 8; ++nt) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hr = e >> 1;
        const float p = (s[nt][e] == -INFINITY) ? 0.f : __expf(s[nt][e] - m[hr]);
        l[hr] += p;
        float pd = p;
        if (seed_ptr)
          pd = (p != 0.f && keep_elem(seed, row_idx[hr] * uint64_t(Lk) + uint64_t(t0 + 8 * nt + 2 * t + (e & 1)), keep_thresh))
                   ? p * inv_keep : 0.f;
        s[nt][e] = pd;
      }
      // P V over the 8 keys of this n-tile.  The A fragment takes key 2t in k-slot t and key 2t+1 in slot t+4, so the
      // accumulator layout of P is used as is; the B fragment reads V rows in the same order.
      const Split pa[4] = {split(s[nt][0]), split(s[nt][2]), split(s[nt][1]), split(s[nt][3])};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        mma3(o[j], pa, split(sv[buf][8 * nt + 2 * t][8 * j + g]), split(sv[buf][8 * nt + 2 * t + 1][8 * j + g]));
    }
    __syncthreads();                                               // buffer `buf` is restaged by the next iteration
  }

#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    l[hr] += __shfl_xor_sync(0xffffffffu, l[hr], 1);
    l[hr] += __shfl_xor_sync(0xffffffffu, l[hr], 2);
    const int r = r0 + g + 8 * hr;
    if (r >= Lq) continue;
    const float inv = l[hr] > 0.f ? 1.f / l[hr] : 0.f;             // fully masked row -> zeros
    float* op = out + int64_t(r) * st.o_l + int64_t(b) * st.o_b + h * kD;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<float2*>(op + 8 * j + 2 * t) = make_float2(o[j][2 * hr] * inv, o[j][2 * hr + 1] * inv);
    if (t == 0) lse[int64_t(bh) * Lq + r] = l[hr] > 0.f ? m[hr] + __logf(l[hr]) : INFINITY;
  }
}

// ---------------------------------------------------------------------------------------------- backward: D
__global__ void __launch_bounds__(256)
dense_attn_bwd_delta_kernel(const float* __restrict__ out, const float* __restrict__ dout, float* __restrict__ delta, int B,
                            int H, int Lq, int64_t o_l, int64_t o_b, int64_t do_l, int64_t do_b) {
  const int lane = threadIdx.x & 31;
  const int64_t row = int64_t(blockIdx.x) * 8 + (threadIdx.x >> 5);          // (b, h, q) in [B][H][Lq] order
  if (row >= int64_t(B) * H * Lq) return;
  const int qi = int(row % Lq), bh = int(row / Lq), b = bh / H, h = bh - b * H;
  float x = __ldg(out + int64_t(qi) * o_l + int64_t(b) * o_b + h * kD + lane) *
            __ldg(dout + int64_t(qi) * do_l + int64_t(b) * do_b + h * kD + lane);
#pragma unroll
  for (int s = 16; s > 0; s >>= 1) x += __shfl_xor_sync(0xffffffffu, x, s);
  if (lane == 0) delta[row] = x;
}

// ---------------------------------------------------------------------------------------------- backward: dq
__global__ void __launch_bounds__(kWarps * 32)
dense_attn_bwd_dq_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                         const uint8_t* __restrict__ key_pad, const int64_t* __restrict__ seed_ptr,
                         const float* __restrict__ lse, const float* __restrict__ delta, const float* __restrict__ dout,
                         float* __restrict__ dq, int H, int Lq, int Lk, float scale, float inv_keep, uint32_t keep_thresh,
                         Strides st, int64_t do_l, int64_t do_b, int64_t dq_l, int64_t dq_b) {
  __shared__ __align__(16) float sk[2][kTile][kPitch];
  __shared__ __align__(16) float sv[2][kTile][kPitch];
  __shared__ uint8_t sm[2][kTile];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
  const int r0 = blockIdx.x * kRows + w * 16;
  const uint64_t seed = seed_ptr ? uint64_t(__ldg(seed_ptr)) : 0;
  const float* kb = k + int64_t(b) * st.k_b + h * kD;
  const float* vb = v + int64_t(b) * st.v_b + h * kD;
  const uint8_t* pad = key_pad ? key_pad + int64_t(b) * Lk : nullptr;
  auto stage = [&](int buf, int t0) {
    stage_rows(sk[buf], kb, st.k_l, t0, Lk);
    stage_rows(sv[buf], vb, st.v_l, t0, Lk);
    if (threadIdx.x < kTile) {
      const int key = t0 + threadIdx.x;
      sm[buf][threadIdx.x] = key >= Lk || (pad && pad[key]);
    }
    cp_async_commit();
  };
  stage(0, 0);

  Split qa[4][4], ga[4][4];
  load_a_rows(qa, q + int64_t(b) * st.q_b + h * kD, st.q_l, r0, Lq, scale);
  load_a_rows(ga, dout + int64_t(b) * do_b + h * kD, do_l, r0, Lq, 1.f);
  float ls[2], dl[2];
  uint64_t row_idx[2];
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int r = r0 + g + 8 * hr;
    ls[hr] = r < Lq ? __ldg(lse + int64_t(bh) * Lq + r) : INFINITY;
    dl[hr] = r < Lq ? __ldg(delta + int64_t(bh) * Lq + r) : 0.f;
    row_idx[hr] = uint64_t(bh) * Lq + uint64_t(r);
  }
  float acc[4][4] = {};                                            // dq channels 8j + {2t, 2t+1}, rows {g, g+8}

  const int n_tiles = (Lk + kTile - 1) / kTile;
  for (int it = 0; it < n_tiles; ++it) {
    const int buf = it & 1, t0 = it * kTile;
    if (it + 1 < n_tiles) stage(buf ^ 1, t0 + kTile);
    else cp_async_commit();
    cp_async_wait_1();
    __syncthreads();
#pragma unroll 2
    for (int nt = 0; nt < 8; ++nt) {
      float s[4] = {}, dp[4] = {};
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        mma3(s, qa[ks], split(sk[buf][8 * nt + g][8 * ks + t]), split(sk[buf][8 * nt + g][8 * ks + t + 4]));
        mma3(dp, ga[ks], split(sv[buf][8 * nt + g][8 * ks + t]), split(sv[buf][8 * nt + g][8 * ks + t + 4]));
      }
      float ds[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hr = e >> 1, key = t0 + 8 * nt + 2 * t + (e & 1);
        ds[e] = 0.f;
        if (!sm[buf][8 * nt + 2 * t + (e & 1)] && ls[hr] != INFINITY) {
          const float p = __expf(s[e] - ls[hr]);
          float u = dp[e];
          if (seed_ptr) u = keep_elem(seed, row_idx[hr] * uint64_t(Lk) + uint64_t(key), keep_thresh) ? u * inv_keep : 0.f;
          ds[e] = p * (u - dl[hr]);
        }
      }
      const Split da[4] = {split(ds[0]), split(ds[2]), split(ds[1]), split(ds[3])};
#pragma unroll
      for (int j = 0; j < 4; ++j)
        mma3(acc[j], da, split(sk[buf][8 * nt + 2 * t][8 * j + g]), split(sk[buf][8 * nt + 2 * t + 1][8 * j + g]));
    }
    __syncthreads();
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int r = r0 + g + 8 * hr;
    if (r >= Lq) continue;
    float* p = dq + int64_t(r) * dq_l + int64_t(b) * dq_b + h * kD;
#pragma unroll
    for (int j = 0; j < 4; ++j)
      *reinterpret_cast<float2*>(p + 8 * j + 2 * t) = make_float2(acc[j][2 * hr] * scale, acc[j][2 * hr + 1] * scale);
  }
}

// ---------------------------------------------------------------------------------------------- backward: dk, dv
__global__ void __launch_bounds__(kWarps * 32)
dense_attn_bwd_dkv_kernel(const float* __restrict__ q, const float* __restrict__ k, const float* __restrict__ v,
                          const uint8_t* __restrict__ key_pad, const int64_t* __restrict__ seed_ptr,
                          const float* __restrict__ lse, const float* __restrict__ delta, const float* __restrict__ dout,
                          float* __restrict__ dk, float* __restrict__ dv, int H, int Lq, int Lk, float scale,
                          float inv_keep, uint32_t keep_thresh, Strides st, int64_t do_l, int64_t do_b, int64_t dk_l,
                          int64_t dk_b, int64_t dv_l, int64_t dv_b) {
  __shared__ __align__(16) float sq[2][kTile][kPitch];
  __shared__ __align__(16) float sg[2][kTile][kPitch];
  __shared__ float s_lse[2][kTile], s_dl[2][kTile];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
  const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
  const int r0 = blockIdx.x * kRows + w * 16;                      // first key of this warp
  const uint64_t seed = seed_ptr ? uint64_t(__ldg(seed_ptr)) : 0;
  const float* qb = q + int64_t(b) * st.q_b + h * kD;
  const float* gb = dout + int64_t(b) * do_b + h * kD;
  auto stage = [&](int buf, int t0) {
    stage_rows(sq[buf], qb, st.q_l, t0, Lq);
    stage_rows(sg[buf], gb, do_l, t0, Lq);
    if (threadIdx.x < kTile) {
      const int qi = t0 + threadIdx.x;
      s_lse[buf][threadIdx.x] = qi < Lq ? __ldg(lse + int64_t(bh) * Lq + qi) : INFINITY;
      s_dl[buf][threadIdx.x] = qi < Lq ? __ldg(delta + int64_t(bh) * Lq + qi) : 0.f;
    }
    cp_async_commit();
  };
  stage(0, 0);

  Split ka[4][4], va[4][4];
  load_a_rows(ka, k + int64_t(b) * st.k_b + h * kD, st.k_l, r0, Lk, scale);
  load_a_rows(va, v + int64_t(b) * st.v_b + h * kD, st.v_l, r0, Lk, 1.f);
  bool live[2];                                                    // key exists and is not padding
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int key = r0 + g + 8 * hr;
    live[hr] = key < Lk && !(key_pad && key_pad[int64_t(b) * Lk + key]);
  }
  float ak[4][4] = {}, av[4][4] = {};                              // dk / dv channels 8j + {2t, 2t+1}, keys {g, g+8}

  const int n_tiles = (Lq + kTile - 1) / kTile;
  for (int it = 0; it < n_tiles; ++it) {
    const int buf = it & 1, t0 = it * kTile;
    if (it + 1 < n_tiles) stage(buf ^ 1, t0 + kTile);
    else cp_async_commit();
    cp_async_wait_1();
    __syncthreads();
#pragma unroll 2
    for (int nt = 0; nt < 8; ++nt) {
      float s[4] = {}, dp[4] = {};                                 // transposed: rows = keys, columns = queries
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        mma3(s, ka[ks], split(sq[buf][8 * nt + g][8 * ks + t]), split(sq[buf][8 * nt + g][8 * ks + t + 4]));
        mma3(dp, va[ks], split(sg[buf][8 * nt + g][8 * ks + t]), split(sg[buf][8 * nt + g][8 * ks + t + 4]));
      }
      float ds[4], pa[4];
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int hr = e >> 1, c = 8 * nt + 2 * t + (e & 1);
        const float ls = s_lse[buf][c];
        ds[e] = pa[e] = 0.f;
        if (live[hr] && ls != INFINITY) {
          const float p = __expf(s[e] - ls);
          float u = dp[e], a = p;
          if (seed_ptr) {
            const bool keep = keep_elem(seed, (uint64_t(bh) * Lq + uint64_t(t0 + c)) * uint64_t(Lk) + uint64_t(r0 + g + 8 * hr),
                                        keep_thresh);
            u = keep ? u * inv_keep : 0.f;
            a = keep ? p * inv_keep : 0.f;
          }
          ds[e] = p * (u - s_dl[buf][c]);
          pa[e] = a;
        }
      }
      const Split da[4] = {split(ds[0]), split(ds[2]), split(ds[1]), split(ds[3])};
      const Split pf[4] = {split(pa[0]), split(pa[2]), split(pa[1]), split(pa[3])};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        mma3(ak[j], da, split(sq[buf][8 * nt + 2 * t][8 * j + g]), split(sq[buf][8 * nt + 2 * t + 1][8 * j + g]));
        mma3(av[j], pf, split(sg[buf][8 * nt + 2 * t][8 * j + g]), split(sg[buf][8 * nt + 2 * t + 1][8 * j + g]));
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int hr = 0; hr < 2; ++hr) {
    const int key = r0 + g + 8 * hr;
    if (key >= Lk) continue;
    float* pk = dk + int64_t(key) * dk_l + int64_t(b) * dk_b + h * kD;
    float* pv = dv + int64_t(key) * dv_l + int64_t(b) * dv_b + h * kD;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      *reinterpret_cast<float2*>(pk + 8 * j + 2 * t) = make_float2(ak[j][2 * hr] * scale, ak[j][2 * hr + 1] * scale);
      *reinterpret_cast<float2*>(pv + 8 * j + 2 * t) = make_float2(av[j][2 * hr], av[j][2 * hr + 1]);
    }
  }
}

// ---------------------------------------------------------------------------------------------- head-averaged weights
// W[b, r, c] = (1/H) sum_h exp(scale q_h[r] . k_h[c] - lse[b, h, r]): the probabilities of the forward, averaged over
// heads (nn.MultiheadAttention's need_weights=True, average_attn_weights=True), from the forward's own log-sum-exp.
// CTA = 64 rows x 64 keys of one image, 16 x 16 threads with 4 x 4 outputs each (rows ty + 16i, keys tx + 16j); the
// head loop stages that head's q / k tiles in shared memory and accumulates in registers, so every output element is
// written once, in a fixed order: no atomics, bitwise reproducible.  Scores are fp32 FMA dot products (32 channels).
constexpr int kWTile = 64;
constexpr int kWPitch = kD + 1;        // odd pitch: the 16 keys / 2 rows a warp reads per channel hit distinct banks

__global__ void __launch_bounds__(256)
dense_attn_weights_kernel(const float* __restrict__ q, const float* __restrict__ k, const uint8_t* __restrict__ key_pad,
                          const float* __restrict__ lse, float* __restrict__ weights, int H, int Lq, int Lk, float scale,
                          int64_t q_l, int64_t q_b, int64_t k_l, int64_t k_b) {
  __shared__ float sq[kWTile][kWPitch];
  __shared__ float sk[kWTile][kWPitch];
  __shared__ float s_lse[kWTile];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int c0 = blockIdx.x * kWTile, r0 = blockIdx.y * kWTile, b = blockIdx.z;
  float acc[4][4] = {};
  for (int h = 0; h < H; ++h) {
    for (int i = threadIdx.x; i < kWTile * (kD / 4); i += 256) {
      const int r = i >> 3, c = (i & 7) * 4;
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f), y = x;
      if (r0 + r < Lq) x = __ldg(reinterpret_cast<const float4*>(q + int64_t(r0 + r) * q_l + int64_t(b) * q_b + h * kD + c));
      if (c0 + r < Lk) y = __ldg(reinterpret_cast<const float4*>(k + int64_t(c0 + r) * k_l + int64_t(b) * k_b + h * kD + c));
      sq[r][c] = x.x * scale; sq[r][c + 1] = x.y * scale; sq[r][c + 2] = x.z * scale; sq[r][c + 3] = x.w * scale;
      sk[r][c] = y.x; sk[r][c + 1] = y.y; sk[r][c + 2] = y.z; sk[r][c + 3] = y.w;
    }
    if (threadIdx.x < kWTile) {
      const int r = r0 + threadIdx.x;
      s_lse[threadIdx.x] = r < Lq ? __ldg(lse + (int64_t(b) * H + h) * Lq + r) : INFINITY;
    }
    __syncthreads();
    float s[4][4] = {};
#pragma unroll 8
    for (int c = 0; c < kD; ++c) {
      float a[4], kk[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = sq[ty + 16 * i][c];
#pragma unroll
      for (int j = 0; j < 4; ++j) kk[j] = sk[tx + 16 * j][c];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) s[i][j] = fmaf(a[i], kk[j], s[i][j]);
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const float ls = s_lse[ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] += ls == INFINITY ? 0.f : expf(s[i][j] - ls);   // fully masked row -> 0
    }
    __syncthreads();                   // the tiles are restaged for the next head
  }
  const float inv_h = 1.f / float(H);
  bool live[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int c = c0 + tx + 16 * j;
    live[j] = c < Lk && !(key_pad && key_pad[int64_t(b) * Lk + c]);
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int r = r0 + ty + 16 * i;
    if (r >= Lq) continue;
    float* w = weights + (int64_t(b) * Lq + r) * Lk;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int c = c0 + tx + 16 * j;
      if (c < Lk) w[c] = live[j] ? acc[i][j] * inv_h : 0.f;
    }
  }
}

bool aligned_view(const void* p, const int64_t* strides, int n) {
  if (reinterpret_cast<uintptr_t>(p) & 15u) return false;
  for (int i = 0; i < n; ++i)
    if (strides[i] % 4) return false;
  return true;
}

}  // namespace

extern "C" int tfb200_dense_attn_fwd_f32(const float* q, const float* k, const float* v, const uint8_t* key_pad,
                                         const int64_t* seed_dev, float* out, float* lse, int B, int H, int Lq, int Lk,
                                         const int64_t* strides8, float scale, float keep_prob, void* stream) {
  if (!q || !k || !v || !out || !lse || !strides8) return TFB200_E_NULLPTR;
  if (B < 1 || H < 1 || Lq < 1 || Lk < 1 || keep_prob <= 0.f || keep_prob > 1.f || int64_t(B) * H > 65535)
    return TFB200_E_SHAPE;
  if (!aligned_view(q, strides8, 2) || !aligned_view(k, strides8 + 2, 2) || !aligned_view(v, strides8 + 4, 2) ||
      !aligned_view(out, strides8 + 6, 2))
    return TFB200_E_SHAPE;
  Strides st{strides8[0], strides8[1], strides8[2], strides8[3], strides8[4], strides8[5], strides8[6], strides8[7]};
  const dim3 grid((Lq + kRows - 1) / kRows, B * H);
  dense_attn_fwd_kernel<<<grid, kWarps * 32, 0, cudaStream_t(stream)>>>(q, k, v, key_pad, seed_dev, out, lse, H, Lq, Lk,
                                                                       scale, 1.f / keep_prob, keep_threshold(keep_prob), st);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_dense_attn_weights_f32(const float* q, const float* k, const uint8_t* key_pad, const float* lse,
                                             float* weights, int B, int H, int Lq, int Lk, const int64_t* strides4,
                                             float scale, void* stream) {
  if (!q || !k || !lse || !weights || !strides4) return TFB200_E_NULLPTR;
  if (B < 1 || H < 1 || Lq < 1 || Lk < 1 || B > 65535 || (Lq + kWTile - 1) / kWTile > 65535) return TFB200_E_SHAPE;
  if (!aligned_view(q, strides4, 2) || !aligned_view(k, strides4 + 2, 2)) return TFB200_E_SHAPE;
  const dim3 grid((Lk + kWTile - 1) / kWTile, (Lq + kWTile - 1) / kWTile, B);
  dense_attn_weights_kernel<<<grid, 256, 0, cudaStream_t(stream)>>>(q, k, key_pad, lse, weights, H, Lq, Lk, scale,
                                                                     strides4[0], strides4[1], strides4[2], strides4[3]);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_dense_attn_bwd_f32(const float* q, const float* k, const float* v, const uint8_t* key_pad,
                                         const int64_t* seed_dev, const float* out, const float* lse, const float* dout,
                                         float* dq, float* dk, float* dv, float* delta_ws, int B, int H, int Lq, int Lk,
                                         const int64_t* strides16, float scale, float keep_prob, void* stream) {
  if (!q || !k || !v || !out || !lse || !dout || !dq || !dk || !dv || !delta_ws || !strides16) return TFB200_E_NULLPTR;
  if (B < 1 || H < 1 || Lq < 1 || Lk < 1 || keep_prob <= 0.f || keep_prob > 1.f || int64_t(B) * H > 65535)
    return TFB200_E_SHAPE;
  const int64_t* s = strides16;
  if (!aligned_view(q, s, 2) || !aligned_view(k, s + 2, 2) || !aligned_view(v, s + 4, 2) || !aligned_view(out, s + 6, 2) ||
      !aligned_view(dout, s + 8, 2) || !aligned_view(dq, s + 10, 2) || !aligned_view(dk, s + 12, 2) ||
      !aligned_view(dv, s + 14, 2))
    return TFB200_E_SHAPE;
  Strides st{s[0], s[1], s[2], s[3], s[4], s[5], s[6], s[7]};
  cudaStream_t cs = cudaStream_t(stream);
  const float inv_keep = 1.f / keep_prob;
  const uint32_t th = keep_threshold(keep_prob);
  const int64_t rows = int64_t(B) * H * Lq;
  dense_attn_bwd_delta_kernel<<<unsigned((rows + 7) / 8), 256, 0, cs>>>(out, dout, delta_ws, B, H, Lq, s[6], s[7], s[8], s[9]);
  dense_attn_bwd_dq_kernel<<<dim3((Lq + kRows - 1) / kRows, B * H), kWarps * 32, 0, cs>>>(
      q, k, v, key_pad, seed_dev, lse, delta_ws, dout, dq, H, Lq, Lk, scale, inv_keep, th, st, s[8], s[9], s[10], s[11]);
  dense_attn_bwd_dkv_kernel<<<dim3((Lk + kRows - 1) / kRows, B * H), kWarps * 32, 0, cs>>>(
      q, k, v, key_pad, seed_dev, lse, delta_ws, dout, dk, dv, H, Lq, Lk, scale, inv_keep, th, st, s[8], s[9], s[12], s[13],
      s[14], s[15]);
  msda_b200_count_launches(3);
  return int(cudaGetLastError());
}
