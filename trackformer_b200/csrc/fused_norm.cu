// Fused residual + dropout + LayerNorm for the transformer layers of the hot path (sm_90a).
//
// The reference's encoder/decoder layers compute   x = norm(x + dropout(branch))
// (src/trackformer/models/deformable_transformer.py:291-292, 284-285, 370-371, 377-378, 360-361) as three
// PyTorch ops forward (dropout, add, LayerNorm) and four backward (LayerNorm input grad, gamma/beta grad,
// add, dropout grad).  On a C2 frame each of these is a pass over a [22223, 256] fp32 tensor (22.8 MB) and
// PyTorch's LayerNorm backward alone makes several passes over it.  These kernels do each direction in ONE
// streaming pass (HBM-bound: forward reads x, branch, mask and writes s = x + drop(branch), y; backward reads
// dy, s, mask and writes dx, dbranch) with a deterministic two-stage column reduction for dgamma / dbeta.
//
//   forward : s = x + branch * mask * (1/keep)        (mask optional: no dropout in eval mode)
//             y = (s - mean) * rstd * gamma + beta    mean/rstd per row, biased variance, eps inside the sqrt
//   backward: xhat = (s - mean) * rstd;  g = dy * gamma
//             ds = rstd * (g - mean_c(g) - xhat * mean_c(g * xhat))
//             dx = ds;  dbranch = ds * mask * (1/keep);  dgamma = sum_r dy * xhat;  dbeta = sum_r dy
//
// One warp owns one row; a lane owns float4 packs lane, lane+32, ... (C % 4 == 0, C <= 1024 forward / 512 backward), so
// all global accesses are 128-bit and coalesced and the row statistics are two warp-shuffle reductions.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "dropout_hash.cuh"
#include "launch_counter.h"

using tfb200::keep_elem;
using tfb200::keep_threshold;

namespace {

constexpr int kWarpsPerCta = 8;
constexpr int kMaxPacks = 8;     // float4 packs per lane -> C <= 32 * 4 * 8 = 1024

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// PACKS = ceil(C / 128): a lane owns float4 packs lane, lane + 32, ...; packs beyond C/4 are masked, so any C % 4 == 0
// up to PACKS * 128 works (256 for the shipped models, 288 for the multi-frame TrackFormer configuration).
template <int PACKS>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
add_dropout_ln_fwd_kernel(const float* __restrict__ x, const float* __restrict__ branch,
                          const uint8_t* __restrict__ mask, const float* __restrict__ gamma,
                          const float* __restrict__ beta, float* __restrict__ s_out, float* __restrict__ y,
                          float* __restrict__ mean_out, float* __restrict__ rstd_out, int64_t rows, int C, float inv_keep,
                          float eps, const int64_t* __restrict__ seed_ptr, uint32_t keep_thresh) {
  const uint64_t seed = seed_ptr != nullptr ? uint64_t(__ldg(seed_ptr)) : 0;
  const int npk = C >> 2;
  const float inv_c = 1.f / float(C);
  const int lane = threadIdx.x & 31;
  const int64_t warp = int64_t(blockIdx.x) * kWarpsPerCta + (threadIdx.x >> 5);
  const int64_t nwarps = int64_t(gridDim.x) * kWarpsPerCta;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 ga[PACKS], be[PACKS];
#pragma unroll
  for (int k = 0; k < PACKS; ++k) {
    const bool on = k * 32 + lane < npk;
    ga[k] = on ? __ldg(reinterpret_cast<const float4*>(gamma) + k * 32 + lane) : zero4;
    be[k] = on ? __ldg(reinterpret_cast<const float4*>(beta) + k * 32 + lane) : zero4;
  }
  for (int64_t r = warp; r < rows; r += nwarps) {
    const float4* xr = reinterpret_cast<const float4*>(x + r * C);
    const float4* br = reinterpret_cast<const float4*>(branch + r * C);
    float4 s[PACKS];
    float sum = 0.f;
#pragma unroll
    for (int k = 0; k < PACKS; ++k) {
      s[k] = zero4;
      if (k * 32 + lane < npk) {
        const float4 a = __ldg(xr + k * 32 + lane);
        float4 b = __ldg(br + k * 32 + lane);
        if (mask != nullptr) {
          const uchar4 m = __ldg(reinterpret_cast<const uchar4*>(mask + r * C) + k * 32 + lane);
          b.x = m.x ? b.x * inv_keep : 0.f;
          b.y = m.y ? b.y * inv_keep : 0.f;
          b.z = m.z ? b.z * inv_keep : 0.f;
          b.w = m.w ? b.w * inv_keep : 0.f;
        } else if (seed_ptr != nullptr) {
          const uint64_t e = uint64_t(r) * C + 4 * (k * 32 + lane);
          b.x = keep_elem(seed, e + 0, keep_thresh) ? b.x * inv_keep : 0.f;
          b.y = keep_elem(seed, e + 1, keep_thresh) ? b.y * inv_keep : 0.f;
          b.z = keep_elem(seed, e + 2, keep_thresh) ? b.z * inv_keep : 0.f;
          b.w = keep_elem(seed, e + 3, keep_thresh) ? b.w * inv_keep : 0.f;
        }
        s[k] = make_float4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w);
        sum += (s[k].x + s[k].y) + (s[k].z + s[k].w);
      }
    }
    const float mean = warp_sum(sum) * inv_c;
    float var = 0.f;
#pragma unroll
    for (int k = 0; k < PACKS; ++k) {
      if (k * 32 + lane < npk) {
        const float dx = s[k].x - mean, dy = s[k].y - mean, dz = s[k].z - mean, dw = s[k].w - mean;
        var += (dx * dx + dy * dy) + (dz * dz + dw * dw);
      }
    }
    const float rstd = rsqrtf(warp_sum(var) * inv_c + eps);
#pragma unroll
    for (int k = 0; k < PACKS; ++k) {
      if (k * 32 + lane < npk) {
        float4 o;
        o.x = (s[k].x - mean) * rstd * ga[k].x + be[k].x;
        o.y = (s[k].y - mean) * rstd * ga[k].y + be[k].y;
        o.z = (s[k].z - mean) * rstd * ga[k].z + be[k].z;
        o.w = (s[k].w - mean) * rstd * ga[k].w + be[k].w;
        reinterpret_cast<float4*>(y + r * C)[k * 32 + lane] = o;
        if (s_out != nullptr) reinterpret_cast<float4*>(s_out + r * C)[k * 32 + lane] = s[k];
      }
    }
    if (lane == 0 && mean_out != nullptr) {
      mean_out[r] = mean;
      rstd_out[r] = rstd;
    }
  }
}

// partial[blockIdx][0][c] = sum over this CTA's rows of dy*xhat, partial[blockIdx][1][c] = sum of dy
template <int PACKS>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
add_dropout_ln_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ s, const uint8_t* __restrict__ mask,
                          const float* __restrict__ gamma, const float* __restrict__ mean_in,
                          const float* __restrict__ rstd_in, float* __restrict__ dx, float* __restrict__ dbranch,
                          float* __restrict__ partial, int64_t rows, int C, float inv_keep,
                          const int64_t* __restrict__ seed_ptr, uint32_t keep_thresh) {
  const uint64_t seed = seed_ptr != nullptr ? uint64_t(__ldg(seed_ptr)) : 0;
  constexpr int CP = PACKS * 128;                  // padded width of the shared reduction buffer
  __shared__ float red[kWarpsPerCta][2][CP];
  const int npk = C >> 2;
  const float inv_c = 1.f / float(C);
  const int lane = threadIdx.x & 31;
  const int wid = threadIdx.x >> 5;
  const int64_t warp = int64_t(blockIdx.x) * kWarpsPerCta + wid;
  const int64_t nwarps = int64_t(gridDim.x) * kWarpsPerCta;
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  float4 ga[PACKS], dg[PACKS], db[PACKS];
#pragma unroll
  for (int k = 0; k < PACKS; ++k) {
    ga[k] = (k * 32 + lane < npk) ? __ldg(reinterpret_cast<const float4*>(gamma) + k * 32 + lane) : zero4;
    dg[k] = zero4;
    db[k] = zero4;
  }
  for (int64_t r = warp; r < rows; r += nwarps) {
    const float mean = __ldg(mean_in + r), rstd = __ldg(rstd_in + r);
    float4 g[PACKS], xh[PACKS];
    float sg = 0.f, sgx = 0.f;
#pragma unroll
    for (int k = 0; k < PACKS; ++k) {
      g[k] = zero4;
      xh[k] = zero4;
      if (k * 32 + lane < npk) {
        const float4 d = __ldg(reinterpret_cast<const float4*>(dy + r * C) + k * 32 + lane);
        const float4 sv = __ldg(reinterpret_cast<const float4*>(s + r * C) + k * 32 + lane);
        xh[k] = make_float4((sv.x - mean) * rstd, (sv.y - mean) * rstd, (sv.z - mean) * rstd, (sv.w - mean) * rstd);
        g[k] = make_float4(d.x * ga[k].x, d.y * ga[k].y, d.z * ga[k].z, d.w * ga[k].w);
        dg[k].x += d.x * xh[k].x; dg[k].y += d.y * xh[k].y; dg[k].z += d.z * xh[k].z; dg[k].w += d.w * xh[k].w;
        db[k].x += d.x; db[k].y += d.y; db[k].z += d.z; db[k].w += d.w;
        sg += (g[k].x + g[k].y) + (g[k].z + g[k].w);
        sgx += (g[k].x * xh[k].x + g[k].y * xh[k].y) + (g[k].z * xh[k].z + g[k].w * xh[k].w);
      }
    }
    const float mg = warp_sum(sg) * inv_c;
    const float mgx = warp_sum(sgx) * inv_c;
#pragma unroll
    for (int k = 0; k < PACKS; ++k) {
      if (k * 32 + lane < npk) {
        float4 ds;
        ds.x = rstd * (g[k].x - mg - xh[k].x * mgx);
        ds.y = rstd * (g[k].y - mg - xh[k].y * mgx);
        ds.z = rstd * (g[k].z - mg - xh[k].z * mgx);
        ds.w = rstd * (g[k].w - mg - xh[k].w * mgx);
        reinterpret_cast<float4*>(dx + r * C)[k * 32 + lane] = ds;
        if (dbranch != nullptr) {
          if (mask != nullptr) {
            const uchar4 m = __ldg(reinterpret_cast<const uchar4*>(mask + r * C) + k * 32 + lane);
            ds.x = m.x ? ds.x * inv_keep : 0.f;
            ds.y = m.y ? ds.y * inv_keep : 0.f;
            ds.z = m.z ? ds.z * inv_keep : 0.f;
            ds.w = m.w ? ds.w * inv_keep : 0.f;
          } else if (seed_ptr != nullptr) {
            const uint64_t e = uint64_t(r) * C + 4 * (k * 32 + lane);
            ds.x = keep_elem(seed, e + 0, keep_thresh) ? ds.x * inv_keep : 0.f;
            ds.y = keep_elem(seed, e + 1, keep_thresh) ? ds.y * inv_keep : 0.f;
            ds.z = keep_elem(seed, e + 2, keep_thresh) ? ds.z * inv_keep : 0.f;
            ds.w = keep_elem(seed, e + 3, keep_thresh) ? ds.w * inv_keep : 0.f;
          }
          reinterpret_cast<float4*>(dbranch + r * C)[k * 32 + lane] = ds;
        }
      }
    }
  }
  // CTA-level column reduction of the 8 warps' partial sums, then one partial row per CTA
#pragma unroll
  for (int k = 0; k < PACKS; ++k) {
    reinterpret_cast<float4*>(&red[wid][0][0])[k * 32 + lane] = dg[k];
    reinterpret_cast<float4*>(&red[wid][1][0])[k * 32 + lane] = db[k];
  }
  __syncthreads();
  for (int c = threadIdx.x; c < 2 * C; c += kWarpsPerCta * 32) {
    const int which = c / C, col = c - which * C;
    float acc = 0.f;
#pragma unroll
    for (int w = 0; w < kWarpsPerCta; ++w) acc += red[w][which][col];
    partial[(size_t(blockIdx.x) * 2 + which) * C + col] = acc;
  }
}

// out[c] = sum_b partial[b][c] for c < width, written to out0 (c < split) / out1 (c >= split).  One warp per 32
// output columns: lane = column (coalesced 128-byte reads of each partial row), the 8 warps of a CTA split the partial
// rows and combine through shared memory in a fixed order -> deterministic.
constexpr int kFinishWarps = 32;
__global__ void __launch_bounds__(kFinishWarps * 32)
column_partials_finish_kernel(const float* __restrict__ partial, float* __restrict__ out0, float* __restrict__ out1,
                              int nblocks, int width, int split) {
  // 8 CTAs x 8 warps walking 592 partial rows one dependent load at a time took ~9 us (latency-bound, 63 calls per
  // step); 32 warps with four independent loads in flight each bring that to the launch floor.  Fixed order -> deterministic.
  __shared__ float acc_s[kFinishWarps][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  if (c < width) {
    int b = w;
    for (; b + 3 * kFinishWarps < nblocks; b += 4 * kFinishWarps) {
      a0 += partial[size_t(b) * width + c];
      a1 += partial[size_t(b + kFinishWarps) * width + c];
      a2 += partial[size_t(b + 2 * kFinishWarps) * width + c];
      a3 += partial[size_t(b + 3 * kFinishWarps) * width + c];
    }
    for (; b < nblocks; b += kFinishWarps) a0 += partial[size_t(b) * width + c];
  }
  acc_s[w][lane] = (a0 + a1) + (a2 + a3);
  __syncthreads();
  if (w == 0 && c < width) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < kFinishWarps; ++k) t += acc_s[k][lane];
    if (c < split) out0[c] = t; else out1[c - split] = t;
  }
}

// Column sums of a [rows, C] matrix (bias gradients of the big encoder Linears): same row-per-warp streaming as the
// LayerNorm backward, partial[blockIdx][c].
template <int PACKS>
__global__ void __launch_bounds__(kWarpsPerCta * 32)
colsum_kernel(const float* __restrict__ x, float* __restrict__ partial, int64_t rows, int C) {
  constexpr int CP = PACKS * 128;
  __shared__ float red[kWarpsPerCta][CP];
  const int npk = C >> 2;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int64_t warp = int64_t(blockIdx.x) * kWarpsPerCta + wid;
  const int64_t nwarps = int64_t(gridDim.x) * kWarpsPerCta;
  float4 acc[PACKS];
#pragma unroll
  for (int k = 0; k < PACKS; ++k) acc[k] = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int64_t r = warp; r < rows; r += nwarps) {
#pragma unroll
    for (int k = 0; k < PACKS; ++k) {
      if (k * 32 + lane < npk) {
        const float4 v = __ldg(reinterpret_cast<const float4*>(x + r * C) + k * 32 + lane);
        acc[k].x += v.x; acc[k].y += v.y; acc[k].z += v.z; acc[k].w += v.w;
      }
    }
  }
#pragma unroll
  for (int k = 0; k < PACKS; ++k) reinterpret_cast<float4*>(&red[wid][0])[k * 32 + lane] = acc[k];
  __syncthreads();
  for (int c = threadIdx.x; c < C; c += kWarpsPerCta * 32) {
    float t = 0.f;
#pragma unroll
    for (int w = 0; w < kWarpsPerCta; ++w) t += red[w][c];
    partial[size_t(blockIdx.x) * C + c] = t;
  }
}

// Small matrices (the decoder side: a few hundred rows): ONE launch, CTA = 32 columns x 8 warps striding the rows,
// fixed summation order.  (The generic ATen reduction needs 7-16 us for a [300, 256] column sum, ~50 of them per step.)
constexpr int kSmallWarps = 32;
__global__ void __launch_bounds__(kSmallWarps * 32)
colsum_small_kernel(const float* __restrict__ x, float* __restrict__ out, int rows, int C) {
  // (first version: 8 warps per CTA, 10.7 us per [300, 256] call under ncu -- latency bound; 32 warps x 4 loads in flight)
  __shared__ float red[kSmallWarps][32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const int c = blockIdx.x * 32 + lane;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
  if (c < C) {
    int r = w;
    for (; r + 3 * kSmallWarps < rows; r += 4 * kSmallWarps) {
      a0 += __ldg(x + size_t(r) * C + c);
      a1 += __ldg(x + size_t(r + kSmallWarps) * C + c);
      a2 += __ldg(x + size_t(r + 2 * kSmallWarps) * C + c);
      a3 += __ldg(x + size_t(r + 3 * kSmallWarps) * C + c);
    }
    for (; r < rows; r += kSmallWarps) a0 += __ldg(x + size_t(r) * C + c);
  }
  red[w][lane] = (a0 + a1) + (a2 + a3);
  __syncthreads();
  if (w == 0 && c < C) {
    float t = 0.f;
#pragma unroll
    for (int k = 0; k < kSmallWarps; ++k) t += red[k][lane];
    out[c] = t;
  }
}

// Fused ReLU + inverted dropout for the FFN hidden activation, mask-free: the keep decision is a counter-based hash
// of (seed, element index); the backward needs no mask because h > 0 <=> (a > 0 and kept).

__global__ void __launch_bounds__(256)
relu_dropout_fwd_kernel(const float* __restrict__ a, float* __restrict__ h, const int64_t* __restrict__ seed_ptr,
                        int64_t n4, float inv_keep, uint32_t keep_thresh, int training) {
  const uint64_t seed = training ? uint64_t(__ldg(seed_ptr)) : 0;
  for (int64_t i = int64_t(blockIdx.x) * 256 + threadIdx.x; i < n4; i += int64_t(gridDim.x) * 256) {
    const float4 v = __ldg(reinterpret_cast<const float4*>(a) + i);
    float4 o;
    if (training) {
      o.x = (v.x > 0.f && keep_elem(seed, 4 * i + 0, keep_thresh)) ? v.x * inv_keep : 0.f;
      o.y = (v.y > 0.f && keep_elem(seed, 4 * i + 1, keep_thresh)) ? v.y * inv_keep : 0.f;
      o.z = (v.z > 0.f && keep_elem(seed, 4 * i + 2, keep_thresh)) ? v.z * inv_keep : 0.f;
      o.w = (v.w > 0.f && keep_elem(seed, 4 * i + 3, keep_thresh)) ? v.w * inv_keep : 0.f;
    } else {
      o = make_float4(fmaxf(v.x, 0.f), fmaxf(v.y, 0.f), fmaxf(v.z, 0.f), fmaxf(v.w, 0.f));
    }
    reinterpret_cast<float4*>(h)[i] = o;
  }
}

__global__ void __launch_bounds__(256)
relu_dropout_bwd_kernel(const float* __restrict__ gh, const float* __restrict__ h, float* __restrict__ ga, int64_t n4,
                        float inv_keep) {
  for (int64_t i = int64_t(blockIdx.x) * 256 + threadIdx.x; i < n4; i += int64_t(gridDim.x) * 256) {
    const float4 g = __ldg(reinterpret_cast<const float4*>(gh) + i);
    const float4 o = __ldg(reinterpret_cast<const float4*>(h) + i);
    reinterpret_cast<float4*>(ga)[i] = make_float4(o.x > 0.f ? g.x * inv_keep : 0.f, o.y > 0.f ? g.y * inv_keep : 0.f,
                                                   o.z > 0.f ? g.z * inv_keep : 0.f, o.w > 0.f ? g.w * inv_keep : 0.f);
  }
}

int grid_for(int64_t rows) {
  const int64_t need = (rows + kWarpsPerCta - 1) / kWarpsPerCta;
  const int64_t cap = TFB200_LN_MAX_CTAS;          // persistent: 132 SMs x 4 resident CTAs
  return int(need < cap ? (need > 0 ? need : 1) : cap);
}

}  // namespace

extern "C" {

int tfb200_ln_partial_ctas(int64_t rows) { return grid_for(rows); }

static int ln_forward(const float* x, const float* branch, const uint8_t* keep_mask, const int64_t* seed_dev,
                      const float* gamma, const float* beta, float* s_out, float* y, float* mean, float* rstd,
                      int64_t rows, int C, float keep_prob, float eps, void* stream) {
  if (!x || !branch || !gamma || !beta || !y) return TFB200_E_NULLPTR;
  if (rows < 0 || C <= 0 || C % 4 != 0 || C > 128 * kMaxPacks) return TFB200_E_SHAPE;
  if (rows == 0) return 0;
  const float inv_keep = (keep_mask || seed_dev) ? 1.f / keep_prob : 1.f;
  const uint32_t thresh = keep_threshold(keep_prob);
  const int grid = grid_for(rows);
  cudaStream_t st = cudaStream_t(stream);
#define TFB200_FWD(P)                                                                                          \
  add_dropout_ln_fwd_kernel<P><<<grid, kWarpsPerCta * 32, 0, st>>>(x, branch, keep_mask, gamma, beta, s_out, y, \
                                                                   mean, rstd, rows, C, inv_keep, eps, seed_dev, thresh)
  switch ((C + 127) / 128) {
    case 1: TFB200_FWD(1); break;
    case 2: TFB200_FWD(2); break;
    case 3: TFB200_FWD(3); break;
    case 4: TFB200_FWD(4); break;
    case 5: case 6: case 7: case 8: TFB200_FWD(8); break;
    default: return TFB200_E_SHAPE;
  }
#undef TFB200_FWD
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

static int ln_backward(const float* dy, const float* s, const uint8_t* keep_mask, const int64_t* seed_dev,
                       const float* gamma, const float* mean, const float* rstd, float* dx, float* dbranch,
                       float* dgamma, float* dbeta, float* partial_ws, int64_t rows, int C, float keep_prob,
                       void* stream) {
  if (!dy || !s || !gamma || !mean || !rstd || !dx || !dgamma || !dbeta || !partial_ws) return TFB200_E_NULLPTR;
  if (rows < 0 || C <= 0 || C % 4 != 0 || C > 512) return TFB200_E_SHAPE;
  cudaStream_t st = cudaStream_t(stream);
  if (rows == 0) {
    cudaMemsetAsync(dgamma, 0, sizeof(float) * C, st);
    cudaMemsetAsync(dbeta, 0, sizeof(float) * C, st);
    return int(cudaGetLastError());
  }
  const float inv_keep = (keep_mask || seed_dev) ? 1.f / keep_prob : 1.f;
  const uint32_t thresh = keep_threshold(keep_prob);
  const int grid = grid_for(rows);
#define TFB200_BWD(P)                                                                                           \
  add_dropout_ln_bwd_kernel<P><<<grid, kWarpsPerCta * 32, 0, st>>>(dy, s, keep_mask, gamma, mean, rstd, dx, dbranch, \
                                                                   partial_ws, rows, C, inv_keep, seed_dev, thresh)
  switch ((C + 127) / 128) {
    case 1: TFB200_BWD(1); break;
    case 2: TFB200_BWD(2); break;
    case 3: TFB200_BWD(3); break;
    case 4: TFB200_BWD(4); break;
    default: return TFB200_E_SHAPE;   // the 48 KB static shared-memory reduction buffer bounds C at 512 here
  }
#undef TFB200_BWD
  column_partials_finish_kernel<<<(2 * C + 31) / 32, kFinishWarps * 32, 0, st>>>(partial_ws, dgamma, dbeta, grid, 2 * C, C);
  msda_b200_count_launches(2);
  return int(cudaGetLastError());
}

int tfb200_add_dropout_layernorm_fwd_f32(const float* x, const float* branch, const uint8_t* keep_mask,
                                         const float* gamma, const float* beta, float* s_out, float* y,
                                         float* mean, float* rstd, int64_t rows, int C, float keep_prob, float eps,
                                         void* stream) {
  return ln_forward(x, branch, keep_mask, nullptr, gamma, beta, s_out, y, mean, rstd, rows, C, keep_prob, eps, stream);
}

int tfb200_add_dropout_layernorm_seeded_fwd_f32(const float* x, const float* branch, const int64_t* seed_dev,
                                                const float* gamma, const float* beta, float* s_out, float* y,
                                                float* mean, float* rstd, int64_t rows, int C, float keep_prob,
                                                float eps, void* stream) {
  if (!seed_dev) return TFB200_E_NULLPTR;
  return ln_forward(x, branch, nullptr, seed_dev, gamma, beta, s_out, y, mean, rstd, rows, C, keep_prob, eps, stream);
}

int tfb200_add_dropout_layernorm_bwd_f32(const float* dy, const float* s, const uint8_t* keep_mask,
                                         const float* gamma, const float* mean, const float* rstd, float* dx,
                                         float* dbranch, float* dgamma, float* dbeta, float* partial_ws,
                                         int64_t rows, int C, float keep_prob, void* stream) {
  return ln_backward(dy, s, keep_mask, nullptr, gamma, mean, rstd, dx, dbranch, dgamma, dbeta, partial_ws, rows, C,
                     keep_prob, stream);
}

int tfb200_add_dropout_layernorm_seeded_bwd_f32(const float* dy, const float* s, const int64_t* seed_dev,
                                                const float* gamma, const float* mean, const float* rstd, float* dx,
                                                float* dbranch, float* dgamma, float* dbeta, float* partial_ws,
                                                int64_t rows, int C, float keep_prob, void* stream) {
  if (!seed_dev) return TFB200_E_NULLPTR;
  return ln_backward(dy, s, nullptr, seed_dev, gamma, mean, rstd, dx, dbranch, dgamma, dbeta, partial_ws, rows, C,
                     keep_prob, stream);
}

int tfb200_colsum_f32(const float* x, float* out, float* partial_ws, int64_t rows, int C, void* stream) {
  if (!x || !out || !partial_ws) return TFB200_E_NULLPTR;
  if (rows < 0 || C <= 0 || C % 4 != 0 || C > 128 * kMaxPacks) return TFB200_E_SHAPE;
  cudaStream_t st = cudaStream_t(stream);
  if (rows == 0) {
    cudaMemsetAsync(out, 0, sizeof(float) * C, st);
    return int(cudaGetLastError());
  }
  if (rows <= 2048) {
    colsum_small_kernel<<<(C + 31) / 32, kSmallWarps * 32, 0, st>>>(x, out, int(rows), C);
    msda_b200_count_launches(1);
    return int(cudaGetLastError());
  }
  const int grid = grid_for(rows);
#define TFB200_CS(P) colsum_kernel<P><<<grid, kWarpsPerCta * 32, 0, st>>>(x, partial_ws, rows, C)
  switch ((C + 127) / 128) {
    case 1: TFB200_CS(1); break;
    case 2: TFB200_CS(2); break;
    case 3: TFB200_CS(3); break;
    case 4: TFB200_CS(4); break;
    case 5: case 6: case 7: case 8: TFB200_CS(8); break;
    default: return TFB200_E_SHAPE;
  }
#undef TFB200_CS
  column_partials_finish_kernel<<<(C + 31) / 32, kFinishWarps * 32, 0, st>>>(partial_ws, out, out, grid, C, C);
  msda_b200_count_launches(2);
  return int(cudaGetLastError());
}

int tfb200_relu_dropout_fwd_f32(const float* a, float* h, const int64_t* seed_dev, int64_t n, float keep_prob,
                                int training, void* stream) {
  if (!a || !h || (training && !seed_dev)) return TFB200_E_NULLPTR;
  if (n < 0 || n % 4 != 0) return TFB200_E_SHAPE;
  if (n == 0) return 0;
  const int64_t n4 = n / 4;
  const int grid = int(n4 / 256 < 132 * 16 ? (n4 + 255) / 256 : 132 * 16);
  const uint32_t thresh = keep_threshold(keep_prob);
  relu_dropout_fwd_kernel<<<grid, 256, 0, cudaStream_t(stream)>>>(a, h, seed_dev, n4, training ? 1.f / keep_prob : 1.f,
                                                                  thresh, training);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

int tfb200_relu_dropout_bwd_f32(const float* grad_h, const float* h, float* grad_a, int64_t n, float keep_prob,
                                int training, void* stream) {
  if (!grad_h || !h || !grad_a) return TFB200_E_NULLPTR;
  if (n < 0 || n % 4 != 0) return TFB200_E_SHAPE;
  if (n == 0) return 0;
  const int64_t n4 = n / 4;
  const int grid = int(n4 / 256 < 132 * 16 ? (n4 + 255) / 256 : 132 * 16);
  relu_dropout_bwd_kernel<<<grid, 256, 0, cudaStream_t(stream)>>>(grad_h, h, grad_a, n4, training ? 1.f / keep_prob : 1.f);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

}  // extern "C"

// ------------------------------------------------------------------------------------------------------------------
// Sampling prep: proj = [offsets (M*L*P*2) | logits (M*L*P)] per query  ->  sampling locations + attention weights.
// Fuses what the reference's MSDeformAttn.forward does with five PyTorch ops per call (ops/modules/ms_deform_attn.py:
// 69-82): split + view of the two projections, softmax over the L*P logits of each head, offset normalisation and the
// reference-point add.  One thread per sample; the LP (power of two <= 32) samples of one (query, head) sit in
// consecutive lanes, so the softmax is a segmented warp-shuffle reduction and every stream is read/written coalesced.
//   2-d reference points: loc = ref[l] + off / (shape_l[0], shape_l[1])      (the reference divides (x, y) by (H, W))
//   4-d reference boxes : loc = ref_xy[l] + off / P * ref_wh[l] * 0.5
// ------------------------------------------------------------------------------------------------------------------
namespace {

template <int LP>
__device__ __forceinline__ float seg_max(float v) {
#pragma unroll
  for (int o = LP / 2; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
template <int LP>
__device__ __forceinline__ float seg_sum(float v) {
#pragma unroll
  for (int o = LP / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// proj: [rows][3*M*LP] (row = (n, q)); ref: [rows][L][RD]; shapes: [L][2] float; loc: [rows][M][LP][2]; attn: [rows][M][LP]
template <int LP, int RD>
__global__ void __launch_bounds__(256)
sampling_prep_fwd_kernel(const float* __restrict__ proj, const float* __restrict__ ref, const float* __restrict__ shapes,
                         float* __restrict__ loc, float* __restrict__ attn, int64_t total, int M, int P) {
  const int64_t stride_t = int64_t(gridDim.x) * 256;
  const int mlp = M * LP;
  for (int64_t t0 = int64_t(blockIdx.x) * 256; t0 < total; t0 += stride_t) {   // whole warps stay together (total % 32 == 0)
    const int64_t t = t0 + threadIdx.x;
    const bool ok = t < total;
    const int64_t tt = ok ? t : total - 1;
    const int64_t row = tt / mlp;
    const int rem = int(tt - row * mlp);          // m * LP + s
    const int s = rem % LP, l = s / P;
    const float* prow = proj + row * 3 * mlp;
    const float2 off = __ldg(reinterpret_cast<const float2*>(prow) + rem);
    const float logit = __ldg(prow + 2 * mlp + rem);
    const float mx = seg_max<LP>(logit);
    const float e = expf(logit - mx);
    const float a = e / seg_sum<LP>(e);
    float2 o;
    if (RD == 2) {
      const float2 r = __ldg(reinterpret_cast<const float2*>(ref) + row * (LP / P) + l);
      o.x = r.x + off.x / __ldg(shapes + 2 * l);
      o.y = r.y + off.y / __ldg(shapes + 2 * l + 1);
    } else {
      const float4 r = __ldg(reinterpret_cast<const float4*>(ref) + row * (LP / P) + l);
      o.x = r.x + off.x / float(P) * r.z * 0.5f;
      o.y = r.y + off.y / float(P) * r.w * 0.5f;
    }
    if (ok) {
      reinterpret_cast<float2*>(loc)[t] = o;
      attn[t] = a;
    }
  }
}

// grad_proj offsets part = grad_loc * d(loc)/d(off); logits part = attn * (ga - sum_s attn*ga)
template <int LP, int RD>
__global__ void __launch_bounds__(256)
sampling_prep_bwd_kernel(const float* __restrict__ grad_loc, const float* __restrict__ grad_attn,
                         const float* __restrict__ attn, const float* __restrict__ ref, const float* __restrict__ shapes,
                         float* __restrict__ grad_proj, int64_t total, int M, int P) {
  const int64_t stride_t = int64_t(gridDim.x) * 256;
  const int mlp = M * LP;
  for (int64_t t0 = int64_t(blockIdx.x) * 256; t0 < total; t0 += stride_t) {
    const int64_t t = t0 + threadIdx.x;
    const bool ok = t < total;
    const int64_t tt = ok ? t : total - 1;
    const int64_t row = tt / mlp;
    const int rem = int(tt - row * mlp);
    const int s = rem % LP, l = s / P;
    const float2 gl = __ldg(reinterpret_cast<const float2*>(grad_loc) + tt);
    const float ga = __ldg(grad_attn + tt), a = __ldg(attn + tt);
    const float dot = seg_sum<LP>(a * ga);
    float2 go;
    if (RD == 2) {
      go.x = gl.x / __ldg(shapes + 2 * l);
      go.y = gl.y / __ldg(shapes + 2 * l + 1);
    } else {
      const float4 r = __ldg(reinterpret_cast<const float4*>(ref) + row * (LP / P) + l);
      go.x = gl.x / float(P) * r.z * 0.5f;
      go.y = gl.y / float(P) * r.w * 0.5f;
    }
    if (ok) {
      float* grow = grad_proj + row * 3 * mlp;
      reinterpret_cast<float2*>(grow)[rem] = go;
      grow[2 * mlp + rem] = a * (ga - dot);
    }
  }
}

int prep_grid(int64_t total) {
  const int64_t need = (total + 255) / 256;
  return int(need < 132 * 16 ? need : 132 * 16);
}

}  // namespace

extern "C" {

int tfb200_sampling_prep_fwd_f32(const float* proj, const float* ref, const float* shapes_f32, float* loc, float* attn,
                                 int64_t rows, int M, int L, int P, int ref_dim, void* stream) {
  if (!proj || !ref || !loc || !attn || (ref_dim == 2 && !shapes_f32)) return TFB200_E_NULLPTR;
  const int LP = L * P;
  if (rows < 0 || M <= 0 || (ref_dim != 2 && ref_dim != 4) || (LP != 4 && LP != 8 && LP != 16 && LP != 32) ||
      (int64_t(M) * LP) % 32 != 0)
    return TFB200_E_SHAPE;
  const int64_t total = rows * M * LP;
  if (total == 0) return 0;
  cudaStream_t st = cudaStream_t(stream);
#define TFB200_PREP(LP_, RD_) \
  sampling_prep_fwd_kernel<LP_, RD_><<<prep_grid(total), 256, 0, st>>>(proj, ref, shapes_f32, loc, attn, total, M, P)
  if (ref_dim == 2) {
    if (LP == 4) TFB200_PREP(4, 2); else if (LP == 8) TFB200_PREP(8, 2); else if (LP == 16) TFB200_PREP(16, 2); else TFB200_PREP(32, 2);
  } else {
    if (LP == 4) TFB200_PREP(4, 4); else if (LP == 8) TFB200_PREP(8, 4); else if (LP == 16) TFB200_PREP(16, 4); else TFB200_PREP(32, 4);
  }
#undef TFB200_PREP
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

int tfb200_sampling_prep_bwd_f32(const float* grad_loc, const float* grad_attn, const float* attn, const float* ref,
                                 const float* shapes_f32, float* grad_proj, int64_t rows, int M, int L, int P, int ref_dim,
                                 void* stream) {
  if (!grad_loc || !grad_attn || !attn || !ref || !grad_proj || (ref_dim == 2 && !shapes_f32)) return TFB200_E_NULLPTR;
  const int LP = L * P;
  if (rows < 0 || M <= 0 || (ref_dim != 2 && ref_dim != 4) || (LP != 4 && LP != 8 && LP != 16 && LP != 32) ||
      (int64_t(M) * LP) % 32 != 0)
    return TFB200_E_SHAPE;
  const int64_t total = rows * M * LP;
  if (total == 0) return 0;
  cudaStream_t st = cudaStream_t(stream);
#define TFB200_PREPB(LP_, RD_) \
  sampling_prep_bwd_kernel<LP_, RD_><<<prep_grid(total), 256, 0, st>>>(grad_loc, grad_attn, attn, ref, shapes_f32, \
                                                                       grad_proj, total, M, P)
  if (ref_dim == 2) {
    if (LP == 4) TFB200_PREPB(4, 2); else if (LP == 8) TFB200_PREPB(8, 2); else if (LP == 16) TFB200_PREPB(16, 2); else TFB200_PREPB(32, 2);
  } else {
    if (LP == 4) TFB200_PREPB(4, 4); else if (LP == 8) TFB200_PREPB(8, 4); else if (LP == 16) TFB200_PREPB(16, 4); else TFB200_PREPB(32, 4);
  }
#undef TFB200_PREPB
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

}  // extern "C"
