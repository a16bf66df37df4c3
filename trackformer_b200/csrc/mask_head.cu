// Segmentation mask head of DETRSegm between its convolutions, and its loss (sm_90a).
//
// Reference: src/trackformer/models/detr_segmentation.py:111-216 (MaskHeadSmallConv, MHAttentionMap) and
// src/trackformer/models/detr.py:330-357 + util/misc.py:522-571 (loss_masks: bilinear upsampling, sigmoid focal
// loss, dice).  The reference concatenates `_expand(src, Q)` -- one copy of the image's 256-channel stride-16 map per
// query -- with the per-query attention maps and convolves the result, and expands every adapter output the same
// way.  Here the convolutions run per image for the image part and per query for the query part, and these kernels
// take the image part as a broadcast operand instead:
//   group_norm_relu : relu(GroupNorm(x[n] + addend[n / per_image]))   channels-last [N][HW][C]
//   upsample_add    : a[n / per_image] + nearest_upsample(x[n])      channels-last
// Every reduction over the queries of an image (addend / adapter gradients) and over samples (GroupNorm affine
// gradients) runs in a fixed order: no float atomics, so results are reproducible run to run.
//
// Layouts: per-query maps are NHWC ("channels_last") as the cuDNN convolutions around them produce; the attention
// maps are [B][Q][heads][HW] as the reference's bbox_mask.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "launch_counter.h"

namespace {

constexpr int kHeadDim = 32;

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// block-wide sum / max for blockDim.x <= 1024; `red` holds >= 32 floats; every thread gets the result
__device__ float block_sum(float v, float* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  float t = 0.f;
  for (int i = 0; i < nw; ++i) t += red[i];
  return t;
}

__device__ float block_max(float v, float* red) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  float t = -INFINITY;
  for (int i = 0; i < nw; ++i) t = fmaxf(t, red[i]);
  return t;
}

// ------------------------------------------------------------------------------------------------------------------
// MHAttentionMap core: w[b][q][h][:] = softmax_p(scale * q[b][q][h] . k[b][p][h], -inf where pad[b][p])
// one CTA per (b, q, h)
__global__ void __launch_bounds__(256)
mask_attn_fwd_kernel(const float* __restrict__ q, const float* __restrict__ k, const uint8_t* __restrict__ pad,
                     float* __restrict__ w, int Q, int HW, int heads, float scale) {
  __shared__ float4 qs[kHeadDim / 4];
  __shared__ float red[32];
  const int row = blockIdx.x;                       // (b * Q + q) * heads + h
  const int h = row % heads, bq = row / heads, b = bq / Q;
  const int D = heads * kHeadDim;
  if (threadIdx.x < kHeadDim / 4)
    qs[threadIdx.x] = reinterpret_cast<const float4*>(q + int64_t(bq) * D + h * kHeadDim)[threadIdx.x];
  __syncthreads();
  float* out = w + int64_t(row) * HW;
  const float* kb = k + int64_t(b) * HW * D + h * kHeadDim;
  float m = -INFINITY;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    const float4* kp = reinterpret_cast<const float4*>(kb + int64_t(p) * D);
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < kHeadDim / 4; ++i) {
      const float4 a = qs[i], c = kp[i];
      s = fmaf(a.x, c.x, s); s = fmaf(a.y, c.y, s); s = fmaf(a.z, c.z, s); s = fmaf(a.w, c.w, s);
    }
    s *= scale;
    if (pad != nullptr && pad[int64_t(b) * HW + p]) s = -INFINITY;
    out[p] = s;
    m = fmaxf(m, s);
  }
  m = block_max(m, red);
  float sum = 0.f;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    const float e = expf(out[p] - m);
    out[p] = e;
    sum += e;
  }
  sum = block_sum(sum, red);
  for (int p = threadIdx.x; p < HW; p += blockDim.x) out[p] = out[p] / sum;
}

// ds = w * (dw - sum(dw * w)) (softmax backward), dq = scale * ds . k; one CTA per (b, q, h)
__global__ void __launch_bounds__(256)
mask_attn_bwd_dq_kernel(const float* __restrict__ k, const float* __restrict__ w, const float* __restrict__ dw,
                        float* __restrict__ ds, float* __restrict__ dq, int Q, int HW, int heads, float scale) {
  __shared__ float red[32];
  __shared__ float part[8][kHeadDim];
  const int row = blockIdx.x;
  const int h = row % heads, bq = row / heads, b = bq / Q;
  const int D = heads * kHeadDim;
  const float* wr = w + int64_t(row) * HW;
  const float* dwr = dw + int64_t(row) * HW;
  float* dsr = ds + int64_t(row) * HW;
  float dot = 0.f;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) dot = fmaf(wr[p], dwr[p], dot);
  dot = block_sum(dot, red);
  float acc[kHeadDim];
#pragma unroll
  for (int c = 0; c < kHeadDim; ++c) acc[c] = 0.f;
  const float* kb = k + int64_t(b) * HW * D + h * kHeadDim;
  for (int p = threadIdx.x; p < HW; p += blockDim.x) {
    const float g = wr[p] * (dwr[p] - dot);
    dsr[p] = g;
    const float4* kp = reinterpret_cast<const float4*>(kb + int64_t(p) * D);
#pragma unroll
    for (int i = 0; i < kHeadDim / 4; ++i) {
      const float4 c = kp[i];
      acc[4 * i] = fmaf(g, c.x, acc[4 * i]);
      acc[4 * i + 1] = fmaf(g, c.y, acc[4 * i + 1]);
      acc[4 * i + 2] = fmaf(g, c.z, acc[4 * i + 2]);
      acc[4 * i + 3] = fmaf(g, c.w, acc[4 * i + 3]);
    }
  }
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
#pragma unroll
  for (int c = 0; c < kHeadDim; ++c) {
    const float v = warp_sum(acc[c]);
    if (lane == 0) part[wid][c] = v;
  }
  __syncthreads();
  if (threadIdx.x < kHeadDim) {
    float t = 0.f;
    for (int i = 0; i < int(blockDim.x >> 5); ++i) t += part[i][threadIdx.x];
    dq[int64_t(bq) * D + h * kHeadDim + threadIdx.x] = scale * t;
  }
}

// dk[b][p][h][:] = scale * sum_q ds[b][q][h][p] * q[b][q][h][:]; grid (ceil(HW / 128), heads, B), thread per p
__global__ void __launch_bounds__(128)
mask_attn_bwd_dk_kernel(const float* __restrict__ q, const float* __restrict__ ds, float* __restrict__ dk, int Q,
                        int HW, int heads, float scale) {
  __shared__ float qt[32][kHeadDim];
  const int p = blockIdx.x * 128 + threadIdx.x, h = blockIdx.y, b = blockIdx.z;
  const int D = heads * kHeadDim;
  float acc[kHeadDim];
#pragma unroll
  for (int c = 0; c < kHeadDim; ++c) acc[c] = 0.f;
  for (int q0 = 0; q0 < Q; q0 += 32) {
    const int nq = min(32, Q - q0);
    __syncthreads();
    for (int i = threadIdx.x; i < nq * kHeadDim; i += 128)
      qt[i / kHeadDim][i % kHeadDim] = q[(int64_t(b) * Q + q0 + i / kHeadDim) * D + h * kHeadDim + i % kHeadDim];
    __syncthreads();
    if (p < HW) {
      for (int j = 0; j < nq; ++j) {
        const float g = ds[((int64_t(b) * Q + q0 + j) * heads + h) * HW + p];
#pragma unroll
        for (int c = 0; c < kHeadDim; ++c) acc[c] = fmaf(g, qt[j][c], acc[c]);
      }
    }
  }
  if (p < HW) {
    float4* o = reinterpret_cast<float4*>(dk + (int64_t(b) * HW + p) * D + h * kHeadDim);
#pragma unroll
    for (int i = 0; i < kHeadDim / 4; ++i)
      o[i] = make_float4(scale * acc[4 * i], scale * acc[4 * i + 1], scale * acc[4 * i + 2], scale * acc[4 * i + 3]);
  }
}

// ------------------------------------------------------------------------------------------------------------------
// GroupNorm + ReLU over one (sample, group) per CTA.  Thread t owns channel t % cpg of the group and walks the pixels
// t / cpg, t / cpg + step, ...: a warp reads contiguous runs of the group's channels, and per-channel partial sums
// (affine gradients) stay in registers until one ordered reduction at the end.
__device__ __forceinline__ int gn_threads(int cpg) { return cpg * (256 / cpg); }

__global__ void __launch_bounds__(256)
group_norm_relu_fwd_kernel(const float* __restrict__ x, const float* __restrict__ addend,
                           const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ y,
                           float* __restrict__ mean_out, float* __restrict__ rstd_out, int per_image, int64_t HW, int C,
                           int groups, float eps) {
  __shared__ float red[32];
  const int n = blockIdx.x / groups, g = blockIdx.x % groups, cpg = C / groups;
  const int nt = gn_threads(cpg);
  const bool active = threadIdx.x < nt;
  const int ch = g * cpg + threadIdx.x % cpg;
  const int64_t p0 = threadIdx.x / cpg, step = nt / cpg;
  const float* xs = x + int64_t(n) * HW * C + ch;
  const float* as = addend != nullptr ? addend + int64_t(n / per_image) * HW * C + ch : nullptr;
  float s = 0.f;
  if (active)
    for (int64_t p = p0; p < HW; p += step) s += xs[p * C] + (as ? as[p * C] : 0.f);
  const float cnt = float(HW * cpg);
  const float mean = block_sum(s, red) / cnt;
  float v = 0.f;
  if (active)
    for (int64_t p = p0; p < HW; p += step) {
      const float d = xs[p * C] + (as ? as[p * C] : 0.f) - mean;
      v = fmaf(d, d, v);
    }
  const float rstd = rsqrtf(block_sum(v, red) / cnt + eps);
  if (active) {
    const float ga = gamma[ch] * rstd, be = beta[ch];
    float* ys = y + int64_t(n) * HW * C + ch;
    for (int64_t p = p0; p < HW; p += step)
      ys[p * C] = fmaxf(fmaf(xs[p * C] + (as ? as[p * C] : 0.f) - mean, ga, be), 0.f);
  }
  if (threadIdx.x == 0) {
    mean_out[blockIdx.x] = mean;
    rstd_out[blockIdx.x] = rstd;
  }
}

// dx of GroupNorm + ReLU, and per-sample affine partials partial[n][0][c] (dgamma) / partial[n][1][c] (dbeta)
__global__ void __launch_bounds__(256)
group_norm_relu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ addend,
                           const float* __restrict__ y, const float* __restrict__ gamma,
                           const float* __restrict__ mean_in, const float* __restrict__ rstd_in, float* __restrict__ dx,
                           float* __restrict__ partial, int per_image, int64_t HW, int C, int groups) {
  __shared__ float red[32];
  __shared__ float pg[256], pb[256];
  const int n = blockIdx.x / groups, g = blockIdx.x % groups, cpg = C / groups;
  const int nt = gn_threads(cpg);
  const bool active = threadIdx.x < nt;
  const int ch = g * cpg + threadIdx.x % cpg;
  const int64_t p0 = threadIdx.x / cpg, step = nt / cpg;
  const int64_t base = int64_t(n) * HW * C + ch;
  const float* as = addend != nullptr ? addend + int64_t(n / per_image) * HW * C + ch : nullptr;
  const float mean = mean_in[blockIdx.x], rstd = rstd_in[blockIdx.x];
  const float ga = active ? gamma[ch] : 0.f;
  float sd = 0.f, sdx = 0.f, dg = 0.f, db = 0.f;
  if (active)
    for (int64_t p = p0; p < HW; p += step) {
      const int64_t i = base + p * C;
      const float gy = y[i] > 0.f ? dy[i] : 0.f;
      const float xh = (x[i] + (as ? as[p * C] : 0.f) - mean) * rstd;
      dg = fmaf(gy, xh, dg);
      db += gy;
      sd = fmaf(gy, ga, sd);
      sdx = fmaf(gy * ga, xh, sdx);
    }
  const float cnt = float(HW * cpg);
  const float m1 = block_sum(sd, red) / cnt;
  const float m2 = block_sum(sdx, red) / cnt;
  if (active)
    for (int64_t p = p0; p < HW; p += step) {
      const int64_t i = base + p * C;
      const float gy = y[i] > 0.f ? dy[i] : 0.f;
      const float xh = (x[i] + (as ? as[p * C] : 0.f) - mean) * rstd;
      dx[i] = rstd * (gy * ga - m1 - xh * m2);
    }
  pg[threadIdx.x] = dg;
  pb[threadIdx.x] = db;
  __syncthreads();
  if (threadIdx.x < cpg) {
    float tg = 0.f, tb = 0.f;
    for (int t = threadIdx.x; t < nt; t += cpg) {
      tg += pg[t];
      tb += pb[t];
    }
    partial[(int64_t(n) * 2) * C + ch] = tg;
    partial[(int64_t(n) * 2 + 1) * C + ch] = tb;
  }
}

// out[r][c] = sum_n in[n][r][c] over n in [0, N) -- affine gradients from the per-sample partials
__global__ void sum_rows_kernel(const float* __restrict__ in, float* __restrict__ out, int N, int64_t inner) {
  const int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= inner) return;
  float t = 0.f;
  for (int n = 0; n < N; ++n) t += in[int64_t(n) * inner + e];
  out[e] = t;
}

// out[b][e] = sum_q in[b * per_image + q][e]: gradient of an operand broadcast over the queries of an image
__global__ void sum_queries_kernel(const float* __restrict__ in, float* __restrict__ out, int per_image,
                                   int64_t inner) {
  const int64_t e = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (e >= inner) return;
  const int b = blockIdx.y;
  const float* src = in + int64_t(b) * per_image * inner + e;
  float t = 0.f;
  for (int q = 0; q < per_image; ++q) t += src[int64_t(q) * inner];
  out[int64_t(b) * inner + e] = t;
}

// ------------------------------------------------------------------------------------------------------------------
// nearest source index of F.interpolate(mode="nearest") (aten/src/ATen/native/UpSample.h nearest_idx)
__device__ __forceinline__ int nearest_src(int o, int in, int out) {
  if (in == out) return o;
  if (out == 2 * in) return o >> 1;
  const float scale = float(in) / float(out);
  return min(int(floorf(float(o) * scale)), in - 1);
}

__global__ void upsample_add_fwd_kernel(const float* __restrict__ x, const float* __restrict__ a,
                                        float* __restrict__ out, int per_image, int Hi, int Wi, int Ho, int Wo, int C,
                                        int64_t total) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = int(i % C);
  int64_t r = i / C;
  const int wo = int(r % Wo);
  r /= Wo;
  const int ho = int(r % Ho);
  const int n = int(r / Ho);
  const int hi = nearest_src(ho, Hi, Ho), wi = nearest_src(wo, Wi, Wo);
  out[i] = a[((int64_t(n / per_image) * Ho + ho) * Wo + wo) * C + c] + x[((int64_t(n) * Hi + hi) * Wi + wi) * C + c];
}

// dx[n][hi][wi][c] = sum of dout over the output pixels whose nearest source is (hi, wi)
__global__ void upsample_add_bwd_dx_kernel(const float* __restrict__ dout, float* __restrict__ dx, int Hi, int Wi,
                                           int Ho, int Wo, int C, int64_t total) {
  const int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (i >= total) return;
  const int c = int(i % C);
  int64_t r = i / C;
  const int wi = int(r % Wi);
  r /= Wi;
  const int hi = int(r % Hi);
  const int n = int(r / Hi);
  const int ho0 = max(0, int(floorf(float(hi) * float(Ho) / float(Hi))) - 2);
  const int wo0 = max(0, int(floorf(float(wi) * float(Wo) / float(Wi))) - 2);
  float t = 0.f;
  for (int ho = ho0; ho < Ho; ++ho) {
    const int sh = nearest_src(ho, Hi, Ho);
    if (sh > hi) break;
    if (sh != hi) continue;
    for (int wo = wo0; wo < Wo; ++wo) {
      const int sw = nearest_src(wo, Wi, Wo);
      if (sw > wi) break;
      if (sw == wi) t += dout[((int64_t(n) * Ho + ho) * Wo + wo) * C + c];
    }
  }
  dx[i] = t;
}

// ------------------------------------------------------------------------------------------------------------------
// loss_masks.  Source coordinate of F.interpolate(mode="bilinear", align_corners=False)
// (aten/src/ATen/native/UpSample.h area_pixel_compute_source_index / compute_source_index_and_lambda)
struct Lerp {
  int i0, i1;
  float l0, l1;
};

__device__ __forceinline__ Lerp bilinear_src(int o, int in, float scale) {
  float s = scale * (float(o) + 0.5f) - 0.5f;
  s = s < 0.f ? 0.f : s;
  Lerp r;
  r.i0 = min(int(s), in - 1);
  r.i1 = r.i0 + (r.i0 < in - 1 ? 1 : 0);
  r.l1 = s - float(r.i0);
  r.l0 = 1.f - r.l1;
  return r;
}

__device__ __forceinline__ float sample_logit(const float* __restrict__ m, int w, const Lerp& ly, const Lerp& lx) {
  return ly.l0 * (lx.l0 * m[ly.i0 * w + lx.i0] + lx.l1 * m[ly.i0 * w + lx.i1]) +
         ly.l1 * (lx.l0 * m[ly.i1 * w + lx.i0] + lx.l1 * m[ly.i1 * w + lx.i1]);
}

struct PixelTerms {
  float focal, p;
};

// sigmoid focal loss of one pixel (util/misc.py:556-563) and its probability
__device__ __forceinline__ PixelTerms focal_pixel(float z, float t, float alpha, float gamma) {
  const float p = 1.f / (1.f + expf(-z));
  const float ce = fmaxf(z, 0.f) - z * t + log1pf(expf(-fabsf(z)));
  const float pt = p * t + (1.f - p) * (1.f - t);
  float l = ce * powf(1.f - pt, gamma);
  if (alpha >= 0.f) l *= alpha * t + (1.f - alpha) * (1.f - t);
  return {l, p};
}

constexpr int kLossChunk = 8192;   // target pixels per CTA of the forward

// partial sums {focal, sum p*t, sum p, sum t} of one chunk of one matched pair; grid (chunks, M)
__global__ void __launch_bounds__(256)
mask_loss_fwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ src,
                     const uint8_t* __restrict__ tmasks, const int64_t* __restrict__ tgt, float* __restrict__ ws, int h,
                     int w, int Ht, int Wt, float alpha, float gamma) {
  __shared__ float red[32];
  const int m = blockIdx.y, chunk = blockIdx.x;
  const float* lm = logits + src[m] * int64_t(h) * w;
  const uint8_t* tm = tmasks + tgt[m] * int64_t(Ht) * Wt;
  const float sy = float(h) / float(Ht), sx = float(w) / float(Wt);
  const int64_t npix = int64_t(Ht) * Wt;
  const int64_t beg = int64_t(chunk) * kLossChunk, end = min(npix, beg + kLossChunk);
  float f = 0.f, pt = 0.f, sp = 0.f, st = 0.f;
  for (int64_t i = beg + threadIdx.x; i < end; i += blockDim.x) {
    const int y = int(i / Wt), x = int(i % Wt);
    const float z = sample_logit(lm, w, bilinear_src(y, h, sy), bilinear_src(x, w, sx));
    const float t = tm[i] ? 1.f : 0.f;
    const PixelTerms r = focal_pixel(z, t, alpha, gamma);
    f += r.focal;
    pt = fmaf(r.p, t, pt);
    sp += r.p;
    st += t;
  }
  f = block_sum(f, red);
  pt = block_sum(pt, red);
  sp = block_sum(sp, red);
  st = block_sum(st, red);
  if (threadIdx.x == 0) {
    float* o = ws + (int64_t(m) * gridDim.x + chunk) * 4;
    o[0] = f; o[1] = pt; o[2] = sp; o[3] = st;
  }
}

// stats[m] = chunk sums in order; out2 = {sum_m focal_m / npix, sum_m dice_m} / num_boxes
__global__ void mask_loss_finish_kernel(const float* __restrict__ ws, float* __restrict__ stats,
                                        const float* __restrict__ num_boxes, float* __restrict__ out2, int M,
                                        int chunks, float npix) {
  __shared__ float red[32];
  float lf = 0.f, ld = 0.f;
  for (int m = threadIdx.x; m < M; m += blockDim.x) {
    float a[4] = {0.f, 0.f, 0.f, 0.f};
    for (int c = 0; c < chunks; ++c)
      for (int j = 0; j < 4; ++j) a[j] += ws[(int64_t(m) * chunks + c) * 4 + j];
    for (int j = 0; j < 4; ++j) stats[m * 4 + j] = a[j];
    lf += a[0] / npix;
    ld += 1.f - (2.f * a[1] + 1.f) / (a[2] + a[3] + 1.f);
  }
  lf = block_sum(lf, red);
  ld = block_sum(ld, red);
  if (threadIdx.x == 0) {
    out2[0] = lf / num_boxes[0];
    out2[1] = ld / num_boxes[0];
  }
}

// gradient of the low-resolution logits: each logit gathers the target pixels whose bilinear footprint contains it
// (no atomics); thread per (pair, low-res pixel), grid (ceil(h * w / 256), M)
__global__ void __launch_bounds__(256)
mask_loss_bwd_kernel(const float* __restrict__ logits, const int64_t* __restrict__ src,
                     const uint8_t* __restrict__ tmasks, const int64_t* __restrict__ tgt,
                     const float* __restrict__ stats, const float* __restrict__ num_boxes, const float* __restrict__ g2,
                     float* __restrict__ grad, int h, int w, int Ht, int Wt, float alpha, float gamma) {
  const int m = blockIdx.y;
  const int e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= h * w) return;
  const int iy = e / w, ix = e % w;
  const float* lm = logits + src[m] * int64_t(h) * w;
  const uint8_t* tm = tmasks + tgt[m] * int64_t(Ht) * Wt;
  const float sy = float(h) / float(Ht), sx = float(w) / float(Wt);
  const float nb = num_boxes[0];
  const float c_focal = g2[0] / (nb * float(int64_t(Ht) * Wt));
  const float I = stats[m * 4 + 1], D = stats[m * 4 + 2] + stats[m * 4 + 3] + 1.f;
  const float c_dice = g2[1] / nb;
  const int y0 = max(0, int(floorf((float(iy - 1) + 0.5f) / sy - 0.5f)) - 2);
  const int x0 = max(0, int(floorf((float(ix - 1) + 0.5f) / sx - 0.5f)) - 2);
  float acc = 0.f;
  for (int y = y0; y < Ht; ++y) {
    const Lerp ly = bilinear_src(y, h, sy);
    if (ly.i0 > iy) break;
    const float wy = (ly.i0 == iy ? ly.l0 : 0.f) + (ly.i1 == iy ? ly.l1 : 0.f);
    if (ly.i0 != iy && ly.i1 != iy) continue;
    for (int x = x0; x < Wt; ++x) {
      const Lerp lx = bilinear_src(x, w, sx);
      if (lx.i0 > ix) break;
      if (lx.i0 != ix && lx.i1 != ix) continue;
      const float wx = (lx.i0 == ix ? lx.l0 : 0.f) + (lx.i1 == ix ? lx.l1 : 0.f);
      const float z = sample_logit(lm, w, ly, lx);
      const float t = tm[int64_t(y) * Wt + x] ? 1.f : 0.f;
      // d focal / dz  (util/misc.py:556-563 differentiated)
      const float p = 1.f / (1.f + expf(-z));
      const float ce = fmaxf(z, 0.f) - z * t + log1pf(expf(-fabsf(z)));
      const float mdl = 1.f - (p * t + (1.f - p) * (1.f - t));
      const float dmdz = -(2.f * t - 1.f) * p * (1.f - p);
      float dfocal = (p - t) * powf(mdl, gamma) + ce * gamma * powf(mdl, gamma - 1.f) * dmdz;
      if (alpha >= 0.f) dfocal *= alpha * t + (1.f - alpha) * (1.f - t);
      // d dice / dz  (util/misc.py:532-537 differentiated)
      const float ddice = -(2.f * t * D - (2.f * I + 1.f)) / (D * D) * p * (1.f - p);
      acc = fmaf(wy * wx, c_focal * dfocal + c_dice * ddice, acc);
    }
  }
  grad[src[m] * int64_t(h) * w + e] = acc;
}

inline unsigned blocks_for(int64_t n, int t) { return unsigned((n + t - 1) / t); }

// the attention kernels move q / k rows and dk rows as float4
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------
extern "C" int tfb200_mask_attn_fwd_f32(const float* q, const float* k, const uint8_t* pad, float* w, int B, int Q,
                                        int HW, int heads, float scale, void* stream) {
  if (!q || !k || !w) return TFB200_E_NULLPTR;
  if (B < 0 || Q < 0 || HW <= 0 || heads <= 0 || !aligned16(q) || !aligned16(k)) return TFB200_E_SHAPE;
  if (int64_t(B) * Q * heads == 0) return 0;
  mask_attn_fwd_kernel<<<unsigned(B * Q * heads), 256, 0, cudaStream_t(stream)>>>(q, k, pad, w, Q, HW, heads, scale);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_mask_attn_bwd_f32(const float* q, const float* k, const float* w, const float* dw, float* ds_ws,
                                        float* dq, float* dk, int B, int Q, int HW, int heads, float scale,
                                        void* stream) {
  if (!q || !k || !w || !dw || !ds_ws || !dq || !dk) return TFB200_E_NULLPTR;
  if (B < 0 || Q < 0 || HW <= 0 || heads <= 0 || !aligned16(k) || !aligned16(dk)) return TFB200_E_SHAPE;
  if (B == 0) return 0;
  const cudaStream_t s = cudaStream_t(stream);
  if (Q == 0) return int(cudaMemsetAsync(dk, 0, sizeof(float) * size_t(B) * HW * heads * kHeadDim, s));
  mask_attn_bwd_dq_kernel<<<unsigned(B * Q * heads), 256, 0, s>>>(k, w, dw, ds_ws, dq, Q, HW, heads, scale);
  mask_attn_bwd_dk_kernel<<<dim3(blocks_for(HW, 128), heads, B), 128, 0, s>>>(q, ds_ws, dk, Q, HW, heads, scale);
  msda_b200_count_launches(2);
  return int(cudaGetLastError());
}

static int gn_check(int N, int per_image, int64_t HW, int C, int groups) {
  if (N < 0 || per_image <= 0 || HW <= 0 || C <= 0 || groups <= 0 || C % groups != 0 || C / groups > 256 ||
      N % per_image != 0)
    return TFB200_E_SHAPE;
  return 0;
}

extern "C" int tfb200_group_norm_relu_fwd_f32(const float* x, const float* addend, const float* gamma,
                                              const float* beta, float* y, float* mean, float* rstd, int N,
                                              int per_image, int64_t HW, int C, int groups, float eps, void* stream) {
  if (!x || !gamma || !beta || !y || !mean || !rstd) return TFB200_E_NULLPTR;
  if (const int rc = gn_check(N, per_image, HW, C, groups)) return rc;
  if (N == 0) return 0;
  group_norm_relu_fwd_kernel<<<unsigned(N * groups), 256, 0, cudaStream_t(stream)>>>(
      x, addend, gamma, beta, y, mean, rstd, per_image, HW, C, groups, eps);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_group_norm_relu_bwd_f32(const float* dy, const float* x, const float* addend, const float* y,
                                              const float* gamma, const float* mean, const float* rstd, float* dx,
                                              float* daddend, float* daffine, float* partial_ws, int N,
                                              int per_image, int64_t HW, int C, int groups, void* stream) {
  if (!dy || !x || !y || !gamma || !mean || !rstd || !dx || !daffine || !partial_ws) return TFB200_E_NULLPTR;
  if (addend != nullptr && daddend == nullptr) return TFB200_E_NULLPTR;
  if (const int rc = gn_check(N, per_image, HW, C, groups)) return rc;
  const cudaStream_t s = cudaStream_t(stream);
  if (N == 0) return int(cudaMemsetAsync(daffine, 0, 2 * sizeof(float) * C, s));
  group_norm_relu_bwd_kernel<<<unsigned(N * groups), 256, 0, s>>>(dy, x, addend, y, gamma, mean, rstd, dx, partial_ws,
                                                                   per_image, HW, C, groups);
  // partial_ws is [N][2][C]: daffine = {dgamma, dbeta} is its sum over the samples
  sum_rows_kernel<<<blocks_for(2 * C, 256), 256, 0, s>>>(partial_ws, daffine, N, int64_t(2 * C));
  int launches = 2;
  if (addend != nullptr) {
    const int64_t inner = HW * C;
    sum_queries_kernel<<<dim3(blocks_for(inner, 256), N / per_image), 256, 0, s>>>(dx, daddend, per_image, inner);
    ++launches;
  }
  msda_b200_count_launches(launches);
  return int(cudaGetLastError());
}

extern "C" int tfb200_upsample_add_fwd_f32(const float* x, const float* a, float* out, int N, int per_image, int Hi,
                                           int Wi, int Ho, int Wo, int C, void* stream) {
  if (!x || !a || !out) return TFB200_E_NULLPTR;
  if (N < 0 || per_image <= 0 || N % per_image != 0 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0 || C <= 0)
    return TFB200_E_SHAPE;
  const int64_t total = int64_t(N) * Ho * Wo * C;
  if (total == 0) return 0;
  upsample_add_fwd_kernel<<<blocks_for(total, 256), 256, 0, cudaStream_t(stream)>>>(x, a, out, per_image, Hi, Wi, Ho,
                                                                                     Wo, C, total);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_upsample_add_bwd_f32(const float* dout, float* dx, float* da, int N, int per_image, int Hi,
                                           int Wi, int Ho, int Wo, int C, void* stream) {
  if (!dout || !dx || !da) return TFB200_E_NULLPTR;
  if (N < 0 || per_image <= 0 || N % per_image != 0 || Hi <= 0 || Wi <= 0 || Ho <= 0 || Wo <= 0 || C <= 0)
    return TFB200_E_SHAPE;
  if (N == 0) return 0;
  const cudaStream_t s = cudaStream_t(stream);
  const int64_t total = int64_t(N) * Hi * Wi * C, inner = int64_t(Ho) * Wo * C;
  upsample_add_bwd_dx_kernel<<<blocks_for(total, 256), 256, 0, s>>>(dout, dx, Hi, Wi, Ho, Wo, C, total);
  sum_queries_kernel<<<dim3(blocks_for(inner, 256), N / per_image), 256, 0, s>>>(dout, da, per_image, inner);
  msda_b200_count_launches(2);
  return int(cudaGetLastError());
}

extern "C" int tfb200_mask_loss_partial_chunks(int Ht, int Wt) {
  return int((int64_t(Ht) * Wt + kLossChunk - 1) / kLossChunk);
}

extern "C" int tfb200_mask_loss_fwd_f32(const float* logits, const int64_t* src, const uint8_t* tgt_masks,
                                        const int64_t* tgt, const float* num_boxes, float* stats, float* partial_ws,
                                        float* out2, int M, int h, int w, int Ht, int Wt, float alpha, float gamma,
                                        void* stream) {
  if (!logits || !tgt_masks || !num_boxes || !out2 || (M > 0 && (!src || !tgt || !stats || !partial_ws)))
    return TFB200_E_NULLPTR;
  if (M < 0 || h <= 0 || w <= 0 || Ht <= 0 || Wt <= 0) return TFB200_E_SHAPE;
  const cudaStream_t s = cudaStream_t(stream);
  if (M == 0) return int(cudaMemsetAsync(out2, 0, 2 * sizeof(float), s));   // no matches: zero loss
  const int chunks = tfb200_mask_loss_partial_chunks(Ht, Wt);
  mask_loss_fwd_kernel<<<dim3(chunks, M), 256, 0, s>>>(logits, src, tgt_masks, tgt, partial_ws, h, w, Ht, Wt, alpha,
                                                        gamma);
  mask_loss_finish_kernel<<<1, 256, 0, s>>>(partial_ws, stats, num_boxes, out2, M, chunks, float(int64_t(Ht) * Wt));
  msda_b200_count_launches(2);
  return int(cudaGetLastError());
}

extern "C" int tfb200_mask_loss_bwd_f32(const float* logits, const int64_t* src, const uint8_t* tgt_masks,
                                        const int64_t* tgt, const float* stats, const float* num_boxes, const float* g2,
                                        float* grad_logits, int R, int M, int h, int w, int Ht, int Wt, float alpha,
                                        float gamma, void* stream) {
  if (!logits || !tgt_masks || !num_boxes || !g2 || !grad_logits || (M > 0 && (!src || !tgt || !stats)))
    return TFB200_E_NULLPTR;
  if (R < 0 || M < 0 || h <= 0 || w <= 0 || Ht <= 0 || Wt <= 0) return TFB200_E_SHAPE;
  const cudaStream_t s = cudaStream_t(stream);
  const cudaError_t e = cudaMemsetAsync(grad_logits, 0, sizeof(float) * size_t(R) * h * w, s);
  if (e != cudaSuccess || M == 0) return int(e);
  mask_loss_bwd_kernel<<<dim3(blocks_for(int64_t(h) * w, 256), M), 256, 0, s>>>(
      logits, src, tgt_masks, tgt, stats, num_boxes, g2, grad_logits, h, w, Ht, Wt, alpha, gamma);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}
