// Kernels specialised for the shipped geometry: fp32, D = 32 channels per head (one head row of
// `value` = 128 bytes = exactly one L1/L2 line), any M / L / P with L*P <= kMaxLP.
//
// What bounds these kernels: every bilinear corner is a 128-byte row that has to
// cross the SM's L1 data stage -- 4 wavefronts per warp-level LDG.128 -- so a C2 encoder call moves
// 1.46 GB through L1 although only 80 MB are compulsory HBM traffic.  The design therefore minimises
// every OTHER wavefront and instruction around those loads:
//
//  * a CTA owns 32 consecutive (n,q,m) groups per iteration; a cooperative prologue turns each of their
//    L*P samples into a "tap" exactly once (8 lanes of a group would otherwise redo the same
//    floor/compare/weight arithmetic) and parks it in shared memory;
//  * tap tables are pitched (odd pitch) so that the 4 groups of a warp hit 4 distinct bank groups:
//    one LDS.128 + one LDS.32 per sample = 2 wavefronts, conflict-free;
//  * "shifted window": instead of predicating dead corners, the 2x2 window is moved inside the image
//    ([xb, xb+1] x [yb, yb+1] with xb = clamp(x0, 0, W-2)) and the weights are permuted/zeroed to match,
//    so all four loads are unconditional and in-bounds, corner 2/4 are immediate offsets of corner 1/3,
//    and fully dead samples degenerate to four zero weights.  (Levels with H < 2 or W < 2 take an
//    on-the-fly predicated path.)  For finite inputs the result equals the reference's zero-padding
//    rule exactly; a non-finite value next to the border can turn into NaN where the reference gives inf.
//  * a CTA walks a contiguous strip of groups (`iters` iterations) so that consecutive iterations --
//    neighbouring queries, whose samples overlap -- reuse each other's lines in L1.
#pragma once

#include "msda_common.cuh"

namespace msda {

constexpr int kMaxLP = 64;          // L*P supported by the staged kernels (C5 decoder: 8*4 = 32)
constexpr int kGroupsPerCta = 32;   // 256 threads / 8 lanes
constexpr int kD32Threads = 256;

struct LevelTable {
  int H[MSDA_B200_MAX_LEVELS];
  int W[MSDA_B200_MAX_LEVELS];
  int start[MSDA_B200_MAX_LEVELS];   // first pixel of the level inside one sample's slab
};

__host__ __device__ inline int tap_pitch(int LP) { return LP | 1; }

__host__ __device__ inline size_t fwd_d32_smem_bytes(int LP) {
  return size_t(kGroupsPerCta) * tap_pitch(LP) * (16 + 4);          // float4 weights + int offset
}
__host__ __device__ inline size_t bwd_d32_smem_bytes(int LP) {
  return size_t(kGroupsPerCta) * tap_pitch(LP) * (16 + 16 + 8);     // col/row weights, derivatives, (a, offset)
}

__device__ __forceinline__ void load_level_table(LevelTable& t, unsigned char* lvl_of,
                                                 const int64_t* __restrict__ shapes, int L, int P) {
  if (threadIdx.x == 0) {
    int acc = 0;
    for (int l = 0; l < L; ++l) {
      const int h = int(__ldg(shapes + 2 * l)), w = int(__ldg(shapes + 2 * l + 1));
      t.H[l] = h;
      t.W[l] = w;
      t.start[l] = acc;
      acc += h * w;
    }
  }
  if (int(threadIdx.x) < L * P) lvl_of[threadIdx.x] = (unsigned char)(threadIdx.x / P);
}

// One axis of the shifted window.  Returns the window base b in [0, size-2] and the weights (wa, wb) of
// columns b and b+1 that reproduce the reference's zero-padded interpolation at coordinate t in (-1, size);
// (da, db) are d(wa)/dt, d(wb)/dt.  Requires size >= 2.
__device__ __forceinline__ void axis_window(float t, int size, int& b, float& wa, float& wb, float& da,
                                            float& db) {
  const float f = floorf(t);
  const int t0 = int(f);
  const float frac = t - f;
  b = min(max(t0, 0), size - 2);
  if (t0 == b) {            // both taps inside
    wa = 1.f - frac; wb = frac; da = -1.f; db = 1.f;
  } else if (t0 < b) {      // t0 = -1: only the upper tap (pixel 0 = b) is inside
    wa = frac; wb = 0.f; da = 1.f; db = 0.f;
  } else {                  // t0 = size-1: only the lower tap (pixel size-1 = b+1) is inside
    wa = 0.f; wb = 1.f - frac; da = 0.f; db = -1.f;
  }
}

// Which of the CTA's 32 consecutive (q, m) groups the 8-lane group `gl` (= tid/8) works on.
// With M = 8 heads (STRIDE_CT = 256) a CTA covers 4 queries x 8 heads; mapping warp w -> head w and the
// warp's four 8-lane groups -> the four queries makes the 4 rows touched by one warp-level LDG/RED belong to
// NEIGHBOURING QUERIES OF ONE HEAD.  On the coarser levels neighbouring queries sample the same pixels, so
// the LSU sees 1-2 distinct 128-byte lines per request instead of 4 (an L1 request costs ~2 cycles per
// distinct line).  Other head counts keep memory order.
template <int STRIDE_CT>
__device__ __forceinline__ int group_slot(int gl) {
  return STRIDE_CT == 256 ? ((gl & 3) * 8 + (gl >> 2)) : gl;
}

__device__ __forceinline__ float4 ldg4(const float* p) { return __ldg(reinterpret_cast<const float4*>(p)); }

__device__ __forceinline__ void fma4(float4& acc, float w, const float4& v) {
  acc.x = fmaf(w, v.x, acc.x);
  acc.y = fmaf(w, v.y, acc.y);
  acc.z = fmaf(w, v.z, acc.z);
  acc.w = fmaf(w, v.w, acc.w);
}

// ------------------------------------------------------------------------------------------------
// Forward
// ------------------------------------------------------------------------------------------------
// STRIDE_CT: M*D in elements when known at compile time (256 for the shipped M = 8), else 0.
template <int STRIDE_CT, int UNROLL = 4, int MINB = 1>
__global__ void __launch_bounds__(kD32Threads, MINB)
msda_fwd_d32_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                    const float* __restrict__ loc, const float* __restrict__ attn,
                    float* __restrict__ out, int S, int M, int L, int Lq, int P, uint32_t groups, int iters) {
  constexpr int D = 32;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ LevelTable lv;
  __shared__ unsigned char lvl_of[kMaxLP];

  const int LP = L * P;
  const int pitch = tap_pitch(LP);
  float4* s_w = reinterpret_cast<float4*>(smem_raw);                    // [32][pitch] corner weights * attn
  int* s_o = reinterpret_cast<int*>(s_w + kGroupsPerCta * pitch);        // [32][pitch] element offset of corner 1
  const int stride = STRIDE_CT ? STRIDE_CT : M * D;
  const int tid = threadIdx.x;
  const int gl = tid >> 3;      // tap-table row of this thread's group (4 consecutive rows per warp)
  const int gm = group_slot<STRIDE_CT>(gl);   // which of the CTA's 32 consecutive groups that is
  const int j = tid & 7;        // 16-byte pack inside the head row / tap column inside the prologue

  load_level_table(lv, lvl_of, shapes, L, P);
  __syncthreads();

  for (int it = 0; it < iters; ++it) {
    const uint32_t g0 = (uint32_t(blockIdx.x) * iters + it) * kGroupsPerCta;
    if (g0 >= groups) break;                                    // uniform
    const bool active = g0 + gm < groups;
    const uint32_t gid = active ? g0 + gm : groups - 1;

    // ---- prologue: every lane builds taps j, j+8, ... of its own group (rows are read coalesced)
    {
      const float2* gxy = reinterpret_cast<const float2*>(loc) + size_t(gid) * LP;
      const float* ga = attn + size_t(gid) * LP;
      for (int s = j; s < LP; s += 8) {
        const float2 xy = __ldg(gxy + s);
        const float a = __ldg(ga + s);
        const int l = lvl_of[s];
        const int H = lv.H[l], W = lv.W[l];
        float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
        int o = lv.start[l] * stride;                           // dead sample: pixel (0,0), zero weights
        if (H >= 2 && W >= 2) {
          const float x = xy.x * float(W) - 0.5f, y = xy.y * float(H) - 0.5f;
          if (y > -1.f && x > -1.f && y < float(H) && x < float(W)) {
            int xb, yb;
            float wxa, wxb, wya, wyb, d0, d1;
            axis_window(x, W, xb, wxa, wxb, d0, d1);
            axis_window(y, H, yb, wya, wyb, d0, d1);
            w = make_float4(wya * wxa * a, wya * wxb * a, wyb * wxa * a, wyb * wxb * a);
            o += (yb * W + xb) * stride;
          }
        }
        s_w[gl * pitch + s] = w;
        s_o[gl * pitch + s] = o;
      }
    }
    __syncthreads();

    if (active) {
      const uint32_t m = gid % uint32_t(M);
      const uint32_t n = gid / (uint32_t(M) * uint32_t(Lq));
      const float* vb = value + size_t(n) * S * stride + m * D + j * 4;
      const float4* rw = s_w + gl * pitch;
      const int* ro = s_o + gl * pitch;
      float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int l = 0; l < L; ++l) {
        const int H = lv.H[l], W = lv.W[l];
        if (H >= 2 && W >= 2) {
          const int rowpitch = W * stride;
#pragma unroll UNROLL
          for (int p = 0; p < P; ++p) {
            const int s = l * P + p;
            const float4 w = rw[s];
            const float* c1 = vb + ro[s];
            const float* c3 = c1 + rowpitch;
            const float4 v1 = ldg4(c1), v2 = ldg4(c1 + stride), v3 = ldg4(c3), v4 = ldg4(c3 + stride);
            fma4(acc, w.x, v1);
            fma4(acc, w.y, v2);
            fma4(acc, w.z, v3);
            fma4(acc, w.w, v4);
          }
        } else {
          // degenerate level (a single row or column): predicated taps computed on the fly
          const float* vl = vb + size_t(lv.start[l]) * stride;
          for (int p = 0; p < P; ++p) {
            const size_t sidx = size_t(gid) * LP + l * P + p;
            const Tap<float> t = make_tap<float>(__ldg(loc + 2 * sidx), __ldg(loc + 2 * sidx + 1), H, W, stride);
            if (!t.live) continue;
            const float a = __ldg(attn + sidx);
            const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
            fma4(acc, t.w1 * a, t.k1 ? ldg4(vl + t.o1) : z);
            fma4(acc, t.w2 * a, t.k2 ? ldg4(vl + t.o2) : z);
            fma4(acc, t.w3 * a, t.k3 ? ldg4(vl + t.o3) : z);
            fma4(acc, t.w4 * a, t.k4 ? ldg4(vl + t.o4) : z);
          }
        }
      }
      *reinterpret_cast<float4*>(out + size_t(gid) * D + j * 4) = acc;
    }
    __syncthreads();    // taps are rebuilt by the next iteration
  }
}

// ------------------------------------------------------------------------------------------------
// Backward (fused): grad_value (128-bit vector reductions), grad_sampling_loc, grad_attn_weight
// ------------------------------------------------------------------------------------------------
__device__ __forceinline__ float dot4(const float4& a, const float4& b) {
  return fmaf(a.x, b.x, fmaf(a.y, b.y, fmaf(a.z, b.z, a.w * b.w)));
}
__device__ __forceinline__ float4 lin2(float ca, const float4& a, float cb, const float4& b) {
  return make_float4(fmaf(ca, a.x, cb * b.x), fmaf(ca, a.y, cb * b.y), fmaf(ca, a.z, cb * b.z),
                     fmaf(ca, a.w, cb * b.w));
}
__device__ __forceinline__ void red4(float* p, float c, const float4& g) {
  Pack<float, 4> r;
  r.v[0] = c * g.x; r.v[1] = c * g.y; r.v[2] = c * g.z; r.v[3] = c * g.w;
  red_add_pack<float, 4>(p, r);
}

template <int STRIDE_CT, int MINB = 4>
__global__ void __launch_bounds__(kD32Threads, MINB)
msda_bwd_d32_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                    const float* __restrict__ loc, const float* __restrict__ attn,
                    const float* __restrict__ grad_out, float* __restrict__ grad_value,
                    float* __restrict__ grad_loc, float* __restrict__ grad_attn,
                    int S, int M, int L, int Lq, int P, uint32_t groups, int iters) {
  constexpr int D = 32;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ LevelTable lv;
  __shared__ unsigned char lvl_of[kMaxLP];

  const int LP = L * P;
  const int pitch = tap_pitch(LP);
  float4* s_w = reinterpret_cast<float4*>(smem_raw);                    // (wxa, wxb, wya, wyb)
  float4* s_d = s_w + kGroupsPerCta * pitch;                            // (dxa, dxb, dya, dyb)
  float2* s_ao = reinterpret_cast<float2*>(s_d + kGroupsPerCta * pitch); // (attn, int offset as bits)
  const int stride = STRIDE_CT ? STRIDE_CT : M * D;
  const int tid = threadIdx.x;
  const int gl = tid >> 3;
  const int gm = group_slot<STRIDE_CT>(gl);
  const int j = tid & 7;

  load_level_table(lv, lvl_of, shapes, L, P);
  __syncthreads();

  for (int it = 0; it < iters; ++it) {
    const uint32_t g0 = (uint32_t(blockIdx.x) * iters + it) * kGroupsPerCta;
    if (g0 >= groups) break;
    const bool active = g0 + gm < groups;
    const uint32_t gid = active ? g0 + gm : groups - 1;
    const size_t sbase = size_t(gid) * LP;

    {
      const float2* gxy = reinterpret_cast<const float2*>(loc) + sbase;
      const float* ga = attn + sbase;
      for (int s = j; s < LP; s += 8) {
        const float2 xy = __ldg(gxy + s);
        const float a = __ldg(ga + s);
        const int l = lvl_of[s];
        const int H = lv.H[l], W = lv.W[l];
        float4 w = make_float4(0.f, 0.f, 0.f, 0.f), d = w;
        int o = lv.start[l] * stride;
        if (H >= 2 && W >= 2) {
          const float x = xy.x * float(W) - 0.5f, y = xy.y * float(H) - 0.5f;
          if (y > -1.f && x > -1.f && y < float(H) && x < float(W)) {
            int xb, yb;
            axis_window(x, W, xb, w.x, w.y, d.x, d.y);
            axis_window(y, H, yb, w.z, w.w, d.z, d.w);
            o += (yb * W + xb) * stride;
          }
        }
        s_w[gl * pitch + s] = w;
        s_d[gl * pitch + s] = d;
        s_ao[gl * pitch + s] = make_float2(a, __int_as_float(o));
      }
    }
    __syncthreads();

    // NB: no early-out for inactive groups -- the warp shuffles below need all 32 lanes; their loads hit
    // the clamped last group and their stores / reductions are masked by `active`.
    {
      const uint32_t m = gid % uint32_t(M);
      const uint32_t n = gid / (uint32_t(M) * uint32_t(Lq));
      const size_t head = size_t(n) * S * stride + m * D + j * 4;
      const float* vb = value + head;
      float* gvb = grad_value + head;
      const float4 g = active ? ldg4(grad_out + size_t(gid) * D + j * 4) : make_float4(0.f, 0.f, 0.f, 0.f);
      const float4* rw = s_w + gl * pitch;
      const float4* rd = s_d + gl * pitch;
      const float2* rao = s_ao + gl * pitch;

      for (int l = 0; l < L; ++l) {
        const int H = lv.H[l], W = lv.W[l];
        const bool fast = (H >= 2 && W >= 2);
        const int rowpitch = W * stride;
        for (int p0 = 0; p0 < P; p0 += 4) {
          // up to 4 samples per round: 12 partial sums (attn, x, y) x 4 reduced over the 8 lanes with a
          // transposing butterfly (12 shuffles instead of 36)
          float part[12];
#pragma unroll
          for (int u = 0; u < 4; ++u) {
            float s_a = 0.f, s_x = 0.f, s_y = 0.f;
            const int p = p0 + u;
            if (p < P) {
              const int s = l * P + p;
              if (fast) {
                const float4 w = rw[s];
                const float4 d = rd[s];
                const float2 ao = rao[s];
                const int o = __float_as_int(ao.y);
                const float* c1 = vb + o;
                const float* c3 = c1 + rowpitch;
                const float4 v1 = ldg4(c1), v2 = ldg4(c1 + stride), v3 = ldg4(c3), v4 = ldg4(c3 + stride);
                const float4 top = lin2(w.x, v1, w.y, v2), bot = lin2(w.x, v3, w.y, v4);   // row interpolants
                const float4 dtop = lin2(d.x, v1, d.y, v2), dbot = lin2(d.x, v3, d.y, v4); // d/dx of them
                s_a = dot4(g, lin2(w.z, top, w.w, bot));
                s_x = dot4(g, lin2(w.z, dtop, w.w, dbot)) * ao.x * float(W);
                s_y = dot4(g, lin2(d.z, top, d.w, bot)) * ao.x * float(H);
                if (active) {
                  // zero coefficients (dead samples, window corners outside the image, masked attention)
                  // are skipped: they would only hammer one L2 line with +0
                  float* q1 = gvb + o;
                  float* q3 = q1 + rowpitch;
                  const float ra = w.z * ao.x, rb = w.w * ao.x;
                  const float k1 = ra * w.x, k2 = ra * w.y, k3 = rb * w.x, k4 = rb * w.y;
                  if (k1 != 0.f) red4(q1, k1, g);
                  if (k2 != 0.f) red4(q1 + stride, k2, g);
                  if (k3 != 0.f) red4(q3, k3, g);
                  if (k4 != 0.f) red4(q3 + stride, k4, g);
                }
              } else {
                // degenerate level: predicated taps on the fly (reference formulas, .cuh:96-163)
                const size_t sidx = sbase + s;
                const float a = __ldg(attn + sidx);
                const Tap<float> t = make_tap<float>(__ldg(loc + 2 * sidx), __ldg(loc + 2 * sidx + 1), H, W, stride);
                if (t.live) {
                  const size_t lofs = size_t(lv.start[l]) * stride;
                  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
                  const float4 v1 = t.k1 ? ldg4(vb + lofs + t.o1) : z, v2 = t.k2 ? ldg4(vb + lofs + t.o2) : z;
                  const float4 v3 = t.k3 ? ldg4(vb + lofs + t.o3) : z, v4 = t.k4 ? ldg4(vb + lofs + t.o4) : z;
                  const float hx = 1.f - t.lx, hy = 1.f - t.ly;
                  const float4 top = lin2(hx, v1, t.lx, v2), bot = lin2(hx, v3, t.lx, v4);
                  const float4 dtop = lin2(-1.f, v1, 1.f, v2), dbot = lin2(-1.f, v3, 1.f, v4);
                  s_a = dot4(g, lin2(hy, top, t.ly, bot));
                  s_x = dot4(g, lin2(hy, dtop, t.ly, dbot)) * a * float(W);
                  s_y = dot4(g, lin2(-1.f, top, 1.f, bot)) * a * float(H);
                  if (active) {
                    if (t.k1) red4(gvb + lofs + t.o1, t.w1 * a, g);
                    if (t.k2) red4(gvb + lofs + t.o2, t.w2 * a, g);
                    if (t.k3) red4(gvb + lofs + t.o3, t.w3 * a, g);
                    if (t.k4) red4(gvb + lofs + t.o4, t.w4 * a, g);
                  }
                }
              }
            }
            part[3 * u + 0] = s_a;
            part[3 * u + 1] = s_x;
            part[3 * u + 2] = s_y;
          }
          // butterfly: after the three steps lane j holds the full sums of sample u = j >> 1
          float r6[6], r3[3];
          {
            const bool hi = j & 4;
#pragma unroll
            for (int k = 0; k < 6; ++k) {
              const float mine = hi ? part[6 + k] : part[k];
              const float give = hi ? part[k] : part[6 + k];
              r6[k] = mine + __shfl_xor_sync(0xffffffffu, give, 4);
            }
          }
          {
            const bool hi = j & 2;
#pragma unroll
            for (int k = 0; k < 3; ++k) {
              const float mine = hi ? r6[3 + k] : r6[k];
              const float give = hi ? r6[k] : r6[3 + k];
              r3[k] = mine + __shfl_xor_sync(0xffffffffu, give, 2);
            }
          }
#pragma unroll
          for (int k = 0; k < 3; ++k) r3[k] += __shfl_xor_sync(0xffffffffu, r3[k], 1);
          const int p = p0 + (j >> 1);
          if (active && !(j & 1) && p < P) {
            const size_t sidx = sbase + l * P + p;
            grad_attn[sidx] = r3[0];
            *reinterpret_cast<float2*>(grad_loc + 2 * sidx) = make_float2(r3[1], r3[2]);
          }
        }
      }
    }
    __syncthreads();
  }
}

}  // namespace msda
