// Backward of the encoder self-attention with TMA-staged value tiles (fp32, D = 32, P = 4, L <= 4): grad_value,
// grad_sampling_loc and grad_attn_weight in one pass.  Companion of msda_enc_tma.cuh (same tiles, same box staging,
// same plan pass); reference semantics: ms_deform_im2col_cuda.cuh:85-163 (ms_deform_attn_col2im_bilinear) and
// :239-378 (the backward kernels) -- identical formulas, different data movement.
//
// What the measurements say about the direct backward (msda_bwd_d32_kernel, 245 us per C2 encoder call): it reads the
// same 11.4 M corner rows as the forward through L1 AND sends one 128-bit vector reduction per corner row to L2 (another
// 1.46 GB; ~3.7 SM-cycles per row).  Here
//   * the corner rows come out of the staged box (LDS.128, ~0.3 rows per corner thanks to the register-resident window),
//   * the grad_value contributions of a window column are ACCUMULATED IN REGISTERS while the window stays (same window:
//     nothing leaves the SM; slid by one: one column = 2 reductions) and only flushed to L2 when the register set is
//     reloaded -- the reductions shrink by the same ~0.3x as the loads;
//   * grad_attn / grad_loc partial sums are reduced over the 8 lanes of a group with the transposing butterfly of
//     msda_run.cuh (12 shuffles per 4 steps), parked in the consumed tap entries and streamed out coalesced at the end.
// Taps whose window is outside the staged box and taps on levels finer than the tile's own take the paths described in
// msda_enc_tma.cuh (global-memory run walk / per-sample evaluation); values are the same either way.
#pragma once

#include "msda_enc_tma.cuh"

namespace msda {

constexpr int kEbHaloX = 6, kEbHaloY = 7;                     // one column narrower than the forward: 24-byte tap entries
__host__ __device__ constexpr int eb_bw(int d) { return (kEtTX >> d) + kEbHaloX; }
__host__ __device__ constexpr int eb_bh(int d) { return (kEtTY >> d) + kEbHaloY; }
constexpr int kEbBuf0Rows = eb_bw(0) * eb_bh(0);              // 330
constexpr int kEbBuf1Rows = eb_bw(1) * eb_bh(1);              // 154
constexpr size_t kEbSmemBytes = 128 + size_t(kEbBuf0Rows + kEbBuf1Rows) * 128 + size_t(kEtEntries) * (16 + 4 + 4) +
                                kEtQ * 4 + 2 * kEtMaxL * 4 + kEtMaxL * 8;
constexpr int kEbThreads = 256;

// derivative sign codes: 0 -> 0, 1 -> +1, 2 -> -1
__device__ __forceinline__ unsigned eb_enc(float d) { return d > 0.f ? 1u : (d < 0.f ? 2u : 0u); }
__device__ __forceinline__ float eb_dec(unsigned c) { return (c & 1u) ? 1.f : ((c & 2u) ? -1.f : 0.f); }
// all four signs of a tap at once: one indexed 128-bit constant load instead of ~20 select instructions per step
struct EbSigns { float4 v[256]; };
__host__ __device__ constexpr float eb_dec_c(unsigned c) { return (c & 1u) ? 1.f : ((c & 2u) ? -1.f : 0.f); }
__constant__ EbSigns kEbSigns;
inline void eb_fill_signs(EbSigns* t) {
  for (unsigned c = 0; c < 256; ++c)
    t->v[c] = make_float4(eb_dec_c(c), eb_dec_c(c >> 2), eb_dec_c(c >> 4), eb_dec_c(c >> 6));
}

// two-lane fp32 helpers on 64-bit register pairs: sm_90 has no packed fp32 arithmetic, so each lane is one IEEE op
__device__ __forceinline__ float2 unpk2(u64 a) {
  float2 r;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(a));
  return r;
}
__device__ __forceinline__ u64 pk2(float x, float y) {
  u64 d;
  asm("mov.b64 %0, {%1, %2};" : "=l"(d) : "f"(x), "f"(y));
  return d;
}
__device__ __forceinline__ u64 fmul2(u64 a, u64 b) {
  const float2 x = unpk2(a), y = unpk2(b);
  return pk2(__fmul_rn(x.x, y.x), __fmul_rn(x.y, y.y));
}
__device__ __forceinline__ u64 ffma2v(u64 a, u64 b, u64 c) {
  const float2 x = unpk2(a), y = unpk2(b), z = unpk2(c);
  return pk2(__fmaf_rn(x.x, y.x, z.x), __fmaf_rn(x.y, y.y, z.y));
}
__device__ __forceinline__ float hsum2(u64 v) {
  float a, b;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(a), "=f"(b) : "l"(v));
  return a + b;
}
// g . v for 16-byte packs held as two f32x2 registers
__device__ __forceinline__ float dot2(const u64 (&g)[2], const u64 (&v)[2]) { return hsum2(ffma2v(g[1], v[1], fmul2(g[0], v[0]))); }
__device__ __forceinline__ void red2(float* p, const u64 (&v)[2]) {
  asm volatile(
      "{\n\t.reg .f32 a, b, c, d;\n\tmov.b64 {a, b}, %1;\n\tmov.b64 {c, d}, %2;\n\t"
      "red.relaxed.gpu.global.add.v4.f32 [%0], {a, b, c, d};\n\t}" ::"l"(p), "l"(v[0]), "l"(v[1])
      : "memory");
}

// predicated helpers (straight-line code: the flush / reset decisions are per 8-lane group, branches would diverge)
__device__ __forceinline__ void red2_if(const float* p, const u64 (&v)[2], bool pred) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t.reg .f32 a, b, c, d;\n\tsetp.ne.b32 p, %3, 0;\n\tmov.b64 {a, b}, %1;\n\tmov.b64 {c, d}, %2;\n\t"
      "@p red.relaxed.gpu.global.add.v4.f32 [%0], {a, b, c, d};\n\t}" ::"l"(p), "l"(v[0]), "l"(v[1]), "r"(int(pred))
      : "memory");
}
// acc = acc * keep + k * g  (keep = 0 right after the set was flushed, else 1; both lanes of the f32x2).  Arithmetic
// instead of a select: ptxas turns a predicated mul / fma pair into both products plus two SELs per register pair.
__device__ __forceinline__ void acc2(u64& acc, float k, u64 g, float keep) {
  const float2 a = unpk2(acc), v = unpk2(g);
  acc = pk2(__fmaf_rn(a.x, keep, __fmul_rn(k, v.x)), __fmaf_rn(a.y, keep, __fmul_rn(k, v.y)));
}

// One sample slot of one level for one warp: the run of R queries, forward values + all three gradients.
//   staged (GLOBAL = false): s_o = rowA | rowB << 9 | codes << 18 (0x1FF = keep the set)
//   global (GLOBAL = true) : s_o = pixel of the NEW right column | load A << 20 | load B << 21 | reload << 22 | codes << 23
// First version: 190 SASS instructions per step (ncu: 164 M per C2 call, issue bound) -- 25 of them re-deriving the
// grad_output address from the thread index every step (rematerialised under the 128-register cap), ~50 in the two
// divergent flush branches with their register copies, 16 in 64-bit reduction addresses.  Now: the grad_output pointer is
// an opaque register pair that only gets incremented, flush / reset are predicated instructions, addresses are 32-bit
// offsets + one mad.wide each.
template <bool GLOBAL>
__device__ __forceinline__ void eb_slot_pass(uint32_t sw_addr, uint32_t sa_addr, uint32_t so_addr, uint32_t slot, float4* s_w_e0,
                                             uint32_t bufa, uint32_t pitch, int BW, unsigned gbox, const float* vh, float* gvh,
                                             unsigned gstride, unsigned rowpitch, float fW, float fH, const float* gout0,
                                             int gq_stride, unsigned valid_mask, int lane, int k, int j) {
  constexpr int R = kEtR;
  u64 A1[2] = {0ull, 0ull}, A3[2] = {0ull, 0ull}, B1[2] = {0ull, 0ull}, B3[2] = {0ull, 0ull};     // window columns (top, bottom)
  u64 GA1[2] = {0ull, 0ull}, GA3[2] = {0ull, 0ull}, GB1[2] = {0ull, 0ull}, GB3[2] = {0ull, 0ull}; // pending grad_value
  unsigned gA = 0u, gB = 0u;                                     // element offsets of the rows the pending sums belong to
  int nzA = 0, nzB = 0;                                          // OR of the coefficient bits seen since the last flush
  const unsigned magic = (65536u + unsigned(BW) - 1u) / unsigned(BW);
  // box row (y * BW + x) -> element offset of that pixel in the head's value / grad_value plane
  auto to_global = [&](unsigned h) -> unsigned {
    const unsigned ry = (h * magic) >> 16, rx = h - ry * unsigned(BW);
    return gbox + ry * rowpitch + rx * gstride;
  };
  const float* gp = gout0;
  asm volatile("" : "+l"(gp));                                   // opaque: keep the pointer, do not rematerialise it
  const size_t gstep = size_t(gq_stride) * 4;

  float4 wn;
  float an;
  unsigned on;
  u64 gn[2];
  auto fetch = [&](int r) {
    const uint32_t eo = uint32_t(r * kEtLP) + slot;
    asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(wn.x), "=f"(wn.y), "=f"(wn.z), "=f"(wn.w) : "r"(sw_addr + eo * 16u));
    asm volatile("ld.shared.f32 %0, [%1];" : "=f"(an) : "r"(sa_addr + eo * 4u));
    asm volatile("ld.shared.b32 %0, [%1];" : "=r"(on) : "r"(so_addr + eo * 4u));
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\tmov.b64 %0, 0;\n\tmov.b64 %1, 0;\n\t"
                 "@p ld.global.nc.v2.b64 {%0, %1}, [%2];\n\t}"
                 : "=l"(gn[0]), "=l"(gn[1])
                 : "l"(gp), "r"(int((valid_mask >> r) & 1u)));
    gp = reinterpret_cast<const float*>(reinterpret_cast<const char*>(gp) + gstep);
  };
  fetch(0);
  float part[12];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const float4 w = wn;
    const float a = an;
    const unsigned o = on;
    const u64 g[2] = {gn[0], gn[1]};
    if (r + 1 < R) fetch(r + 1);

    bool la, lb;
    unsigned codes, ngA, ngB;
    if (GLOBAL) {
      la = (o >> 20) & 1u; lb = (o >> 21) & 1u;
      codes = o >> 23;
      const unsigned ob = (o & 0xFFFFFu) * gstride;
      const unsigned oa = ((o >> 22) & 1u) ? ob - gstride : ob;
      ngA = la ? oa : gA;
      ngB = lb ? ob : gB;
    } else {
      const unsigned rowA = o & 0x1FFu, rowB = (o >> 9) & 0x1FFu;
      la = rowA != 0x1FFu; lb = rowB != 0x1FFu;
      codes = o >> 18;
      ngA = la ? rowA : gA;                                     // staged: gA / gB hold the BOX ROW of the column a set keeps;
      ngB = lb ? rowB : gB;                                     // it is turned into a global offset only when the set is flushed
    }
    // a set that is about to be reloaded first sends what it has collected for its old rows
    if (la && (unsigned(nzA) << 1) != 0u) {
      const unsigned f = GLOBAL ? gA : to_global(gA);
      red2(const_cast<float*>(row_ptr(gvh, f)), GA1);
      red2(const_cast<float*>(row_ptr(gvh, f + rowpitch)), GA3);
    }
    if (lb && (unsigned(nzB) << 1) != 0u) {
      const unsigned f = GLOBAL ? gB : to_global(gB);
      red2(const_cast<float*>(row_ptr(gvh, f)), GB1);
      red2(const_cast<float*>(row_ptr(gvh, f + rowpitch)), GB3);
    }
    gA = ngA; gB = ngB;
    if (GLOBAL) {
      ldg2_if(A1[0], A1[1], row_ptr(vh, gA), la);
      ldg2_if(A3[0], A3[1], row_ptr(vh, gA + rowpitch), la);
      ldg2_if(B1[0], B1[1], row_ptr(vh, gB), lb);
      ldg2_if(B3[0], B3[1], row_ptr(vh, gB + rowpitch), lb);
    } else {
      const uint32_t pa = bufa + (o & 0x1FFu) * 128u, pb = bufa + ((o >> 9) & 0x1FFu) * 128u;
      lds2_if(A1[0], A1[1], pa, la);
      lds2_if(A3[0], A3[1], pa + pitch, la);
      lds2_if(B1[0], B1[1], pb, lb);
      lds2_if(B3[0], B3[1], pb + pitch, lb);
    }

    // w = (x-weight of set A, x-weight of set B, y-weight of the top row, y-weight of the bottom row)
    const float4 sg = kEbSigns.v[codes & 0xFFu];
    const float dA = sg.x, dB = sg.y, dya = sg.z, dyb = sg.w;
    const float e1 = dot2(g, A1), e3 = dot2(g, A3), f1 = dot2(g, B1), f3 = dot2(g, B3);
    const float T = fmaf(w.x, e1, w.y * f1), Bo = fmaf(w.x, e3, w.y * f3);          // g . top / bottom interpolant
    const float DT = fmaf(dA, e1, dB * f1), DB = fmaf(dA, e3, dB * f3);            // g . d/dx of them
    part[3 * (r & 3) + 0] = fmaf(w.z, T, w.w * Bo);
    part[3 * (r & 3) + 1] = fmaf(w.z, DT, w.w * DB) * a * fW;
    part[3 * (r & 3) + 2] = fmaf(dya, T, dyb * Bo) * a * fH;
    const float ya = w.z * a, yb = w.w * a;
    const float kA1 = ya * w.x, kA3 = yb * w.x, kB1 = ya * w.y, kB3 = yb * w.y;
    const float keepA = la ? 0.f : 1.f, keepB = lb ? 0.f : 1.f;
    acc2(GA1[0], kA1, g[0], keepA); acc2(GA1[1], kA1, g[1], keepA);
    acc2(GA3[0], kA3, g[0], keepA); acc2(GA3[1], kA3, g[1], keepA);
    acc2(GB1[0], kB1, g[0], keepB); acc2(GB1[1], kB1, g[1], keepB);
    acc2(GB3[0], kB3, g[0], keepB); acc2(GB3[1], kB3, g[1], keepB);
    nzA = (nzA & (int(la) - 1)) | __float_as_int(kA1) | __float_as_int(kA3);
    nzB = (nzB & (int(lb) - 1)) | __float_as_int(kB1) | __float_as_int(kB3);

    if ((r & 3) == 3) {
      float r3[3];
      reduce_steps<8>(part, r3, lane, k, j);
      if (!(j & 1)) {
        // the entries of these four steps have been consumed by every lane of the group: park the three gradients there
        s_w_e0[(r - 3 + (j >> 1)) * kEtLP + int(slot)] = make_float4(r3[0], r3[1], r3[2], 0.f);
      }
    }
  }
  if ((unsigned(nzA) << 1) != 0u) {
    const unsigned f = GLOBAL ? gA : to_global(gA);
    red2(const_cast<float*>(row_ptr(gvh, f)), GA1);
    red2(const_cast<float*>(row_ptr(gvh, f + rowpitch)), GA3);
  }
  if ((unsigned(nzB) << 1) != 0u) {
    const unsigned f = GLOBAL ? gB : to_global(gB);
    red2(const_cast<float*>(row_ptr(gvh, f)), GB1);
    red2(const_cast<float*>(row_ptr(gvh, f + rowpitch)), GB3);
  }
}

// PREP = true: `loc` / `attn` are the raw projection / reference points (see msda_enc_tma.cuh) and `grad_loc` receives the
// gradient of the PROJECTION row ([M][16][2] offset gradients, then [M][16] logit gradients = softmax backward);
// `grad_attn` is unused.
template <bool PREP = false>
__global__ void __launch_bounds__(kEbThreads, 2)
msda_bwd_enc_tma_kernel(const float* __restrict__ value, const float* __restrict__ loc, const float* __restrict__ attn,
                        const float* __restrict__ grad_out, float* __restrict__ grad_value, float* __restrict__ grad_loc,
                        float* __restrict__ grad_attn, const __grid_constant__ EtGeom g, const __grid_constant__ EtMaps maps) {
  constexpr int D = 32, R = kEtR, T = kEbThreads;
  extern __shared__ unsigned char et_smem_raw[];
  unsigned char* base = et_smem_raw + ((128u - (et_smem(et_smem_raw) & 127u)) & 127u);
  float* buf0 = reinterpret_cast<float*>(base);
  float* buf1 = buf0 + kEbBuf0Rows * D;
  float4* s_w = reinterpret_cast<float4*>(buf1 + kEbBuf1Rows * D);      // x / y weights (plan: x-weights in set order); later the gradients
  float* s_a = reinterpret_cast<float*>(s_w + kEtEntries);               // attention weight
  unsigned* s_o = reinterpret_cast<unsigned*>(s_a + kEtEntries);         // window word (see eb_slot_pass)
  unsigned* s_far = s_o + kEtEntries;
  int* s_box = reinterpret_cast<int*>(s_far + kEtQ);
  unsigned long long* s_bar = reinterpret_cast<unsigned long long*>(s_box + 2 * kEtMaxL);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wset = warp >> 2, wq = warp & 3;
  const int k = lane >> 3, j = lane & 7;
  const int L = g.L, M = g.M, Lq = g.Lq, LPr = L * kEtP;
  const int stride = M * D;

  const int tiles = g.tiles_used;
  const int m = blockIdx.x % M;
  const int t = tiles - 1 - int((blockIdx.x / M) % tiles);
  const int n = blockIdx.x / (M * tiles);
  int lq = 0;
#pragma unroll
  for (int l = 1; l < kEtMaxL; ++l)
    if (l < L && t >= g.tile_begin[l]) lq = l;
  const int tt = t - g.tile_begin[lq];
  const int ty = tt / g.tiles_x[lq], tx = tt - ty * g.tiles_x[lq];
  const int Wq = g.W[lq], Hq = g.H[lq];
  const int x0 = tx * kEtTX, y0 = ty * kEtTY;
  const int qbase = g.start[lq] + y0 * Wq + x0;

  if (tid < 2 * kEtMaxL) s_box[tid] = INT_MAX;
  if (tid < kEtMaxL) et_mbar_init(et_smem(s_bar + tid), 1);
  if (tid == 0) asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  if (tid < kEtQ) s_far[tid] = 0u;
  __syncthreads();

  // ---- phase 1: taps (x / y weights, attention weight, derivative signs, window corner)
  {
    constexpr int NIT = kEtQ * 16 / T;
    const int s = tid & 15, l = s >> 2;
    const bool slot_ok = s < LPr;
    const int Hl = slot_ok ? g.H[l] : 2, Wl = slot_ok ? g.W[l] : 2;
    int mnx = INT_MAX, mny = INT_MAX;
    float2 xy[NIT], rf[PREP ? NIT : 1];
    float at[NIT];
    const size_t srow = size_t(M) * LPr;
#pragma unroll
    for (int it = 0; it < NIT; ++it) {
      const int qi = (tid >> 4) + (T / 16) * it;
      const int ix = qi & 15, iy = qi >> 4;
      const bool valid = slot_ok && (x0 + ix < Wq) && (y0 + iy < Hq);
      if (PREP) {
        const size_t nq = size_t(n) * Lq + (valid ? qbase + iy * Wq + ix : qbase);
        const float* prow = loc + nq * size_t(3 * M * 16);
        xy[it] = __ldg(reinterpret_cast<const float2*>(prow) + m * 16 + s);
        at[it] = __ldg(prow + 2 * M * 16 + m * 16 + s);
        rf[it] = __ldg(reinterpret_cast<const float2*>(attn) + nq * L + l);
      } else {
        const size_t sidx = (size_t(n) * Lq + qbase + iy * Wq + ix) * srow + size_t(m) * LPr + s;
        xy[it] = valid ? __ldg(reinterpret_cast<const float2*>(loc) + sidx) : make_float2(-8.f, -8.f);
        at[it] = valid ? __ldg(attn + sidx) : 0.f;
      }
    }
#pragma unroll
    for (int it = 0; it < NIT; ++it) {
      const int qi = (tid >> 4) + (T / 16) * it;
      float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
      float a = 0.f;
      unsigned code = kEtNone;
      float lx = xy[it].x, ly = xy[it].y, aw = at[it];
      if (PREP) {
        float mx = aw;
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        const float e = expf(aw - mx);
        float sum = e;
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        aw = e / sum;
        const int ix = qi & 15, iy = qi >> 4;
        const bool valid = (x0 + ix < Wq) && (y0 + iy < Hq);
        lx = valid ? rf[it].x + lx / float(Hl) : -8.f;
        ly = valid ? rf[it].y + ly / float(Wl) : -8.f;
        a = valid ? aw : 0.f;               // the softmax backward needs the weight of EVERY sample, dead ones included
      }
      const float x = lx * float(Wl) - 0.5f, y = ly * float(Hl) - 0.5f;
      if (y > -1.f && x > -1.f && y < float(Hl) && x < float(Wl)) {
        int xb, yb;
        float dxa, dxb, dya, dyb;
        axis_window(x, Wl, xb, w.x, w.y, dxa, dxb);
        axis_window(y, Hl, yb, w.z, w.w, dya, dyb);
        a = aw;
        const unsigned codes = eb_enc(dxa) | (eb_enc(dxb) << 2) | (eb_enc(dya) << 4) | (eb_enc(dyb) << 6);
        if (l < lq) {
          code = unsigned(g.start[l] + yb * Wl + xb) | (codes << 20);        // pixel of the window's first corner
        } else {
          code = unsigned(xb) | (unsigned(yb) << 12) | (codes << 24);
          mnx = min(mnx, xb);
          mny = min(mny, yb);
        }
      }
      const int e = qi * kEtLP + s + (qi >> 3);
      s_w[e] = w;
      s_a[e] = a;
      s_o[e] = code;
    }
#pragma unroll
    for (int lv = 0; lv < kEtMaxL; ++lv) {
      const int vx = __reduce_min_sync(0xffffffffu, l == lv ? mnx : INT_MAX);
      const int vy = __reduce_min_sync(0xffffffffu, l == lv ? mny : INT_MAX);
      if (lane == 0 && vx != INT_MAX) {
        atomicMin(&s_box[2 * lv], vx);
        atomicMin(&s_box[2 * lv + 1], vy);
      }
    }
  }
  __syncthreads();

  auto issue = [&](int l) {
    const int d = l - lq;
    const int bx = s_box[2 * l], by = s_box[2 * l + 1];
    if (bx == INT_MAX) return;
    const uint32_t bar = et_smem(s_bar + l);
    et_mbar_expect(bar, uint32_t(eb_bw(d) * eb_bh(d) * 128));
    et_tma_box(et_smem((d & 1) ? buf1 : buf0), &maps.m[et_map_index(lq, l)], bar, m, bx, by, n);
  };
  if (tid == 0) {
    issue(lq);
    if (lq + 1 < L) issue(lq + 1);
  }

  // ---- phase 2 (plan): one thread per (run, slot) chain
  {
    const int s = tid & 15, l = s >> 2, run = tid >> 4;
    if (s < LPr) {
      const bool glob = l < lq;
      const int d = glob ? 0 : l - lq;
      const int BW = eb_bw(d), BH = eb_bh(d);
      const int bx = glob ? 0 : s_box[2 * l], by = glob ? 0 : s_box[2 * l + 1];
      unsigned co = 0u;
      bool have = false, par = false;
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int qi = (run >> 1) * kEtTX + (run & 1) * R + r;
        const int e = qi * kEtLP + s + run;
        const unsigned code = s_o[e];
        bool live = code != kEtNone;
        unsigned o = 0u, codes = 0u;
        if (live) {
          if (glob) {
            o = code & 0xFFFFFu;
            codes = code >> 20;
          } else {
            const int rx = int(code & 0xFFFu) - bx, ry = int((code >> 12) & 0xFFFu) - by;
            o = unsigned(ry * BW + rx);
            codes = code >> 24;
            if (rx > BW - 2 || ry > BH - 2) {
              atomicOr(&s_far[qi], 1u << s);
              s_w[e] = make_float4(0.f, 0.f, 0.f, 0.f);
              s_a[e] = 0.f;
              live = false;
            }
          }
        }
        if (!live) {
          s_o[e] = glob ? 0u : 0x3FFFFu;
          continue;
        }
        const bool same = have && (o == co);
        const bool shift = have && (o == co + 1u);
        const bool reload = !(same || shift);
        const bool ldA = reload || (shift && !par);
        const bool ldB = reload || (shift && par);
        par = reload ? false : (par != shift);
        co = o;
        have = true;
        if (par) {                                            // set A holds the right column: x-weights / x-signs in set order
          const float4 w = s_w[e];
          s_w[e] = make_float4(w.y, w.x, w.z, w.w);
          codes = ((codes >> 2) & 3u) | ((codes & 3u) << 2) | (codes & 0xF0u);
        }
        if (glob) {
          s_o[e] = (o + 1u) | (unsigned(ldA) << 20) | (unsigned(ldB) << 21) | (unsigned(reload) << 22) | (codes << 23);
        } else {
          const unsigned oa = ldA ? (reload ? o : o + 1u) : 0x1FFu;
          const unsigned ob = ldB ? o + 1u : 0x1FFu;
          s_o[e] = oa | (ob << 9) | (codes << 18);
        }
      }
    }
  }
  __syncthreads();

  // ---- hot loops: warp = two tile rows; warp set = two of a level's four slots, one after the other
  const int row_t = 2 * wq + (k >> 1);
  const int run_g = 2 * row_t + (k & 1);
  const int e0 = (row_t * kEtTX + (k & 1) * R) * kEtLP + run_g;
  const uint32_t sw_addr = et_smem(s_w + e0), sa_addr = et_smem(s_a + e0), so_addr = et_smem(s_o + e0);
  const uint32_t lane_off = uint32_t(j) * 16u;
  const size_t img = size_t(n) * g.S * stride + m * D + j * 4;
  const float* vh = value + img;
  float* gvh = grad_value + img;
  const int ix0 = (k & 1) * R;
  const bool row_ok = (y0 + row_t) < Hq;
  unsigned valid_mask = 0u;
#pragma unroll
  for (int r = 0; r < R; ++r)
    if (row_ok && (x0 + ix0 + r) < Wq) valid_mask |= 1u << r;
  const float* gout0 = grad_out + ((size_t(n) * Lq + qbase + row_t * Wq + ix0) * M + m) * D + j * 4;

#pragma unroll 1
  for (int l = 0; l < lq; ++l) {
#pragma unroll 1
    for (int p = 0; p < 2; ++p)
      eb_slot_pass<true>(sw_addr, sa_addr, so_addr, uint32_t(l * kEtP + wset * 2 + p), s_w + e0, 0u, 0u, 1, 0u, vh, gvh,
                         unsigned(stride), unsigned(g.W[l]) * unsigned(stride), float(g.W[l]), float(g.H[l]), gout0, stride,
                         valid_mask, lane, k, j);
  }
#pragma unroll 1
  for (int l = lq; l < L; ++l) {
    const int d = l - lq;
    if (s_box[2 * l] != INT_MAX) {
      et_mbar_wait(et_smem(s_bar + l), 0);
      const unsigned gbox = unsigned(g.start[l] + s_box[2 * l + 1] * g.W[l] + s_box[2 * l]) * unsigned(stride);
#pragma unroll 1
      for (int p = 0; p < 2; ++p)
        eb_slot_pass<false>(sw_addr, sa_addr, so_addr, uint32_t(l * kEtP + wset * 2 + p), s_w + e0,
                            et_smem((d & 1) ? buf1 : buf0) + lane_off, uint32_t(eb_bw(d)) * 128u, eb_bw(d), gbox, vh, gvh,
                            unsigned(stride), unsigned(g.W[l]) * unsigned(stride), float(g.W[l]), float(g.H[l]), gout0, stride,
                            valid_mask, lane, k, j);
    }
    if (l + 2 < L) {
      __syncthreads();
      if (tid == 0) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        issue(l + 2);
      }
    }
  }

  // ---- samples flagged "far": per sample from global memory with the reference's predicated corners (col2im formulas)
  {
    const unsigned gmask = 0xFFu << (8 * k);
#pragma unroll 1
    for (int r = 0; r < R; ++r) {
      unsigned fm = s_far[row_t * kEtTX + ix0 + r] & (0x3333u << (wset * 2));
      if (fm == 0u) continue;
      const size_t qidx = size_t(n) * Lq + qbase + row_t * Wq + ix0 + r;
      const float4 gr = ldg4(gout0 + size_t(r) * stride);
      while (fm) {
        const int s = __ffs(int(fm)) - 1;
        fm &= fm - 1;
        const int l = s >> 2;
        const int H = g.H[l], W = g.W[l];
        float2 xy;
        float a;
        if (PREP) {
          prep_sample_serial(loc, attn, qidx, m, s, l, M, L, H, W, xy.x, xy.y, a);
        } else {
          const size_t sidx = (qidx * M + m) * LPr + s;
          xy = __ldg(reinterpret_cast<const float2*>(loc) + sidx);
          a = __ldg(attn + sidx);
        }
        const Tap<float> tp = make_tap<float>(xy.x, xy.y, H, W, stride);
        float s_at = 0.f, s_x = 0.f, s_y = 0.f;
        if (tp.live) {
          const size_t lofs = size_t(g.start[l]) * stride;
          const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
          const float4 v1 = tp.k1 ? ldg4(vh + lofs + tp.o1) : z, v2 = tp.k2 ? ldg4(vh + lofs + tp.o2) : z;
          const float4 v3 = tp.k3 ? ldg4(vh + lofs + tp.o3) : z, v4 = tp.k4 ? ldg4(vh + lofs + tp.o4) : z;
          const float hx = 1.f - tp.lx, hy = 1.f - tp.ly;
          const float4 top = lin2(hx, v1, tp.lx, v2), bot = lin2(hx, v3, tp.lx, v4);
          const float4 dtop = lin2(-1.f, v1, 1.f, v2), dbot = lin2(-1.f, v3, 1.f, v4);
          s_at = dot4(gr, lin2(hy, top, tp.ly, bot));
          s_x = dot4(gr, lin2(hy, dtop, tp.ly, dbot)) * a * float(W);
          s_y = dot4(gr, lin2(-1.f, top, 1.f, bot)) * a * float(H);
          const float k1 = tp.w1 * a, k2 = tp.w2 * a, k3 = tp.w3 * a, k4 = tp.w4 * a;
          if (tp.k1 && k1 != 0.f) red4(gvh + lofs + tp.o1, k1, gr);
          if (tp.k2 && k2 != 0.f) red4(gvh + lofs + tp.o2, k2, gr);
          if (tp.k3 && k3 != 0.f) red4(gvh + lofs + tp.o3, k3, gr);
          if (tp.k4 && k4 != 0.f) red4(gvh + lofs + tp.o4, k4, gr);
        }
#pragma unroll
        for (int sh = 4; sh > 0; sh >>= 1) {
          s_at += __shfl_xor_sync(gmask, s_at, sh);
          s_x += __shfl_xor_sync(gmask, s_x, sh);
          s_y += __shfl_xor_sync(gmask, s_y, sh);
        }
        if (j == 0) {
          s_w[e0 + r * kEtLP + s] = make_float4(s_at, s_x, s_y, 0.f);
          if (PREP) s_a[e0 + r * kEtLP + s] = a;             // (the plan zeroed it when it flagged the sample)
        }
      }
    }
  }
  __syncthreads();

  // ---- grad_attn / grad_loc out of the tap entries, coalesced (same thread -> sample mapping as phase 1)
  {
    constexpr int NIT = kEtQ * 16 / T;
    const int s = tid & 15;
    if (s < LPr) {
      const size_t srow = size_t(M) * LPr;
#pragma unroll
      for (int it = 0; it < NIT; ++it) {
        const int qi = (tid >> 4) + (T / 16) * it;
        const int ix = qi & 15, iy = qi >> 4;
        const bool valid = x0 + ix < Wq && y0 + iy < Hq;
        const int e = qi * kEtLP + s + (qi >> 3);
        const float4 r = s_w[e];
        if (PREP) {
          // projection gradient: offsets through d(loc) / d(offset) = 1 / (H, W); logits through the softmax Jacobian
          // a_s * (g_s - sum_j a_j g_j), the sum taken over the 16 consecutive lanes of the head
          const float a = s_a[e];
          float dot = a * r.x;
#pragma unroll
          for (int o = 8; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
          if (valid) {
            const int l = s >> 2;
            float* grow = grad_loc + (size_t(n) * Lq + qbase + iy * Wq + ix) * size_t(3 * M * 16);
            reinterpret_cast<float2*>(grow)[m * 16 + s] = make_float2(r.y / float(g.H[l]), r.z / float(g.W[l]));
            grow[2 * M * 16 + m * 16 + s] = a * (r.x - dot);
          }
        } else if (valid) {
          const size_t sidx = (size_t(n) * Lq + qbase + iy * Wq + ix) * srow + size_t(m) * LPr + s;
          grad_attn[sidx] = r.x;
          *reinterpret_cast<float2*>(grad_loc + 2 * sidx) = make_float2(r.y, r.z);
        }
      }
    }
  }
}

}  // namespace msda
