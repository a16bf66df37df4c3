// Second-generation "run" kernels (fp32, D = 32): same register-resident sliding windows over runs of consecutive
// queries as msda_run.cuh, rebuilt around the instruction stream, because after the rows were cut to ~0.3x the
// kernels became ISSUE bound (SASS of the first generation: 56 instructions per (query, sample slot) step, of which
// 16 are the FFMAs that do the work, 16 are register copies the compiler inserts around the predicated window loads
// and ~20 are 64-bit address arithmetic and window-state logic):
//
//   * PLAN pass.  The window state machine (same / slid by one / reload, which register set holds the left column)
//     depends only on the tap offsets, so it is run ONCE per (run, head, slot) chain by one thread after the tap
//     prologue and its decisions are written back into the tap table: the bilinear weights already permuted into
//     register-set order (A-top, B-top, A-bottom, B-bottom) and two 32-bit element offsets (column to load into set A,
//     column to load into set B; kNoLoad = keep).  The hot loop has no state logic left.
//   * Packed pairs.  Window values travel as 64-bit register pairs (two fp32 lanes); sm_90 has no packed fp32 FMA,
//     so ffma2 issues one IEEE fp32 FMA per lane (the pair moves are register renames and cost no instruction).
//   * lean addressing: unsigned 32-bit element offsets + one IMAD.WIDE.U32 per row address.
//   * NS sample slots of a level walk the run INTERLEAVED (their windows live in separate registers): the loads of
//     all NS slots of a step are issued before the first FMA of the step, so NS x 4 row loads are in flight per lane
//     without the compiler having to rename window registers.
//
// Semantics as in msda_run.cuh / msda_d32.cuh (shifted window == the reference's zero padding for finite inputs,
// ms_deform_im2col_cuda.cuh:24-83,165-237).
#pragma once

#include "msda_run.cuh"

namespace msda {

typedef unsigned long long u64;
constexpr unsigned kNoLoad = 0xFFFFFFFFu;

__host__ __device__ inline int run2_entries(int R, int LP) { return 4 * R * kRunHeads * LP + 4; }
__host__ __device__ inline size_t fwd_run2_smem_bytes(int R, int LP) { return size_t(run2_entries(R, LP)) * (16 + 8); }

__device__ __forceinline__ void ffma2(u64& acc, float w, u64 v) {
  float a0, a1, v0, v1;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(a0), "=f"(a1) : "l"(acc));
  asm("mov.b64 {%0, %1}, %2;" : "=f"(v0), "=f"(v1) : "l"(v));
  a0 = __fmaf_rn(w, v0, a0);
  a1 = __fmaf_rn(w, v1, a1);
  asm("mov.b64 %0, {%1, %2};" : "=l"(acc) : "f"(a0), "f"(a1));
}
__device__ __forceinline__ void ldg2_if(u64& lo, u64& hi, const float* p, bool pred) {
  asm("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\t@p ld.global.nc.v2.b64 {%0, %1}, [%2];\n\t}"
      : "+l"(lo), "+l"(hi)
      : "l"(p), "r"(int(pred)));
}
// vb + o (elements) as ONE instruction (IMAD.WIDE.U32); the compiler's own lowering of `vb + o` re-derives the lane's
// 64-bit base from the uniform kernel argument every time (IADD3 + IMAD.X + LEA + LEA.HI.X per address)
__device__ __forceinline__ const float* row_ptr(const float* vb, unsigned o) {
  u64 a;
  asm("mad.wide.u32 %0, %1, 4, %2;" : "=l"(a) : "r"(o), "l"(vb));
  return reinterpret_cast<const float*>(a);
}
__device__ __forceinline__ float4 unpack4(u64 lo, u64 hi) {
  float4 r;
  asm("mov.b64 {%0, %1}, %2;" : "=f"(r.x), "=f"(r.y) : "l"(lo));
  asm("mov.b64 {%0, %1}, %2;" : "=f"(r.z), "=f"(r.w) : "l"(hi));
  return r;
}
__device__ __forceinline__ void pack4(const float4& v, u64& lo, u64& hi) {
  asm("mov.b64 %0, {%1, %2};" : "=l"(lo) : "f"(v.x), "f"(v.y));
  asm("mov.b64 %0, {%1, %2};" : "=l"(hi) : "f"(v.z), "f"(v.w));
}

// ------------------------------------------------------------------------------------------------
// Forward.  Unit = 4 runs x R queries x 4 heads; CTA = 4 warps (warp = head, 8-lane group = run).
// NS = sample slots walked together (must divide P; slots of one group share their level).
// ------------------------------------------------------------------------------------------------
template <int R, int NS, int LP_CT>
__global__ void __launch_bounds__(kRunThreads, 4)
msda_fwd_run2_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                     const float* __restrict__ loc, const float* __restrict__ attn, float* __restrict__ out,
                     int S, int M, int L, int Lq, int P, int qblocks) {
  constexpr int D = 32, RUNS = 4, QB = RUNS * R, ROWS = QB * kRunHeads;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ LevelTable lv;
  __shared__ unsigned char lvl_of[kMaxLP];

  const int LP = LP_CT ? LP_CT : L * P;
  const int entries = run2_entries(R, LP);
  float4* s_w = reinterpret_cast<float4*>(smem_raw);              // plan output: weights * attn in (A1, B1, A3, B3) order
  uint2* s_o = reinterpret_cast<uint2*>(s_w + entries);            // plan output: element offsets of the columns to load
  const unsigned stride = unsigned(M) * D;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const int k = lane >> 3, j = lane & 7;

  const int hblocks = M / kRunHeads;
  const int unit = blockIdx.x;
  const int hb = unit % hblocks;
  const int qb = (unit / hblocks) % qblocks;
  const int n = unit / (hblocks * qblocks);
  const int q0 = qb * QB;

  load_level_table(lv, lvl_of, shapes, L, P);
  __syncthreads();

  // ---- phase 1: one tap per (row, sample), read coalesced: corner weights * attn, offset of the window's first corner
  for (int i = tid; i < ROWS * LP; i += kRunThreads) {
    const int row = i / LP, s = i - row * LP;
    const int gq = q0 + (row >> 2);
    const int l = lvl_of[s];
    const int H = lv.H[l], W = lv.W[l];
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
    unsigned o = unsigned(lv.start[l]) * stride;
    if (gq < Lq) {
      const size_t sidx = ((size_t(n) * Lq + gq) * M + hb * kRunHeads + (row & 3)) * LP + s;
      const float2 xy = __ldg(reinterpret_cast<const float2*>(loc) + sidx);
      const float a = __ldg(attn + sidx);
      if (H >= 2 && W >= 2) {
        const float x = xy.x * float(W) - 0.5f, y = xy.y * float(H) - 0.5f;
        if (y > -1.f && x > -1.f && y < float(H) && x < float(W)) {
          int xb, yb;
          float wxa, wxb, wya, wyb, d0, d1;
          axis_window(x, W, xb, wxa, wxb, d0, d1);
          axis_window(y, H, yb, wya, wyb, d0, d1);
          w = make_float4(wya * wxa * a, wya * wxb * a, wyb * wxa * a, wyb * wxb * a);
          o += unsigned(yb * W + xb) * stride;
        }
      } else {
        w = make_float4(xy.x, xy.y, a, 0.f);       // degenerate level: raw sample, predicated taps on the fly
      }
    }
    const int slot = run_slot<R>(row, s, LP);
    s_w[slot] = w;
    s_o[slot] = make_uint2(o, 0u);
  }
  __syncthreads();

  // ---- phase 2 (plan): one thread per (run, head, slot) chain walks the R steps and fixes the window decisions
  for (int c = tid; c < RUNS * kRunHeads * LP; c += kRunThreads) {
    const int s = c % LP, kh = c / LP;
    const int h = kh & 3, kk = kh >> 2;
    const int l = lvl_of[s];
    if (lv.H[l] < 2 || lv.W[l] < 2) continue;
    unsigned co = 0;
    bool par = false;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const int slot = run_slot<R>((kk * R + r) * kRunHeads + h, s, LP);
      const unsigned o = s_o[slot].x;
      const float4 w = s_w[slot];
      const unsigned d = o - co;
      const bool same = (r > 0) && (d == 0u);
      const bool shift = (r > 0) && (d == stride);
      const bool reload = !(same || shift);
      const bool ldA = reload || (shift && !par);
      const bool ldB = reload || (shift && par);
      par = reload ? false : (par != shift);
      co = o;
      // after this step set A holds the right column iff par; w = (top-left, top-right, bottom-left, bottom-right)
      s_w[slot] = par ? make_float4(w.y, w.x, w.w, w.z) : w;
      s_o[slot] = make_uint2(ldA ? (reload ? o : o + stride) : kNoLoad, ldB ? o + stride : kNoLoad);
    }
  }
  __syncthreads();

  const int m = hb * kRunHeads + warp;
  const float* vb = value + size_t(n) * S * stride + m * D + j * 4;
  const int slot0 = run_slot<R>((k * R) * kRunHeads + warp, 0, LP);     // slot of (first query of the run, s = 0)

  u64 acc[R][2];
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r][0] = acc[r][1] = 0ull;

#pragma unroll 1
  for (int s0 = 0; s0 < LP; s0 += NS) {
    const int l = lvl_of[s0];
    const int H = lv.H[l], W = lv.W[l];
    if (H >= 2 && W >= 2) {
      const unsigned rowpitch = unsigned(W) * stride;
      u64 A1[NS][2], A3[NS][2], B1[NS][2], B3[NS][2];
#pragma unroll
      for (int p = 0; p < NS; ++p)
        A1[p][0] = A1[p][1] = A3[p][0] = A3[p][1] = B1[p][0] = B1[p][1] = B3[p][0] = B3[p][1] = 0ull;
#pragma unroll
      for (int r = 0; r < R; ++r) {
        float4 w[NS];
        uint2 o[NS];
#pragma unroll
        for (int p = 0; p < NS; ++p) {
          const int slot = slot0 + r * kRunHeads * LP + s0 + p;
          w[p] = s_w[slot];
          o[p] = s_o[slot];
        }
#pragma unroll
        for (int p = 0; p < NS; ++p) {
          const bool la = o[p].x != kNoLoad, lb = o[p].y != kNoLoad;
          ldg2_if(A1[p][0], A1[p][1], row_ptr(vb, o[p].x), la);
          ldg2_if(A3[p][0], A3[p][1], row_ptr(vb, o[p].x + rowpitch), la);
          ldg2_if(B1[p][0], B1[p][1], row_ptr(vb, o[p].y), lb);
          ldg2_if(B3[p][0], B3[p][1], row_ptr(vb, o[p].y + rowpitch), lb);
        }
#pragma unroll
        for (int p = 0; p < NS; ++p) {
          ffma2(acc[r][0], w[p].x, A1[p][0]);
          ffma2(acc[r][1], w[p].x, A1[p][1]);
          ffma2(acc[r][0], w[p].y, B1[p][0]);
          ffma2(acc[r][1], w[p].y, B1[p][1]);
          ffma2(acc[r][0], w[p].z, A3[p][0]);
          ffma2(acc[r][1], w[p].z, A3[p][1]);
          ffma2(acc[r][0], w[p].w, B3[p][0]);
          ffma2(acc[r][1], w[p].w, B3[p][1]);
        }
      }
    } else {
      // degenerate level (a single row or column): predicated taps built from the raw (x, y, attn) in the slot
      const float* vl = vb + size_t(lv.start[l]) * stride;
      for (int p = 0; p < NS; ++p) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const int gq = q0 + k * R + r;
          if (gq >= Lq) continue;
          const float4 raw = s_w[slot0 + r * kRunHeads * LP + s0 + p];
          const Tap<float> t = make_tap<float>(raw.x, raw.y, H, W, int(stride));
          if (!t.live) continue;
          const float a = raw.z;
          const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
          float4 av = unpack4(acc[r][0], acc[r][1]);
          fma4(av, t.w1 * a, t.k1 ? ldg4(vl + t.o1) : z);
          fma4(av, t.w2 * a, t.k2 ? ldg4(vl + t.o2) : z);
          fma4(av, t.w3 * a, t.k3 ? ldg4(vl + t.o3) : z);
          fma4(av, t.w4 * a, t.k4 ? ldg4(vl + t.o4) : z);
          pack4(av, acc[r][0], acc[r][1]);
        }
      }
    }
  }

#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int gq = q0 + k * R + r;
    if (gq < Lq) {
      float* dst = out + ((size_t(n) * Lq + gq) * M + m) * D + j * 4;
      asm volatile("st.global.v2.b64 [%0], {%1, %2};" ::"l"(dst), "l"(acc[r][0]), "l"(acc[r][1]) : "memory");
    }
  }
}

}  // namespace msda
