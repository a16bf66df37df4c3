// "Run" kernels for fp32, D = 32 (128-byte head rows), large query sets (the encoder: Lq = S, raster order).
//
// Why: the gather is bound by L1 wavefronts (one per 128-byte corner row) and, in the backward, by the
// L2 reduction units (one RED.128 per corner row) -- not by HBM.  In the encoder, consecutive
// queries are neighbouring pixels and their sampling windows on a level overlap: on the query's own level the
// 2x2 window slides by one pixel per query (the right column becomes the left one), on the coarser levels it
// mostly does not move at all.  So instead of giving a query's 16 samples to one 8-lane group (which reads
// 64 rows per query), an 8-lane group here walks a RUN of R consecutive queries for ONE sample slot (level,
// point) at a time and keeps the current 2x2 window in registers:
//     same window      -> no load                      (backward: keep accumulating, no reduction)
//     slid by +1 pixel -> load one new column (2 rows) (backward: flush one column = 2 RED.128)
//     anything else    -> load both columns  (4 rows)  (backward: flush both)
// For a C2 encoder call with model-like sampling locations that is ~0.3x of the rows of the per-query scheme,
// for forward loads and backward reductions alike; with scattered locations it degenerates to the old cost.
// The two register sets (A, B) never move: a parity bit says which one currently holds the left column and
// the bilinear weights are swapped instead of the data.
//
// Work unit = QB = 4*R consecutive queries x HB = 4 heads; CTA = 4 warps; warp = head, the warp's four
// 8-lane groups = four adjacent runs.  A cooperative prologue turns every sample of the unit into a tap
// exactly once (coalesced reads of sampling_loc / attn_weight) and parks it in shared memory; the backward
// writes grad_attn / grad_loc back into the tap slots and streams them out coalesced at the end.
// Semantics as in msda_d32.cuh (shifted window == the reference's zero padding for finite inputs).
//
// LG = lanes per group = 16-byte packs per head row: 8 for D = 32, 9 for the multi-frame geometry D = 36 (a warp then
// carries three runs, lanes 27..31 shadow the last lane of run 2 with every store / reduction masked).
#pragma once

#include "msda_d32.cuh"

namespace msda {

constexpr int kRunThreads = 128;
constexpr int kRunHeads = 4;            // heads per unit (= warps per CTA)

__host__ __device__ constexpr int run_runs(int LG) { return 32 / LG; }                          // runs per warp: 4 or 3
__host__ __device__ inline int run_entries(int LG, int R, int LP) { return run_runs(LG) * R * kRunHeads * LP + 4; }
__host__ __device__ inline size_t fwd_run_smem_bytes(int LG, int R, int LP) { return size_t(run_entries(LG, R, LP)) * (16 + 4); }
__host__ __device__ inline size_t bwd_run_smem_bytes(int LG, int R, int LP) { return size_t(run_entries(LG, R, LP)) * (16 + 8); }

// tap slot of (row, s): rows are (query-in-unit * 4 + head); every run's block is skewed by one slot so that the
// four 8-lane groups of a warp (same head, same step, four runs) hit four different bank groups
template <int R>
__device__ __forceinline__ int run_slot(int row, int s, int LP) { return row * LP + s + row / (4 * R); }

// predicated 128-bit read-only load that leaves the destination untouched when the predicate is false
__device__ __forceinline__ void ldg4_if(float4& v, const float* p, bool pred) {
  asm("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %5, 0;\n\t@p ld.global.nc.v4.f32 {%0, %1, %2, %3}, [%4];\n\t}"
      : "+f"(v.x), "+f"(v.y), "+f"(v.z), "+f"(v.w)
      : "l"(p), "r"(int(pred)));
}

__device__ __forceinline__ void red4v(float* p, const float4& g) {
  asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p), "f"(g.x), "f"(g.y), "f"(g.z),
               "f"(g.w)
               : "memory");
}

// One sample's normalised location and attention weight.
//   PREP = false: read from sampling_loc / attn_weight (the reference's operands).
//   PREP = true : computed from the module's raw projection, never materialised (ops/modules/ms_deform_attn.py:69-79):
//                 `a` = the row [n, q] of the [offsets | logits] GEMM ([M][LP][2] offsets, then [M][LP] logits),
//                 `b` = reference points [n, q][L][2];  loc = ref + offset / (H, W) -- the reference divides the (x, y)
//                 offset by spatial_shapes AS STORED, i.e. by (H, W) -- and attn = softmax of the LP logits of the head,
//                 reduced over the LP consecutive lanes that hold them (LP = 16).
template <bool PREP, int LPC>
__device__ __forceinline__ void run_sample(const float* __restrict__ a, const float* __restrict__ b, size_t nq, int m, int s,
                                           int l, int M, int L, int LP, int H, int W, float& x, float& y, float& w) {
  if (!PREP) {
    const size_t sidx = (nq * M + m) * LP + s;
    const float2 xy = __ldg(reinterpret_cast<const float2*>(a) + sidx);
    x = xy.x; y = xy.y;
    w = __ldg(b + sidx);
  } else {
    const float* prow = a + nq * size_t(3 * M * LPC);
    const float2 off = __ldg(reinterpret_cast<const float2*>(prow) + m * LPC + s);
    const float logit = __ldg(prow + 2 * M * LPC + m * LPC + s);
    float mx = logit;
#pragma unroll
    for (int o = LPC / 2; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    const float e = expf(logit - mx);
    float sum = e;
#pragma unroll
    for (int o = LPC / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    w = e / sum;
    const float2 r = __ldg(reinterpret_cast<const float2*>(b) + nq * L + l);
    x = r.x + off.x / float(H);
    y = r.y + off.y / float(W);
  }
}

// ------------------------------------------------------------------------------------------------
// Forward
// ------------------------------------------------------------------------------------------------
template <int LG, int R, int LP_CT, bool PREP = false>
__global__ void __launch_bounds__(kRunThreads, 4)
msda_fwd_run_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                    const float* __restrict__ loc, const float* __restrict__ attn, float* __restrict__ out,
                    int S, int M, int L, int Lq, int P, int qblocks) {
  constexpr int D = 4 * LG, RUNS = run_runs(LG), QB = RUNS * R, ROWS = QB * kRunHeads;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ LevelTable lv;
  __shared__ unsigned char lvl_of[kMaxLP];

  const int LP = LP_CT ? LP_CT : L * P;
  const int entries = run_entries(LG, R, LP);
  float4* s_w = reinterpret_cast<float4*>(smem_raw);             // corner weights * attn
  int* s_o = reinterpret_cast<int*>(s_w + entries);               // element offset of the window's first corner
  const int stride = M * D;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const bool live = lane < RUNS * LG;                             // (LG = 9: lanes 27..31 shadow lane 26)
  const int k = live ? lane / LG : RUNS - 1, j = live ? lane - k * LG : LG - 1;

  const int hblocks = M / kRunHeads;
  const int unit = blockIdx.x;
  const int hb = unit % hblocks;
  const int qb = (unit / hblocks) % qblocks;
  const int n = unit / (hblocks * qblocks);
  const int q0 = qb * QB;

  load_level_table(lv, lvl_of, shapes, L, P);
  __syncthreads();

  // ---- prologue: one tap per (row, sample), read coalesced.  Degenerate levels (a single row or column) keep the raw
  //      (x, y, attn) in the slot instead; the main loop builds their predicated taps on the fly.
  static_assert(!PREP || LP_CT == 16, "the fused sampling prologue reduces over 16 consecutive lanes");
  for (int i = tid; i < ROWS * LP; i += kRunThreads) {
    const int row = i / LP, s = i - row * LP;
    const int gq = q0 + (row >> 2);
    const int l = lvl_of[s];
    const int H = lv.H[l], W = lv.W[l];
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
    int o = lv.start[l] * stride;
    float lx, ly, a;
    run_sample<PREP, LP_CT ? LP_CT : 2>(loc, attn, size_t(n) * Lq + min(gq, Lq - 1), hb * kRunHeads + (row & 3), s, l, M, L,
                                        LP, H, W, lx, ly, a);
    if (gq < Lq) {
      if (H >= 2 && W >= 2) {
        const float x = lx * float(W) - 0.5f, y = ly * float(H) - 0.5f;
        if (y > -1.f && x > -1.f && y < float(H) && x < float(W)) {
          int xb, yb;
          float wxa, wxb, wya, wyb, d0, d1;
          axis_window(x, W, xb, wxa, wxb, d0, d1);
          axis_window(y, H, yb, wya, wyb, d0, d1);
          w = make_float4(wya * wxa * a, wya * wxb * a, wyb * wxa * a, wyb * wxb * a);
          o += (yb * W + xb) * stride;
        }
      } else {
        w = make_float4(lx, ly, a, 0.f);
      }
    }
    const int slot = run_slot<R>(row, s, LP);
    s_w[slot] = w;
    s_o[slot] = o;
  }
  __syncthreads();

  const int m = hb * kRunHeads + warp;
  const float* vb = value + size_t(n) * S * stride + m * D + j * 4;
  const int row0 = (k * R) * kRunHeads + warp;            // row of this group's first query

  float4 acc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r] = make_float4(0.f, 0.f, 0.f, 0.f);

  for (int s = 0; s < LP; ++s) {
    const int l = lvl_of[s];
    const int H = lv.H[l], W = lv.W[l];
    if (H >= 2 && W >= 2) {
      const int rowpitch = W * stride;
      float4 A1 = make_float4(0.f, 0.f, 0.f, 0.f), A3 = A1, B1 = A1, B3 = A1;
      int co = 0;
      bool par = false;
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int slot = run_slot<R>(row0 + r * kRunHeads, s, LP);
        const float4 w = s_w[slot];
        const int o = s_o[slot];
        const int d = o - co;
        const bool same = (r > 0) && (d == 0);
        const bool shift = (r > 0) && (d == stride);
        const bool reload = !(same || shift);
        const bool ldA = reload || (shift && !par);
        const bool ldB = reload || (shift && par);
        const float* pB = vb + o + stride;                 // the (new) right column in every load case
        const float* pA = reload ? vb + o : pB;
        ldg4_if(A1, pA, ldA);
        ldg4_if(A3, pA + rowpitch, ldA);
        ldg4_if(B1, pB, ldB);
        ldg4_if(B3, pB + rowpitch, ldB);
        par = reload ? false : (par != shift);
        co = o;
        // w = (top-left, top-right, bottom-left, bottom-right) * attn; A holds the left column unless par
        fma4(acc[r], par ? w.y : w.x, A1);
        fma4(acc[r], par ? w.x : w.y, B1);
        fma4(acc[r], par ? w.w : w.z, A3);
        fma4(acc[r], par ? w.z : w.w, B3);
      }
    } else {
      // degenerate level (a single row or column): predicated taps built from the raw (x, y, attn) in the slot
      const float* vl = vb + size_t(lv.start[l]) * stride;
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const int gq = q0 + k * R + r;
        if (gq >= Lq) continue;
        const float4 raw = s_w[run_slot<R>(row0 + r * kRunHeads, s, LP)];
        const Tap<float> t = make_tap<float>(raw.x, raw.y, H, W, stride);
        if (!t.live) continue;
        const float a = raw.z;
        const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
        fma4(acc[r], t.w1 * a, t.k1 ? ldg4(vl + t.o1) : z);
        fma4(acc[r], t.w2 * a, t.k2 ? ldg4(vl + t.o2) : z);
        fma4(acc[r], t.w3 * a, t.k3 ? ldg4(vl + t.o3) : z);
        fma4(acc[r], t.w4 * a, t.k4 ? ldg4(vl + t.o4) : z);
      }
    }
  }

#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int gq = q0 + k * R + r;
    if (live && gq < Lq)
      *reinterpret_cast<float4*>(out + ((size_t(n) * Lq + gq) * M + m) * D + j * 4) = acc[r];
  }
}

// ------------------------------------------------------------------------------------------------
// Backward (fused): grad_value with per-column register accumulation, grad_sampling_loc, grad_attn_weight
// ------------------------------------------------------------------------------------------------
// Tap: s_w = (wxa, wxb, wya, wyb), s_ao = (attn, offset | cx | cy << 2) where cx, cy in {0: both taps inside
// (d = -1, +1), 1: only the upper tap (d = +1, 0), 2: only the lower tap (d = 0, -1), 3: dead (0, 0)}; the offset is
// a multiple of M*32 >= 128, so its low bits are free.
__device__ __forceinline__ int axis_code(float da, float db) { return da < 0.f ? 0 : (da > 0.f ? 1 : (db < 0.f ? 2 : 3)); }
__device__ __forceinline__ float code_da(int c) { return c == 0 ? -1.f : (c == 1 ? 1.f : 0.f); }
__device__ __forceinline__ float code_db(int c) { return c == 0 ? 1.f : (c == 2 ? -1.f : 0.f); }

// Sums the 12 per-lane partials of four steps over the LG lanes of every group: afterwards lanes j = 0, 2, 4, 6 of a
// group hold (grad_attn, grad_loc.x, grad_loc.y) of step j >> 1.  LG = 8: transposing xor butterfly (12 shuffles);
// LG = 9: lane 8 is folded into lanes 0..7 first (12 more), then the same butterfly with explicit partner lanes.
template <int LG>
__device__ __forceinline__ void reduce_steps(float (&part)[12], float (&r3)[3], int lane, int k, int j) {
  int p4, p2, p1;
  if (LG == 8) {
    p4 = lane ^ 4; p2 = lane ^ 2; p1 = lane ^ 1;
  } else {
    const int base = k * LG;
#pragma unroll
    for (int c = 0; c < 12; ++c) {
      const float v = __shfl_sync(0xffffffffu, part[c], base + 8);
      if (j == (c & 7)) part[c] += v;
    }
    const int jj = j < 8 ? j : 0;                   // lane 8 (and the shadow lanes): harmless partners, result unused
    p4 = base + (jj ^ 4); p2 = base + (jj ^ 2); p1 = base + (jj ^ 1);
  }
  float r6[6];
  {
    const bool hi = j & 4;
#pragma unroll
    for (int c = 0; c < 6; ++c) {
      const float mine = hi ? part[6 + c] : part[c];
      const float give = hi ? part[c] : part[6 + c];
      r6[c] = mine + __shfl_sync(0xffffffffu, give, p4);
    }
  }
  {
    const bool hi = j & 2;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const float mine = hi ? r6[3 + c] : r6[c];
      const float give = hi ? r6[c] : r6[3 + c];
      r3[c] = mine + __shfl_sync(0xffffffffu, give, p2);
    }
  }
#pragma unroll
  for (int c = 0; c < 3; ++c) r3[c] += __shfl_sync(0xffffffffu, r3[c], p1);
}

// PREP = true: `loc` / `attn` are the raw projection / reference points (see run_sample) and `grad_loc` receives the
// gradient of the PROJECTION row ([M][LP][2] offset gradients, then [M][LP] logit gradients = softmax backward);
// `grad_attn` is unused.
template <int LG, int R, int LP_CT, bool PREP = false>
__global__ void __launch_bounds__(kRunThreads, 4)
msda_bwd_run_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                    const float* __restrict__ loc, const float* __restrict__ attn,
                    const float* __restrict__ grad_out, float* __restrict__ grad_value,
                    float* __restrict__ grad_loc, float* __restrict__ grad_attn,
                    int S, int M, int L, int Lq, int P, int qblocks) {
  constexpr int D = 4 * LG, RUNS = run_runs(LG), QB = RUNS * R, ROWS = QB * kRunHeads;
  static_assert(R % 4 == 0, "the lane butterfly reduces four steps at a time");
  extern __shared__ __align__(16) unsigned char smem_raw[];
  __shared__ LevelTable lv;
  __shared__ unsigned char lvl_of[kMaxLP];

  const int LP = LP_CT ? LP_CT : L * P;
  const int entries = run_entries(LG, R, LP);
  float4* s_w = reinterpret_cast<float4*>(smem_raw);
  float2* s_ao = reinterpret_cast<float2*>(s_w + entries);
  const int stride = M * D;
  const int tid = threadIdx.x;
  const int warp = tid >> 5, lane = tid & 31;
  const bool live = lane < RUNS * LG;                             // shadow lanes: no reductions, no stores
  const int k = live ? lane / LG : RUNS - 1, j = live ? lane - k * LG : LG - 1;

  const int hblocks = M / kRunHeads;
  const int unit = blockIdx.x;
  const int hb = unit % hblocks;
  const int qb = (unit / hblocks) % qblocks;
  const int n = unit / (hblocks * qblocks);
  const int q0 = qb * QB;

  load_level_table(lv, lvl_of, shapes, L, P);
  __syncthreads();

  static_assert(!PREP || LP_CT == 16, "the fused sampling prologue reduces over 16 consecutive lanes");
  for (int i = tid; i < ROWS * LP; i += kRunThreads) {
    const int row = i / LP, s = i - row * LP;
    const int gq = q0 + (row >> 2);
    const int l = lvl_of[s];
    const int H = lv.H[l], W = lv.W[l];
    float4 w = make_float4(0.f, 0.f, 0.f, 0.f);
    int o = lv.start[l] * stride + 15;                      // dead: codes (3, 3)
    float lx, ly, a;
    run_sample<PREP, LP_CT ? LP_CT : 2>(loc, attn, size_t(n) * Lq + min(gq, Lq - 1), hb * kRunHeads + (row & 3), s, l, M, L,
                                        LP, H, W, lx, ly, a);
    if (gq >= Lq) {
      a = 0.f;
    } else if (H >= 2 && W >= 2) {
      const float x = lx * float(W) - 0.5f, y = ly * float(H) - 0.5f;
      if (y > -1.f && x > -1.f && y < float(H) && x < float(W)) {
        int xb, yb;
        float dxa, dxb, dya, dyb;
        axis_window(x, W, xb, w.x, w.y, dxa, dxb);
        axis_window(y, H, yb, w.z, w.w, dya, dyb);
        o = (lv.start[l] + yb * W + xb) * stride + axis_code(dxa, dxb) + 4 * axis_code(dya, dyb);
      }
    } else {
      w = make_float4(lx, ly, 0.f, 0.f);                   // degenerate level: raw location, taps on the fly
    }
    const int slot = run_slot<R>(row, s, LP);
    s_w[slot] = w;
    s_ao[slot] = make_float2(a, __int_as_float(o));
  }
  __syncthreads();

  const int m = hb * kRunHeads + warp;
  const size_t head = size_t(n) * S * stride + m * D + j * 4;
  const float* vb = value + head;
  float* gvb = grad_value + head;
  const int row0 = (k * R) * kRunHeads + warp;

  float4 g[R];
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int gq = q0 + k * R + r;
    g[r] = (live && gq < Lq) ? ldg4(grad_out + ((size_t(n) * Lq + gq) * M + m) * D + j * 4)
                             : make_float4(0.f, 0.f, 0.f, 0.f);
  }

  for (int s = 0; s < LP; ++s) {
    const int l = lvl_of[s];
    const int H = lv.H[l], W = lv.W[l];
    const bool fast = (H >= 2 && W >= 2);
    const int rowpitch = W * stride;
    const float fW = float(W), fH = float(H);
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 A1 = zero4, A3 = zero4, B1 = zero4, B3 = zero4;          // window columns (top, bottom)
    float4 GA1 = zero4, GA3 = zero4, GB1 = zero4, GB3 = zero4;      // their pending grad_value contributions
    int oA = 0, oB = 0;                                              // element offsets of A1 / B1
    int nzA = 0, nzB = 0;                                            // OR of the coefficient bits seen so far
    int co = 0;
    bool par = false;

#pragma unroll
    for (int r0 = 0; r0 < R; r0 += 4) {
      float part[12];
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        const int r = r0 + u;
        float s_a = 0.f, s_x = 0.f, s_y = 0.f;
        if (fast) {
          const int slot = run_slot<R>(row0 + r * kRunHeads, s, LP);
          const float4 w = s_w[slot];
          const float2 ao = s_ao[slot];
          const int oc = __float_as_int(ao.y);
          const int o = oc & ~15;
          const int cx = oc & 3, cy = (oc >> 2) & 3;
          const int d = o - co;
          const bool same = (r > 0) && (d == 0);
          const bool shift = (r > 0) && (d == stride);
          const bool reload = !(same || shift);
          const bool ldA = reload || (shift && !par);
          const bool ldB = reload || (shift && par);
          if (ldA) {
            if (live && (unsigned(nzA) << 1) != 0) { red4v(gvb + oA, GA1); red4v(gvb + oA + rowpitch, GA3); }
            GA1 = zero4; GA3 = zero4; nzA = 0;
            oA = reload ? o : o + stride;
          }
          if (ldB) {
            if (live && (unsigned(nzB) << 1) != 0) { red4v(gvb + oB, GB1); red4v(gvb + oB + rowpitch, GB3); }
            GB1 = zero4; GB3 = zero4; nzB = 0;
            oB = o + stride;
          }
          ldg4_if(A1, vb + oA, ldA);
          ldg4_if(A3, vb + oA + rowpitch, ldA);
          ldg4_if(B1, vb + oB, ldB);
          ldg4_if(B3, vb + oB + rowpitch, ldB);
          par = reload ? false : (par != shift);
          co = o;

          const float dxa = code_da(cx), dxb = code_db(cx), dya = code_da(cy), dyb = code_db(cy);
          const float xa = par ? w.y : w.x, xb = par ? w.x : w.y;       // x-weights of columns A, B
          const float da = par ? dxb : dxa, db = par ? dxa : dxb;
          const float e1 = dot4(g[r], A1), e3 = dot4(g[r], A3), f1 = dot4(g[r], B1), f3 = dot4(g[r], B3);
          const float T = fmaf(xa, e1, xb * f1), Bo = fmaf(xa, e3, xb * f3);       // g . top / bottom interpolant
          const float DT = fmaf(da, e1, db * f1), DB = fmaf(da, e3, db * f3);     // g . d/dx of them
          s_a = fmaf(w.z, T, w.w * Bo);
          s_x = fmaf(w.z, DT, w.w * DB) * ao.x * fW;
          s_y = fmaf(dya, T, dyb * Bo) * ao.x * fH;
          const float ya = w.z * ao.x, yb = w.w * ao.x;
          const float kA1 = ya * xa, kA3 = yb * xa, kB1 = ya * xb, kB3 = yb * xb;
          fma4(GA1, kA1, g[r]);
          fma4(GA3, kA3, g[r]);
          fma4(GB1, kB1, g[r]);
          fma4(GB3, kB3, g[r]);
          nzA |= __float_as_int(kA1) | __float_as_int(kA3);
          nzB |= __float_as_int(kB1) | __float_as_int(kB3);
        } else {
          // degenerate level: predicated taps on the fly (reference formulas, .cuh:96-163), direct reductions
          const int gq = q0 + k * R + r;
          if (live && gq < Lq) {
            const int slot = run_slot<R>(row0 + r * kRunHeads, s, LP);
            const float4 raw = s_w[slot];
            const float a = s_ao[slot].x;
            const Tap<float> t = make_tap<float>(raw.x, raw.y, H, W, stride);
            if (t.live) {
              const size_t lofs = size_t(lv.start[l]) * stride;
              const float4 v1 = t.k1 ? ldg4(vb + lofs + t.o1) : zero4, v2 = t.k2 ? ldg4(vb + lofs + t.o2) : zero4;
              const float4 v3 = t.k3 ? ldg4(vb + lofs + t.o3) : zero4, v4 = t.k4 ? ldg4(vb + lofs + t.o4) : zero4;
              const float hx = 1.f - t.lx, hy = 1.f - t.ly;
              const float4 top = lin2(hx, v1, t.lx, v2), bot = lin2(hx, v3, t.lx, v4);
              const float4 dtop = lin2(-1.f, v1, 1.f, v2), dbot = lin2(-1.f, v3, 1.f, v4);
              s_a = dot4(g[r], lin2(hy, top, t.ly, bot));
              s_x = dot4(g[r], lin2(hy, dtop, t.ly, dbot)) * a * fW;
              s_y = dot4(g[r], lin2(-1.f, top, 1.f, bot)) * a * fH;
              if (t.k1) red4(gvb + lofs + t.o1, t.w1 * a, g[r]);
              if (t.k2) red4(gvb + lofs + t.o2, t.w2 * a, g[r]);
              if (t.k3) red4(gvb + lofs + t.o3, t.w3 * a, g[r]);
              if (t.k4) red4(gvb + lofs + t.o4, t.w4 * a, g[r]);
            }
          }
        }
        part[3 * u + 0] = s_a;
        part[3 * u + 1] = s_x;
        part[3 * u + 2] = s_y;
      }
      float r3[3];
      reduce_steps<LG>(part, r3, lane, k, j);
      if (live && j < 8 && !(j & 1)) {
        // the tap slot of (step, s) has been consumed by all lanes of the group: reuse it for the three gradients
        const int slot = run_slot<R>(row0 + (r0 + (j >> 1)) * kRunHeads, s, LP);
        s_w[slot] = make_float4(r3[0], r3[1], r3[2], 0.f);
      }
    }
    if (fast && live) {
      if ((unsigned(nzA) << 1) != 0) { red4v(gvb + oA, GA1); red4v(gvb + oA + rowpitch, GA3); }
      if ((unsigned(nzB) << 1) != 0) { red4v(gvb + oB, GB1); red4v(gvb + oB + rowpitch, GB3); }
    }
  }
  __syncthreads();

  // ---- stream the gradients out of the tap slots, coalesced
  for (int i = tid; i < ROWS * LP; i += kRunThreads) {
    const int row = i / LP, s = i - row * LP;
    const int gq = q0 + (row >> 2);
    const int slot = run_slot<R>(row, s, LP);
    const float4 r = s_w[slot];
    if (!PREP) {
      if (gq >= Lq) continue;
      const size_t sidx = ((size_t(n) * Lq + gq) * M + hb * kRunHeads + (row & 3)) * LP + s;
      grad_attn[sidx] = r.x;
      *reinterpret_cast<float2*>(grad_loc + 2 * sidx) = make_float2(r.y, r.z);
    } else {
      // projection gradient: offsets via d(loc)/d(off) = 1 / (H, W); logits via the softmax Jacobian
      // a * (g - sum_s a_s g_s), the sum taken over the LP consecutive lanes of the head (all lanes take part)
      const float a = s_ao[slot].x;
      float dot = a * r.x;
#pragma unroll
      for (int o = (LP_CT ? LP_CT : 2) / 2; o > 0; o >>= 1) dot += __shfl_xor_sync(0xffffffffu, dot, o);
      if (gq >= Lq) continue;
      const int l = lvl_of[s];
      const int mm = hb * kRunHeads + (row & 3);
      float* grow = grad_loc + (size_t(n) * Lq + gq) * size_t(3 * M * LP);
      reinterpret_cast<float2*>(grow)[mm * LP + s] = make_float2(r.y / float(lv.H[l]), r.z / float(lv.W[l]));
      grow[2 * M * LP + mm * LP + s] = a * (r.x - dot);
    }
  }
}

// ------------------------------------------------------------------------------------------------
// "Wide" kernels for small query sets (the decoder: a few hundred queries, scattered locations): one WARP per
// (n, q, m) group, lane = (sample quarter, 16-byte channel pack), so that 2 400 groups become 600 CTAs with
// 16 independent row loads in flight per lane instead of 75 CTAs walking 16 samples serially.
// ------------------------------------------------------------------------------------------------
constexpr int kWideThreads = 128;       // 4 groups per CTA

__global__ void __launch_bounds__(kWideThreads)
msda_fwd_wide_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                     const float* __restrict__ loc, const float* __restrict__ attn, float* __restrict__ out,
                     int S, int M, int L, int Lq, int P, uint32_t groups) {
  constexpr int D = 32;
  __shared__ LevelTable lv;
  __shared__ unsigned char lvl_of[kMaxLP];
  const int LP = L * P;
  const int stride = M * D;
  const int lane = threadIdx.x & 31;
  const int q4 = lane >> 3, j = lane & 7;
  load_level_table(lv, lvl_of, shapes, L, P);
  __syncthreads();
  const uint32_t gid = blockIdx.x * (kWideThreads / 32) + (threadIdx.x >> 5);
  if (gid >= groups) return;                                   // warp-uniform
  const uint32_t m = gid % uint32_t(M);
  const uint32_t n = gid / (uint32_t(M) * uint32_t(Lq));
  const float* vb = value + size_t(n) * S * stride + m * D + j * 4;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll 4
  for (int s = q4; s < LP; s += 4) {
    const int l = lvl_of[s];
    const int H = lv.H[l], W = lv.W[l];
    const size_t sidx = size_t(gid) * LP + s;
    const float2 xy = __ldg(reinterpret_cast<const float2*>(loc) + sidx);
    const float a = __ldg(attn + sidx);
    const Tap<float> t = make_tap<float>(xy.x, xy.y, H, W, stride);
    if (!t.live) continue;
    const float* vl = vb + size_t(lv.start[l]) * stride;
    const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 v1 = t.k1 ? ldg4(vl + t.o1) : z, v2 = t.k2 ? ldg4(vl + t.o2) : z;
    const float4 v3 = t.k3 ? ldg4(vl + t.o3) : z, v4 = t.k4 ? ldg4(vl + t.o4) : z;
    fma4(acc, t.w1 * a, v1);
    fma4(acc, t.w2 * a, v2);
    fma4(acc, t.w3 * a, v3);
    fma4(acc, t.w4 * a, v4);
  }
#pragma unroll
  for (int sh = 8; sh <= 16; sh <<= 1) {
    acc.x += __shfl_xor_sync(0xffffffffu, acc.x, sh);
    acc.y += __shfl_xor_sync(0xffffffffu, acc.y, sh);
    acc.z += __shfl_xor_sync(0xffffffffu, acc.z, sh);
    acc.w += __shfl_xor_sync(0xffffffffu, acc.w, sh);
  }
  if (q4 == 0) *reinterpret_cast<float4*>(out + size_t(gid) * D + j * 4) = acc;
}

__global__ void __launch_bounds__(kWideThreads)
msda_bwd_wide_kernel(const float* __restrict__ value, const int64_t* __restrict__ shapes,
                     const float* __restrict__ loc, const float* __restrict__ attn,
                     const float* __restrict__ grad_out, float* __restrict__ grad_value,
                     float* __restrict__ grad_loc, float* __restrict__ grad_attn,
                     int S, int M, int L, int Lq, int P, uint32_t groups) {
  constexpr int D = 32;
  __shared__ LevelTable lv;
  __shared__ unsigned char lvl_of[kMaxLP];
  const int LP = L * P;
  const int stride = M * D;
  const int lane = threadIdx.x & 31;
  const int q4 = lane >> 3, j = lane & 7;
  load_level_table(lv, lvl_of, shapes, L, P);
  __syncthreads();
  const uint32_t gid = blockIdx.x * (kWideThreads / 32) + (threadIdx.x >> 5);
  if (gid >= groups) return;                                   // warp-uniform
  const uint32_t m = gid % uint32_t(M);
  const uint32_t n = gid / (uint32_t(M) * uint32_t(Lq));
  const size_t head = size_t(n) * S * stride + m * D + j * 4;
  const float* vb = value + head;
  float* gvb = grad_value + head;
  const float4 g = ldg4(grad_out + size_t(gid) * D + j * 4);
  const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
  // every 8-lane quarter takes samples q4, q4+4, ...; four of them per butterfly round
  for (int s0 = q4; s0 < LP; s0 += 16) {
    float part[12];
#pragma unroll
    for (int u = 0; u < 4; ++u) {
      const int s = s0 + 4 * u;
      float s_a = 0.f, s_x = 0.f, s_y = 0.f;
      if (s < LP) {
        const int l = lvl_of[s];
        const int H = lv.H[l], W = lv.W[l];
        const size_t sidx = size_t(gid) * LP + s;
        const float2 xy = __ldg(reinterpret_cast<const float2*>(loc) + sidx);
        const float a = __ldg(attn + sidx);
        const Tap<float> t = make_tap<float>(xy.x, xy.y, H, W, stride);
        if (t.live) {
          const size_t lofs = size_t(lv.start[l]) * stride;
          const float4 v1 = t.k1 ? ldg4(vb + lofs + t.o1) : z, v2 = t.k2 ? ldg4(vb + lofs + t.o2) : z;
          const float4 v3 = t.k3 ? ldg4(vb + lofs + t.o3) : z, v4 = t.k4 ? ldg4(vb + lofs + t.o4) : z;
          const float hx = 1.f - t.lx, hy = 1.f - t.ly;
          const float4 top = lin2(hx, v1, t.lx, v2), bot = lin2(hx, v3, t.lx, v4);
          const float4 dtop = lin2(-1.f, v1, 1.f, v2), dbot = lin2(-1.f, v3, 1.f, v4);
          s_a = dot4(g, lin2(hy, top, t.ly, bot));
          s_x = dot4(g, lin2(hy, dtop, t.ly, dbot)) * a * float(W);
          s_y = dot4(g, lin2(-1.f, top, 1.f, bot)) * a * float(H);
          const float k1 = t.w1 * a, k2 = t.w2 * a, k3 = t.w3 * a, k4 = t.w4 * a;
          if (t.k1 && k1 != 0.f) red4(gvb + lofs + t.o1, k1, g);
          if (t.k2 && k2 != 0.f) red4(gvb + lofs + t.o2, k2, g);
          if (t.k3 && k3 != 0.f) red4(gvb + lofs + t.o3, k3, g);
          if (t.k4 && k4 != 0.f) red4(gvb + lofs + t.o4, k4, g);
        }
      }
      part[3 * u + 0] = s_a;
      part[3 * u + 1] = s_x;
      part[3 * u + 2] = s_y;
    }
    float r6[6], r3[3];
    {
      const bool hi = j & 4;
#pragma unroll
      for (int c = 0; c < 6; ++c) {
        const float mine = hi ? part[6 + c] : part[c];
        const float give = hi ? part[c] : part[6 + c];
        r6[c] = mine + __shfl_xor_sync(0xffffffffu, give, 4);
      }
    }
    {
      const bool hi = j & 2;
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        const float mine = hi ? r6[3 + c] : r6[c];
        const float give = hi ? r6[c] : r6[3 + c];
        r3[c] = mine + __shfl_xor_sync(0xffffffffu, give, 2);
      }
    }
#pragma unroll
    for (int c = 0; c < 3; ++c) r3[c] += __shfl_xor_sync(0xffffffffu, r3[c], 1);
    const int s = s0 + 4 * (j >> 1);
    if (!(j & 1) && s < LP) {
      const size_t sidx = size_t(gid) * LP + s;
      grad_attn[sidx] = r3[0];
      *reinterpret_cast<float2*>(grad_loc + 2 * sidx) = make_float2(r3[1], r3[2]);
    }
  }
}

}  // namespace msda
