// Encoder self-attention (queries == pixels, raster order) with TMA-staged value tiles -- fp32, D = 32, P = 4, L <= 4.
//
// Reference semantics: ms_deform_im2col_cuda.cuh:165-237 (forward sampling kernel) -- identical taps, weights and zero
// padding; only the data movement differs.
//
// What the measurements of the direct kernels say : a C2 encoder call gathers 11.4 M corner
// rows of 128 bytes (1.46 GB, 18x the compulsory bytes).  Through L1 a row costs ~2 cycles of the data stage no matter
// how the request is shaped (92 us); cutting the rows with register-resident windows (msda_run*.cuh) made the direct
// kernels latency bound instead (one window load per group in flight, L2 latency, little L1 left beside 41-49 KB of
// tap tables per CTA).  Shared memory serves a 128-byte row per cycle at ~30 cycles latency, and in the encoder the rows
// a tile of neighbouring queries needs form a compact box per level.  So:
//
//   * CTA = 16 x 8 tile of queries of one level x ONE head (8 warps; warp = two tile rows x two of a level's four
//     sample slots; 8-lane group = run of 8 consecutive queries; the two warp sets' partial sums meet in shared memory).  One cooperative pass turns the tile's 2 048 samples into taps and reduces the EXACT lower
//     corner of their windows per level (REDUX.MIN + shared-memory atomicMin).
//   * The box [corner, corner + (16 >> d) + 7) x [.., (8 >> d) + 7) of sample level l = lq + d is fetched by ONE TMA
//     instruction (cp.async.bulk.tensor.5d over value viewed as [N][H_l][W_l][M][32], zero fill outside the level) into
//     one of two shared-memory buffers; levels lq and lq+1 are in flight while the plan pass runs, level l+2 is
//     issued as soon as level l has been gathered (mbarrier completion, no thread ever waits for a load it issued).
//   * PLAN pass + hot loop as in msda_run2.cuh (window state machine run once per chain, weights stored in register-set
//     order, FFMA2), but the window rows are 16-bit row indices into the staged box and the loads are LDS.128:
//     ~0.3 rows per (query, sample, corner) at one row per cycle.
//   * Nothing is assumed about where samples fall.  A tap whose window is not inside its level's box (wide trained
//     offsets, random locations) and every tap on a level FINER than the tile's own level (footprint 2-8x the tile) is
//     flagged in a per-query bit mask and evaluated afterwards straight from global memory with the reference's
//     predicated corners; the results are the same numbers either way.
//
// Needs the level sizes on the HOST (grid = tiles, tensor maps): entry point msda_b200_forward_enc_tiled_f32.
#pragma once

#include <cuda.h>

#include <climits>

#include "msda_run2.cuh"

namespace msda {

constexpr int kEtThreads = 256;                                // 8 warps: two warp sets share a tile, two slots of a level each
constexpr int kEtTX = 16, kEtTY = 8, kEtQ = kEtTX * kEtTY;     // query tile
constexpr int kEtMaxL = 4, kEtP = 4, kEtLP = 16;               // table geometry (L <= 4 levels x 4 points)
constexpr int kEtR = 8;                                        // run length
constexpr int kEtHalo = 7;                                     // 4 points along the head's direction + bilinear + slack
__host__ __device__ constexpr int et_bw(int d) { return (kEtTX >> d) + kEtHalo; }
__host__ __device__ constexpr int et_bh(int d) { return (kEtTY >> d) + kEtHalo; }
constexpr int kEtBuf0Rows = et_bw(0) * et_bh(0);              // 345 rows (d = 0; d = 2 needs 99)
constexpr int kEtBuf1Rows = et_bw(1) * et_bh(1);              // 165 rows (d = 1; d = 3 needs 72)
constexpr int kEtEntries = kEtQ * kEtLP + 16;                 // + one-entry skew per run of 8 queries (bank spread)
constexpr unsigned kEtNone = 0xFFFFFFFFu;                      // tap: dead / far;  after the plan: no load for either set
constexpr size_t kEtSmemBytes = 128 + size_t(kEtBuf0Rows + kEtBuf1Rows) * 128 + size_t(kEtEntries) * (16 + 4) +
                                kEtQ * 4 + 2 * kEtMaxL * 4 + kEtMaxL * 8;

struct EtGeom {
  int L, S, M, Lq;
  int tiles_used;                                             // tiles the grid covers (all, or only those of query level 0)
  int H[kEtMaxL], W[kEtMaxL], start[kEtMaxL];
  int tiles_x[kEtMaxL], tile_begin[kEtMaxL + 1];
};
// tensor map of sample level l as seen from a tile of query level lq <= l (the box size depends on l - lq)
__host__ __device__ constexpr int et_map_index(int lq, int l) { return lq * 4 - lq * (lq - 1) / 2 + (l - lq); }
struct EtMaps { CUtensorMap m[10]; };

__device__ __forceinline__ uint32_t et_smem(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }
__device__ __forceinline__ void et_mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void et_mbar_expect(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void et_mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!ok);
}
// box (32 channels, head m, BW pixels from x0, BH pixels from y0, image n) -> dense [BH][BW][32] floats at dst
__device__ __forceinline__ void et_tma_box(uint32_t dst, const CUtensorMap* map, uint32_t bar, int m, int x0, int y0, int n) {
  asm volatile(
      "cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(0), "r"(m), "r"(x0), "r"(y0), "r"(n)
      : "memory");
}
__device__ __forceinline__ void lds2_if(u64& lo, u64& hi, uint32_t addr, bool pred) {
  asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %3, 0;\n\t@p ld.shared.v2.b64 {%0, %1}, [%2];\n\t}"
               : "+l"(lo), "+l"(hi)
               : "r"(addr), "r"(int(pred)));
}

// One level for one warp: NS slots walk the run of R queries together.  GLOBAL = false: window rows are row indices
// into the staged box (LDS.128); GLOBAL = true: element offsets into `value` (levels finer than the tile's own).
// Taps of step r + 1 are requested before the FMAs of step r.
// accumulators per query: (low / high half of the 16-byte pack) x (even / odd slot when a warp walks four slots, so
// that consecutive FFMA2s of a step never depend on each other; with two slots per warp and 16 warps per SM the other
// warps cover the FFMA2 latency and the registers are better spent on occupancy)
__host__ __device__ constexpr int et_nacc(int NS) { return NS == 4 ? 4 : 2; }

template <int NS, bool GLOBAL>
__device__ __forceinline__ void et_level_pass(u64 (&acc)[kEtR][et_nacc(NS)], uint32_t sw_addr, uint32_t so_addr, uint32_t slot0,
                                              uint32_t bufa, uint32_t pitch, const float* vh, unsigned gstride,
                                              unsigned rowpitch) {
  constexpr int R = kEtR;
  u64 A1[NS][2], A3[NS][2], B1[NS][2], B3[NS][2];
#pragma unroll
  for (int p = 0; p < NS; ++p)
    A1[p][0] = A1[p][1] = A3[p][0] = A3[p][1] = B1[p][0] = B1[p][1] = B3[p][0] = B3[p][1] = 0ull;
  float4 wn[NS];
  unsigned on[NS];
  auto taps = [&](int r) {
#pragma unroll
    for (int p = 0; p < NS; ++p) {
      const uint32_t eo = uint32_t(r * kEtLP) + slot0 + uint32_t(p);
      asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
                   : "=f"(wn[p].x), "=f"(wn[p].y), "=f"(wn[p].z), "=f"(wn[p].w)
                   : "r"(sw_addr + eo * 16u));
      asm volatile("ld.shared.b32 %0, [%1];" : "=r"(on[p]) : "r"(so_addr + eo * 4u));
    }
  };
  taps(0);
#pragma unroll
  for (int r = 0; r < R; ++r) {
    float4 w[NS];
    unsigned o[NS];
#pragma unroll
    for (int p = 0; p < NS; ++p) { w[p] = wn[p]; o[p] = on[p]; }
#pragma unroll
    for (int p = 0; p < NS; ++p) {
      if (GLOBAL) {
        const unsigned ob = o[p] & ~7u;
        const bool la = o[p] & 1u, lb = o[p] & 2u;
        const unsigned oa = (o[p] & 4u) ? ob - gstride : ob;
        ldg2_if(A1[p][0], A1[p][1], row_ptr(vh, oa), la);
        ldg2_if(A3[p][0], A3[p][1], row_ptr(vh, oa + rowpitch), la);
        ldg2_if(B1[p][0], B1[p][1], row_ptr(vh, ob), lb);
        ldg2_if(B3[p][0], B3[p][1], row_ptr(vh, ob + rowpitch), lb);
      } else {
        const unsigned oa = o[p] & 0xFFFFu, ob = o[p] >> 16;
        const bool la = oa != 0xFFFFu, lb = ob != 0xFFFFu;
        const uint32_t pa = bufa + oa * 128u, pb = bufa + ob * 128u;
        lds2_if(A1[p][0], A1[p][1], pa, la);
        lds2_if(A3[p][0], A3[p][1], pa + pitch, la);
        lds2_if(B1[p][0], B1[p][1], pb, lb);
        lds2_if(B3[p][0], B3[p][1], pb + pitch, lb);
      }
    }
    if (r + 1 < R) taps(r + 1);
#pragma unroll
    for (int c = 0; c < 4; ++c) {
#pragma unroll
      for (int p = 0; p < NS; ++p) {
        const float wc = c == 0 ? w[p].x : (c == 1 ? w[p].y : (c == 2 ? w[p].z : w[p].w));
        const u64* v = c == 0 ? A1[p] : (c == 1 ? B1[p] : (c == 2 ? A3[p] : B3[p]));
        constexpr int kSplit = et_nacc(NS) == 4 ? 2 : 0;
        ffma2(acc[r][kSplit * (p & 1)], wc, v[0]);
        ffma2(acc[r][kSplit * (p & 1) + 1], wc, v[1]);
      }
    }
  }
}

// One sample's (normalised location, attention weight) from the module's raw projection, evaluated by a single thread
// (far path of the fused-prologue kernels; the tap pass uses run_sample<true, 16>, one lane per slot).
//   proj row [n, q]: [M][16][2] offsets, then [M][16] logits;  ref [n, q][L][2];  loc = ref + offset / (H, W) as stored.
__device__ __forceinline__ void prep_sample_serial(const float* __restrict__ proj, const float* __restrict__ ref, size_t nq,
                                                   int m, int s, int l, int M, int L, int H, int W, float& x, float& y,
                                                   float& a) {
  const float* prow = proj + nq * size_t(3 * M * 16);
  const float* lg = prow + 2 * M * 16 + m * 16;
  float v[16], mx = -INFINITY, sum = 0.f;
#pragma unroll
  for (int i = 0; i < 16; i += 4) {
    const float4 t = __ldg(reinterpret_cast<const float4*>(lg + i));
    v[i] = t.x; v[i + 1] = t.y; v[i + 2] = t.z; v[i + 3] = t.w;
  }
#pragma unroll
  for (int i = 0; i < 16; ++i) mx = fmaxf(mx, v[i]);
  float mine = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    const float e = expf(v[i] - mx);
    sum += e;
    if (i == s) mine = e;
  }
  a = mine / sum;
  const float2 off = __ldg(reinterpret_cast<const float2*>(prow) + m * 16 + s);
  const float2 r = __ldg(reinterpret_cast<const float2*>(ref) + nq * L + l);
  x = r.x + off.x / float(H);
  y = r.y + off.y / float(W);
}

// PREP = true (module-level fusion, ops/modules/ms_deform_attn.py:69-87 inside the kernel): `loc` is the raw output of
// the [sampling_offsets | attention_weights] projections and `attn` the reference points; sampling locations and softmax
// weights are computed in the tap pass and never materialised.  Needs L * P == 16.
template <int NS, bool PREP = false>
__global__ void __launch_bounds__(512 / NS, 2)
msda_fwd_enc_tma_kernel(const float* __restrict__ value, const float* __restrict__ loc, const float* __restrict__ attn,
                        float* __restrict__ out, const __grid_constant__ EtGeom g, const __grid_constant__ EtMaps maps) {
  constexpr int D = 32, R = kEtR;
  constexpr int WS = 4 / NS;                                  // warp sets: each takes NS of a level's 4 slots
  constexpr int T = 128 * WS;                                 // threads
  extern __shared__ unsigned char et_smem_raw[];
  unsigned char* base = et_smem_raw + ((128u - (et_smem(et_smem_raw) & 127u)) & 127u);       // TMA destinations: 128-byte aligned
  float* buf0 = reinterpret_cast<float*>(base);
  float* buf1 = buf0 + kEtBuf0Rows * D;
  float4* s_w = reinterpret_cast<float4*>(buf1 + kEtBuf1Rows * D);
  unsigned* s_o = reinterpret_cast<unsigned*>(s_w + kEtEntries);
  unsigned* s_far = s_o + kEtEntries;                       // [128] per-query mask of the slots evaluated from global memory
  int* s_box = reinterpret_cast<int*>(s_far + kEtQ);        // [L][2] lower corner (x, y) of the windows of level l
  unsigned long long* s_bar = reinterpret_cast<unsigned long long*>(s_box + 2 * kEtMaxL);    // [L] one-shot barriers

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int wset = warp >> 2, wq = warp & 3;                // warp set (slots), warp within the set (tile rows)
  const int k = lane >> 3, j = lane & 7;
  const int L = g.L, M = g.M, Lq = g.Lq, LPr = L * kEtP;
  const int stride = M * D;

  // ---- which head / tile / image
  const int tiles = g.tiles_used;
  const int m = blockIdx.x % M;
  const int t = tiles - 1 - int((blockIdx.x / M) % tiles);     // coarse query levels (the longest CTAs) first
  const int n = blockIdx.x / (M * tiles);
  int lq = 0;
#pragma unroll
  for (int l = 1; l < kEtMaxL; ++l)
    if (l < L && t >= g.tile_begin[l]) lq = l;
  const int tt = t - g.tile_begin[lq];
  const int ty = tt / g.tiles_x[lq], tx = tt - ty * g.tiles_x[lq];
  const int Wq = g.W[lq], Hq = g.H[lq];
  const int x0 = tx * kEtTX, y0 = ty * kEtTY;
  const int qbase = g.start[lq] + y0 * Wq + x0;            // query (iy, ix) of the tile = qbase + iy * Wq + ix

  if (tid < 2 * kEtMaxL) s_box[tid] = INT_MAX;
  if (tid < kEtMaxL) et_mbar_init(et_smem(s_bar + tid), 1);
  if (tid == 0) asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  if (tid < kEtQ) s_far[tid] = 0u;
  __syncthreads();

  // ---- phase 1: taps.  Thread -> slot s = tid % 16 (fixed), queries qi = tid / 16 + (T / 16) * it.
  {
    constexpr int NIT = kEtQ * 16 / T;
    const int s = tid & 15, l = s >> 2;
    const bool slot_ok = s < LPr;
    const int Hl = slot_ok ? g.H[l] : 2, Wl = slot_ok ? g.W[l] : 2;
    int mnx = INT_MAX, mny = INT_MAX;
    // all samples of the thread are requested before the first one is used: one HBM round trip per CTA instead of one
    // per sample (ncu, first version: 61 % of the kernel's stall samples sat on the first use of these loads)
    float2 xy[NIT], rf[PREP ? NIT : 1];
    float at[NIT];
    const size_t srow = size_t(M) * LPr;                      // floats of attn per query
#pragma unroll
    for (int it = 0; it < NIT; ++it) {
      const int qi = (tid >> 4) + (T / 16) * it;
      const int ix = qi & 15, iy = qi >> 4;
      const bool valid = slot_ok && (x0 + ix < Wq) && (y0 + iy < Hq);
      if (PREP) {
        // raw projection: offset pair and logit of (head m, slot s); reference point of (query, level)
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
      unsigned code = kEtNone;
      float a = at[it];
      float lx = xy[it].x, ly = xy[it].y;
      if (PREP) {
        // softmax over the head's 16 logits (16 consecutive lanes), location = reference + offset / (H, W) as stored
        float mx = a;
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        const float e = expf(a - mx);
        float sum = e;
#pragma unroll
        for (int o = 8; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
        a = e / sum;
        const int ix = qi & 15, iy = qi >> 4;
        const bool valid = (x0 + ix < Wq) && (y0 + iy < Hq);
        lx = valid ? rf[it].x + lx / float(Hl) : -8.f;
        ly = valid ? rf[it].y + ly / float(Wl) : -8.f;
      }
      const float x = lx * float(Wl) - 0.5f, y = ly * float(Hl) - 0.5f;                 // invalid queries: far outside
      if (y > -1.f && x > -1.f && y < float(Hl) && x < float(Wl)) {
        int xb, yb;
        float wxa, wxb, wya, wyb, d0, d1;
        axis_window(x, Wl, xb, wxa, wxb, d0, d1);
        axis_window(y, Hl, yb, wya, wyb, d0, d1);
        w = make_float4(wya * wxa * a, wya * wxb * a, wyb * wxa * a, wyb * wxb * a);
        if (l < lq) {
          // finer level than the tile's own (footprint 2-8x the tile): gathered from global memory by the same
          // run machinery; the tap is the element offset of the window's first corner (a multiple of M * 32)
          code = unsigned(g.start[l] + yb * Wl + xb) * unsigned(stride);
        } else {
          code = unsigned(xb) | (unsigned(yb) << 16);
          mnx = min(mnx, xb);
          mny = min(mny, yb);
        }
      }
      const int e = qi * kEtLP + s + (qi >> 3);
      s_w[e] = w;
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

  // ---- the first two staged levels go in flight; the plan pass below runs under them
  auto issue = [&](int l) {
    const int d = l - lq;
    const int bx = s_box[2 * l], by = s_box[2 * l + 1];
    if (bx == INT_MAX) return;                               // no live sample on this level: nothing will read the buffer
    const uint32_t bar = et_smem(s_bar + l);
    et_mbar_expect(bar, uint32_t(et_bw(d) * et_bh(d) * 128));
    et_tma_box(et_smem((d & 1) ? buf1 : buf0), &maps.m[et_map_index(lq, l)], bar, m, bx, by, n);
  };
  if (tid == 0) {
    issue(lq);
    if (lq + 1 < L) issue(lq + 1);
  }

  // ---- phase 2 (plan): one thread per (run of 8 queries, slot) chain (256 chains); with 128 threads a thread owns two
  //      chains (same slot, runs 8 apart) and walks them in lockstep so that their shared-memory round trips overlap
  {
    constexpr int NCH = 256 / T;
    const int s = tid & 15, l = s >> 2;
    if (s < LPr) {
      const bool glob = l < lq;                               // finer level than the tile's own: global-memory taps
      const int d = glob ? 0 : l - lq;
      const int BW = et_bw(d), BH = et_bh(d);
      const int bx = glob ? 0 : s_box[2 * l], by = glob ? 0 : s_box[2 * l + 1];
      const unsigned step = glob ? unsigned(stride) : 1u;     // offset of the right-hand neighbour
      unsigned co[NCH];
      bool have[NCH], par[NCH];
#pragma unroll
      for (int h = 0; h < NCH; ++h) { co[h] = 0u; have[h] = false; par[h] = false; }
#pragma unroll
      for (int r = 0; r < R; ++r) {
#pragma unroll
        for (int h = 0; h < NCH; ++h) {
          const int run = (tid >> 4) + (T / 16) * h;
          const int qi = (run >> 1) * kEtTX + (run & 1) * R + r;
          const int e = qi * kEtLP + s + run;
          const unsigned code = s_o[e];
          unsigned o = code;
          bool live = code != kEtNone;
          if (live && !glob) {
            const int rx = int(code & 0xFFFFu) - bx, ry = int(code >> 16) - by;
            o = unsigned(ry * BW + rx);
            if (rx > BW - 2 || ry > BH - 2) {                 // window not inside the staged box
              atomicOr(&s_far[qi], 1u << s);
              s_w[e] = make_float4(0.f, 0.f, 0.f, 0.f);
              live = false;
            }
          }
          if (!live) {                                        // dead / far sample: zero weights, no load, window untouched
            s_o[e] = glob ? 0u : kEtNone;
            continue;
          }
          const float4 w = s_w[e];
          const bool same = have[h] && (o == co[h]);
          const bool shift = have[h] && (o == co[h] + step);
          const bool reload = !(same || shift);
          const bool ldA = reload || (shift && !par[h]);
          const bool ldB = reload || (shift && par[h]);
          par[h] = reload ? false : (par[h] != shift);
          co[h] = o;
          have[h] = true;
          s_w[e] = par[h] ? make_float4(w.y, w.x, w.w, w.z) : w;
          if (glob) {
            // (element offset of the NEW right column) | load A | load B << 1 | reload << 2
            s_o[e] = (o + step) | unsigned(ldA) | (unsigned(ldB) << 1) | (unsigned(reload) << 2);
          } else {
            const unsigned oa = ldA ? (reload ? o : o + 1u) : 0xFFFFu;
            const unsigned ob = ldB ? o + 1u : 0xFFFFu;
            s_o[e] = oa | (ob << 16);
          }
        }
      }
    }
  }
  __syncthreads();

  // ---- hot loops
  const int row_t = 2 * wq + (k >> 1);                       // tile row of this group
  const int run_g = 2 * row_t + (k & 1);                     // run index (= skew of its entries)
  const int e0 = (row_t * kEtTX + (k & 1) * R) * kEtLP + run_g;
  const uint32_t sw_addr = et_smem(s_w + e0), so_addr = et_smem(s_o + e0);
  const uint32_t lane_off = uint32_t(j) * 16u;
  const float* vh = value + size_t(n) * g.S * stride + m * D + j * 4;

  constexpr int NACC = et_nacc(NS);
  u64 acc[R][NACC];
#pragma unroll
  for (int r = 0; r < R; ++r)
#pragma unroll
    for (int c = 0; c < NACC; ++c) acc[r][c] = 0ull;
  auto total = [&](int r) {                                   // sum of the query's partial accumulators
    float4 e = unpack4(acc[r][0], acc[r][1]);
    if (NACC == 4) {
      const float4 o = unpack4(acc[r][2], acc[r][3]);
      e.x += o.x; e.y += o.y; e.z += o.z; e.w += o.w;
    }
    return e;
  };

  // levels finer than the tile's own: the same walk, window rows straight from global memory
#pragma unroll 1
  for (int l = 0; l < lq; ++l)
    et_level_pass<NS, true>(acc, sw_addr, so_addr, uint32_t(l * kEtP + wset * NS), 0u, 0u, vh, unsigned(stride),
                            unsigned(g.W[l]) * unsigned(stride));

#pragma unroll 1
  for (int l = lq; l < L; ++l) {
    const int d = l - lq;
    if (s_box[2 * l] != INT_MAX) {                            // uniform
      et_mbar_wait(et_smem(s_bar + l), 0);
      et_level_pass<NS, false>(acc, sw_addr, so_addr, uint32_t(l * kEtP + wset * NS),
                               et_smem((d & 1) ? buf1 : buf0) + lane_off, uint32_t(et_bw(d)) * 128u, nullptr, 0u, 0u);
    }
    if (l + 2 < L) {                                          // this level's buffer is free: fetch level l + 2 into it
      __syncthreads();
      if (tid == 0) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        issue(l + 2);
      }
    }
  }

  // ---- samples flagged "far": straight from global memory, the reference's predicated corners; two at a time so that
  //      their dependent load chains (location -> corner rows) overlap.  Each warp set takes the bits of its own slots.
  constexpr unsigned kSetMask = NS == 4 ? 0xFFFFu : 0x3333u;
#pragma unroll                                              // (unrolled: acc[] must stay in registers)
  for (int r = 0; r < R; ++r) {
    const int ix = (k & 1) * R + r;
    unsigned fm = s_far[row_t * kEtTX + ix] & (kSetMask << (wset * NS));
    if (fm == 0u) continue;
    const size_t qidx = size_t(n) * Lq + qbase + row_t * Wq + ix;
    float4 av = unpack4(acc[r][0], acc[r][1]);
    while (fm) {
      int sl[2];
      float2 xy[2];
      float a[2];
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        sl[u] = fm ? __ffs(int(fm)) - 1 : -1;
        fm &= fm - 1;                                         // (0 stays 0)
        const int su = sl[u] < 0 ? 0 : sl[u];
        if (PREP) {
          prep_sample_serial(loc, attn, qidx, m, su, su >> 2, M, L, g.H[su >> 2], g.W[su >> 2], xy[u].x, xy[u].y, a[u]);
          if (sl[u] < 0) a[u] = 0.f;
        } else {
          const size_t sidx = (qidx * M + m) * LPr + su;
          xy[u] = __ldg(reinterpret_cast<const float2*>(loc) + sidx);
          a[u] = sl[u] < 0 ? 0.f : __ldg(attn + sidx);
        }
      }
      Tap<float> tp[2];
      float4 v[2][4];
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        const int l = (sl[u] < 0 ? 0 : sl[u]) >> 2;
        tp[u] = make_tap<float>(xy[u].x, xy[u].y, g.H[l], g.W[l], stride);
        const float* vl = vh + size_t(g.start[l]) * stride;
        const bool on = tp[u].live && sl[u] >= 0;
        v[u][0] = (on && tp[u].k1) ? ldg4(vl + tp[u].o1) : z;
        v[u][1] = (on && tp[u].k2) ? ldg4(vl + tp[u].o2) : z;
        v[u][2] = (on && tp[u].k3) ? ldg4(vl + tp[u].o3) : z;
        v[u][3] = (on && tp[u].k4) ? ldg4(vl + tp[u].o4) : z;
      }
#pragma unroll
      for (int u = 0; u < 2; ++u) {
        fma4(av, tp[u].w1 * a[u], v[u][0]);
        fma4(av, tp[u].w2 * a[u], v[u][1]);
        fma4(av, tp[u].w3 * a[u], v[u][2]);
        fma4(av, tp[u].w4 * a[u], v[u][3]);
      }
    }
    pack4(av, acc[r][0], acc[r][1]);
  }

  // ---- combine the warp sets' partial sums (through shared memory, over the first value buffer) and store
  if (WS == 2) {
    __syncthreads();                                          // every warp is done with the value buffers
    float4* comb = reinterpret_cast<float4*>(buf0);           // [128 queries][8 lanes]
    if (wset == 1) {
#pragma unroll
      for (int r = 0; r < R; ++r) {
        comb[(row_t * kEtTX + (k & 1) * R + r) * 8 + j] = total(r);
      }
    }
    __syncthreads();
    if (wset == 1) return;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const float4 c = comb[(row_t * kEtTX + (k & 1) * R + r) * 8 + j];
      float4 e = unpack4(acc[r][0], acc[r][1]);
      e.x += c.x; e.y += c.y; e.z += c.z; e.w += c.w;
      pack4(e, acc[r][0], acc[r][1]);
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) {
    const int ix = (k & 1) * R + r;
    if (x0 + ix < Wq && y0 + row_t < Hq) {
      float* dst = out + ((size_t(n) * Lq + qbase + row_t * Wq + ix) * M + m) * D + j * 4;
      *reinterpret_cast<float4*>(dst) = total(r);
    }
  }
}

}  // namespace msda
