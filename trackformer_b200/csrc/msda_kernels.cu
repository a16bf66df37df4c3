// libmsda_b200: hand-written sm_90a kernels for multi-scale deformable attention
// (forward + fused backward) behind the C ABI declared in include/msda_b200.h.
//
// Replaces the reference's three kernels + host wrappers
//   ms_deformable_im2col_gpu_kernel        ms_deform_im2col_cuda.cuh:165-237  (+ at::sum, ms_deform_attn_cuda.cu:80)
//   ms_deformable_col2im_gpu_kernel        ms_deform_im2col_cuda.cuh:239-306
//   ms_deformable_col2im_coord_gpu_kernel  ms_deform_im2col_cuda.cuh:308-378
// with ONE forward kernel (no L*P-times inflated `columns` tensor, no separate reduction,
// level starts derived in-kernel) and ONE backward kernel (corners are read once and feed
// grad_value, grad_sampling_loc and grad_attn_weight together).
//
// Work decomposition ("group" = one (n, q, m) triple = one head of one query):
//   * G lanes of a warp own a group; lane j owns channel packs j, j+G, ... (ITERS of them),
//     each pack = VEC contiguous channels = 16 bytes when the layout allows.  For the shipped
//     geometry (fp32, D=32) G=8, VEC=4: the 8 lanes of a group read one full 128-byte row of
//     `value` per bilinear corner -> every warp-level load touches exactly 4 full L1 lines.
//   * groups are numbered n-major, then q, then m, i.e. exactly the memory order of
//     sampling_loc / attn_weight / output, so those streams are read/written fully coalesced.
//   * backward: per-sample partial dot products are reduced over the G lanes with
//     warp shuffles; grad_value uses 128-bit vector reductions (red.global.add.v4.f32).
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>
#include <mutex>

#include "../../include/msda_b200.h"
#include "launch_counter.h"
#include "msda_common.cuh"
#include "msda_d32.cuh"
#include "msda_d36.cuh"
#include "msda_run2.cuh"
#include "msda_enc_tma_bwd.cuh"
#include "tma_host.h"

namespace msda {

static std::atomic<uint64_t> g_launches{0};
static std::atomic<int> g_fwd_variant{0};
static std::atomic<int> g_bwd_variant{0};

constexpr int kThreads = 256;

// ------------------------------------------------------------------------------------
// Forward: out[n,q,m,:] = sum_{l,p} attn * bilinear(value_l, loc)
// ------------------------------------------------------------------------------------
template <typename T, int VEC, int G, int ITERS>
__global__ void __launch_bounds__(kThreads)
msda_fwd_kernel(const T* __restrict__ value, const int64_t* __restrict__ shapes,
                const T* __restrict__ loc, const T* __restrict__ attn, T* __restrict__ out,
                int S, int M, int D, int L, int Lq, int P, int64_t groups) {
  const int64_t gid_raw = (int64_t(blockIdx.x) * kThreads + threadIdx.x) / G;
  const int lane = threadIdx.x % G;
  const bool active = gid_raw < groups;
  const int64_t gid = active ? gid_raw : groups - 1;

  const int m = int(gid % M);
  const int64_t n = gid / (int64_t(M) * Lq);
  const int stride = M * D;
  const int npacks = D / VEC;

  const T* vhead = value + n * int64_t(S) * stride + m * D;
  const T* lp = loc + gid * (int64_t(L) * P * 2);
  const T* ap = attn + gid * (int64_t(L) * P);

  Pack<T, VEC> acc[ITERS];
#pragma unroll
  for (int i = 0; i < ITERS; ++i) acc[i] = pack_zero<T, VEC>();

  int64_t start = 0;
  for (int l = 0; l < L; ++l) {
    const int H = int(__ldg(shapes + 2 * l));
    const int W = int(__ldg(shapes + 2 * l + 1));
    const T* vl = vhead + start * stride;
    start += int64_t(H) * W;
    for (int p = 0; p < P; ++p) {
      const T lx = __ldg(lp), ly = __ldg(lp + 1), a = __ldg(ap);
      lp += 2;
      ap += 1;
      const Tap<T> t = make_tap<T>(lx, ly, H, W, stride);
      if (!t.live) continue;
      const T a1 = t.w1 * a, a2 = t.w2 * a, a3 = t.w3 * a, a4 = t.w4 * a;
#pragma unroll
      for (int i = 0; i < ITERS; ++i) {
        const int pk = lane + i * G;
        if (pk >= npacks) break;
        const int co = pk * VEC;
        const Pack<T, VEC> v1 = t.k1 ? ldg_pack<T, VEC>(vl + t.o1 + co) : pack_zero<T, VEC>();
        const Pack<T, VEC> v2 = t.k2 ? ldg_pack<T, VEC>(vl + t.o2 + co) : pack_zero<T, VEC>();
        const Pack<T, VEC> v3 = t.k3 ? ldg_pack<T, VEC>(vl + t.o3 + co) : pack_zero<T, VEC>();
        const Pack<T, VEC> v4 = t.k4 ? ldg_pack<T, VEC>(vl + t.o4 + co) : pack_zero<T, VEC>();
#pragma unroll
        for (int c = 0; c < VEC; ++c)
          acc[i].v[c] += a1 * v1.v[c] + a2 * v2.v[c] + a3 * v3.v[c] + a4 * v4.v[c];
      }
    }
  }
  if (active) {
    T* o = out + gid * D;
#pragma unroll
    for (int i = 0; i < ITERS; ++i) {
      const int pk = lane + i * G;
      if (pk < npacks) st_pack<T, VEC>(o + pk * VEC, acc[i]);
    }
  }
}

// ------------------------------------------------------------------------------------
// Backward (fused): grad_value (vector reductions), grad_sampling_loc, grad_attn_weight
// ------------------------------------------------------------------------------------
template <typename T, int G>
__device__ __forceinline__ T group_sum(T v) {
#pragma unroll
  for (int o = G / 2; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

template <typename T, int VEC, int G, int ITERS>
__global__ void __launch_bounds__(kThreads)
msda_bwd_kernel(const T* __restrict__ value, const int64_t* __restrict__ shapes,
                const T* __restrict__ loc, const T* __restrict__ attn,
                const T* __restrict__ grad_out, T* __restrict__ grad_value,
                T* __restrict__ grad_loc, T* __restrict__ grad_attn,
                int S, int M, int D, int L, int Lq, int P, int64_t groups) {
  const int64_t gid_raw = (int64_t(blockIdx.x) * kThreads + threadIdx.x) / G;
  const int lane = threadIdx.x % G;
  const bool active = gid_raw < groups;
  const int64_t gid = active ? gid_raw : groups - 1;

  const int m = int(gid % M);
  const int64_t n = gid / (int64_t(M) * Lq);
  const int stride = M * D;
  const int npacks = D / VEC;

  const int64_t head_ofs = n * int64_t(S) * stride + m * D;
  const T* vhead = value + head_ofs;
  T* gvhead = grad_value + head_ofs;
  const int64_t sbase = gid * (int64_t(L) * P);
  const T* lp = loc + sbase * 2;
  const T* ap = attn + sbase;
  T* glp = grad_loc + sbase * 2;
  T* gap = grad_attn + sbase;

  Pack<T, VEC> g[ITERS];
#pragma unroll
  for (int i = 0; i < ITERS; ++i) {
    const int pk = lane + i * G;
    g[i] = (active && pk < npacks) ? ldg_pack<T, VEC>(grad_out + gid * D + pk * VEC)
                                   : pack_zero<T, VEC>();
  }

  int64_t start = 0;
  for (int l = 0; l < L; ++l) {
    const int H = int(__ldg(shapes + 2 * l));
    const int W = int(__ldg(shapes + 2 * l + 1));
    const int64_t lofs = start * stride;
    start += int64_t(H) * W;
    for (int p = 0; p < P; ++p) {
      const T lx = __ldg(lp), ly = __ldg(lp + 1), a = __ldg(ap);
      const Tap<T> t = make_tap<T>(lx, ly, H, W, stride);
      T s_a = T(0), s_x = T(0), s_y = T(0);
      if (t.live) {  // uniform across the G lanes of a group
        const T hx = T(1) - t.lx, hy = T(1) - t.ly;
        const T a1 = t.w1 * a, a2 = t.w2 * a, a3 = t.w3 * a, a4 = t.w4 * a;
#pragma unroll
        for (int i = 0; i < ITERS; ++i) {
          const int pk = lane + i * G;
          if (pk >= npacks) break;
          const int co = pk * VEC;
          const T* vl = vhead + lofs + co;
          const Pack<T, VEC> v1 = t.k1 ? ldg_pack<T, VEC>(vl + t.o1) : pack_zero<T, VEC>();
          const Pack<T, VEC> v2 = t.k2 ? ldg_pack<T, VEC>(vl + t.o2) : pack_zero<T, VEC>();
          const Pack<T, VEC> v3 = t.k3 ? ldg_pack<T, VEC>(vl + t.o3) : pack_zero<T, VEC>();
          const Pack<T, VEC> v4 = t.k4 ? ldg_pack<T, VEC>(vl + t.o4) : pack_zero<T, VEC>();
          Pack<T, VEC> r1, r2, r3, r4;
#pragma unroll
          for (int c = 0; c < VEC; ++c) {
            const T gc = g[i].v[c];
            s_a += gc * (t.w1 * v1.v[c] + t.w2 * v2.v[c] + t.w3 * v3.v[c] + t.w4 * v4.v[c]);
            s_x += gc * (hy * (v2.v[c] - v1.v[c]) + t.ly * (v4.v[c] - v3.v[c]));
            s_y += gc * (hx * (v3.v[c] - v1.v[c]) + t.lx * (v4.v[c] - v2.v[c]));
            r1.v[c] = a1 * gc;
            r2.v[c] = a2 * gc;
            r3.v[c] = a3 * gc;
            r4.v[c] = a4 * gc;
          }
          if (active) {
            T* gl = gvhead + lofs + co;
            if (t.k1) red_add_pack<T, VEC>(gl + t.o1, r1);
            if (t.k2) red_add_pack<T, VEC>(gl + t.o2, r2);
            if (t.k3) red_add_pack<T, VEC>(gl + t.o3, r3);
            if (t.k4) red_add_pack<T, VEC>(gl + t.o4, r4);
          }
        }
      }
      s_a = group_sum<T, G>(s_a);
      s_x = group_sum<T, G>(s_x);
      s_y = group_sum<T, G>(s_y);
      if (active && lane == 0) {
        gap[0] = s_a;
        glp[0] = s_x * a * T(W);
        glp[1] = s_y * a * T(H);
      }
      lp += 2;
      ap += 1;
      glp += 2;
      gap += 1;
    }
  }
}

// ------------------------------------------------------------------------------------
// Host side: dispatch on (VEC, G, ITERS), launch, error reporting
// ------------------------------------------------------------------------------------
struct Dims {
  int N, S, M, D, L, Lq, P;
};

static int check_dims(const Dims& d) {
  if (d.N < 0 || d.Lq < 0 || d.S <= 0 || d.M <= 0 || d.D <= 0 || d.L <= 0 || d.P <= 0)
    return MSDA_E_DIMS;
  if (d.L > MSDA_B200_MAX_LEVELS) return MSDA_E_LEVELS;
  if (int64_t(d.S) * d.M * d.D > int64_t(INT32_MAX)) return MSDA_E_TOO_LARGE;
  return 0;
}

template <typename T>
static bool aligned16(const T* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// Opts `kernel` in to `bytes` of dynamic shared memory when that exceeds the 48 KB default (the attribute is sticky,
// so it is raised at most a few times per kernel over the life of the process).
template <typename K>
static cudaError_t ensure_dyn_smem(K kernel, size_t bytes, std::atomic<size_t>& granted) {
  if (bytes <= 48 * 1024 || bytes <= granted.load(std::memory_order_relaxed)) return cudaSuccess;
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes));
  if (e == cudaSuccess) granted.store(bytes, std::memory_order_relaxed);
  return e;
}
#define MSDA_ENSURE_SMEM(kernel, bytes)                                         \
  do {                                                                          \
    static std::atomic<size_t> granted__{0};                                    \
    cudaError_t e__ = ensure_dyn_smem(kernel, bytes, granted__);                \
    if (e__ != cudaSuccess) return int(e__);                                    \
  } while (0)

// Which specialised fp32 / D = 32 kernel family serves a problem (variant 0 = automatic):
//   run  : large query sets (encoder) -- register-resident sliding windows over runs of consecutive queries
//   wide : small query sets (decoder) -- one warp per (n, q, m) group
//   d32  : everything in between (and M % 4 != 0): one 8-lane group per (n, q, m), tap tables in shared memory
enum class Family { kD32, kRun8, kRun4, kRun2, kWide };
static Family pick_family(int variant, int64_t groups, const struct Dims& d);

#define MSDA_LAUNCH_FWD(VEC_, G_, IT_)                                                       \
  msda_fwd_kernel<T, VEC_, G_, IT_><<<grid_for(G_), kThreads, 0, st>>>(                      \
      value, shapes, loc, attn, out, d.S, d.M, d.D, d.L, d.Lq, d.P, groups)
#define MSDA_LAUNCH_BWD(VEC_, G_, IT_)                                                       \
  msda_bwd_kernel<T, VEC_, G_, IT_><<<grid_for(G_), kThreads, 0, st>>>(                      \
      value, shapes, loc, attn, gout, gval, gloc, gattn, d.S, d.M, d.D, d.L, d.Lq, d.P, groups)

// Strip length (iterations of 32 groups) per CTA for the d32 kernels: keep at least ~2 waves of CTAs in
// flight on the device's SMs (132 on an H100 SXM), but let big problems walk contiguous strips so neighbouring queries share L1 lines.
static int pick_iters(int64_t ctas) {
  static std::atomic<int> sms{0};
  int n = sms.load(std::memory_order_relaxed);
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
      n = 132;
    sms.store(n, std::memory_order_relaxed);
  }
  const int64_t two_waves = int64_t(n) * 8 * 2;
  int it = int(ctas / two_waves);
  return it < 1 ? 1 : (it > 8 ? 8 : it);
}

// Picks lanes-per-group G and packs-per-lane ITERS for `npacks` 16-byte packs per head.
static void pick_shape(int npacks, int* G, int* iters) {
  int g = 1;
  while (g < 8 && g < npacks) g <<= 1;           // 1,2,4,8
  if (npacks == 9) g = 4;                        // D=36 fp32: 3 iterations at 75% lane use beats 2 at 56%
  *G = g;
  *iters = (npacks + g - 1) / g;
}

static Family pick_family(int variant, int64_t groups, const Dims& d) {
  const bool run_ok = (d.M % kRunHeads == 0);
  if (variant == 100) return run_ok ? Family::kRun8 : Family::kD32;
  if (variant == 101) return run_ok ? Family::kRun4 : Family::kD32;
  if (variant == 120 || variant == 121) return run_ok ? Family::kRun2 : Family::kD32;
  if (variant == 110) return Family::kWide;
  if (variant != 0) return Family::kD32;                    // the older tuning codes address the d32 kernels
  if (groups <= 32768) return Family::kWide;
  // The run kernels cut the rows through L1 to ~0.3x but serialise one window load per group and need 41-49 KB of
  // shared memory per CTA (little L1 left), and end up latency bound at the C2 encoder geometry, so the 8-lane-group
  // kernels serve it; the run kernels stay selectable (variants 100, 101, 120, 121).  The multi-frame geometry
  // (D = 36, C5 encoder call) is the exception, where R = 4 runs beat the nine-lane / generic kernels.  This selection
  // has not been re-timed on H100 (tools/opbench.py times every variant).
  if (run_ok && d.D == 36 && d.Lq >= 2048) return Family::kRun4;
  return Family::kD32;
}

template <typename T>
static int forward_impl(const T* value, const int64_t* shapes, const T* loc, const T* attn, T* out,
                        const Dims& d, cudaStream_t st) {
  if (int rc = check_dims(d)) return rc;
  const int64_t groups = int64_t(d.N) * d.Lq * d.M;
  if (groups == 0) return 0;                       // empty batch / no queries: nothing to do (pointers may be NULL)
  if (!value || !shapes || !loc || !attn || !out) return MSDA_E_NULLPTR;
  constexpr int V16 = 16 / int(sizeof(T));
  const bool vec_ok = (d.D % V16 == 0) && aligned16(value) && aligned16(out);
  auto grid_for = [&](int G) { return unsigned((groups * G + kThreads - 1) / kThreads); };
  bool launched = false;
  if constexpr (sizeof(T) == 4) {
    // run kernels (msda_run.cuh): large query sets, D = 32 (8 lanes per head row) or D = 36 (9 lanes)
    const int variant = g_fwd_variant.load(std::memory_order_relaxed);
    const int LP = d.L * d.P;
    if (variant != 1 && vec_ok && (d.D == 32 || d.D == 36) && LP <= kMaxLP && aligned16(loc) && aligned16(attn) &&
        groups < (int64_t(1) << 31)) {
      const Family fam = pick_family(variant, groups, d);
      if (fam == Family::kRun2 && d.D == 32) {
        // second-generation run kernels (msda_run2.cuh): planned windows, FFMA2, NS interleaved slots
        const int NS = (variant == 121 || d.P % 4 != 0) ? 2 : 4;
        constexpr int R = 8;
        const int qblocks = (d.Lq + 4 * R - 1) / (4 * R);
        const int64_t units = int64_t(d.N) * qblocks * (d.M / kRunHeads);
        const size_t smem = fwd_run2_smem_bytes(R, LP);
        if (units < (int64_t(1) << 31) && d.P % NS == 0 && smem <= 220 * 1024) {
#define MSDA_FWD_RUN2(NS_, LPCT_)                                                                                   \
  do {                                                                                                              \
    MSDA_ENSURE_SMEM((msda_fwd_run2_kernel<R, NS_, LPCT_>), smem);                                                  \
    msda_fwd_run2_kernel<R, NS_, LPCT_><<<unsigned(units), kRunThreads, smem, st>>>(value, shapes, loc, attn, out,   \
                                                                                   d.S, d.M, d.L, d.Lq, d.P, qblocks); \
  } while (0)
          if (NS == 4 && LP == 16) MSDA_FWD_RUN2(4, 16);
          else if (NS == 4) MSDA_FWD_RUN2(4, 0);
          else if (LP == 16) MSDA_FWD_RUN2(2, 16);
          else MSDA_FWD_RUN2(2, 0);
#undef MSDA_FWD_RUN2
          g_launches.fetch_add(1, std::memory_order_relaxed);
          return int(cudaGetLastError());
        }
      }
      if (fam == Family::kRun8 || fam == Family::kRun4 || fam == Family::kRun2) {
        const int R = fam == Family::kRun4 ? 4 : 8, LG = d.D / 4;
        const int QB = run_runs(LG) * R;
        const int qblocks = (d.Lq + QB - 1) / QB;
        const int64_t units = int64_t(d.N) * qblocks * (d.M / kRunHeads);
        const size_t smem = fwd_run_smem_bytes(LG, R, LP);
        if (units < (int64_t(1) << 31) && smem <= 220 * 1024) {
#define MSDA_FWD_RUN(LG_, R_, LPCT_)                                                                                \
  do {                                                                                                              \
    MSDA_ENSURE_SMEM((msda_fwd_run_kernel<LG_, R_, LPCT_>), smem);                                                  \
    msda_fwd_run_kernel<LG_, R_, LPCT_><<<unsigned(units), kRunThreads, smem, st>>>(value, shapes, loc, attn, out,   \
                                                                                   d.S, d.M, d.L, d.Lq, d.P, qblocks); \
  } while (0)
          if (LG == 8) {
            if (R == 8 && LP == 16) MSDA_FWD_RUN(8, 8, 16);
            else if (R == 8) MSDA_FWD_RUN(8, 8, 0);
            else if (LP == 16) MSDA_FWD_RUN(8, 4, 16);
            else MSDA_FWD_RUN(8, 4, 0);
          } else {
            if (R == 8 && LP == 16) MSDA_FWD_RUN(9, 8, 16);
            else if (R == 8) MSDA_FWD_RUN(9, 8, 0);
            else if (LP == 16) MSDA_FWD_RUN(9, 4, 16);
            else MSDA_FWD_RUN(9, 4, 0);
          }
#undef MSDA_FWD_RUN
          g_launches.fetch_add(1, std::memory_order_relaxed);
          return int(cudaGetLastError());
        }
      }
    }
  }
  if constexpr (sizeof(T) == 4) {
    // specialised kernels for the shipped geometry (fp32, 128-byte head rows); variant 1 forces the generic path
    const int variant = g_fwd_variant.load(std::memory_order_relaxed);
    const int LP = d.L * d.P;
    if (variant != 1 && vec_ok && d.D == 32 && LP <= kMaxLP && aligned16(loc) && aligned16(attn) &&
        groups < (int64_t(1) << 31)) {
      const Family fam = pick_family(variant, groups, d);
      if (fam == Family::kWide) {
        const unsigned grid = unsigned((groups + kWideThreads / 32 - 1) / (kWideThreads / 32));
        msda_fwd_wide_kernel<<<grid, kWideThreads, 0, st>>>(value, shapes, loc, attn, out, d.S, d.M, d.L, d.Lq, d.P,
                                                            uint32_t(groups));
        g_launches.fetch_add(1, std::memory_order_relaxed);
        return int(cudaGetLastError());
      }
      const int64_t ctas = (groups + kGroupsPerCta - 1) / kGroupsPerCta;
      // variant = 10 * tuning + iters_code: iters_code >= 2 forces iters = code - 1; tuning picks (unroll, min CTAs/SM)
      const int tuning = variant >= 100 ? 0 : variant / 10, icode = variant >= 100 ? 0 : variant % 10;
      const int iters = icode >= 2 ? icode - 1 : pick_iters(ctas);
      const unsigned grid = unsigned((ctas + iters - 1) / iters);
      const size_t smem = fwd_d32_smem_bytes(LP);
#define MSDA_FWD_D32(U, B)                                                                                          \
  do {                                                                                                              \
    MSDA_ENSURE_SMEM((msda_fwd_d32_kernel<256, U, B>), smem);                                                       \
    msda_fwd_d32_kernel<256, U, B><<<grid, kD32Threads, smem, st>>>(value, shapes, loc, attn, out, d.S, d.M, d.L,    \
                                                                    d.Lq, d.P, uint32_t(groups), iters);            \
  } while (0)
      if (d.M == 8 && tuning == 1) MSDA_FWD_D32(2, 5);
      else if (d.M == 8 && tuning == 2) MSDA_FWD_D32(2, 6);
      else if (d.M == 8 && tuning == 3) MSDA_FWD_D32(4, 5);
      else if (d.M == 8 && tuning == 4) MSDA_FWD_D32(1, 6);
      else if (d.M == 8 && tuning == 5) MSDA_FWD_D32(4, 3);
      else if (d.M == 8 && tuning == 6) MSDA_FWD_D32(4, 4);
      else if (d.M == 8 && tuning == 7) MSDA_FWD_D32(8, 2);
      else if (d.M == 8 && tuning == 8) MSDA_FWD_D32(4, 1);
      else if (d.M == 8) MSDA_FWD_D32(4, 4);          // measured best overall: 64 registers, 4 CTAs/SM
#undef MSDA_FWD_D32
      else {
        MSDA_ENSURE_SMEM((msda_fwd_d32_kernel<0>), smem);
        msda_fwd_d32_kernel<0><<<grid, kD32Threads, smem, st>>>(value, shapes, loc, attn, out, d.S, d.M, d.L, d.Lq,
                                                                d.P, uint32_t(groups), iters);
      }
      launched = true;
    }
  }
  if constexpr (sizeof(T) == 4) {
    // multi-frame geometry (D = 36): nine-lane groups, forward only (msda_d36.cuh); variant 1 forces the generic path
    const int LP = d.L * d.P;
    if (!launched && g_fwd_variant.load(std::memory_order_relaxed) != 1 && vec_ok && d.D == 36 && LP <= kMaxLP &&
        aligned16(loc) && aligned16(attn) && groups < (int64_t(1) << 31)) {
      const int64_t ctas = (groups + kD36GroupsPerCta - 1) / kD36GroupsPerCta;
      const int iters = pick_iters(ctas);
      const unsigned grid = unsigned((ctas + iters - 1) / iters);
      const size_t smem = fwd_d36_smem_bytes(LP);
      if (d.M == 8)
        msda_fwd_d36_kernel<288><<<grid, kD32Threads, smem, st>>>(value, shapes, loc, attn, out, d.S, d.M, d.L, d.Lq,
                                                                  d.P, uint32_t(groups), iters);
      else
        msda_fwd_d36_kernel<0><<<grid, kD32Threads, smem, st>>>(value, shapes, loc, attn, out, d.S, d.M, d.L, d.Lq,
                                                                d.P, uint32_t(groups), iters);
      launched = true;
    }
  }
  if (!launched && vec_ok) {
    int G, it;
    pick_shape(d.D / V16, &G, &it);
    launched = true;
    if (G == 8 && it == 1) MSDA_LAUNCH_FWD(V16, 8, 1);
    else if (G == 8 && it == 2) MSDA_LAUNCH_FWD(V16, 8, 2);
    else if (G == 8 && it <= 4) MSDA_LAUNCH_FWD(V16, 8, 4);
    else if (G == 4 && it == 1) MSDA_LAUNCH_FWD(V16, 4, 1);
    else if (G == 4 && it <= 3) MSDA_LAUNCH_FWD(V16, 4, 3);
    else if (G == 2) MSDA_LAUNCH_FWD(V16, 2, 2);
    else if (G == 1) MSDA_LAUNCH_FWD(V16, 1, 1);
    else launched = false;
  }
  if (!launched) {
    // odd channel counts / unaligned views / very wide heads: scalar lanes, strided channels
    if (d.D <= 8) MSDA_LAUNCH_FWD(1, 8, 1);
    else if (d.D <= 32) MSDA_LAUNCH_FWD(1, 8, 4);
    else if (d.D <= 128) MSDA_LAUNCH_FWD(1, 8, 16);
    else return MSDA_E_TOO_LARGE;
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return int(cudaGetLastError());
}

template <typename T>
static int backward_impl(const T* value, const int64_t* shapes, const T* loc, const T* attn,
                         const T* gout, T* gval, T* gloc, T* gattn, const Dims& d, cudaStream_t st) {
  if (int rc = check_dims(d)) return rc;
  if (d.N > 0) {
    if (!gval) return MSDA_E_NULLPTR;
    cudaError_t e = cudaMemsetAsync(gval, 0, sizeof(T) * size_t(d.N) * d.S * d.M * d.D, st);
    if (e != cudaSuccess) return int(e);
  }
  const int64_t groups = int64_t(d.N) * d.Lq * d.M;
  if (groups == 0) return 0;                       // no queries: grad_value is all zeros, the rest is empty
  if (!value || !shapes || !loc || !attn || !gout || !gloc || !gattn) return MSDA_E_NULLPTR;
  constexpr int V16 = 16 / int(sizeof(T));
  const bool vec_ok = (d.D % V16 == 0) && aligned16(value) && aligned16(gout) && aligned16(gval);
  auto grid_for = [&](int G) { return unsigned((groups * G + kThreads - 1) / kThreads); };
  bool launched = false;
  if constexpr (sizeof(T) == 4) {
    const int variant = g_bwd_variant.load(std::memory_order_relaxed);
    const int LP = d.L * d.P;
    if (variant != 1 && vec_ok && (d.D == 32 || d.D == 36) && LP <= kMaxLP && aligned16(loc) && aligned16(attn) &&
        aligned16(gloc) && aligned16(gattn) && groups < (int64_t(1) << 31)) {
      const Family fam = pick_family(variant, groups, d);
      if (fam == Family::kRun8 || fam == Family::kRun4 || fam == Family::kRun2) {
        const int R = fam == Family::kRun4 ? 4 : 8, LG = d.D / 4;
        const int QB = run_runs(LG) * R;
        const int qblocks = (d.Lq + QB - 1) / QB;
        const int64_t units = int64_t(d.N) * qblocks * (d.M / kRunHeads);
        const size_t smem = bwd_run_smem_bytes(LG, R, LP);
        if (units < (int64_t(1) << 31) && smem <= 220 * 1024) {
#define MSDA_BWD_RUN(LG_, R_, LPCT_)                                                                                \
  do {                                                                                                              \
    MSDA_ENSURE_SMEM((msda_bwd_run_kernel<LG_, R_, LPCT_>), smem);                                                  \
    msda_bwd_run_kernel<LG_, R_, LPCT_><<<unsigned(units), kRunThreads, smem, st>>>(                                \
        value, shapes, loc, attn, gout, gval, gloc, gattn, d.S, d.M, d.L, d.Lq, d.P, qblocks);                      \
  } while (0)
          if (LG == 8) {
            if (R == 8 && LP == 16) MSDA_BWD_RUN(8, 8, 16);
            else if (R == 8) MSDA_BWD_RUN(8, 8, 0);
            else if (LP == 16) MSDA_BWD_RUN(8, 4, 16);
            else MSDA_BWD_RUN(8, 4, 0);
          } else {
            if (R == 8 && LP == 16) MSDA_BWD_RUN(9, 8, 16);
            else if (R == 8) MSDA_BWD_RUN(9, 8, 0);
            else if (LP == 16) MSDA_BWD_RUN(9, 4, 16);
            else MSDA_BWD_RUN(9, 4, 0);
          }
#undef MSDA_BWD_RUN
          g_launches.fetch_add(1, std::memory_order_relaxed);
          return int(cudaGetLastError());
        }
      }
    }
  }
  if constexpr (sizeof(T) == 4) {
    const int variant = g_bwd_variant.load(std::memory_order_relaxed);
    const int LP = d.L * d.P;
    if (variant != 1 && vec_ok && d.D == 32 && LP <= kMaxLP && aligned16(loc) && aligned16(attn) &&
        aligned16(gloc) && aligned16(gattn) && groups < (int64_t(1) << 31)) {
      const Family fam = pick_family(variant, groups, d);
      if (fam == Family::kWide) {
        const unsigned grid = unsigned((groups + kWideThreads / 32 - 1) / (kWideThreads / 32));
        msda_bwd_wide_kernel<<<grid, kWideThreads, 0, st>>>(value, shapes, loc, attn, gout, gval, gloc, gattn, d.S, d.M,
                                                            d.L, d.Lq, d.P, uint32_t(groups));
        g_launches.fetch_add(1, std::memory_order_relaxed);
        return int(cudaGetLastError());
      }
      const int64_t ctas = (groups + kGroupsPerCta - 1) / kGroupsPerCta;
      const int tuning = variant >= 100 ? 0 : variant / 10, icode = variant >= 100 ? 0 : variant % 10;
      const int iters = icode >= 2 ? icode - 1 : pick_iters(ctas);
      const unsigned grid = unsigned((ctas + iters - 1) / iters);
      const size_t smem = bwd_d32_smem_bytes(LP);
#define MSDA_BWD_D32(B)                                                                                              \
  do {                                                                                                               \
    MSDA_ENSURE_SMEM((msda_bwd_d32_kernel<256, B>), smem);                                                           \
    msda_bwd_d32_kernel<256, B><<<grid, kD32Threads, smem, st>>>(value, shapes, loc, attn, gout, gval, gloc, gattn,   \
                                                                 d.S, d.M, d.L, d.Lq, d.P, uint32_t(groups), iters); \
  } while (0)
      if (d.M == 8 && tuning == 1) MSDA_BWD_D32(2);
      else if (d.M == 8 && tuning == 2) MSDA_BWD_D32(3);
      else if (d.M == 8 && tuning == 3) MSDA_BWD_D32(5);
      else if (d.M == 8 && tuning == 4) MSDA_BWD_D32(6);
      else if (d.M == 8) MSDA_BWD_D32(4);
#undef MSDA_BWD_D32
      else {
        MSDA_ENSURE_SMEM((msda_bwd_d32_kernel<0>), smem);
        msda_bwd_d32_kernel<0><<<grid, kD32Threads, smem, st>>>(value, shapes, loc, attn, gout, gval, gloc, gattn,
                                                                d.S, d.M, d.L, d.Lq, d.P, uint32_t(groups), iters);
      }
      launched = true;
    }
  }
  if (!launched && vec_ok) {
    int G, it;
    pick_shape(d.D / V16, &G, &it);
    launched = true;
    if (G == 8 && it == 1) MSDA_LAUNCH_BWD(V16, 8, 1);
    else if (G == 8 && it == 2) MSDA_LAUNCH_BWD(V16, 8, 2);
    else if (G == 8 && it <= 4) MSDA_LAUNCH_BWD(V16, 8, 4);
    else if (G == 4 && it == 1) MSDA_LAUNCH_BWD(V16, 4, 1);
    else if (G == 4 && it <= 3) MSDA_LAUNCH_BWD(V16, 4, 3);
    else if (G == 2) MSDA_LAUNCH_BWD(V16, 2, 2);
    else if (G == 1) MSDA_LAUNCH_BWD(V16, 1, 1);
    else launched = false;
  }
  if (!launched) {
    // odd channel counts / unaligned views / very wide heads: scalar lanes, strided channels
    if (d.D <= 8) MSDA_LAUNCH_BWD(1, 8, 1);
    else if (d.D <= 32) MSDA_LAUNCH_BWD(1, 8, 4);
    else if (d.D <= 128) MSDA_LAUNCH_BWD(1, 8, 16);
    else return MSDA_E_TOO_LARGE;
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return int(cudaGetLastError());
}

// ---- measurement aid: what can the L1 data stage deliver for THIS access pattern? -------------------------------
// Every warp issues LDG.128 requests shaped exactly like the gather's: 4 groups x 8 lanes, each group reading one
// 128-byte row chosen pseudo-randomly from a table of `rows` rows (table small => L1 hits; 22.8 MB => L2 hits).
// Nothing else happens, so bytes/time is the ceiling the MSDeformAttn gather can reach on this part.
__global__ void __launch_bounds__(256)
l1_gather_probe_kernel(const float4* __restrict__ table, float4* __restrict__ sink, uint32_t rows, int iters) {
  const uint32_t gid = (blockIdx.x * 256u + threadIdx.x) >> 3;
  const int j = threadIdx.x & 7;
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  uint32_t h = gid * 2654435761u + 12345u;
#pragma unroll 8
  for (int i = 0; i < iters; ++i) {
    h = h * 1664525u + 1013904223u;
    const float4 v = __ldg(table + size_t((h >> 8) % rows) * 8 + j);
    acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
  }
  if (acc.x == 1.2345e30f) sink[gid] = acc;        // never true: keeps the loads alive
}

// ---- host-buffer convenience path (end-to-end timing, C callers without a CUDA runtime) ---
struct DevBuf {
  void* p = nullptr;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t alloc(size_t bytes) { return cudaMalloc(&p, bytes ? bytes : 1); }
};
#define MSDA_CUDA_TRY(expr)                   \
  do {                                        \
    cudaError_t e__ = (expr);                 \
    if (e__ != cudaSuccess) return int(e__);  \
  } while (0)

}  // namespace msda

using namespace msda;

extern "C" {

int msda_b200_abi_version(void) { return MSDA_B200_ABI_VERSION; }

const char* msda_b200_error_string(int code) {
  switch (code) {
    case 0: return "success";
    case MSDA_E_NULLPTR: return "msda_b200: NULL pointer argument";
    case MSDA_E_DIMS: return "msda_b200: non-positive dimension";
    case MSDA_E_TOO_LARGE: return "msda_b200: S*M*D exceeds 2^31-1 elements or D unsupported";
    case MSDA_E_LEVELS: return "msda_b200: too many levels";
    case MSDA_E_UNSUPPORTED: return "msda_b200: geometry not supported by this specialised entry point";
    default: break;
  }
  if (code > 0) return cudaGetErrorString(cudaError_t(code));
  return "msda_b200: unknown error";
}

void msda_b200_set_variant(int fwd_variant, int bwd_variant) {
  g_fwd_variant.store(fwd_variant);
  g_bwd_variant.store(bwd_variant);
}

uint64_t msda_b200_launch_count(void) { return g_launches.load(); }
void msda_b200_count_launches(int n) { g_launches.fetch_add(uint64_t(n), std::memory_order_relaxed); }

int msda_b200_l1_gather_probe(const float* table, float* sink, int64_t rows, int iters, int ctas, void* stream) {
  if (!table || !sink || rows <= 0 || iters <= 0 || ctas <= 0) return MSDA_E_DIMS;
  l1_gather_probe_kernel<<<ctas, 256, 0, cudaStream_t(stream)>>>(reinterpret_cast<const float4*>(table),
                                                                 reinterpret_cast<float4*>(sink), uint32_t(rows), iters);
  return int(cudaGetLastError());
}

int msda_b200_variant_allows_tiles(void) {
  const int v = g_fwd_variant.load(), b = g_bwd_variant.load();
  return ((v == 0 || v >= 200) && (b == 0 || b >= 200)) ? 1 : 0;
}

int msda_b200_forward_f32(const float* value, const int64_t* spatial_shapes, const float* sampling_loc,
                          const float* attn_weight, float* output, int N, int S, int M, int D, int L,
                          int Lq, int P, void* stream) {
  return forward_impl<float>(value, spatial_shapes, sampling_loc, attn_weight, output,
                             Dims{N, S, M, D, L, Lq, P}, cudaStream_t(stream));
}

int msda_b200_forward_f64(const double* value, const int64_t* spatial_shapes, const double* sampling_loc,
                          const double* attn_weight, double* output, int N, int S, int M, int D, int L,
                          int Lq, int P, void* stream) {
  return forward_impl<double>(value, spatial_shapes, sampling_loc, attn_weight, output,
                              Dims{N, S, M, D, L, Lq, P}, cudaStream_t(stream));
}

int msda_b200_backward_f32(const float* value, const int64_t* spatial_shapes, const float* sampling_loc,
                           const float* attn_weight, const float* grad_output, float* grad_value,
                           float* grad_sampling_loc, float* grad_attn_weight, int N, int S, int M, int D,
                           int L, int Lq, int P, void* stream) {
  return backward_impl<float>(value, spatial_shapes, sampling_loc, attn_weight, grad_output, grad_value,
                              grad_sampling_loc, grad_attn_weight, Dims{N, S, M, D, L, Lq, P},
                              cudaStream_t(stream));
}

int msda_b200_backward_f64(const double* value, const int64_t* spatial_shapes, const double* sampling_loc,
                           const double* attn_weight, const double* grad_output, double* grad_value,
                           double* grad_sampling_loc, double* grad_attn_weight, int N, int S, int M, int D,
                           int L, int Lq, int P, void* stream) {
  return backward_impl<double>(value, spatial_shapes, sampling_loc, attn_weight, grad_output, grad_value,
                               grad_sampling_loc, grad_attn_weight, Dims{N, S, M, D, L, Lq, P},
                               cudaStream_t(stream));
}

// ---- fused-prologue entry points: sampling locations / attention weights are computed inside the kernel from the
//      module's raw [offsets | logits] projection and the reference points (ops/modules/ms_deform_attn.py:69-79) and
//      never written to HBM.  Domain: fp32, D = 32 or 36, M % 4 == 0, L * P == 16, 2-d reference points.
static int fused_domain(const Dims& d, const void* a, const void* b, const void* c, const void* e) {
  if (int rc = check_dims(d)) return rc;
  if ((d.D != 32 && d.D != 36) || d.M % kRunHeads != 0 || d.L * d.P != 16 || d.N < 1 || d.Lq < 1) return MSDA_E_UNSUPPORTED;
  if (!aligned16(a) || !aligned16(b) || !aligned16(c) || !aligned16(e)) return MSDA_E_UNSUPPORTED;
  return 0;
}

int msda_b200_forward_fused_f32(const float* value, const int64_t* spatial_shapes, const float* proj, const float* ref,
                                float* output, int N, int S, int M, int D, int L, int Lq, int P, void* stream) {
  const Dims d{N, S, M, D, L, Lq, P};
  if (!value || !spatial_shapes || !proj || !ref || !output) return MSDA_E_NULLPTR;
  if (int rc = fused_domain(d, value, proj, ref, output)) return rc;
  cudaStream_t st = cudaStream_t(stream);
  const int LG = D / 4, R = 8, QB = run_runs(LG) * R;
  const int qblocks = (Lq + QB - 1) / QB;
  const int64_t units = int64_t(N) * qblocks * (M / kRunHeads);
  if (units >= (int64_t(1) << 31)) return MSDA_E_TOO_LARGE;
  const size_t smem = fwd_run_smem_bytes(LG, R, 16);
  if (LG == 8) {
    MSDA_ENSURE_SMEM((msda_fwd_run_kernel<8, 8, 16, true>), smem);
    msda_fwd_run_kernel<8, 8, 16, true><<<unsigned(units), kRunThreads, smem, st>>>(value, spatial_shapes, proj, ref, output, S,
                                                                                   M, L, Lq, P, qblocks);
  } else {
    MSDA_ENSURE_SMEM((msda_fwd_run_kernel<9, 8, 16, true>), smem);
    msda_fwd_run_kernel<9, 8, 16, true><<<unsigned(units), kRunThreads, smem, st>>>(value, spatial_shapes, proj, ref, output, S,
                                                                                   M, L, Lq, P, qblocks);
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return int(cudaGetLastError());
}

int msda_b200_backward_fused_f32(const float* value, const int64_t* spatial_shapes, const float* proj, const float* ref,
                                 const float* grad_output, float* grad_value, float* grad_proj, int N, int S, int M, int D,
                                 int L, int Lq, int P, void* stream) {
  const Dims d{N, S, M, D, L, Lq, P};
  if (!value || !spatial_shapes || !proj || !ref || !grad_output || !grad_value || !grad_proj) return MSDA_E_NULLPTR;
  if (int rc = fused_domain(d, value, proj, ref, grad_output)) return rc;
  if (!aligned16(grad_value) || !aligned16(grad_proj)) return MSDA_E_UNSUPPORTED;
  cudaStream_t st = cudaStream_t(stream);
  cudaError_t e = cudaMemsetAsync(grad_value, 0, sizeof(float) * size_t(N) * S * M * D, st);
  if (e != cudaSuccess) return int(e);
  const int LG = D / 4, R = 8, QB = run_runs(LG) * R;
  const int qblocks = (Lq + QB - 1) / QB;
  const int64_t units = int64_t(N) * qblocks * (M / kRunHeads);
  if (units >= (int64_t(1) << 31)) return MSDA_E_TOO_LARGE;
  const size_t smem = bwd_run_smem_bytes(LG, R, 16);
  if (LG == 8) {
    MSDA_ENSURE_SMEM((msda_bwd_run_kernel<8, 8, 16, true>), smem);
    msda_bwd_run_kernel<8, 8, 16, true><<<unsigned(units), kRunThreads, smem, st>>>(
        value, spatial_shapes, proj, ref, grad_output, grad_value, grad_proj, nullptr, S, M, L, Lq, P, qblocks);
  } else {
    MSDA_ENSURE_SMEM((msda_bwd_run_kernel<9, 8, 16, true>), smem);
    msda_bwd_run_kernel<9, 8, 16, true><<<unsigned(units), kRunThreads, smem, st>>>(
        value, spatial_shapes, proj, ref, grad_output, grad_value, grad_proj, nullptr, S, M, L, Lq, P, qblocks);
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return int(cudaGetLastError());
}

// value of image n, level l, viewed as [N][H_l][W_l][M][32] floats; box = 32 channels x 1 head x bw x bh pixels
static bool et_make_map(CUtensorMap* map, const float* level_base, int N, int S, int M, int H, int W, int bw, int bh) {
  tfb200::EncodeTiledFn fn = tfb200::tensor_map_encoder();
  if (!fn) return false;
  const cuuint64_t dims[5] = {32, cuuint64_t(M), cuuint64_t(W), cuuint64_t(H), cuuint64_t(N)};
  const cuuint64_t strides[4] = {128, cuuint64_t(M) * 128, cuuint64_t(W) * M * 128, cuuint64_t(S) * M * 128};
  const cuuint32_t box[5] = {32, 1, cuuint32_t(bw), cuuint32_t(bh), 1};
  const cuuint32_t estr[5] = {1, 1, 1, 1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 5, const_cast<float*>(level_base), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int eb_upload_signs() {
  static std::once_flag signs_once;
  static cudaError_t signs_rc = cudaSuccess;
  std::call_once(signs_once, [] {
    EbSigns t;
    eb_fill_signs(&t);
    signs_rc = cudaMemcpyToSymbol(kEbSigns, &t, sizeof(t));     // (per device context: one GPU per process)
  });
  return int(signs_rc);
}

// Fills the tile geometry and the tensor maps of the encoder tile kernels; MSDA_E_UNSUPPORTED outside their domain.
static int et_prepare(const float* value, const int64_t* spatial_shapes_host, int N, int S, int M, int D, int L, int Lq,
                      int P, EtGeom* g, EtMaps* maps, int64_t* grid, bool backward) {
  if (D != 32 || L > kEtMaxL || P != kEtP || Lq != S || N < 1 || M > 65535) return MSDA_E_UNSUPPORTED;
  if (backward && S >= (1 << 20)) return MSDA_E_UNSUPPORTED;          // 20-bit pixel indices in the backward's tap words
  if (!aligned16(value)) return MSDA_E_UNSUPPORTED;
  g->L = L; g->S = S; g->M = M; g->Lq = Lq;
  int64_t acc = 0;
  int tiles = 0;
  for (int l = 0; l < kEtMaxL; ++l) {
    g->H[l] = g->W[l] = 2; g->start[l] = 0; g->tiles_x[l] = 1; g->tile_begin[l + 1] = 0;
  }
  for (int l = 0; l < L; ++l) {
    const int64_t h = spatial_shapes_host[2 * l], w = spatial_shapes_host[2 * l + 1];
    if (h < 2 || w < 2 || h > 32767 || w > 32767) return MSDA_E_UNSUPPORTED;
    if (backward && (h > 4095 || w > 4095)) return MSDA_E_UNSUPPORTED;  // 12-bit window corners in the backward's tap words
    g->H[l] = int(h); g->W[l] = int(w); g->start[l] = int(acc);
    g->tiles_x[l] = int((w + kEtTX - 1) / kEtTX);
    g->tile_begin[l] = tiles;
    tiles += g->tiles_x[l] * int((h + kEtTY - 1) / kEtTY);
    acc += h * w;
  }
  for (int l = L; l <= kEtMaxL; ++l) g->tile_begin[l] = tiles;
  g->tiles_used = tiles;
  if (acc != S) return MSDA_E_UNSUPPORTED;
  *grid = int64_t(tiles) * M * N;
  if (*grid > INT32_MAX) return MSDA_E_UNSUPPORTED;
  for (int lq = 0; lq < L; ++lq)
    for (int l = lq; l < L; ++l)
      if (!et_make_map(&maps->m[et_map_index(lq, l)], value + size_t(g->start[l]) * M * 32, N, S, M, g->H[l], g->W[l],
                       backward ? eb_bw(l - lq) : et_bw(l - lq), backward ? eb_bh(l - lq) : et_bh(l - lq)))
        return MSDA_E_UNSUPPORTED;
  return 0;
}

int msda_b200_forward_enc_tiled_f32(const float* value, const int64_t* spatial_shapes_host, const float* sampling_loc,
                                    const float* attn_weight, float* output, int N, int S, int M, int D, int L,
                                    int Lq, int P, void* stream) {
  const Dims d{N, S, M, D, L, Lq, P};
  if (int rc = check_dims(d)) return rc;
  if (!value || !spatial_shapes_host || !sampling_loc || !attn_weight || !output) return MSDA_E_NULLPTR;
  if (!aligned16(sampling_loc) || !aligned16(attn_weight) || !aligned16(output)) return MSDA_E_UNSUPPORTED;
  EtGeom g;
  EtMaps maps;
  int64_t grid = 0;
  if (int rc = et_prepare(value, spatial_shapes_host, N, S, M, D, L, Lq, P, &g, &maps, &grid, false)) return rc;
  if (g_fwd_variant.load(std::memory_order_relaxed) == 201) {        // A/B: four warps, four slots per warp
    MSDA_ENSURE_SMEM((msda_fwd_enc_tma_kernel<4, false>), kEtSmemBytes);
    msda_fwd_enc_tma_kernel<4, false><<<unsigned(grid), 128, kEtSmemBytes, cudaStream_t(stream)>>>(value, sampling_loc, attn_weight,
                                                                                           output, g, maps);
  } else {
    MSDA_ENSURE_SMEM((msda_fwd_enc_tma_kernel<2, false>), kEtSmemBytes);
    msda_fwd_enc_tma_kernel<2, false><<<unsigned(grid), kEtThreads, kEtSmemBytes, cudaStream_t(stream)>>>(value, sampling_loc,
                                                                                                  attn_weight, output, g, maps);
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return int(cudaGetLastError());
}

// 8-lane-group backward on the queries [q_first, Lq) of every image (no zero-fill: the caller did it)
static int bwd_d32_query_range(const float* value, const int64_t* shapes_dev, const float* loc, const float* attn,
                               const float* gout, float* gval, float* gloc, float* gattn, const Dims& d, int q_first,
                               cudaStream_t st) {
  const int LP = d.L * d.P;
  const int nq = d.Lq - q_first;
  if (nq <= 0) return 0;
  const size_t smem = bwd_d32_smem_bytes(LP);
  for (int n = 0; n < d.N; ++n) {
    const size_t qo = size_t(n) * d.Lq + q_first;
    const float* v = value + size_t(n) * d.S * d.M * d.D;
    float* gv = gval + size_t(n) * d.S * d.M * d.D;
    const float* lc = loc + qo * d.M * LP * 2;
    const float* at = attn + qo * d.M * LP;
    const float* go = gout + qo * d.M * d.D;
    float* gl = gloc + qo * d.M * LP * 2;
    float* ga = gattn + qo * d.M * LP;
    const int64_t groups = int64_t(nq) * d.M;
    const int64_t ctas = (groups + kGroupsPerCta - 1) / kGroupsPerCta;
    const int iters = pick_iters(ctas);
    const unsigned grid = unsigned((ctas + iters - 1) / iters);
    if (d.M == 8) {
      MSDA_ENSURE_SMEM((msda_bwd_d32_kernel<256, 4>), smem);
      msda_bwd_d32_kernel<256, 4><<<grid, kD32Threads, smem, st>>>(v, shapes_dev, lc, at, go, gv, gl, ga, d.S, d.M, d.L, nq, d.P,
                                                                   uint32_t(groups), iters);
    } else {
      MSDA_ENSURE_SMEM((msda_bwd_d32_kernel<0>), smem);
      msda_bwd_d32_kernel<0><<<grid, kD32Threads, smem, st>>>(v, shapes_dev, lc, at, go, gv, gl, ga, d.S, d.M, d.L, nq, d.P,
                                                              uint32_t(groups), iters);
    }
    g_launches.fetch_add(1, std::memory_order_relaxed);
  }
  return int(cudaGetLastError());
}

int msda_b200_backward_enc_tiled_f32(const float* value, const int64_t* spatial_shapes_host,
                                     const int64_t* spatial_shapes_dev, const float* sampling_loc, const float* attn_weight,
                                     const float* grad_output, float* grad_value, float* grad_sampling_loc,
                                     float* grad_attn_weight, int N, int S, int M, int D, int L, int Lq, int P, void* stream) {
  const Dims d{N, S, M, D, L, Lq, P};
  if (int rc = check_dims(d)) return rc;
  if (!value || !spatial_shapes_host || !sampling_loc || !attn_weight || !grad_output || !grad_value || !grad_sampling_loc ||
      !grad_attn_weight)
    return MSDA_E_NULLPTR;
  if (!aligned16(sampling_loc) || !aligned16(attn_weight) || !aligned16(grad_output) || !aligned16(grad_value) ||
      !aligned16(grad_sampling_loc) || !aligned16(grad_attn_weight))
    return MSDA_E_UNSUPPORTED;
  EtGeom g;
  EtMaps maps;
  int64_t grid = 0;
  if (int rc = et_prepare(value, spatial_shapes_host, N, S, M, D, L, Lq, P, &g, &maps, &grid, true)) return rc;
  cudaStream_t st = cudaStream_t(stream);
  cudaError_t e = cudaMemsetAsync(grad_value, 0, sizeof(float) * size_t(N) * S * M * D, st);
  if (e != cudaSuccess) return int(e);
  if (int rc = eb_upload_signs()) return rc;
  // Queries of the coarser levels (25 % of a C2 call) sample the finer levels with a footprint of 2-8x the tile: the tile
  // kernel walks those levels from global memory, one L2 round trip per step, and its slowest CTAs are exactly these
  // (16 % of the kernel's time for 8 % of the samples, ncu).  Experiment: with the device copy of the level sizes at hand
  // they can go to the 8-lane-group kernel instead while the tile kernel keeps the level-0 tiles.
  // The 8-lane-group kernel needs about as long for that quarter of the queries as the tile kernel's slow CTAs, so the
  // split did not pay and is OFF unless asked for (variant 203).
  const bool split = spatial_shapes_dev != nullptr && L > 1 && g_bwd_variant.load(std::memory_order_relaxed) == 203;
  if (split) {
    g.tiles_used = g.tile_begin[1];
    grid = int64_t(g.tiles_used) * M * N;
  }
  MSDA_ENSURE_SMEM(msda_bwd_enc_tma_kernel<false>, kEbSmemBytes);
  msda_bwd_enc_tma_kernel<false><<<unsigned(grid), kEbThreads, kEbSmemBytes, st>>>(
      value, sampling_loc, attn_weight, grad_output, grad_value, grad_sampling_loc, grad_attn_weight, g, maps);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  if (int rc = int(cudaGetLastError())) return rc;
  if (split)
    return bwd_d32_query_range(value, spatial_shapes_dev, sampling_loc, attn_weight, grad_output, grad_value, grad_sampling_loc,
                               grad_attn_weight, d, g.start[1], st);
  return 0;
}

// Encoder tile kernels with the module's location / softmax arithmetic inside (ops/modules/ms_deform_attn.py:69-87):
// proj [N][Lq][3*M*16] = [offsets | logits], ref [N][Lq][L][2].  Domain: the tile kernels' (fp32, D = 32, Lq == S) and L == 4.
int msda_b200_forward_enc_tiled_fused_f32(const float* value, const int64_t* spatial_shapes_host, const float* proj,
                                          const float* ref, float* output, int N, int S, int M, int D, int L, int Lq,
                                          int P, void* stream) {
  const Dims d{N, S, M, D, L, Lq, P};
  if (int rc = check_dims(d)) return rc;
  if (!value || !spatial_shapes_host || !proj || !ref || !output) return MSDA_E_NULLPTR;
  if (L != 4 || !aligned16(proj) || !aligned16(ref) || !aligned16(output)) return MSDA_E_UNSUPPORTED;
  EtGeom g;
  EtMaps maps;
  int64_t grid = 0;
  if (int rc = et_prepare(value, spatial_shapes_host, N, S, M, D, L, Lq, P, &g, &maps, &grid, false)) return rc;
  MSDA_ENSURE_SMEM((msda_fwd_enc_tma_kernel<2, true>), kEtSmemBytes);
  msda_fwd_enc_tma_kernel<2, true><<<unsigned(grid), kEtThreads, kEtSmemBytes, cudaStream_t(stream)>>>(value, proj, ref, output,
                                                                                                    g, maps);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return int(cudaGetLastError());
}

int msda_b200_backward_enc_tiled_fused_f32(const float* value, const int64_t* spatial_shapes_host, const float* proj,
                                           const float* ref, const float* grad_output, float* grad_value, float* grad_proj,
                                           int N, int S, int M, int D, int L, int Lq, int P, void* stream) {
  const Dims d{N, S, M, D, L, Lq, P};
  if (int rc = check_dims(d)) return rc;
  if (!value || !spatial_shapes_host || !proj || !ref || !grad_output || !grad_value || !grad_proj) return MSDA_E_NULLPTR;
  if (L != 4 || !aligned16(proj) || !aligned16(ref) || !aligned16(grad_output) || !aligned16(grad_value) || !aligned16(grad_proj))
    return MSDA_E_UNSUPPORTED;
  EtGeom g;
  EtMaps maps;
  int64_t grid = 0;
  if (int rc = et_prepare(value, spatial_shapes_host, N, S, M, D, L, Lq, P, &g, &maps, &grid, true)) return rc;
  cudaStream_t st = cudaStream_t(stream);
  cudaError_t e = cudaMemsetAsync(grad_value, 0, sizeof(float) * size_t(N) * S * M * D, st);
  if (e != cudaSuccess) return int(e);
  if (int rc = eb_upload_signs()) return rc;
  MSDA_ENSURE_SMEM(msda_bwd_enc_tma_kernel<true>, kEbSmemBytes);
  msda_bwd_enc_tma_kernel<true><<<unsigned(grid), kEbThreads, kEbSmemBytes, st>>>(value, proj, ref, grad_output, grad_value,
                                                                                 grad_proj, nullptr, g, maps);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  return int(cudaGetLastError());
}

int msda_b200_forward_host_f32(const float* value, const int64_t* spatial_shapes, const float* sampling_loc,
                               const float* attn_weight, float* output, int N, int S, int M, int D, int L,
                               int Lq, int P, int device) {
  const Dims d{N, S, M, D, L, Lq, P};
  if (int rc = check_dims(d)) return rc;
  if (!value || !spatial_shapes || !sampling_loc || !attn_weight || !output) return MSDA_E_NULLPTR;
  MSDA_CUDA_TRY(cudaSetDevice(device));
  const size_t nv = size_t(N) * S * M * D, ns = size_t(N) * Lq * M * L * P, no = size_t(N) * Lq * M * D;
  DevBuf dv, dsz, dl, da, dout;
  MSDA_CUDA_TRY(dv.alloc(nv * 4));
  MSDA_CUDA_TRY(dsz.alloc(size_t(L) * 16));
  MSDA_CUDA_TRY(dl.alloc(ns * 8));
  MSDA_CUDA_TRY(da.alloc(ns * 4));
  MSDA_CUDA_TRY(dout.alloc(no * 4));
  cudaStream_t st = nullptr;
  MSDA_CUDA_TRY(cudaMemcpyAsync(dv.p, value, nv * 4, cudaMemcpyHostToDevice, st));
  MSDA_CUDA_TRY(cudaMemcpyAsync(dsz.p, spatial_shapes, size_t(L) * 16, cudaMemcpyHostToDevice, st));
  MSDA_CUDA_TRY(cudaMemcpyAsync(dl.p, sampling_loc, ns * 8, cudaMemcpyHostToDevice, st));
  MSDA_CUDA_TRY(cudaMemcpyAsync(da.p, attn_weight, ns * 4, cudaMemcpyHostToDevice, st));
  int rc = forward_impl<float>((const float*)dv.p, (const int64_t*)dsz.p, (const float*)dl.p,
                               (const float*)da.p, (float*)dout.p, d, st);
  if (rc) return rc;
  MSDA_CUDA_TRY(cudaMemcpyAsync(output, dout.p, no * 4, cudaMemcpyDeviceToHost, st));
  MSDA_CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

int msda_b200_backward_host_f32(const float* value, const int64_t* spatial_shapes, const float* sampling_loc,
                                const float* attn_weight, const float* grad_output, float* grad_value,
                                float* grad_sampling_loc, float* grad_attn_weight, int N, int S, int M,
                                int D, int L, int Lq, int P, int device) {
  const Dims d{N, S, M, D, L, Lq, P};
  if (int rc = check_dims(d)) return rc;
  if (!value || !spatial_shapes || !sampling_loc || !attn_weight || !grad_output || !grad_value ||
      !grad_sampling_loc || !grad_attn_weight)
    return MSDA_E_NULLPTR;
  MSDA_CUDA_TRY(cudaSetDevice(device));
  const size_t nv = size_t(N) * S * M * D, ns = size_t(N) * Lq * M * L * P, no = size_t(N) * Lq * M * D;
  DevBuf dv, dsz, dl, da, dgo, dgv, dgl, dga;
  MSDA_CUDA_TRY(dv.alloc(nv * 4));
  MSDA_CUDA_TRY(dsz.alloc(size_t(L) * 16));
  MSDA_CUDA_TRY(dl.alloc(ns * 8));
  MSDA_CUDA_TRY(da.alloc(ns * 4));
  MSDA_CUDA_TRY(dgo.alloc(no * 4));
  MSDA_CUDA_TRY(dgv.alloc(nv * 4));
  MSDA_CUDA_TRY(dgl.alloc(ns * 8));
  MSDA_CUDA_TRY(dga.alloc(ns * 4));
  cudaStream_t st = nullptr;
  MSDA_CUDA_TRY(cudaMemcpyAsync(dv.p, value, nv * 4, cudaMemcpyHostToDevice, st));
  MSDA_CUDA_TRY(cudaMemcpyAsync(dsz.p, spatial_shapes, size_t(L) * 16, cudaMemcpyHostToDevice, st));
  MSDA_CUDA_TRY(cudaMemcpyAsync(dl.p, sampling_loc, ns * 8, cudaMemcpyHostToDevice, st));
  MSDA_CUDA_TRY(cudaMemcpyAsync(da.p, attn_weight, ns * 4, cudaMemcpyHostToDevice, st));
  MSDA_CUDA_TRY(cudaMemcpyAsync(dgo.p, grad_output, no * 4, cudaMemcpyHostToDevice, st));
  int rc = backward_impl<float>((const float*)dv.p, (const int64_t*)dsz.p, (const float*)dl.p,
                                (const float*)da.p, (const float*)dgo.p, (float*)dgv.p, (float*)dgl.p,
                                (float*)dga.p, d, st);
  if (rc) return rc;
  MSDA_CUDA_TRY(cudaMemcpyAsync(grad_value, dgv.p, nv * 4, cudaMemcpyDeviceToHost, st));
  MSDA_CUDA_TRY(cudaMemcpyAsync(grad_sampling_loc, dgl.p, ns * 8, cudaMemcpyDeviceToHost, st));
  MSDA_CUDA_TRY(cudaMemcpyAsync(grad_attn_weight, dga.p, ns * 4, cudaMemcpyDeviceToHost, st));
  MSDA_CUDA_TRY(cudaStreamSynchronize(st));
  return 0;
}

}  // extern "C"
