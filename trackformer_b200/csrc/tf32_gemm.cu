// Y[M,N] = act(X[M,K] . W[N,K]^T + bias[N]) -- fp32 in HBM, TF32 tensor-core products, fp32 accumulation.
//
// Hand-written sm_90a kernel for the long-token Linear layers of the deformable transformer
// (reference: nn.Linear calls in ops/modules/ms_deform_attn.py:64,69,70,88 and
// models/deformable_transformer.py:282-286 -- value / [offsets|logits] / output projections and the FFN over the
// S = 22 223 encoder tokens).  These products are HBM-bound (read X once, write Y once), so the kernel is built to
// stream:
//
//   * TMA (cp.async.bulk.tensor) stages 128 x 32 fp32 operand tiles through a 4-deep mbarrier ring filled by one
//     producer warp; out-of-range rows of the last token block are zero-filled by the TMA unit and the store is
//     clipped by it -- no tail code anywhere;
//   * two consumer warpgroups each own 64 rows of the 128 x 128 output tile and issue
//     wgmma.mma_async.m64n128k8.f32.tf32.tf32 (persistent CTAs, one per SM);
//   * the epilogue adds the bias, applies the activation (ReLU, ReLU + dropout, or the dropout gradient), writes
//     128-byte rows into a swizzled staging buffer and hands it to TMA stores (or TMA reductions).
//
// wgmma reads a TF32 operand from shared memory only K-major (contraction index contiguous).  The two products:
//   linear  Y  = X . W^T        A = X tile [128 rows][32 k] and B = W tile, both K-major SWIZZLE_128B and both read
//                               by wgmma straight from shared memory.  One wgmma group stays in flight: a ring slot
//                               is released once the group after the one that read it has been issued and the
//                               older group has retired (wait_group 1).
//                               dgrad dX = dY . W runs as this product on W^T ([K, N], transposed once per call).
//   wgrad   dW = dY^T . X       A = dY^T from a [32 tokens][128 n] tile (MN-major, so it goes through registers);
//                               B = X^T, whose [32 tokens][128 k] tile the consumers transpose into a K-major swizzled
//                               buffer first.  The token axis (22 223 long) is split into slabs over all SMs and every
//                               CTA adds its 128 x 128 partial product into dW with a TMA reduction
//                               (cp.reduce.async.bulk.tensor .add).
#include <cuda.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <atomic>

#include "../../include/tfb200_fused.h"
#include "dropout_hash.cuh"
#include "launch_counter.h"
#include "tma_host.h"

namespace tfb200 {
namespace gemm {

constexpr int BM = 128, BN = 128, BK = 32;          // BK fp32 = 128 bytes = one swizzle span
constexpr int STAGES = 4;
constexpr int CONSUMERS = 256;                       // two warpgroups, 64 accumulator rows each
constexpr int THREADS = CONSUMERS + 32;              // + one TMA producer warp
constexpr int TILE_BYTES = BM * BK * 4;              // 16 KB (A and B tiles have the same size)
constexpr int OUT_BYTES = BM * BN * 4;               // epilogue staging: four 128-row x 32-column chunks
constexpr int SMEM_BYTES = STAGES * 2 * TILE_BYTES + 2 * TILE_BYTES + OUT_BYTES + 256 + 1024;   // + barriers + align

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return uint32_t(__cvta_generic_to_shared(p)); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.b32 %0, 1, 0, p;\n\t}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!ok);
}

__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
      : "memory");
}
__device__ __forceinline__ void tma_reduce_add_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.reduce.async.bulk.tensor.2d.global.shared::cta.add.tile.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(
                   reinterpret_cast<uint64_t>(map)),
               "r"(src), "r"(c0), "r"(c1)
               : "memory");
}

__device__ __forceinline__ uint32_t lds(uint32_t a) {
  uint32_t v;
  asm volatile("ld.shared.b32 %0, [%1];" : "=r"(v) : "r"(a));
  return v;
}
// byte offset of element (row, col) in a [rows][32] fp32 tile with 128-byte swizzle (16-byte chunk ^= row % 8)
__device__ __forceinline__ uint32_t sw128(int row, int col) {
  return uint32_t(row * 128 + ((((col & 31) >> 2) ^ (row & 7)) << 4) + (col & 3) * 4);
}

// K-major tile [rows][32 fp32], SWIZZLE_128B, 8-row groups 1024 bytes apart (sm_90 wgmma descriptor)
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr) {
  uint64_t d = uint64_t((saddr & 0x3FFFFu) >> 4);       // start address, 16-byte units          bits [0,14)
  d |= uint64_t(1) << 16;                                // leading byte offset (unused here)     bits [16,30)
  d |= uint64_t(1024 >> 4) << 32;                        // stride byte offset: 8 rows x 128 B    bits [32,46)
  d |= uint64_t(1) << 62;                                // layout: SWIZZLE_128B                  bits [62,64)
  return d;
}

#define TFB200_ACC64                                                                                                   \
  "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),          \
      "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]),           \
      "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),          \
      "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]),          \
      "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]),          \
      "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),          \
      "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]),          \
      "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
#define TFB200_D64                                                                                                     \
  "{"                                                                                                                  \
  "%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, "     \
  "%24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, "     \
  "%46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63 "                         \
  "}"

// d[64x128] (+)= a[64x8] . b[128x8]^T; A fragment in registers: rows lane/4 (+8), columns lane%4 (+4) of the warp's
// 16-row slice
__device__ __forceinline__ void wgmma_tf32_rs(float (&d)[64], const uint32_t (&a)[4], uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " TFB200_D64 ", {%64, %65, %66, %67}, %68, p, 1, 1;\n\t}"
      : TFB200_ACC64
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(accumulate)
      : "memory");
}
// the same product with A read from a K-major shared-memory tile through its descriptor
__device__ __forceinline__ void wgmma_tf32_ss(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " TFB200_D64 ", %64, %65, p, 1, 1;\n\t}"
      : TFB200_ACC64
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}
#undef TFB200_ACC64
#undef TFB200_D64

// keeps the compiler from touching the accumulators while a wgmma is in flight
__device__ __forceinline__ void fence_acc(float (&d)[64]) {
#pragma unroll
  for (int i = 0; i < 64; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// MODE linear: y = epi(x . w^T + bias)   accumulator [out rows, out cols]
// MODE wgrad:  dw += dy^T . x            accumulator [N, K]; token axis split into `splits` slabs, TMA reduce-add into dw
// "a" / "b" index 128-wide blocks of the accumulator rows / columns; k_blocks counts 32-wide contraction blocks.
enum { kModeLinear = 0, kModeWgrad = 1 };
// Epilogues of the linear mode, on v = acc + bias at output element (row, col), idx = row * cols + col:
//   none          v
//   relu          max(v, 0)
//   relu_dropout  (v > 0 && keep_elem(seed, idx)) ? v * inv_keep : 0     -- relu_dropout_fwd_kernel's mask, bit for
//                 bit; seed == nullptr (eval) is plain ReLU
//   dropout_grad  h[idx] > 0 ? v * inv_keep : 0                          -- relu_dropout_bwd_kernel on the product
enum { kEpiNone = 0, kEpiRelu = 1, kEpiReluDropout = 2, kEpiDropoutGrad = 3 };

struct Epilogue {
  const float* bias;       // [cols] or nullptr
  const float* h;          // dropout_grad: the forward's [rows, cols] output
  const int64_t* seed;     // relu_dropout: device seed, nullptr in eval mode
  int64_t rows;
  int cols;
  float inv_keep;
  uint32_t keep_thresh;
};

template <int MODE, int EPI>
__global__ void __launch_bounds__(THREADS, 1)
tf32_gemm_kernel(const __grid_constant__ CUtensorMap map_a, const __grid_constant__ CUtensorMap map_b,
                 const __grid_constant__ CUtensorMap map_y, const Epilogue ep, int a_tiles, int b_tiles, int k_blocks,
                 int splits) {
  constexpr bool MN = (MODE == kModeWgrad);   // both tiles staged [32 contraction rows][128]
  extern __shared__ unsigned char smem_dyn[];
  const uint32_t base = (smem_u32(smem_dyn) + 1023u) & ~1023u;          // SWIZZLE_128B tiles need 1024-byte alignment
  const uint32_t s_a = base;                                            // [STAGES][16 KB]
  const uint32_t s_b = s_a + STAGES * TILE_BYTES;                       // [STAGES][16 KB]
  const uint32_t s_t = s_b + STAGES * TILE_BYTES;                       // [2][16 KB] transposed B (wgrad)
  const uint32_t s_c = s_t + 2 * TILE_BYTES;                            // [4][16 KB] epilogue staging
  const uint32_t bar_full = s_c + OUT_BYTES, bar_empty = bar_full + 8 * STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int total_tiles = a_tiles * b_tiles * splits;     // work units: (output tile, contraction slab)

  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(bar_full + 8 * i, 1);
      mbar_init(bar_empty + 8 * i, CONSUMERS / 32);                     // one arrival per consumer warp
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp == CONSUMERS / 32) {
    // ===== TMA producer =====
    if (lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
        const int tile = t / splits, slab = t - tile * splits;
        const int a_blk = tile / b_tiles, b_blk = tile - a_blk * b_tiles;
        const int kb0 = int(int64_t(k_blocks) * slab / splits), kb1 = int(int64_t(k_blocks) * (slab + 1) / splits);
        for (int kb = kb0; kb < kb1; ++kb) {
          mbar_wait(bar_empty + 8 * stage, phase ^ 1);
          const uint32_t bar = bar_full + 8 * stage;
          mbar_expect_tx(bar, 2 * TILE_BYTES);
          if (MN) {
            tma_load_2d(s_a + stage * TILE_BYTES, &map_a, bar, a_blk * BM, kb * BK);
            tma_load_2d(s_b + stage * TILE_BYTES, &map_b, bar, b_blk * BN, kb * BK);
          } else {
            tma_load_2d(s_a + stage * TILE_BYTES, &map_a, bar, kb * BK, a_blk * BM);
            tma_load_2d(s_b + stage * TILE_BYTES, &map_b, bar, kb * BK, b_blk * BN);
          }
          if (++stage == STAGES) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===== consumers =====
  const int g = lane >> 2, tq = lane & 3;
  const int r0 = (warp >> 2) * 64 + (warp & 3) * 16 + g;                // accumulator rows r0 and r0 + 8
  const uint64_t seed = (EPI == kEpiReluDropout && ep.seed != nullptr) ? uint64_t(__ldg(ep.seed)) : 0;
  int stage = 0;
  uint32_t phase = 0, kcount = 0;
  for (int t = blockIdx.x; t < total_tiles; t += gridDim.x) {
    const int tile = t / splits, slab = t - tile * splits;
    const int a_blk = tile / b_tiles, b_blk = tile - a_blk * b_tiles;
    const int kb0 = int(int64_t(k_blocks) * slab / splits), kb1 = int(int64_t(k_blocks) * (slab + 1) / splits);
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    if (MODE == kModeLinear) {
      const uint32_t a_rows = uint32_t(warp >> 2) * 64 * 128;           // this warpgroup's 64 rows of the X tile
      int held = -1;                                                     // slot read by the wgmma group in flight
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(bar_full + 8 * stage, phase);
        fence_acc(acc);
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
        const uint64_t adesc = smem_desc(s_a + stage * TILE_BYTES + a_rows), bdesc = smem_desc(s_b + stage * TILE_BYTES);
#pragma unroll
        for (int ks = 0; ks < BK / 8; ++ks)                              // k step = 32 bytes = 2 desc units
          wgmma_tf32_ss(acc, adesc + 2 * ks, bdesc + 2 * ks, ((kb - kb0) | ks) ? 1u : 0u);
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 1;" ::: "memory");  // the previous k-block's group has retired
        fence_acc(acc);
        if (held >= 0) {
          __syncwarp();
          if (lane == 0) mbar_arrive(bar_empty + 8 * held);
        }
        held = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
      fence_acc(acc);
      if (held >= 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * held);
      }
    } else {
      for (int kb = kb0; kb < kb1; ++kb) {
        mbar_wait(bar_full + 8 * stage, phase);
        const uint32_t sa = s_a + stage * TILE_BYTES;
        // [32 tokens][128 k] -> [128 k][32 tokens] swizzled; double-buffered: the barrier below also orders the
        // wgmma of step kcount - 2 (both warpgroups waited for it before this step's barrier) before this overwrite
        const uint32_t sb = s_b + stage * TILE_BYTES, dst = s_t + (kcount++ & 1) * TILE_BYTES;
        {
          const int row = threadIdx.x & (BN - 1), c0 = (threadIdx.x >> 7) * 4;
#pragma unroll
          for (int c = c0; c < c0 + 4; ++c) {
            uint32_t v[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) v[j] = lds(sb + uint32_t((4 * c + j) * BN * 4 + row * 4));
            asm volatile("st.shared.v4.b32 [%0], {%1, %2, %3, %4};" ::"r"(dst + sw128(row, 4 * c)), "r"(v[0]),
                         "r"(v[1]), "r"(v[2]), "r"(v[3])
                         : "memory");
          }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to wgmma
        asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
        // A fragment from the MN-major [32 tokens][128 n] tile; the registers stay live until the group retires,
        // so this loop waits for its group before the next fragment load (wait_group 0)
        uint32_t a[BK / 8][4];
#pragma unroll
        for (int ks = 0; ks < BK / 8; ++ks) {
          const int k = ks * 8 + tq;
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            const int r = r0 + 8 * (j & 1), kk = k + 4 * (j >> 1);
            a[ks][j] = lds(sa + uint32_t(kk * BM * 4 + r * 4));
          }
        }
        fence_acc(acc);
        asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
        const uint64_t bdesc = smem_desc(dst);
#pragma unroll
        for (int ks = 0; ks < BK / 8; ++ks) wgmma_tf32_rs(acc, a[ks], bdesc + 2 * ks, ((kb - kb0) | ks) ? 1u : 0u);
        asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
        asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory");
        fence_acc(acc);
        __syncwarp();
        if (lane == 0) mbar_arrive(bar_empty + 8 * stage);              // frees the smem slot
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }

    // ===== epilogue: registers -> (+bias, epilogue op) -> swizzled smem -> TMA store =====
    if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // last tile's stores read
    asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
    const int64_t row_base = int64_t(a_blk) * BM;
    const int col_base = b_blk * BN;
#pragma unroll
    for (int i = 0; i < 64; i += 2) {
      const int r = r0 + 8 * ((i >> 1) & 1), c = (i >> 2) * 8 + tq * 2;   // columns c, c + 1
      float v0 = acc[i], v1 = acc[i + 1];
      if (MODE == kModeLinear) {
        if (ep.bias != nullptr) {
          const float2 b = __ldg(reinterpret_cast<const float2*>(ep.bias + col_base + c));
          v0 += b.x;
          v1 += b.y;
        }
        const int64_t row = row_base + r, idx = row * ep.cols + col_base + c;
        if (EPI == kEpiRelu || (EPI == kEpiReluDropout && ep.seed == nullptr)) {
          v0 = fmaxf(v0, 0.f);
          v1 = fmaxf(v1, 0.f);
        } else if (EPI == kEpiReluDropout) {
          v0 = (v0 > 0.f && keep_elem(seed, uint64_t(idx), ep.keep_thresh)) ? v0 * ep.inv_keep : 0.f;
          v1 = (v1 > 0.f && keep_elem(seed, uint64_t(idx) + 1, ep.keep_thresh)) ? v1 * ep.inv_keep : 0.f;
        } else if (EPI == kEpiDropoutGrad) {
          const float2 h = row < ep.rows ? __ldg(reinterpret_cast<const float2*>(ep.h + idx)) : make_float2(0.f, 0.f);
          v0 = h.x > 0.f ? v0 * ep.inv_keep : 0.f;
          v1 = h.y > 0.f ? v1 * ep.inv_keep : 0.f;
        }
      }
      asm volatile("st.shared.v2.f32 [%0], {%1, %2};" ::"r"(s_c + (c >> 5) * TILE_BYTES + sw128(r, c)), "f"(v0), "f"(v1)
                   : "memory");
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");       // generic-proxy writes -> visible to the TMA unit
    asm volatile("bar.sync 1, %0;" ::"n"(CONSUMERS) : "memory");
    if (threadIdx.x == 0) {
      const int row0 = a_blk * BM, col0 = b_blk * BN;
#pragma unroll
      for (int ch = 0; ch < BN / 32; ++ch) {
        if (MODE == kModeWgrad) tma_reduce_add_2d(&map_y, s_c + ch * TILE_BYTES, col0 + 32 * ch, row0);
        else tma_store_2d(&map_y, s_c + ch * TILE_BYTES, col0 + 32 * ch, row0);
      }
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
  }
  if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // all stores land before exit
}

// wt[K][N] = w[N][K]: the dgrad's weight operand in the linear mode's K-major layout (at most 1 MB per call)
__global__ void __launch_bounds__(256) transpose_kernel(const float* __restrict__ w, float* __restrict__ wt, int N, int K) {
  __shared__ float tile[32][33];
  const int k0 = blockIdx.x * 32, n0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += 8) tile[j][threadIdx.x] = w[int64_t(n0 + j) * K + k0 + threadIdx.x];
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += 8) wt[int64_t(k0 + j) * N + n0 + threadIdx.x] = tile[threadIdx.x][j];
}

// ---- host side ----------------------------------------------------------------------------------------------
// row-major [rows, cols] fp32 matrix; box = 32 columns x 128 rows with 128-byte swizzle (K-major tiles, output
// chunks), or 128 columns x 32 rows unswizzled (the [32 contraction rows][128] tiles of an MN-major operand)
static bool make_map(CUtensorMap* map, const float* ptr, int64_t rows, int64_t cols, bool mn_major = false) {
  tfb200::EncodeTiledFn fn = tfb200::tensor_map_encoder();
  if (!fn) return false;
  const cuuint64_t dims[2] = {cuuint64_t(cols), cuuint64_t(rows)};
  const cuuint64_t strides[1] = {cuuint64_t(cols) * 4};
  const cuuint32_t box[2] = {mn_major ? 128u : 32u, mn_major ? 32u : 128u};
  const cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(ptr), dims, strides, box, estr,
            CU_TENSOR_MAP_INTERLEAVE_NONE, mn_major ? CU_TENSOR_MAP_SWIZZLE_NONE : CU_TENSOR_MAP_SWIZZLE_128B,
            CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int sm_count() {
  static std::atomic<int> cached{0};
  int v = cached.load(std::memory_order_relaxed);
  if (v == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess ||
        v <= 0)
      v = 132;
    cached.store(v, std::memory_order_relaxed);
  }
  return v;
}

}  // namespace gemm
}  // namespace tfb200

using namespace tfb200::gemm;

static bool misaligned(const void* a, const void* b, const void* c, const void* d = nullptr, const void* e = nullptr) {
  return ((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b) | reinterpret_cast<uintptr_t>(c) |
           reinterpret_cast<uintptr_t>(d) | reinterpret_cast<uintptr_t>(e)) & 15u) != 0;
}

template <int MODE, int EPI>
static int launch(const CUtensorMap& ma, const CUtensorMap& mb, const CUtensorMap& mo, const Epilogue& ep, int a_tiles,
                  int b_tiles, int k_blocks, int splits, cudaStream_t st) {
  static std::atomic<bool> attr_set{false};
  if (!attr_set.load()) {
    cudaError_t e = cudaFuncSetAttribute(tf32_gemm_kernel<MODE, EPI>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES);
    if (e != cudaSuccess) return int(e);
    attr_set.store(true);
  }
  const int64_t units = int64_t(a_tiles) * b_tiles * splits;
  const unsigned grid = unsigned(units < sm_count() ? units : sm_count());
  tf32_gemm_kernel<MODE, EPI><<<grid, THREADS, SMEM_BYTES, st>>>(ma, mb, mo, ep, a_tiles, b_tiles, k_blocks, splits);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

// y[M, N] = epi(x[M, K] . w[N, K]^T + bias) in the linear mode
template <int EPI>
static int linear(const float* x, const float* w, float* y, const Epilogue& ep, int64_t M, int N, int K, cudaStream_t st) {
  CUtensorMap mx, mw, my;
  if (!make_map(&mx, x, M, K) || !make_map(&mw, w, N, K) || !make_map(&my, y, M, N)) return -7;
  return launch<kModeLinear, EPI>(mx, mw, my, ep, int((M + BM - 1) / BM), N / BN, K / BK, 1, st);
}

static Epilogue make_epilogue(const float* bias, int64_t M, int N) {
  return Epilogue{bias, nullptr, nullptr, M, N, 1.f, 0xFFFFFFFFu};
}

extern "C" int tfb200_tf32_linear_supported(int64_t M, int N, int K) {
  return (M >= 1 && N >= BN && N % BN == 0 && K >= BN && K % BN == 0) ? 1 : 0;     // K % 128: dgrad / wgrad tile it too
}

extern "C" int tfb200_tf32_linear_f32(const float* x, const float* w, const float* bias, float* y, int64_t M, int N,
                                      int K, int relu, void* stream) {
  if (!x || !w || !y) return -1;
  if (M < 1 || N % BN || K % BK || N < BN || K < BK) return -5;
  if (misaligned(x, w, y, bias)) return -6;
  const Epilogue ep = make_epilogue(bias, M, N);
  return relu ? linear<kEpiRelu>(x, w, y, ep, M, N, K, cudaStream_t(stream))
              : linear<kEpiNone>(x, w, y, ep, M, N, K, cudaStream_t(stream));
}

extern "C" int tfb200_tf32_linear_relu_dropout_f32(const float* x, const float* w, const float* bias,
                                                   const int64_t* seed_dev, float* h, int64_t M, int N, int K,
                                                   float keep_prob, int training, void* stream) {
  if (!x || !w || !h || (training && !seed_dev)) return -1;
  if (M < 1 || N % BN || K % BK || N < BN || K < BK || (training && !(keep_prob > 0.f && keep_prob <= 1.f))) return -5;
  if (misaligned(x, w, h, bias)) return -6;
  Epilogue ep = make_epilogue(bias, M, N);
  if (training) {
    ep.seed = seed_dev;
    ep.inv_keep = 1.f / keep_prob;
    ep.keep_thresh = tfb200::keep_threshold(keep_prob);
  }
  return linear<kEpiReluDropout>(x, w, h, ep, M, N, K, cudaStream_t(stream));
}

// dx[M, K] = dy[M, N] . w[N, K] as the linear mode on wt = w^T [K, N]; h != nullptr applies the dropout gradient
static int dgrad(const float* dy, const float* w, float* wt, const float* h, float* dx, int64_t M, int N, int K,
                 float inv_keep, cudaStream_t st) {
  if (!dy || !w || !wt || !dx) return -1;
  if (M < 1 || N % BK || K % BN || N < BK || K < BN) return -5;
  if (misaligned(dy, w, wt, dx, h)) return -6;
  transpose_kernel<<<dim3(K / 32, N / 32), dim3(32, 8), 0, st>>>(w, wt, N, K);
  msda_b200_count_launches(1);
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return int(e);
  Epilogue ep = make_epilogue(nullptr, M, K);
  if (h == nullptr) return linear<kEpiNone>(dy, wt, dx, ep, M, K, N, st);
  ep.h = h;
  ep.inv_keep = inv_keep;
  return linear<kEpiDropoutGrad>(dy, wt, dx, ep, M, K, N, st);
}

extern "C" int tfb200_tf32_linear_dgrad_f32(const float* dy, const float* w, float* wt, float* dx, int64_t M, int N,
                                            int K, void* stream) {
  return dgrad(dy, w, wt, nullptr, dx, M, N, K, 1.f, cudaStream_t(stream));
}

extern "C" int tfb200_tf32_linear_dgrad_relu_dropout_f32(const float* dy, const float* w, float* wt, const float* h,
                                                         float* ga, int64_t M, int N, int K, float keep_prob,
                                                         int training, void* stream) {
  if (!h) return -1;
  if (training && !(keep_prob > 0.f && keep_prob <= 1.f)) return -5;
  return dgrad(dy, w, wt, h, ga, M, N, K, training ? 1.f / keep_prob : 1.f, cudaStream_t(stream));
}

extern "C" int tfb200_tf32_linear_wgrad_f32(const float* dy, const float* x, float* dw, int64_t M, int N, int K,
                                            void* stream) {
  if (!dy || !x || !dw) return -1;
  if (M < 1 || N % BM || K % BN || N < BM || K < BN) return -5;
  if (misaligned(dy, x, dw)) return -6;
  cudaStream_t st = cudaStream_t(stream);
  cudaError_t e = cudaMemsetAsync(dw, 0, size_t(N) * K * 4, st);       // the slabs are ADDED into dw
  if (e != cudaSuccess) return int(e);
  CUtensorMap ma, mb, mo;
  if (!make_map(&ma, dy, M, N, true) || !make_map(&mb, x, M, K, true) || !make_map(&mo, dw, N, K)) return -7;
  const int m_tiles = N / BM, n_tiles = K / BN, k_blocks = int((M + BK - 1) / BK);
  int splits = sm_count() / (m_tiles * n_tiles);
  if (splits < 1) splits = 1;
  if (splits > k_blocks) splits = k_blocks;
  return launch<kModeWgrad, kEpiNone>(ma, mb, mo, make_epilogue(nullptr, N, K), m_tiles, n_tiles, k_blocks, splits, st);
}
