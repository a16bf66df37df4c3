// Segmentation masks of the online tracker's active tracks, resolved in one launch (sm_90a).
//
// Reference: src/trackformer/models/detr_segmentation.py:219-253 (PostProcessSegm with return_probs=True) followed by
// src/trackformer/models/tracker.py:509-521.  The reference upsamples the stride-4 mask logits of EVERY query row
// bilinearly to the padded input size, applies the sigmoid, copies all of it to the host, crops each row to the image
// and nearest-resizes it to the original size; at the end of the frame the active tracks' masks are stacked (a track
// that did not take a new mask keeps the boolean mask of the previous frame, promoted to 0 / 1 by torch.stack) and every
// pixel goes to the FIRST track of maximal value when that value exceeds 0.5.
//
// Here the same value is computed per output pixel, for the active tracks only, and the resolved masks leave the device
// as one int32 label map (track id, or -1 for background):
//   * the nearest and bilinear source indices / weights of a pixel are computed once and serve every track;
//   * the low-resolution footprint of an output tile is staged in shared memory for a chunk of tracks at a time, so the
//     number of tracks is unbounded (a footprint larger than the stage reads global memory instead);
//   * the running (best value, first position) pair of each pixel stays in registers; a strict '>' in list order keeps
//     the first maximum, so exact ties (saturated sigmoids, stale masks at exactly 1.0) resolve like torch.argmax;
//   * stale tracks cost one read of the previous label map per pixel and one lookup in a shared-memory hash table
//     (id -> list position), never a scan over the stale tracks.
// Index maths is ATen's (UpSample.h): nearest_idx with its identity and 2x cases and fp32 scale, and
// area_pixel_compute_source_index (align_corners=False) with the clamp at 0 and the "+1 if < size - 1" neighbour.  The
// interpolation and the sigmoid are evaluated in fp32 without contraction, in the order of ATen's CPU kernel.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "interp_index.h"
#include "launch_counter.h"

namespace {

constexpr int kTileW = 64;                 // output tile: 64 columns x 16 rows, 256 threads, 4 rows per thread
constexpr int kTileH = 16;
constexpr int kThreads = 256;
constexpr int kRows = kTileH / (kThreads / kTileW);
constexpr int kMaxChunk = 256;             // tracks per pass over the output tile
constexpr int kStageFloats = 8192;         // 32 KB of staged logits per pass
constexpr int kMaxSmem = 200 * 1024;
constexpr int kMaxBatch = 16;             // images per launch

using tfb200_interp::Lin;
using tfb200_interp::linear_src;
using tfb200_interp::nearest_src;

__device__ __forceinline__ unsigned slot_of(int id, int mask) {
  unsigned x = unsigned(id);
  x = (x ^ (x >> 16)) * 0x45d9f3bu;
  x = (x ^ (x >> 16)) * 0x45d9f3bu;
  return (x ^ (x >> 16)) & unsigned(mask);
}

// The images of one launch.  Image b owns the output tiles [tile_end[b - 1], tile_end[b]) of the 1-D grid; every CTA
// works on one tile of one image, so the body below is the single-image kernel with that image's arguments.
// tfb200_track_masks_f32 is the launch of one image.
// kCap is the table's capacity: 1 for a single image (a one-entry table, the image known at compile time), else
// kMaxBatch.
template <int kCap>
struct MasksBatch {
  TfbTrackMasksArgs a[kCap];
  int tiles_x[kCap];
  int tile_end[kCap];
  int hash_slots;                          // the largest stale set's table; a larger table maps ids to the same t
};

template <int kCap>
__global__ void __launch_bounds__(kThreads, 2)
track_masks_kernel(const __grid_constant__ MasksBatch<kCap> batch) {
  int b = 0;
  if (kCap > 1)
    while (int(blockIdx.x) >= batch.tile_end[b]) ++b;
  const TfbTrackMasksArgs& a = batch.a[b];
  const float* __restrict__ logits = a.logits;
  const int32_t* __restrict__ src = a.src;
  const int32_t* __restrict__ ids = a.ids;
  const int32_t* __restrict__ prev = a.prev_label;
  int32_t* __restrict__ label = a.label;
  const int T = a.T, h = a.h, w = a.w, size_h = a.size_h, size_w = a.size_w, crop_h = a.crop_h, crop_w = a.crop_w;
  const int H = a.H, W = a.W, hash_slots = batch.hash_slots;
  const int tile = int(blockIdx.x) - (b ? batch.tile_end[b - 1] : 0);
  const int tile_x = tile % batch.tiles_x[b], tile_y = tile / batch.tiles_x[b];
  extern __shared__ int smem[];
  int* hkey = smem;
  int* hval = hkey + hash_slots;
  int* csrc = hval + hash_slots;
  float* stage = reinterpret_cast<float*>(csrc + kMaxChunk);
  const int tid = threadIdx.x, tx = tid % kTileW, ty = tid / kTileW;

  // ---- stale tracks: id -> list position
  if (prev != nullptr) {
    for (int i = tid; i < hash_slots; i += kThreads) hkey[i] = -1;
    __syncthreads();
    for (int t = tid; t < T; t += kThreads) {
      if (src[t] >= 0) continue;
      const int id = ids[t];
      unsigned s = slot_of(id, hash_slots - 1);
      while (true) {
        const int old = atomicCAS(hkey + s, -1, id);
        if (old == -1 || old == id) { hval[s] = t; break; }
        s = (s + 1) & unsigned(hash_slots - 1);
      }
    }
  }

  // ---- source indices of this thread's pixels, and the tile's low-resolution footprint (indices are monotone)
  const int x0_tile = tile_x * kTileW, y0_tile = tile_y * kTileH;
  const int x_last = min(x0_tile + kTileW, W) - 1, y_last = min(y0_tile + kTileH, H) - 1;
  const int fx0 = linear_src(nearest_src(x0_tile, crop_w, W), w, size_w).i0;
  const int fx1 = linear_src(nearest_src(x_last, crop_w, W), w, size_w).i1;
  const int fy0 = linear_src(nearest_src(y0_tile, crop_h, H), h, size_h).i0;
  const int fy1 = linear_src(nearest_src(y_last, crop_h, H), h, size_h).i1;
  const int fw = fx1 - fx0 + 1, fp = (fy1 - fy0 + 1) * fw;
  const bool staged = fp <= kStageFloats;
  const int chunk = staged ? min(kMaxChunk, kStageFloats / fp) : kMaxChunk;
  const int row_stride = staged ? fw : w;

  const int x = x0_tile + tx;
  const Lin lx = linear_src(nearest_src(min(x, W - 1), crop_w, W), w, size_w);
  const int c0 = staged ? lx.i0 - fx0 : lx.i0, c1 = staged ? lx.i1 - fx0 : lx.i1;
  int r0[kRows], r1[kRows];
  float h0[kRows], h1[kRows], best[kRows];
  int pos[kRows];
#pragma unroll
  for (int r = 0; r < kRows; ++r) {
    const int y = min(y0_tile + ty + r * (kThreads / kTileW), H - 1);
    const Lin ly = linear_src(nearest_src(y, crop_h, H), h, size_h);
    r0[r] = (staged ? ly.i0 - fy0 : ly.i0) * row_stride;
    r1[r] = (staged ? ly.i1 - fy0 : ly.i1) * row_stride;
    h0[r] = ly.l0;
    h1[r] = ly.l1;
    best[r] = -1.f;                        // below every probability
    pos[r] = -1;
  }

  // ---- fresh tracks, in list order, a chunk at a time
  const int64_t plane = int64_t(h) * w;
  for (int t0 = 0; t0 < T; t0 += chunk) {
    const int n = min(chunk, T - t0);
    __syncthreads();                       // previous chunk fully consumed (and the hash table built)
    for (int i = tid; i < n; i += kThreads) csrc[i] = src[t0 + i];
    __syncthreads();
    if (staged) {
      for (int e = tid; e < n * fp; e += kThreads) {
        const int k = e / fp, q = e - k * fp;
        const int s = csrc[k];
        if (s >= 0) stage[e] = __ldg(logits + s * plane + int64_t(fy0 + q / fw) * w + fx0 + q % fw);
      }
      __syncthreads();
    }
    for (int k = 0; k < n; ++k) {
      const int s = csrc[k];
      if (s < 0) continue;
      const float* base = staged ? stage + k * fp : logits + s * plane;
#pragma unroll
      for (int r = 0; r < kRows; ++r) {
        const float a = __fadd_rn(__fmul_rn(base[r0[r] + c0], lx.l0), __fmul_rn(base[r0[r] + c1], lx.l1));
        const float b = __fadd_rn(__fmul_rn(base[r1[r] + c0], lx.l0), __fmul_rn(base[r1[r] + c1], lx.l1));
        const float v = __fadd_rn(__fmul_rn(a, h0[r]), __fmul_rn(b, h1[r]));
        const float p = 1.f / (1.f + expf(-v));
        if (p > best[r]) { best[r] = p; pos[r] = t0 + k; }
      }
    }
  }
  // (T > 0, so the first pass's barrier has also published the hash table)

  // ---- stale candidate (value exactly 1.0), threshold, label
  if (x >= W) return;
#pragma unroll
  for (int r = 0; r < kRows; ++r) {
    const int y = y0_tile + ty + r * (kThreads / kTileW);
    if (y >= H) continue;
    const int64_t o = int64_t(y) * W + x;
    if (prev != nullptr) {
      const int id = prev[o];
      if (id >= 0) {
        unsigned s = slot_of(id, hash_slots - 1);
        while (hkey[s] != -1 && hkey[s] != id) s = (s + 1) & unsigned(hash_slots - 1);
        if (hkey[s] == id) {
          const int t = hval[s];
          if (1.f > best[r] || (1.f == best[r] && t < pos[r])) { best[r] = 1.f; pos[r] = t; }
        }
      }
    }
    label[o] = best[r] > 0.5f ? ids[pos[r]] : -1;
  }
}

int next_pow2(int v) {
  int p = 64;
  while (p < v) p <<= 1;
  return p;
}

template <int kCap>
cudaError_t launch(const MasksBatch<kCap>& batch, int tiles, size_t smem, cudaStream_t s) {
  if (smem > 48 * 1024) {
    const cudaError_t e =
        cudaFuncSetAttribute(track_masks_kernel<kCap>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    if (e != cudaSuccess) return e;
  }
  track_masks_kernel<kCap><<<tiles, kThreads, smem, s>>>(batch);
  return cudaSuccess;
}

bool bad_args(const TfbTrackMasksArgs& a) {
  return a.T < 0 || a.h <= 0 || a.w <= 0 || a.size_h <= 0 || a.size_w <= 0 || a.crop_h <= 0 || a.crop_w <= 0 ||
         a.crop_h > a.size_h || a.crop_w > a.size_w || a.H <= 0 || a.W <= 0 || a.T > (1 << 24);
}

}  // namespace

extern "C" int tfb200_track_masks_batched_f32(const TfbTrackMasksArgs* args, int n, void* stream) {
  if (!args) return TFB200_E_NULLPTR;
  if (n <= 0 || n > kMaxBatch) return TFB200_E_SHAPE;
  MasksBatch<kMaxBatch> batch;
  int tiles = 0, max_stale = 0;
  for (int b = 0; b < n; ++b) {
    const TfbTrackMasksArgs& a = args[b];
    if (!a.src || !a.ids || !a.label) return TFB200_E_NULLPTR;
    if (bad_args(a)) return TFB200_E_SHAPE;
    batch.a[b] = a;
    batch.tiles_x[b] = (a.W + kTileW - 1) / kTileW;
    const int64_t own = a.T == 0 ? 0 : int64_t(batch.tiles_x[b]) * ((a.H + kTileH - 1) / kTileH);   // T == 0: untouched
    if (tiles + own > int64_t(INT32_MAX)) return TFB200_E_SHAPE;
    tiles += int(own);
    batch.tile_end[b] = tiles;
    if (a.T > 0 && a.prev_label) max_stale = a.T > max_stale ? a.T : max_stale;
  }
  for (int b = n; b < kMaxBatch; ++b) batch.tile_end[b] = tiles;
  if (tiles == 0) return 0;
  batch.hash_slots = max_stale ? next_pow2(2 * max_stale) : 0;
  const size_t smem = (size_t(2) * batch.hash_slots + kMaxChunk) * sizeof(int) + kStageFloats * sizeof(float);
  if (smem > size_t(kMaxSmem)) return TFB200_E_SHAPE;
  const cudaStream_t s = cudaStream_t(stream);
  cudaError_t e;
  if (n == 1) {
    MasksBatch<1> one;
    one.a[0] = batch.a[0];
    one.tiles_x[0] = batch.tiles_x[0];
    one.tile_end[0] = batch.tile_end[0];
    one.hash_slots = batch.hash_slots;
    e = launch(one, tiles, smem, s);
  } else {
    e = launch(batch, tiles, smem, s);
  }
  if (e != cudaSuccess) return int(e);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_track_masks_f32(const float* logits, const int32_t* src, const int32_t* ids,
                                      const int32_t* prev_label, int32_t* label, int T, int h, int w, int size_h,
                                      int size_w, int crop_h, int crop_w, int H, int W, void* stream) {
  const TfbTrackMasksArgs a = {logits, src, ids, prev_label, label, T, h, w, size_h, size_w, crop_h, crop_w, H, W};
  return tfb200_track_masks_batched_f32(&a, 1, stream);
}
