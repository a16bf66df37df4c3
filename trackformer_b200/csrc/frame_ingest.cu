// Frame ingest: uint8 H x W x 3 video frame -> antialiased bilinear resize -> normalised fp32 3 x h x w, one launch (sm_90a).
//
// Reference: what the sequence datasets do per frame on the host (src/trackformer/datasets/tracking/mot17_sequence.py:68-81
// through datasets/coco.py:270-312 and datasets/transforms.py:115-145, 381-383, 457-463): Pillow's bilinear resize of
// the 8-bit image, to_tensor (byte / 255) and Normalize(mean, std).  Pillow's 8-bit resampler is integer arithmetic, so
// this kernel is bit-identical to it, not close to it:
//   * per axis a table row {lo, cnt, k_0 .. k_{ksize-1}} per output index, built by the host in double and quantised to
//     22 fractional bits (frame_ingest.py); one pass is  byte = clamp((2^21 + sum_j pixel[lo + j] * k_j) >> 22, 0, 255)
//     in 32-bit integers (255 * 2^22 < 2^31);
//   * the horizontal pass runs first and is rounded to a byte before the vertical pass, as Pillow rounds its
//     intermediate image; an axis whose length does not change has no table and is skipped, not run with unit weights;
//   * the last byte goes through a 3 x 256 fp32 table made by the host with the reference's own torch ops, so the kernel
//     takes no floating-point rounding decision at all.
//
// One fused kernel: a block owns a 64-column x tile_h-row output tile.  It stages the tile's table rows in shared
// memory, runs the horizontal pass for the input rows the tile's vertical footprint covers into a uint8 shared-memory
// tile (the intermediate image never exists in global memory), then the vertical pass and the look-up from there.
// The input is interleaved bytes, the output planar floats: output rows are written as 16-byte vectors whose phase
// follows each row's own address (a 1333-float row stride moves it from row to row), scalars only at the tile's edges.
// ksize is a runtime value: the launcher derives the most input rows a tile can need from the axis scale and halves
// tile_h until the footprint fits in shared memory.  The destination has row and plane strides, so the same kernel
// writes one image of a zero-padded batch.
#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "launch_counter.h"

namespace {

constexpr int kTileW = 64;                 // output columns per block
constexpr int kMaxTileH = 16;              // output rows per block (halved for strong vertical reductions)
constexpr int kThreads = 256;
constexpr int kPitch = kTileW * 3;         // bytes per row of the shared-memory tile (interleaved RGB)
constexpr int kChunks = kTileW / 4 + 1;    // 16-byte store slots per output row: 16 aligned ones + a split edge pair
constexpr int kBits = 22;                  // fractional bits of the quantised weights (Pillow's PRECISION_BITS)
constexpr int kMaxSmem = 200 * 1024;

__device__ __forceinline__ int to_byte(int acc) { return min(max(acc >> kBits, 0), 255); }

__global__ void __launch_bounds__(kThreads)
frame_ingest_kernel(const uint8_t* __restrict__ src, int64_t src_row_stride, const int32_t* __restrict__ xtab, int ksx,
                    const int32_t* __restrict__ ytab, int ksy, const float* __restrict__ lut, float* __restrict__ dst,
                    int64_t dst_row_stride, int64_t dst_plane_stride, int h, int w, int tile_h, int rows_cap) {
  extern __shared__ int smem[];
  int* xlo = smem;
  int* xcnt = xlo + kTileW;
  int* ylo = xcnt + kTileW;
  int* ycnt = ylo + kMaxTileH;
  int* xk = ycnt + kMaxTileH;
  int* yk = xk + kTileW * ksx;
  uint8_t* tile = reinterpret_cast<uint8_t*>(yk + tile_h * ksy);

  const int tid = threadIdx.x;
  const int x0 = blockIdx.x * kTileW, y0 = blockIdx.y * tile_h;
  const int tw = min(kTileW, w - x0), th = min(tile_h, h - y0);

  // ---- this tile's table rows
  if (xtab != nullptr) {
    const int rw = 2 + ksx;
    for (int e = tid; e < tw * rw; e += kThreads) {
      const int i = e / rw, f = e - i * rw;
      const int v = __ldg(xtab + int64_t(x0) * rw + e);
      if (f == 0) xlo[i] = v;
      else if (f == 1) xcnt[i] = min(v, ksx);
      else xk[i * ksx + f - 2] = v;
    }
  }
  if (ytab != nullptr) {
    const int rw = 2 + ksy;
    for (int e = tid; e < th * rw; e += kThreads) {
      const int i = e / rw, f = e - i * rw;
      const int v = __ldg(ytab + int64_t(y0) * rw + e);
      if (f == 0) ylo[i] = v;
      else if (f == 1) ycnt[i] = min(v, ksy);
      else yk[i * ksy + f - 2] = v;
    }
  }
  __syncthreads();

  // ---- horizontal pass (or a plain copy) of the input rows under the tile -> uint8 tile[row][x][c]
  const int ry0 = ytab != nullptr ? ylo[0] : y0;
  const int nrows = ytab != nullptr ? min(ylo[th - 1] + ycnt[th - 1] - ry0, rows_cap) : th;
  for (int e = tid; e < nrows * kPitch; e += kThreads) {
    const int r = e / kPitch, q = e - r * kPitch;
    if (q >= tw * 3) continue;
    const int x = q / 3, c = q - x * 3;
    const uint8_t* row = src + int64_t(ry0 + r) * src_row_stride;
    int v;
    if (xtab != nullptr) {
      const uint8_t* p = row + xlo[x] * 3 + c;
      const int* k = xk + x * ksx;
      const int n = xcnt[x];
      int acc = 1 << (kBits - 1);
      for (int j = 0; j < n; ++j) acc += int(__ldg(p + 3 * j)) * k[j];
      v = to_byte(acc);
    } else {
      v = __ldg(row + (x0 + x) * 3 + c);
    }
    tile[e] = uint8_t(v);
  }
  __syncthreads();

  // ---- vertical pass + look-up, four neighbouring columns per item, stored as one aligned 16-byte vector
  for (int it = tid; it < 3 * th * kChunks; it += kThreads) {
    const int k = it % kChunks, rc = it / kChunks;
    const int yy = rc % th, c = rc / th;
    float* out = dst + c * dst_plane_stride + int64_t(y0 + yy) * dst_row_stride + x0;
    const int phase = int((reinterpret_cast<uintptr_t>(out) >> 2) & 3);
    const int xs = 4 * k - phase;                        // first column of this slot, relative to the tile
    if (xs >= tw) continue;
    int acc[4];
    if (ytab != nullptr) {
      const int r0 = ylo[yy] - ry0;
      const int n = min(ycnt[yy], nrows - r0);
      const int* kk = yk + yy * ksy;
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] = 1 << (kBits - 1);
      for (int j = 0; j < n; ++j) {
        const uint8_t* t = tile + (r0 + j) * kPitch + c;
        const int wj = kk[j];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const int xr = min(max(xs + i, 0), tw - 1);
          acc[i] += int(t[xr * 3]) * wj;
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] = to_byte(acc[i]);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i) acc[i] = tile[yy * kPitch + min(max(xs + i, 0), tw - 1) * 3 + c];
    }
    float v[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) v[i] = __ldg(lut + c * 256 + acc[i]);
    if (xs >= 0 && xs + 4 <= tw) {
      *reinterpret_cast<float4*>(out + xs) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int i = 0; i < 4; ++i)
        if (xs + i >= 0 && xs + i < tw) out[xs + i] = v[i];
    }
  }
}

}  // namespace

extern "C" int tfb200_frame_ingest_u8_f32(const uint8_t* src, int64_t src_row_stride, int H, int W, const int32_t* xtab,
                                          int ksize_x, int cnt_max_x, const int32_t* ytab, int ksize_y, int cnt_max_y,
                                          const float* lut, float* dst, int64_t dst_row_stride,
                                          int64_t dst_plane_stride, int h, int w, void* stream) {
  if (!src || !lut || !dst) return TFB200_E_NULLPTR;
  if (H <= 0 || W <= 0 || h <= 0 || w <= 0 || src_row_stride < int64_t(3) * W || dst_row_stride < w ||
      dst_plane_stride <= 0)
    return TFB200_E_SHAPE;
  if (xtab ? (ksize_x < 1 || cnt_max_x < 1 || cnt_max_x > ksize_x) : w != W) return TFB200_E_SHAPE;
  if (ytab ? (ksize_y < 1 || cnt_max_y < 1 || cnt_max_y > ksize_y) : h != H) return TFB200_E_SHAPE;
  if ((reinterpret_cast<uintptr_t>(dst) & 3) != 0) return TFB200_E_SHAPE;
  const int ksx = xtab ? ksize_x : 0, ksy = ytab ? ksize_y : 0;

  // input rows under tile_h output rows: lo moves by at most ceil((tile_h - 1) * H / h), the last row adds its cnt
  int tile_h = kMaxTileH, rows_cap = 0;
  size_t smem = 0;
  while (true) {
    rows_cap = ytab ? int(ceil(double(tile_h - 1) * H / h)) + cnt_max_y + 1 : tile_h;
    smem = size_t(2 * kTileW + 2 * kMaxTileH + kTileW * ksx + tile_h * ksy) * sizeof(int) + size_t(rows_cap) * kPitch;
    if (smem <= size_t(kMaxSmem) || tile_h == 1) break;
    tile_h /= 2;
  }
  const int64_t grid_y = (int64_t(h) + tile_h - 1) / tile_h;
  if (smem > size_t(kMaxSmem) || grid_y > 65535) return TFB200_E_SHAPE;
  if (smem > 48 * 1024) {
    const cudaError_t e = cudaFuncSetAttribute(frame_ingest_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    if (e != cudaSuccess) return int(e);
  }
  const dim3 grid((w + kTileW - 1) / kTileW, unsigned(grid_y));
  frame_ingest_kernel<<<grid, kThreads, smem, cudaStream_t(stream)>>>(src, src_row_stride, xtab, ksx, ytab, ksy, lut, dst,
                                                                      dst_row_stride, dst_plane_stride, h, w, tile_h,
                                                                      rows_cap);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}
