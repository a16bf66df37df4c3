// Shared device helpers for the sm_90a multi-scale deformable attention kernels.
//
// Semantics follow the reference CUDA op (timmeinhardt/trackformer,
// src/trackformer/models/ops/src/cuda/ms_deform_im2col_cuda.cuh):
//   pixel coords       x = loc_x*W - 0.5, y = loc_y*H - 0.5            (:227-228)
//   sample is live iff y > -1 && x > -1 && y < H && x < W              (:229)
//   corners outside [0,H-1]x[0,W-1] read as zero                       (:38-61)
// None of the reference's code is reused; the kernels are organised differently
// (one fused pass, no `columns` tensor, vector lanes per head, sub-warp reductions).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace msda {

// ---- fixed-size channel packs: 16-byte lanes whenever the layout allows -------------
template <typename T, int VEC> struct Pack { T v[VEC]; };

template <typename T, int VEC>
__device__ __forceinline__ Pack<T, VEC> pack_zero() {
  Pack<T, VEC> r;
#pragma unroll
  for (int i = 0; i < VEC; ++i) r.v[i] = T(0);
  return r;
}

// read-only (non-coherent) global load of one pack
template <typename T, int VEC>
__device__ __forceinline__ Pack<T, VEC> ldg_pack(const T* __restrict__ p) {
  Pack<T, VEC> r;
  if constexpr (sizeof(T) * VEC == 16) {
    const uint4 t = __ldg(reinterpret_cast<const uint4*>(p));
    *reinterpret_cast<uint4*>(&r) = t;
  } else if constexpr (sizeof(T) * VEC == 8 && VEC > 1) {
    const uint2 t = __ldg(reinterpret_cast<const uint2*>(p));
    *reinterpret_cast<uint2*>(&r) = t;
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) r.v[i] = __ldg(p + i);
  }
  return r;
}

template <typename T, int VEC>
__device__ __forceinline__ void st_pack(T* __restrict__ p, const Pack<T, VEC>& r) {
  if constexpr (sizeof(T) * VEC == 16) {
    *reinterpret_cast<uint4*>(p) = *reinterpret_cast<const uint4*>(&r);
  } else if constexpr (sizeof(T) * VEC == 8 && VEC > 1) {
    *reinterpret_cast<uint2*>(p) = *reinterpret_cast<const uint2*>(&r);
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) p[i] = r.v[i];
  }
}

// Fire-and-forget reduction into global memory (no return value -> RED, not ATOM).
// fp32 x4 uses the sm_90+ 128-bit vector reduction: one L2 transaction per lane
// instead of four.
template <typename T, int VEC>
__device__ __forceinline__ void red_add_pack(T* p, const Pack<T, VEC>& r) {
  if constexpr (sizeof(T) == 4 && VEC == 4) {
    asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p),
                 "f"(r.v[0]), "f"(r.v[1]), "f"(r.v[2]), "f"(r.v[3])
                 : "memory");
  } else if constexpr (sizeof(T) == 4 && VEC == 2) {
    asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(r.v[0]),
                 "f"(r.v[1])
                 : "memory");
  } else {
#pragma unroll
    for (int i = 0; i < VEC; ++i) atomicAdd(p + i, r.v[i]);
  }
}

template <typename T> __device__ __forceinline__ T floor_t(T x);
template <> __device__ __forceinline__ float floor_t<float>(float x) { return floorf(x); }
template <> __device__ __forceinline__ double floor_t<double>(double x) { return floor(x); }

// Everything a sample needs besides the value rows themselves.
template <typename T>
struct Tap {
  T w1, w2, w3, w4;    // bilinear weights of (y0,x0) (y0,x1) (y1,x0) (y1,x1)
  T lx, ly;            // fractional parts (backward needs them for d/dx, d/dy)
  int o1, o2, o3, o4;  // element offsets of the four corner rows inside the level slab
  bool k1, k2, k3, k4; // corner inside the image?
  bool live;           // reference validity test
};

// stride = M*D (elements between neighbouring pixels)
template <typename T>
__device__ __forceinline__ Tap<T> make_tap(T locx, T locy, int H, int W, int stride) {
  Tap<T> t;
  const T x = locx * T(W) - T(0.5);
  const T y = locy * T(H) - T(0.5);
  t.live = (y > T(-1)) && (x > T(-1)) && (y < T(H)) && (x < T(W));
  const T fx = floor_t(x), fy = floor_t(y);
  const int x0 = int(fx), y0 = int(fy);
  t.lx = x - fx;
  t.ly = y - fy;
  const T hx = T(1) - t.lx, hy = T(1) - t.ly;
  t.w1 = hy * hx;
  t.w2 = hy * t.lx;
  t.w3 = t.ly * hx;
  t.w4 = t.ly * t.lx;
  const bool xl = x0 >= 0, xh = x0 + 1 <= W - 1, yl = y0 >= 0, yh = y0 + 1 <= H - 1;
  t.k1 = t.live && yl && xl;
  t.k2 = t.live && yl && xh;
  t.k3 = t.live && yh && xl;
  t.k4 = t.live && yh && xh;
  t.o1 = (y0 * W + x0) * stride;
  t.o2 = t.o1 + stride;
  t.o3 = t.o1 + W * stride;
  t.o4 = t.o3 + stride;
  return t;
}

}  // namespace msda
