// The portability layer of the sources compiled twice: by nvcc into kernels, and by g++ into test-only host builds in
// which one "thread" runs each CTA in turn (mot_eval_core.h, mots_eval_core.h, track_step_core.h, two_stage_core.h,
// panoptic_core.h, coco_eval_core.h, coco_poly_core.h, interp_index.h, lsa_core.h).
//
// The CPU suites stand in for the GPU on one promise: the host build performs exactly the device's arithmetic.  So the
// rounding helpers are typed -- hd_f* take and return float like __f*_rn, hd_d* double like __d*_rn -- and the host
// twin is compiled with -ffp-contract=off, so that its plain operators round every operation separately too.  Where
// the two differ, the device is the product: the host follows it.
#pragma once

#include <stdint.h>

#include <type_traits>

#if defined(__CUDACC__)
#define HD_FN __device__ inline
#define HD_FORCEINLINE __device__ __forceinline__
#define HD_SYNC() __syncthreads()
#define HD_SYNCWARP() __syncwarp()
#define HD_TID (int(threadIdx.x))
#define HD_NT (int(blockDim.x))
#define HD_LANE (int(threadIdx.x) & 31)
#define HD_NLANES 32
#else
#include <string.h>
#define HD_FN inline
#define HD_FORCEINLINE inline
#define HD_SYNC() ((void)0)
#define HD_SYNCWARP() ((void)0)
#define HD_TID 0
#define HD_NT 1
#define HD_LANE 0
#define HD_NLANES 1
#endif

// ---- separately rounded arithmetic, round to nearest ----
#if defined(__CUDACC__)
HD_FORCEINLINE float hd_fadd(float a, float b) { return __fadd_rn(a, b); }
HD_FORCEINLINE float hd_fsub(float a, float b) { return __fsub_rn(a, b); }
HD_FORCEINLINE float hd_fmul(float a, float b) { return __fmul_rn(a, b); }
HD_FORCEINLINE float hd_fdiv(float a, float b) { return __fdiv_rn(a, b); }
HD_FORCEINLINE double hd_dadd(double a, double b) { return __dadd_rn(a, b); }
HD_FORCEINLINE double hd_dsub(double a, double b) { return __dsub_rn(a, b); }
HD_FORCEINLINE double hd_dmul(double a, double b) { return __dmul_rn(a, b); }
HD_FORCEINLINE double hd_ddiv(double a, double b) { return __ddiv_rn(a, b); }
#else
HD_FORCEINLINE float hd_fadd(float a, float b) { return a + b; }
HD_FORCEINLINE float hd_fsub(float a, float b) { return a - b; }
HD_FORCEINLINE float hd_fmul(float a, float b) { return a * b; }
HD_FORCEINLINE float hd_fdiv(float a, float b) { return a / b; }
HD_FORCEINLINE double hd_dadd(double a, double b) { return a + b; }
HD_FORCEINLINE double hd_dsub(double a, double b) { return a - b; }
HD_FORCEINLINE double hd_dmul(double a, double b) { return a * b; }
HD_FORCEINLINE double hd_ddiv(double a, double b) { return a / b; }
#endif

// ---- atomics on 32- and 64-bit integers (plain read-modify-write on the host); the value converts to *p's type ----
template <class T> struct hd_same { using type = T; };

// hd_atomic_add returns the old value
template <class T> HD_FN T hd_atomic_add(T* p, typename hd_same<T>::type v) {
#if defined(__CUDACC__)
  if constexpr (sizeof(T) == 8)
    return T(atomicAdd(reinterpret_cast<unsigned long long*>(p), static_cast<unsigned long long>(v)));
  else
    return atomicAdd(p, v);
#else
  const T o = *p;
  *p = o + v;
  return o;
#endif
}
template <class T> HD_FN void hd_atomic_min(T* p, typename hd_same<T>::type v) {
#if defined(__CUDACC__)
  if constexpr (sizeof(T) == 8 && std::is_signed<T>::value) atomicMin(reinterpret_cast<long long*>(p), (long long)v);
  else if constexpr (sizeof(T) == 8) atomicMin(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v);
  else atomicMin(p, v);
#else
  if (v < *p) *p = v;
#endif
}
template <class T> HD_FN void hd_atomic_max(T* p, typename hd_same<T>::type v) {
#if defined(__CUDACC__)
  if constexpr (sizeof(T) == 8 && std::is_signed<T>::value) atomicMax(reinterpret_cast<long long*>(p), (long long)v);
  else if constexpr (sizeof(T) == 8) atomicMax(reinterpret_cast<unsigned long long*>(p), (unsigned long long)v);
  else atomicMax(p, v);
#else
  if (v > *p) *p = v;
#endif
}
template <class T> HD_FN void hd_atomic_or(T* p, typename hd_same<T>::type v) {
#if defined(__CUDACC__)
  if constexpr (sizeof(T) == 8) atomicOr(reinterpret_cast<unsigned long long*>(p), static_cast<unsigned long long>(v));
  else atomicOr(p, v);
#else
  *p |= v;
#endif
}

// ---- bits ----
HD_FORCEINLINE uint32_t hd_float_bits(float f) {
#if defined(__CUDACC__)
  return __float_as_uint(f);
#else
  uint32_t u;
  memcpy(&u, &f, 4);
  return u;
#endif
}
HD_FORCEINLINE float hd_bits_float(uint32_t u) {
#if defined(__CUDACC__)
  return __uint_as_float(u);
#else
  float f;
  memcpy(&f, &u, 4);
  return f;
#endif
}
#if defined(__CUDACC__)
HD_FORCEINLINE int hd_popc(uint32_t v) { return __popc(v); }
HD_FORCEINLINE int hd_ctz(uint32_t v) { return __ffs(int(v)) - 1; }       // v != 0
HD_FORCEINLINE int hd_clz(uint32_t v) { return __clz(int(v)); }
#else
HD_FORCEINLINE int hd_popc(uint32_t v) { return __builtin_popcount(v); }
HD_FORCEINLINE int hd_ctz(uint32_t v) { return __builtin_ctz(v); }        // v != 0
HD_FORCEINLINE int hd_clz(uint32_t v) { return __builtin_clz(v); }        // v != 0
#endif
