// Source indices of ATen's F.interpolate (aten/src/ATen/native/UpSample.h), shared by the kernels that reproduce it
// (track_masks.cu, mask_head.cu, panoptic_core.h) and by the g++ host builds of those routines.  All arithmetic is
// separately rounded fp32, as ATen's CPU kernels evaluate it.
#pragma once

#if defined(__CUDACC__)
#define II_FN __device__ __forceinline__
#define ii_mul(a, b) __fmul_rn((a), (b))
#define ii_add(a, b) __fadd_rn((a), (b))
#define ii_sub(a, b) __fsub_rn((a), (b))
#else
#include <math.h>
#define II_FN static inline
#define ii_mul(a, b) ((a) * (b))
#define ii_add(a, b) ((a) + (b))
#define ii_sub(a, b) ((a) - (b))
#endif

namespace tfb200_interp {

#if defined(__CUDACC__)
II_FN int ii_min(int a, int b) { return min(a, b); }
#else
II_FN int ii_min(int a, int b) { return a < b ? a : b; }
#endif

// nearest_idx: output index o of a resize from `in` to `out` elements (mode="nearest"), with its identity and 2x cases
II_FN int nearest_src(int o, int in, int out) {
  if (out == in) return o;
  if (out == 2 * in) return o >> 1;
  const float scale = float(in) / float(out);
  return ii_min(int(floorf(ii_mul(float(o), scale))), in - 1);
}

struct Lin {
  int i0, i1;
  float l0, l1;
};

// compute_source_index_and_lambda, linear mode, align_corners=False: the two neighbours and their weights
II_FN Lin linear_src(int o, int in, int out) {
  if (out == in) return {o, o, 1.f, 0.f};
  const float scale = float(in) / float(out);
  float s = ii_sub(ii_mul(scale, ii_add(float(o), 0.5f)), 0.5f);
  s = s < 0.f ? 0.f : s;
  const int i0 = ii_min(int(floorf(s)), in - 1);
  const float l1 = fminf(fmaxf(ii_sub(s, float(i0)), 0.f), 1.f);
  return {i0, i0 + (i0 < in - 1 ? 1 : 0), ii_sub(1.f, l1), l1};
}

// bilinear value of a row-major [.][w] plane at (ly, lx), in the order of ATen's CPU kernel
II_FN float bilinear_at(const float* m, int w, const Lin& ly, const Lin& lx) {
  const float a = ii_add(ii_mul(m[ly.i0 * w + lx.i0], lx.l0), ii_mul(m[ly.i0 * w + lx.i1], lx.l1));
  const float b = ii_add(ii_mul(m[ly.i1 * w + lx.i0], lx.l0), ii_mul(m[ly.i1 * w + lx.i1], lx.l1));
  return ii_add(ii_mul(a, ly.l0), ii_mul(b, ly.l1));
}

}  // namespace tfb200_interp
