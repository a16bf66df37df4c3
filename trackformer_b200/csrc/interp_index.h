// Source indices of ATen's F.interpolate (aten/src/ATen/native/UpSample.h), shared by the kernels that reproduce it
// (track_masks.cu, mask_head.cu, panoptic_core.h) and by the g++ host builds of those routines.  All arithmetic is
// separately rounded fp32, as ATen's CPU kernels evaluate it.
#pragma once

#include <math.h>

#include "host_device.h"

namespace tfb200_interp {

#if defined(__CUDACC__)
HD_FORCEINLINE int ii_min(int a, int b) { return min(a, b); }
#else
HD_FORCEINLINE int ii_min(int a, int b) { return a < b ? a : b; }
#endif

// nearest_idx: output index o of a resize from `in` to `out` elements (mode="nearest"), with its identity and 2x cases
HD_FORCEINLINE int nearest_src(int o, int in, int out) {
  if (out == in) return o;
  if (out == 2 * in) return o >> 1;
  const float scale = float(in) / float(out);
  return ii_min(int(floorf(hd_fmul(float(o), scale))), in - 1);
}

struct Lin {
  int i0, i1;
  float l0, l1;
};

// compute_source_index_and_lambda, linear mode, align_corners=False: the two neighbours and their weights
HD_FORCEINLINE Lin linear_src(int o, int in, int out) {
  if (out == in) return {o, o, 1.f, 0.f};
  const float scale = float(in) / float(out);
  float s = hd_fsub(hd_fmul(scale, hd_fadd(float(o), 0.5f)), 0.5f);
  s = s < 0.f ? 0.f : s;
  const int i0 = ii_min(int(floorf(s)), in - 1);
  const float l1 = fminf(fmaxf(hd_fsub(s, float(i0)), 0.f), 1.f);
  return {i0, i0 + (i0 < in - 1 ? 1 : 0), hd_fsub(1.f, l1), l1};
}

// bilinear value of a row-major [.][w] plane at (ly, lx), in the order of ATen's CPU kernel
HD_FORCEINLINE float bilinear_at(const float* m, int w, const Lin& ly, const Lin& lx) {
  const float a = hd_fadd(hd_fmul(m[ly.i0 * w + lx.i0], lx.l0), hd_fmul(m[ly.i0 * w + lx.i1], lx.l1));
  const float b = hd_fadd(hd_fmul(m[ly.i1 * w + lx.i0], lx.l0), hd_fmul(m[ly.i1 * w + lx.i1], lx.l1));
  return hd_fadd(hd_fmul(a, ly.l0), hd_fmul(b, ly.l1));
}

}  // namespace tfb200_interp
