// COCO polygon ground truth as mask runs (what pycocotools 2.0's frPyObjects / rleFrPoly / rleFrBbox + merge compute
// for COCO.annToRLE, and what the reference's datasets/coco.py convert_coco_poly_to_mask decodes), written once as
// routines:
//
//   cp_edge_points  (one thread per edge)         the polygon vertices on pycocotools' 5x integer grid, checked, and
//                                                 the edge's boundary-point count
//   cp_edge_toggles (one thread per edge)         walk the edge's boundary points as rleFrPoly does and count, or
//                                                 write, the y-boundary toggles of each consecutive pair (the first
//                                                 point of an edge pairs with the last point of the previous one)
//   cp_sweep        (one thread per annotation)   the toggles of all parts of an annotation sorted by position (the
//                                                 caller's segmented sort, values = part): a part covers a pixel when
//                                                 an odd number of its toggles lie at or before it, the annotation
//                                                 when any part does; count, or write, the runs of that union
//   cp_rle_decode   (one thread per string)       a compressed COCO RLE counts string into the same runs
//   cp_mask_pixel   (one thread per output pixel) a [H][W] uint8 mask byte from its runs
//
// nvcc compiles them into csrc/coco_poly.cu's kernels (the sort: CUB), g++ (one "thread", std::sort) into the
// test-only host build tests/host_build/coco_poly_host.cpp.  The grid arithmetic is fp64 with separately rounded
// operations, as pycocotools' x86-64 build computes it: on the device through __dmul_rn / __dadd_rn / __ddiv_rn /
// __dsub_rn, on the host with -ffp-contract=off.  A contracted ys + s * t + .5 moves a boundary point on long edges.
//
// Runs are column-major like COCO RLE: (start, length) of each run of ones, pixel (y, x) at index x * h + y.
#pragma once

#include <limits.h>
#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "host_device.h"

namespace tfb200_poly {

constexpr int kThreads = 256;
constexpr double kScale = 5.0;                       // rleFrPoly's upsampling of the boundary
constexpr double kIntLimit = 2147483648.0;           // |5 x + .5| below 2^31: the grid value fits a C int

// sizes [TFB200_POLY_SIZES] int64, written by the count entry
enum {
  kSzPoints = TFB200_POLY_SIZE_POINTS, kSzToggles = TFB200_POLY_SIZE_TOGGLES, kSzStatus = TFB200_POLY_SIZE_STATUS,
  kSzBadFinite = TFB200_POLY_SIZE_BAD_FINITE, kSzBadRange = TFB200_POLY_SIZE_BAD_RANGE
};

struct PolyParams {
  const double* xy;        // [V][2] vertices of every part, parts in order
  const int64_t* part_off; // [n_parts + 1] vertex offsets; edge e joins vertex e to the next one of its part
  const int32_t* part_ann; // [n_parts] annotation of each part
  const int64_t* ann_part; // [n_ann + 1] part offsets (an annotation's parts are consecutive)
  const int32_t* ann_hw;   // [n_ann][2] h, w
  int n_parts, n_ann;
  int64_t n_edges;         // = V
};

// (int)(5 c + .5) with C's truncation toward zero; false when c is not finite or the value overflows an int
HD_FN bool cp_grid(double c, int64_t* g) {
  const double q = hd_dadd(hd_dmul(kScale, c), 0.5);
  if (!(q > -kIntLimit && q < kIntLimit)) return false;
  *g = int64_t(q);
  return true;
}

// (int)q as x86-64's cvttsd2si computes it: NaN (the 0 / 0 slope of a zero-length edge) gives INT_MIN
HD_FN int64_t cp_trunc(double q) {
  if (!(q > -kIntLimit - 1.0 && q < kIntLimit)) return INT_MIN;
  return int64_t(q);
}

// the part holding edge e: the last p with part_off[p] <= e
HD_FN int cp_part_of(const PolyParams& P, int64_t e) {
  int lo = 0, hi = P.n_parts;                        // part_off[lo] <= e < part_off[hi]
  while (hi - lo > 1) {
    const int mid = (lo + hi) >> 1;
    if (P.part_off[mid] <= e) lo = mid; else hi = mid;
  }
  return lo;
}

// one edge of rleFrPoly after the flip
struct Edge {
  int64_t xs, ys, dx, dy, n;                         // n = boundary points of the edge, max(dx, dy) + 1
  double s;
  bool flip, xmajor;
};

HD_FN Edge cp_edge(const PolyParams& P, int p, int64_t e) {
  const int64_t b = e + 1 == P.part_off[p + 1] ? P.part_off[p] : e + 1;   // x[k] = x[0]
  int64_t xs = 0, ys = 0, xe = 0, ye = 0;
  cp_grid(P.xy[2 * e], &xs); cp_grid(P.xy[2 * e + 1], &ys);
  cp_grid(P.xy[2 * b], &xe); cp_grid(P.xy[2 * b + 1], &ye);
  Edge E;
  E.dx = xe > xs ? xe - xs : xs - xe;
  E.dy = ye > ys ? ye - ys : ys - ye;
  E.xmajor = E.dx >= E.dy;
  E.flip = (E.xmajor && xs > xe) || (!E.xmajor && ys > ye);
  if (E.flip) {
    int64_t t = xs; xs = xe; xe = t;
    t = ys; ys = ye; ye = t;
  }
  E.xs = xs; E.ys = ys;
  E.s = E.xmajor ? hd_ddiv(double(ye - ys), double(E.dx)) : hd_ddiv(double(xe - xs), double(E.dy));
  E.n = (E.xmajor ? E.dx : E.dy) + 1;
  return E;
}

HD_FN void cp_point(const Edge& E, int64_t d, int64_t* u, int64_t* v) {
  if (E.xmajor) {
    const int64_t t = E.flip ? E.dx - d : d;
    *u = t + E.xs;
    *v = cp_trunc(hd_dadd(hd_dadd(double(E.ys), hd_dmul(E.s, double(t))), 0.5));
  } else {
    const int64_t t = E.flip ? E.dy - d : d;
    *v = t + E.ys;
    *u = cp_trunc(hd_dadd(hd_dadd(double(E.xs), hd_dmul(E.s, double(t))), 0.5));
  }
}

// the toggle x * h + y of the pair (u0, v0) -> (u1, v1), or -1
HD_FN int64_t cp_toggle(int64_t u0, int64_t v0, int64_t u1, int64_t v1, int64_t h, int64_t w) {
  if (u1 == u0) return -1;
  const double xd = hd_dsub(hd_ddiv(hd_dadd(double(u1 < u0 ? u1 : u1 - 1), 0.5), kScale), 0.5);
  if (floor(xd) != xd || xd < 0 || xd > double(w - 1)) return -1;
  double yd = hd_dsub(hd_ddiv(hd_dadd(double(v1 < v0 ? v1 : v0), 0.5), kScale), 0.5);
  if (yd < 0) yd = 0;
  else if (yd > double(h)) yd = double(h);
  return int64_t(xd) * h + int64_t(ceil(yd));
}

// Edge e: validates its first vertex (status bit 1 not finite, 2 out of the int range; *ann = its annotation) and
// returns its boundary-point count (0 when the edge cannot be walked).
HD_FN int64_t cp_edge_points(const PolyParams& P, int64_t e, int* bad, int* ann) {
  const int p = cp_part_of(P, e);
  *ann = P.part_ann[p];
  *bad = 0;
  const int64_t b = e + 1 == P.part_off[p + 1] ? P.part_off[p] : e + 1;
  int64_t g = 0;
  for (int c = 0; c < 2; ++c) {
    const double z = P.xy[2 * e + c];
    if (!isfinite(z)) *bad |= 1;
    else if (!cp_grid(z, &g)) *bad |= 2;
  }
  if (*bad) return 0;
  for (int c = 0; c < 2; ++c)
    if (!isfinite(P.xy[2 * b + c]) || !cp_grid(P.xy[2 * b + c], &g)) return 0;   // reported by edge b
  return cp_edge(P, p, e).n;
}

// Edge e's toggles: the pairs (previous point, point) for every point of the edge, the first point of the part
// excepted.  Returns the count; kWrite stores them at key[at ..] with the part as value.
template <bool kWrite>
HD_FN int64_t cp_edge_toggles(const PolyParams& P, int64_t e, int64_t at, uint32_t* key, int32_t* val) {
  const int p = cp_part_of(P, e);
  const int a = P.part_ann[p];
  const int64_t h = P.ann_hw[2 * a], w = P.ann_hw[2 * a + 1];
  if (h <= 0 || w <= 0) return 0;
  const Edge E = cp_edge(P, p, e);
  int64_t u0 = 0, v0 = 0, u1 = 0, v1 = 0, n = 0;
  int64_t d = 0;
  if (e == P.part_off[p]) {
    cp_point(E, 0, &u0, &v0);
    d = 1;
  } else {
    const Edge Q = cp_edge(P, p, e - 1);
    cp_point(Q, Q.n - 1, &u0, &v0);
  }
  for (; d < E.n; ++d) {
    cp_point(E, d, &u1, &v1);
    const int64_t t = cp_toggle(u0, v0, u1, v1, h, w);
    if (t >= 0) {
      if (kWrite) { key[at + n] = uint32_t(t); val[at + n] = p; }
      ++n;
    }
    u0 = u1; v0 = v1;
  }
  return n;
}

// Annotation a: its toggles key[seg[a] .. seg[a + 1]) sorted by position, val = their part; par [n_parts] zero on
// entry for a's parts (left as the parts' final parities).  Counts the runs of the union, or writes them to run.
template <bool kWrite>
HD_FN int64_t cp_sweep(const PolyParams& P, int a, const int32_t* seg, const uint32_t* key, const int32_t* val,
                       uint8_t* par, uint32_t* run) {
  const int64_t hw = int64_t(P.ann_hw[2 * a]) * P.ann_hw[2 * a + 1];
  int64_t i = seg[a], n = 0, start = 0, cover = 0;
  const int64_t end = seg[a + 1];
  bool in = false;
  while (i < end) {
    const uint32_t pos = key[i];
    for (; i < end && key[i] == pos; ++i) {
      const int q = val[i];
      par[q] ^= 1;
      cover += par[q] ? 1 : -1;
    }
    if ((cover > 0) == in) continue;
    in = cover > 0;
    if (in) {
      start = pos;
    } else {
      if (kWrite) { run[2 * n] = uint32_t(start); run[2 * n + 1] = uint32_t(pos - start); }
      ++n;
    }
  }
  if (in && start < hw) {
    if (kWrite) { run[2 * n] = uint32_t(start); run[2 * n + 1] = uint32_t(hw - start); }
    ++n;
  }
  return n;
}

// A compressed COCO counts string (pycocotools rleFrString) of an h x w mask: the number of runs of ones, -1 when
// malformed (a character outside '0' .. 'o', a value cut short or over 7 characters, a negative count, or counts that
// do not sum to h * w).  kWrite stores the runs at run[0 ..].
template <bool kWrite>
HD_FN int64_t cp_rle_decode(const uint8_t* c, int64_t len, int64_t hw, uint32_t* run) {
  int64_t pos = 0, c1 = 0, c2 = 0, n = 0;
  if (len == 0) return -1;
  for (int64_t j = 0, i = 0; j < len; ++i) {
    int64_t x = 0;
    int k = 0, v = 0;
    do {
      if (j >= len || k >= 7) return -1;
      v = int(c[j++]) - 48;
      if (v < 0 || v > 63) return -1;
      x |= int64_t(v & 0x1F) << (5 * k);
      ++k;
    } while (v & 0x20);
    if (v & 0x10) x |= -(int64_t(1) << (5 * k));
    const int64_t cnt = i > 2 ? x + c2 : x;
    if (cnt < 0 || cnt > hw - pos) return -1;
    if ((i & 1) && cnt > 0) {
      if (kWrite) { run[2 * n] = uint32_t(pos); run[2 * n + 1] = uint32_t(cnt); }
      ++n;
    }
    pos += cnt; c2 = c1; c1 = cnt;
  }
  return pos == hw ? n : -1;
}

// Byte (y, x) of an H x W mask whose runs are run[b .. e)
HD_FN uint8_t cp_mask_pixel(const uint32_t* run, int64_t b, int64_t e, int64_t H, int64_t y, int64_t x) {
  const int64_t i = x * H + y;
  int64_t lo = b, hi = e;                            // the first run starting after i
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (int64_t(run[2 * mid]) <= i) lo = mid + 1; else hi = mid;
  }
  return lo > b && i < int64_t(run[2 * (lo - 1)]) + run[2 * (lo - 1) + 1] ? 1 : 0;
}

// Argument ranges: 0 or TFB200_E_SHAPE.
static inline int cp_check(int n_parts, int n_ann, int64_t n_edges) {
  if (n_parts < 0 || n_ann < 0 || n_edges < 0 || n_edges >= INT32_MAX) return TFB200_E_SHAPE;
  return 0;
}

}  // namespace tfb200_poly
