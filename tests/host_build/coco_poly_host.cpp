// TEST-ONLY host build of the polygon rasteriser: the very routines csrc/coco_poly.cu's kernels are compiled from
// (trackformer_b200/csrc/coco_poly_core.h), each thread run in turn and the segmented sort done by std::sort, so the
// CPU suite can compare the device algorithm with the oracle of tests/coco_poly_reference.py.  Built by
// tests/test_coco_poly_cpu.py with -ffp-contract=off; never shipped, never loaded by the package.  Same arguments as
// the tfb200_coco_poly_* / tfb200_coco_rle_runs / tfb200_coco_masks_u8 entries, host memory, no stream or workspace.
#include <string.h>

#include <algorithm>
#include <utility>
#include <vector>

#include "../../trackformer_b200/csrc/coco_poly_core.h"

using namespace tfb200_poly;

static PolyParams params(const double* xy, const int64_t* part_off, const int32_t* part_ann, const int64_t* ann_part,
                         const int32_t* ann_hw, int n_parts, int n_ann, int64_t n_edges) {
  PolyParams P{};
  P.xy = xy; P.part_off = part_off; P.part_ann = part_ann; P.ann_part = ann_part; P.ann_hw = ann_hw;
  P.n_parts = n_parts; P.n_ann = n_ann; P.n_edges = n_edges;
  return P;
}

extern "C" int tfb200_coco_poly_count_host(const double* xy, const int64_t* part_off, const int32_t* part_ann,
                                           const int64_t* ann_part, const int32_t* ann_hw, int n_parts, int n_ann,
                                           int64_t n_edges, int32_t* toggle_off, int64_t* ann_points,
                                           int64_t* sizes) {
  if (int rc = cp_check(n_parts, n_ann, n_edges)) return rc;
  const PolyParams P = params(xy, part_off, part_ann, ann_part, ann_hw, n_parts, n_ann, n_edges);
  memset(ann_points, 0, size_t(n_ann) * 8);
  sizes[kSzPoints] = 0; sizes[kSzToggles] = 0; sizes[kSzStatus] = 0;
  sizes[kSzBadFinite] = n_ann; sizes[kSzBadRange] = n_ann;
  for (int64_t e = 0; e < n_edges; ++e) {
    int bad = 0, a = 0;
    const int64_t n = cp_edge_points(P, e, &bad, &a);
    sizes[kSzStatus] |= bad;
    if ((bad & 1) && a < sizes[kSzBadFinite]) sizes[kSzBadFinite] = a;
    if ((bad & 2) && a < sizes[kSzBadRange]) sizes[kSzBadRange] = a;
    ann_points[a] += n;
    sizes[kSzPoints] += n;
  }
  const bool ok = sizes[kSzStatus] == 0 && sizes[kSzPoints] <= INT32_MAX;
  toggle_off[0] = 0;
  for (int64_t e = 0; e < n_edges; ++e)
    toggle_off[e + 1] = toggle_off[e] + (ok ? int32_t(cp_edge_toggles<false>(P, e, 0, nullptr, nullptr)) : 0);
  if (sizes[kSzPoints] > INT32_MAX) sizes[kSzStatus] |= 4;
  sizes[kSzToggles] = sizes[kSzStatus] ? 0 : toggle_off[n_edges];
  return 0;
}

extern "C" int tfb200_coco_poly_runs_host(const double* xy, const int64_t* part_off, const int32_t* part_ann,
                                          const int64_t* ann_part, const int32_t* ann_hw, int n_parts, int n_ann,
                                          int64_t n_edges, const int32_t* toggle_off, int64_t n_toggles,
                                          int64_t* run_off, uint32_t* runs) {
  if (int rc = cp_check(n_parts, n_ann, n_edges)) return rc;
  const PolyParams P = params(xy, part_off, part_ann, ann_part, ann_hw, n_parts, n_ann, n_edges);
  std::vector<uint32_t> key(size_t(n_toggles) + 1);
  std::vector<int32_t> val(size_t(n_toggles) + 1), seg(size_t(n_ann) + 1);
  std::vector<uint8_t> par(size_t(n_parts) + 1, 0);
  for (int64_t e = 0; e < n_edges; ++e) cp_edge_toggles<true>(P, e, toggle_off[e], key.data(), val.data());
  for (int a = 0; a <= n_ann; ++a) seg[a] = toggle_off[part_off[ann_part[a]]];
  std::vector<std::pair<uint32_t, int32_t>> kv;
  for (int a = 0; a < n_ann; ++a) {                  // each annotation's toggles by position
    kv.clear();
    for (int32_t i = seg[a]; i < seg[a + 1]; ++i) kv.emplace_back(key[i], val[i]);
    std::sort(kv.begin(), kv.end());
    for (size_t i = 0; i < kv.size(); ++i) { key[seg[a] + i] = kv[i].first; val[seg[a] + i] = kv[i].second; }
  }
  run_off[0] = 0;
  for (int a = 0; a < n_ann; ++a)
    run_off[a + 1] = run_off[a] + cp_sweep<false>(P, a, seg.data(), key.data(), val.data(), par.data(), nullptr);
  std::fill(par.begin(), par.end(), 0);
  for (int a = 0; a < n_ann; ++a)
    cp_sweep<true>(P, a, seg.data(), key.data(), val.data(), par.data(), runs + 2 * run_off[a]);
  return 0;
}

extern "C" int tfb200_coco_rle_runs_host(const uint8_t* chars, const int64_t* str_off, const int64_t* run_cap_off,
                                         int n, int h, int w, int64_t* bounds, uint32_t* runs, int64_t* first_bad) {
  const int64_t hw = int64_t(h) * w;
  for (int k = 0; k < n; ++k) {
    const int64_t len = str_off[k + 1] - str_off[k], at = run_cap_off[k];
    const int64_t m = cp_rle_decode<false>(chars + str_off[k], len, hw, nullptr);
    if (m < 0 && k < *first_bad) *first_bad = k;
    if (m >= 0) cp_rle_decode<true>(chars + str_off[k], len, hw, runs + 2 * at);
    bounds[2 * k] = at;
    bounds[2 * k + 1] = at + (m < 0 ? 0 : m);
  }
  return 0;
}

extern "C" int tfb200_coco_masks_u8_host(const int32_t* src, int N, int H, int W, const int64_t* poly_run_off,
                                         const uint32_t* poly_runs, const int64_t* rle_bounds,
                                         const uint32_t* rle_runs, uint8_t* out) {
  for (int m = 0; m < N; ++m) {
    const int s = src[m];
    const uint32_t* run = s >= 0 ? poly_runs : rle_runs;
    const int64_t b = s >= 0 ? poly_run_off[s] : rle_bounds[2 * (-1 - s)];
    const int64_t e = s >= 0 ? poly_run_off[s + 1] : rle_bounds[2 * (-1 - s) + 1];
    for (int64_t y = 0; y < H; ++y)
      for (int64_t x = 0; x < W; ++x) out[(int64_t(m) * H + y) * W + x] = cp_mask_pixel(run, b, e, H, y, x);
  }
  return 0;
}
