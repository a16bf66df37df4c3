// TEST-ONLY host build of the panoptic post-processing and PQ scoring: the very routines csrc/panoptic.cu's kernels
// are compiled from (trackformer_b200/csrc/panoptic_core.h), each CTA run in turn by one "thread".  The entries have
// the names and arguments of the device entries (host pointers; the stream is ignored), so the CPU suite drives the
// product's own host code (segmentation.PostProcessPanoptic, panoptic_eval.PQScorer) with CPU tensors.  Built by
// tests/test_panoptic_cpu.py; never shipped, never loaded by the package.
#include <string.h>

#include <vector>

#include "../../trackformer_b200/csrc/panoptic_core.h"

using namespace tfb200_panoptic;

extern "C" int tfb200_panoptic_classes_f32(const float* logits, int B, int Q, int C, float threshold, int32_t* cls,
                                           float* score, uint8_t* keep, void*) {
  PpParams p{};
  p.B = B; p.Q = Q; p.C = C; p.threshold = threshold;
  p.logits = logits; p.cls = cls; p.score = score; p.keep = keep;
  for (int64_t r = 0; r < int64_t(B) * Q; ++r) pp_classes(p, r);
  return 0;
}

extern "C" int tfb200_panoptic_label_f32(const float* masks, int B, int Q, int h, int w, const int64_t* img, int,
                                         const int32_t* kept_q, const int32_t* kept_alive, const int32_t* kept_rep,
                                         const int32_t* idx, int32_t* map, unsigned long long* area, int blocks,
                                         void*) {
  PpParams p{};
  p.B = B; p.Q = Q; p.h = h; p.w = w;
  p.masks = masks; p.img = img; p.kept_q = kept_q; p.kept_alive = kept_alive; p.kept_rep = kept_rep; p.idx = idx;
  p.map = map; p.area = area;
  static unsigned long long hist[kMaxKept];
  for (int b = 0; b < B; ++b)
    for (int k = 0; k < blocks; ++k) pp_label(p, b, k, hist);
  return 0;
}

extern "C" int tfb200_panoptic_final_f32(const int64_t* img, int B, const int32_t* kept_alive, const int32_t* kept_pos,
                                         const int32_t* idx, const int32_t* map, int32_t* out, int blocks, void*) {
  PpParams p{};
  p.B = B; p.img = img; p.kept_alive = kept_alive; p.kept_pos = kept_pos; p.idx = idx;
  p.map = const_cast<int32_t*>(map);
  p.out = out;
  for (int b = 0; b < B; ++b)
    for (int k = 0; k < blocks; ++k) pp_final(p, b, k);
  return 0;
}

extern "C" int tfb200_pq_update(const int64_t* img, int B, int Kc, int, const int32_t* maps, const int32_t* gt_id,
                                const int32_t* gt_cat, const int32_t* gt_crowd, const double* gt_area,
                                const int32_t* gt_json, const int32_t* pred_id, const int32_t* pred_cat, int* cells,
                                int64_t n_cells, int64_t* pred_area, int32_t* stat_i, double* stat_iou, long long* err,
                                int blocks, void*) {
  PqParams p{};
  p.B = B; p.Kc = Kc; p.img = img; p.maps = maps; p.gt_id = gt_id; p.gt_cat = gt_cat; p.gt_crowd = gt_crowd;
  p.gt_area = gt_area; p.gt_json = gt_json; p.pred_id = pred_id; p.pred_cat = pred_cat; p.cells = cells;
  p.pred_area = pred_area; p.stat_i = stat_i; p.stat_iou = stat_iou; p.err = err;
  memset(cells, 0, size_t(n_cells) * sizeof(int));
  static int sh[kSharedCells];
  static MatchShared msh;
  for (int b = 0; b < B; ++b)
    for (int k = 0; k < blocks; ++k) pq_count(p, b, k, sh);
  for (int b = 0; b < B; ++b) pq_match(p, b, msh);
  return 0;
}

extern "C" int tfb200_pq_reduce(const int32_t* stat_i, const double* stat_iou, const long long* err,
                                const int64_t* rows, int64_t n, int Kc, double* out, int64_t* err_out, void*) {
  for (int k = 0; k <= Kc; ++k) pq_reduce(stat_i, stat_iou, err, rows, n, Kc, k, out, err_out);
  return 0;
}
