// TEST-ONLY host build of the COCO evaluation: the very routines csrc/coco_eval.cu's kernels are compiled from
// (trackformer_b200/csrc/coco_eval_core.h), each CTA run in turn by one "thread", so the CPU suite can compare the
// device algorithm with the oracle of tests/coco_eval_reference.py.  Built by tests/test_coco_eval_cpu.py; never
// shipped, never loaded by the package.  The arguments of the C entries, host memory, no stream, the workspace
// allocated here; iou_out (may be NULL) receives the IoU workspace (per image [n_det][n_gt]) so that tests can read
// the IoUs themselves.  The radix sort of the device entry is std::stable_sort on the same keys here.
#include <string.h>

#include <algorithm>
#include <numeric>
#include <vector>

#include "../../trackformer_b200/csrc/coco_eval_core.h"

using namespace tfb200_coco;

extern "C" int tfb200_coco_match_host(const int64_t* img, int B, int max_n, int max_g, const float* boxes,
                                      const float* scores, const int64_t* labels, int64_t N, const int64_t* cat_ids,
                                      int K, const int64_t* gt_off, const int32_t* gt_k, const double* gt_box,
                                      const double* gt_area, const uint8_t* gt_crowd, const int64_t* gt_id,
                                      const int64_t* gt_run_off, const uint32_t* gt_runs, const int32_t* gt_bbox,
                                      const int64_t* gt_px, const double* area_rng, int A, const double* iou_thr,
                                      int T, int max_det, int segm, int64_t iou_cells, int64_t dbit_words,
                                      int64_t gbit_words, int64_t gtm_bytes, uint64_t* key, int32_t* rank,
                                      uint32_t* state, int32_t* status, double* iou_out) {
  if (int rc = ce_check_match(B, N, K, A, T, max_det)) return rc;
  if (max_n < 0 || max_n > kMaxDets || max_g < 0) return TFB200_E_SHAPE;
  MatchParams p{};
  p.B = B; p.K = K; p.A = A; p.T = T; p.max_det = max_det; p.segm = segm;
  p.img = img; p.boxes = boxes; p.scores = scores; p.labels = labels; p.cat_ids = cat_ids;
  p.gt_off = gt_off; p.gt_k = gt_k; p.gt_box = gt_box; p.gt_area = gt_area; p.gt_crowd = gt_crowd; p.gt_id = gt_id;
  p.gt_run_off = gt_run_off; p.gt_runs = gt_runs; p.gt_bbox = gt_bbox; p.gt_px = gt_px;
  p.area_rng = area_rng; p.iou_thr = iou_thr; p.key = key; p.rank = rank; p.state = state; p.status = status;
  std::vector<int32_t> dk(N), dord(N), dbox(N * 4);
  std::vector<double> iou(iou_cells);
  std::vector<uint32_t> dbits(dbit_words), gbits(gbit_words, 0u);
  std::vector<int64_t> dpx(N);
  std::vector<uint8_t> gtm(gtm_bytes, 0);
  p.dk = dk.data(); p.dord = dord.data(); p.dbox = dbox.data(); p.iou = iou.data(); p.dbits = dbits.data();
  p.gbits = gbits.data(); p.dpx = dpx.data(); p.gtm = gtm.data();
  for (int b = 0; b < B; ++b) ce_rank(p, b);
  PackShared psh;
  IouShared ish;
  if (segm) {
    for (int b = 0; b < B; ++b) for (int j = 0; j < max_n; ++j) ce_pack_dt(p, b, j, psh);
    for (int b = 0; b < B; ++b) for (int g = 0; g < max_g; ++g) ce_decode_gt(p, b, g);
  }
  for (int b = 0; b < B; ++b) for (int j = 0; j < max_n; ++j) ce_iou(p, b, j, ish);
  for (int b = 0; b < B; ++b) ce_match(p, b);
  if (iou_out) memcpy(iou_out, iou.data(), size_t(iou_cells) * sizeof(double));
  return 0;
}

extern "C" int tfb200_coco_accumulate_host(const uint64_t* key, const int32_t* rank, const uint32_t* state,
                                           int64_t n_rec, const int64_t* kept, int n_kept, int64_t n,
                                           const int64_t* npig, const double* rec_thr, const int32_t* max_dets,
                                           const int32_t* status, int K, int A, int T, int R, int M,
                                           double* precision, double* recall, double* scores, double* status_out) {
  if (int rc = ce_check_acc(K, A, T, R, M, n_kept, n_rec, n)) return rc;
  AccParams p{};
  p.K = K; p.A = A; p.T = T; p.R = R; p.M = M; p.n_kept = n_kept; p.n_rec = n_rec; p.n = n;
  p.key = key; p.rank = rank; p.state = state; p.kept = kept; p.npig = npig; p.rec_thr = rec_thr;
  p.max_dets = max_dets; p.status_in = status; p.precision = precision; p.recall = recall; p.scores = scores;
  p.status_out = status_out;
  std::vector<uint64_t> key_in(n), key_out(n);
  std::vector<int64_t> val_in(n), val_out(n);
  p.key_in = key_in.data(); p.key_out = key_out.data(); p.val_in = val_in.data(); p.val_out = val_out.data();
  for (int i = 0; i < n_kept; ++i) ce_gather(p, i);
  std::vector<int64_t> order(n);
  std::iota(order.begin(), order.end(), 0);
  std::stable_sort(order.begin(), order.end(), [&](int64_t x, int64_t y) { return key_in[x] < key_in[y]; });
  for (int64_t i = 0; i < n; ++i) { key_out[i] = key_in[order[i]]; val_out[i] = val_in[order[i]]; }
  static AccShared sh;
  for (int c = 0; c < K * A * M * T; ++c) ce_acc(p, c, sh);
  status_out[0] = double(status[0]);
  return 0;
}
