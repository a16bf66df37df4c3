// TEST-ONLY host build of the MOT evaluation: the very routines csrc/mot_eval.cu's kernels are compiled from
// (trackformer_b200/csrc/mot_eval_core.h), each CTA run in turn by one "thread", so the CPU suite can compare the
// device algorithm with the oracle of tests/mot_eval_reference.py.  Built by tests/test_mot_eval_cpu.py; never shipped,
// never loaded by the package.  Same arguments as tfb200_mot_eval_f32, host memory, no stream.
#include <string.h>

#include "../../trackformer_b200/csrc/mot_eval_core.h"

using namespace tfb200_mot;

extern "C" size_t tfb200_mot_eval_host_workspace_bytes(int S, int F, int64_t n_gt, int64_t n_trk, int64_t tp_cells,
                                                       int max_obj, int max_hyp, int64_t pair_cap) {
  if (me_check(S, F, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap)) return 0;
  Params p{};
  return me_carve(p, nullptr, S, F, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap);
}

extern "C" int tfb200_mot_eval_host(const int64_t* seq, const int32_t* frame_obj, const int32_t* frame_hyp,
                                    const int32_t* obj_id, const float* obj_box, const int32_t* hyp_id,
                                    const float* hyp_box, int S, int F, int64_t n_gt, int64_t n_trk, int64_t tp_cells,
                                    int max_obj, int max_hyp, int64_t pair_cap, void* workspace,
                                    size_t workspace_bytes, int64_t* out) {
  if (int rc = me_check(S, F, n_gt, n_trk, tp_cells, max_obj, max_hyp, pair_cap)) return rc;
  Params p{};
  if (workspace_bytes < me_carve(p, static_cast<char*>(workspace), S, F, n_gt, n_trk, tp_cells, max_obj, max_hyp,
                                 pair_cap))
    return TFB200_E_SHAPE;
  p.S = S; p.F = F; p.max_obj = max_obj; p.max_hyp = max_hyp; p.pair_cap = pair_cap;
  p.seq = seq; p.fobj = frame_obj; p.fhyp = frame_hyp; p.obj_id = obj_id; p.obj_box = obj_box; p.hyp_id = hyp_id;
  p.hyp_box = hyp_box; p.out = out;
  static Shared sh;
  memset(p.tp, 0, size_t(tp_cells) * 4);
  for (int s = 0; s < S; ++s) me_init_seq(p, s);
  for (int f = 0; f < F; ++f) me_pairs_frame<false>(p, f, sh);
  me_scan(p, sh);
  for (int f = 0; f < F; ++f) me_pairs_frame<true>(p, f, sh);
  for (int s = 0; s < S; ++s) me_clear_seq(p, s, sh);
  for (int s = 0; s < S; ++s) me_id_label(p, s, sh);
  for (int64_t k = 0; k < n_gt; ++k) me_id_comp(p, k, sh);
  return 0;
}
