// TEST-ONLY host build of the two-stage proposal and selection routines: the very code csrc/two_stage.cu's kernels are
// compiled from (trackformer_b200/csrc/two_stage_core.h), each CTA run by one "thread", so the CPU suite can compare
// the device algorithm with fixtures recorded from the reference.  Built by tests/test_two_stage_cpu.py; never shipped,
// never loaded by the package.  Same arguments as the C entries, host memory, no stream.
#include "../../trackformer_b200/csrc/two_stage_core.h"

using namespace tfb200_two_stage;

extern "C" int tfb200_two_stage_proposals_host(const uint8_t* mask, const float* memory, float* masked, float* prop,
                                               uint8_t* valid, int B, int S, int L, int C, const int* hw) {
  if (int rc = ts_check_proposals(B, S, L, memory ? C : 0, hw)) return rc;
  ProposalParams p{};
  p.B = B; p.S = S; p.L = L; p.C = memory ? C : 0;
  ts_levels(p, hw);
  p.mask = mask; p.memory = memory; p.masked = masked; p.prop = prop; p.valid = valid;
  int vw[kMaxLevels], vh[kMaxLevels];
  for (int b = 0; b < B; ++b) {
    ts_valid_counts(p, b, vw, vh);
    for (int s = 0; s < S; ++s) {
      const bool ok = ts_proposal(p, b, s, vw, vh);
      if (memory)
        for (int c = 0; c < C; ++c)
          masked[(size_t(b) * S + s) * C + c] = ok ? memory[(size_t(b) * S + s) * C + c] : 0.f;
    }
  }
  return 0;
}

extern "C" int tfb200_two_stage_select_host(const float* logits, const float* unact, const float* dim_t, uint32_t* keys,
                                            int64_t* index, float* boxes, float* ref, float* embed, int B, int S,
                                            int C, int k) {
  if (int rc = ts_check_select(B, S, C, k)) return rc;
  SelectParams p{};
  p.B = B; p.S = S; p.C = C; p.k = k;
  p.logits = logits; p.unact = unact; p.dim_t = dim_t; p.keys = keys;
  p.index = index; p.boxes = boxes; p.ref = ref; p.embed = embed;
  static SelectShared sh;
  for (int b = 0; b < B; ++b) {
    ts_select(p, b, sh);
    ts_select_outputs(p, b, sh);
  }
  return 0;
}
