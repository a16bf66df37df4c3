// TEST-ONLY host build of tfb200_track_step_batched_f32: the routine the batched kernel's CTA b runs on args[b]
// (trackformer_b200/csrc/track_step_core.h), here one sequence after the other.  Built by
// tests/test_multi_tracker_cpu.py; never shipped, never loaded by the package.
#include "../../trackformer_b200/csrc/track_step_core.h"

extern "C" int tfb200_track_step_batched_host(const TfbTrackStepArgs* args, int n) {
  static tfb200_track::Shared sh;
  for (int b = 0; b < n; ++b) tfb200_track::ts_step(args[b], sh);
  return 0;
}
