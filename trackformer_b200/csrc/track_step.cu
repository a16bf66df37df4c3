// Tracker.step bookkeeping on the device (sm_90a): one CTA runs tfb200_track::ts_step (track_step_core.h) -- every
// threshold, both NMS passes, public-detection gating, ReID and the result rows of src/trackformer/models/tracker.py:
// 266-548 -- so a tracked frame costs one launch after the detector and one small device->host copy of the results,
// instead of the reference's several .cpu() synchronisations per track per frame.
//
// tfb200_track_step_batched_f32 steps up to kMaxBatch independent sequences in one launch: CTA b runs the same routine
// on args[b].  The arguments travel by value in the kernel's parameter space (16 x 312 B, inside the 32 KB that CUDA
// 12.1+ allows on sm_90), so the launch needs no host->device copy and can be captured in a CUDA graph.
#include <cuda_runtime.h>

#include "launch_counter.h"
#include "track_step_core.h"

namespace {

constexpr int kMaxBatch = 16;

struct TrackStepBatch {
  TfbTrackStepArgs a[kMaxBatch];
};

__global__ void __launch_bounds__(tfb200_track::kThreads)
track_step_kernel(const __grid_constant__ TfbTrackStepArgs args) {
  __shared__ tfb200_track::Shared sh;
  tfb200_track::ts_step(args, sh);
}

__global__ void __launch_bounds__(tfb200_track::kThreads)
track_step_batched_kernel(const __grid_constant__ TrackStepBatch batch) {
  __shared__ tfb200_track::Shared sh;
  tfb200_track::ts_step(batch.a[blockIdx.x], sh);
}

int check_args(const TfbTrackStepArgs* a) {
  if (!a) return TFB200_E_NULLPTR;
  if (!a->rows || !a->hs_embeds || !a->q_boxes || !a->q_embeds || !a->result || !a->iscratch || !a->fscratch ||
      !a->dscratch)
    return TFB200_E_NULLPTR;
  const TfbTrackState* st[2] = {&a->in, &a->out};
  for (const TfbTrackState* s : st)
    if (!s->header || !s->ids || !s->pos || !s->anchor || !s->score || !s->obj_ind || !s->count_inactive ||
        !s->count_termination || !s->bank)
      return TFB200_E_NULLPTR;
  if (a->capacity <= 0 || a->capacity > tfb200_track::kMaxRows || a->hidden <= 0 || a->nq < 0 || a->n_query < 0 ||
      a->n_public < 0 || a->n_query + a->nq > a->capacity || a->public_mode < 0 || a->public_mode > 2 ||
      (a->public_mode != 0 && a->n_public > 0 && !a->public_dets))
    return TFB200_E_SHAPE;
  return 0;
}

}  // namespace

extern "C" int tfb200_track_step_f32(const TfbTrackStepArgs* a, void* stream) {
  if (int rc = check_args(a)) return rc;
  track_step_kernel<<<1, tfb200_track::kThreads, 0, cudaStream_t(stream)>>>(*a);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

extern "C" int tfb200_track_step_batched_f32(const TfbTrackStepArgs* args, int n, void* stream) {
  if (!args) return TFB200_E_NULLPTR;
  if (n <= 0 || n > kMaxBatch) return TFB200_E_SHAPE;
  TrackStepBatch batch;
  for (int b = 0; b < n; ++b) {
    if (int rc = check_args(args + b)) return rc;
    batch.a[b] = args[b];
  }
  track_step_batched_kernel<<<n, tfb200_track::kThreads, 0, cudaStream_t(stream)>>>(batch);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}
