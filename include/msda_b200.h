/*
 * msda_b200.h -- C ABI of the H100 (sm_90a) multi-scale deformable attention library
 * (libmsda_b200.so).  Plain pointers and sizes only; no torch types.
 *
 * Every entry point replaces a piece of the reference's compiled extension
 * `MultiScaleDeformableAttention` (timmeinhardt/trackformer @ e468bf1,
 * paths relative to src/trackformer/models/ops/):
 *
 *   msda_b200_forward_{f32,f64}   <- ms_deform_attn_cuda_forward          src/cuda/ms_deform_attn_cuda.cu:19-86
 *                                    (= ms_deformable_im2col_cuda         src/cuda/ms_deform_im2col_cuda.cuh:380-410
 *                                       + at::sum over the L*P columns    src/cuda/ms_deform_attn_cuda.cu:80)
 *   msda_b200_backward_{f32,f64}  <- ms_deform_attn_cuda_backward         src/cuda/ms_deform_attn_cuda.cu:89-168
 *                                    (= ms_deformable_col2im_coord_cuda   src/cuda/ms_deform_im2col_cuda.cuh:454-496
 *                                       + ms_deformable_col2im_cuda       src/cuda/ms_deform_im2col_cuda.cuh:412-452)
 *   msda_b200_*_host_*            <- the same two calls for callers that hold HOST buffers (the
 *                                    reference has no such path: its CPU entry throws,
 *                                    src/cpu/ms_deform_attn_cpu.cpp:15,27); used for end-to-end timing.
 *
 * The Python-visible module built on top of this ABI keeps the reference's pybind surface
 * (src/vision.cpp:4-7, src/ms_deform_attn.h:10-50): see trackformer_b200/csrc/msda_torch.cpp.
 *
 * Tensor layouts (contiguous, last index fastest) -- identical to the reference:
 *   value           [N][S][M][D]      s = level_start[l] + y*W_l + x,  S = sum_l H_l*W_l
 *   spatial_shapes  [L][2] int64      (H_l, W_l), DEVICE memory (the reference keeps it on the GPU,
 *                                     models/deformable_transformer.py:156); level starts are derived
 *                                     in-kernel, the old 5-argument API has no level_start_index
 *   sampling_loc    [N][Lq][M][L][P][2]   (x, y) normalised to [0,1] over the padded level
 *   attn_weight     [N][Lq][M][L][P]
 *   output / grad_output                  [N][Lq][M*D]
 *   grad_value / grad_sampling_loc / grad_attn_weight : shapes of value / sampling_loc / attn_weight
 *
 * Ownership: the caller owns every buffer.  The backward call zero-fills grad_value itself
 * (the reference does at::zeros_like, ms_deform_attn_cuda.cu:119) and overwrites the other two.
 * All work is enqueued on `stream` (a cudaStream_t, passed as void*; NULL = legacy default
 * stream); the device-pointer calls never synchronise.  Re-entrant, no global state.
 *
 * Errors: every function returns 0 on success, a negative MSDA_E_* code for argument
 * errors, or a positive cudaError_t value when a CUDA call / kernel launch failed (the
 * reference only printf()s launch errors, ms_deform_im2col_cuda.cuh:404-408 -- here they are
 * returned, and the Python binding raises).  msda_b200_error_string() renders either kind.
 */
#ifndef MSDA_B200_H_
#define MSDA_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MSDA_B200_ABI_VERSION 1

#define MSDA_E_NULLPTR   (-1)  /* a required pointer is NULL                       */
#define MSDA_E_DIMS      (-2)  /* a dimension is <= 0 (N, Lq may be 0: no-op)      */
#define MSDA_E_TOO_LARGE (-3)  /* a per-sample slab exceeds 2^31-1 elements        */
#define MSDA_E_LEVELS    (-4)  /* L > MSDA_B200_MAX_LEVELS                         */

#define MSDA_E_UNSUPPORTED (-5) /* geometry outside a specialised entry point's domain */

#define MSDA_B200_MAX_LEVELS 32

int msda_b200_abi_version(void);
const char* msda_b200_error_string(int code);

/* ---- device-pointer entry points (the hot path) -------------------------------------- */
int msda_b200_forward_f32(const float* value, const int64_t* spatial_shapes,
                          const float* sampling_loc, const float* attn_weight, float* output,
                          int N, int S, int M, int D, int L, int Lq, int P, void* stream);
int msda_b200_forward_f64(const double* value, const int64_t* spatial_shapes,
                          const double* sampling_loc, const double* attn_weight, double* output,
                          int N, int S, int M, int D, int L, int Lq, int P, void* stream);

int msda_b200_backward_f32(const float* value, const int64_t* spatial_shapes,
                           const float* sampling_loc, const float* attn_weight,
                           const float* grad_output, float* grad_value, float* grad_sampling_loc,
                           float* grad_attn_weight,
                           int N, int S, int M, int D, int L, int Lq, int P, void* stream);
int msda_b200_backward_f64(const double* value, const int64_t* spatial_shapes,
                           const double* sampling_loc, const double* attn_weight,
                           const double* grad_output, double* grad_value, double* grad_sampling_loc,
                           double* grad_attn_weight,
                           int N, int S, int M, int D, int L, int Lq, int P, void* stream);

/* ---- encoder self-attention (queries == pixels, Lq == S) with shared-memory staged value tiles -----------
 * Same contract and same results as msda_b200_forward_f32, but the level sizes are ALSO given on the host
 * (spatial_shapes_host, [L][2] int64 (H, W) in HOST memory): the grid is one CTA per 16x4 tile of queries per head.
 * Returns MSDA_E_UNSUPPORTED (nothing launched) unless fp32, D == 32, L <= 8, L*P <= 64, Lq == S == sum(H*W),
 * every H, W >= 2 and the buffers are 16-byte aligned -- callers then use msda_b200_forward_f32.
 * No reference counterpart (the reference has a single kernel for every call site).                         */
/* ---- fused-prologue variant (module-level fusion, SURVEY 8(f1)) ------------------------------------------------------
 * The sampling locations and attention weights of ops/modules/ms_deform_attn.py:69-79 are computed INSIDE the kernel:
 *   proj [N][Lq][3*M*L*P]  the raw output of the module's [sampling_offsets | attention_weights] projections:
 *                          [M][L][P][2] offsets followed by [M][L*P] logits (softmax over L*P per head in-kernel)
 *   ref  [N][Lq][L][2]     reference points;  loc = ref + offset / spatial_shapes (divided as stored, like the reference)
 * backward writes grad_proj (same layout: offset gradients, then the logit gradients through the softmax) and
 * zero-fills + accumulates grad_value.  Domain: fp32, D = 32 or 36, M % 4 == 0, L*P == 16; MSDA_E_UNSUPPORTED otherwise
 * (callers then materialise loc / attn and use msda_b200_forward_f32 / _backward_f32).                              */
int msda_b200_forward_fused_f32(const float* value, const int64_t* spatial_shapes, const float* proj, const float* ref,
                                float* output, int N, int S, int M, int D, int L, int Lq, int P, void* stream);
int msda_b200_backward_fused_f32(const float* value, const int64_t* spatial_shapes, const float* proj, const float* ref,
                                 const float* grad_output, float* grad_value, float* grad_proj, int N, int S, int M, int D,
                                 int L, int Lq, int P, void* stream);

int msda_b200_forward_enc_tiled_f32(const float* value, const int64_t* spatial_shapes_host,
                                    const float* sampling_loc, const float* attn_weight, float* output,
                                    int N, int S, int M, int D, int L, int Lq, int P, void* stream);
/* Backward twin (same contract as msda_b200_backward_f32: grad_value is zero-filled and accumulated, the other two are
 * overwritten; replaces ms_deform_attn_cuda_backward, ms_deform_attn_cuda.cu:89-168, for encoder call sites).  Domain as
 * the forward, plus H, W <= 4095 and S < 2^20.  With the device copy of the level sizes given, the queries of levels >= 1
 * (whose samples on finer levels cannot be staged) are served by the 8-lane-group kernel in a second launch.            */
int msda_b200_backward_enc_tiled_f32(const float* value, const int64_t* spatial_shapes_host,
                                     const int64_t* spatial_shapes_dev /* device copy, or NULL */,
                                     const float* sampling_loc, const float* attn_weight, const float* grad_output,
                                     float* grad_value, float* grad_sampling_loc, float* grad_attn_weight,
                                     int N, int S, int M, int D, int L, int Lq, int P, void* stream);

/* Tile kernels with the fused prologue (proj / ref as in msda_b200_forward_fused_f32); additionally L == 4. */
int msda_b200_forward_enc_tiled_fused_f32(const float* value, const int64_t* spatial_shapes_host, const float* proj,
                                          const float* ref, float* output, int N, int S, int M, int D, int L, int Lq,
                                          int P, void* stream);
int msda_b200_backward_enc_tiled_fused_f32(const float* value, const int64_t* spatial_shapes_host, const float* proj,
                                           const float* ref, const float* grad_output, float* grad_value,
                                           float* grad_proj, int N, int S, int M, int D, int L, int Lq, int P, void* stream);

/* ---- host-buffer entry points (H2D + kernel + D2H inside the call; synchronous) -------- */
int msda_b200_forward_host_f32(const float* value, const int64_t* spatial_shapes,
                               const float* sampling_loc, const float* attn_weight, float* output,
                               int N, int S, int M, int D, int L, int Lq, int P, int device);
int msda_b200_backward_host_f32(const float* value, const int64_t* spatial_shapes,
                                const float* sampling_loc, const float* attn_weight,
                                const float* grad_output, float* grad_value,
                                float* grad_sampling_loc, float* grad_attn_weight,
                                int N, int S, int M, int D, int L, int Lq, int P, int device);

/* ---- introspection / tuning (not part of the reference surface) ------------------------ */
/* Selects a kernel variant for experiments (0 = library default). Process-wide.            */
void msda_b200_set_variant(int fwd_variant, int bwd_variant);
/* 1 unless a non-default forward variant is forced (then the tiled encoder path is bypassed, for A/B timing) */
int msda_b200_variant_allows_tiles(void);
/* Measurement aid: `ctas` CTAs of 256 threads each issue `iters` gather-shaped LDG.128 requests (4 x 128-byte rows
 * per warp request, rows drawn pseudo-randomly from table[rows][32] floats).  Bytes moved = ctas*256*iters*16.
 * Used by tools/l1_gather_peak.py to measure the L1-data-stage ceiling the gather kernels are compared against.   */
int msda_b200_l1_gather_probe(const float* table, float* sink, int64_t rows, int iters, int ctas, void* stream);
/* Number of kernel launches this library has enqueued since load (bench.py's gpu_launches). */
uint64_t msda_b200_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* MSDA_B200_H_ */
