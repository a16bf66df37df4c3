/*
 * tfb200_fused.h -- C ABI of the fused transformer-layer kernels in libmsda_b200.so (sm_90a).
 *
 * These have NO counterpart in the reference's native code: the reference runs them as chains of PyTorch ops
 *   x = norm(x + dropout(branch))        src/trackformer/models/deformable_transformer.py:284-285, 291-292,
 *                                        360-361, 370-371, 377-378
 * They sit on the hot path (SURVEY section 8, rows a10/a11) and are exposed through the same Python module as extra
 * functions; the reference-facing surface stays include/msda_b200.h.
 *
 * Conventions as in msda_b200.h: caller owns all (device) buffers, work is enqueued on `stream`, 0 = success,
 * negative = argument error, positive = cudaError_t.
 */
#ifndef TFB200_FUSED_H_
#define TFB200_FUSED_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TFB200_E_NULLPTR (-1)
#define TFB200_E_SHAPE   (-2)   /* C must be a multiple of 4, <= 512 (LayerNorm backward) / 1024 (forward, colsum) */
#define TFB200_LN_MAX_CTAS 528  /* persistent grid: 132 SMs x 4 CTAs; also the row count of `partial_ws` */

/* number of CTAs (= rows of the [ctas][2][C] fp32 workspace the backward needs) for a problem of `rows` rows */
int tfb200_ln_partial_ctas(int64_t rows);

/* s = x + branch * keep_mask / keep_prob   (keep_mask == NULL: s = x + branch)
 * y = LayerNorm(s) * gamma + beta          mean/rstd [rows] and s_out [rows][C] are optional outputs (NULL to skip) */
int tfb200_add_dropout_layernorm_fwd_f32(const float* x, const float* branch, const uint8_t* keep_mask,
                                         const float* gamma, const float* beta, float* s_out, float* y,
                                         float* mean, float* rstd, int64_t rows, int C, float keep_prob, float eps,
                                         void* stream);

/* dx = dL/dx (= dL/ds), dbranch = dL/dbranch (NULL to skip), dgamma/dbeta [C]; partial_ws: [ctas][2][C] fp32 */
int tfb200_add_dropout_layernorm_bwd_f32(const float* dy, const float* s, const uint8_t* keep_mask,
                                         const float* gamma, const float* mean, const float* rstd, float* dx,
                                         float* dbranch, float* dgamma, float* dbeta, float* partial_ws,
                                         int64_t rows, int C, float keep_prob, void* stream);

/* Same pair with mask-free dropout: keep decisions are a counter-based hash of (*seed_dev, element index) against
 * keep_prob (the scheme of tfb200_relu_dropout_*), so no mask tensor is drawn, stored or read; forward and backward
 * must be given the same seed.                                                                                        */
int tfb200_add_dropout_layernorm_seeded_fwd_f32(const float* x, const float* branch, const int64_t* seed_dev,
                                                const float* gamma, const float* beta, float* s_out, float* y,
                                                float* mean, float* rstd, int64_t rows, int C, float keep_prob,
                                                float eps, void* stream);
int tfb200_add_dropout_layernorm_seeded_bwd_f32(const float* dy, const float* s, const int64_t* seed_dev,
                                                const float* gamma, const float* mean, const float* rstd, float* dx,
                                                float* dbranch, float* dgamma, float* dbeta, float* partial_ws,
                                                int64_t rows, int C, float keep_prob, void* stream);

/* out[c] = sum_r x[r][c]  (bias gradient of a Linear over a long token axis); C % 4 == 0, C <= 1024;
 * partial_ws: [tfb200_ln_partial_ctas(rows)][C] fp32.  Deterministic (fixed summation order).                      */
int tfb200_colsum_f32(const float* x, float* out, float* partial_ws, int64_t rows, int C, void* stream);

/* h = dropout(relu(a)) in one pass (FFN hidden activation, deformable_transformer.py:283,359).  Inverted dropout with a
 * counter-based keep decision hashed from (*seed_dev, element index): no mask tensor.  backward: grad_a from grad_h and
 * h alone (h > 0 <=> a > 0 and kept).  n % 4 == 0.  training == 0: plain ReLU.                                        */
int tfb200_relu_dropout_fwd_f32(const float* a, float* h, const int64_t* seed_dev, int64_t n, float keep_prob,
                                int training, void* stream);
int tfb200_relu_dropout_bwd_f32(const float* grad_h, const float* h, float* grad_a, int64_t n, float keep_prob,
                                int training, void* stream);

/* proj [rows][3*M*L*P] = per query [offsets (M,L,P,2) | attention logits (M,L*P)]  ->  sampling locations
 * loc [rows][M][L][P][2] and softmax attention weights attn [rows][M][L][P] in one pass (ms_deform_attn.py:69-82).
 * ref: [rows][L][ref_dim] reference points (ref_dim 2) or boxes (4); shapes_f32: [L][2] level sizes AS STORED (H, W)
 * in fp32 (only read for ref_dim == 2).  L*P in {4, 8, 16, 32}, (M*L*P) % 32 == 0.  backward: grad_proj from grad_loc,
 * grad_attn and the saved attn (no gradient for ref: callers use it only when ref does not require one).            */
int tfb200_sampling_prep_fwd_f32(const float* proj, const float* ref, const float* shapes_f32, float* loc, float* attn,
                                 int64_t rows, int M, int L, int P, int ref_dim, void* stream);
int tfb200_sampling_prep_bwd_f32(const float* grad_loc, const float* grad_attn, const float* attn, const float* ref,
                                 const float* shapes_f32, float* grad_proj, int64_t rows, int M, int L, int P, int ref_dim,
                                 void* stream);

/* Device-side Hungarian matching (replaces the host scipy.optimize.linear_sum_assignment calls of
 * src/trackformer/models/matcher.py:104,127).  cost: [K][B][Q][T] fp32 (K decoder layers, B images, Q queries, T = all
 * ground-truth boxes of the batch, image b owning columns offsets[b] .. offsets[b+1]-1; offsets_dev: int32 [B+1] on the
 * device).  Every (k, b) problem assigns each of image b's boxes to a distinct query (boxes per image <= max_targets <= Q).
 * src/tgt: int64 [K][T]; for each problem the pairs are written to columns offsets[b].. in ascending query order:
 * src = query index, tgt = global box index.  *status_dev (int32, caller-zeroed) becomes 1 (more boxes than queries)
 * or 2 (infeasible: a box whose costs are all +inf).  Double-precision duals, like scipy.                           */
int tfb200_lsa_f32(const float* cost, const int* offsets_dev, int64_t* src, int64_t* tgt, int K, int B, int Q, int T,
                   int max_targets, int* status_dev, void* stream);

/* Detection post-processing for the online tracker (deformable_detr.py:286-334 + the per-track read-backs of
 * tracker.py:306-330): logits [N][Q][C], boxes [N][Q][4] (cx, cy, w, h normalised), sizes_hw [N][2] int64 (h, w) on the
 * DEVICE  ->  packed [N][Q][6] = {sigmoid score of the best class, its index, x0, y0, x1, y1 in pixels (unclipped)} and,
 * optionally, labels [N][Q] int64.  Ties between classes resolve to the smallest index (torch.max).                 */
int tfb200_detect_postprocess_f32(const float* logits, const float* boxes, const int64_t* sizes_hw, float* packed,
                                  int64_t* labels, int N, int Q, int C, void* stream);
/* The same rows for the softmax classifier of vanilla DETR (PostProcess, detr.py:446-490): logits [N][Q][C] with the
 * last column "no object" (C >= 2); score = softmax probability of the best of the first C - 1 classes.            */
int tfb200_detect_postprocess_softmax_f32(const float* logits, const float* boxes, const int64_t* sizes_hw,
                                          float* packed, int64_t* labels, int N, int Q, int C, void* stream);

/* clip_grad_norm_ + AdamW (decoupled weight decay) over one contiguous fp32 range of n parameters in one pass
 * (engine.py:147-151 + torch.optim.AdamW of train.py:118).  grad_norm_dev: device scalar holding the global gradient
 * 2-norm, or NULL for no clipping; the clip coefficient min(1, max_norm / (norm + 1e-6)) is applied on the fly, the
 * gradient buffer is not modified.  step >= 1 is the update count (bias correction).  Pointers 16-byte aligned.      */
int tfb200_flat_adamw_f32(float* param, const float* grad, float* exp_avg, float* exp_avg_sq, int64_t n,
                          const float* grad_norm_dev, float max_norm, float lr, float beta1, float beta2, float eps,
                          float weight_decay, int64_t step, void* stream);

/* Frozen batch-norm + optional residual add + optional ReLU over channels-last activations ([pixels][C], C % 4 == 0):
 *   y = act(x * scale[c] + shift[c] (+ residual))          backbone.py:46-55 + torchvision Bottleneck.forward
 * backward: g = relu ? dy * (y > 0) : dy;  dx = g * scale[c] (NULL to skip);  dresidual = g (NULL when there was no
 * residual).  scale / shift are the folded per-channel terms (weight * rsqrt(var + eps), bias - mean * scale).        */
int tfb200_frozen_bn_act_fwd_f32(const float* x, const float* residual, const float* scale, const float* shift,
                                 float* y, int64_t pixels, int C, int relu, void* stream);
int tfb200_frozen_bn_act_bwd_f32(const float* dy, const float* y, const float* scale, float* dx, float* dresidual,
                                 int64_t pixels, int C, int relu, void* stream);

/* y[M][N] = act(x[M][K] . w[N][K]^T + bias[N])  -- the nn.Linear of the long-token projections / FFN
 * (ops/modules/ms_deform_attn.py:64,69,70,88; models/deformable_transformer.py:282-286) as ONE hand-written
 * wgmma kernel: TMA-staged 128x32 fp32 tiles, TF32 tensor-core products (wgmma.mma_async .tf32), fp32
 * accumulation in registers, bias (+ optional ReLU) in the epilogue, TMA store.  All row-major, contiguous, 16-byte aligned.
 * Requires N % 128 == 0 and K % 32 == 0 (tfb200_tf32_linear_supported); M is arbitrary.  bias may be NULL.
 * Returns -5 (unsupported) outside that domain: the caller keeps the library GEMM for those.                          */
int tfb200_tf32_linear_supported(int64_t M, int N, int K);
int tfb200_tf32_linear_f32(const float* x, const float* w, const float* bias, float* y, int64_t M, int N, int K,
                           int relu, void* stream);
/* The FFN's first Linear with its activation fused into the epilogue (models/deformable_transformer.py:282):
 *   h = (a > 0 && keep(seed, row * N + col)) ? a / keep_prob : 0,   a = x . w^T + bias
 * -- the mask of tfb200_relu_dropout_fwd_f32 on the same a, bit for bit.  seed_dev: the device int64 seed (read by
 * the kernel, so a captured graph draws a fresh mask per replay); training == 0 is plain ReLU and needs no seed. */
int tfb200_tf32_linear_relu_dropout_f32(const float* x, const float* w, const float* bias, const int64_t* seed_dev,
                                        float* h, int64_t M, int N, int K, float keep_prob, int training, void* stream);
/* The layer's two backward products on the same pipeline:
 *   dx[M][K]  = dy[M][N] . w[N][K]            (N % 32 == 0, K % 128 == 0; run as the forward product on wt = w^T,
 *                                              which is written into the caller's [K][N] workspace wt first)
 *   dw[N][K]  = dy[M][N]^T . x[M][K]          (N, K % 128 == 0; the token axis M is split over all SMs, the partial
 *                                              products are added into dw by TMA reductions; dw is zero-filled here)
 * dgrad_relu_dropout fuses the gradient of tfb200_tf32_linear_relu_dropout_f32's activation into the dgrad epilogue:
 *   ga[M][K]  = h[M][K] > 0 ? (dy . w) / keep_prob : 0          (training == 0: keep_prob is taken as 1)      */
int tfb200_tf32_linear_dgrad_f32(const float* dy, const float* w, float* wt, float* dx, int64_t M, int N, int K,
                                 void* stream);
int tfb200_tf32_linear_dgrad_relu_dropout_f32(const float* dy, const float* w, float* wt, const float* h, float* ga,
                                              int64_t M, int N, int K, float keep_prob, int training, void* stream);
int tfb200_tf32_linear_wgrad_f32(const float* dy, const float* x, float* dw, int64_t M, int N, int K, void* stream);

/* out[r][c] = sigmoid(delta[r][c] + inverse_sigmoid(ref[r][c]))  for c < ref_dim (2 or 4), sigmoid(delta[r][c]) beyond;
 * inverse_sigmoid(x) = log(clamp(clamp(x,0,1), eps) / clamp(1 - clamp(x,0,1), eps))  (util/misc.py:515-519) -- the box
 * refinement of deformable_transformer.py:412-422 / deformable_detr.py:229-248 in one launch.  delta/out [rows][4],
 * ref [rows][ref_dim].  backward: grad_delta [rows][4], grad_ref [rows][ref_dim] (NULL to skip), from grad_out and out. */
int tfb200_refine_boxes_fwd_f32(const float* delta, const float* ref, float* out, int64_t rows, int ref_dim, float eps,
                                void* stream);
int tfb200_refine_boxes_bwd_f32(const float* grad_out, const float* out, const float* ref, float* grad_delta,
                                float* grad_ref, int64_t rows, int ref_dim, float eps, void* stream);

/* SetCriterion / HungarianMatcher on the device (csrc/set_loss.cu; reference: models/matcher.py:60-100,
 * models/detr.py:213-328, util/misc.py:540-571, util/box_ops.py:24-61).  R = K*B*Q rows (layer, image, query).
 *   match_cost : cost[R][T] = w_bbox * L1 + w_class * focal class cost - w_giou * GIoU against the T boxes of the batch
 *   set_loss_fwd: src/tgt [K][T] are the matched (query, global box) pairs, columns offsets[b]..offsets[b+1]-1 belong to
 *                 image b; writes out5k[5][K] = loss_ce, loss_bbox, loss_giou, cardinality_error, class_error and the
 *                 UNIT gradients (unit_logits [R][C], unit_l1 / unit_giou [R][4]) that set_loss_bwd scales by the incoming
 *                 gradients g_*[K] / num_boxes.  n_gt [B] = boxes per image (float), num_boxes = device scalar.
 *                 row_loss [R], row_flags [R], pair_l1 / pair_giou [K][T] are scratch.                                  */
int tfb200_match_cost_f32(const float* logits, const float* boxes, const int64_t* tgt_ids, const float* tgt_boxes,
                          float* cost, int64_t R, int C, int T, float w_class, float w_bbox, float w_giou, float alpha,
                          float gamma, void* stream);
int tfb200_set_loss_fwd_f32(const float* logits, const float* boxes, const int64_t* src, const int64_t* tgt,
                            const int64_t* tgt_ids, const float* tgt_boxes, const int* offsets, const float* n_gt,
                            const float* num_boxes, float* unit_logits, float* unit_l1, float* unit_giou, float* row_loss,
                            int* row_flags, float* pair_l1, float* pair_giou, float* out5k, int K, int B, int Q, int C,
                            int T, float alpha, float gamma, void* stream);
/* Track-query training (models/matcher.py:112-128, models/detr_tracking.py):
 *   match_cost_track : match_cost for logits / boxes [K][B][Q] with the forcing of row_pin [B*Q] (int32, the same for all
 *                      K layers) applied in the same pass: -1 free row; c in [0, T) row pinned to global box c (its row
 *                      is +inf except -1 at c; column c is +inf for every other row of the image); any other value an
 *                      excluded row (all +inf: false-positive or filler track query).  T <= 49152.  Feeds tfb200_lsa_f32.
 *   set_loss_fwd_masked: set_loss_fwd with row_valid [B*Q] (uint8, the same for all layers): a zero row adds nothing to
 *                      loss_ce, is not counted by cardinality_error, has no pair terms and gets zero unit gradients (so
 *                      set_loss_bwd gives it a zero gradient).                                                        */
int tfb200_match_cost_track_f32(const float* logits, const float* boxes, const int64_t* tgt_ids, const float* tgt_boxes,
                                const int* row_pin, float* cost, int K, int B, int Q, int C, int T, float w_class,
                                float w_bbox, float w_giou, float alpha, float gamma, void* stream);
int tfb200_set_loss_fwd_masked_f32(const float* logits, const float* boxes, const int64_t* src, const int64_t* tgt,
                                   const int64_t* tgt_ids, const float* tgt_boxes, const int* offsets, const float* n_gt,
                                   const float* num_boxes, const uint8_t* row_valid, float* unit_logits, float* unit_l1,
                                   float* unit_giou, float* row_loss, int* row_flags, float* pair_l1, float* pair_giou,
                                   float* out5k, int K, int B, int Q, int C, int T, float alpha, float gamma,
                                   void* stream);
int tfb200_set_loss_bwd_f32(const float* unit_logits, const float* unit_l1, const float* unit_giou, const float* g_ce,
                            const float* g_l1, const float* g_giou, const float* num_boxes, float* grad_logits,
                            float* grad_boxes, int K, int B, int Q, int C, void* stream);
/* The same with the softmax classifier (focal_loss: false; models/matcher.py:77, models/detr.py:172-211).  Logits have
 * C = classes + 1 columns, the last one "no object" (C >= 2).
 *   match_cost_softmax / match_cost_track_softmax: class cost -softmax(logit_r)[label_t] (one log-sum-exp per row);
 *                      otherwise as match_cost / match_cost_track.
 *   set_loss_fwd_softmax: the weighted cross-entropy of loss_labels: target = matched label with weight 1, else no
 *                      object with weight eos_coef (> 0); loss_ce[k] = sum_r w_r ce_r / sum_r w_r.  row_valid [B*Q]
 *                      (optional) as in set_loss_fwd_masked.  row_pin [B*Q] (optional, see match_cost_track): when
 *                      given, a valid unmatched row with pin -2 (false-positive track query) has its ce scaled by
 *                      1 / eos_coef and counts 1 in the normaliser.  out6k[6][K] = out5k rows + the normaliser sum_r
 *                      w_r; row_norm [R] is scratch.  Box terms, cardinality_error and class_error as set_loss_fwd.
 *   set_loss_bwd_softmax: set_loss_bwd with the logit gradient scaled by g_ce[k] / ce_norm[k] (ce_norm = out6k + 5K). */
int tfb200_match_cost_softmax_f32(const float* logits, const float* boxes, const int64_t* tgt_ids,
                                  const float* tgt_boxes, float* cost, int64_t R, int C, int T, float w_class,
                                  float w_bbox, float w_giou, void* stream);
int tfb200_match_cost_track_softmax_f32(const float* logits, const float* boxes, const int64_t* tgt_ids,
                                        const float* tgt_boxes, const int* row_pin, float* cost, int K, int B, int Q,
                                        int C, int T, float w_class, float w_bbox, float w_giou, void* stream);
int tfb200_set_loss_fwd_softmax_f32(const float* logits, const float* boxes, const int64_t* src, const int64_t* tgt,
                                    const int64_t* tgt_ids, const float* tgt_boxes, const int* offsets,
                                    const float* n_gt, const float* num_boxes, const uint8_t* row_valid,
                                    const int* row_pin, float* unit_logits, float* unit_l1, float* unit_giou,
                                    float* row_loss, float* row_norm, int* row_flags, float* pair_l1, float* pair_giou,
                                    float* out6k, int K, int B, int Q, int C, int T, float eos_coef, void* stream);
int tfb200_set_loss_bwd_softmax_f32(const float* unit_logits, const float* unit_l1, const float* unit_giou,
                                    const float* g_ce, const float* g_l1, const float* g_giou, const float* num_boxes,
                                    const float* ce_norm, float* grad_logits, float* grad_boxes, int K, int B, int Q,
                                    int C, void* stream);

/* Stem of the ResNet trunk in one pass (csrc/frozen_bn_act.cu): y = maxpool 3x3 / stride 2 / pad 1 of
 * relu(x * scale[c] + shift[c]); x [N][H][W][C] channels-last, y [N][(H+1)/2][(W+1)/2][C]; forward only (frozen stem). */
int tfb200_frozen_bn_relu_maxpool_f32(const float* x, const float* scale, const float* shift, float* y, int N, int H, int W,
                                      int C, void* stream);

/* Dense self-attention over a few hundred positions, 32 channels per head (csrc/small_attn.cu; replaces the core of the
 * decoder's nn.MultiheadAttention, reference models/deformable_transformer.py:342,366-368).  q / k / v / out (and dout /
 * dq / dk / dv) are [L][B][H][32] VIEWS: channel stride 1, head stride 32, sequence / batch strides (in elements) in
 *   strides8  = {q_l, q_b, k_l, k_b, v_l, v_b, out_l, out_b}
 *   strides16 = strides8 + {dout_l, dout_b, dq_l, dq_b, dk_l, dk_b, dv_l, dv_b}
 * out = dropout(softmax(scale * q k^T + mask)) v; key_pad [B][L] (1 = ignore that key) or NULL; seed_dev NULL = no
 * dropout, else keep_prob in (0, 1] with the mask-free hash RNG; lse [B][H][L] (saved for the backward);
 * delta_ws [B][H][L] scratch.                                                                                       */
int tfb200_small_attn_fwd_f32(const float* q, const float* k, const float* v, const uint8_t* key_pad,
                              const int64_t* seed_dev, float* out, float* lse, int B, int H, int L,
                              const int64_t* strides8, float scale, float keep_prob, void* stream);
int tfb200_small_attn_bwd_f32(const float* q, const float* k, const float* v, const uint8_t* key_pad,
                              const int64_t* seed_dev, const float* out, const float* lse, const float* dout,
                              float* dq, float* dk, float* dv, float* delta_ws, int B, int H, int L,
                              const int64_t* strides16, float scale, float keep_prob, void* stream);

/* Dense multi-head attention over long key sequences, 32 channels per head (csrc/dense_attn.cu; replaces the core of the
 * three nn.MultiheadAttention calls of the vanilla transformer, reference models/transformer.py: encoder
 * self-attention, decoder self- and cross-attention).  Flash-style tiles, both products on tensor cores as split-TF32
 * (fp32-level accuracy), online softmax in fp32.  q / out / dout / dq are [Lq][B][H][32] VIEWS, k / v / dk / dv
 * [Lk][B][H][32] VIEWS: channel stride 1, head stride 32, 16-byte aligned base, sequence / batch strides (in elements,
 * multiples of 4) in
 *   strides8  = {q_l, q_b, k_l, k_b, v_l, v_b, out_l, out_b}
 *   strides16 = strides8 + {dout_l, dout_b, dq_l, dq_b, dk_l, dk_b, dv_l, dv_b}
 * out = dropout(softmax(scale * q k^T + mask)) v; Lq, Lk >= 1 independent; key_pad [B][Lk] (nonzero = ignore that key,
 * any pattern) or NULL; a query whose keys are all ignored gets a zero output.  seed_dev NULL = no dropout, else
 * keep_prob in (0, 1] with the mask-free hash RNG keyed by the element index ((b*H + h)*Lq + q)*Lk + k; lse [B][H][Lq]
 * (saved for the backward); delta_ws [B][H][Lq] scratch.  B*H <= 65535.  The backward uses no atomics: bitwise
 * reproducible.                                                                                                      */
int tfb200_dense_attn_fwd_f32(const float* q, const float* k, const float* v, const uint8_t* key_pad,
                              const int64_t* seed_dev, float* out, float* lse, int B, int H, int Lq, int Lk,
                              const int64_t* strides8, float scale, float keep_prob, void* stream);
int tfb200_dense_attn_bwd_f32(const float* q, const float* k, const float* v, const uint8_t* key_pad,
                              const int64_t* seed_dev, const float* out, const float* lse, const float* dout,
                              float* dq, float* dk, float* dv, float* delta_ws, int B, int H, int Lq, int Lk,
                              const int64_t* strides16, float scale, float keep_prob, void* stream);
/* The attention probabilities of the forward averaged over heads (nn.MultiheadAttention's need_weights=True,
 * average_attn_weights=True): weights [B][Lq][Lk] (contiguous) = (1/H) sum_h exp(scale q_h . k_h - lse[b][h][q]),
 * from the same q / k views (strides4 = {q_l, q_b, k_l, k_b}, alignment as above) and the lse [B][H][Lq] of
 * tfb200_dense_attn_fwd_f32; dropout does not enter.  Ignored keys (key_pad nonzero) get exactly 0, and so does every
 * key of a query whose keys are all ignored.  One launch, no atomics: bitwise reproducible.  B <= 65535.          */
int tfb200_dense_attn_weights_f32(const float* q, const float* k, const uint8_t* key_pad, const float* lse,
                                  float* weights, int B, int H, int Lq, int Lk, const int64_t* strides4, float scale,
                                  void* stream);

/* One frame of the online tracker's bookkeeping on the device (csrc/track_step.cu; reference models/tracker.py:266-548:
 * score thresholds 337-373 / 425-436, both NMS passes 388-406 / 494-515, public-detection gating 122-164, ReID 166-264,
 * results 533-545, reid_sim_only 547-548).  One CTA takes every decision of Tracker.step in the reference's order.
 *
 * State is a struct of arrays in track order: entries [0, n_active) are the active tracks, [n_active, n_active +
 * n_inactive) the inactive ones, both in the reference's list order.  header = {n_active, n_inactive, track_num,
 * num_reids, n_query_next, error, n_results, 0}.  `in` is CONSUMED (it is the kernel's work table, rows beyond the
 * tracks are used for this frame's object queries: capacity >= n_active + n_inactive + nq, <= 2048); `out` receives
 * the new state, `q_boxes` / `q_embeds` the track queries of the next frame (active tracks, then the inactive ones that
 * survive the patience / positive-area test, boxes as cx, cy, w, h divided by the image size), and `result` the header
 * followed by n_results rows of 8 words {id, obj_ind, score, x0, y0, x1, y1, src} (ints and fp32 bit patterns); src is
 * the query row whose embedding -- and so whose segmentation mask -- the track took this frame, or -1 if it took none.
 * error: 1 = n_query does not match the state, 2 = capacity.                                                         */
typedef struct TfbTrackState {
  int32_t* header;             /* [8] */
  int32_t* ids;                /* [capacity] */
  float* pos;                  /* [capacity][4]  x0, y0, x1, y1 in pixels */
  float* anchor;               /* [capacity][4]  position at the start of the step (Track.last_pos[-1]) */
  float* score;                /* [capacity] */
  int32_t* obj_ind;            /* [capacity] */
  int32_t* count_inactive;     /* [capacity] */
  int32_t* count_termination;  /* [capacity] */
  float* bank;                 /* [capacity][hidden] last output embedding of every track */
} TfbTrackState;

typedef struct TfbTrackStepArgs {
  const float* rows;           /* [n_query + nq][6] packed detections of this frame (tfb200_detect_postprocess_f32) */
  const float* hs_embeds;      /* [n_query + nq][hidden] decoder output embeddings */
  const float* public_dets;    /* [n_public][4] pixel xyxy, or NULL */
  TfbTrackState in, out;
  float* q_boxes;              /* [capacity][4] */
  float* q_embeds;             /* [capacity][hidden] */
  int32_t* result;             /* [8 + 8 * capacity] */
  int32_t* iscratch;           /* [16 * capacity] */
  float* fscratch;             /* [8 * capacity + capacity * max(nq, n_public, 1)] */
  double* dscratch;            /* [4 * capacity] */
  double inactive_patience, reid_sim_threshold;
  float detection_obj_score_thresh, track_obj_score_thresh, reid_score_thresh, detection_nms_thresh, track_nms_thresh;
  int32_t capacity, hidden, nq, n_query, n_public, img_h, img_w;
  int32_t overflow_boxes, public_mode /* 0 off, 1 center_distance, 2 min_iou_0_5 */, reid_greedy_matching,
      reid_sim_only, steps_termination, detection_nms_on, track_nms_on;
} TfbTrackStepArgs;

int tfb200_track_step_f32(const TfbTrackStepArgs* args, void* stream);

/* n independent sequences in ONE launch of n CTAs: CTA b takes every decision of tfb200_track_step_f32 on args[b]
 * (its own state, scratch, result buffer, public detections and thresholds), so the results are those of n single
 * calls.  The n structs are passed by value (kernel parameter space), so the launch reads no host memory and can be
 * captured in a CUDA graph.  n must be 1..16, else TFB200_E_SHAPE; any invalid args[b] returns what
 * tfb200_track_step_f32 returns for it.  On an error nothing is launched.                                          */
int tfb200_track_step_batched_f32(const TfbTrackStepArgs* args, int n, void* stream);

/* Segmentation mask head between its convolutions, and its loss (csrc/mask_head.cu; reference
 * models/detr_segmentation.py:111-216, models/detr.py:330-357).  Per-query maps are channels-last [N][HW][C] with
 * N = images * per_image; an operand "per image" is [N / per_image][...] and is broadcast over that image's queries
 * instead of being expanded.  Reductions over queries and samples run in a fixed order (no float atomics).
 *
 * mask_attn: w [B][Q][heads][HW] = scale * q . k per head, -inf where pad, then one softmax over each query's
 *   heads * HW entries together (MHAttentionMap, head width 32): the heads of a query share one partition sum.
 *   q [B][Q][heads*32], k [B][HW][heads*32] token-major, pad [B][HW] bool or NULL; heads <= 256.  q, k (and dk)
 *   must be 16-byte aligned, else TFB200_E_SHAPE.  backward: dq, dk from dw; ds_ws [B][Q][heads][HW] scratch.     */
int tfb200_mask_attn_fwd_f32(const float* q, const float* k, const uint8_t* pad, float* w, int B, int Q, int HW,
                             int heads, float scale, void* stream);
int tfb200_mask_attn_bwd_f32(const float* q, const float* k, const float* w, const float* dw, float* ds_ws, float* dq,
                             float* dk, int B, int Q, int HW, int heads, float scale, void* stream);
/* group_norm_relu: y = relu(GroupNorm_groups(x + addend) * gamma + beta), addend [N / per_image][HW][C] or NULL;
 * mean / rstd [N][groups] are saved for the backward.  C / groups <= 256.  backward: dx, daddend (summed over each
 * image's queries; required when addend is given), daffine [2][C] = {dgamma, dbeta}; partial_ws [N][2][C] scratch. */
int tfb200_group_norm_relu_fwd_f32(const float* x, const float* addend, const float* gamma, const float* beta, float* y,
                                   float* mean, float* rstd, int N, int per_image, int64_t HW, int C, int groups,
                                   float eps, void* stream);
int tfb200_group_norm_relu_bwd_f32(const float* dy, const float* x, const float* addend, const float* y,
                                   const float* gamma, const float* mean, const float* rstd, float* dx, float* daddend,
                                   float* daffine, float* partial_ws, int N, int per_image, int64_t HW, int C,
                                   int groups, void* stream);
/* upsample_add: out [N][Ho][Wo][C] = a[n / per_image] + x[n] nearest-upsampled from [Hi][Wi] (F.interpolate's
 * nearest rule).  backward: dx [N][Hi][Wi][C] (block sums) and da [N / per_image][Ho][Wo][C] (sum over queries).    */
int tfb200_upsample_add_fwd_f32(const float* x, const float* a, float* out, int N, int per_image, int Hi, int Wi,
                                int Ho, int Wo, int C, void* stream);
int tfb200_upsample_add_bwd_f32(const float* dout, float* dx, float* da, int N, int per_image, int Hi, int Wi, int Ho,
                                int Wo, int C, void* stream);
/* Ragged variants of the three (the matched query rows of a training step): P rows over B images, image b owning
 * rows row_offsets[b] .. row_offsets[b + 1] (int32 [B + 1] on the device: row_offsets[0] = 0, non-decreasing,
 * row_offsets[B] = P -- not checked on the host, which never reads it).  An image may own no rows: its attention-key
 * gradient and its per-image operand gradients are then zero.  Same kernels, arithmetic and summation order as the
 * per_image entry points, which equal these with row_offsets[b] = b * per_image.  mask_attn: q [P][heads*32],
 * w / ds_ws [P][heads][HW], k / dk [B][HW][heads*32].  group_norm_relu: addend [B][HW][C] is required, mean / rstd
 * [P][groups], partial_ws [P][2][C].  upsample_add: x [P][Hi][Wi][C], a / da [B][Ho][Wo][C].  P = 0 is legal
 * (forwards: no-ops; backwards: zero per-image gradients); B = 0 requires P = 0.                                    */
int tfb200_mask_attn_rows_fwd_f32(const float* q, const float* k, const uint8_t* pad, const int32_t* row_offsets,
                                  float* w, int B, int P, int HW, int heads, float scale, void* stream);
int tfb200_mask_attn_rows_bwd_f32(const float* q, const float* k, const int32_t* row_offsets, const float* w,
                                  const float* dw, float* ds_ws, float* dq, float* dk, int B, int P, int HW, int heads,
                                  float scale, void* stream);
int tfb200_group_norm_relu_rows_fwd_f32(const float* x, const float* addend, const int32_t* row_offsets,
                                        const float* gamma, const float* beta, float* y, float* mean, float* rstd,
                                        int B, int P, int64_t HW, int C, int groups, float eps, void* stream);
int tfb200_group_norm_relu_rows_bwd_f32(const float* dy, const float* x, const float* addend,
                                        const int32_t* row_offsets, const float* y, const float* gamma,
                                        const float* mean, const float* rstd, float* dx, float* daddend,
                                        float* daffine, float* partial_ws, int B, int P, int64_t HW, int C, int groups,
                                        void* stream);
int tfb200_upsample_add_rows_fwd_f32(const float* x, const float* a, const int32_t* row_offsets, float* out, int B,
                                     int P, int Hi, int Wi, int Ho, int Wo, int C, void* stream);
int tfb200_upsample_add_rows_bwd_f32(const float* dout, const int32_t* row_offsets, float* dx, float* da, int B, int P,
                                     int Hi, int Wi, int Ho, int Wo, int C, void* stream);
/* mask_loss: M matched pairs (logits row src[m] of [R][h][w], target mask tgt[m] of [T][Ht][Wt] bool).  The logits
 * are sampled bilinearly (align_corners=False) at every target pixel on the fly; out2 = {sigmoid focal loss (mean
 * over pixels), dice} summed over pairs and divided by the device scalar *num_boxes.  M == 0 gives zeros.
 * stats [M][4] are saved for the backward; partial_ws [M][tfb200_mask_loss_partial_chunks(Ht, Wt)][4] scratch.
 * backward: grad_logits [R][h][w] (zero outside the matched rows) from g2 = {dL/dloss_mask, dL/dloss_dice}.
 * Precondition: src holds no row twice (a one-to-one matching guarantees it); each matched row's gradient is written,
 * not accumulated.                                                                                                */
int tfb200_mask_loss_partial_chunks(int Ht, int Wt);
int tfb200_mask_loss_fwd_f32(const float* logits, const int64_t* src, const uint8_t* tgt_masks, const int64_t* tgt,
                             const float* num_boxes, float* stats, float* partial_ws, float* out2, int M, int h, int w,
                             int Ht, int Wt, float alpha, float gamma, void* stream);
int tfb200_mask_loss_bwd_f32(const float* logits, const int64_t* src, const uint8_t* tgt_masks, const int64_t* tgt,
                             const float* stats, const float* num_boxes, const float* g2, float* grad_logits, int R,
                             int M, int h, int w, int Ht, int Wt, float alpha, float gamma, void* stream);

/* Segmentation masks of the tracker's active tracks resolved into one label map (csrc/track_masks.cu; reference
 * models/detr_segmentation.py:219-253 with return_probs=True, models/tracker.py:509-521).  T tracks in active-list
 * order; src[t] is the row of logits [K][h][w] (stride-4 mask logits) the track takes this frame, or -1 for a track
 * that keeps its previous mask, which is prev_label == ids[t] (value exactly 1.0).  A fresh track's value at output
 * pixel (y, x) of [H][W] is sigmoid(bilinear (align_corners=False) upsampling to [size_h][size_w]) at the nearest
 * source pixel of the [crop_h][crop_w] crop.  label[y][x] = ids[first t of maximal value] if that value > 0.5, else
 * -1.  ids >= 0 and unique; logits may be NULL when no src is >= 0; prev_label [H][W] or NULL (no stale tracks).
 * T == 0 writes nothing.                                                                                          */
int tfb200_track_masks_f32(const float* logits, const int32_t* src, const int32_t* ids, const int32_t* prev_label,
                           int32_t* label, int T, int h, int w, int size_h, int size_w, int crop_h, int crop_w, int H,
                           int W, void* stream);

/* tfb200_track_masks_f32 for n images (1..16, else TFB200_E_SHAPE) in ONE launch: args[b] holds image b's arguments,
 * each with its own logits, src, ids, prev_label, label and sizes (label sizes may differ).  Image b's label map equals
 * tfb200_track_masks_f32 on args[b] bit for bit; tfb200_track_masks_f32 is this entry with n = 1.  The structs are
 * passed by value (kernel parameter space).  A NULL args or an invalid args[b] returns what tfb200_track_masks_f32
 * returns for it, and nothing is launched; images with T == 0 are not written.                                    */
typedef struct TfbTrackMasksArgs {
  const float* logits;
  const int32_t* src;
  const int32_t* ids;
  const int32_t* prev_label;
  int32_t* label;
  int T, h, w, size_h, size_w, crop_h, crop_w, H, W;
} TfbTrackMasksArgs;

int tfb200_track_masks_batched_f32(const TfbTrackMasksArgs* args, int n, void* stream);

/* COCO run-length encodings of the masks label == ids[t] of a label map (csrc/mask_rle.cu; what pycocotools
 * mask.encode(np.asfortranarray(label == ids[t]))["counts"] holds, for MOTS20Sequence.write_results,
 * datasets/tracking/mots20_sequence.py:72-91).  label [H][W] int32 row-major (e.g. tfb200_track_masks_f32's output);
 * ids [T] int32, >= 0, in any order, duplicates allowed (they get equal strings); label values that are not in ids,
 * negative ones included, are background for every track.  Writes header [2 + 2T] int64 = {status, total bytes,
 * offset[T], length[T]} and the T strings back to back into chars (offset[t] .. offset[t] + length[t]).  status bit 1:
 * a negative id (its string is that of an empty mask); bit 2: total > chars_capacity, and chars is left untouched.
 * tfb200_mask_rle_max_bytes(H, W, T) bounds the total for any label map.  workspace: tfb200_mask_rle_workspace_bytes
 * bytes, 256-byte aligned (0 for a bad shape).  H * W <= 2^28, T <= 2^24.  T == 0 writes nothing.  Deterministic.  */
size_t tfb200_mask_rle_workspace_bytes(int H, int W, int T);
int64_t tfb200_mask_rle_max_bytes(int H, int W, int T);
int tfb200_mask_rle_i32(const int32_t* label, const int32_t* ids, int H, int W, int T, void* workspace,
                        size_t workspace_bytes, int64_t* header, char* chars, int64_t chars_capacity, void* stream);

/* tfb200_mask_rle_i32 for n label maps (1..16, else TFB200_E_SHAPE) at once: map b is maps[b].label [H][W] with its
 * own H, W, ids and T.  ONE header [2 + 2 * sum(T)] int64 = {status, total bytes, offset[sum T], length[sum T]} and one
 * character buffer hold every string, tracks ordered map after map and in ids order within a map; each string is
 * byte-equal to tfb200_mask_rle_i32's for its map.  Each stage is one launch over all maps (nine launches and four
 * memsets, whatever n), and tfb200_mask_rle_i32 is this entry with n = 1.  Every map must satisfy the single entry's
 * limits, sum T <= 2^24, and the boundary lists of all maps share int32 offsets: sum over maps of 2 H W must be
 * < 2^31, else TFB200_E_SHAPE (and the size queries return 0).  A map with T == 0 has no strings.                 */
typedef struct TfbMaskRleMap {
  const int32_t* label;
  const int32_t* ids;
  int H, W, T;
} TfbMaskRleMap;

size_t tfb200_mask_rle_batched_workspace_bytes(const TfbMaskRleMap* maps, int n);
int64_t tfb200_mask_rle_batched_max_bytes(const TfbMaskRleMap* maps, int n);
int tfb200_mask_rle_batched_i32(const TfbMaskRleMap* maps, int n, void* workspace, size_t workspace_bytes,
                                int64_t* header, char* chars, int64_t chars_capacity, void* stream);

/* MOTChallenge CLEAR-MOT and identity metrics of S sequences at once (csrc/mot_eval.cu; what motmetrics 1.2.0
 * computes for get_mot_accum / evaluate_mot_accums, src/trackformer/util/track_utils.py:354-417).  F frames over all
 * sequences in order; frame f holds object rows frame_obj[f] .. frame_obj[f + 1] and hypothesis rows frame_hyp[f] ..
 * frame_hyp[f + 1] (int32 [F + 1], non-decreasing, from 0), in the order motmetrics is given them.  obj_id / hyp_id:
 * the row's dense GT / track id within its sequence; obj_box / hyp_box [rows][4] float32 x, y, w, h.  seq [S][8]
 * int64 = {frame begin, frame end, GT-id begin, GT-id count, track-id begin, track-id count, tp-cell begin, 0}: the
 * GT ids of sequence s are n_gt's entries from its begin (likewise tracks), its tp matrix [GT-id count][track-id
 * count] int32 starts at its tp-cell begin of tp_cells.  A pair is valid when 1 - IoU <= 0.5 (fp64 IoU of the boxes
 * extended to x + w, y + h).  Writes out [S][16] 8-byte slots = {status, valid pairs, matches, switches, misses, false
 * positives, fragmentations, mostly tracked, partially tracked, mostly lost, IDTP, largest residual component of a
 * frame (objects, hypotheses), largest identity component (GT ids, track ids), sum of d over matches and switches as
 * a double}.  status bit 1: more than pair_cap valid pairs (slot 1 holds the count; nothing past the pairs is
 * computed: call again with pair_cap >= the sum of slot 1); bit 2: a frame with more than max_obj objects or max_hyp
 * hypotheses; bit 4: a residual component over 64 objects or 64 hypotheses; bit 8: an identity component whose
 * smaller side (GT ids or track ids) is over 8192 or larger side over 65536.  A set bit leaves that sequence's counts
 * incomplete.  Workspace: tfb200_mot_eval_workspace_bytes(...) bytes (0 for bad sizes), about 16 B per pair of
 * pair_cap plus 4 B per tp cell.  Integer counts are exact and every output is the same run to run.  Sizes out of
 * range: TFB200_E_SHAPE.                                                                                           */
size_t tfb200_mot_eval_workspace_bytes(int S, int F, int64_t n_gt, int64_t n_trk, int64_t tp_cells, int max_obj,
                                       int max_hyp, int64_t pair_cap);
int tfb200_mot_eval_f32(const int64_t* seq, const int32_t* frame_obj, const int32_t* frame_hyp, const int32_t* obj_id,
                        const float* obj_box, const int32_t* hyp_id, const float* hyp_box, int S, int F, int64_t n_gt,
                        int64_t n_trk, int64_t tp_cells, int max_obj, int max_hyp, int64_t pair_cap, void* workspace,
                        size_t workspace_bytes, int64_t* out, void* stream);

/* MOTS metrics of S sequences at once (csrc/mots_eval.cu, csrc/mots_eval_core.h): the pairs of tfb200_mot_eval_f32
 * from masks given as COCO RLE counts strings (pycocotools rleToString), then its matching unchanged.  seq [S][8] as
 * tfb200_mot_eval_f32's; seq_hw [S][2] int32 the sequence's H, W (H x W < 2^28).  F frames over all sequences in
 * order; frame_mask int32 [3F + 1]: frame f's GT masks are rows frame_mask[3f] .., its ignore regions frame_mask[3f +
 * 1] .., its hypotheses frame_mask[3f + 2] .. frame_mask[3f + 3]; frame_cell int64 [F + 1] the prefix sums of (GT
 * masks + 1) x hypotheses per frame (cells = the total); frame_obj int32 [F + 1] the prefix sums of GT masks, obj_id
 * [n_obj] their dense GT ids.  mask [n_masks][4] int32 = {frame, dense id (GT id, track id or 0), H, W}; mask k's
 * string is chars[str_off[k] .. str_off[k + 1]) (str_off int64 [n_masks + 1]).  interval_cap >= the sum over masks
 * of floor(string length / 2), < 2^31; pair_cap >= min(sum of GT x hypotheses per frame, 2 x GT masks) (a GT mask
 * has at most two partners with IoU >= 0.5 when hypotheses do not overlap).  A pair is valid when its pixel counts
 * give inter > 0 and 2 inter >= union, with d = 1 - inter / union; a hypothesis with no valid pair and 2 |h & ignore| >
 * |h| is removed.  Writes out [S][16] as tfb200_mot_eval_f32 (hypotheses = the kept ones) followed by [S][11] =
 * {status, GT masks, kept hypotheses, removed hypotheses, intervals, intersecting (GT, hypothesis) pairs, then the
 * first sequence-local frame of status bits 1, 2, 4, 8, 16 (INT64_MAX when unset)}.  status bit 1: GT masks or ignore
 * regions of a frame overlap; 2: hypotheses of a frame overlap; 4: a mask whose size differs from its sequence's (or
 * H x W out of range); 8: a malformed string (a character outside '0' .. 'o', a value cut short or of more than 7
 * characters, a negative count) or runs that do not cover H x W; 16: more intervals than interval_cap (nothing is
 * decoded).  A bad mask contributes no pixels; a set bit leaves the sequence's counts meaningless.  Workspace:
 * tfb200_mots_eval_workspace_bytes(...) (0 for bad sizes), about 32 B per interval of interval_cap plus 4 B per cell
 * and tfb200_mot_eval_f32's.  Integer counts are exact and every output is the same run to run.  Sizes out of range:
 * TFB200_E_SHAPE.                                                                                                  */
size_t tfb200_mots_eval_workspace_bytes(int S, int F, int n_masks, int64_t n_gt, int64_t n_trk, int64_t tp_cells,
                                        int max_obj, int max_hyp, int64_t pair_cap, int64_t interval_cap,
                                        int64_t cells);
int tfb200_mots_eval(const int64_t* seq, const int32_t* seq_hw, const int32_t* frame_mask, const int64_t* frame_cell,
                     const int32_t* frame_obj, const int32_t* obj_id, const int32_t* mask, const int64_t* str_off,
                     const uint8_t* chars, int S, int F, int n_masks, int64_t n_gt, int64_t n_trk, int64_t tp_cells,
                     int max_obj, int max_hyp, int64_t pair_cap, int64_t interval_cap, int64_t cells, void* workspace,
                     size_t workspace_bytes, int64_t* out, void* stream);

/* COCO box / mask AP (csrc/coco_eval.cu; what pycocotools 2.0's COCOeval computes for the reference's CocoEvaluator,
 * datasets/coco_eval.py).  tfb200_coco_match_f32 evaluates the B images of one update.  img [B][10] int64 = {GT image
 * row, first detection row, detection count, H, W, device address of the image's masks uint8/bool [n][H][W] (segm),
 * IoU-matrix offset (cells), detection bit-plane offset (words), GT bit-plane offset (words), matched-flag offset
 * (bytes)}, the offsets laid out by the caller (per image n x G IoU cells, n x W x ceil(H / 32) and G x W x ceil(H / 32)
 * words, A x T x G bytes, G = the image's GT rows); max_n / max_g the largest n / G.  boxes [N][4] float32 x0, y0,
 * x1, y1, scores [N] float32, labels [N] int64 (category id = label + 1), cat_ids [K] ascending.  Ground truth of the
 * whole dataset: gt_off [images + 1], per row (sorted by category index within an image, JSON order otherwise) gt_k,
 * gt_box [4] x, y, w, h fp64, gt_area fp64, gt_crowd, gt_id int64; segm: gt_run_off / gt_runs [runs][2] (column-major
 * start, length of each run of ones), gt_bbox [4] int32 inclusive tight box, gt_px pixel count.  area_rng [A][2],
 * iou_thr [T] (min(t, 1 - 1e-10)), max_det (maxDets[-1]).  Writes per detection the sort key ((category index << 32)
 * | descending-score bits, K << 32 when it is not evaluated), its rank within (image, category) and state [N][A]
 * 2 bits per threshold (0 false positive, 1 true positive, 2 ignored), and ors 1 into status for a non-finite score.
 * Limits: n <= TFB200_COCO_MAX_DETS detections per image (TFB200_E_SHAPE beyond), A <= 8, T <= 16; the evaluator
 * also keeps an image's ground truths of one category <= TFB200_COCO_MAX_GT.  Sizes out of range: TFB200_E_SHAPE.
 * tfb200_coco_accumulate_f32 runs accumulate over the records of all updates (key, rank, state as written above,
 * n_rec rows): kept [n_kept][3] = {record begin, destination begin, count} of every evaluated image in image-id order
 * (n = the sum of counts), npig [K][A] non-ignored GT counts, rec_thr [R] (R <= 1024), max_dets [M] (M <= 8).  Writes
 * precision / scores [T][R][K][A][M] and recall [T][K][A][M] fp64 (-1 where npig is 0), and status_out = status.
 * Deterministic.  Workspaces: the *_workspace_bytes queries (0 for bad sizes), 256-byte aligned.  The match
 * workspace is laid out for every detection and ground truth of each image (the caller cannot know which detections
 * rank within the first max_det of their category without reading the scores back): 8 B per IoU cell, plus for segm
 * 4 B x W x ceil(H / 32) per detection and per ground truth, e.g. about 78 MB for 300 detections at 1080 x 1920. */
#define TFB200_COCO_MAX_DETS 4096
#define TFB200_COCO_MAX_GT 4096
size_t tfb200_coco_match_workspace_bytes(int64_t N, int64_t iou_cells, int64_t dbit_words, int64_t gbit_words,
                                         int64_t gtm_bytes);
int tfb200_coco_match_f32(const int64_t* img, int B, int max_n, int max_g, const float* boxes, const float* scores,
                          const int64_t* labels, int64_t N, const int64_t* cat_ids, int K, const int64_t* gt_off,
                          const int32_t* gt_k, const double* gt_box, const double* gt_area, const uint8_t* gt_crowd,
                          const int64_t* gt_id, const int64_t* gt_run_off, const uint32_t* gt_runs,
                          const int32_t* gt_bbox, const int64_t* gt_px, const double* area_rng, int A,
                          const double* iou_thr, int T, int max_det, int segm, int64_t iou_cells, int64_t dbit_words,
                          int64_t gbit_words, int64_t gtm_bytes, void* workspace, size_t workspace_bytes,
                          uint64_t* key, int32_t* rank, uint32_t* state, int32_t* status, void* stream);
size_t tfb200_coco_accumulate_workspace_bytes(int64_t n);
int tfb200_coco_accumulate_f32(const uint64_t* key, const int32_t* rank, const uint32_t* state, int64_t n_rec,
                               const int64_t* kept, int n_kept, int64_t n, const int64_t* npig, const double* rec_thr,
                               const int32_t* max_dets, const int32_t* status, int K, int A, int T, int R, int M,
                               void* workspace, size_t workspace_bytes, double* precision, double* recall,
                               double* scores, double* status_out, void* stream);

/* Frame ingest (csrc/frame_ingest.cu; reference: the per-frame host work of datasets/tracking/mot17_sequence.py:68-81,
 * i.e. Pillow's bilinear resize of the 8-bit image, to_tensor and Normalize): src [H][W][3] interleaved uint8 with
 * src_row_stride bytes between rows (>= 3 * W)  ->  dst[c * dst_plane_stride + y * dst_row_stride + x] fp32, c < 3,
 * y < h, x < w (strides in elements, so dst may be one image of a padded batch; 4-byte aligned).  Bit-identical to
 * Pillow: per axis a device table of w (h) rows {lo, cnt, k_0 .. k_{ksize-1}} int32, weights quantised to 22 fractional
 * bits; a pass is clamp((2^21 + sum_{j < cnt} pixel[lo + j] * k_j) >> 22, 0, 255), horizontal first, rounded to a byte
 * between the passes.  xtab == NULL skips the horizontal pass and requires w == W, ytab == NULL likewise for rows; with
 * both NULL the call only converts.  cnt_max_* is the largest cnt of that table (it bounds the shared-memory footprint
 * of a tile); cnt_max > ksize is TFB200_E_SHAPE, as are non-positive sizes, and nothing is launched.  Every table row
 * must satisfy lo >= 0, lo + cnt <= the input length and lo non-decreasing -- not checked, the host never reads the
 * tables.  lut [3][256] fp32 maps the final byte of channel c to its normalised value.  Any ksize is handled until one
 * output row's footprint exceeds 200 KB of shared memory (a reduction by several hundred: TFB200_E_SHAPE).        */
int tfb200_frame_ingest_u8_f32(const uint8_t* src, int64_t src_row_stride, int H, int W, const int32_t* xtab,
                               int ksize_x, int cnt_max_x, const int32_t* ytab, int ksize_y, int cnt_max_y,
                               const float* lut, float* dst, int64_t dst_row_stride, int64_t dst_plane_stride, int h,
                               int w, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* TFB200_FUSED_H_ */
