// Python module `MultiScaleDeformableAttention` -- same name and same two entry points as the
// reference's pybind surface (src/trackformer/models/ops/src/vision.cpp:4-7,
// src/ms_deform_attn.h:10-50), so `import MultiScaleDeformableAttention as MSDA` in the
// reference's ops/functions/ms_deform_attn_func.py:11 resolves to this library unchanged.
//
// This file is glue only: argument validation, output allocation, current-stream lookup and
// a call through the C ABI of libmsda_b200 (include/msda_b200.h).  Differences from the
// reference glue, all deliberate:
//   * kernel-launch / CUDA errors raise (the reference printf()s them, ms_deform_im2col_cuda.cuh:404-408)
//   * no `columns` scratch tensor, no at::sum, no per-level ATen ops for level_start_index
//   * im2col_step is validated exactly like the reference (ms_deform_attn_cuda.cu:46-48) and then
//     ignored: one launch covers the whole batch
//   * CPU tensors raise "Not implemented on the CPU" like ms_deform_attn.h:27 -- there is no CPU fallback
#include <torch/extension.h>

#include <c10/cuda/CUDAGuard.h>
#include <c10/cuda/CUDAStream.h>

#include <algorithm>
#include <vector>

#include "../../include/msda_b200.h"
#include "../../include/tfb200_fused.h"

namespace {

struct Geometry {
  int N, S, M, D, L, Lq, P;
};

Geometry validate(const at::Tensor& value, const at::Tensor& spatial_shapes,
                  const at::Tensor& sampling_loc, const at::Tensor& attn_weight,
                  int64_t im2col_step) {
  TORCH_CHECK(value.is_cuda(), "Not implemented on the CPU");
  TORCH_CHECK(spatial_shapes.is_cuda(), "spatial_shapes must be a CUDA tensor");
  TORCH_CHECK(sampling_loc.is_cuda(), "sampling_loc must be a CUDA tensor");
  TORCH_CHECK(attn_weight.is_cuda(), "attn_weight must be a CUDA tensor");
  TORCH_CHECK(value.is_contiguous(), "value tensor has to be contiguous");
  TORCH_CHECK(value.scalar_type() == at::kFloat || value.scalar_type() == at::kDouble,
              "ms_deform_attn: value must be float32 or float64, got ", value.scalar_type());
  TORCH_CHECK(sampling_loc.scalar_type() == value.scalar_type() &&
                  attn_weight.scalar_type() == value.scalar_type(),
              "ms_deform_attn: value, sampling_loc and attn_weight must share one dtype");
  TORCH_CHECK(spatial_shapes.scalar_type() == at::kLong, "spatial_shapes must be int64");
  TORCH_CHECK(value.dim() == 4, "value must be [N, S, M, D]");
  TORCH_CHECK(spatial_shapes.dim() == 2 && spatial_shapes.size(1) == 2, "spatial_shapes must be [L, 2]");
  TORCH_CHECK(sampling_loc.dim() == 6 && sampling_loc.size(5) == 2,
              "sampling_loc must be [N, Lq, M, L, P, 2]");
  TORCH_CHECK(attn_weight.dim() == 5, "attn_weight must be [N, Lq, M, L, P]");
  Geometry g;
  g.N = int(value.size(0));
  g.S = int(value.size(1));
  g.M = int(value.size(2));
  g.D = int(value.size(3));
  g.L = int(spatial_shapes.size(0));
  g.Lq = int(sampling_loc.size(1));
  g.P = int(sampling_loc.size(4));
  TORCH_CHECK(sampling_loc.size(0) == g.N && sampling_loc.size(2) == g.M && sampling_loc.size(3) == g.L,
              "sampling_loc shape does not match value / spatial_shapes");
  TORCH_CHECK(attn_weight.size(0) == g.N && attn_weight.size(1) == g.Lq && attn_weight.size(2) == g.M &&
                  attn_weight.size(3) == g.L && attn_weight.size(4) == g.P,
              "attn_weight shape does not match sampling_loc");
  TORCH_CHECK(value.device() == spatial_shapes.device() && value.device() == sampling_loc.device() &&
                  value.device() == attn_weight.device(),
              "ms_deform_attn: all tensors must live on the same device");
  const int64_t step = std::min<int64_t>(g.N, im2col_step);
  TORCH_CHECK(g.N == 0 || (step > 0 && g.N % step == 0), "batch(", g.N, ") must divide im2col_step(", step, ")");
  return g;
}

void raise_on_error(int rc, const char* what) {
  TORCH_CHECK(rc == 0, what, " failed: ", msda_b200_error_string(rc), " (code ", rc, ")");
}

}  // namespace

at::Tensor ms_deform_attn_forward(const at::Tensor& value, const at::Tensor& spatial_shapes,
                                  const at::Tensor& sampling_loc, const at::Tensor& attn_weight,
                                  const int64_t im2col_step) {
  const Geometry g = validate(value, spatial_shapes, sampling_loc, attn_weight, im2col_step);
  const c10::cuda::CUDAGuard guard(value.device());
  const at::Tensor shapes = spatial_shapes.contiguous();
  const at::Tensor loc = sampling_loc.contiguous();
  const at::Tensor attn = attn_weight.contiguous();
  at::Tensor out = at::empty({g.N, g.Lq, int64_t(g.M) * g.D}, value.options());
  void* stream = c10::cuda::getCurrentCUDAStream().stream();
  int rc;
  if (value.scalar_type() == at::kFloat) {
    rc = msda_b200_forward_f32(value.data_ptr<float>(), shapes.data_ptr<int64_t>(), loc.data_ptr<float>(),
                               attn.data_ptr<float>(), out.data_ptr<float>(), g.N, g.S, g.M, g.D, g.L,
                               g.Lq, g.P, stream);
  } else {
    rc = msda_b200_forward_f64(value.data_ptr<double>(), shapes.data_ptr<int64_t>(), loc.data_ptr<double>(),
                               attn.data_ptr<double>(), out.data_ptr<double>(), g.N, g.S, g.M, g.D, g.L,
                               g.Lq, g.P, stream);
  }
  raise_on_error(rc, "ms_deform_attn_forward");
  return out;
}

std::vector<at::Tensor> ms_deform_attn_backward(const at::Tensor& value, const at::Tensor& spatial_shapes,
                                                const at::Tensor& sampling_loc,
                                                const at::Tensor& attn_weight,
                                                const at::Tensor& grad_output, const int64_t im2col_step) {
  const Geometry g = validate(value, spatial_shapes, sampling_loc, attn_weight, im2col_step);
  TORCH_CHECK(grad_output.is_cuda(), "grad_output must be a CUDA tensor");
  TORCH_CHECK(grad_output.scalar_type() == value.scalar_type(), "grad_output dtype mismatch");
  TORCH_CHECK(grad_output.numel() == int64_t(g.N) * g.Lq * g.M * g.D, "grad_output must be [N, Lq, M*D]");
  const c10::cuda::CUDAGuard guard(value.device());
  const at::Tensor shapes = spatial_shapes.contiguous();
  const at::Tensor loc = sampling_loc.contiguous();
  const at::Tensor attn = attn_weight.contiguous();
  const at::Tensor gout = grad_output.contiguous();
  at::Tensor grad_value = at::empty_like(value);  // zero-filled inside the C-ABI call
  at::Tensor grad_loc = at::empty_like(loc);
  at::Tensor grad_attn = at::empty_like(attn);
  void* stream = c10::cuda::getCurrentCUDAStream().stream();
  int rc;
  if (value.scalar_type() == at::kFloat) {
    rc = msda_b200_backward_f32(value.data_ptr<float>(), shapes.data_ptr<int64_t>(), loc.data_ptr<float>(),
                                attn.data_ptr<float>(), gout.data_ptr<float>(), grad_value.data_ptr<float>(),
                                grad_loc.data_ptr<float>(), grad_attn.data_ptr<float>(), g.N, g.S, g.M, g.D,
                                g.L, g.Lq, g.P, stream);
  } else {
    rc = msda_b200_backward_f64(value.data_ptr<double>(), shapes.data_ptr<int64_t>(),
                                loc.data_ptr<double>(), attn.data_ptr<double>(), gout.data_ptr<double>(),
                                grad_value.data_ptr<double>(), grad_loc.data_ptr<double>(),
                                grad_attn.data_ptr<double>(), g.N, g.S, g.M, g.D, g.L, g.Lq, g.P, stream);
  }
  raise_on_error(rc, "ms_deform_attn_backward");
  return {grad_value, grad_loc, grad_attn};
}

// Backward of the encoder self-attention: tiled kernel when the geometry allows, the general kernel otherwise
// (strict: raise instead).  `hw` is the host copy of spatial_shapes ([H0, W0, H1, W1, ...]).
static std::vector<at::Tensor> backward_enc_impl(const at::Tensor& value, const at::Tensor& spatial_shapes,
                                                 const at::Tensor& sampling_loc, const at::Tensor& attn_weight,
                                                 const at::Tensor& grad_output, const std::vector<int64_t>& hw,
                                                 const int64_t im2col_step, bool strict) {
  const Geometry g = validate(value, spatial_shapes, sampling_loc, attn_weight, im2col_step);
  TORCH_CHECK(grad_output.is_cuda() && grad_output.scalar_type() == value.scalar_type() &&
              grad_output.numel() == int64_t(g.N) * g.Lq * g.M * g.D, "grad_output must be a CUDA tensor [N, Lq, M*D]");
  if (value.scalar_type() == at::kFloat && int64_t(hw.size()) == 2 * int64_t(g.L) && msda_b200_variant_allows_tiles()) {
    const c10::cuda::CUDAGuard guard(value.device());
    const at::Tensor loc = sampling_loc.contiguous(), attn = attn_weight.contiguous(), gout = grad_output.contiguous();
    at::Tensor grad_value = at::empty_like(value), grad_loc = at::empty_like(loc), grad_attn = at::empty_like(attn);
    const at::Tensor shapes = spatial_shapes.contiguous();
    const int rc = msda_b200_backward_enc_tiled_f32(
        value.data_ptr<float>(), hw.data(), shapes.data_ptr<int64_t>(), loc.data_ptr<float>(), attn.data_ptr<float>(),
        gout.data_ptr<float>(),
        grad_value.data_ptr<float>(), grad_loc.data_ptr<float>(), grad_attn.data_ptr<float>(), g.N, g.S, g.M, g.D, g.L, g.Lq,
        g.P, c10::cuda::getCurrentCUDAStream().stream());
    if (rc == 0) return {grad_value, grad_loc, grad_attn};
    if (rc != MSDA_E_UNSUPPORTED) raise_on_error(rc, "ms_deform_attn_backward_enc");
  }
  TORCH_CHECK(!strict, "ms_deform_attn_backward_enc: outside the tiled kernel's domain (fp32, D = 32, P = 4, L <= 4, Lq == S)");
  return ms_deform_attn_backward(value, spatial_shapes, sampling_loc, attn_weight, grad_output, im2col_step);
}
std::vector<at::Tensor> ms_deform_attn_backward_enc(const at::Tensor& value, const at::Tensor& spatial_shapes,
                                                    const at::Tensor& sampling_loc, const at::Tensor& attn_weight,
                                                    const at::Tensor& grad_output, const std::vector<int64_t>& hw,
                                                    const int64_t im2col_step) {
  return backward_enc_impl(value, spatial_shapes, sampling_loc, attn_weight, grad_output, hw, im2col_step, false);
}
std::vector<at::Tensor> ms_deform_attn_backward_enc_strict(const at::Tensor& value, const at::Tensor& spatial_shapes,
                                                           const at::Tensor& sampling_loc, const at::Tensor& attn_weight,
                                                           const at::Tensor& grad_output, const std::vector<int64_t>& hw,
                                                           const int64_t im2col_step) {
  return backward_enc_impl(value, spatial_shapes, sampling_loc, attn_weight, grad_output, hw, im2col_step, true);
}

// fused-prologue variant: proj [N, Lq, 3*M*L*P] (raw [offsets | logits]), ref [N, Lq, L, 2]
at::Tensor ms_deform_attn_forward_fused(const at::Tensor& value, const at::Tensor& spatial_shapes, const at::Tensor& proj,
                                        const at::Tensor& ref, int64_t n_points) {
  TORCH_CHECK(value.is_cuda() && proj.is_cuda() && ref.is_cuda() && spatial_shapes.is_cuda(), "Not implemented on the CPU");
  TORCH_CHECK(value.scalar_type() == at::kFloat && proj.scalar_type() == at::kFloat && ref.scalar_type() == at::kFloat &&
              spatial_shapes.scalar_type() == at::kLong && value.dim() == 4 && proj.dim() == 3 && ref.dim() == 4 &&
              ref.size(3) == 2, "ms_deform_attn_forward_fused: dtypes / ranks");
  const at::Tensor v = value.contiguous(), pr = proj.contiguous(), rf = ref.contiguous(), sh = spatial_shapes.contiguous();
  const int64_t N = v.size(0), S = v.size(1), M = v.size(2), D = v.size(3), L = sh.size(0), Lq = pr.size(1), P = n_points;
  TORCH_CHECK(pr.size(0) == N && pr.size(2) == 3 * M * L * P && rf.size(0) == N && rf.size(1) == Lq && rf.size(2) == L,
              "ms_deform_attn_forward_fused: shapes");
  const c10::cuda::CUDAGuard guard(value.device());
  at::Tensor out = at::empty({N, Lq, M * D}, v.options());
  const int rc = msda_b200_forward_fused_f32(v.data_ptr<float>(), sh.data_ptr<int64_t>(), pr.data_ptr<float>(), rf.data_ptr<float>(),
                                             out.data_ptr<float>(), int(N), int(S), int(M), int(D), int(L), int(Lq), int(P),
                                             c10::cuda::getCurrentCUDAStream().stream());
  raise_on_error(rc, "ms_deform_attn_forward_fused");
  return out;
}

std::vector<at::Tensor> ms_deform_attn_backward_fused(const at::Tensor& value, const at::Tensor& spatial_shapes,
                                                      const at::Tensor& proj, const at::Tensor& ref, const at::Tensor& grad_output,
                                                      int64_t n_points) {
  const at::Tensor v = value.contiguous(), pr = proj.contiguous(), rf = ref.contiguous(), sh = spatial_shapes.contiguous();
  const at::Tensor go = grad_output.contiguous();
  const int64_t N = v.size(0), S = v.size(1), M = v.size(2), D = v.size(3), L = sh.size(0), Lq = pr.size(1), P = n_points;
  const c10::cuda::CUDAGuard guard(value.device());
  at::Tensor gv = at::empty_like(v), gp = at::empty_like(pr);
  const int rc = msda_b200_backward_fused_f32(v.data_ptr<float>(), sh.data_ptr<int64_t>(), pr.data_ptr<float>(), rf.data_ptr<float>(),
                                              go.data_ptr<float>(), gv.data_ptr<float>(), gp.data_ptr<float>(), int(N), int(S),
                                              int(M), int(D), int(L), int(Lq), int(P), c10::cuda::getCurrentCUDAStream().stream());
  raise_on_error(rc, "ms_deform_attn_backward_fused");
  return {gv, gp};
}

// Encoder tile kernels with the fused prologue: proj [N, Lq, 3*M*16], ref [N, Lq, 4, 2], hw = host level sizes.
// Raise (no fallback: the caller chose this path) outside the domain.
at::Tensor ms_deform_attn_forward_enc_fused(const at::Tensor& value, const at::Tensor& proj, const at::Tensor& ref,
                                            const std::vector<int64_t>& hw) {
  TORCH_CHECK(value.is_cuda() && proj.is_cuda() && ref.is_cuda(), "Not implemented on the CPU");
  TORCH_CHECK(value.scalar_type() == at::kFloat && proj.scalar_type() == at::kFloat && ref.scalar_type() == at::kFloat &&
              value.dim() == 4 && proj.dim() == 3 && ref.dim() == 4 && ref.size(3) == 2 && hw.size() == 8,
              "ms_deform_attn_forward_enc_fused: dtypes / ranks (four levels)");
  const at::Tensor v = value.contiguous(), pr = proj.contiguous(), rf = ref.contiguous();
  const int64_t N = v.size(0), S = v.size(1), M = v.size(2), D = v.size(3), L = 4, Lq = pr.size(1), P = 4;
  TORCH_CHECK(pr.size(0) == N && pr.size(2) == 3 * M * L * P && rf.size(0) == N && rf.size(1) == Lq && rf.size(2) == L,
              "ms_deform_attn_forward_enc_fused: shapes");
  const c10::cuda::CUDAGuard guard(value.device());
  at::Tensor out = at::empty({N, Lq, M * D}, v.options());
  const int rc = msda_b200_forward_enc_tiled_fused_f32(v.data_ptr<float>(), hw.data(), pr.data_ptr<float>(), rf.data_ptr<float>(),
                                                       out.data_ptr<float>(), int(N), int(S), int(M), int(D), int(L), int(Lq),
                                                       int(P), c10::cuda::getCurrentCUDAStream().stream());
  raise_on_error(rc, "ms_deform_attn_forward_enc_fused");
  return out;
}

std::vector<at::Tensor> ms_deform_attn_backward_enc_fused(const at::Tensor& value, const at::Tensor& proj, const at::Tensor& ref,
                                                          const at::Tensor& grad_output, const std::vector<int64_t>& hw) {
  const at::Tensor v = value.contiguous(), pr = proj.contiguous(), rf = ref.contiguous(), go = grad_output.contiguous();
  const int64_t N = v.size(0), S = v.size(1), M = v.size(2), D = v.size(3), L = 4, Lq = pr.size(1), P = 4;
  TORCH_CHECK(hw.size() == 8 && go.numel() == N * Lq * M * D, "ms_deform_attn_backward_enc_fused: shapes");
  const c10::cuda::CUDAGuard guard(value.device());
  at::Tensor gv = at::empty_like(v), gp = at::empty_like(pr);
  const int rc = msda_b200_backward_enc_tiled_fused_f32(v.data_ptr<float>(), hw.data(), pr.data_ptr<float>(), rf.data_ptr<float>(),
                                                        go.data_ptr<float>(), gv.data_ptr<float>(), gp.data_ptr<float>(), int(N),
                                                        int(S), int(M), int(D), int(L), int(Lq), int(P),
                                                        c10::cuda::getCurrentCUDAStream().stream());
  raise_on_error(rc, "ms_deform_attn_backward_enc_fused");
  return {gv, gp};
}

static at::Tensor forward_enc_impl(const at::Tensor& value, const at::Tensor& spatial_shapes,
                                   const at::Tensor& sampling_loc, const at::Tensor& attn_weight,
                                   const std::vector<int64_t>& hw, const int64_t im2col_step, bool strict);

at::Tensor ms_deform_attn_forward_enc(const at::Tensor& value, const at::Tensor& spatial_shapes,
                                      const at::Tensor& sampling_loc, const at::Tensor& attn_weight,
                                      const std::vector<int64_t>& hw, const int64_t im2col_step) {
  return forward_enc_impl(value, spatial_shapes, sampling_loc, attn_weight, hw, im2col_step, false);
}

// the same, but raises instead of falling back to the general kernel (tests: proves which kernel produced the numbers)
at::Tensor ms_deform_attn_forward_enc_strict(const at::Tensor& value, const at::Tensor& spatial_shapes,
                                             const at::Tensor& sampling_loc, const at::Tensor& attn_weight,
                                             const std::vector<int64_t>& hw, const int64_t im2col_step) {
  return forward_enc_impl(value, spatial_shapes, sampling_loc, attn_weight, hw, im2col_step, true);
}

static at::Tensor forward_enc_impl(const at::Tensor& value, const at::Tensor& spatial_shapes,
                                   const at::Tensor& sampling_loc, const at::Tensor& attn_weight,
                                   const std::vector<int64_t>& hw, const int64_t im2col_step, bool strict) {
  const Geometry g = validate(value, spatial_shapes, sampling_loc, attn_weight, im2col_step);
  if (value.scalar_type() == at::kFloat && int64_t(hw.size()) == 2 * int64_t(g.L) && msda_b200_variant_allows_tiles()) {
    const c10::cuda::CUDAGuard guard(value.device());
    const at::Tensor loc = sampling_loc.contiguous();
    const at::Tensor attn = attn_weight.contiguous();
    at::Tensor out = at::empty({g.N, g.Lq, int64_t(g.M) * g.D}, value.options());
    const int rc = msda_b200_forward_enc_tiled_f32(value.data_ptr<float>(), hw.data(), loc.data_ptr<float>(),
                                                   attn.data_ptr<float>(), out.data_ptr<float>(), g.N, g.S, g.M, g.D,
                                                   g.L, g.Lq, g.P, c10::cuda::getCurrentCUDAStream().stream());
    if (rc == 0) return out;
    if (rc != MSDA_E_UNSUPPORTED) raise_on_error(rc, "ms_deform_attn_forward_enc");
  }
  TORCH_CHECK(!strict, "ms_deform_attn_forward_enc: outside the tiled kernel's domain (fp32, D = 32, P = 4, L <= 4, Lq == S)");
  return ms_deform_attn_forward(value, spatial_shapes, sampling_loc, attn_weight, im2col_step);
}

// ---- fused residual + dropout + LayerNorm (include/tfb200_fused.h) -------------------------------------------
// forward: returns {y, s, mean, rstd}; keep_mask is an optional bool/uint8 tensor of x's shape
std::vector<at::Tensor> add_dropout_layernorm_forward(const at::Tensor& x, const at::Tensor& branch,
                                                      const c10::optional<at::Tensor>& keep_mask,
                                                      const at::Tensor& gamma, const at::Tensor& beta,
                                                      double keep_prob, double eps) {
  TORCH_CHECK(x.is_cuda() && branch.is_cuda(), "add_dropout_layernorm: CUDA tensors required (no CPU path)");
  TORCH_CHECK(x.scalar_type() == at::kFloat && branch.scalar_type() == at::kFloat, "fp32 only");
  TORCH_CHECK(x.sizes() == branch.sizes(), "x and branch must have the same shape");
  const int64_t C = x.size(-1);
  const at::Tensor xc = x.contiguous(), bc = branch.contiguous(), g = gamma.contiguous(), b = beta.contiguous();
  const int64_t rows = xc.numel() / C;
  const c10::cuda::CUDAGuard guard(x.device());
  at::Tensor y = at::empty_like(xc), s = at::empty_like(xc);
  at::Tensor mean = at::empty({rows}, xc.options()), rstd = at::empty({rows}, xc.options());
  const uint8_t* mptr = nullptr;
  at::Tensor mk;
  if (keep_mask.has_value() && keep_mask->defined()) {
    mk = keep_mask->contiguous();
    TORCH_CHECK(mk.numel() == xc.numel() && mk.element_size() == 1, "keep_mask must be a bool/uint8 tensor shaped like x");
    mptr = static_cast<const uint8_t*>(mk.data_ptr());
  }
  const int rc = tfb200_add_dropout_layernorm_fwd_f32(
      xc.data_ptr<float>(), bc.data_ptr<float>(), mptr, g.data_ptr<float>(), b.data_ptr<float>(), s.data_ptr<float>(),
      y.data_ptr<float>(), mean.data_ptr<float>(), rstd.data_ptr<float>(), rows, int(C), float(keep_prob), float(eps),
      c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "add_dropout_layernorm_forward failed (code ", rc, "): C must be a multiple of 4 and <= 512");
  return {y, s, mean, rstd};
}

// backward: returns {dx, dbranch, dgamma, dbeta}
std::vector<at::Tensor> add_dropout_layernorm_backward(const at::Tensor& dy, const at::Tensor& s,
                                                       const c10::optional<at::Tensor>& keep_mask,
                                                       const at::Tensor& gamma, const at::Tensor& mean,
                                                       const at::Tensor& rstd, double keep_prob) {
  TORCH_CHECK(dy.is_cuda() && s.is_cuda(), "add_dropout_layernorm: CUDA tensors required (no CPU path)");
  const int64_t C = s.size(-1);
  const at::Tensor dyc = dy.contiguous(), g = gamma.contiguous();
  const int64_t rows = s.numel() / C;
  const c10::cuda::CUDAGuard guard(s.device());
  at::Tensor dx = at::empty_like(s), db = at::empty_like(s);
  at::Tensor dgamma = at::empty({C}, s.options()), dbeta = at::empty({C}, s.options());
  at::Tensor ws = at::empty({tfb200_ln_partial_ctas(rows), 2, C}, s.options());
  const uint8_t* mptr = nullptr;
  at::Tensor mk;
  if (keep_mask.has_value() && keep_mask->defined()) {
    mk = keep_mask->contiguous();
    mptr = static_cast<const uint8_t*>(mk.data_ptr());
  }
  const int rc = tfb200_add_dropout_layernorm_bwd_f32(
      dyc.data_ptr<float>(), s.data_ptr<float>(), mptr, g.data_ptr<float>(), mean.data_ptr<float>(),
      rstd.data_ptr<float>(), dx.data_ptr<float>(), db.data_ptr<float>(), dgamma.data_ptr<float>(),
      dbeta.data_ptr<float>(), ws.data_ptr<float>(), rows, int(C), float(keep_prob),
      c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "add_dropout_layernorm_backward failed (code ", rc, ")");
  return {dx, db, dgamma, dbeta};
}

at::Tensor colsum(const at::Tensor& x) {
  TORCH_CHECK(x.is_cuda() && x.scalar_type() == at::kFloat && x.dim() >= 2, "colsum: fp32 CUDA matrix required");
  const at::Tensor xc = x.contiguous();
  const int64_t C = xc.size(-1), rows = xc.numel() / C;
  const c10::cuda::CUDAGuard guard(x.device());
  at::Tensor out = at::empty({C}, xc.options());
  at::Tensor ws = at::empty({tfb200_ln_partial_ctas(rows), C}, xc.options());
  const int rc = tfb200_colsum_f32(xc.data_ptr<float>(), out.data_ptr<float>(), ws.data_ptr<float>(), rows, int(C),
                                   c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "colsum failed (code ", rc, "): C must be a multiple of 4 and <= 1024");
  return out;
}

// y = act(x . w^T + bias) on the hand-written wgmma TF32 kernel (csrc/tf32_gemm.cu); x [..., K], w [N, K], bias [N] or None
bool tf32_linear_supported(int64_t rows, int64_t n, int64_t k) { return tfb200_tf32_linear_supported(rows, int(n), int(k)) != 0; }

at::Tensor tf32_linear(const at::Tensor& x, const at::Tensor& w, const c10::optional<at::Tensor>& bias, bool relu) {
  TORCH_CHECK(x.is_cuda() && w.is_cuda() && x.scalar_type() == at::kFloat && w.scalar_type() == at::kFloat && w.dim() == 2,
              "tf32_linear: fp32 CUDA tensors required");
  const int64_t K = w.size(1), N = w.size(0);
  TORCH_CHECK(x.dim() >= 1 && x.size(-1) == K, "tf32_linear: x[..., K] against w[N, K]");
  const at::Tensor xc = x.contiguous(), wc = w.contiguous();
  const int64_t M = xc.numel() / K;
  const float* bp = nullptr;
  at::Tensor bc;
  if (bias.has_value() && bias->defined()) {
    TORCH_CHECK(bias->is_cuda() && bias->scalar_type() == at::kFloat && bias->numel() == N, "tf32_linear: bias[N]");
    bc = bias->contiguous();
    bp = bc.data_ptr<float>();
  }
  const c10::cuda::CUDAGuard guard(x.device());
  auto sizes = xc.sizes().vec();
  sizes.back() = N;
  at::Tensor y = at::empty(sizes, xc.options());
  if (M == 0) return y;
  const int rc = tfb200_tf32_linear_f32(xc.data_ptr<float>(), wc.data_ptr<float>(), bp, y.data_ptr<float>(), M, int(N),
                                        int(K), relu ? 1 : 0, c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "tf32_linear failed (code ", rc, "): needs N % 128 == 0, K % 32 == 0, 16-byte aligned operands");
  return y;
}

// dx = dy . w  and  dw = dy^T . x  of the same layer (csrc/tf32_gemm.cu, modes dgrad / wgrad)
at::Tensor tf32_linear_dgrad(const at::Tensor& dy, const at::Tensor& w) {
  TORCH_CHECK(dy.is_cuda() && w.is_cuda() && dy.scalar_type() == at::kFloat && w.scalar_type() == at::kFloat && w.dim() == 2 &&
              dy.size(-1) == w.size(0), "tf32_linear_dgrad: dy[..., N] against w[N, K]");
  const at::Tensor g = dy.contiguous(), wc = w.contiguous();
  const int64_t N = wc.size(0), K = wc.size(1), M = g.numel() / N;
  const c10::cuda::CUDAGuard guard(dy.device());
  auto sizes = g.sizes().vec();
  sizes.back() = K;
  at::Tensor dx = at::empty(sizes, g.options());
  if (M == 0) return dx;
  const int rc = tfb200_tf32_linear_dgrad_f32(g.data_ptr<float>(), wc.data_ptr<float>(), dx.data_ptr<float>(), M, int(N),
                                              int(K), c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "tf32_linear_dgrad failed (code ", rc, ")");
  return dx;
}

at::Tensor tf32_linear_wgrad(const at::Tensor& dy, const at::Tensor& x) {
  TORCH_CHECK(dy.is_cuda() && x.is_cuda() && dy.scalar_type() == at::kFloat && x.scalar_type() == at::kFloat,
              "tf32_linear_wgrad: fp32 CUDA tensors required");
  const at::Tensor g = dy.contiguous(), xc = x.contiguous();
  const int64_t N = g.size(-1), K = xc.size(-1), M = g.numel() / N;
  TORCH_CHECK(xc.numel() / K == M, "tf32_linear_wgrad: dy[M, N] and x[M, K] must agree on M");
  const c10::cuda::CUDAGuard guard(dy.device());
  at::Tensor dw = at::empty({N, K}, g.options());
  const int rc = tfb200_tf32_linear_wgrad_f32(g.data_ptr<float>(), xc.data_ptr<float>(), dw.data_ptr<float>(), M, int(N),
                                              int(K), c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "tf32_linear_wgrad failed (code ", rc, ")");
  return dw;
}

// Dense self-attention of the decoder queries (csrc/small_attn.cu): q, k, v are [L, B, H, 32] views (channel stride 1,
// head stride 32); key_pad [B, L] bool or None; seed None = no dropout.  Returns {out [L, B, H, 32], lse [B, H, L]}.
static void check_view(const at::Tensor& t, const char* name) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat && t.dim() == 4 && t.size(3) == 32 && t.stride(3) == 1 &&
                  t.stride(2) == 32 && (reinterpret_cast<uintptr_t>(t.data_ptr()) & 15u) == 0 && t.stride(0) % 4 == 0 &&
                  t.stride(1) % 4 == 0,
              "small_attention: ", name, " must be an fp32 CUDA [L, B, H, 32] view with 16-byte aligned rows");
}
std::vector<at::Tensor> small_attention_forward(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v,
                                                const c10::optional<at::Tensor>& key_pad,
                                                const c10::optional<at::Tensor>& seed, double scale, double keep_prob) {
  check_view(q, "q"); check_view(k, "k"); check_view(v, "v");
  const int64_t L = q.size(0), B = q.size(1), H = q.size(2);
  TORCH_CHECK(k.sizes() == q.sizes() && v.sizes() == q.sizes(), "small_attention: q, k, v must have the same shape");
  const c10::cuda::CUDAGuard guard(q.device());
  at::Tensor out = at::empty({L, B, H, 32}, q.options());
  at::Tensor lse = at::empty({B, H, L}, q.options());
  const uint8_t* kp = nullptr;
  at::Tensor kpc;
  if (key_pad.has_value() && key_pad->defined()) {
    kpc = key_pad->contiguous();
    TORCH_CHECK(kpc.numel() == B * L && kpc.element_size() == 1, "small_attention: key_pad must be a bool [B, L] tensor");
    kp = static_cast<const uint8_t*>(kpc.data_ptr());
  }
  const int64_t* sp = (seed.has_value() && seed->defined()) ? seed->data_ptr<int64_t>() : nullptr;
  const int64_t st[8] = {q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1), out.stride(0), out.stride(1)};
  const int rc = tfb200_small_attn_fwd_f32(q.data_ptr<float>(), k.data_ptr<float>(), v.data_ptr<float>(), kp, sp,
                                           out.data_ptr<float>(), lse.data_ptr<float>(), int(B), int(H), int(L), st,
                                           float(scale), float(keep_prob), c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "small_attention_forward failed (code ", rc, ")");
  return {out, lse};
}

std::vector<at::Tensor> small_attention_backward(const at::Tensor& q, const at::Tensor& k, const at::Tensor& v,
                                                 const c10::optional<at::Tensor>& key_pad,
                                                 const c10::optional<at::Tensor>& seed, const at::Tensor& out,
                                                 const at::Tensor& lse, const at::Tensor& grad_out, double scale,
                                                 double keep_prob) {
  check_view(q, "q"); check_view(k, "k"); check_view(v, "v"); check_view(out, "out");
  const at::Tensor go = grad_out.contiguous();
  check_view(go, "grad_out");
  const int64_t L = q.size(0), B = q.size(1), H = q.size(2);
  const c10::cuda::CUDAGuard guard(q.device());
  at::Tensor dq = at::empty({L, B, H, 32}, q.options()), dk = at::empty({L, B, H, 32}, q.options()),
             dv = at::empty({L, B, H, 32}, q.options());
  at::Tensor delta = at::empty({B, H, L}, q.options());
  const uint8_t* kp = nullptr;
  at::Tensor kpc;
  if (key_pad.has_value() && key_pad->defined()) {
    kpc = key_pad->contiguous();
    kp = static_cast<const uint8_t*>(kpc.data_ptr());
  }
  const int64_t* sp = (seed.has_value() && seed->defined()) ? seed->data_ptr<int64_t>() : nullptr;
  const int64_t st[16] = {q.stride(0), q.stride(1), k.stride(0), k.stride(1), v.stride(0), v.stride(1), out.stride(0),
                          out.stride(1), go.stride(0), go.stride(1), dq.stride(0), dq.stride(1), dk.stride(0), dk.stride(1),
                          dv.stride(0), dv.stride(1)};
  const int rc = tfb200_small_attn_bwd_f32(q.data_ptr<float>(), k.data_ptr<float>(), v.data_ptr<float>(), kp, sp,
                                           out.data_ptr<float>(), lse.data_ptr<float>(), go.data_ptr<float>(),
                                           dq.data_ptr<float>(), dk.data_ptr<float>(), dv.data_ptr<float>(),
                                           delta.data_ptr<float>(), int(B), int(H), int(L), st, float(scale),
                                           float(keep_prob), c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "small_attention_backward failed (code ", rc, ")");
  return {dq, dk, dv};
}

// boxes = sigmoid(delta + inverse_sigmoid(ref)) (csrc/box_refine.cu); delta [..., 4], ref [..., 2 or 4]
at::Tensor refine_boxes_forward(const at::Tensor& delta, const at::Tensor& ref, double eps) {
  TORCH_CHECK(delta.is_cuda() && ref.is_cuda() && delta.scalar_type() == at::kFloat && ref.scalar_type() == at::kFloat &&
              delta.size(-1) == 4 && (ref.size(-1) == 2 || ref.size(-1) == 4) &&
              delta.numel() / 4 == ref.numel() / ref.size(-1), "refine_boxes: delta [..., 4], ref [..., 2|4]");
  const at::Tensor d = delta.contiguous(), r = ref.contiguous();
  const c10::cuda::CUDAGuard guard(delta.device());
  at::Tensor out = at::empty_like(d);
  const int rc = tfb200_refine_boxes_fwd_f32(d.data_ptr<float>(), r.data_ptr<float>(), out.data_ptr<float>(), d.numel() / 4,
                                             int(r.size(-1)), float(eps), c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "refine_boxes_forward failed (code ", rc, ")");
  return out;
}

std::vector<at::Tensor> refine_boxes_backward(const at::Tensor& grad_out, const at::Tensor& out, const at::Tensor& ref,
                                              bool need_ref_grad, double eps) {
  const at::Tensor g = grad_out.contiguous(), o = out.contiguous(), r = ref.contiguous();
  const c10::cuda::CUDAGuard guard(out.device());
  at::Tensor gd = at::empty_like(o);
  at::Tensor gr = need_ref_grad ? at::empty_like(r) : at::Tensor();
  const int rc = tfb200_refine_boxes_bwd_f32(g.data_ptr<float>(), o.data_ptr<float>(), r.data_ptr<float>(),
                                             gd.data_ptr<float>(), need_ref_grad ? gr.data_ptr<float>() : nullptr,
                                             o.numel() / 4, int(r.size(-1)), float(eps),
                                             c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "refine_boxes_backward failed (code ", rc, ")");
  return {gd, gr};
}

at::Tensor relu_dropout_forward(const at::Tensor& a, const c10::optional<at::Tensor>& seed, double keep_prob, bool training) {
  TORCH_CHECK(a.is_cuda() && a.scalar_type() == at::kFloat, "relu_dropout: fp32 CUDA tensor required");
  const at::Tensor ac = a.contiguous();
  const c10::cuda::CUDAGuard guard(a.device());
  at::Tensor h = at::empty_like(ac);
  const int64_t* sp = nullptr;
  if (training) {
    TORCH_CHECK(seed.has_value() && seed->is_cuda() && seed->scalar_type() == at::kLong && seed->numel() >= 1,
                "relu_dropout: training mode needs an int64 CUDA seed tensor");
    sp = seed->data_ptr<int64_t>();
  }
  const int rc = tfb200_relu_dropout_fwd_f32(ac.data_ptr<float>(), h.data_ptr<float>(), sp, ac.numel(), float(keep_prob),
                                             training ? 1 : 0, c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "relu_dropout_forward failed (code ", rc, ")");
  return h;
}

at::Tensor relu_dropout_backward(const at::Tensor& grad_h, const at::Tensor& h, double keep_prob, bool training) {
  const at::Tensor g = grad_h.contiguous();
  const c10::cuda::CUDAGuard guard(h.device());
  at::Tensor ga = at::empty_like(h);
  const int rc = tfb200_relu_dropout_bwd_f32(g.data_ptr<float>(), h.data_ptr<float>(), ga.data_ptr<float>(), h.numel(),
                                             float(keep_prob), training ? 1 : 0, c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "relu_dropout_backward failed (code ", rc, ")");
  return ga;
}

// proj [N,Lq,3*M*L*P], ref [N,Lq,L,2|4], shapes_f32 [L,2] -> {loc [N,Lq,M,L,P,2], attn [N,Lq,M,L,P]}
std::vector<at::Tensor> sampling_prep_forward(const at::Tensor& proj, const at::Tensor& ref, const at::Tensor& shapes_f32,
                                              int64_t M, int64_t L, int64_t P) {
  TORCH_CHECK(proj.is_cuda() && proj.scalar_type() == at::kFloat && proj.dim() == 3, "sampling_prep: proj must be [N,Lq,3*M*L*P] fp32 CUDA");
  const at::Tensor p = proj.contiguous(), r = ref.contiguous(), sh = shapes_f32.contiguous();
  const int64_t N = p.size(0), Lq = p.size(1);
  TORCH_CHECK(p.size(2) == 3 * M * L * P && r.size(0) == N && r.size(1) == Lq && r.size(2) == L, "sampling_prep: shape mismatch");
  const c10::cuda::CUDAGuard guard(proj.device());
  at::Tensor loc = at::empty({N, Lq, M, L, P, 2}, p.options()), attn = at::empty({N, Lq, M, L, P}, p.options());
  const int rc = tfb200_sampling_prep_fwd_f32(p.data_ptr<float>(), r.data_ptr<float>(), sh.data_ptr<float>(),
                                              loc.data_ptr<float>(), attn.data_ptr<float>(), N * Lq, int(M), int(L), int(P),
                                              int(r.size(3)), c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "sampling_prep_forward failed (code ", rc, ")");
  return {loc, attn};
}

at::Tensor sampling_prep_backward(const at::Tensor& grad_loc, const at::Tensor& grad_attn, const at::Tensor& attn,
                                  const at::Tensor& ref, const at::Tensor& shapes_f32, int64_t M, int64_t L, int64_t P) {
  const at::Tensor gl = grad_loc.contiguous(), ga = grad_attn.contiguous(), r = ref.contiguous(), sh = shapes_f32.contiguous();
  const int64_t N = attn.size(0), Lq = attn.size(1);
  const c10::cuda::CUDAGuard guard(attn.device());
  at::Tensor gp = at::empty({N, Lq, 3 * M * L * P}, attn.options());
  const int rc = tfb200_sampling_prep_bwd_f32(gl.data_ptr<float>(), ga.data_ptr<float>(), attn.data_ptr<float>(),
                                              r.data_ptr<float>(), sh.data_ptr<float>(), gp.data_ptr<float>(), N * Lq, int(M),
                                              int(L), int(P), int(r.size(3)), c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "sampling_prep_backward failed (code ", rc, ")");
  return gp;
}

// cost [K,B,Q,T] fp32, offsets int32 [B+1] (device) -> {src [K,T] int64, tgt [K,T] int64, status int32 [1]}
std::vector<at::Tensor> lsa(const at::Tensor& cost, const at::Tensor& offsets, int64_t max_targets) {
  TORCH_CHECK(cost.is_cuda() && cost.scalar_type() == at::kFloat && cost.dim() == 4, "lsa: cost must be a [K,B,Q,T] fp32 CUDA tensor");
  TORCH_CHECK(offsets.is_cuda() && offsets.scalar_type() == at::kInt && offsets.numel() == cost.size(1) + 1,
              "lsa: offsets must be an int32 CUDA tensor of B+1 entries");
  const at::Tensor c = cost.contiguous();
  const c10::cuda::CUDAGuard guard(cost.device());
  const int64_t K = c.size(0), B = c.size(1), Q = c.size(2), T = c.size(3);
  auto iopt = c.options().dtype(at::kLong);
  at::Tensor src = at::zeros({K, T}, iopt), tgt = at::zeros({K, T}, iopt);
  at::Tensor status = at::zeros({1}, c.options().dtype(at::kInt));
  const int rc = tfb200_lsa_f32(c.data_ptr<float>(), offsets.data_ptr<int>(), src.data_ptr<int64_t>(), tgt.data_ptr<int64_t>(),
                                int(K), int(B), int(Q), int(T), int(max_targets), status.data_ptr<int>(),
                                c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "lsa failed (code ", rc, ")");
  return {src, tgt, status};
}

// ---- SetCriterion / matcher on the device (csrc/set_loss.cu) ------------------------------------------------------------
at::Tensor match_cost(const at::Tensor& logits, const at::Tensor& boxes, const at::Tensor& tgt_ids, const at::Tensor& tgt_boxes,
                      double w_class, double w_bbox, double w_giou, double alpha, double gamma) {
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == at::kFloat && boxes.scalar_type() == at::kFloat &&
              tgt_ids.scalar_type() == at::kLong && tgt_boxes.scalar_type() == at::kFloat, "match_cost: dtypes");
  const at::Tensor lg = logits.contiguous(), bx = boxes.contiguous(), ti = tgt_ids.contiguous(), tb = tgt_boxes.contiguous();
  const int64_t C = lg.size(-1), R = lg.numel() / C, T = ti.numel();
  TORCH_CHECK(bx.numel() == R * 4 && tb.numel() == T * 4 && T > 0, "match_cost: shapes");
  const c10::cuda::CUDAGuard guard(logits.device());
  at::Tensor cost = at::empty({R, T}, lg.options());
  const int rc = tfb200_match_cost_f32(lg.data_ptr<float>(), bx.data_ptr<float>(), ti.data_ptr<int64_t>(), tb.data_ptr<float>(),
                                       cost.data_ptr<float>(), R, int(C), int(T), float(w_class), float(w_bbox), float(w_giou),
                                       float(alpha), float(gamma), c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "match_cost failed (code ", rc, ")");
  return cost;
}

// returns {out5k [5][K], unit_logits [K,B,Q,C], unit_l1 [K,B,Q,4], unit_giou [K,B,Q,4]}
std::vector<at::Tensor> set_loss_forward(const at::Tensor& logits, const at::Tensor& boxes, const at::Tensor& src,
                                         const at::Tensor& tgt, const at::Tensor& tgt_ids, const at::Tensor& tgt_boxes,
                                         const at::Tensor& offsets, const at::Tensor& n_gt, const at::Tensor& num_boxes,
                                         double alpha, double gamma) {
  TORCH_CHECK(logits.is_cuda() && logits.dim() == 4 && boxes.dim() == 4 && logits.scalar_type() == at::kFloat &&
              boxes.scalar_type() == at::kFloat && src.scalar_type() == at::kLong && tgt.scalar_type() == at::kLong &&
              tgt_ids.scalar_type() == at::kLong && tgt_boxes.scalar_type() == at::kFloat &&
              offsets.scalar_type() == at::kInt && n_gt.scalar_type() == at::kFloat && num_boxes.scalar_type() == at::kFloat &&
              num_boxes.is_cuda() && n_gt.is_cuda() && offsets.is_cuda(), "set_loss_forward: dtypes / devices");
  const at::Tensor lg = logits.contiguous(), bx = boxes.contiguous(), s = src.contiguous(), t = tgt.contiguous();
  const at::Tensor ti = tgt_ids.contiguous(), tb = tgt_boxes.contiguous();
  const int64_t K = lg.size(0), B = lg.size(1), Q = lg.size(2), C = lg.size(3), T = s.size(-1);
  TORCH_CHECK(s.numel() == K * T && t.numel() == K * T && ti.numel() == T && tb.numel() == 4 * T && offsets.numel() == B + 1 &&
              n_gt.numel() == B, "set_loss_forward: shapes");
  const c10::cuda::CUDAGuard guard(logits.device());
  at::Tensor out = at::empty({5, K}, lg.options());
  at::Tensor ul = at::empty_like(lg), u1 = at::empty_like(bx), ug = at::empty_like(bx);
  at::Tensor row_loss = at::empty({K * B * Q}, lg.options()), row_flags = at::empty({K * B * Q}, lg.options().dtype(at::kInt));
  at::Tensor pl = at::zeros({K, T}, lg.options()), pg = at::zeros({K, T}, lg.options());
  const int rc = tfb200_set_loss_fwd_f32(lg.data_ptr<float>(), bx.data_ptr<float>(), s.data_ptr<int64_t>(), t.data_ptr<int64_t>(),
                                         ti.data_ptr<int64_t>(), tb.data_ptr<float>(), offsets.data_ptr<int>(),
                                         n_gt.data_ptr<float>(), num_boxes.data_ptr<float>(), ul.data_ptr<float>(),
                                         u1.data_ptr<float>(), ug.data_ptr<float>(), row_loss.data_ptr<float>(),
                                         row_flags.data_ptr<int>(), pl.data_ptr<float>(), pg.data_ptr<float>(),
                                         out.data_ptr<float>(), int(K), int(B), int(Q), int(C), int(T), float(alpha),
                                         float(gamma), c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "set_loss_forward failed (code ", rc, ")");
  return {out, ul, u1, ug};
}

std::vector<at::Tensor> set_loss_backward(const at::Tensor& unit_logits, const at::Tensor& unit_l1, const at::Tensor& unit_giou,
                                          const at::Tensor& g_ce, const at::Tensor& g_l1, const at::Tensor& g_giou,
                                          const at::Tensor& num_boxes) {
  const int64_t K = unit_logits.size(0), B = unit_logits.size(1), Q = unit_logits.size(2), C = unit_logits.size(3);
  const at::Tensor a = g_ce.contiguous(), b = g_l1.contiguous(), c = g_giou.contiguous();
  TORCH_CHECK(a.numel() == K && b.numel() == K && c.numel() == K && a.scalar_type() == at::kFloat, "set_loss_backward: gradient vectors [K]");
  const c10::cuda::CUDAGuard guard(unit_logits.device());
  at::Tensor gl = at::empty_like(unit_logits), gb = at::empty_like(unit_l1);
  const int rc = tfb200_set_loss_bwd_f32(unit_logits.data_ptr<float>(), unit_l1.data_ptr<float>(), unit_giou.data_ptr<float>(),
                                         a.data_ptr<float>(), b.data_ptr<float>(), c.data_ptr<float>(),
                                         num_boxes.data_ptr<float>(), gl.data_ptr<float>(), gb.data_ptr<float>(), int(K), int(B),
                                         int(Q), int(C), c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "set_loss_backward failed (code ", rc, ")");
  return {gl, gb};
}

// ---- detection post-processing for the tracker (deformable_detr.py:286-334) ------------------------------------------
std::vector<at::Tensor> detect_postprocess(const at::Tensor& logits, const at::Tensor& boxes, const at::Tensor& sizes_hw) {
  TORCH_CHECK(logits.is_cuda() && logits.scalar_type() == at::kFloat && logits.dim() == 3, "detect_postprocess: logits must be [N,Q,C] fp32 CUDA");
  TORCH_CHECK(boxes.is_cuda() && boxes.scalar_type() == at::kFloat && boxes.dim() == 3 && boxes.size(2) == 4, "detect_postprocess: boxes must be [N,Q,4] fp32 CUDA");
  TORCH_CHECK(sizes_hw.is_cuda() && sizes_hw.scalar_type() == at::kLong && sizes_hw.dim() == 2 && sizes_hw.size(1) == 2, "detect_postprocess: sizes must be [N,2] int64 CUDA");
  const int64_t N = logits.size(0), Q = logits.size(1), C = logits.size(2);
  TORCH_CHECK(boxes.size(0) == N && boxes.size(1) == Q && sizes_hw.size(0) == N, "detect_postprocess: shape mismatch");
  c10::cuda::CUDAGuard guard(logits.device());
  auto lg = logits.contiguous(), bx = boxes.contiguous(), sz = sizes_hw.contiguous();
  auto packed = at::empty({N, Q, 6}, lg.options());
  auto labels = at::empty({N, Q}, lg.options().dtype(at::kLong));
  const int rc = tfb200_detect_postprocess_f32(lg.data_ptr<float>(), bx.data_ptr<float>(), sz.data_ptr<int64_t>(),
                                               packed.data_ptr<float>(), labels.data_ptr<int64_t>(), int(N), int(Q), int(C),
                                               at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "detect_postprocess failed (code ", rc, ")");
  return {packed, labels};
}

// ---- clip + AdamW over a flat parameter range (engine.py:147-151) ---------------------------------------------------
void flat_adamw(at::Tensor param, const at::Tensor& grad, at::Tensor exp_avg, at::Tensor exp_avg_sq, int64_t begin,
                int64_t end, const c10::optional<at::Tensor>& grad_norm, double max_norm, double lr, double beta1,
                double beta2, double eps, double weight_decay, int64_t step) {
  for (const at::Tensor* t : std::initializer_list<const at::Tensor*>{&param, &grad, &exp_avg, &exp_avg_sq})
    TORCH_CHECK(t->is_cuda() && t->scalar_type() == at::kFloat && t->dim() == 1 && t->is_contiguous() &&
                t->numel() == param.numel(), "flat_adamw: buffers must be flat contiguous fp32 CUDA tensors of one length");
  TORCH_CHECK(0 <= begin && begin <= end && end <= param.numel() && begin % 4 == 0, "flat_adamw: bad range");
  const float* norm = nullptr;
  if (grad_norm.has_value()) {
    TORCH_CHECK(grad_norm->is_cuda() && grad_norm->scalar_type() == at::kFloat && grad_norm->numel() == 1, "flat_adamw: grad_norm must be a CUDA fp32 scalar");
    norm = grad_norm->data_ptr<float>();
  }
  const c10::cuda::CUDAGuard guard(param.device());
  const int rc = tfb200_flat_adamw_f32(param.data_ptr<float>() + begin, grad.data_ptr<float>() + begin,
                                       exp_avg.data_ptr<float>() + begin, exp_avg_sq.data_ptr<float>() + begin, end - begin,
                                       norm, float(max_norm), float(lr), float(beta1), float(beta2), float(eps),
                                       float(weight_decay), step, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "flat_adamw failed (code ", rc, ")");
}

// ---- frozen batch-norm + residual + ReLU over NHWC activations (backbone.py:46-55) ------------------------------------
static bool nhwc_dense(const at::Tensor& t) {
  return t.is_cuda() && t.scalar_type() == at::kFloat && t.dim() == 4 && t.is_contiguous(at::MemoryFormat::ChannelsLast);
}

at::Tensor frozen_bn_act_forward(const at::Tensor& x, const c10::optional<at::Tensor>& residual, const at::Tensor& scale,
                                 const at::Tensor& shift, bool relu) {
  TORCH_CHECK(nhwc_dense(x), "frozen_bn_act: x must be a channels-last fp32 CUDA tensor [N,C,H,W]");
  const int64_t C = x.size(1);
  TORCH_CHECK(C % 4 == 0 && scale.numel() == C && shift.numel() == C && scale.is_cuda() && shift.is_cuda() &&
              scale.scalar_type() == at::kFloat && shift.scalar_type() == at::kFloat, "frozen_bn_act: bad scale/shift");
  const float* res = nullptr;
  if (residual.has_value()) {
    TORCH_CHECK(nhwc_dense(*residual) && residual->sizes() == x.sizes(), "frozen_bn_act: residual must match x");
    res = residual->data_ptr<float>();
  }
  const c10::cuda::CUDAGuard guard(x.device());
  auto sc = scale.contiguous().view({C}), sh = shift.contiguous().view({C});
  auto y = at::empty_like(x, x.options().memory_format(at::MemoryFormat::ChannelsLast));
  const int rc = tfb200_frozen_bn_act_fwd_f32(x.data_ptr<float>(), res, sc.data_ptr<float>(), sh.data_ptr<float>(),
                                              y.data_ptr<float>(), x.numel() / C, int(C), relu ? 1 : 0,
                                              at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "frozen_bn_act_forward failed (code ", rc, ")");
  return y;
}

at::Tensor frozen_bn_relu_maxpool(const at::Tensor& x, const at::Tensor& scale, const at::Tensor& shift) {
  TORCH_CHECK(nhwc_dense(x), "frozen_bn_relu_maxpool: x must be a channels-last fp32 CUDA tensor [N,C,H,W]");
  const int64_t N = x.size(0), C = x.size(1), H = x.size(2), W = x.size(3);
  TORCH_CHECK(C % 4 == 0 && scale.numel() == C && shift.numel() == C && scale.is_cuda() && shift.is_cuda() &&
              scale.scalar_type() == at::kFloat && shift.scalar_type() == at::kFloat, "frozen_bn_relu_maxpool: bad scale/shift");
  const c10::cuda::CUDAGuard guard(x.device());
  auto sc = scale.contiguous().view({C}), sh = shift.contiguous().view({C});
  auto y = at::empty({N, C, (H + 1) / 2, (W + 1) / 2}, x.options().memory_format(at::MemoryFormat::ChannelsLast));
  const int rc = tfb200_frozen_bn_relu_maxpool_f32(x.data_ptr<float>(), sc.data_ptr<float>(), sh.data_ptr<float>(),
                                                   y.data_ptr<float>(), int(N), int(H), int(W), int(C),
                                                   at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "frozen_bn_relu_maxpool failed (code ", rc, ")");
  return y;
}

std::vector<at::Tensor> frozen_bn_act_backward(const at::Tensor& dy, const at::Tensor& y, const at::Tensor& scale, bool relu,
                                               bool need_dx, bool need_dres) {
  TORCH_CHECK(nhwc_dense(y) && dy.is_cuda() && dy.scalar_type() == at::kFloat && dy.sizes() == y.sizes(), "frozen_bn_act_backward: bad dy / y");
  TORCH_CHECK(need_dx || need_dres, "frozen_bn_act_backward: nothing to compute");
  const int64_t C = y.size(1);
  const c10::cuda::CUDAGuard guard(y.device());
  auto g = dy.contiguous(at::MemoryFormat::ChannelsLast);
  auto sc = scale.contiguous().view({C});
  at::Tensor dx, dres;
  if (need_dx) dx = at::empty_like(y, y.options().memory_format(at::MemoryFormat::ChannelsLast));
  if (need_dres) dres = at::empty_like(y, y.options().memory_format(at::MemoryFormat::ChannelsLast));
  const int rc = tfb200_frozen_bn_act_bwd_f32(g.data_ptr<float>(), y.data_ptr<float>(), sc.data_ptr<float>(),
                                              need_dx ? dx.data_ptr<float>() : nullptr,
                                              need_dres ? dres.data_ptr<float>() : nullptr, y.numel() / C, int(C),
                                              relu ? 1 : 0, at::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "frozen_bn_act_backward failed (code ", rc, ")");
  return {dx, dres};
}

// ---- residual + dropout + LayerNorm with mask-free (seeded) dropout --------------------------------------------------
std::vector<at::Tensor> add_dropout_layernorm_seeded_forward(const at::Tensor& x, const at::Tensor& branch, const at::Tensor& seed,
                                                             const at::Tensor& gamma, const at::Tensor& beta,
                                                             double keep_prob, double eps) {
  TORCH_CHECK(x.is_cuda() && branch.is_cuda(), "add_dropout_layernorm: CUDA tensors required (no CPU path)");
  TORCH_CHECK(x.scalar_type() == at::kFloat && branch.scalar_type() == at::kFloat, "fp32 only");
  TORCH_CHECK(x.sizes() == branch.sizes(), "x and branch must have the same shape");
  TORCH_CHECK(seed.is_cuda() && seed.scalar_type() == at::kLong && seed.numel() >= 1, "seed must be an int64 CUDA tensor");
  const int64_t C = x.size(-1);
  const at::Tensor xc = x.contiguous(), bc = branch.contiguous(), g = gamma.contiguous(), b = beta.contiguous();
  const int64_t rows = xc.numel() / C;
  const c10::cuda::CUDAGuard guard(x.device());
  at::Tensor y = at::empty_like(xc), s = at::empty_like(xc);
  at::Tensor mean = at::empty({rows}, xc.options()), rstd = at::empty({rows}, xc.options());
  const int rc = tfb200_add_dropout_layernorm_seeded_fwd_f32(
      xc.data_ptr<float>(), bc.data_ptr<float>(), seed.data_ptr<int64_t>(), g.data_ptr<float>(), b.data_ptr<float>(),
      s.data_ptr<float>(), y.data_ptr<float>(), mean.data_ptr<float>(), rstd.data_ptr<float>(), rows, int(C),
      float(keep_prob), float(eps), c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "add_dropout_layernorm_seeded_forward failed (code ", rc, ")");
  return {y, s, mean, rstd};
}

std::vector<at::Tensor> add_dropout_layernorm_seeded_backward(const at::Tensor& dy, const at::Tensor& s, const at::Tensor& seed,
                                                              const at::Tensor& gamma, const at::Tensor& mean,
                                                              const at::Tensor& rstd, double keep_prob) {
  TORCH_CHECK(dy.is_cuda() && s.is_cuda(), "add_dropout_layernorm: CUDA tensors required (no CPU path)");
  TORCH_CHECK(seed.is_cuda() && seed.scalar_type() == at::kLong && seed.numel() >= 1, "seed must be an int64 CUDA tensor");
  const int64_t C = s.size(-1);
  const at::Tensor dyc = dy.contiguous(), g = gamma.contiguous();
  const int64_t rows = s.numel() / C;
  const c10::cuda::CUDAGuard guard(s.device());
  at::Tensor dx = at::empty_like(s), db = at::empty_like(s);
  at::Tensor dgamma = at::empty({C}, s.options()), dbeta = at::empty({C}, s.options());
  at::Tensor ws = at::empty({tfb200_ln_partial_ctas(rows), 2, C}, s.options());
  const int rc = tfb200_add_dropout_layernorm_seeded_bwd_f32(
      dyc.data_ptr<float>(), s.data_ptr<float>(), seed.data_ptr<int64_t>(), g.data_ptr<float>(), mean.data_ptr<float>(),
      rstd.data_ptr<float>(), dx.data_ptr<float>(), db.data_ptr<float>(), dgamma.data_ptr<float>(),
      dbeta.data_ptr<float>(), ws.data_ptr<float>(), rows, int(C), float(keep_prob),
      c10::cuda::getCurrentCUDAStream().stream());
  TORCH_CHECK(rc == 0, "add_dropout_layernorm_seeded_backward failed (code ", rc, ")");
  return {dx, db, dgamma, dbeta};
}

// ---- segmentation mask head (csrc/mask_head.cu) ----
static void check_f32(const at::Tensor& t, const char* what) {
  TORCH_CHECK(t.is_cuda() && t.scalar_type() == at::kFloat, what, ": fp32 CUDA tensor required (no CPU path)");
}

static void check_nhwc(const at::Tensor& t, const char* what) {
  check_f32(t, what);
  TORCH_CHECK(t.dim() == 4 && t.is_contiguous(at::MemoryFormat::ChannelsLast), what,
              ": [N, C, H, W] channels-last contiguous tensor required");
}

static at::Tensor empty_nhwc(at::IntArrayRef sizes, const at::Tensor& like) {
  return at::empty(sizes, like.options().memory_format(at::MemoryFormat::ChannelsLast));
}

static void raise_rc(int rc, const char* what) { TORCH_CHECK(rc == 0, what, " failed (code ", rc, ")"); }

// q [B, Q, heads*32], k [B, HW, heads*32], pad [B, HW] bool or None -> w [B, Q, heads, HW]
at::Tensor mask_attn_forward(const at::Tensor& q, const at::Tensor& k, const c10::optional<at::Tensor>& pad, int64_t heads,
                             double scale) {
  check_f32(q, "mask_attn q");
  check_f32(k, "mask_attn k");
  TORCH_CHECK(q.dim() == 3 && k.dim() == 3 && heads > 0 && q.size(2) == heads * 32 && k.size(2) == q.size(2) &&
              k.size(0) == q.size(0) && k.size(1) > 0, "mask_attn: q [B, Q, heads*32], k [B, HW, heads*32]");
  const at::Tensor qc = q.contiguous(), kc = k.contiguous();
  TORCH_CHECK(reinterpret_cast<uintptr_t>(qc.data_ptr()) % 16 == 0 && reinterpret_cast<uintptr_t>(kc.data_ptr()) % 16 == 0,
              "mask_attn: q and k must be 16-byte aligned");
  const int B = int(q.size(0)), Q = int(q.size(1)), HW = int(k.size(1));
  const uint8_t* pp = nullptr;
  at::Tensor pc;
  if (pad.has_value() && pad->defined()) {
    pc = pad->contiguous();
    TORCH_CHECK(pc.is_cuda() && pc.element_size() == 1 && pc.numel() == int64_t(B) * HW, "mask_attn: pad must be a bool [B, HW] CUDA tensor");
    pp = reinterpret_cast<const uint8_t*>(pc.data_ptr());
  }
  const c10::cuda::CUDAGuard guard(q.device());
  at::Tensor w = at::empty({B, Q, heads, HW}, qc.options());
  raise_rc(tfb200_mask_attn_fwd_f32(qc.data_ptr<float>(), kc.data_ptr<float>(), pp, w.data_ptr<float>(), B, Q, HW,
                                    int(heads), float(scale), c10::cuda::getCurrentCUDAStream().stream()),
           "mask_attn_forward");
  return w;
}

std::vector<at::Tensor> mask_attn_backward(const at::Tensor& q, const at::Tensor& k, const at::Tensor& w,
                                           const at::Tensor& dw, double scale) {
  check_f32(dw, "mask_attn dw");
  TORCH_CHECK(w.dim() == 4 && dw.sizes() == w.sizes() && q.is_contiguous() && k.is_contiguous() && w.is_contiguous(),
              "mask_attn_backward: saved tensors and dw [B, Q, heads, HW]");
  const int B = int(w.size(0)), Q = int(w.size(1)), heads = int(w.size(2)), HW = int(w.size(3));
  const at::Tensor dwc = dw.contiguous();
  const c10::cuda::CUDAGuard guard(w.device());
  at::Tensor ds = at::empty_like(w), dq = at::empty_like(q), dk = at::empty_like(k);
  raise_rc(tfb200_mask_attn_bwd_f32(q.data_ptr<float>(), k.data_ptr<float>(), w.data_ptr<float>(), dwc.data_ptr<float>(),
                                    ds.data_ptr<float>(), dq.data_ptr<float>(), dk.data_ptr<float>(), B, Q, HW, heads,
                                    float(scale), c10::cuda::getCurrentCUDAStream().stream()),
           "mask_attn_backward");
  return {dq, dk};
}

static const float* opt_addend(const c10::optional<at::Tensor>& addend, const at::Tensor& x, int per_image) {
  if (!addend.has_value() || !addend->defined()) return nullptr;
  check_nhwc(*addend, "group_norm_relu addend");
  TORCH_CHECK(addend->size(0) * per_image == x.size(0) && addend->size(1) == x.size(1) && addend->size(2) == x.size(2) &&
              addend->size(3) == x.size(3), "group_norm_relu: addend must be [N / per_image, C, H, W]");
  return addend->data_ptr<float>();
}

// x [N, C, H, W] channels-last (+ addend [N / per_image, C, H, W]) -> {y, mean [N, G], rstd [N, G]}
std::vector<at::Tensor> group_norm_relu_forward(const at::Tensor& x, const c10::optional<at::Tensor>& addend,
                                                const at::Tensor& gamma, const at::Tensor& beta, int64_t groups,
                                                int64_t per_image, double eps) {
  check_nhwc(x, "group_norm_relu x");
  TORCH_CHECK(per_image > 0 && x.size(0) % per_image == 0, "group_norm_relu: N must be a multiple of per_image");
  const int64_t C = x.size(1);
  check_f32(gamma, "group_norm_relu gamma");
  check_f32(beta, "group_norm_relu beta");
  TORCH_CHECK(gamma.numel() == C && beta.numel() == C && gamma.is_contiguous() && beta.is_contiguous(),
              "group_norm_relu: gamma / beta [C]");
  const float* ap = opt_addend(addend, x, int(per_image));
  const c10::cuda::CUDAGuard guard(x.device());
  at::Tensor y = empty_nhwc(x.sizes(), x);
  at::Tensor mean = at::empty({x.size(0), groups}, x.options()), rstd = at::empty({x.size(0), groups}, x.options());
  raise_rc(tfb200_group_norm_relu_fwd_f32(x.data_ptr<float>(), ap, gamma.data_ptr<float>(), beta.data_ptr<float>(),
                                          y.data_ptr<float>(), mean.data_ptr<float>(), rstd.data_ptr<float>(),
                                          int(x.size(0)), int(per_image), x.size(2) * x.size(3), int(C), int(groups),
                                          float(eps), c10::cuda::getCurrentCUDAStream().stream()),
           "group_norm_relu_forward");
  return {y, mean, rstd};
}

// -> {dx, daddend (undefined without addend), dgamma, dbeta}
std::vector<at::Tensor> group_norm_relu_backward(const at::Tensor& dy, const at::Tensor& x,
                                                 const c10::optional<at::Tensor>& addend, const at::Tensor& y,
                                                 const at::Tensor& gamma, const at::Tensor& mean, const at::Tensor& rstd,
                                                 int64_t per_image) {
  check_nhwc(x, "group_norm_relu x");
  check_nhwc(y, "group_norm_relu y");
  check_f32(dy, "group_norm_relu dy");
  TORCH_CHECK(dy.sizes() == x.sizes() && y.sizes() == x.sizes() && per_image > 0 && x.size(0) % per_image == 0,
              "group_norm_relu_backward: dy, x, y must have one shape");
  const at::Tensor dyc = dy.contiguous(at::MemoryFormat::ChannelsLast);
  const int64_t N = x.size(0), C = x.size(1);
  const float* ap = opt_addend(addend, x, int(per_image));
  const c10::cuda::CUDAGuard guard(x.device());
  at::Tensor dx = empty_nhwc(x.sizes(), x);
  at::Tensor da = ap ? empty_nhwc(addend->sizes(), x) : at::Tensor();
  at::Tensor daff = at::empty({2, C}, x.options()), ws = at::empty({N, 2, C}, x.options());
  raise_rc(tfb200_group_norm_relu_bwd_f32(dyc.data_ptr<float>(), x.data_ptr<float>(), ap, y.data_ptr<float>(),
                                          gamma.data_ptr<float>(), mean.data_ptr<float>(), rstd.data_ptr<float>(),
                                          dx.data_ptr<float>(), ap ? da.data_ptr<float>() : nullptr, daff.data_ptr<float>(),
                                          ws.data_ptr<float>(), int(N), int(per_image), x.size(2) * x.size(3), int(C),
                                          int(mean.size(1)), c10::cuda::getCurrentCUDAStream().stream()),
           "group_norm_relu_backward");
  return {dx, da, daff[0], daff[1]};
}

// a [N / per_image, C, Ho, Wo] + nearest_upsample(x [N, C, Hi, Wi]), both channels-last
at::Tensor upsample_add_forward(const at::Tensor& x, const at::Tensor& a) {
  check_nhwc(x, "upsample_add x");
  check_nhwc(a, "upsample_add a");
  TORCH_CHECK(a.size(0) > 0 && x.size(0) % a.size(0) == 0 && a.size(1) == x.size(1),
              "upsample_add: x [N, C, Hi, Wi] and a [N / per_image, C, Ho, Wo]");
  const c10::cuda::CUDAGuard guard(x.device());
  at::Tensor out = empty_nhwc({x.size(0), x.size(1), a.size(2), a.size(3)}, x);
  raise_rc(tfb200_upsample_add_fwd_f32(x.data_ptr<float>(), a.data_ptr<float>(), out.data_ptr<float>(), int(x.size(0)),
                                       int(x.size(0) / a.size(0)), int(x.size(2)), int(x.size(3)), int(a.size(2)),
                                       int(a.size(3)), int(x.size(1)), c10::cuda::getCurrentCUDAStream().stream()),
           "upsample_add_forward");
  return out;
}

std::vector<at::Tensor> upsample_add_backward(const at::Tensor& dout, int64_t images, int64_t Hi, int64_t Wi) {
  check_f32(dout, "upsample_add dout");
  TORCH_CHECK(dout.dim() == 4 && images > 0 && dout.size(0) % images == 0 && Hi > 0 && Wi > 0,
              "upsample_add_backward: dout [N, C, Ho, Wo]");
  const at::Tensor g = dout.contiguous(at::MemoryFormat::ChannelsLast);
  const int64_t N = g.size(0), C = g.size(1);
  const c10::cuda::CUDAGuard guard(g.device());
  at::Tensor dx = empty_nhwc({N, C, Hi, Wi}, g), da = empty_nhwc({images, C, g.size(2), g.size(3)}, g);
  raise_rc(tfb200_upsample_add_bwd_f32(g.data_ptr<float>(), dx.data_ptr<float>(), da.data_ptr<float>(), int(N),
                                       int(N / images), int(Hi), int(Wi), int(g.size(2)), int(g.size(3)), int(C),
                                       c10::cuda::getCurrentCUDAStream().stream()),
           "upsample_add_backward");
  return {dx, da};
}

static void check_mask_loss_args(const at::Tensor& logits, const at::Tensor& src, const at::Tensor& tgt_masks,
                                 const at::Tensor& tgt, const at::Tensor& num_boxes) {
  check_f32(logits, "mask_loss logits");
  TORCH_CHECK(logits.dim() == 3 && logits.is_contiguous(), "mask_loss: logits must be a contiguous [R, h, w] tensor");
  TORCH_CHECK(tgt_masks.is_cuda() && tgt_masks.dim() == 3 && tgt_masks.element_size() == 1 &&
              tgt_masks.scalar_type() != at::kChar && tgt_masks.is_contiguous(),
              "mask_loss: target masks must be a contiguous bool/uint8 [T, Ht, Wt] CUDA tensor");
  TORCH_CHECK(src.is_cuda() && tgt.is_cuda() && src.scalar_type() == at::kLong && tgt.scalar_type() == at::kLong &&
              src.dim() == 1 && src.sizes() == tgt.sizes() && src.is_contiguous() && tgt.is_contiguous(),
              "mask_loss: src / tgt must be int64 [M] CUDA tensors");
  check_f32(num_boxes, "mask_loss num_boxes");
  TORCH_CHECK(num_boxes.numel() == 1, "mask_loss: num_boxes must be a one-element tensor");
}

// -> {out [2] = (loss_mask, loss_dice), stats [M, 4]}
std::vector<at::Tensor> mask_loss_forward(const at::Tensor& logits, const at::Tensor& src, const at::Tensor& tgt_masks,
                                          const at::Tensor& tgt, const at::Tensor& num_boxes, double alpha, double gamma) {
  check_mask_loss_args(logits, src, tgt_masks, tgt, num_boxes);
  const int M = int(src.numel()), Ht = int(tgt_masks.size(1)), Wt = int(tgt_masks.size(2));
  const c10::cuda::CUDAGuard guard(logits.device());
  at::Tensor out = at::empty({2}, logits.options()), stats = at::empty({M, 4}, logits.options());
  at::Tensor ws = at::empty({M, tfb200_mask_loss_partial_chunks(Ht, Wt), 4}, logits.options());
  raise_rc(tfb200_mask_loss_fwd_f32(logits.data_ptr<float>(), src.data_ptr<int64_t>(),
                                    reinterpret_cast<const uint8_t*>(tgt_masks.data_ptr()), tgt.data_ptr<int64_t>(),
                                    num_boxes.data_ptr<float>(), stats.data_ptr<float>(), ws.data_ptr<float>(),
                                    out.data_ptr<float>(), M, int(logits.size(1)), int(logits.size(2)), Ht, Wt,
                                    float(alpha), float(gamma), c10::cuda::getCurrentCUDAStream().stream()),
           "mask_loss_forward");
  return {out, stats};
}

at::Tensor mask_loss_backward(const at::Tensor& logits, const at::Tensor& src, const at::Tensor& tgt_masks,
                              const at::Tensor& tgt, const at::Tensor& stats, const at::Tensor& num_boxes,
                              const at::Tensor& g2, double alpha, double gamma) {
  check_mask_loss_args(logits, src, tgt_masks, tgt, num_boxes);
  check_f32(g2, "mask_loss g2");
  TORCH_CHECK(g2.numel() == 2 && stats.numel() == src.numel() * 4, "mask_loss_backward: g2 [2], stats [M, 4]");
  const at::Tensor gc = g2.contiguous();
  const c10::cuda::CUDAGuard guard(logits.device());
  at::Tensor grad = at::empty_like(logits);
  raise_rc(tfb200_mask_loss_bwd_f32(logits.data_ptr<float>(), src.data_ptr<int64_t>(),
                                    reinterpret_cast<const uint8_t*>(tgt_masks.data_ptr()), tgt.data_ptr<int64_t>(),
                                    stats.data_ptr<float>(), num_boxes.data_ptr<float>(), gc.data_ptr<float>(),
                                    grad.data_ptr<float>(), int(logits.size(0)), int(src.numel()), int(logits.size(1)),
                                    int(logits.size(2)), int(tgt_masks.size(1)), int(tgt_masks.size(2)), float(alpha),
                                    float(gamma), c10::cuda::getCurrentCUDAStream().stream()),
           "mask_loss_backward");
  return grad;
}

PYBIND11_MODULE(TORCH_EXTENSION_NAME, m) {
  m.doc() = "H100 (sm_90a) multi-scale deformable attention; drop-in for the reference extension";
  m.def("ms_deform_attn_forward", &ms_deform_attn_forward, "ms_deform_attn_forward");
  m.def("ms_deform_attn_backward", &ms_deform_attn_backward, "ms_deform_attn_backward");
  // extras (not in the reference surface)
  m.def("abi_version", []() { return msda_b200_abi_version(); });
  m.def("launch_count", []() { return msda_b200_launch_count(); });
  m.def("set_variant", [](int f, int b) { msda_b200_set_variant(f, b); });
  m.def("ms_deform_attn_forward_enc", &ms_deform_attn_forward_enc);
  m.def("ms_deform_attn_forward_enc_strict", &ms_deform_attn_forward_enc_strict);
  m.def("ms_deform_attn_backward_enc", &ms_deform_attn_backward_enc);
  m.def("ms_deform_attn_backward_enc_strict", &ms_deform_attn_backward_enc_strict);
  m.def("ms_deform_attn_forward_enc_fused", &ms_deform_attn_forward_enc_fused);
  m.def("ms_deform_attn_backward_enc_fused", &ms_deform_attn_backward_enc_fused);
  m.def("ms_deform_attn_forward_fused", &ms_deform_attn_forward_fused);
  m.def("ms_deform_attn_backward_fused", &ms_deform_attn_backward_fused);
  m.def("add_dropout_layernorm_forward", &add_dropout_layernorm_forward);
  m.def("add_dropout_layernorm_backward", &add_dropout_layernorm_backward);
  m.def("add_dropout_layernorm_seeded_forward", &add_dropout_layernorm_seeded_forward);
  m.def("add_dropout_layernorm_seeded_backward", &add_dropout_layernorm_seeded_backward);
  m.def("colsum", &colsum);
  m.def("lsa", &lsa);
  m.def("match_cost", &match_cost);
  m.def("set_loss_forward", &set_loss_forward);
  m.def("set_loss_backward", &set_loss_backward);
  m.def("sampling_prep_forward", &sampling_prep_forward);
  m.def("sampling_prep_backward", &sampling_prep_backward);
  m.def("small_attention_forward", &small_attention_forward);
  m.def("small_attention_backward", &small_attention_backward);
  m.def("refine_boxes_forward", &refine_boxes_forward);
  m.def("refine_boxes_backward", &refine_boxes_backward);
  m.def("tf32_linear", &tf32_linear);
  m.def("tf32_linear_supported", &tf32_linear_supported);
  m.def("tf32_linear_dgrad", &tf32_linear_dgrad);
  m.def("tf32_linear_wgrad", &tf32_linear_wgrad);
  m.def("relu_dropout_forward", &relu_dropout_forward);
  m.def("relu_dropout_backward", &relu_dropout_backward);
  m.def("detect_postprocess", &detect_postprocess);
  m.def("flat_adamw", &flat_adamw);
  m.def("frozen_bn_act_forward", &frozen_bn_act_forward);
  m.def("frozen_bn_act_backward", &frozen_bn_act_backward);
  m.def("frozen_bn_relu_maxpool", &frozen_bn_relu_maxpool);
  m.def("mask_attn_forward", &mask_attn_forward);
  m.def("mask_attn_backward", &mask_attn_backward);
  m.def("group_norm_relu_forward", &group_norm_relu_forward);
  m.def("group_norm_relu_backward", &group_norm_relu_backward);
  m.def("upsample_add_forward", &upsample_add_forward);
  m.def("upsample_add_backward", &upsample_add_backward);
  m.def("mask_loss_forward", &mask_loss_forward);
  m.def("mask_loss_backward", &mask_loss_backward);
}
