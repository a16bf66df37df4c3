// ORACLE -- TEST INFRASTRUCTURE ONLY.  C-ABI around the REFERENCE's own CUDA kernels, compiled from the reference
// sources where they lie (/root/reference/src/trackformer/models/ops/src/cuda/ms_deform_im2col_cuda.cuh, pulled in by
// the include below; nothing from it is copied into this repository).  Built only in the build container
// (`make -f oracle/Makefile ref` -> oracle/_ref/libmsda_refcuda.so, git-ignored, shipped to the GPU box by gpurun) and
// used by tests/test_refcuda_gpu.py and tools/opbench.py as (a) a GPU-vs-GPU parity check against the real reference
// kernels and (b) "the kernel to beat" on the same GPU.
//
// The reference's host wrappers (ms_deform_attn_cuda.cu) depend on ATen; this file restates only their launch
// sequence: forward = im2col kernel into a [L*P, N, Lq, M, D] `columns` buffer + sum over L*P (at::sum there,
// ms_deform_attn_cuda.cu:80); backward = coord kernel + col2im kernel on zero-filled outputs (:119-160); level start
// indices as the reference derives them (:52-58).
#include <cuda_runtime.h>
#include <stdint.h>

#include MSDA_REF_CUH

namespace {

template <typename T>
__global__ void sum_columns(const T* __restrict__ columns, T* __restrict__ out, int64_t n_out, int planes) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n_out; i += int64_t(gridDim.x) * blockDim.x) {
    T acc = 0;
    for (int p = 0; p < planes; ++p) acc += columns[int64_t(p) * n_out + i];
    out[i] = acc;
  }
}

__global__ void level_starts(const int64_t* shapes, int64_t* start, int L) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    int64_t acc = 0;
    for (int l = 0; l < L; ++l) { start[l] = acc; acc += shapes[2 * l] * shapes[2 * l + 1]; }
  }
}

}  // namespace

extern "C" {

// workspace: columns [L*P*N*Lq*M*D] T followed by level_start [L] int64 (caller allocates; see refcuda_ws_bytes)
int64_t refcuda_ws_bytes(int N, int M, int D, int L, int Lq, int P, int elem) {
  return int64_t(L) * P * N * Lq * M * D * elem + int64_t(L) * 8 + 64;
}

int refcuda_forward_f32(const float* value, const int64_t* shapes, const float* loc, const float* attn, float* out,
                        void* ws, int N, int S, int M, int D, int L, int Lq, int P, void* stream) {
  cudaStream_t st = cudaStream_t(stream);
  float* columns = static_cast<float*>(ws);
  const int64_t n_out = int64_t(N) * Lq * M * D;
  int64_t* start = reinterpret_cast<int64_t*>((reinterpret_cast<uintptr_t>(columns + int64_t(L) * P * n_out) + 63) & ~uintptr_t(63));
  level_starts<<<1, 32, 0, st>>>(shapes, start, L);
  ms_deformable_im2col_cuda<float>(st, value, shapes, start, loc, attn, N, S, M, D, L, Lq, P, columns);
  sum_columns<float><<<int((n_out + 255) / 256), 256, 0, st>>>(columns, out, n_out, L * P);
  return int(cudaGetLastError());
}

int refcuda_backward_f32(const float* value, const int64_t* shapes, const float* loc, const float* attn,
                         const float* grad_out, float* grad_value, float* grad_loc, float* grad_attn, void* ws,
                         int N, int S, int M, int D, int L, int Lq, int P, void* stream) {
  cudaStream_t st = cudaStream_t(stream);
  int64_t* start = static_cast<int64_t*>(ws);
  level_starts<<<1, 32, 0, st>>>(shapes, start, L);
  cudaMemsetAsync(grad_value, 0, sizeof(float) * size_t(N) * S * M * D, st);
  cudaMemsetAsync(grad_loc, 0, sizeof(float) * size_t(N) * Lq * M * L * P * 2, st);
  cudaMemsetAsync(grad_attn, 0, sizeof(float) * size_t(N) * Lq * M * L * P, st);
  ms_deformable_col2im_coord_cuda<float>(st, grad_out, value, shapes, start, loc, attn, N, S, M, D, L, Lq, P, grad_loc,
                                         grad_attn);
  ms_deformable_col2im_cuda<float>(st, grad_out, shapes, start, loc, attn, N, S, M, D, L, Lq, P, grad_value);
  return int(cudaGetLastError());
}

}  // extern "C"
