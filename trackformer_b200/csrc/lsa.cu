// Device-side Hungarian matching for the set-prediction loss (sm_90a).
//
// The reference computes the matching cost on the GPU, copies it to the host and calls
// scipy.optimize.linear_sum_assignment once per decoder layer (src/trackformer/models/matcher.py:104,127 -- six
// device->host synchronisations per training step).  This kernel solves the same rectangular assignment problems
// on the device: one CTA per (decoder layer, batch element) problem, queries x that element's ground-truth boxes,
// by shortest augmenting paths with dual variables (the Jonker-Volgenant scheme scipy's solver is built on; lsa_core.h,
// the solver the tracker and the MOT evaluators share), in double precision like scipy (which promotes the float32
// cost matrix to float64).  The optimum of a cost matrix
// without exact ties is unique, so the assignment equals scipy's; pairs are emitted sorted by query index, the order
// linear_sum_assignment returns.  (With exact float ties the two solvers may pick different, equally optimal pairs.)
//
// Problem p = (k, b): cost(query j, target i) = cost[((k*B + b)*Q + j) * T + off[b] + i], i < off[b+1]-off[b] <= Q.
// Outputs, for every p and rank r in query order:  src[k*T + off[b] + r] = query index,
//                                                    tgt[k*T + off[b] + r] = off[b] + target index.
//
// tfb200_lsa_f32 keeps a problem's whole state in shared memory (25 B per query), so it takes Q up to about 8,000.  The
// encoder loss of two-stage Deformable DETR matches every memory token (22,223 at 800x1333), which
// tfb200_lsa_wide_f32 solves with the same routine over a global workspace: the cost block transposed to
// [target][query], so that each row scan reads contiguous memory, and the column state (L2-resident at these sizes).
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "launch_counter.h"
#include "lsa_core.h"

namespace {

namespace lsa = tfb200_lsa;

constexpr int kLsaThreads = 256;

// One (layer, image) problem, shared by both kernels: the solve, then the pairs sorted by query index (rank = number
// of targets matched to a smaller query).  The solver state lives where the caller points it: shared memory in
// lsa_kernel, a global workspace in lsa_wide_kernel.
template <int NT>
__device__ __forceinline__ void lsa_problem(const lsa::Strided& cost, int nr, int nc, const lsa::Rows& R,
                                            const lsa::Cols& C, int64_t* __restrict__ src, int64_t* __restrict__ tgt,
                                            size_t out0, int t0, int* __restrict__ status) {
  __shared__ typename lsa::Cta<NT>::Scratch scratch;
  if (!lsa::solve<lsa::Cta<NT>>(nr, nc, cost, R, C, scratch)) {
    if (threadIdx.x == 0) atomicExch(status, 2);   // infeasible (all +inf)
    return;
  }
  for (int i = threadIdx.x; i < nr; i += NT) {
    const int q = R.col4row[i];
    int rank = 0;
    for (int o = 0; o < nr; ++o) rank += R.col4row[o] < q;
    src[out0 + rank] = q;
    tgt[out0 + rank] = t0 + i;
  }
}

__global__ void __launch_bounds__(kLsaThreads)
lsa_kernel(const float* __restrict__ cost, const int* __restrict__ off, int64_t* __restrict__ src,
           int64_t* __restrict__ tgt, int B, int Q, int T, int* __restrict__ status) {
  extern __shared__ __align__(8) unsigned char smem[];
  const int k = blockIdx.x / B, b = blockIdx.x % B;
  const int t0 = off[b], nr = off[b + 1] - t0, nc = Q;       // rows = targets, columns = queries
  if (nr <= 0) return;
  if (nr > nc) {                                               // caller guarantees nr <= nc; flag instead of UB
    if (threadIdx.x == 0) atomicExch(status, 1);
    return;
  }
  const float* C = cost + (size_t(k) * B + b) * size_t(Q) * T + t0;   // C[j * T + i]
  double* shortest = reinterpret_cast<double*>(smem);          // [nc]
  double* v = shortest + nc;                                   // [nc]
  double* u = v + nc;                                          // [nr]
  int* path = reinterpret_cast<int*>(u + nr);                  // [nc]
  int* row4col = path + nc;                                    // [nc]
  int* col4row = row4col + nc;                                 // [nr]
  int* visited = col4row + nr;                                 // [nr]
  uint8_t* in_sc = reinterpret_cast<uint8_t*>(visited + nr);   // [nc]
  lsa_problem<kLsaThreads>(lsa::Strided{C, 1, size_t(T)}, nr, nc, lsa::Rows{u, col4row, visited},
                           lsa::Cols{shortest, v, path, row4col, in_sc}, src, tgt, size_t(k) * T + t0, t0, status);
}

// ---- wide problems: column state in a global workspace, cost transposed to [target][query] -----------------------
constexpr int kWideThreads = 1024;

// Per-problem workspace layout (all problems alike, sized for max_targets rows): see lsa_wide_bytes.
struct WideLayout {
  size_t cost, shortest, v, u, path, row4col, col4row, visited, in_sc, total;
};

__host__ __device__ inline size_t wide_align(size_t x) { return (x + 255) & ~size_t(255); }

__host__ __device__ inline WideLayout wide_layout(int Q, int R) {
  WideLayout l;
  size_t o = 0;
  l.cost = o;     o = wide_align(o + size_t(R) * Q * 4);
  l.shortest = o; o = wide_align(o + size_t(Q) * 8);
  l.v = o;        o = wide_align(o + size_t(Q) * 8);
  l.u = o;        o = wide_align(o + size_t(R) * 8);
  l.path = o;     o = wide_align(o + size_t(Q) * 4);
  l.row4col = o;  o = wide_align(o + size_t(Q) * 4);
  l.col4row = o;  o = wide_align(o + size_t(R) * 4);
  l.visited = o;  o = wide_align(o + size_t(R) * 4);
  l.in_sc = o;    o = wide_align(o + size_t(Q));
  l.total = o;
  return l;
}

// cost[(k*B + b)*Q + j][t0 + i] -> ws(problem)[i * Q + j], 32 x 32 tiles through shared memory.
// grid (ceil(Q/32), ceil(max_targets/32), K*B), block (32, 8)
__global__ void lsa_wide_transpose_kernel(const float* __restrict__ cost, const int* __restrict__ off,
                                          unsigned char* __restrict__ ws, int B, int Q, int T, int R) {
  __shared__ float tile[32][33];
  const int p = blockIdx.z, k = p / B, b = p % B;
  const int t0 = off[b], nr = off[b + 1] - t0;
  if (nr <= 0 || nr > Q || nr > R) return;
  const WideLayout l = wide_layout(Q, R);
  float* dst = reinterpret_cast<float*>(ws + size_t(p) * l.total + l.cost);
  const float* C = cost + (size_t(k) * B + b) * size_t(Q) * T + t0;
  const int j0 = blockIdx.x * 32, i0 = blockIdx.y * 32;
  if (i0 >= nr) return;
  for (int y = threadIdx.y; y < 32; y += 8) {
    const int j = j0 + y, i = i0 + threadIdx.x;
    if (j < Q && i < nr) tile[y][threadIdx.x] = C[size_t(j) * T + i];
  }
  __syncthreads();
  for (int y = threadIdx.y; y < 32; y += 8) {
    const int i = i0 + y, j = j0 + threadIdx.x;
    if (i < nr && j < Q) dst[size_t(i) * Q + j] = tile[threadIdx.x][y];
  }
}

__global__ void __launch_bounds__(kWideThreads)
lsa_wide_kernel(const int* __restrict__ off, unsigned char* __restrict__ ws, int64_t* __restrict__ src,
                int64_t* __restrict__ tgt, int B, int Q, int T, int R, int* __restrict__ status) {
  const int p = blockIdx.x, k = p / B, b = p % B;
  const int t0 = off[b], nr = off[b + 1] - t0, nc = Q;
  if (nr <= 0) return;
  if (nr > nc || nr > R) {
    if (threadIdx.x == 0) atomicExch(status, 1);
    return;
  }
  const WideLayout l = wide_layout(Q, R);
  unsigned char* w = ws + size_t(p) * l.total;
  const lsa::Rows rows{reinterpret_cast<double*>(w + l.u), reinterpret_cast<int*>(w + l.col4row),
                       reinterpret_cast<int*>(w + l.visited)};
  const lsa::Cols cols{reinterpret_cast<double*>(w + l.shortest), reinterpret_cast<double*>(w + l.v),
                       reinterpret_cast<int*>(w + l.path), reinterpret_cast<int*>(w + l.row4col), w + l.in_sc};
  lsa_problem<kWideThreads>(lsa::Strided{reinterpret_cast<const float*>(w + l.cost), size_t(Q), 1}, nr, nc, rows,
                            cols, src, tgt, size_t(k) * T + t0, t0, status);
}

}  // namespace

extern "C" {

size_t tfb200_lsa_shared_bytes(int Q, int max_targets) {
  return size_t(Q) * (8 + 8 + 4 + 4 + 1) + size_t(max_targets > 0 ? max_targets : 0) * (8 + 4 + 4) + 64;
}

int tfb200_lsa_f32(const float* cost, const int* offsets_dev, int64_t* src, int64_t* tgt, int K, int B, int Q, int T,
                   int max_targets, int* status_dev, void* stream) {
  if (!cost || !offsets_dev || !src || !tgt || !status_dev) return TFB200_E_NULLPTR;
  if (K <= 0 || B <= 0 || Q <= 0 || T < 0 || max_targets < 0 || max_targets > Q) return TFB200_E_SHAPE;
  if (T == 0) return 0;
  const size_t smem = tfb200_lsa_shared_bytes(Q, max_targets);
  if (smem > TFB200_LSA_SHARED_MAX) return TFB200_E_SHAPE;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(lsa_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    if (e != cudaSuccess) return int(e);
  }
  lsa_kernel<<<K * B, kLsaThreads, smem, cudaStream_t(stream)>>>(cost, offsets_dev, src, tgt, B, Q, T, status_dev);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

size_t tfb200_lsa_wide_workspace_bytes(int K, int B, int Q, int max_targets) {
  if (K <= 0 || B <= 0 || Q <= 0 || max_targets <= 0) return 0;
  return size_t(K) * B * wide_layout(Q, max_targets).total;
}

int tfb200_lsa_wide_f32(const float* cost, const int* offsets_dev, int64_t* src, int64_t* tgt, int K, int B, int Q,
                        int T, int max_targets, void* workspace, size_t workspace_bytes, int* status_dev,
                        void* stream) {
  if (!cost || !offsets_dev || !src || !tgt || !status_dev) return TFB200_E_NULLPTR;
  if (K <= 0 || B <= 0 || Q <= 0 || T < 0 || max_targets < 0 || max_targets > Q) return TFB200_E_SHAPE;
  if (T == 0 || max_targets == 0) return 0;
  if (size_t(K) * B > 0x7fffffffu || size_t(Q) > 0x7fffffffu / 32) return TFB200_E_SHAPE;
  if (!workspace) return TFB200_E_NULLPTR;
  if (workspace_bytes < tfb200_lsa_wide_workspace_bytes(K, B, Q, max_targets)) return TFB200_E_SHAPE;
  const cudaStream_t st = cudaStream_t(stream);
  const dim3 tgrid(unsigned((Q + 31) / 32), unsigned((max_targets + 31) / 32), unsigned(K * B));
  if (tgrid.y > 65535 || tgrid.z > 65535) return TFB200_E_SHAPE;
  lsa_wide_transpose_kernel<<<tgrid, dim3(32, 8), 0, st>>>(cost, offsets_dev, static_cast<unsigned char*>(workspace),
                                                          B, Q, T, max_targets);
  lsa_wide_kernel<<<K * B, kWideThreads, 0, st>>>(offsets_dev, static_cast<unsigned char*>(workspace), src, tgt, B, Q,
                                                  T, max_targets, status_dev);
  msda_b200_count_launches(2);
  return int(cudaGetLastError());
}

}  // extern "C"
