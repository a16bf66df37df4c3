// Device-side Hungarian matching for the set-prediction loss (sm_90a).
//
// The reference computes the matching cost on the GPU, copies it to the host and calls
// scipy.optimize.linear_sum_assignment once per decoder layer (src/trackformer/models/matcher.py:104,127 -- six
// device->host synchronisations per training step).  This kernel solves the same rectangular assignment problems
// on the device: one CTA per (decoder layer, batch element) problem, queries x that element's ground-truth boxes,
// by shortest augmenting paths with dual variables (the Jonker-Volgenant scheme scipy's solver is built on),
// in double precision like scipy (which promotes the float32 cost matrix to float64).  The optimum of a cost matrix
// without exact ties is unique, so the assignment equals scipy's; pairs are emitted sorted by query index, the order
// linear_sum_assignment returns.  (With exact float ties the two solvers may pick different, equally optimal pairs.)
//
// Problem p = (k, b): cost(query j, target i) = cost[((k*B + b)*Q + j) * T + off[b] + i], i < off[b+1]-off[b] <= Q.
// Outputs, for every p and rank r in query order:  src[k*T + off[b] + r] = query index,
//                                                    tgt[k*T + off[b] + r] = off[b] + target index.
#include <cuda_runtime.h>
#include <float.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "launch_counter.h"

namespace {

constexpr int kLsaThreads = 256;

struct MinKey {
  double val;
  int tie;    // 0: column unassigned (preferred on equal value), 1: assigned
  int idx;
};

__device__ __forceinline__ bool better(const MinKey& a, const MinKey& b) {
  if (a.val != b.val) return a.val < b.val;
  if (a.tie != b.tie) return a.tie < b.tie;
  return a.idx < b.idx;
}

__device__ __forceinline__ MinKey warp_min(MinKey k) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    MinKey other;
    other.val = __shfl_xor_sync(0xffffffffu, k.val, o);
    other.tie = __shfl_xor_sync(0xffffffffu, k.tie, o);
    other.idx = __shfl_xor_sync(0xffffffffu, k.idx, o);
    if (better(other, k)) k = other;
  }
  return k;
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
  int* visited = col4row + nr;                                 // [nr] rows in SR, in visiting order
  unsigned char* in_sc = reinterpret_cast<unsigned char*>(visited + nr);   // [nc]
  __shared__ MinKey s_key[kLsaThreads / 32];
  __shared__ MinKey s_best;
  __shared__ int s_i, s_sink, s_nvisited, s_fail;

  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int j = tid; j < nc; j += kLsaThreads) { v[j] = 0.0; row4col[j] = -1; }
  for (int i = tid; i < nr; i += kLsaThreads) { u[i] = 0.0; col4row[i] = -1; }
  if (tid == 0) s_fail = 0;
  __syncthreads();

  for (int cur = 0; cur < nr; ++cur) {
    for (int j = tid; j < nc; j += kLsaThreads) { shortest[j] = DBL_MAX; path[j] = -1; in_sc[j] = 0; }
    if (tid == 0) { s_i = cur; s_sink = -1; s_nvisited = 0; }
    __syncthreads();
    double min_val = 0.0;
    while (true) {
      const int i = s_i;
      if (tid == 0) visited[s_nvisited++] = i;
      const double ui = u[i];
      MinKey best{DBL_MAX, 1, INT32_MAX};
      for (int j = tid; j < nc; j += kLsaThreads) {
        if (in_sc[j]) continue;
        const double r = min_val + double(C[size_t(j) * T + i]) - ui - v[j];
        if (r < shortest[j]) { shortest[j] = r; path[j] = i; }
        const MinKey cand{shortest[j], row4col[j] == -1 ? 0 : 1, j};
        if (better(cand, best)) best = cand;
      }
      best = warp_min(best);
      if (lane == 0) s_key[wid] = best;
      __syncthreads();
      if (wid == 0) {
        MinKey kk = lane < kLsaThreads / 32 ? s_key[lane] : MinKey{DBL_MAX, 1, INT32_MAX};
        kk = warp_min(kk);
        if (lane == 0) {
          s_best = kk;
          if (kk.val == DBL_MAX || kk.idx == INT32_MAX) { s_fail = 1; s_sink = 0; }   // infeasible (all +inf)
          else {
            in_sc[kk.idx] = 1;
            if (row4col[kk.idx] == -1) s_sink = kk.idx; else s_i = row4col[kk.idx];
          }
        }
      }
      __syncthreads();
      min_val = s_best.val;
      if (s_sink != -1) break;
    }
    if (s_fail) break;
    // ---- dual update
    const int nvis = s_nvisited, sink = s_sink;
    for (int t = tid; t < nvis; t += kLsaThreads) {
      const int i = visited[t];
      if (i == cur) u[i] += min_val;
      else u[i] += min_val - shortest[col4row[i]];
    }
    for (int j = tid; j < nc; j += kLsaThreads)
      if (in_sc[j]) v[j] -= min_val - shortest[j];
    __syncthreads();
    // ---- augment along the path (short: at most nvis hops)
    if (tid == 0) {
      int j = sink;
      while (true) {
        const int i = path[j];
        row4col[j] = i;
        const int prev = col4row[i];
        col4row[i] = j;
        j = prev;
        if (i == cur) break;
      }
    }
    __syncthreads();
  }
  if (s_fail) {
    if (tid == 0) atomicExch(status, 2);
    return;
  }
  // ---- emit pairs sorted by query index (rank = number of targets matched to a smaller query)
  for (int i = tid; i < nr; i += kLsaThreads) {
    const int q = col4row[i];
    int rank = 0;
    for (int o = 0; o < nr; ++o) rank += col4row[o] < q;
    src[size_t(k) * T + t0 + rank] = q;
    tgt[size_t(k) * T + t0 + rank] = t0 + i;
  }
}

}  // namespace

extern "C" {

int tfb200_lsa_f32(const float* cost, const int* offsets_dev, int64_t* src, int64_t* tgt, int K, int B, int Q, int T,
                   int max_targets, int* status_dev, void* stream) {
  if (!cost || !offsets_dev || !src || !tgt || !status_dev) return TFB200_E_NULLPTR;
  if (K <= 0 || B <= 0 || Q <= 0 || T < 0 || max_targets < 0 || max_targets > Q) return TFB200_E_SHAPE;
  if (T == 0) return 0;
  const size_t smem = size_t(Q) * (8 + 8 + 4 + 4 + 1) + size_t(max_targets) * (8 + 4 + 4) + 64;
  if (smem > 200 * 1024) return TFB200_E_SHAPE;
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(lsa_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem));
    if (e != cudaSuccess) return int(e);
  }
  lsa_kernel<<<K * B, kLsaThreads, smem, cudaStream_t(stream)>>>(cost, offsets_dev, src, tgt, B, Q, T, status_dev);
  msda_b200_count_launches(1);
  return int(cudaGetLastError());
}

}  // extern "C"
