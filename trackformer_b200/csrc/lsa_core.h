// The rectangular assignment solver of the set-criterion matcher (lsa.cu), the device tracker's ReID matching
// (track_step_core.h) and the MOT evaluators' CLEAR-MOT and identity matchings (mot_eval_core.h): the shortest
// augmenting path method scipy.optimize.linear_sum_assignment is built on (Crouse 2016, after Jonker-Volgenant), with
// the duals in double precision like scipy.
//
// Each scan takes its minimum under a total order -- lower reduced cost, then an unassigned column, then the lower
// index -- so the result does not depend on how a thread group splits the columns: a CTA, one warp, one thread, and
// the g++ host build (where every group is the one calling thread) all produce the same assignment bit for bit.  The
// optimum of a cost matrix without exact ties is unique, so it is scipy's; among equally optimal assignments scipy's
// choice may differ.
#pragma once

#include <float.h>
#include <stddef.h>
#include <stdint.h>

#include "host_device.h"

namespace tfb200_lsa {

// a column of the scan: its shortest path length, whether it is assigned, its index
struct Key {
  double val;
  int tie;    // 0: column unassigned (preferred on equal value), 1: assigned
  int idx;
};

HD_FORCEINLINE bool better(const Key& a, const Key& b) {
  if (a.val != b.val) return a.val < b.val;
  if (a.tie != b.tie) return a.tie < b.tie;
  return a.idx < b.idx;
}

#if defined(__CUDACC__)
__device__ __forceinline__ Key warp_min(Key k) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    Key other;
    other.val = __shfl_xor_sync(0xffffffffu, k.val, o);
    other.tie = __shfl_xor_sync(0xffffffffu, k.tie, o);
    other.idx = __shfl_xor_sync(0xffffffffu, k.idx, o);
    if (better(other, k)) k = other;
  }
  return k;
}
#endif

// Thread groups.  min() hands every thread of the group the group's minimum key, and orders the group's memory
// accesses before it against those after it.

// the calling thread alone
struct Thread {
  struct Scratch {};
  static constexpr int kSize = 1;
  HD_FORCEINLINE static int rank() { return 0; }
  HD_FORCEINLINE static void sync() {}
  HD_FORCEINLINE static Key min(Key k, Scratch&) { return k; }
};

// one whole warp
struct Warp {
  struct Scratch {};
  static constexpr int kSize = HD_NLANES;
  HD_FORCEINLINE static int rank() { return HD_LANE; }
  HD_FORCEINLINE static void sync() { HD_SYNCWARP(); }
  HD_FORCEINLINE static Key min(Key k, Scratch&) {
#if defined(__CUDACC__)
    k = warp_min(k);
    __syncwarp();
#endif
    return k;
  }
};

// a whole CTA of NT threads (blockDim.x == NT); the cross-warp keys go through the caller's shared Scratch
template <int NT>
struct Cta {
  static_assert(NT % 32 == 0 && NT <= 1024, "a CTA of whole warps");
  struct Scratch {
    Key warp[NT / 32];
    Key best;
  };
#if defined(__CUDACC__)
  static constexpr int kSize = NT;
#else
  static constexpr int kSize = 1;
#endif
  HD_FORCEINLINE static int rank() { return HD_TID; }
  HD_FORCEINLINE static void sync() { HD_SYNC(); }
  HD_FORCEINLINE static Key min(Key k, Scratch& s) {
#if defined(__CUDACC__)
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    k = warp_min(k);
    if (lane == 0) s.warp[wid] = k;
    __syncthreads();
    if (wid == 0) {
      k = lane < NT / 32 ? s.warp[lane] : Key{DBL_MAX, 1, INT32_MAX};
      k = warp_min(k);
      if (lane == 0) s.best = k;
    }
    __syncthreads();
    k = s.best;
#endif
    return k;
  }
};

// Solver state, where the caller puts it.  Per column: shortest path length, dual, predecessor row, assigned row (-1:
// none), in the scanned set.  Per row: dual, assigned column, and the rows of the current search in visiting order.
struct Cols {
  double* shortest;
  double* v;
  int* path;
  int* row4col;
  uint8_t* in_sc;
};
struct Rows {
  double* u;
  int* col4row;
  int* visited;
};

// cost(i, j) = c[i * rs + j * cs] of a float matrix, promoted to double like scipy does
struct Strided {
  const float* c;
  size_t rs, cs;
  HD_FORCEINLINE double operator()(int i, int j) const { return double(c[size_t(i) * rs + size_t(j) * cs]); }
};

// Assigns each of nr rows a distinct one of nc >= nr columns at minimum total cost(i, j) (a double).  Fills
// R.col4row and C.row4col.  Returns false, on every thread of the group, when some row reaches no column below
// DBL_MAX (non-finite costs); the assignment is then incomplete.  Every thread of the group calls it.  Column j is
// scanned by thread j % kSize throughout, so only that thread ever touches in_sc[j].
template <class G, class Cost>
HD_FORCEINLINE bool solve(int nr, int nc, const Cost& cost, const Rows& R, const Cols& C,
                          typename G::Scratch& scratch) {
  const int t = G::rank(), nt = G::kSize;
  for (int j = t; j < nc; j += nt) { C.v[j] = 0.0; C.row4col[j] = -1; }
  for (int i = t; i < nr; i += nt) { R.u[i] = 0.0; R.col4row[i] = -1; }
  G::sync();
  for (int cur = 0; cur < nr; ++cur) {
    // path[j] needs no reset: a column enters the scanned set only once shortest[j] < DBL_MAX, which sets it
    for (int j = t; j < nc; j += nt) { C.shortest[j] = DBL_MAX; C.in_sc[j] = 0; }
    int i = cur, sink = -1, nvis = 0;
    double min_val = 0.0;
    while (sink == -1) {
      if (t == 0) R.visited[nvis] = i;
      ++nvis;
      const double ui = R.u[i];
      Key best{DBL_MAX, 1, INT32_MAX};
      for (int j = t; j < nc; j += nt) {
        if (C.in_sc[j]) continue;
        const double r = min_val + cost(i, j) - ui - C.v[j];
        if (r < C.shortest[j]) { C.shortest[j] = r; C.path[j] = i; }
        const Key k{C.shortest[j], C.row4col[j] == -1 ? 0 : 1, j};
        if (better(k, best)) best = k;
      }
      best = G::min(best, scratch);
      if (best.val == DBL_MAX || best.idx == INT32_MAX) return false;
      if (best.idx % nt == t) C.in_sc[best.idx] = 1;
      min_val = best.val;
      if (C.row4col[best.idx] == -1) sink = best.idx;
      else i = C.row4col[best.idx];
    }
    // ---- dual update
    for (int k = t; k < nvis; k += nt) {
      const int r = R.visited[k];
      if (r == cur) R.u[r] += min_val;
      else R.u[r] += min_val - C.shortest[R.col4row[r]];
    }
    for (int j = t; j < nc; j += nt)
      if (C.in_sc[j]) C.v[j] -= min_val - C.shortest[j];
    G::sync();
    // ---- augment along the path (at most nvis hops)
    if (t == 0) {
      for (int j = sink;;) {
        const int r = C.path[j];
        C.row4col[j] = r;
        const int prev = R.col4row[r];
        R.col4row[r] = j;
        j = prev;
        if (r == cur) break;
      }
    }
    G::sync();
  }
  return true;
}

}  // namespace tfb200_lsa
