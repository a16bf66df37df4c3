// COCO run-length encodings of the tracker's per-track masks, straight from the device label map (sm_90a).
//
// Reference: the result writer of MOTS20 (datasets/tracking/mots20_sequence.py:72-91) calls pycocotools
// `mask.encode(np.asfortranarray(label == id))` on one full-size host bool array per track and frame.  Here the strings
// are made on the device from the int32 label map that csrc/track_masks.cu writes, so only the strings leave it.
//
// The mask of track t is label == ids[t].  Its runs alternate in column-major order (p = x * H + y), starting with the
// zero run (length 0 if pixel 0 is set); the last run is always written; an empty mask is the single count H * W.  A
// count becomes characters as in pycocotools rleToString: x = cnts[i] - (i > 2 ? cnts[i - 2] : 0), then 5-bit groups,
// least significant first, bit 0x20 set while more follow (arithmetic shift; a group with bit 0x10 ends at x == -1),
// plus 48.
//
// Pipeline (nine launches, all deterministic: a position's place in a track's list is a rank, never an atomic's turn):
//   1. hash ids -> lowest t holding that id (duplicate ids share one boundary list and get equal strings)
//   2. label map -> track index per pixel, transposed to column-major through a shared-memory tile
//   3. one warp per chunk of kChunk positions: boundary events (the track index differs from the previous pixel's), a
//      boundary of track a and of track b; count them per (track, chunk)
//   4. per track: exclusive scan of its chunk counts -> its boundary count
//   5. exclusive scan of the boundary counts over tracks -> where each track's boundary list starts
//   6. the warp of step 3 again, writing each boundary at its rank: within a chunk, the lanes of one 32-position step
//      that touch track X are ranked by lane (= position) order, and steps run in position order
//   7. per track: characters of its counts -> its string length
//   8. exclusive scan of the lengths -> the header (status, total bytes, offsets, lengths)
//   9. per track: characters written at their offsets (a block scan of the per-count character counts)
// Buffers are sized for the worst case (every pixel a boundary of two tracks: 2 H W boundaries); a character buffer
// smaller than the total is reported in the header's status, never truncated.
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "launch_counter.h"

namespace {

constexpr int kChunk = 2048;              // positions per warp in the event passes
constexpr int kEventWarps = 4;            // warps (chunks) per block there
constexpr int kTile = 32;                 // transpose tile
constexpr int kThreads = 256;             // per-track and scan kernels
constexpr int kEmpty = -1;                // free hash slot (ids are >= 0)

__device__ __forceinline__ unsigned slot_of(int id, int mask) {
  unsigned x = unsigned(id);
  x = (x ^ (x >> 16)) * 0x45d9f3bu;
  x = (x ^ (x >> 16)) * 0x45d9f3bu;
  return (x ^ (x >> 16)) & unsigned(mask);
}

__device__ __forceinline__ int lookup(const int* __restrict__ keys, const int* __restrict__ vals, int id, int mask) {
  if (id < 0) return -1;
  unsigned s = slot_of(id, mask);
  while (true) {
    const int k = __ldg(keys + s);
    if (k == id) return __ldg(vals + s);
    if (k == kEmpty) return -1;
    s = (s + 1) & unsigned(mask);
  }
}

// characters of one count difference (pycocotools rleToString)
__device__ __forceinline__ int rle_chars(long long x) {
  int n = 0;
  bool more = true;
  while (more) {
    const long long c = x & 0x1f;
    x >>= 5;
    more = (c & 0x10) ? x != -1 : x != 0;
    ++n;
  }
  return n;
}

// exclusive scan over the block (blockDim.x == kThreads); returns the prefix, *total the block's sum
__device__ __forceinline__ long long block_excl_scan(long long v, long long* warp_sums, long long* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  long long inc = v;
#pragma unroll
  for (int d = 1; d < 32; d <<= 1) {
    const long long o = __shfl_up_sync(0xffffffffu, inc, d);
    if (lane >= d) inc += o;
  }
  __syncthreads();                          // warp_sums free from any previous use
  if (lane == 31) warp_sums[warp] = inc;
  __syncthreads();
  long long before = 0, sum = 0;
#pragma unroll
  for (int w = 0; w < kThreads / 32; ++w) {
    const long long s = warp_sums[w];
    before += w < warp ? s : 0;
    sum += s;
  }
  *total = sum;
  return before + inc - v;
}

// ---- 1. ids -> lowest list position (status bit 1: a negative id)
__global__ void rle_hash_kernel(const int32_t* __restrict__ ids, int T, int* keys, int* vals, int mask,
                                unsigned long long* status) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  const int id = ids[t];
  if (id < 0) {
    atomicOr(status, 1ull);
    return;
  }
  unsigned s = slot_of(id, mask);
  while (true) {
    const int old = atomicCAS(keys + s, kEmpty, id);
    if (old == kEmpty || old == id) {
      atomicMin(vals + s, t);
      return;
    }
    s = (s + 1) & unsigned(mask);
  }
}

// ---- 2. row-major label map -> column-major track index (-1: no track)
__global__ void __launch_bounds__(kTile * 8)
rle_classify_kernel(const int32_t* __restrict__ label, const int* __restrict__ keys, const int* __restrict__ vals,
                    int mask, int* __restrict__ tcm, int H, int W) {
  __shared__ int tile[kTile][kTile + 1];
  const int x0 = blockIdx.x * kTile, y0 = blockIdx.y * kTile;
  const int tx = threadIdx.x, ty = threadIdx.y;
#pragma unroll
  for (int r = 0; r < kTile; r += 8) {
    const int y = y0 + ty + r, x = x0 + tx;
    if (y < H && x < W) tile[ty + r][tx] = lookup(keys, vals, label[int64_t(y) * W + x], mask);
  }
  __syncthreads();
#pragma unroll
  for (int r = 0; r < kTile; r += 8) {
    const int x = x0 + ty + r, y = y0 + tx;
    if (y < H && x < W) tcm[int64_t(x) * H + y] = tile[tx][ty + r];
  }
}

// ---- 3 / 6. boundary events of one chunk per warp.  counts[t * n_chunks + c]: pass 3 counts, pass 6 consumes them as
// running offsets (after step 4 made them exclusive prefixes) and writes bnd[tbase[t] + offset].
template <bool kWrite>
__global__ void __launch_bounds__(32 * kEventWarps)
rle_events_kernel(const int* __restrict__ tcm, int N, int n_chunks, int* counts, const int* __restrict__ tbase,
                  int* __restrict__ bnd) {
  const int lane = threadIdx.x & 31;
  const int c = blockIdx.x * kEventWarps + (threadIdx.x >> 5);
  if (c >= n_chunks) return;                // whole warps leave together
  const unsigned lt = (1u << lane) - 1u;
  const int end = min(N, (c + 1) * kChunk);
  for (int p0 = c * kChunk; p0 < end; p0 += 32) {
    const int p = p0 + lane;
    const int cur = p < end ? tcm[p] : -1;
    const int prev = p == 0 ? -1 : (p < end ? tcm[p - 1] : -1);
    const bool ev = p < end && cur != prev;
    bool need_a = ev && prev >= 0, need_b = ev && cur >= 0;   // prev's run ends at p, cur's starts at p
    while (true) {
      const unsigned pa = __ballot_sync(0xffffffffu, need_a), pb = __ballot_sync(0xffffffffu, need_b);
      if (!(pa | pb)) break;
      const int src = pa ? __ffs(pa) - 1 : __ffs(pb) - 1;
      const int ka = __shfl_sync(0xffffffffu, prev, src), kb = __shfl_sync(0xffffffffu, cur, src);
      const int X = pa ? ka : kb;
      const bool in_a = need_a && prev == X, in_b = need_b && cur == X;   // at most one: prev != cur
      const unsigned m = __ballot_sync(0xffffffffu, in_a || in_b);
      int* slot = counts + int64_t(X) * n_chunks + c;
      const int before = *slot;
      if (kWrite && (in_a || in_b)) bnd[tbase[X] + before + __popc(m & lt)] = p;
      __syncwarp();
      if (lane == 0) *slot = before + __popc(m);
      __syncwarp();
      need_a = need_a && !in_a;
      need_b = need_b && !in_b;
    }
  }
}

// ---- 4. per track: exclusive scan of its chunk counts; also its list's owner (lowest t of the same id)
__global__ void __launch_bounds__(kThreads)
rle_track_scan_kernel(const int32_t* __restrict__ ids, const int* __restrict__ keys, const int* __restrict__ vals,
                      int mask, int* counts, int n_chunks, int* __restrict__ nb, int* __restrict__ rep) {
  __shared__ long long ws[kThreads / 32];
  const int t = blockIdx.x;
  int* row = counts + int64_t(t) * n_chunks;
  long long carry = 0;
  for (int i0 = 0; i0 < n_chunks; i0 += kThreads) {
    const int i = i0 + threadIdx.x;
    const int v = i < n_chunks ? row[i] : 0;
    long long total;
    const long long e = block_excl_scan(v, ws, &total);
    if (i < n_chunks) row[i] = int(carry + e);
    carry += total;
  }
  if (threadIdx.x == 0) {
    nb[t] = int(carry);
    const int r = lookup(keys, vals, ids[t], mask);
    rep[t] = r < 0 ? t : r;                 // a negative id has no list (status bit 1 reports it)
  }
}

// ---- 5 / 8. exclusive scan over tracks (one block).  5: int boundary counts -> list starts.  8: int64 string lengths
// -> header {status, total, offsets[T], lengths[T]}; status bit 2 when the total exceeds the character buffer.
__global__ void __launch_bounds__(kThreads)
rle_scan_tracks_kernel(const int* __restrict__ nb, int* __restrict__ tbase, const long long* __restrict__ len,
                       long long* __restrict__ header, int T, long long capacity) {
  __shared__ long long ws[kThreads / 32];
  long long carry = 0;
  for (int i0 = 0; i0 < T; i0 += kThreads) {
    const int i = i0 + threadIdx.x;
    const long long v = i < T ? (len ? len[i] : nb[i]) : 0;
    long long total;
    const long long e = block_excl_scan(v, ws, &total);
    if (i < T) {
      if (len) {
        header[2 + i] = carry + e;
        header[2 + T + i] = v;
      } else {
        tbase[i] = int(carry + e);
      }
    }
    carry += total;
  }
  if (len && threadIdx.x == 0) {
    header[1] = carry;
    if (carry > capacity) header[0] |= 2;
  }
}

// count i of a track whose k ascending boundaries are b[0..k): runs between 0, the boundaries and N
__device__ __forceinline__ long long run_count(const int* b, int k, int N, int i) {
  return (long long)(i < k ? b[i] : N) - (i > 0 ? b[i - 1] : 0);
}

__device__ __forceinline__ long long count_diff(const int* b, int k, int N, int i) {
  return run_count(b, k, N, i) - (i > 2 ? run_count(b, k, N, i - 2) : 0);
}

// ---- 7 / 9. per track: 7 sums the characters of its k + 1 counts; 9 writes them at header offsets
template <bool kWrite>
__global__ void __launch_bounds__(kThreads)
rle_chars_kernel(const int* __restrict__ bnd, const int* __restrict__ tbase, const int* __restrict__ nb,
                 const int* __restrict__ rep, int N, long long* __restrict__ len, const long long* __restrict__ header,
                 int T, long long capacity, char* __restrict__ chars) {
  __shared__ long long ws[kThreads / 32];
  const int t = blockIdx.x;
  const int r = rep[t];
  const int k = nb[r];
  const int* b = bnd + tbase[r];
  if (kWrite && header[1] > capacity) return;             // reported in the header's status
  char* out = kWrite ? chars + header[2 + t] : nullptr;
  long long carry = 0;
  for (int i0 = 0; i0 <= k; i0 += kThreads) {
    const int i = i0 + threadIdx.x;
    long long x = 0;
    int n = 0;
    if (i <= k) {
      x = count_diff(b, k, N, i);
      n = rle_chars(x);
    }
    long long total;
    const long long e = block_excl_scan(n, ws, &total);
    if (kWrite && i <= k) {
      char* o = out + carry + e;
      bool more = true;
      while (more) {
        long long c = x & 0x1f;
        x >>= 5;
        more = (c & 0x10) ? x != -1 : x != 0;
        if (more) c |= 0x20;
        *o++ = char(c + 48);
      }
    }
    carry += total;
  }
  if (!kWrite && threadIdx.x == 0) len[t] = carry;
}

size_t align256(size_t v) { return (v + 255) & ~size_t(255); }

int hash_slots(int T) {
  int p = 64;
  while (p < 2 * T) p <<= 1;
  return p;
}

struct Layout {
  size_t keys, vals, rep, nb, tbase, len, counts, tcm, bnd, total;
};

Layout layout(int H, int W, int T) {
  const size_t N = size_t(H) * W, S = size_t(hash_slots(T)), n_chunks = (N + kChunk - 1) / kChunk;
  Layout l;
  size_t o = 0;
  l.keys = o;   o += align256(S * 4);
  l.vals = o;   o += align256(S * 4);
  l.rep = o;    o += align256(size_t(T) * 4);
  l.nb = o;     o += align256(size_t(T) * 4);
  l.tbase = o;  o += align256(size_t(T) * 4);
  l.len = o;    o += align256(size_t(T) * 8);
  l.counts = o; o += align256(size_t(T) * n_chunks * 4);
  l.tcm = o;    o += align256(N * 4);
  l.bnd = o;    o += align256(2 * N * 4);               // each pixel ends at most one run and starts at most one
  l.total = o;
  return l;
}

bool bad_shape(int H, int W, int T) {
  return H <= 0 || W <= 0 || T < 0 || T > (1 << 24) || int64_t(H) * W > (int64_t(1) << 28);
}

}  // namespace

extern "C" size_t tfb200_mask_rle_workspace_bytes(int H, int W, int T) {
  return bad_shape(H, W, T) ? 0 : layout(H, W, T).total;
}

extern "C" int64_t tfb200_mask_rle_max_bytes(int H, int W, int T) {
  if (bad_shape(H, W, T)) return 0;
  const int64_t N = int64_t(H) * W;
  int per = 1;                              // characters of any |difference| <= N: 2^(5 per - 1) > N
  while ((int64_t(1) << (5 * per - 1)) <= N) ++per;
  return per * (2 * N + T);                 // at most 2N boundaries over all tracks, k + 1 counts per track
}

extern "C" int tfb200_mask_rle_i32(const int32_t* label, const int32_t* ids, int H, int W, int T, void* workspace,
                                   size_t workspace_bytes, int64_t* header, char* chars, int64_t chars_capacity,
                                   void* stream) {
  if (!label || !ids || !workspace || !header || !chars) return TFB200_E_NULLPTR;
  if (bad_shape(H, W, T) || chars_capacity < 0) return TFB200_E_SHAPE;
  if (T == 0) return 0;
  const Layout l = layout(H, W, T);
  if (workspace_bytes < l.total) return TFB200_E_SHAPE;
  const cudaStream_t s = cudaStream_t(stream);
  char* ws = static_cast<char*>(workspace);
  int* keys = reinterpret_cast<int*>(ws + l.keys);
  int* vals = reinterpret_cast<int*>(ws + l.vals);
  int* rep = reinterpret_cast<int*>(ws + l.rep);
  int* nb = reinterpret_cast<int*>(ws + l.nb);
  int* tbase = reinterpret_cast<int*>(ws + l.tbase);
  long long* len = reinterpret_cast<long long*>(ws + l.len);
  int* counts = reinterpret_cast<int*>(ws + l.counts);
  int* tcm = reinterpret_cast<int*>(ws + l.tcm);
  int* bnd = reinterpret_cast<int*>(ws + l.bnd);
  long long* hdr = reinterpret_cast<long long*>(header);
  const int N = H * W, S = hash_slots(T), n_chunks = (N + kChunk - 1) / kChunk;

  cudaError_t e;
  if ((e = cudaMemsetAsync(keys, 0xff, size_t(S) * 4, s)) != cudaSuccess) return int(e);     // kEmpty
  if ((e = cudaMemsetAsync(vals, 0x7f, size_t(S) * 4, s)) != cudaSuccess) return int(e);     // > any t (atomicMin)
  if ((e = cudaMemsetAsync(counts, 0, size_t(T) * n_chunks * 4, s)) != cudaSuccess) return int(e);
  if ((e = cudaMemsetAsync(hdr, 0, sizeof(long long), s)) != cudaSuccess) return int(e);
  rle_hash_kernel<<<(T + 255) / 256, 256, 0, s>>>(ids, T, keys, vals, S - 1,
                                                 reinterpret_cast<unsigned long long*>(hdr));
  rle_classify_kernel<<<dim3((W + kTile - 1) / kTile, (H + kTile - 1) / kTile), dim3(kTile, 8), 0, s>>>(
      label, keys, vals, S - 1, tcm, H, W);
  const int event_blocks = (n_chunks + kEventWarps - 1) / kEventWarps;
  rle_events_kernel<false><<<event_blocks, 32 * kEventWarps, 0, s>>>(tcm, N, n_chunks, counts, nullptr, nullptr);
  rle_track_scan_kernel<<<T, kThreads, 0, s>>>(ids, keys, vals, S - 1, counts, n_chunks, nb, rep);
  rle_scan_tracks_kernel<<<1, kThreads, 0, s>>>(nb, tbase, nullptr, nullptr, T, 0);
  rle_events_kernel<true><<<event_blocks, 32 * kEventWarps, 0, s>>>(tcm, N, n_chunks, counts, tbase, bnd);
  rle_chars_kernel<false><<<T, kThreads, 0, s>>>(bnd, tbase, nb, rep, N, len, nullptr, T, 0, nullptr);
  rle_scan_tracks_kernel<<<1, kThreads, 0, s>>>(nullptr, nullptr, len, hdr, T, chars_capacity);
  rle_chars_kernel<true><<<T, kThreads, 0, s>>>(bnd, tbase, nb, rep, N, nullptr, hdr, T, chars_capacity, chars);
  msda_b200_count_launches(9);
  return int(cudaGetLastError());
}
