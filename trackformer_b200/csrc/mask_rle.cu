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
//
// tfb200_mask_rle_batched_i32 runs the same nine launches over up to 16 maps: every stage's grid covers the items
// (tracks, tiles, chunks) of all maps, and a CTA or warp finds its map in prefix tables passed by value.  Tracks are
// numbered map after map, so steps 5 and 8 scan all of them at once into one boundary array and one header;
// tfb200_mask_rle_i32 is the case of one map.
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
constexpr int kMaxBatch = 16;             // maps per call

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

// The maps of one call.  Map b owns the global tracks [t_end[b - 1], t_end[b]), the classify tiles [tile_end[b - 1],
// tile_end[b]) and the event chunks [chunk_end[b - 1], chunk_end[b]); its hash table, column-major track indices and
// chunk counts start at hash_off / pix_off / count_off.  A map with T == 0 owns no track, tile or chunk.  Track and chunk indices
// inside a map are the single-map pipeline's, so each stage runs the single-map body on the map it finds.
// kCap is the table's capacity: 1 for a single map (the launch then carries a one-entry table and finds its map at
// compile time), kMaxBatch otherwise.
template <int kCap>
struct RleBatch {
  const int32_t* label[kCap];
  const int32_t* ids[kCap];
  int64_t pix_off[kCap];
  int64_t count_off[kCap];
  int H[kCap], W[kCap];
  int t_end[kCap], tile_end[kCap], chunk_end[kCap];
  int hash_off[kCap], hash_mask[kCap], n_chunks[kCap], tiles_x[kCap];
};

// the map owning item v of a prefix `end` (v < end[kCap - 1])
template <int kCap>
__device__ __forceinline__ int map_of(const int* end, int v) {
  int b = 0;
  if (kCap > 1)
    while (v >= end[b]) ++b;
  return b;
}

__device__ __forceinline__ int begin_of(const int* end, int b) { return b ? end[b - 1] : 0; }

// ---- 1. ids -> lowest list position within the map (status bit 1: a negative id)
template <int kCap>
__global__ void rle_hash_kernel(const __grid_constant__ RleBatch<kCap> m, int T, int* keys, int* vals,
                                unsigned long long* status) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= T) return;
  const int b = map_of<kCap>(m.t_end, g), t = g - begin_of(m.t_end, b);
  const int id = m.ids[b][t];
  if (id < 0) {
    atomicOr(status, 1ull);
    return;
  }
  const int mask = m.hash_mask[b];
  keys += m.hash_off[b];
  vals += m.hash_off[b];
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

// ---- 2. row-major label map -> column-major track index within the map (-1: no track)
template <int kCap>
__global__ void __launch_bounds__(kTile * 8)
rle_classify_kernel(const __grid_constant__ RleBatch<kCap> m, const int* __restrict__ keys, const int* __restrict__ vals,
                    int* __restrict__ tcm) {
  __shared__ int tile[kTile][kTile + 1];
  const int b = map_of<kCap>(m.tile_end, blockIdx.x), i = blockIdx.x - begin_of(m.tile_end, b);
  const int H = m.H[b], W = m.W[b], mask = m.hash_mask[b];
  const int32_t* __restrict__ label = m.label[b];
  keys += m.hash_off[b];
  vals += m.hash_off[b];
  tcm += m.pix_off[b];
  const int x0 = (i % m.tiles_x[b]) * kTile, y0 = (i / m.tiles_x[b]) * kTile;
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

// ---- 3 / 6. boundary events of one chunk per warp.  counts[t * n_chunks + c] of the chunk's map: pass 3 counts, pass
// 6 consumes them as running offsets (after step 4 made them exclusive prefixes) and writes bnd[tbase[t] + offset].
template <bool kWrite, int kCap>
__global__ void __launch_bounds__(32 * kEventWarps)
rle_events_kernel(const __grid_constant__ RleBatch<kCap> m, int total_chunks, const int* __restrict__ tcm, int* counts,
                  const int* __restrict__ tbase, int* __restrict__ bnd) {
  const int lane = threadIdx.x & 31;
  const int cg = blockIdx.x * kEventWarps + (threadIdx.x >> 5);
  if (cg >= total_chunks) return;           // whole warps leave together
  const int b = map_of<kCap>(m.chunk_end, cg), c = cg - begin_of(m.chunk_end, b);
  const int N = m.H[b] * m.W[b], n_chunks = m.n_chunks[b];
  tcm += m.pix_off[b];
  counts += m.count_off[b];
  if (kWrite) tbase += begin_of(m.t_end, b);
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
      const unsigned msk = __ballot_sync(0xffffffffu, in_a || in_b);
      int* slot = counts + int64_t(X) * n_chunks + c;
      const int before = *slot;
      if (kWrite && (in_a || in_b)) bnd[tbase[X] + before + __popc(msk & lt)] = p;
      __syncwarp();
      if (lane == 0) *slot = before + __popc(msk);
      __syncwarp();
      need_a = need_a && !in_a;
      need_b = need_b && !in_b;
    }
  }
}

// ---- 4. per track: exclusive scan of its chunk counts; also its list's owner (lowest t of the same id in its map)
template <int kCap>
__global__ void __launch_bounds__(kThreads)
rle_track_scan_kernel(const __grid_constant__ RleBatch<kCap> m, const int* __restrict__ keys, const int* __restrict__ vals,
                      int* counts, int* __restrict__ nb, int* __restrict__ rep) {
  __shared__ long long ws[kThreads / 32];
  const int g = blockIdx.x;
  const int b = map_of<kCap>(m.t_end, g), t0 = begin_of(m.t_end, b), t = g - t0;
  const int n_chunks = m.n_chunks[b];
  int* row = counts + m.count_off[b] + int64_t(t) * n_chunks;
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
    nb[g] = int(carry);
    const int r = lookup(keys + m.hash_off[b], vals + m.hash_off[b], m.ids[b][t], m.hash_mask[b]);
    rep[g] = t0 + (r < 0 ? t : r);          // a negative id has no list (status bit 1 reports it)
  }
}

// ---- 5 / 8. exclusive scan over all tracks (one block).  5: int boundary counts -> list starts.  8: int64 string
// lengths -> header {status, total, offsets[T], lengths[T]}; status bit 2 when the total exceeds the character buffer.
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
template <bool kWrite, int kCap>
__global__ void __launch_bounds__(kThreads)
rle_chars_kernel(const __grid_constant__ RleBatch<kCap> m, const int* __restrict__ bnd, const int* __restrict__ tbase,
                 const int* __restrict__ nb, const int* __restrict__ rep, long long* __restrict__ len,
                 const long long* __restrict__ header, long long capacity, char* __restrict__ chars) {
  __shared__ long long ws[kThreads / 32];
  const int t = blockIdx.x;
  const int mb = map_of<kCap>(m.t_end, t);
  const int N = m.H[mb] * m.W[mb];
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
  int T, slots, tiles, chunks;
};

bool bad_shape(int H, int W, int T) {
  return H <= 0 || W <= 0 || T < 0 || T > (1 << 24) || int64_t(H) * W > (int64_t(1) << 28);
}

// Checks the maps (TFB200_E_SHAPE for any bad one, or for sum 2 H W >= 2^31) and lays the workspace out: each region
// holds the maps' parts back to back, so one map lays out exactly as the single-map pipeline always has.
int plan(const TfbMaskRleMap* maps, int n, RleBatch<kMaxBatch>* m, Layout* l) {
  if (n <= 0 || n > kMaxBatch) return TFB200_E_SHAPE;
  int64_t T = 0, S = 0, N = 0, counts = 0, tiles = 0, chunks = 0, all_pixels = 0;
  for (int b = 0; b < n; ++b) {
    const TfbMaskRleMap& a = maps[b];
    if (bad_shape(a.H, a.W, a.T)) return TFB200_E_SHAPE;
    all_pixels += int64_t(a.H) * a.W;
    const bool on = a.T > 0;                // a map without tracks keeps its regions but owns no tiles or chunks
    const int64_t pixels = int64_t(a.H) * a.W, n_chunks = (pixels + kChunk - 1) / kChunk;
    const int slots = hash_slots(a.T);
    m->label[b] = a.label;
    m->ids[b] = a.ids;
    m->H[b] = a.H;
    m->W[b] = a.W;
    m->hash_off[b] = int(S);
    m->hash_mask[b] = slots - 1;
    m->pix_off[b] = N;
    m->count_off[b] = counts;
    m->n_chunks[b] = int(n_chunks);
    m->tiles_x[b] = (a.W + kTile - 1) / kTile;
    T += a.T;
    S += slots;
    N += pixels;
    counts += int64_t(a.T) * n_chunks;
    chunks += on ? n_chunks : 0;
    tiles += on ? int64_t(m->tiles_x[b]) * ((a.H + kTile - 1) / kTile) : 0;
    m->t_end[b] = int(T);
    m->chunk_end[b] = int(chunks);
    m->tile_end[b] = int(tiles);
  }
  if (2 * all_pixels >= (int64_t(1) << 31) || T > (1 << 24)) return TFB200_E_SHAPE;
  for (int b = n; b < kMaxBatch; ++b) {
    m->t_end[b] = int(T);
    m->chunk_end[b] = int(chunks);
    m->tile_end[b] = int(tiles);
  }
  size_t o = 0;
  l->keys = o;   o += align256(size_t(S) * 4);
  l->vals = o;   o += align256(size_t(S) * 4);
  l->rep = o;    o += align256(size_t(T) * 4);
  l->nb = o;     o += align256(size_t(T) * 4);
  l->tbase = o;  o += align256(size_t(T) * 4);
  l->len = o;    o += align256(size_t(T) * 8);
  l->counts = o; o += align256(size_t(counts) * 4);
  l->tcm = o;    o += align256(size_t(N) * 4);
  l->bnd = o;    o += align256(2 * size_t(N) * 4);       // each pixel ends at most one run and starts at most one
  l->total = o;
  l->T = int(T);
  l->slots = int(S);
  l->tiles = int(tiles);
  l->chunks = int(chunks);
  return 0;
}

// characters of all strings of one H x W map with T tracks, at most
int64_t max_bytes(int H, int W, int T) {
  const int64_t N = int64_t(H) * W;
  int per = 1;                              // characters of any |difference| <= N: 2^(5 per - 1) > N
  while ((int64_t(1) << (5 * per - 1)) <= N) ++per;
  return per * (2 * N + T);                 // at most 2N boundaries over all tracks, k + 1 counts per track
}

// the nine launches of one call (after the four memsets)
template <int kCap>
void launch_stages(const RleBatch<kCap>& m, const Layout& l, int T, int* keys, int* vals, int* rep, int* nb,
                   int* tbase, long long* len, int* counts, int* tcm, int* bnd, long long* hdr, char* chars,
                   int64_t chars_capacity, cudaStream_t s) {
  rle_hash_kernel<kCap><<<(T + 255) / 256, 256, 0, s>>>(m, T, keys, vals, reinterpret_cast<unsigned long long*>(hdr));
  rle_classify_kernel<kCap><<<l.tiles, dim3(kTile, 8), 0, s>>>(m, keys, vals, tcm);
  const int event_blocks = (l.chunks + kEventWarps - 1) / kEventWarps;
  rle_events_kernel<false, kCap><<<event_blocks, 32 * kEventWarps, 0, s>>>(m, l.chunks, tcm, counts, nullptr, nullptr);
  rle_track_scan_kernel<kCap><<<T, kThreads, 0, s>>>(m, keys, vals, counts, nb, rep);
  rle_scan_tracks_kernel<<<1, kThreads, 0, s>>>(nb, tbase, nullptr, nullptr, T, 0);
  rle_events_kernel<true, kCap><<<event_blocks, 32 * kEventWarps, 0, s>>>(m, l.chunks, tcm, counts, tbase, bnd);
  rle_chars_kernel<false, kCap><<<T, kThreads, 0, s>>>(m, bnd, tbase, nb, rep, len, nullptr, 0, nullptr);
  rle_scan_tracks_kernel<<<1, kThreads, 0, s>>>(nullptr, nullptr, len, hdr, T, chars_capacity);
  rle_chars_kernel<true, kCap><<<T, kThreads, 0, s>>>(m, bnd, tbase, nb, rep, nullptr, hdr, chars_capacity, chars);
}

}  // namespace

extern "C" size_t tfb200_mask_rle_batched_workspace_bytes(const TfbMaskRleMap* maps, int n) {
  RleBatch<kMaxBatch> m;
  Layout l;
  return maps && plan(maps, n, &m, &l) == 0 ? l.total : 0;
}

extern "C" int64_t tfb200_mask_rle_batched_max_bytes(const TfbMaskRleMap* maps, int n) {
  RleBatch<kMaxBatch> m;
  Layout l;
  if (!maps || plan(maps, n, &m, &l) != 0) return 0;
  int64_t total = 0;
  for (int b = 0; b < n; ++b) total += maps[b].T > 0 ? max_bytes(maps[b].H, maps[b].W, maps[b].T) : 0;
  return total;
}

extern "C" size_t tfb200_mask_rle_workspace_bytes(int H, int W, int T) {
  const TfbMaskRleMap map = {nullptr, nullptr, H, W, T};
  return tfb200_mask_rle_batched_workspace_bytes(&map, 1);
}

extern "C" int64_t tfb200_mask_rle_max_bytes(int H, int W, int T) {
  return bad_shape(H, W, T) ? 0 : max_bytes(H, W, T);
}

extern "C" int tfb200_mask_rle_batched_i32(const TfbMaskRleMap* maps, int n, void* workspace, size_t workspace_bytes,
                                           int64_t* header, char* chars, int64_t chars_capacity, void* stream) {
  if (!maps || !workspace || !header || !chars) return TFB200_E_NULLPTR;
  if (n <= 0 || n > kMaxBatch) return TFB200_E_SHAPE;
  for (int b = 0; b < n; ++b)
    if (!maps[b].label || !maps[b].ids) return TFB200_E_NULLPTR;
  RleBatch<kMaxBatch> m;
  Layout l;
  if (const int rc = plan(maps, n, &m, &l)) return rc;
  if (chars_capacity < 0) return TFB200_E_SHAPE;
  const int T = l.T;
  if (T == 0) return 0;
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

  cudaError_t e;
  if ((e = cudaMemsetAsync(keys, 0xff, size_t(l.slots) * 4, s)) != cudaSuccess) return int(e);   // kEmpty
  if ((e = cudaMemsetAsync(vals, 0x7f, size_t(l.slots) * 4, s)) != cudaSuccess) return int(e);   // > any t (atomicMin)
  if ((e = cudaMemsetAsync(counts, 0, l.tcm - l.counts, s)) != cudaSuccess) return int(e);
  if ((e = cudaMemsetAsync(hdr, 0, sizeof(long long), s)) != cudaSuccess) return int(e);
  if (n == 1) {
    RleBatch<1> one;
    one.label[0] = m.label[0];
    one.ids[0] = m.ids[0];
    one.pix_off[0] = m.pix_off[0];
    one.count_off[0] = m.count_off[0];
    one.H[0] = m.H[0];
    one.W[0] = m.W[0];
    one.t_end[0] = m.t_end[0];
    one.tile_end[0] = m.tile_end[0];
    one.chunk_end[0] = m.chunk_end[0];
    one.hash_off[0] = m.hash_off[0];
    one.hash_mask[0] = m.hash_mask[0];
    one.n_chunks[0] = m.n_chunks[0];
    one.tiles_x[0] = m.tiles_x[0];
    launch_stages(one, l, T, keys, vals, rep, nb, tbase, len, counts, tcm, bnd, hdr, chars, chars_capacity, s);
  } else {
    launch_stages(m, l, T, keys, vals, rep, nb, tbase, len, counts, tcm, bnd, hdr, chars, chars_capacity, s);
  }
  msda_b200_count_launches(9);
  return int(cudaGetLastError());
}

extern "C" int tfb200_mask_rle_i32(const int32_t* label, const int32_t* ids, int H, int W, int T, void* workspace,
                                   size_t workspace_bytes, int64_t* header, char* chars, int64_t chars_capacity,
                                   void* stream) {
  const TfbMaskRleMap map = {label, ids, H, W, T};
  return tfb200_mask_rle_batched_i32(&map, 1, workspace, workspace_bytes, header, chars, chars_capacity, stream);
}
