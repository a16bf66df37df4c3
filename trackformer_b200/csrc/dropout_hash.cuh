// Counter-based keep decision of the mask-free inverted dropout used by every fused dropout site: a hash of
// (per-call seed, logical element index) compared against floor(keep_prob * 2^32).  One definition, so that every
// kernel that fuses a dropout draws the same mask for the same (seed, index) -- tests/dropout_hash.py restates it.
#pragma once

#include <stdint.h>

namespace tfb200 {

__device__ __forceinline__ uint32_t mix32(uint32_t x) {
  x ^= x >> 16; x *= 0x7feb352du; x ^= x >> 15; x *= 0x846ca68bu; x ^= x >> 16;
  return x;
}

__device__ __forceinline__ bool keep_elem(uint64_t seed, uint64_t idx, uint32_t keep_thresh) {
  const uint32_t h = mix32(uint32_t(idx) ^ mix32(uint32_t(idx >> 32) + uint32_t(seed)) ^ uint32_t(seed >> 32) * 0x9e3779b9u);
  return h < keep_thresh;
}

// floor(keep_prob * 2^32), saturating: keep_prob = 1 keeps every element
inline uint32_t keep_threshold(float keep_prob) {
  const double t = double(keep_prob) * 4294967296.0;
  return t >= 4294967295.0 ? 0xFFFFFFFFu : uint32_t(t);
}

}  // namespace tfb200
