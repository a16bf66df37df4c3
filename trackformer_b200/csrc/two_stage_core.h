// Two-stage Deformable DETR (src/trackformer/models/deformable_transformer.py:77-122, 180-194): encoder proposals and
// top-k query selection, written once as cooperative routines:
//
//   ts_valid_counts  (per image)   unpadded width / height of every level: the first row / column of its padding mask
//   ts_proposal      (per token)   level, (cx, cy, w, h) = ((x+.5)/valid_W, (y+.5)/valid_H, .05*2^l, .05*2^l), the valid
//                                  flag (all four in (0.01, 0.99), token not padded) and log(p / (1 - p)), +inf if invalid
//   ts_select        (per image)   the k largest class-0 logits over the S tokens, by a 4 x 8-bit radix select over the
//                                  order-preserving 32-bit key of the logit (no S-sized buffer in shared memory), ties at
//                                  the threshold taken in token order, the k winners sorted by (logit desc, token asc)
//   ts_select_outputs(per image)   the gathered (detached) unactivated boxes, their sigmoid (reference points) and the
//                                  512-wide sine embedding of get_proposal_pos_embed
//
// nvcc compiles them into csrc/two_stage.cu's kernels, g++ (one "thread") into the test-only host build
// tests/host_build/two_stage_host.cpp.  All arithmetic is fp32 with separately rounded operations, in torch's order;
// sinf / cosf / expf / logf are the full-precision functions (the build has no fast-math).
#pragma once

#include <math.h>
#include <stddef.h>
#include <stdint.h>

#include "../../include/tfb200_fused.h"
#include "host_device.h"

namespace tfb200_two_stage {

constexpr int kMaxLevels = 8;
constexpr int kMaxK = 2048;            // queries selected per image
constexpr int kSelThreads = 1024;
constexpr int kEmbed = 128;            // sine features per box coordinate (get_proposal_pos_embed's num_pos_feats)

struct ProposalParams {
  int B, S, L, C;
  int H[kMaxLevels], W[kMaxLevels], start[kMaxLevels];
  const uint8_t* mask;                 // [B][S], nonzero = padded; nullptr: no padding
  const float* memory;                 // [B][S][C] or nullptr
  float* masked;                       // [B][S][C] (with memory)
  float* prop;                         // [B][S][4] proposal logits
  uint8_t* valid;                      // [B][S]
};

// the unpadded width (row 0) and height (column 0) of every level of image b
HD_FN void ts_valid_counts(const ProposalParams& p, int b, int* vw, int* vh) {
  for (int l = HD_TID; l < p.L; l += HD_NT) { vw[l] = 0; vh[l] = 0; }
  HD_SYNC();
  if (p.mask == nullptr) {
    for (int l = HD_TID; l < p.L; l += HD_NT) { vw[l] = p.W[l]; vh[l] = p.H[l]; }
  } else {
    const uint8_t* m = p.mask + size_t(b) * p.S;
    for (int l = 0; l < p.L; ++l) {
      for (int x = HD_TID; x < p.W[l]; x += HD_NT)
        if (!m[p.start[l] + x]) hd_atomic_add(&vw[l], 1);
      for (int y = HD_TID; y < p.H[l]; y += HD_NT)
        if (!m[p.start[l] + y * p.W[l]]) hd_atomic_add(&vh[l], 1);
    }
  }
  HD_SYNC();
}

// proposal logits and valid flag of token s of image b; returns the flag
HD_FN bool ts_proposal(const ProposalParams& p, int b, int s, const int* vw, const int* vh) {
  int l = 0;
  while (l + 1 < p.L && s >= p.start[l + 1]) ++l;
  const int r = s - p.start[l], y = r / p.W[l], x = r - y * p.W[l];
  float v[4];
  v[0] = (float(x) + 0.5f) / float(vw[l]);
  v[1] = (float(y) + 0.5f) / float(vh[l]);
  v[2] = v[3] = 0.05f * float(1 << l);
  const bool padded = p.mask != nullptr && p.mask[size_t(b) * p.S + s] != 0;
  bool ok = !padded;
  for (int c = 0; c < 4; ++c) ok = ok && v[c] > 0.01f && v[c] < 0.99f;
  float* out = p.prop + (size_t(b) * p.S + s) * 4;
  for (int c = 0; c < 4; ++c) out[c] = ok ? logf(v[c] / (1.0f - v[c])) : INFINITY;
  p.valid[size_t(b) * p.S + s] = ok ? 1 : 0;
  return ok;
}

// ---- selection ----------------------------------------------------------------------------------------------------
struct SelectParams {
  int B, S, C, k;
  const float* logits;                 // [B][S][C], class 0 is ranked
  const float* unact;                  // [B][S][4] unactivated boxes
  const float* dim_t;                  // [128]
  uint32_t* keys;                      // [B][S] workspace
  int64_t* index;                      // [B][k] selected tokens, best first
  float* boxes;                        // [B][k][4] gathered unactivated boxes
  float* ref;                          // [B][k][4] their sigmoid
  float* embed;                        // [B][k][4 * 128]
};

struct SelectShared {
  uint32_t hist[256];
  uint32_t wkey[kMaxK];
  int widx[kMaxK];
  int order[kMaxK];
  int cnt[kSelThreads];
  uint32_t prefix, hi_mask;
  int krem, ngt, taken;
};

// order-preserving key: a > b as floats <=> key(a) > key(b) as unsigned (-0 ranks below +0)
HD_FN uint32_t ts_key(float f) {
  const uint32_t u = hd_float_bits(f);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

HD_FN void ts_select(const SelectParams& p, int b, SelectShared& sh) {
  const int S = p.S, k = p.k;
  uint32_t* keys = p.keys + size_t(b) * S;
  if (HD_TID == 0) { sh.prefix = 0; sh.hi_mask = 0; sh.krem = k; sh.taken = 0; }
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (int i = HD_TID; i < 256; i += HD_NT) sh.hist[i] = 0;
    HD_SYNC();
    const uint32_t prefix = sh.prefix, hi = sh.hi_mask;
    for (int s = HD_TID; s < S; s += HD_NT) {
      uint32_t key;
      if (pass == 0) {
        key = ts_key(p.logits[(size_t(b) * S + s) * p.C]);
        keys[s] = key;
      } else {
        key = keys[s];
      }
      if ((key & hi) == prefix) hd_atomic_add(&sh.hist[(key >> shift) & 255u], 1u);
    }
    HD_SYNC();
    if (HD_TID == 0) {
      int above = 0, bin = 255;
      for (; bin > 0; --bin) {
        if (above + int(sh.hist[bin]) >= sh.krem) break;
        above += int(sh.hist[bin]);
      }
      sh.krem -= above;
      sh.prefix |= uint32_t(bin) << shift;
      sh.hi_mask |= 0xffu << shift;
    }
    HD_SYNC();
  }
  // threshold key t = sh.prefix; krem of the tokens with key t are taken, the lowest token indices first
  const uint32_t t = sh.prefix;
  const int krem = sh.krem;
  if (HD_TID == 0) sh.ngt = k - krem;
  HD_SYNC();
  const int ngt = sh.ngt;
  const int nt = HD_NT, seg = (S + nt - 1) / nt;
  const int s0 = HD_TID * seg, s1 = s0 + seg < S ? s0 + seg : S;
  int ties = 0;
  for (int s = HD_TID; s < S; s += HD_NT) {
    const uint32_t key = keys[s];
    if (key > t) {
      const int at = hd_atomic_add(&sh.taken, 1);
      sh.wkey[at] = key;
      sh.widx[at] = s;
    }
  }
  for (int s = s0; s < s1; ++s) ties += keys[s] == t;
  sh.cnt[HD_TID] = ties;
  HD_SYNC();
  if (HD_TID == 0) {
    int acc = 0;
    for (int i = 0; i < nt; ++i) { const int c = sh.cnt[i]; sh.cnt[i] = acc; acc += c; }
  }
  HD_SYNC();
  int run = sh.cnt[HD_TID];
  for (int s = s0; s < s1 && run < krem; ++s)
    if (keys[s] == t) { sh.wkey[ngt + run] = t; sh.widx[ngt + run] = s; ++run; }
  HD_SYNC();
  // rank sort of the k winners: logit descending, token ascending (a total order)
  for (int i = HD_TID; i < k; i += HD_NT) {
    const uint32_t ki = sh.wkey[i];
    const int ii = sh.widx[i];
    int rank = 0;
    for (int j = 0; j < k; ++j) {
      const uint32_t kj = sh.wkey[j];
      rank += kj > ki || (kj == ki && sh.widx[j] < ii);
    }
    sh.order[rank] = ii;
  }
  HD_SYNC();
}

HD_FN float ts_sigmoid(float x) { return 1.0f / (1.0f + expf(-x)); }

HD_FN void ts_select_outputs(const SelectParams& p, int b, const SelectShared& sh) {
  const int k = p.k;
  for (int r = HD_TID; r < k; r += HD_NT) p.index[size_t(b) * k + r] = sh.order[r];
  for (int e = HD_TID; e < k * 4; e += HD_NT) {
    const int r = e >> 2, c = e & 3;
    const float u = p.unact[(size_t(b) * p.S + sh.order[r]) * 4 + c];
    p.boxes[size_t(b) * k * 4 + e] = u;
    p.ref[size_t(b) * k * 4 + e] = ts_sigmoid(u);
  }
  const float scale = 6.28318530717958647692f;          // float(2 * math.pi)
  for (int e = HD_TID; e < k * 4 * kEmbed; e += HD_NT) {
    const int r = e / (4 * kEmbed), c = (e / kEmbed) & 3, j = e % kEmbed;
    const float u = p.unact[(size_t(b) * p.S + sh.order[r]) * 4 + c];
    const float pos = (ts_sigmoid(u) * scale) / p.dim_t[j];
    p.embed[size_t(b) * k * 4 * kEmbed + e] = (j & 1) ? cosf(pos) : sinf(pos);
  }
}

// argument checks shared by the C entries and the host build
static inline int ts_check_proposals(int B, int S, int L, int C, const int* hw) {
  if (B <= 0 || S <= 0 || L <= 0 || L > kMaxLevels || C < 0 || C % 4 != 0) return TFB200_E_SHAPE;
  int64_t total = 0;
  for (int l = 0; l < L; ++l) {
    if (hw[2 * l] <= 0 || hw[2 * l + 1] <= 0) return TFB200_E_SHAPE;
    total += int64_t(hw[2 * l]) * hw[2 * l + 1];
  }
  return total == S ? 0 : TFB200_E_SHAPE;
}

static inline int ts_check_select(int B, int S, int C, int k) {
  if (B <= 0 || S <= 0 || C <= 0 || k <= 0 || k > S || k > kMaxK) return TFB200_E_SHAPE;
  return 0;
}

static inline void ts_levels(ProposalParams& p, const int* hw) {
  int acc = 0;
  for (int l = 0; l < p.L; ++l) {
    p.H[l] = hw[2 * l];
    p.W[l] = hw[2 * l + 1];
    p.start[l] = acc;
    acc += p.H[l] * p.W[l];
  }
}

}  // namespace tfb200_two_stage
