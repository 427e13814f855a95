// attn_dropout.cuh — the attention dropout mask, shared by flash_attn.cu and temporal_attn_long.cu.
//
// SDPA's dropout_p (genie/module/attention.py:229-234) drops softmax probabilities after the causal mask and scales the
// kept ones by 1 / (1 - p). The forward pass and both backward passes regenerate the mask, and they hold the scores in
// different orientations (S in the forward, flash MODE 1 and the tiled dQ kernel; S^T in flash MODE 0 and the tiled
// dK / dV kernel), so the mask is a pure function of (seed, sequence, head, query i, key j):
//
//   z    = sequence * n_head + head        (64-bit; flash: the frame in [0, nseq); tiled temporal: b * P + p)
//   c    = ((j >> 4) * 8 + (j & 7), (i >> 4) * 8 + (i & 7), lo32(z), hi32(z))
//   r    = Philox4x32-10(counter c, key (lo32(seed), hi32(seed)))     (Salmon et al., SC 2011; curand's Philox4_32_10)
//   w    = r[2 * ((i >> 3) & 1) + ((j >> 3) & 1)]
//   keep(i, j)  iff  w >= t,   t = min(round(p * 2^32), 2^32 - 1)
//
// One Philox call covers queries {i, i + 8} x keys {j, j + 8} (i, j with bit 3 clear). In both the wgmma and the
// mma.sync m16n8k16 accumulator fragments a thread holds rows {r, r + 8} and columns {c + 8k}, so each call's four words
// land in one thread whichever operand is the row: about 15 integer instructions per score. The keep probability
// 1 - t / 2^32 is within 2^-33 of 1 - p.
//
// The seed is read from device memory, so a captured CUDA graph draws a fresh one (written by the generator) per replay.
#pragma once
#include <math.h>
#include <stdint.h>

#include "og_host.cuh"

namespace og {

struct DropParams {
  const uint64_t* seed;   // device pointer to the 64-bit seed of this call
  uint32_t thresh;        // t: a score is kept iff its Philox word is >= t
  float rscale;           // 1 / (1 - p)
};

__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k.x, lo1, hi0 ^ c.w ^ k.y, lo0);
    k.x += 0x9E3779B9u;
    k.y += 0xBB67AE85u;
  }
  return c;
}

__device__ __forceinline__ uint2 drop_key(const uint64_t* seed) {
  const uint64_t s = *seed;
  return make_uint2((uint32_t)s, (uint32_t)(s >> 32));
}

// Keep bits of one thread's 16 x 64 share of a 64 x 64 score tile, in the accumulator order of both fragment layouts:
// bit 4 jj + 2 rr + e is element (row + 8 rr, col + 8 jj + e), rr, e in {0, 1}, jj in 0 .. 7. `row` has bit 3 clear and
// `col` is a multiple of 16 plus the thread's column offset (< 8). kT: rows are keys and columns queries (S^T).
template <bool kT>
__device__ __forceinline__ uint32_t drop_keep_tile(uint32_t row, uint32_t col, uint64_t z, uint2 key, uint32_t t) {
  uint32_t m = 0;
#pragma unroll
  for (int pj = 0; pj < 4; ++pj)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const uint32_t cc = col + 16 * pj + e;
      const uint32_t qi = kT ? cc : row, kj = kT ? row : cc;
      const uint4 r = philox4x32_10(
          make_uint4((kj >> 4) * 8 + (kj & 7), (qi >> 4) * 8 + (qi & 7), (uint32_t)z, (uint32_t)(z >> 32)), key);
      const uint32_t w[4] = {r.x, r.y, r.z, r.w};   // word 2a + b: query + 8a, key + 8b
#pragma unroll
      for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 2; ++b) {
          const int rr = kT ? b : a, jj = 2 * pj + (kT ? a : b);
          m |= (uint32_t)(w[2 * a + b] >= t) << (4 * jj + 2 * rr + e);
        }
    }
  return m;
}

// Checks p and the seed pointer of a dropout entry point and derives t and 1 / (1 - p).
static inline int drop_params(float p, const uint64_t* seed, const char* who, DropParams* d) {
  OG_REQUIRE(seed, "%s: null seed pointer", who);
  OG_REQUIRE(p >= 0.f && p < 1.f, "%s: dropout p=%g must lie in [0, 1)", who, (double)p);
  const double t = nearbyint((double)p * 4294967296.0);
  d->seed = seed;
  d->thresh = t > 4294967295.0 ? 0xFFFFFFFFu : (uint32_t)t;
  d->rscale = (float)(1.0 / (1.0 - (double)p));
  return OG_OK;
}

// The same for the entry points that also run without dropout (og_flash_attn_causal_*, og_temporal_attn_bidir_*):
// p = 0 gives *drop = nullptr, the kernels without a mask, and the seed may be null; any other p is checked as above.
static inline int drop_params_opt(float p, const uint64_t* seed, const char* who, DropParams* d,
                                  const DropParams** drop) {
  *drop = nullptr;
  if (p == 0.f) return OG_OK;
  if (const int r = drop_params(p, seed, who, d)) return r;
  *drop = d;
  return OG_OK;
}

}  // namespace og
