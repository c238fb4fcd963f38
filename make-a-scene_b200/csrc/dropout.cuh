// Dropout masks of the token transformer, generated where they are used and regenerated in the backward (never stored).
// Element e of a dropout site with 64-bit seed s is kept iff
//     w = word[e & 3] of Philox4x32-10(counter = (lo32(e >> 2), hi32(e >> 2), 0, 0), key = (lo32(s), hi32(s)))  >=  t,
// t = floor(p * 2^32) (a 64-bit integer in [0, 2^32]: p = 1 keeps nothing).  e is the element's row-major linear index in
// its tensor ([B, heads, S, S] probabilities, [rows, H] activations), so the mask does not depend on any kernel's tiling.
// The seed is read from device memory: a captured CUDA graph draws a fresh mask at each replay.
#pragma once
#include <stdint.h>

namespace mas {

// Philox4x32-10 (Salmon, Moraes, Dror, Shaw, SC'11), the counter-based generator of Random123 and cuRAND.
__device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t lo0 = 0xD2511F53u * c.x, hi0 = __umulhi(0xD2511F53u, c.x);
    const uint32_t lo1 = 0xCD9E8D57u * c.z, hi1 = __umulhi(0xCD9E8D57u, c.z);
    c = make_uint4(hi1 ^ c.y ^ k0, lo1, hi0 ^ c.w ^ k1, lo0);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c;
}

struct DropMask {
  const int64_t* seed;   // device scalar
  uint64_t t;            // keep iff word >= t
  float scale;           // factor of kept elements
};

// Host side: the threshold of probability p (0 <= p <= 1).
static inline uint64_t drop_threshold(double p) {
  const double t = p * 4294967296.0;
  return t <= 0.0 ? 0ull : (t >= 4294967296.0 ? 4294967296ull : (uint64_t)t);
}

// Host side: the factor of kept elements, 1 / (1 - p) (0 for p = 1, like nn.Dropout(p=1)).
static inline float drop_scale(double p) { return p < 1.0 ? (float)(1.0 / (1.0 - p)) : 0.f; }

// Keep bits (bit k <-> element 4 g + k) of the group g of four consecutive elements.
__device__ __forceinline__ uint32_t keep_bits4(uint64_t seed, uint64_t g, uint64_t t) {
  const uint4 w = philox4x32_10(make_uint4((uint32_t)g, (uint32_t)(g >> 32), 0u, 0u), (uint32_t)seed, (uint32_t)(seed >> 32));
  return (uint32_t)((uint64_t)w.x >= t) | ((uint32_t)((uint64_t)w.y >= t) << 1) | ((uint32_t)((uint64_t)w.z >= t) << 2) |
         ((uint32_t)((uint64_t)w.w >= t) << 3);
}

}  // namespace mas
