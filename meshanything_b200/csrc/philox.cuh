// philox.cuh -- Philox4x32-10 (Random123) for the seeded streams of the library: counter (i, tag0, tag1, tag2), key
// (seed mod 2^32, seed >> 32).  Each stream has its own tag (DESIGN.md section 1.5: the surface sampler; section 1.6:
// the plane hypotheses), so two features given the same seed draw unrelated numbers.
#pragma once
#include <cstdint>

namespace ma {

__device__ __forceinline__ uint32_t philox_mulhilo(uint32_t a, uint32_t b, uint32_t* hi) {
  const unsigned long long p = (unsigned long long)a * b;
  *hi = (uint32_t)(p >> 32);
  return (uint32_t)p;
}

// the four output words of Philox4x32-10 for counter (i, tag0, tag1, tag2) under the key of `seed`
__device__ __forceinline__ uint4 philox4x32_10(uint32_t i, uint32_t tag0, uint32_t tag1, uint32_t tag2,
                                               unsigned long long seed) {
  uint32_t c0 = i, c1 = tag0, c2 = tag1, c3 = tag2;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; r++) {
    uint32_t hi0, hi1;
    const uint32_t lo0 = philox_mulhilo(0xD2511F53u, c0, &hi0), lo1 = philox_mulhilo(0xCD9E8D57u, c2, &hi1);
    const uint32_t n0 = hi1 ^ c1 ^ k0, n1 = lo1, n2 = hi0 ^ c3 ^ k1, n3 = lo0;
    c0 = n0; c1 = n1; c2 = n2; c3 = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

}  // namespace ma
