// Philox4x32-10 (Salmon, Moraes, Dror, Shaw, "Parallel random numbers: as easy as 1, 2, 3", SC 2011), the counter-based
// generator of the sampling token picker.  Plain C++ apart from the qualifiers, so that a host compiler builds the same
// function (tests/test_sampling.py compiles this header with g++ and checks it against the published answers).
#ifndef MT3_PHILOX_CUH_
#define MT3_PHILOX_CUH_

#include <stdint.h>

#ifdef __CUDACC__
#define MT3_HD __host__ __device__ __forceinline__
#else
#define MT3_HD inline
#endif

namespace mt3 {

// out = Philox4x32-10(counter c, key (k0, k1)): ten rounds, the key bumped by the Weyl constants between rounds
MT3_HD void philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t out[4]) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    if (r) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    c1 = (uint32_t)p1;
    c3 = (uint32_t)p0;
    c0 = n0;
    c2 = n2;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}

// A uniform float strictly inside (0, 1) from one output word: (2 (w >> 9) + 1) 2^-24, exact in float32
MT3_HD float philox_uniform(uint32_t w) { return (float)(2u * (w >> 9) + 1u) * 5.9604644775390625e-8f; }

}  // namespace mt3

#endif  // MT3_PHILOX_CUH_
