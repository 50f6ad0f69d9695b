// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11): the counter-based generator
// of the on-device samplers (sample_filter.cuh) and of the training dropout masks (dropout.cuh). ops/sampling.py's
// philox4x32_10 is the same function in Python integers.
#pragma once

#include <cstdint>

namespace adapcc {

// the four output words for counter (c0, c1, c2, c3) and key (k0, k1)
__device__ __forceinline__ uint4 philox4(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                         uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    c0 = hi1 ^ c1 ^ k0;
    c1 = lo1;
    c2 = hi0 ^ c3 ^ k1;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

}  // namespace adapcc
