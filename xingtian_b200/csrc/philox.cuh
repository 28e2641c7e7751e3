// philox.cuh -- the Philox4x32-10 counter-based generator (Salmon et al. 2011) every device draw of the library uses.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

namespace xtb {

// Ten rounds on counter c (overwritten by the four output words) with key (k0, k1)
__device__ inline void philox4x32_10(uint32_t c[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int i = 0; i < 10; i++) {
    uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}

}  // namespace xtb
