// philox.cuh -- Philox4x32-10 (Salmon et al., SC'11), the counter-based generator of the device samplers (ffma_launch.cu)
// and of the HMC sampler (hmc.cu).  A draw is a pure function of (counter, key): graph replays and the float64 test
// oracle reproduce every value.
#pragma once
#include <stdint.h>

namespace pinn {

__device__ __forceinline__ void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
    const uint32_t n0 = hi1 ^ c[1] ^ k0, n1 = lo1, n2 = hi0 ^ c[3] ^ k1, n3 = lo0;
    c[0] = n0; c[1] = n1; c[2] = n2; c[3] = n3;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
}

}  // namespace pinn
