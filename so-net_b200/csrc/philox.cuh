// philox.cuh — the library's one counter-based generator: Philox4x32-10 (Salmon et al., SC'11).
// No state to store: the 128-bit counter names the draw, the 64-bit seed is the key. Used by the
// in-kernel jitter of augment.cu, the in-kernel point selection of sample_points.cu and the surface
// draws of mesh_sample.cu, which keep their streams apart through a stream tag in counter word 2
// (augment: 0..2, sample_points: 3..4, mesh_sample: 5..6).
#pragma once
#include <stdint.h>

namespace sonet {

__device__ __forceinline__ void philox_round(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
  const uint32_t hi0 = __umulhi(0xD2511F53u, c[0]), lo0 = 0xD2511F53u * c[0];
  const uint32_t hi1 = __umulhi(0xCD9E8D57u, c[2]), lo1 = 0xCD9E8D57u * c[2];
  const uint32_t n0 = hi1 ^ c[1] ^ k0, n2 = hi0 ^ c[3] ^ k1;
  c[0] = n0; c[1] = lo1; c[2] = n2; c[3] = lo0;
}
__device__ __forceinline__ void philox4x32_10(uint32_t (&c)[4], uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    philox_round(c, k0, k1);
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
}

}  // namespace sonet
