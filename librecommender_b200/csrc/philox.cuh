// Philox4x32-10 counter-based generator and its bounded-integer map, shared by the device samplers
// (csrc/sampler.cu) and BPR's negative draw (csrc/bpr.cu).  oracle/sampling.py restates both bit for bit.
#pragma once
#include <stdint.h>

namespace b200 {

struct U4 { uint32_t x, y, z, w; };

__host__ __device__ __forceinline__ U4 philox4x32_10(U4 ctr, uint32_t k0, uint32_t k1) {
  const uint32_t M0 = 0xD2511F53u, M1 = 0xCD9E8D57u, W0 = 0x9E3779B9u, W1 = 0xBB67AE85u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)M0 * ctr.x;
    const uint64_t p1 = (uint64_t)M1 * ctr.z;
    U4 n;
    n.x = (uint32_t)(p1 >> 32) ^ ctr.y ^ k0;
    n.y = (uint32_t)p1;
    n.z = (uint32_t)(p0 >> 32) ^ ctr.w ^ k1;
    n.w = (uint32_t)p0;
    ctr = n;
    k0 += W0;
    k1 += W1;
  }
  return ctr;
}

// uniform integer in [0, n): high 64 bits of (64-bit random) * n
__device__ __forceinline__ int64_t bounded(uint32_t hi, uint32_t lo, int64_t n) {
  const uint64_t r = ((uint64_t)hi << 32) | lo;
  return (int64_t)__umul64hi(r, (uint64_t)n);
}

}  // namespace b200
