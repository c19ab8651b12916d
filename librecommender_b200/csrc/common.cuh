// Shared helpers for the sm_90a kernels of librecommender_b200.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

namespace b200 {

// ---- error plumbing (thread-local last error string, C-ABI returns <0) ----
void set_last_error(const char* fmt, ...);
int check_cuda(cudaError_t e, const char* what);

#define B200_CUDA_OK(expr)                                   \
  do {                                                       \
    int _rc = ::b200::check_cuda((expr), #expr);             \
    if (_rc != 0) return _rc;                                \
  } while (0)

#define B200_REQUIRE(cond, ...)                              \
  do {                                                       \
    if (!(cond)) {                                           \
      ::b200::set_last_error(__VA_ARGS__);                   \
      return -2;                                             \
    }                                                        \
  } while (0)

// kernel launch counter (bench.py reports gpu_launches from it)
extern unsigned long long g_launch_count;
inline void count_launch(int n = 1) { g_launch_count += (unsigned long long)n; }

// SM count of the current device (0 if it cannot be queried): launch sizing and the fused scorer's plan
inline int num_sms() {
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess)
    return 0;
  return n;
}

__host__ __device__ inline int64_t ceil_div64(int64_t a, int64_t b) { return (a + b - 1) / b; }

// Float bit pattern of a REMOVED entry (a consumed item, an empty candidate slot).  It is a NaN
// that no arithmetic produces (hardware NaNs are 0x7fffffff), and its key is 0: below every real value.
constexpr uint32_t kRemovedBits = 0xffffffffu;

// Order-preserving map float -> uint32 (larger float => larger key), one key per class of values
// the ranking order calls equal: -0.0 takes the key of +0.0, every NaN the top key (a NaN ranks
// above +inf, where numpy's sort puts it), and kRemovedBits key 0.  Keys in [1, key(-inf)) are unused.
// key_to_float inverts it up to that canonicalisation (-0.0 -> +0.0, NaN -> 0x7fffffff).
__device__ __forceinline__ uint32_t float_to_key(float f) {
  uint32_t b = __float_as_uint(f);
  b = b == 0x80000000u ? 0u : b;
  const uint32_t k = (b & 0x80000000u) ? ~b : (b | 0x80000000u);
  // NaNs land in (key(+inf), 2^32) (positive) and [1, key(-inf)) (negative; kRemovedBits gives 0)
  return (k - 1u < 0x007ffffeu || k > 0xff800000u) ? 0xffffffffu : k;
}
__device__ __forceinline__ float key_to_float(uint32_t k) {
  uint32_t b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(b);
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace b200
