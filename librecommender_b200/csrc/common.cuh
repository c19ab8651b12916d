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

// Order-preserving map float -> uint32 (larger float => larger key).
__device__ __forceinline__ uint32_t float_to_key(float f) {
  uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
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
