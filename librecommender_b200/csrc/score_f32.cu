// Exact-fp32 scoring kernels (SIMT).
//
// b200_score_rows_f32 replaces `user_embed @ item_embeds.T` of
// libreco/recommendation/recommend.py:66-68 when the score matrix has to be materialised
// (rank path for arbitrary d / tiny catalogues, and the fallback of the tensor-core path).
// b200_gather_dot replaces libreco/prediction/predict.py:36-40.
//
// Exact-score definition used everywhere in this library: one fp32 accumulator per output,
// acc = fmaf(u[k], i[k], acc) for k = 0..d-1.
#include "common.cuh"
#include "../../include/b200reco.h"

namespace b200 {

constexpr int BM = 128, BN = 128, BK = 8;

// C[BM,BN] tile per CTA, 256 threads, 8x8 micro-tile per thread (strided by 16 so that
// shared-memory reads are conflict-free broadcasts and global stores are 64-B segments).
__global__ void __launch_bounds__(256)
score_rows_f32_kernel(const float* __restrict__ U, int64_t ldu, const int64_t* __restrict__ uid,
                      int64_t B, const float* __restrict__ I, int64_t ldi, int64_t N, int d,
                      float* __restrict__ out, int64_t lds) {
  __shared__ float As[BK][BM + 4];
  __shared__ float Bs[BK][BN + 4];
  __shared__ int64_t urow[BM];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = (int64_t)blockIdx.y * BM;
  const int64_t n0 = (int64_t)blockIdx.x * BN;
  if (tid < BM) {
    const int64_t r = m0 + tid;
    urow[tid] = (r < B) ? (uid ? uid[r] : r) : -1;
  }
  __syncthreads();
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  // loader mapping: thread -> (row = tid / 2, k-offset = (tid % 2) * 4), 4 consecutive k
  const int lrow = tid >> 1, lk = (tid & 1) * 4;
  const int64_t arow = urow[lrow];
  const int64_t brow = n0 + lrow;
  for (int k0 = 0; k0 < d; k0 += BK) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int k = k0 + lk + q;
      // k >= d pads the last BK tile with a product of -0.0: fmaf(0, -0, acc) == acc for every acc, -0.0
      // included (a +0.0 product would turn an accumulated -0.0 into +0.0)
      float a = 0.f, b = -0.f;
      if (k < d) {
        if (arow >= 0) a = __ldg(U + arow * ldu + k);
        if (brow < N) b = __ldg(I + brow * ldi + k);
      }
      As[lk + q][lrow] = a;
      Bs[lk + q][lrow] = b;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < BK; ++k) {
      float a[8], b[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = As[k][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 8; ++j) b[j] = Bs[k][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t r = m0 + ty + 16 * i;
    if (r >= B) continue;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int64_t c = n0 + tx + 16 * j;
      if (c < N) out[r * lds + c] = acc[i][j];
    }
  }
}

// one warp per (user, item) pair: lanes stride over k, but to keep the exact-score definition
// (sequential fma in k) each lane handles whole pairs instead: thread per pair.
__global__ void gather_dot_kernel(const float* __restrict__ U, int64_t ldu,
                                  const int64_t* __restrict__ users, const float* __restrict__ I,
                                  int64_t ldi, const int64_t* __restrict__ items, int64_t n, int d,
                                  int mode, float lo, float hi, float* __restrict__ out) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= n) return;
  const float* u = U + users[r] * ldu;
  const float* it = I + items[r] * ldi;
  float acc = 0.f;
  for (int k = 0; k < d; ++k) acc = fmaf(__ldg(u + k), __ldg(it + k), acc);
  if (mode == 1) acc = 1.f / (1.f + expf(-acc));
  else if (mode == 2) acc = fminf(fmaxf(acc, lo), hi);
  out[r] = acc;
}

}  // namespace b200

using namespace b200;

extern "C" int b200_score_rows_f32(const float* U, int64_t ldu, const int64_t* user_ids, int64_t B,
                                   const float* I, int64_t ldi, int64_t N, int32_t d, float* scores,
                                   int64_t lds, void* stream) {
  B200_REQUIRE(U && I && scores, "b200_score_rows_f32: null pointer");
  B200_REQUIRE(d >= 1 && N >= 1 && B >= 0, "b200_score_rows_f32: bad shape");
  if (B == 0) return 0;
  const int64_t gy = ceil_div64(B, BM);
  B200_REQUIRE(gy <= 65535, "b200_score_rows_f32: too many rows per call");
  dim3 grid((unsigned)ceil_div64(N, BN), (unsigned)gy);
  score_rows_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(U, ldu, user_ids, B, I, ldi, N, d,
                                                                scores, lds);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_gather_dot(const float* U, int64_t ldu, const int64_t* users, const float* I,
                               int64_t ldi, const int64_t* items, int64_t n, int32_t d, int32_t mode,
                               float lo, float hi, float* out, void* stream) {
  B200_REQUIRE(U && I && users && items && out, "b200_gather_dot: null pointer");
  if (n == 0) return 0;
  gather_dot_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(
      U, ldu, users, I, ldi, items, n, d, mode, lo, hi, out);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
