// Caser and WaveNet inference: the convolutional user encoders (libreco/algorithms/caser.py:177-221,
// wave_net.py:181-222).
//
// The user vector of both models is [user_embeds[u] | head(encoder(seq_embeds[seq]))]; the kernels here compute the
// encoder up to the Dense head, which runs on the dense-layer kernels.  One CTA owns a tile of users: each user's
// T x K gathered rows are read from HBM once into shared memory and every intermediate stays on chip (WaveNet's
// per-layer activations ping-pong between two [tile, T, C] buffers); only the pre-head features are written out.
// Weights are read through L1 / L2.
//
// Work item = (user, output column, [block of CONV_PB positions]); the item's output columns vary fastest across the
// threads of a warp, so the threads of a warp read the same shared-memory row (a broadcast) and consecutive weight
// columns.  Each pre-activation is one fmaf chain starting at the bias in the order the header states, a position
// block only shares the weight loads of its chains, and max / ReLU are order-free: a user's bits depend only on its
// own sequence, not on the tile it shares, on n or on the call.
#include <algorithm>

#include "../../include/b200reco.h"
#include "common.cuh"

namespace b200 {
namespace {

constexpr int CONV_MAX_T = 64;
constexpr int CONV_MAX_K = 128;
constexpr int CONV_MAX_FILTERS = 32;     // Caser nh, nv
constexpr int CONV_MAX_F = 128;          // WaveNet filters
constexpr int CONV_MAX_LAYERS = 16;      // WaveNet causal layers
constexpr int CONV_THREADS = 128;
constexpr int CONV_PB = 4;               // positions per work item
constexpr int CONV_MAX_TILE = 32;

// floats of Caser's packed weights: W_1 .. W_T ([h, K, nh] each), b_h [T, nh], Wv [T, nv], bv [nv]
__host__ __device__ inline int64_t caser_floats(int T, int K, int nh, int nv) {
  return (int64_t)K * nh * T * (T + 1) / 2 + (int64_t)T * nh + (int64_t)T * nv + nv;
}

// floats of WaveNet's packed weights: per causal layer W [2, C_in, F], b [F]; then the 1x1 layer W [F, F], b [F]
__host__ __device__ inline int64_t wavenet_floats(int K, int F, int n_conv) {
  return (2 * (int64_t)K * F + F) + (int64_t)(n_conv - 1) * (2 * (int64_t)F * F + F) + (int64_t)F * F + F;
}

struct ConvParams {
  int T, K, tile, us;                    // us: a user's float stride in shared memory (odd: no bank conflicts)
  int nh, nv;                            // Caser
  int F, L, dil[CONV_MAX_LAYERS], ldc;   // WaveNet: filters, causal layers, dilations, buffer row stride
  const int64_t* users;
  int64_t n;
  const int32_t* seqs;
  int64_t ld_seq;
  const float* X;
  int64_t ldx;
  const float* w;
  float* out;
  int64_t ldo;
};

// x[u * us + t * ld + k] = X[seqs[users[s0 + u], t], k] (0 for users past n)
__device__ void gather_tile(const ConvParams& p, float* x, int ld) {
  const int64_t s0 = (int64_t)blockIdx.x * p.tile;
  const int per_user = p.T * p.K;
  for (int i = threadIdx.x; i < p.tile * per_user; i += blockDim.x) {
    const int u = i / per_user, r = i - u * per_user, t = r / p.K, k = r - t * p.K;
    const int64_t s = s0 + u;
    float v = 0.f;
    if (s < p.n) {
      const int64_t item = __ldg(p.seqs + __ldg(p.users + s) * p.ld_seq + t);
      v = __ldg(p.X + item * p.ldx + k);
    }
    x[u * p.us + t * ld + k] = v;
  }
}

__global__ void __launch_bounds__(CONV_THREADS) caser_encode_kernel(const __grid_constant__ ConvParams p) {
  extern __shared__ float sm[];
  const int T = p.T, K = p.K, nh = p.nh, nv = p.nv;
  const int64_t s0 = (int64_t)blockIdx.x * p.tile;
  gather_tile(p, sm, K);
  __syncthreads();
  const float* bh = p.w + (int64_t)K * nh * T * (T + 1) / 2;
  const float* Wv = bh + T * nh;
  const float* bv = Wv + T * nv;
  // horizontal: o_h[f] = max_p relu(b_h[f] + sum_{j<h} sum_k x[p+j, k] W_h[j, k, f]), p = 0 .. T-h
  const int nhor = T * nh;
  for (int it = threadIdx.x; it < p.tile * nhor; it += blockDim.x) {
    const int u = it / nhor, r = it - u * nhor, h = r / nh + 1, f = r - (h - 1) * nh;
    if (s0 + u >= p.n) continue;
    const float* x = sm + u * p.us;
    const float* W = p.w + (int64_t)K * nh * (h - 1) * h / 2 + f;
    const float b = __ldg(bh + (h - 1) * nh + f);
    const int npos = T - h + 1;
    float m = 0.f;
    for (int p0 = 0; p0 < npos; p0 += CONV_PB) {
      int pos[CONV_PB];
      float acc[CONV_PB];
#pragma unroll
      for (int q = 0; q < CONV_PB; ++q) {
        pos[q] = min(p0 + q, npos - 1) * K;   // positions past the end repeat the last one: the max is unchanged
        acc[q] = b;
      }
      for (int j = 0; j < h; ++j)
        for (int k = 0; k < K; ++k) {
          const float wv = __ldg(W + (int64_t)(j * K + k) * nh);
#pragma unroll
          for (int q = 0; q < CONV_PB; ++q) acc[q] = fmaf(x[pos[q] + j * K + k], wv, acc[q]);
        }
#pragma unroll
      for (int q = 0; q < CONV_PB; ++q) m = fmaxf(m, acc[q]);
    }
    p.out[(s0 + u) * p.ldo + r] = m;
  }
  // vertical: v[k, f] = relu(bv[f] + sum_t x[t, k] Wv[t, f]) at column T*nh + k*nv + f
  const int nver = K * nv;
  for (int it = threadIdx.x; it < p.tile * nver; it += blockDim.x) {
    const int u = it / nver, r = it - u * nver, k = r / nv, f = r - k * nv;
    if (s0 + u >= p.n) continue;
    const float* x = sm + u * p.us + k;
    float acc = __ldg(bv + f);
    for (int t = 0; t < T; ++t) acc = fmaf(x[t * K], __ldg(Wv + t * nv + f), acc);
    p.out[(s0 + u) * p.ldo + nhor + r] = fmaxf(acc, 0.f);
  }
}

__global__ void __launch_bounds__(CONV_THREADS) wavenet_encode_kernel(const __grid_constant__ ConvParams p) {
  extern __shared__ float sm[];
  const int T = p.T, F = p.F, ld = p.ldc;
  const int64_t s0 = (int64_t)blockIdx.x * p.tile;
  float* xin = sm;
  float* xout = sm + p.tile * p.us;
  gather_tile(p, xin, ld);
  __syncthreads();
  // causal layer: y[t, f] = relu(b[f] + sum_c x[t-d, c] W[0, c, f] + sum_c x[t, c] W[1, c, f]), terms t-d < 0 absent
  const float* W = p.w;
  const int nblk = (T + CONV_PB - 1) / CONV_PB;
  for (int l = 0; l < p.L; ++l) {
    const int C = l ? F : p.K, d = p.dil[l];
    const float* b = W + 2 * C * F;
    for (int it = threadIdx.x; it < p.tile * nblk * F; it += blockDim.x) {
      const int u = it / (nblk * F), r = it - u * nblk * F, t0 = (r / F) * CONV_PB, f = r - (r / F) * F;
      if (s0 + u >= p.n) continue;
      const float* x = xin + u * p.us;
      int tq[CONV_PB];
      float acc[CONV_PB];
#pragma unroll
      for (int q = 0; q < CONV_PB; ++q) {
        tq[q] = min(t0 + q, T - 1);
        acc[q] = __ldg(b + f);
      }
      for (int c = 0; c < C; ++c) {
        const float wv = __ldg(W + c * F + f);
#pragma unroll
        for (int q = 0; q < CONV_PB; ++q)
          if (tq[q] >= d) acc[q] = fmaf(x[(tq[q] - d) * ld + c], wv, acc[q]);
      }
      for (int c = 0; c < C; ++c) {
        const float wv = __ldg(W + (C + c) * F + f);
#pragma unroll
        for (int q = 0; q < CONV_PB; ++q) acc[q] = fmaf(x[tq[q] * ld + c], wv, acc[q]);
      }
#pragma unroll
      for (int q = 0; q < CONV_PB; ++q)
        if (t0 + q < T) xout[u * p.us + (t0 + q) * ld + f] = fmaxf(acc[q], 0.f);
    }
    __syncthreads();
    W = b + F;
    float* tmp = xin; xin = xout; xout = tmp;
  }
  // the 1x1 layer, ReLU and the max over T: out[f] = max_t relu(b1[f] + sum_c y[t, c] W1[c, f])
  const float* b1 = W + F * F;
  for (int it = threadIdx.x; it < p.tile * F; it += blockDim.x) {
    const int u = it / F, f = it - u * F;
    if (s0 + u >= p.n) continue;
    const float* y = xin + u * p.us;
    float m = 0.f;
    for (int t0 = 0; t0 < T; t0 += CONV_PB) {
      int tq[CONV_PB];
      float acc[CONV_PB];
#pragma unroll
      for (int q = 0; q < CONV_PB; ++q) {
        tq[q] = min(t0 + q, T - 1) * ld;
        acc[q] = __ldg(b1 + f);
      }
      for (int c = 0; c < F; ++c) {
        const float wv = __ldg(W + c * F + f);
#pragma unroll
        for (int q = 0; q < CONV_PB; ++q) acc[q] = fmaf(y[tq[q] + c], wv, acc[q]);
      }
#pragma unroll
      for (int q = 0; q < CONV_PB; ++q) m = fmaxf(m, acc[q]);
    }
    p.out[(s0 + u) * p.ldo + f] = m;
  }
}

// the largest tile (at most CONV_MAX_TILE users) whose `buffers` [tile, us] blocks fit 96 KB, so that two CTAs
// share an SM; then the launch
template <typename Kernel>
int conv_launch(const char* who, Kernel kernel, ConvParams& p, int buffers, void* stream) {
  int dev = 0, optin = 0;
  B200_CUDA_OK(cudaGetDevice(&dev));
  B200_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  const int64_t bytes = (int64_t)buffers * p.us * sizeof(float);
  p.tile = (int)std::max<int64_t>(1, std::min<int64_t>(CONV_MAX_TILE, (96 * 1024) / bytes));
  const size_t smem = (size_t)(p.tile * bytes);
  B200_REQUIRE(smem <= (size_t)optin, "%s: a tile of %d users needs %zu B of shared memory, the device allows %d", who,
               p.tile, smem, optin);
  if (smem > 48 * 1024) B200_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<(unsigned)ceil_div64(p.n, p.tile), CONV_THREADS, smem, (cudaStream_t)stream>>>(p);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

bool caser_shape_ok(int T, int K, int nh, int nv) {
  return T >= 1 && T <= CONV_MAX_T && K >= 1 && K <= CONV_MAX_K && nh >= 1 && nh <= CONV_MAX_FILTERS && nv >= 1 &&
         nv <= CONV_MAX_FILTERS;
}

bool wavenet_shape_ok(int K, int F, int n_conv) {
  return K >= 1 && K <= CONV_MAX_K && F >= 1 && F <= CONV_MAX_F && n_conv >= 1 && n_conv <= CONV_MAX_LAYERS;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int64_t b200_caser_weight_floats(int32_t T, int32_t K, int32_t nh, int32_t nv) {
  return caser_shape_ok(T, K, nh, nv) ? caser_floats(T, K, nh, nv) : -2;
}

extern "C" int64_t b200_wavenet_weight_floats(int32_t K, int32_t F, int32_t n_conv) {
  return wavenet_shape_ok(K, F, n_conv) ? wavenet_floats(K, F, n_conv) : -2;
}

extern "C" int b200_caser_encode(const int64_t* users, int64_t n, const int32_t* seqs, int64_t ld_seq, int32_t T,
                                 const float* X, int64_t ldx, int32_t K, int32_t nh, int32_t nv, const float* weights,
                                 float* out, int64_t ldo, void* stream) {
  const char* who = "b200_caser_encode";
  B200_REQUIRE(caser_shape_ok(T, K, nh, nv), "%s: T %d, K %d, nh %d, nv %d outside T <= %d, K <= %d, nh, nv <= %d", who,
               T, K, nh, nv, CONV_MAX_T, CONV_MAX_K, CONV_MAX_FILTERS);
  B200_REQUIRE(n >= 0 && n <= (int64_t)0x7fffffff * CONV_MAX_TILE, "%s: bad slot count %lld", who, (long long)n);
  if (n == 0) return 0;
  B200_REQUIRE(users && seqs && X && weights && out, "%s: null pointer", who);
  B200_REQUIRE(ld_seq >= T && ldx >= K && ldo >= (int64_t)T * nh + (int64_t)K * nv, "%s: bad leading dimension", who);
  ConvParams p{};
  p.T = T; p.K = K; p.nh = nh; p.nv = nv;
  p.users = users; p.n = n; p.seqs = seqs; p.ld_seq = ld_seq; p.X = X; p.ldx = ldx; p.w = weights;
  p.out = out; p.ldo = ldo;
  p.us = (T * K) | 1;
  return conv_launch(who, caser_encode_kernel, p, 1, stream);
}

extern "C" int b200_wavenet_encode(const int64_t* users, int64_t n, const int32_t* seqs, int64_t ld_seq, int32_t T,
                                   const float* X, int64_t ldx, int32_t K, int32_t n_conv, int32_t F,
                                   const int32_t* dilations, const float* weights, float* out, int64_t ldo,
                                   void* stream) {
  const char* who = "b200_wavenet_encode";
  B200_REQUIRE(T >= 1 && T <= CONV_MAX_T && wavenet_shape_ok(K, F, n_conv),
               "%s: T %d, K %d, F %d, %d layers outside T <= %d, K <= %d, F <= %d, 1 to %d layers", who, T, K, F, n_conv,
               CONV_MAX_T, CONV_MAX_K, CONV_MAX_F, CONV_MAX_LAYERS);
  B200_REQUIRE(dilations, "%s: null dilations", who);
  ConvParams p{};
  for (int l = 0; l < n_conv; ++l) {
    B200_REQUIRE(dilations[l] >= 1, "%s: layer %d has dilation %d", who, l, dilations[l]);
    p.dil[l] = dilations[l];
  }
  B200_REQUIRE(n >= 0 && n <= (int64_t)0x7fffffff * CONV_MAX_TILE, "%s: bad slot count %lld", who, (long long)n);
  if (n == 0) return 0;
  B200_REQUIRE(users && seqs && X && weights && out, "%s: null pointer", who);
  B200_REQUIRE(ld_seq >= T && ldx >= K && ldo >= F, "%s: bad leading dimension", who);
  p.T = T; p.K = K; p.F = F; p.L = n_conv; p.ldc = std::max(K, F) | 1; p.us = (T * p.ldc) | 1;
  p.users = users; p.n = n; p.seqs = seqs; p.ld_seq = ld_seq; p.X = X; p.ldx = ldx; p.w = weights;
  p.out = out; p.ldo = ldo;
  return conv_launch(who, wavenet_encode_kernel, p, 2, stream);
}
