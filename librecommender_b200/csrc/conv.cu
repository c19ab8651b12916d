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
//
// Training (caser.py:135-221, wave_net.py:139-222): the same kernels with SAVE = true also write the max-pool argmax
// and WaveNet's layer outputs; Caser's backward routes dF through the saved argmax (caser_dx_kernel, caser_dw_kernel
// + b200_col_reduce, no atomics), WaveNet's backward runs on the dense kernels around three position kernels.
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
  // training forward only (SAVE = true): the max-pool argmax per output column, and WaveNet's causal layer outputs
  int32_t* arg;
  float* ys;
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

// SAVE = true (the training forward) computes the same values in the same order and also writes, per output column
// of the horizontal part, the argmax of the max-pool: the lowest position reaching the maximum (strict > in ascending
// position order; positions clamped to the last one repeat it and cannot move it), -1 when the maximum is <= 0
template <bool SAVE>
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
    float best = 0.f;
    int arg = -1;
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
      for (int q = 0; q < CONV_PB; ++q) {
        m = fmaxf(m, acc[q]);
        if (SAVE && acc[q] > best) {
          best = acc[q];
          arg = min(p0 + q, npos - 1);
        }
      }
    }
    p.out[(s0 + u) * p.ldo + r] = m;
    if (SAVE) p.arg[(s0 + u) * nhor + r] = arg;
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

// SAVE = true also writes every causal layer's output y_l [n * T, F] (ys + l * n * T * F, row s * T + t) and, per
// (slot, f), the argmax over t of the 1x1 layer under the tie rule of caser_encode_kernel (-1 when the max is <= 0)
template <bool SAVE>
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
        if (t0 + q < T) {
          xout[u * p.us + (t0 + q) * ld + f] = fmaxf(acc[q], 0.f);
          if (SAVE) p.ys[((int64_t)l * p.n + s0 + u) * T * F + (int64_t)(t0 + q) * F + f] = fmaxf(acc[q], 0.f);
        }
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
    float best = 0.f;
    int arg = -1;
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
      for (int q = 0; q < CONV_PB; ++q) {
        m = fmaxf(m, acc[q]);
        if (SAVE && acc[q] > best) {
          best = acc[q];
          arg = min(t0 + q, T - 1);
        }
      }
    }
    p.out[(s0 + u) * p.ldo + f] = m;
    if (SAVE) p.arg[(s0 + u) * F + f] = arg;
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

// ---- Caser backward ---------------------------------------------------------------------------------------------
// g = dF masked: a horizontal column passes dF to its saved argmax p* (nothing when p* = -1), a vertical column
// passes dF where the feature is > 0.  Rows s * T + t of X and dX are position t of slot s.
constexpr int CONV_CHUNK_ROWS = 256;           // rows per weight-gradient partial
constexpr int64_t CONV_PART_FLOATS = 1 << 22;  // the partials stay below max(E, this) floats

struct CaserBwdParams {
  int T, K, nh, nv, nchunk, chunk;
  int64_t n, E;
  const float* dF;
  int64_t ldf;
  const float* feat;
  int64_t ldfe;
  const int32_t* arg;   // [n, T * nh]
  const float* X;
  int64_t ldx;
  const float* w;
  float* dX;
  int64_t lddx;
  float* part;          // [nchunk, E]
};

int caser_nchunk(int64_t n, int64_t E) {
  const int64_t by_rows = (n + CONV_CHUNK_ROWS - 1) / CONV_CHUNK_ROWS;
  return (int)std::max<int64_t>(1, std::min<int64_t>({by_rows, CONV_PART_FLOATS / E, 65535}));
}

// one CTA per slot: dX[t, k] = sum over (h, f) with p* <= t < p* + h of g[h, f] W_h[t - p*, k, f] (h, then f
// ascending), then + sum_f gv[k, f] Wv[t, f] (f ascending).  The slot's g, p* and gv are staged in shared memory.
__global__ void __launch_bounds__(CONV_THREADS) caser_dx_kernel(const __grid_constant__ CaserBwdParams q) {
  extern __shared__ float sm[];
  const int T = q.T, K = q.K, nh = q.nh, nv = q.nv, nhor = T * nh, nver = K * nv;
  int* sa = reinterpret_cast<int*>(sm);
  float* sg = sm + nhor;
  float* sv = sg + nhor;
  const int64_t s = blockIdx.x;
  for (int i = threadIdx.x; i < nhor; i += blockDim.x) {
    const int a = __ldg(q.arg + s * nhor + i);
    sa[i] = a;
    sg[i] = a >= 0 ? __ldg(q.dF + s * q.ldf + i) : 0.f;
  }
  for (int i = threadIdx.x; i < nver; i += blockDim.x)
    sv[i] = __ldg(q.feat + s * q.ldfe + nhor + i) > 0.f ? __ldg(q.dF + s * q.ldf + nhor + i) : 0.f;
  __syncthreads();
  const float* Wv = q.w + (int64_t)K * nh * T * (T + 1) / 2 + T * nh;
  for (int it = threadIdx.x; it < T * K; it += blockDim.x) {
    const int t = it / K, k = it - t * K;
    float acc = 0.f;
    for (int h = 1; h <= T; ++h) {
      const float* W = q.w + (int64_t)K * nh * (h - 1) * h / 2 + k * nh;
      for (int f = 0; f < nh; ++f) {
        const int i = (h - 1) * nh + f, j = t - sa[i];
        if (sa[i] >= 0 && j >= 0 && j < h) acc = fmaf(sg[i], __ldg(W + j * K * nh + f), acc);
      }
    }
    for (int f = 0; f < nv; ++f) acc = fmaf(sv[k * nv + f], __ldg(Wv + t * nv + f), acc);
    q.dX[(s * T + t) * q.lddx + k] = acc;
  }
}

// one thread per (weight element e in the packed layout, chunk of rows): the chunk's sum over its rows, ascending,
// into part[chunk, e]; b200_col_reduce then adds the chunks in a fixed order
__global__ void __launch_bounds__(CONV_THREADS) caser_dw_kernel(const __grid_constant__ CaserBwdParams q) {
  const int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= q.E) return;
  const int T = q.T, K = q.K, nh = q.nh, nv = q.nv, nhor = T * nh;
  const int64_t b0 = (int64_t)blockIdx.y * q.chunk, b1 = min(q.n, b0 + (int64_t)q.chunk);
  const int64_t Eh = (int64_t)K * nh * T * (T + 1) / 2;
  float acc = 0.f;
  if (e < Eh) {                                   // W_h[j, k, f] += g[h, f] x[p* + j, k]
    int h = 1;
    while ((int64_t)K * nh * h * (h + 1) / 2 <= e) ++h;
    const int r = (int)(e - (int64_t)K * nh * (h - 1) * h / 2), j = r / (K * nh), k = (r / nh) % K, f = r % nh;
    const int col = (h - 1) * nh + f;
    for (int64_t b = b0; b < b1; ++b) {
      const int a = __ldg(q.arg + b * nhor + col);
      if (a >= 0) acc = fmaf(__ldg(q.dF + b * q.ldf + col), __ldg(q.X + (b * T + a + j) * q.ldx + k), acc);
    }
  } else if (e < Eh + nhor) {                     // b_h[f] += g[h, f]
    const int col = (int)(e - Eh);
    for (int64_t b = b0; b < b1; ++b)
      if (__ldg(q.arg + b * nhor + col) >= 0) acc += __ldg(q.dF + b * q.ldf + col);
  } else if (e < Eh + nhor + T * nv) {            // Wv[t, f] += sum_k gv[k, f] x[t, k]
    const int r = (int)(e - Eh - nhor), t = r / nv, f = r % nv;
    for (int64_t b = b0; b < b1; ++b)
      for (int k = 0; k < K; ++k) {
        const int64_t c = nhor + k * nv + f;
        if (__ldg(q.feat + b * q.ldfe + c) > 0.f)
          acc = fmaf(__ldg(q.dF + b * q.ldf + c), __ldg(q.X + (b * T + t) * q.ldx + k), acc);
      }
  } else {                                        // bv[f] += sum_k gv[k, f]
    const int f = (int)(e - Eh - nhor - T * nv);
    for (int64_t b = b0; b < b1; ++b)
      for (int k = 0; k < K; ++k) {
        const int64_t c = nhor + k * nv + f;
        if (__ldg(q.feat + b * q.ldfe + c) > 0.f) acc += __ldg(q.dF + b * q.ldf + c);
      }
  }
  q.part[blockIdx.y * q.E + e] = acc;
}

// ---- WaveNet backward: the position work around the dense products ------------------------------------------------
// dZ[s * T + t, f] = dF[s, f] where t is the saved argmax of (s, f), else 0
__global__ void wavenet_pool_backward_kernel(int64_t n, int T, int F, const float* __restrict__ dF, int64_t ldf,
                                             const int32_t* __restrict__ arg, float* __restrict__ dZ) {
  const int64_t total = n * T * F;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t s = i / ((int64_t)T * F);
    const int r = (int)(i - s * T * F), t = r / F, f = r - t * F;
    dZ[i] = __ldg(arg + s * F + f) == t ? __ldg(dF + s * ldf + f) : 0.f;
  }
}

// out[s * T + t] = [x[s * T + t - d] (0 for t < d) | x[s * T + t]], [n * T, 2C]
__global__ void wavenet_layer_inputs_kernel(const float* __restrict__ x, int64_t ldx, int64_t n, int T, int C, int d,
                                            float* __restrict__ out) {
  const int64_t total = n * T * 2 * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / (2 * C);
    const int c = (int)(i - row * 2 * C), t = (int)(row % T);
    float v;
    if (c >= C) v = __ldg(x + row * ldx + c - C);
    else v = t >= d ? __ldg(x + (row - d) * ldx + c) : 0.f;
    out[i] = v;
  }
}

// dx[s * T + t, c] = P[s * T + t, C + c] + P[s * T + t + d, c] (the second term while t + d < T, tested as
// d < T - t so that a dilation near INT32_MAX cannot overflow into a read past the slot)
__global__ void wavenet_layer_dx_kernel(const float* __restrict__ P, int64_t n, int T, int C, int d,
                                        float* __restrict__ dx, int64_t lddx) {
  const int64_t total = n * T * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t row = i / C;
    const int c = (int)(i - row * C), t = (int)(row % T);
    float v = __ldg(P + row * 2 * C + C + c);
    if (d < T - t) v += __ldg(P + (row + d) * 2 * C + c);
    dx[row * lddx + c] = v;
  }
}

unsigned elem_blocks(int64_t total) {
  return (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(total, 256), 132 * 32));
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

namespace {

int caser_encode_impl(const char* who, bool save, const int64_t* users, int64_t n, const int32_t* seqs, int64_t ld_seq,
                      int32_t T, const float* X, int64_t ldx, int32_t K, int32_t nh, int32_t nv, const float* weights,
                      float* out, int64_t ldo, int32_t* argmax, void* stream) {
  B200_REQUIRE(caser_shape_ok(T, K, nh, nv), "%s: T %d, K %d, nh %d, nv %d outside T <= %d, K <= %d, nh, nv <= %d", who,
               T, K, nh, nv, CONV_MAX_T, CONV_MAX_K, CONV_MAX_FILTERS);
  B200_REQUIRE(n >= 0 && n <= (int64_t)0x7fffffff * CONV_MAX_TILE, "%s: bad slot count %lld", who, (long long)n);
  if (n == 0) return 0;
  B200_REQUIRE(users && seqs && X && weights && out && (!save || argmax), "%s: null pointer", who);
  B200_REQUIRE(ld_seq >= T && ldx >= K && ldo >= (int64_t)T * nh + (int64_t)K * nv, "%s: bad leading dimension", who);
  ConvParams p{};
  p.T = T; p.K = K; p.nh = nh; p.nv = nv;
  p.users = users; p.n = n; p.seqs = seqs; p.ld_seq = ld_seq; p.X = X; p.ldx = ldx; p.w = weights;
  p.out = out; p.ldo = ldo; p.arg = argmax;
  p.us = (T * K) | 1;
  return save ? conv_launch(who, caser_encode_kernel<true>, p, 1, stream)
              : conv_launch(who, caser_encode_kernel<false>, p, 1, stream);
}

int wavenet_encode_impl(const char* who, bool save, const int64_t* users, int64_t n, const int32_t* seqs,
                        int64_t ld_seq, int32_t T, const float* X, int64_t ldx, int32_t K, int32_t n_conv, int32_t F,
                        const int32_t* dilations, const float* weights, float* out, int64_t ldo, float* layer_out,
                        int32_t* argmax, void* stream) {
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
  B200_REQUIRE(users && seqs && X && weights && out && (!save || (layer_out && argmax)), "%s: null pointer", who);
  B200_REQUIRE(ld_seq >= T && ldx >= K && ldo >= F, "%s: bad leading dimension", who);
  p.T = T; p.K = K; p.F = F; p.L = n_conv; p.ldc = std::max(K, F) | 1; p.us = (T * p.ldc) | 1;
  p.users = users; p.n = n; p.seqs = seqs; p.ld_seq = ld_seq; p.X = X; p.ldx = ldx; p.w = weights;
  p.out = out; p.ldo = ldo; p.ys = layer_out; p.arg = argmax;
  return save ? conv_launch(who, wavenet_encode_kernel<true>, p, 2, stream)
              : conv_launch(who, wavenet_encode_kernel<false>, p, 2, stream);
}

}  // namespace

extern "C" int b200_caser_encode(const int64_t* users, int64_t n, const int32_t* seqs, int64_t ld_seq, int32_t T,
                                 const float* X, int64_t ldx, int32_t K, int32_t nh, int32_t nv, const float* weights,
                                 float* out, int64_t ldo, void* stream) {
  return caser_encode_impl("b200_caser_encode", false, users, n, seqs, ld_seq, T, X, ldx, K, nh, nv, weights, out, ldo,
                           nullptr, stream);
}

extern "C" int b200_wavenet_encode(const int64_t* users, int64_t n, const int32_t* seqs, int64_t ld_seq, int32_t T,
                                   const float* X, int64_t ldx, int32_t K, int32_t n_conv, int32_t F,
                                   const int32_t* dilations, const float* weights, float* out, int64_t ldo,
                                   void* stream) {
  return wavenet_encode_impl("b200_wavenet_encode", false, users, n, seqs, ld_seq, T, X, ldx, K, n_conv, F, dilations,
                             weights, out, ldo, nullptr, nullptr, stream);
}

extern "C" int b200_caser_train_forward(const int64_t* users, int64_t n, const int32_t* seqs, int64_t ld_seq,
                                        int32_t T, const float* X, int64_t ldx, int32_t K, int32_t nh, int32_t nv,
                                        const float* weights, float* out, int64_t ldo, int32_t* argmax, void* stream) {
  return caser_encode_impl("b200_caser_train_forward", true, users, n, seqs, ld_seq, T, X, ldx, K, nh, nv, weights,
                           out, ldo, argmax, stream);
}

extern "C" int b200_wavenet_train_forward(const int64_t* users, int64_t n, const int32_t* seqs, int64_t ld_seq,
                                          int32_t T, const float* X, int64_t ldx, int32_t K, int32_t n_conv, int32_t F,
                                          const int32_t* dilations, const float* weights, float* out, int64_t ldo,
                                          float* layer_out, int32_t* argmax, void* stream) {
  return wavenet_encode_impl("b200_wavenet_train_forward", true, users, n, seqs, ld_seq, T, X, ldx, K, n_conv, F,
                             dilations, weights, out, ldo, layer_out, argmax, stream);
}

extern "C" int64_t b200_caser_backward_workspace_floats(int64_t n, int32_t T, int32_t K, int32_t nh, int32_t nv) {
  if (!caser_shape_ok(T, K, nh, nv) || n < 0) return -2;
  const int64_t E = caser_floats(T, K, nh, nv);
  return n == 0 ? 0 : (int64_t)caser_nchunk(n, E) * E;
}

extern "C" int b200_caser_backward(int64_t n, int32_t T, int32_t K, int32_t nh, int32_t nv, const float* dF,
                                   int64_t ldf, const float* feat, int64_t ldfe, const int32_t* argmax, const float* X,
                                   int64_t ldx, const float* weights, float* dX, int64_t lddx, float* dW,
                                   float* workspace, int64_t workspace_floats, void* stream) {
  const char* who = "b200_caser_backward";
  B200_REQUIRE(caser_shape_ok(T, K, nh, nv), "%s: T %d, K %d, nh %d, nv %d outside T <= %d, K <= %d, nh, nv <= %d", who,
               T, K, nh, nv, CONV_MAX_T, CONV_MAX_K, CONV_MAX_FILTERS);
  B200_REQUIRE(n >= 0 && n <= 0x7fffffff, "%s: bad slot count %lld", who, (long long)n);
  if (n == 0) return 0;
  B200_REQUIRE(dF && feat && argmax && X && weights && dX && dW && workspace, "%s: null pointer", who);
  const int64_t D = (int64_t)T * nh + (int64_t)K * nv;
  B200_REQUIRE(ldf >= D && ldfe >= D && ldx >= K && lddx >= K, "%s: bad leading dimension", who);
  CaserBwdParams q{};
  q.T = T; q.K = K; q.nh = nh; q.nv = nv; q.n = n; q.E = caser_floats(T, K, nh, nv);
  q.nchunk = caser_nchunk(n, q.E);
  q.chunk = (int)((n + q.nchunk - 1) / q.nchunk);
  B200_REQUIRE(workspace_floats >= q.nchunk * q.E, "%s: workspace of %lld floats, %lld needed", who,
               (long long)workspace_floats, (long long)(q.nchunk * q.E));
  q.dF = dF; q.ldf = ldf; q.feat = feat; q.ldfe = ldfe; q.arg = argmax; q.X = X; q.ldx = ldx; q.w = weights;
  q.dX = dX; q.lddx = lddx; q.part = workspace;
  cudaStream_t st = (cudaStream_t)stream;
  const size_t smem = (size_t)(2 * T * nh + K * nv) * sizeof(float);
  caser_dx_kernel<<<(unsigned)n, CONV_THREADS, smem, st>>>(q);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  caser_dw_kernel<<<dim3((unsigned)ceil_div64(q.E, CONV_THREADS), (unsigned)q.nchunk), CONV_THREADS, 0, st>>>(q);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  B200_CUDA_OK(cudaMemsetAsync(dW, 0, (size_t)q.E * sizeof(float), st));
  return b200_col_reduce(workspace, q.E, q.nchunk, (int32_t)q.E, nullptr, nullptr, 0, dW, stream);
}

extern "C" int b200_wavenet_pool_backward(int64_t n, int32_t T, int32_t F, const float* dF, int64_t ldf,
                                          const int32_t* argmax, float* dZ, void* stream) {
  const char* who = "b200_wavenet_pool_backward";
  B200_REQUIRE(T >= 1 && T <= CONV_MAX_T && F >= 1 && F <= CONV_MAX_F, "%s: T %d, F %d outside T <= %d, F <= %d", who,
               T, F, CONV_MAX_T, CONV_MAX_F);
  B200_REQUIRE(n >= 0, "%s: bad slot count %lld", who, (long long)n);
  if (n == 0) return 0;
  B200_REQUIRE(dF && argmax && dZ, "%s: null pointer", who);
  B200_REQUIRE(ldf >= F, "%s: bad leading dimension", who);
  wavenet_pool_backward_kernel<<<elem_blocks(n * T * F), 256, 0, (cudaStream_t)stream>>>(n, T, F, dF, ldf, argmax, dZ);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_wavenet_layer_inputs(const float* x, int64_t ldx, int64_t n, int32_t T, int32_t C,
                                         int32_t dilation, float* out, void* stream) {
  const char* who = "b200_wavenet_layer_inputs";
  B200_REQUIRE(T >= 1 && T <= CONV_MAX_T && C >= 1 && C <= std::max(CONV_MAX_K, CONV_MAX_F) && dilation >= 1,
               "%s: T %d, C %d, dilation %d outside T <= %d, C <= %d, dilation >= 1", who, T, C, dilation, CONV_MAX_T,
               std::max(CONV_MAX_K, CONV_MAX_F));
  B200_REQUIRE(n >= 0, "%s: bad slot count %lld", who, (long long)n);
  if (n == 0) return 0;
  B200_REQUIRE(x && out, "%s: null pointer", who);
  B200_REQUIRE(ldx >= C, "%s: bad leading dimension", who);
  wavenet_layer_inputs_kernel<<<elem_blocks(n * T * 2 * C), 256, 0, (cudaStream_t)stream>>>(x, ldx, n, T, C, dilation,
                                                                                            out);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_wavenet_layer_dx(const float* P, int64_t n, int32_t T, int32_t C, int32_t dilation, float* dx,
                                     int64_t lddx, void* stream) {
  const char* who = "b200_wavenet_layer_dx";
  B200_REQUIRE(T >= 1 && T <= CONV_MAX_T && C >= 1 && C <= std::max(CONV_MAX_K, CONV_MAX_F) && dilation >= 1,
               "%s: T %d, C %d, dilation %d outside T <= %d, C <= %d, dilation >= 1", who, T, C, dilation, CONV_MAX_T,
               std::max(CONV_MAX_K, CONV_MAX_F));
  B200_REQUIRE(n >= 0, "%s: bad slot count %lld", who, (long long)n);
  if (n == 0) return 0;
  B200_REQUIRE(P && dx, "%s: null pointer", who);
  B200_REQUIRE(lddx >= C, "%s: bad leading dimension", who);
  wavenet_layer_dx_kernel<<<elem_blocks(n * T * C), 256, 0, (cudaStream_t)stream>>>(P, n, T, C, dilation, dx, lddx);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
