// AutoInt inference (libreco/algorithms/autoint.py:146-168, layers/attention.py:67-138): L layers of
// multi-head self-attention ACROSS the F field embeddings of one (user, item) pair, then Dense(1) on the
// flattened block.  One warp owns one pair; its block X [F, K] and the per-layer projections stay in
// shared memory, so a pair costs one read of its field embeddings and one logit written.
//
// Every stage is a set of independent outputs spread over the 32 lanes (lane = output index mod 32), and
// each output is ONE thread's fixed chain of fmaf over an ascending index — which lane computes it never
// changes its value.  The rows mode (X materialised as the [R, F*K] concat) and the grid mode (X assembled
// from a user-side and an item-side block) run the same device function on the same numbers, so they agree
// bit for bit.
#include <math.h>

#include <algorithm>

#include "../../include/b200reco.h"
#include "common.cuh"

namespace b200 {
namespace {

constexpr int AI_MAX_K = 64;
constexpr int AI_MAX_D = 64;
constexpr int AI_MAX_LAYERS = 4;
constexpr int AI_MAX_F = 130;   // 2 id fields + up to 128 sparse / dense fields
constexpr int AI_WARPS = 8;     // warps (pairs in flight) per CTA when shared memory allows

struct AutoIntParams {
  int F, K, H, L;
  int hd[AI_MAX_LAYERS];
  int use_residual;
  const float* w;       // per layer: Wq [K, D], Wk [K, D], Wv [K, D], Wo [D, K]; D = H * hd[l], columns head-major
  const float* w_out;   // [F * K]
  float b_out;
  int ldx, ldd, lds;    // shared-memory leading dimensions (odd: lanes reading different rows hit different banks)
};

__host__ __device__ inline int odd_ld(int n) { return n | 1; }

// shared-memory floats one warp needs: X [F, ldx], Q / K / V [F, ldd] each, one 32-row chunk of scores [32, lds]
__host__ __device__ inline int64_t warp_floats(int F, int ldx, int ldd, int lds) {
  return (int64_t)F * ldx + 3 * (int64_t)F * ldd + 32 * (int64_t)lds;
}

// The arithmetic of one pair, X already in shared memory.  Returns the logit (valid in every lane).
__device__ float autoint_pair(const AutoIntParams& p, float* X, float* Q, float* Kt, float* V, float* S, int lane) {
  const int F = p.F, K = p.K, H = p.H, ldx = p.ldx, ldd = p.ldd, lds = p.lds;
  const float* wl = p.w;
  for (int l = 0; l < p.L; ++l) {
    const int hd = p.hd[l], D = H * hd;
    const float* Wq = wl;
    const float* Wo = wl + 3 * K * D;
    // Q, K, V = X Wq, X Wk, X Wv: output (m, f, d), dot over k ascending
    const int FD = F * D;
    for (int idx = lane; idx < 3 * FD; idx += 32) {
      const int m = idx / FD, rem = idx - m * FD, f = rem / D, d = rem - f * D;
      const float* W = Wq + (int64_t)m * K * D + d;
      const float* x = X + f * ldx;
      float acc = 0.f;
      for (int k = 0; k < K; ++k) acc = fmaf(x[k], __ldg(W + (int64_t)k * D), acc);
      float* dst = m == 0 ? Q : (m == 1 ? Kt : V);
      dst[f * ldd + d] = acc;
    }
    __syncwarp();
    // per head h and query field f (row h*F + f): P = softmax_g(<Q_h[f], K_h[g]> / sqrt(hd)), O_h[f] = P V_h;
    // rows in chunks of 32, a lane per row for the scores, then a lane per (row, j) for the weighted sum.
    // O overwrites the Q columns of its own row, which nothing reads afterwards.
    const float scale = 1.0f / sqrtf((float)hd);
    const int HF = H * F;
    for (int c0 = 0; c0 < HF; c0 += 32) {
      const int row = c0 + lane;
      if (row < HF) {
        const int h = row / F, f = row - h * F;
        const float* q = Q + f * ldd + h * hd;
        float* s = S + lane * lds;
        float mx = -INFINITY;
        for (int g = 0; g < F; ++g) {
          const float* kg = Kt + g * ldd + h * hd;
          float acc = 0.f;
          for (int j = 0; j < hd; ++j) acc = fmaf(q[j], kg[j], acc);
          const float v = acc * scale;
          s[g] = v;
          mx = fmaxf(mx, v);
        }
        float sum = 0.f;
        for (int g = 0; g < F; ++g) {
          const float e = expf(s[g] - mx);
          s[g] = e;
          sum += e;
        }
        for (int g = 0; g < F; ++g) s[g] = s[g] / sum;
      }
      __syncwarp();
      const int nrows = min(32, HF - c0);
      for (int idx = lane; idx < nrows * hd; idx += 32) {
        const int rl = idx / hd, j = idx - rl * hd;
        const int r = c0 + rl, h = r / F, f = r - h * F;
        const float* pr = S + rl * lds;
        const float* v = V + h * hd + j;
        float acc = 0.f;
        for (int g = 0; g < F; ++g) acc = fmaf(pr[g], v[g * ldd], acc);
        Q[f * ldd + h * hd + j] = acc;
      }
      __syncwarp();
    }
    // Y = concat_h(O_h) Wo, X = X + Y (use_residual) or X = Y; element (f, k) reads only O and its own X
    for (int idx = lane; idx < F * K; idx += 32) {
      const int f = idx / K, k = idx - f * K;
      const float* o = Q + f * ldd;
      float acc = 0.f;
      for (int d = 0; d < D; ++d) acc = fmaf(o[d], __ldg(Wo + (int64_t)d * K + k), acc);
      X[f * ldx + k] = p.use_residual ? X[f * ldx + k] + acc : acc;
    }
    __syncwarp();
    wl += 4 * (int64_t)K * D;
  }
  // logit = <flatten(X), w_out> + b_out, one chain over the flat index f * K + k
  float acc = 0.f;
  if (lane == 0) {
    for (int f = 0; f < F; ++f)
      for (int k = 0; k < K; ++k) acc = fmaf(X[f * ldx + k], __ldg(p.w_out + f * K + k), acc);
    acc += p.b_out;
  }
  acc = __shfl_sync(0xffffffffu, acc, 0);
  __syncwarp();   // X is rewritten by the next pair
  return acc;
}

// Pair (b, n) for b < B, n < N: warps stride over n, blockIdx.y strides over b (no 64-bit division).
// GRID = false: B = 1, pair n reads X from Xr[n, :F*K], writes out[n].
// GRID = true:  field f reads Xu[b, slot*K..] (map[f] >= 0, slot = map[f]) or Xi[n, slot*K..] (map[f] < 0,
//               slot = -1 - map[f]); writes out[b * ld_out + n].
template <bool GRID>
__global__ void __launch_bounds__(AI_WARPS * 32)
    autoint_kernel(const __grid_constant__ AutoIntParams p, const float* __restrict__ Xr, int64_t ldr,
                   const float* __restrict__ Xi, int64_t ldi, const int32_t* __restrict__ field_map, int64_t B,
                   int64_t N, float* __restrict__ out, int64_t ld_out) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float* X = smem + warp * warp_floats(p.F, p.ldx, p.ldd, p.lds);
  float* Q = X + p.F * p.ldx;
  float* Kt = Q + p.F * p.ldd;
  float* V = Kt + p.F * p.ldd;
  float* S = V + p.F * p.ldd;
  const int K = p.K, FK = p.F * K;
  for (int64_t b = blockIdx.y; b < B; b += gridDim.y) {
    for (int64_t n = (int64_t)blockIdx.x * nw + warp; n < N; n += (int64_t)gridDim.x * nw) {
      if (GRID) {
        const float* xu = Xr + b * ldr;
        const float* xi = Xi + n * ldi;
        for (int idx = lane; idx < FK; idx += 32) {
          const int f = idx / K, k = idx - f * K;
          const int m = __ldg(field_map + f);
          X[f * p.ldx + k] = m >= 0 ? __ldg(xu + m * K + k) : __ldg(xi + (-1 - m) * K + k);
        }
      } else {
        const float* xr = Xr + n * ldr;
        for (int idx = lane; idx < FK; idx += 32) {
          const int f = idx / K, k = idx - f * K;
          X[f * p.ldx + k] = __ldg(xr + idx);
        }
      }
      __syncwarp();
      const float z = autoint_pair(p, X, Q, Kt, V, S, lane);
      if (lane == 0) out[b * ld_out + n] = z;
    }
  }
}

int autoint_setup(AutoIntParams& p, int32_t F, int32_t K, int32_t H, int32_t L, const int32_t* head_dims_host,
                  const float* weights, const float* w_out, float b_out, int32_t use_residual, size_t& warp_bytes,
                  const char* who) {
  B200_REQUIRE(weights && w_out && head_dims_host, "%s: null pointer", who);
  B200_REQUIRE(F >= 2 && F <= AI_MAX_F, "%s: field count %d outside [2, %d]", who, F, AI_MAX_F);
  B200_REQUIRE(K >= 1 && K <= AI_MAX_K, "%s: embed size %d outside [1, %d]", who, K, AI_MAX_K);
  B200_REQUIRE(L >= 1 && L <= AI_MAX_LAYERS, "%s: layer count %d outside [1, %d]", who, L, AI_MAX_LAYERS);
  B200_REQUIRE(H >= 1 && H <= AI_MAX_D, "%s: head count %d outside [1, %d]", who, H, AI_MAX_D);
  int dmax = 1;
  for (int l = 0; l < L; ++l) {
    const int hd = head_dims_host[l];
    B200_REQUIRE(hd >= 1 && H * hd <= AI_MAX_D, "%s: layer %d: num_heads %d x head size %d outside [1, %d]", who, l, H,
                 hd, AI_MAX_D);
    p.hd[l] = hd;
    dmax = dmax > H * hd ? dmax : H * hd;
  }
  p.F = F; p.K = K; p.H = H; p.L = L;
  p.use_residual = use_residual ? 1 : 0;
  p.w = weights; p.w_out = w_out; p.b_out = b_out;
  p.ldx = odd_ld(K); p.ldd = odd_ld(dmax); p.lds = odd_ld(F);
  warp_bytes = (size_t)warp_floats(F, p.ldx, p.ldd, p.lds) * sizeof(float);
  return 0;
}

template <bool GRID>
int autoint_launch(const AutoIntParams& p, size_t warp_bytes, const float* Xr, int64_t ldr, const float* Xi,
                   int64_t ldi, const int32_t* field_map, int64_t B, int64_t N, float* out, int64_t ld_out,
                   void* stream, const char* who) {
  int dev = 0, optin = 0;
  B200_CUDA_OK(cudaGetDevice(&dev));
  B200_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  B200_REQUIRE(warp_bytes <= (size_t)optin, "%s: one pair needs %zu B of shared memory, the device allows %d", who,
               warp_bytes, optin);
  // up to AI_WARPS pairs in flight per CTA, keeping a CTA within ~96 KB so two or more fit on an SM
  int warps = (int)((96 * 1024) / warp_bytes);
  warps = warps < 1 ? 1 : (warps > AI_WARPS ? AI_WARPS : warps);
  const size_t smem = warp_bytes * warps;
  auto kern = autoint_kernel<GRID>;
  if (smem > 48 * 1024) B200_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t cap = (int64_t)(num_sms() > 0 ? num_sms() : 132) * 32;
  const int64_t gx = std::min<int64_t>(ceil_div64(N, warps), cap);
  const int64_t gy = std::min<int64_t>(std::min<int64_t>(B, std::max<int64_t>(1, cap / gx)), 65535);
  kern<<<dim3((unsigned)gx, (unsigned)gy), warps * 32, smem, (cudaStream_t)stream>>>(p, Xr, ldr, Xi, ldi, field_map, B,
                                                                                     N, out, ld_out);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200_autoint_rows(const float* X, int64_t ldx, int64_t R, int32_t F, int32_t K, int32_t num_heads,
                                 int32_t n_layers, const int32_t* head_dims_host, const float* weights,
                                 const float* w_out, float b_out, int32_t use_residual, float* out, void* stream) {
  AutoIntParams p;
  size_t warp_bytes = 0;
  int rc = autoint_setup(p, F, K, num_heads, n_layers, head_dims_host, weights, w_out, b_out, use_residual, warp_bytes,
                         "b200_autoint_rows");
  if (rc != 0) return rc;
  B200_REQUIRE(X && out, "b200_autoint_rows: null pointer");
  B200_REQUIRE(R >= 0 && ldx >= (int64_t)F * K, "b200_autoint_rows: bad shape (R %lld, ldx %lld < F*K %d)", (long long)R,
               (long long)ldx, F * K);
  if (R == 0) return 0;
  return autoint_launch<false>(p, warp_bytes, X, ldx, nullptr, 0, nullptr, 1, R, out, 0, stream, "b200_autoint_rows");
}

extern "C" int b200_autoint_grid(const float* Xu, int64_t ldu, int64_t B, const float* Xi, int64_t ldi, int64_t N,
                                 const int32_t* field_map, int32_t F, int32_t K, int32_t num_heads, int32_t n_layers,
                                 const int32_t* head_dims_host, const float* weights, const float* w_out, float b_out,
                                 int32_t use_residual, float* scores, int64_t ld_scores, void* stream) {
  AutoIntParams p;
  size_t warp_bytes = 0;
  int rc = autoint_setup(p, F, K, num_heads, n_layers, head_dims_host, weights, w_out, b_out, use_residual, warp_bytes,
                         "b200_autoint_grid");
  if (rc != 0) return rc;
  B200_REQUIRE(Xu && Xi && field_map && scores, "b200_autoint_grid: null pointer");
  B200_REQUIRE(B >= 0 && N >= 0 && ld_scores >= N && ldu >= K && ldi >= K, "b200_autoint_grid: bad shape");
  if (B == 0 || N == 0) return 0;
  return autoint_launch<true>(p, warp_bytes, Xu, ldu, Xi, ldi, field_map, B, N, scores, ld_scores, stream,
                              "b200_autoint_grid");
}
