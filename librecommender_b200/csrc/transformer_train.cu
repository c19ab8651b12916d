// Transformer training (libreco/algorithms/transformer.py:203-339 in training mode): the parts of the step that
// are not dense products over the R*T sequence rows.  The Q / K / V / O projections, the FFN and the MLP, with all
// their input and weight gradients, run on the library's dense kernels; what is left is
//   * the masked self-attention core, forward and backward (csrc/attn_core.cuh with the mask on): per (row, head)
//     over T positions, key g visible to query f when g < len or (causal) g <= f;
//   * rms_norm (layers/normalization.py:21-29) forward / backward over rows of width D, saving rstd per row;
//   * the swish / erf-gelu activations from the pre-activation, forward and backward;
//   * the backward of the target attention (tf_attention, layers/attention.py:5-25) whose forward is
//     b200_transformer_target_attention in rows mode.
// lens is clamped to [1, T] everywhere here: the training collator gives every row len >= 1 (position 0 of a
// history is len 1 holding the pad id), so key 0 is always visible and a hidden key's probability is exactly 0
// under either TensorFlow graph's mask (-1e9 added or written).
#include <math.h>

#include <algorithm>

#include "../../include/b200reco.h"
#include "attn_core.cuh"

namespace b200 {
namespace {

constexpr int TT_MAX_T = 64;    // the Transformer envelope of the inference kernels (transformer.cu)
constexpr int TT_MAX_D = 128;
constexpr int ACT_RELU = 1, ACT_SWISH = 2, ACT_GELU = 3;

int tattn_setup(AttnShape& s, int64_t R, int32_t T, int32_t H, int32_t hd, float scale, const int32_t* lens,
                const char* who) {
  B200_REQUIRE(R >= 0, "%s: row count %lld < 0", who, (long long)R);
  B200_REQUIRE(T >= 1 && T <= TT_MAX_T, "%s: sequence length %d outside [1, %d]", who, T, TT_MAX_T);
  B200_REQUIRE(H >= 1 && hd >= 1 && H <= TT_MAX_D && hd <= TT_MAX_D && H * hd <= TT_MAX_D,
               "%s: num_heads %d x head size %d outside [1, %d]", who, H, hd, TT_MAX_D);
  B200_REQUIRE(isfinite(scale), "%s: scale is not finite", who);
  B200_REQUIRE(lens != nullptr, "%s: null lens", who);
  s.F = T; s.H = H; s.hd = hd; s.scale = scale;
  s.ld = odd(hd); s.lds = odd(T);
  return 0;
}

// ---- rms_norm: one warp per row ------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
    rms_forward_kernel(const float* __restrict__ X, int64_t ldx, int64_t R, int D, const float* __restrict__ scale,
                       float* __restrict__ Y, int64_t ldy, float* __restrict__ rstd) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < R; r += nw) {
    const float* x = X + r * ldx;
    float ss = 0.f;
    for (int d = lane; d < D; d += 32) ss = fmaf(x[d], x[d], ss);
    const float rs = rsqrtf(warp_sum(ss) / (float)D + 1e-8f);
    for (int d = lane; d < D; d += 32) Y[r * ldy + d] = x[d] * rs * __ldg(scale + d);
    if (lane == 0) rstd[r] = rs;
  }
}

// dx = rstd (g - x rstd^2 <g, x> / D) with g = dy o scale
__global__ void __launch_bounds__(256)
    rms_backward_kernel(const float* __restrict__ dY, int64_t lddy, const float* __restrict__ X, int64_t ldx,
                        const float* __restrict__ rstd, int64_t R, int D, const float* __restrict__ scale,
                        float* __restrict__ dX, int64_t lddx) {
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < R; r += nw) {
    const float* x = X + r * ldx;
    const float* dy = dY + r * lddy;
    float gx = 0.f;
    for (int d = lane; d < D; d += 32) gx = fmaf(dy[d] * __ldg(scale + d), x[d], gx);
    const float rs = rstd[r];
    const float c = rs * rs * warp_sum(gx) / (float)D;
    for (int d = lane; d < D; d += 32) dX[r * lddx + d] = rs * (dy[d] * __ldg(scale + d) - x[d] * c);
  }
}

// ---- activations from the pre-activation -----------------------------------------------------------------------
__device__ __forceinline__ float act_fwd(int act, float x) {
  if (act == ACT_RELU) return fmaxf(x, 0.f);
  if (act == ACT_SWISH) return x / (1.0f + expf(-x));
  return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f));
}

__device__ __forceinline__ float act_grad(int act, float x) {
  if (act == ACT_RELU) return x > 0.f ? 1.f : 0.f;
  if (act == ACT_SWISH) {
    const float s = 1.0f / (1.0f + expf(-x));
    return s + x * s * (1.0f - s);
  }
  // d/dx 0.5 x (1 + erf(x / sqrt 2)) = 0.5 (1 + erf(x / sqrt 2)) + x exp(-x^2 / 2) / sqrt(2 pi)
  return 0.5f * (1.0f + erff(x * 0.70710678118654752f)) + x * 0.39894228040143268f * expf(-0.5f * x * x);
}

__global__ void act_forward_kernel(const float* __restrict__ x, int64_t n, int act, float* __restrict__ y) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = act_fwd(act, x[i]);
}

__global__ void act_backward_kernel(const float* __restrict__ dy, const float* __restrict__ x, int64_t n, int act,
                                    float* __restrict__ dx) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dx[i] = dy[i] * act_grad(act, x[i]);
}

// ---- target attention backward: one warp per row --------------------------------------------------------------
// p = softmax_t(<q, S_t>) over t < len, out = sum_t p_t S_t (recomputed); ds_t = p_t (<dout, S_t> - <dout, out>),
// dq = sum_t ds_t S_t, dS_t = p_t dout + ds_t q (t < len), 0 (t >= len).  Lane l owns keys l and l + 32 and
// columns l + 32 j.
__global__ void __launch_bounds__(256)
    target_attention_backward_kernel(const float* __restrict__ Qr, int64_t ldq, const float* __restrict__ S, int T,
                                     int D, const int32_t* __restrict__ lens, const float* __restrict__ dout,
                                     int64_t lddo, int64_t R, float* __restrict__ dq, int64_t lddq,
                                     float* __restrict__ dS) {
  constexpr int NJ = TT_MAX_D / 32;
  const int lane = threadIdx.x & 31;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5; r < R; r += nw) {
    const float* q = Qr + r * ldq;
    const float* go = dout + r * lddo;
    const float* s = S + r * T * D;
    const int len = min(max(lens[r], 1), T);
    float l[2], b[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int t = lane + 32 * e;
      float acc = 0.f, accb = 0.f;
      if (t < len) {
        const float* st = s + (int64_t)t * D;
        for (int d = 0; d < D; ++d) {
          const float sv = __ldg(st + d);
          acc = fmaf(__ldg(q + d), sv, acc);
          accb = fmaf(__ldg(go + d), sv, accb);
        }
      }
      l[e] = t < len ? acc : -INFINITY;
      b[e] = accb;
    }
    const float mx = warp_max(fmaxf(l[0], l[1]));
    float ex[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) ex[e] = lane + 32 * e < len ? expf(l[e] - mx) : 0.f;
    const float sum = warp_sum(ex[0] + ex[1]);
    const float pw[2] = {ex[0] / sum, ex[1] / sum};
    float out[NJ], qd[NJ], gd[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int d = lane + 32 * j;
      out[j] = 0.f;
      qd[j] = d < D ? __ldg(q + d) : 0.f;
      gd[j] = d < D ? __ldg(go + d) : 0.f;
    }
    for (int t = 0; t < len; ++t) {
      const float pt = __shfl_sync(0xffffffffu, t < 32 ? pw[0] : pw[1], t & 31);
      const float* st = s + (int64_t)t * D;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int d = lane + 32 * j;
        if (d < D) out[j] = fmaf(pt, __ldg(st + d), out[j]);
      }
    }
    float c = 0.f;
#pragma unroll
    for (int j = 0; j < NJ; ++j) c = fmaf(gd[j], out[j], c);
    c = warp_sum(c);
    const float ds[2] = {pw[0] * (b[0] - c), pw[1] * (b[1] - c)};
    float dqa[NJ];
#pragma unroll
    for (int j = 0; j < NJ; ++j) dqa[j] = 0.f;
    float* dsr = dS + r * T * D;
    for (int t = 0; t < T; ++t) {
      const float pt = __shfl_sync(0xffffffffu, t < 32 ? pw[0] : pw[1], t & 31);
      const float dst = __shfl_sync(0xffffffffu, t < 32 ? ds[0] : ds[1], t & 31);
      const float* st = s + (int64_t)t * D;
      const bool live = t < len;
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int d = lane + 32 * j;
        if (d < D) {
          if (live) dqa[j] = fmaf(dst, __ldg(st + d), dqa[j]);
          dsr[(int64_t)t * D + d] = live ? fmaf(dst, qd[j], pt * gd[j]) : 0.f;
        }
      }
    }
#pragma unroll
    for (int j = 0; j < NJ; ++j) {
      const int d = lane + 32 * j;
      if (d < D) dq[r * lddq + d] = dqa[j];
    }
  }
}

int64_t warp_grid(int64_t rows) {
  return std::max<int64_t>(1, std::min<int64_t>(ceil_div64(rows, 8), (int64_t)(num_sms() > 0 ? num_sms() : 132) * 16));
}

int64_t elem_grid(int64_t n) {
  return std::max<int64_t>(1, std::min<int64_t>(ceil_div64(n, 256), (int64_t)(num_sms() > 0 ? num_sms() : 132) * 16));
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200_transformer_attention_forward(const float* Q, int64_t ldq, const float* K, int64_t ldk,
                                                  const float* V, int64_t ldv, const int32_t* lens, int64_t R,
                                                  int32_t T, int32_t num_heads, int32_t head_dim, int32_t causal,
                                                  float scale, float* O, int64_t ldo, float* lse, void* stream) {
  const char* who = "b200_transformer_attention_forward";
  AttnShape s;
  int rc = tattn_setup(s, R, T, num_heads, head_dim, scale, lens, who);
  if (rc != 0) return rc;
  B200_REQUIRE(Q && K && V && O && lse, "%s: null pointer", who);
  const int64_t D = (int64_t)num_heads * head_dim;
  B200_REQUIRE(ldq >= D && ldk >= D && ldv >= D && ldo >= D, "%s: a row stride is below num_heads x head size %lld",
               who, (long long)D);
  if (R == 0) return 0;
  const int64_t items = R * num_heads;
  return attn_launch(attn_forward_kernel<true>, (size_t)attn_warp_floats(s, 3) * sizeof(float), items, stream, who, s,
                     AttnMask{lens, causal ? 1 : 0}, Q, ldq, K, ldk, V, ldv, items, O, ldo, lse);
}

extern "C" int b200_transformer_attention_backward(const float* Q, int64_t ldq, const float* K, int64_t ldk,
                                                   const float* V, int64_t ldv, const float* O, int64_t ldo,
                                                   const float* lse, const float* dO, int64_t lddo,
                                                   const int32_t* lens, int64_t R, int32_t T, int32_t num_heads,
                                                   int32_t head_dim, int32_t causal, float scale, float* dQ, float* dK,
                                                   float* dV, int64_t ldg, void* stream) {
  const char* who = "b200_transformer_attention_backward";
  AttnShape s;
  int rc = tattn_setup(s, R, T, num_heads, head_dim, scale, lens, who);
  if (rc != 0) return rc;
  B200_REQUIRE(Q && K && V && O && lse && dO && dQ && dK && dV, "%s: null pointer", who);
  const int64_t D = (int64_t)num_heads * head_dim;
  B200_REQUIRE(ldq >= D && ldk >= D && ldv >= D && ldo >= D && lddo >= D && ldg >= D,
               "%s: a row stride is below num_heads x head size %lld", who, (long long)D);
  if (R == 0) return 0;
  const int64_t items = R * num_heads;
  return attn_launch(attn_backward_kernel<true>, (size_t)attn_warp_floats(s, 6) * sizeof(float), items, stream, who, s,
                     AttnMask{lens, causal ? 1 : 0}, Q, ldq, K, ldk, V, ldv, O, ldo, lse, dO, lddo, items, dQ, dK, dV,
                     ldg);
}

extern "C" int b200_rms_norm_forward(const float* X, int64_t ldx, int64_t R, int32_t D, const float* scale, float* Y,
                                     int64_t ldy, float* rstd, void* stream) {
  const char* who = "b200_rms_norm_forward";
  B200_REQUIRE(R >= 0 && D >= 1 && ldx >= D && ldy >= D, "%s: bad shape R %lld, D %d", who, (long long)R, D);
  B200_REQUIRE(X && scale && Y && rstd, "%s: null pointer", who);
  if (R == 0) return 0;
  rms_forward_kernel<<<(unsigned)warp_grid(R), 256, 0, (cudaStream_t)stream>>>(X, ldx, R, D, scale, Y, ldy, rstd);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_rms_norm_backward(const float* dY, int64_t lddy, const float* X, int64_t ldx, const float* rstd,
                                      int64_t R, int32_t D, const float* scale, float* dX, int64_t lddx,
                                      void* stream) {
  const char* who = "b200_rms_norm_backward";
  B200_REQUIRE(R >= 0 && D >= 1 && lddy >= D && ldx >= D && lddx >= D, "%s: bad shape R %lld, D %d", who,
               (long long)R, D);
  B200_REQUIRE(dY && X && rstd && scale && dX, "%s: null pointer", who);
  if (R == 0) return 0;
  rms_backward_kernel<<<(unsigned)warp_grid(R), 256, 0, (cudaStream_t)stream>>>(dY, lddy, X, ldx, rstd, R, D, scale,
                                                                                dX, lddx);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_activation_forward(const float* x, int64_t n, int32_t act, float* y, void* stream) {
  const char* who = "b200_activation_forward";
  B200_REQUIRE(act == ACT_RELU || act == ACT_SWISH || act == ACT_GELU, "%s: activation code %d not in {1, 2, 3}", who,
               act);
  B200_REQUIRE(n >= 0, "%s: n %lld < 0", who, (long long)n);
  B200_REQUIRE(x && y, "%s: null pointer", who);
  if (n == 0) return 0;
  act_forward_kernel<<<(unsigned)elem_grid(n), 256, 0, (cudaStream_t)stream>>>(x, n, act, y);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_activation_backward(const float* dy, const float* x, int64_t n, int32_t act, float* dx,
                                        void* stream) {
  const char* who = "b200_activation_backward";
  B200_REQUIRE(act == ACT_RELU || act == ACT_SWISH || act == ACT_GELU, "%s: activation code %d not in {1, 2, 3}", who,
               act);
  B200_REQUIRE(n >= 0, "%s: n %lld < 0", who, (long long)n);
  B200_REQUIRE(dy && x && dx, "%s: null pointer", who);
  if (n == 0) return 0;
  act_backward_kernel<<<(unsigned)elem_grid(n), 256, 0, (cudaStream_t)stream>>>(dy, x, n, act, dx);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_transformer_target_attention_backward(const float* Q, int64_t ldq, const float* S, int32_t T,
                                                          int32_t D, const int32_t* lens, const float* dout,
                                                          int64_t lddo, int64_t R, float* dq, int64_t lddq, float* dS,
                                                          void* stream) {
  const char* who = "b200_transformer_target_attention_backward";
  B200_REQUIRE(T >= 1 && T <= TT_MAX_T, "%s: sequence length %d outside [1, %d]", who, T, TT_MAX_T);
  B200_REQUIRE(D >= 1 && D <= TT_MAX_D, "%s: model width %d outside [1, %d]", who, D, TT_MAX_D);
  B200_REQUIRE(R >= 0 && ldq >= D && lddo >= D && lddq >= D, "%s: bad shape", who);
  B200_REQUIRE(Q && S && lens && dout && dq && dS, "%s: null pointer", who);
  if (R == 0) return 0;
  target_attention_backward_kernel<<<(unsigned)warp_grid(R), 256, 0, (cudaStream_t)stream>>>(
      Q, ldq, S, T, D, lens, dout, lddo, R, dq, lddq, dS);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
