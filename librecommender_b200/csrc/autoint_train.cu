// AutoInt training: the attention core of one multi-head self-attention layer across the F fields
// (layers/attention.py:67-125), forward and exact backward.  Everything else in a layer (the Q / K / V
// projections, the output projection and all their gradients) is a dense product over R*F rows and runs on
// the library's dense kernels; what is left is, per (row r, head h) with Q_h, K_h, V_h [F, hd]:
//   S = scale * Q_h K_h^T,  P = softmax_rows(S),  O_h = P V_h,  lse_f = log sum_g exp(S_fg)
// and its backward
//   dV_h = P^T dO_h,  dP = dO_h V_h^T,  dS = P o (dP - rowsum(dO_h o O_h)),  dQ_h = scale dS K_h,
//   dK_h = scale dS^T Q_h.
// One warp owns one (row, head).  Its Q, K, V (and for the backward dO, dK, dV) live in shared memory; P is
// never stored in global memory: the backward recomputes it from the saved lse, 32 query fields at a time.
// dK and dV accumulate in shared memory over those query chunks, each element in one lane's fixed chain, so
// there are no atomics and two identical calls give identical bits.
#include <math.h>

#include <algorithm>

#include "../../include/b200reco.h"
#include "common.cuh"

namespace b200 {
namespace {

constexpr int AT_MAX_F = 130;   // the inference engine's envelope (autoint.cu)
constexpr int AT_MAX_D = 64;
constexpr int AT_WARPS = 8;     // warps ((row, head) items in flight) per CTA when shared memory allows

struct AttnShape {
  int F, H, hd, ld, lds;        // ld, lds: odd shared-memory leading dimensions (rows in different banks)
  float scale;
};

__host__ __device__ inline int odd(int n) { return n | 1; }

// shared-memory floats one warp needs: `mats` [F, ld] matrices plus one 32-query chunk of P / dS [32, lds]
__host__ __device__ inline int64_t attn_warp_floats(const AttnShape& s, int mats) {
  return (int64_t)mats * s.F * s.ld + 32 * (int64_t)s.lds;
}

// rows [r*F, r*F + F) of a [R*F, ld_g] matrix, columns [h*hd, h*hd + hd) -> dst [F, ld]
__device__ inline void stage(float* dst, const float* __restrict__ src, int64_t ld_g, int64_t base, int col0,
                             const AttnShape& s, int lane) {
  for (int idx = lane; idx < s.F * s.hd; idx += 32) {
    const int f = idx / s.hd, j = idx - f * s.hd;
    dst[f * s.ld + j] = __ldg(src + (base + f) * ld_g + col0 + j);
  }
}

__device__ inline float dot(const float* a, const float* b, int n) {
  float acc = 0.f;
  for (int j = 0; j < n; ++j) acc = fmaf(a[j], b[j], acc);
  return acc;
}

__global__ void __launch_bounds__(AT_WARPS * 32)
    attn_forward_kernel(const AttnShape s, const float* __restrict__ Q, int64_t ldq, const float* __restrict__ Kg,
                        int64_t ldk, const float* __restrict__ V, int64_t ldv, int64_t items, float* __restrict__ O,
                        int64_t ldo, float* __restrict__ lse) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int F = s.F, hd = s.hd, ld = s.ld, lds = s.lds;
  float* Qs = smem + warp * attn_warp_floats(s, 3);
  float* Ks = Qs + F * ld;
  float* Vs = Ks + F * ld;
  float* S = Vs + F * ld;
  for (int64_t it = (int64_t)blockIdx.x * nw + warp; it < items; it += (int64_t)gridDim.x * nw) {
    const int64_t r = it / s.H;
    const int h = (int)(it - r * s.H), col0 = h * hd;
    const int64_t base = r * F;
    stage(Qs, Q, ldq, base, col0, s, lane);
    stage(Ks, Kg, ldk, base, col0, s, lane);
    stage(Vs, V, ldv, base, col0, s, lane);
    __syncwarp();
    for (int c0 = 0; c0 < F; c0 += 32) {
      const int f = c0 + lane;
      if (f < F) {                                     // a lane per query field: scores, max, sum, P
        const float* q = Qs + f * ld;
        float* p = S + lane * lds;
        float mx = -INFINITY;
        for (int g = 0; g < F; ++g) {
          const float v = dot(q, Ks + g * ld, hd) * s.scale;
          p[g] = v;
          mx = fmaxf(mx, v);
        }
        float sum = 0.f;
        for (int g = 0; g < F; ++g) {
          const float e = expf(p[g] - mx);
          p[g] = e;
          sum += e;
        }
        for (int g = 0; g < F; ++g) p[g] = p[g] / sum;
        lse[it * F + f] = mx + logf(sum);
      }
      __syncwarp();
      const int nrows = min(32, F - c0);               // a lane per (query field, j): O = P V
      for (int idx = lane; idx < nrows * hd; idx += 32) {
        const int rl = idx / hd, j = idx - rl * hd;
        const float* p = S + rl * lds;
        float acc = 0.f;
        for (int g = 0; g < F; ++g) acc = fmaf(p[g], Vs[g * ld + j], acc);
        O[(base + c0 + rl) * ldo + col0 + j] = acc;
      }
      __syncwarp();
    }
  }
}

__global__ void __launch_bounds__(AT_WARPS * 32)
    attn_backward_kernel(const AttnShape s, const float* __restrict__ Q, int64_t ldq, const float* __restrict__ Kg,
                         int64_t ldk, const float* __restrict__ V, int64_t ldv, const float* __restrict__ O,
                         int64_t ldo, const float* __restrict__ lse, const float* __restrict__ dO, int64_t lddo,
                         int64_t items, float* __restrict__ dQ, float* __restrict__ dK, float* __restrict__ dV,
                         int64_t ldg) {
  extern __shared__ float smem[];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  const int F = s.F, hd = s.hd, ld = s.ld, lds = s.lds, Fhd = F * hd;
  float* Qs = smem + warp * attn_warp_floats(s, 6);
  float* Ks = Qs + F * ld;
  float* Vs = Ks + F * ld;
  float* dOs = Vs + F * ld;
  float* dKs = dOs + F * ld;
  float* dVs = dKs + F * ld;
  float* S = dVs + F * ld;
  for (int64_t it = (int64_t)blockIdx.x * nw + warp; it < items; it += (int64_t)gridDim.x * nw) {
    const int64_t r = it / s.H;
    const int h = (int)(it - r * s.H), col0 = h * hd;
    const int64_t base = r * F;
    stage(Qs, Q, ldq, base, col0, s, lane);
    stage(Ks, Kg, ldk, base, col0, s, lane);
    stage(Vs, V, ldv, base, col0, s, lane);
    stage(dOs, dO, lddo, base, col0, s, lane);
    for (int idx = lane; idx < Fhd; idx += 32) {
      const int g = idx / hd, j = idx - g * hd;
      dKs[g * ld + j] = 0.f;
      dVs[g * ld + j] = 0.f;
    }
    __syncwarp();
    for (int c0 = 0; c0 < F; c0 += 32) {
      const int f = c0 + lane, nrows = min(32, F - c0);
      float* p = S + lane * lds;
      if (f < F) {                                     // P of query f, recomputed from its lse
        const float* q = Qs + f * ld;
        const float l = __ldg(lse + it * F + f);
        for (int g = 0; g < F; ++g) p[g] = expf(dot(q, Ks + g * ld, hd) * s.scale - l);
      }
      __syncwarp();
      for (int idx = lane; idx < Fhd; idx += 32) {     // dV += P^T dO over this chunk's query fields
        const int g = idx / hd, j = idx - g * hd;
        float acc = dVs[g * ld + j];
        for (int rl = 0; rl < nrows; ++rl) acc = fmaf(S[rl * lds + g], dOs[(c0 + rl) * ld + j], acc);
        dVs[g * ld + j] = acc;
      }
      __syncwarp();
      if (f < F) {                                     // P -> scale * dS, in place
        const float* dof = dOs + f * ld;
        const float* of = O + (base + f) * ldo + col0;
        float dsum = 0.f;
        for (int j = 0; j < hd; ++j) dsum = fmaf(dof[j], __ldg(of + j), dsum);
        for (int g = 0; g < F; ++g) p[g] = p[g] * (dot(dof, Vs + g * ld, hd) - dsum) * s.scale;
      }
      __syncwarp();
      for (int idx = lane; idx < nrows * hd; idx += 32) {   // dQ rows of this chunk: complete here
        const int rl = idx / hd, j = idx - rl * hd;
        const float* ds = S + rl * lds;
        float acc = 0.f;
        for (int g = 0; g < F; ++g) acc = fmaf(ds[g], Ks[g * ld + j], acc);
        dQ[(base + c0 + rl) * ldg + col0 + j] = acc;
      }
      for (int idx = lane; idx < Fhd; idx += 32) {     // dK += dS^T Q over this chunk's query fields
        const int g = idx / hd, j = idx - g * hd;
        float acc = dKs[g * ld + j];
        for (int rl = 0; rl < nrows; ++rl) acc = fmaf(S[rl * lds + g], Qs[(c0 + rl) * ld + j], acc);
        dKs[g * ld + j] = acc;
      }
      __syncwarp();
    }
    for (int idx = lane; idx < Fhd; idx += 32) {
      const int g = idx / hd, j = idx - g * hd;
      dK[(base + g) * ldg + col0 + j] = dKs[g * ld + j];
      dV[(base + g) * ldg + col0 + j] = dVs[g * ld + j];
    }
    __syncwarp();                                      // shared memory is restaged for the next item
  }
}

int attn_setup(AttnShape& s, int64_t R, int32_t F, int32_t H, int32_t hd, float scale, const char* who) {
  B200_REQUIRE(R >= 0, "%s: row count %lld < 0", who, (long long)R);
  B200_REQUIRE(F >= 2 && F <= AT_MAX_F, "%s: field count %d outside [2, %d]", who, F, AT_MAX_F);
  B200_REQUIRE(H >= 1 && hd >= 1 && H <= AT_MAX_D && hd <= AT_MAX_D && H * hd <= AT_MAX_D,
               "%s: num_heads %d x head size %d outside [1, %d]", who, H, hd, AT_MAX_D);
  B200_REQUIRE(isfinite(scale), "%s: scale is not finite", who);
  s.F = F; s.H = H; s.hd = hd; s.scale = scale;
  s.ld = odd(hd); s.lds = odd(F);
  return 0;
}

// Up to AT_WARPS items per CTA, keeping a CTA within ~96 KB so two or more fit on an SM.
template <typename Kern, typename... Args>
int attn_launch(Kern kern, size_t warp_bytes, int64_t items, void* stream, const char* who, Args... args) {
  int dev = 0, optin = 0;
  B200_CUDA_OK(cudaGetDevice(&dev));
  B200_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  B200_REQUIRE(warp_bytes <= (size_t)optin, "%s: one (row, head) needs %zu B of shared memory, the device allows %d",
               who, warp_bytes, optin);
  int warps = (int)((96 * 1024) / warp_bytes);
  warps = warps < 1 ? 1 : (warps > AT_WARPS ? AT_WARPS : warps);
  const size_t smem = warp_bytes * warps;
  if (smem > 48 * 1024) B200_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t cap = (int64_t)(num_sms() > 0 ? num_sms() : 132) * 32;
  const int64_t grid = std::min<int64_t>(ceil_div64(items, warps), cap);
  kern<<<(unsigned)grid, warps * 32, smem, (cudaStream_t)stream>>>(args...);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200_autoint_attention_forward(const float* Q, int64_t ldq, const float* K, int64_t ldk,
                                              const float* V, int64_t ldv, int64_t R, int32_t F, int32_t num_heads,
                                              int32_t head_dim, float scale, float* O, int64_t ldo, float* lse,
                                              void* stream) {
  const char* who = "b200_autoint_attention_forward";
  AttnShape s;
  int rc = attn_setup(s, R, F, num_heads, head_dim, scale, who);
  if (rc != 0) return rc;
  B200_REQUIRE(Q && K && V && O && lse, "%s: null pointer", who);
  const int64_t D = (int64_t)num_heads * head_dim;
  B200_REQUIRE(ldq >= D && ldk >= D && ldv >= D && ldo >= D, "%s: a row stride is below num_heads x head size %lld",
               who, (long long)D);
  if (R == 0) return 0;
  const int64_t items = R * num_heads;
  return attn_launch(attn_forward_kernel, (size_t)attn_warp_floats(s, 3) * sizeof(float), items, stream, who, s, Q,
                     ldq, K, ldk, V, ldv, items, O, ldo, lse);
}

extern "C" int b200_autoint_attention_backward(const float* Q, int64_t ldq, const float* K, int64_t ldk,
                                               const float* V, int64_t ldv, const float* O, int64_t ldo,
                                               const float* lse, const float* dO, int64_t lddo, int64_t R, int32_t F,
                                               int32_t num_heads, int32_t head_dim, float scale, float* dQ, float* dK,
                                               float* dV, int64_t ldg, void* stream) {
  const char* who = "b200_autoint_attention_backward";
  AttnShape s;
  int rc = attn_setup(s, R, F, num_heads, head_dim, scale, who);
  if (rc != 0) return rc;
  B200_REQUIRE(Q && K && V && O && lse && dO && dQ && dK && dV, "%s: null pointer", who);
  const int64_t D = (int64_t)num_heads * head_dim;
  B200_REQUIRE(ldq >= D && ldk >= D && ldv >= D && ldo >= D && lddo >= D && ldg >= D,
               "%s: a row stride is below num_heads x head size %lld", who, (long long)D);
  if (R == 0) return 0;
  const int64_t items = R * num_heads;
  return attn_launch(attn_backward_kernel, (size_t)attn_warp_floats(s, 6) * sizeof(float), items, stream, who, s, Q,
                     ldq, K, ldk, V, ldv, O, ldo, lse, dO, lddo, items, dQ, dK, dV, ldg);
}
