// The attention core of one multi-head self-attention layer, forward and exact backward, shared by AutoInt
// training (csrc/autoint_train.cu, F fields per row, no mask) and Transformer training (csrc/transformer_train.cu,
// T sequence positions per row, the padding / causal mask).  Per (row r, head h) with Q_h, K_h, V_h [F, hd]:
//   S = scale * Q_h K_h^T,  P = softmax_rows(S),  O_h = P V_h,  lse_f = log sum_g exp(S_fg)
// and its backward
//   dV_h = P^T dO_h,  dP = dO_h V_h^T,  dS = P o (dP - rowsum(dO_h o O_h)),  dQ_h = scale dS K_h,
//   dK_h = scale dS^T Q_h.
// With MASK, key g is visible to query f when g < len_r, or g <= f when `causal` is set; a hidden key gets
// probability exactly 0 (its score is never formed; callers guarantee len_r >= 1, so key 0 is always visible).
// One warp owns one (row, head).  Its Q, K, V (and for the backward dO, dK, dV) live in shared memory; P is
// never stored in global memory: the backward recomputes it from the saved lse, 32 query fields at a time.
// dK and dV accumulate in shared memory over those query chunks, each element in one lane's fixed chain, so
// there are no atomics and two identical calls give identical bits.
#pragma once

#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace b200 {
namespace {

constexpr int AT_WARPS = 8;     // warps ((row, head) items in flight) per CTA when shared memory allows

struct AttnShape {
  int F, H, hd, ld, lds;        // ld, lds: odd shared-memory leading dimensions (rows in different banks)
  float scale;
};

// the mask of one row: lens [R] (already clamped to [1, F] by the caller) and the causal flag
struct AttnMask {
  const int32_t* lens;
  int causal;
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

template <bool MASK>
__device__ inline bool visible(int f, int g, int len, int causal) {
  return !MASK || g < len || (causal && g <= f);
}

template <bool MASK>
__device__ inline int row_len(const AttnMask& m, int64_t r, int F) {
  return MASK ? min(max(__ldg(m.lens + r), 1), F) : F;
}

template <bool MASK>
__global__ void __launch_bounds__(AT_WARPS * 32)
    attn_forward_kernel(const AttnShape s, const AttnMask m, const float* __restrict__ Q, int64_t ldq,
                        const float* __restrict__ Kg, int64_t ldk, const float* __restrict__ V, int64_t ldv,
                        int64_t items, float* __restrict__ O, int64_t ldo, float* __restrict__ lse) {
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
    const int len = row_len<MASK>(m, r, F);
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
          const float v = visible<MASK>(f, g, len, m.causal) ? dot(q, Ks + g * ld, hd) * s.scale : -INFINITY;
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

template <bool MASK>
__global__ void __launch_bounds__(AT_WARPS * 32)
    attn_backward_kernel(const AttnShape s, const AttnMask m, const float* __restrict__ Q, int64_t ldq,
                         const float* __restrict__ Kg, int64_t ldk, const float* __restrict__ V, int64_t ldv,
                         const float* __restrict__ O, int64_t ldo, const float* __restrict__ lse,
                         const float* __restrict__ dO, int64_t lddo, int64_t items, float* __restrict__ dQ,
                         float* __restrict__ dK, float* __restrict__ dV, int64_t ldg) {
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
    const int len = row_len<MASK>(m, r, F);
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
        for (int g = 0; g < F; ++g)
          p[g] = visible<MASK>(f, g, len, m.causal) ? expf(dot(q, Ks + g * ld, hd) * s.scale - l) : 0.f;
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
