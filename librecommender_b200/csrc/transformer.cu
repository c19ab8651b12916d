// Transformer inference (libreco/algorithms/transformer.py:203-339, a BST-style ranking model).
//
// Everything up to the encoded sequence S_u [T, D] depends on the user only, so it runs ONCE per user of a call
// (b200_transformer_encode: one CTA owns one sequence and runs all L layers with it in shared memory).  The
// per-pair part is the target attention of the item query q_n = [rms_item(G[n]) || 1..1] over S_u and the MLP.
// The first MLP layer splits as Pu[u] + Pi[n] + s_u W1_seq, and since s_u = sum_t p_t S_u[t] its last term is
// sum_t p_t V'_u[t] with V'_u = S_u W1_seq [T, H1] made once per user: b200_transformer_pair_scores then costs a
// pair len*D FMAs for the logits, a masked softmax, len*H1 FMAs for the mix and the small swish layers.
// b200_transformer_target_attention is the rows form: one warp per explicit (slot, item) row writes s_u.
//
// Masked attention scores are fl32(score - 1e9) as Keras adds the mask (softmax of MultiHeadAttention, and
// tf.keras.layers.Attention); for a row with every key masked (len = 0) the weights are therefore the softmax
// of those rounded values, uniform whenever |score| < 32.
#include <math.h>

#include <algorithm>

#include "../../include/b200reco.h"
#include "common.cuh"

namespace b200 {
namespace {

constexpr int TF_MAX_T = 64;
constexpr int TF_MAX_D = 128;
constexpr int TF_MAX_LAYERS = 4;
constexpr int ENC_THREADS = 256;
constexpr float MASK_NEG = 1.0e9f;

__host__ __device__ inline int odd_ld(int n) { return n | 1; }
__host__ __device__ inline int round_up(int n, int m) { return (n + m - 1) / m * m; }

__device__ __forceinline__ float gelu_erf(float x) { return 0.5f * x * (1.0f + erff(x * 0.70710678118654752f)); }
__device__ __forceinline__ float swish(float x) { return x / (1.0f + expf(-x)); }

// floats per layer of the packed encoder weights: rms_att [D], Wq, Wk, Wv, Wo [D, D], rms_ffn [D], W1 [D, 4D], W2 [4D, D]
__host__ __device__ inline int64_t layer_floats(int D) { return 2 * (int64_t)D + 12 * (int64_t)D * D; }

struct EncParams {
  int T, Kp, Kpos, D, H, L, causal, ldx, ldp;
  const int64_t* users;
  const int32_t* lens;
  const int32_t* seqs;
  int64_t ld_seq;
  const float* G;
  int64_t ldg;
  const float* pos;
  const float* w;
  const float* rms_last;
  float* S;
};

__host__ __device__ inline int64_t enc_smem_floats(int T, int ldx, int ldp) { return 5 * (int64_t)T * ldx + (int64_t)T * ldp; }

// Xn = X * rsqrt(mean(X^2) + 1e-8) * scale, row by row (layers/normalization.py:21-29); rs: T floats of scratch
__device__ __forceinline__ void rms_rows(const float* X, float* Xn, float* rs, const float* __restrict__ scale, int T, int D, int ldx) {
  const int tid = threadIdx.x, nt = blockDim.x;
  for (int t = tid; t < T; t += nt) {
    const float* x = X + t * ldx;
    float ss = 0.f;
    for (int d = 0; d < D; ++d) ss = fmaf(x[d], x[d], ss);
    rs[t] = rsqrtf(ss / (float)D + 1e-8f);
  }
  __syncthreads();
  for (int i = tid; i < T * D; i += nt) {
    const int t = i / D, d = i - t * D;
    Xn[t * ldx + d] = X[t * ldx + d] * rs[t] * __ldg(scale + d);
  }
  __syncthreads();
}

// One CTA per slot: X = [G[seq_t] || pos_t], L layers of
//   a = MHA(rms(x)) + x;  x = a + W2 gelu(W1 rms(a))
// then S = rms_last(x).  Shared memory: X, Xn, Q, K, V [T, ldx] and the scores P [T, ldp] of one head.
__global__ void __launch_bounds__(ENC_THREADS) transformer_encode_kernel(const __grid_constant__ EncParams p) {
  extern __shared__ float sm[];
  const int T = p.T, D = p.D, ldx = p.ldx, ldp = p.ldp, tid = threadIdx.x, nt = blockDim.x;
  float* X = sm;
  float* Xn = X + T * ldx;
  float* Q = Xn + T * ldx;
  float* Kt = Q + T * ldx;
  float* V = Kt + T * ldx;
  float* P = V + T * ldx;
  const int64_t s = blockIdx.x;
  const int32_t* seq = p.seqs + p.users[s] * p.ld_seq;
  const int len = min(max(p.lens[s], 0), T);
  for (int i = tid; i < T * D; i += nt) {
    const int t = i / D, d = i - t * D;
    X[t * ldx + d] = d < p.Kp ? __ldg(p.G + (int64_t)__ldg(seq + t) * p.ldg + d) : __ldg(p.pos + t * p.Kpos + d - p.Kp);
  }
  __syncthreads();
  const int H = p.H, hd = D / H, TD = T * D;
  const float scale = 1.0f / sqrtf((float)hd);
  const float* wl = p.w;
  for (int l = 0; l < p.L; ++l) {
    const float* Wq = wl + D;
    const float* Wo = Wq + 3 * (int64_t)D * D;
    const float* rms_ffn = Wo + (int64_t)D * D;
    const float* W1 = rms_ffn + D;
    const float* W2 = W1 + 4 * (int64_t)D * D;
    rms_rows(X, Xn, P, wl, T, D, ldx);
    // Q, K, V = Xn Wq, Xn Wk, Xn Wv: output (m, t, d), one chain over k ascending
    for (int i = tid; i < 3 * TD; i += nt) {
      const int m = i / TD, rem = i - m * TD, t = rem / D, d = rem - t * D;
      const float* W = Wq + (int64_t)m * D * D + d;
      const float* x = Xn + t * ldx;
      float acc = 0.f;
      for (int k = 0; k < D; ++k) acc = fmaf(x[k], __ldg(W + (int64_t)k * D), acc);
      Q[(int64_t)m * T * ldx + t * ldx + d] = acc;     // Q, Kt, V are consecutive [T, ldx] blocks
    }
    __syncthreads();
    for (int h = 0; h < H; ++h) {
      const int c0 = h * hd;
      // key k is visible to query q when k < len, OR k <= q under the causal mask (transformer.py:320-326)
      for (int i = tid; i < T * T; i += nt) {
        const int q = i / T, k = i - q * T;
        float acc = 0.f;
        for (int j = 0; j < hd; ++j) acc = fmaf(Q[q * ldx + c0 + j], Kt[k * ldx + c0 + j], acc);
        float v = acc * scale;
        if (!(k < len || (p.causal && k <= q))) v = v - MASK_NEG;
        P[q * ldp + k] = v;
      }
      __syncthreads();
      for (int q = tid; q < T; q += nt) {
        float* row = P + q * ldp;
        float mx = -INFINITY;
        for (int k = 0; k < T; ++k) mx = fmaxf(mx, row[k]);
        float sum = 0.f;
        for (int k = 0; k < T; ++k) {
          const float e = expf(row[k] - mx);
          row[k] = e;
          sum += e;
        }
        for (int k = 0; k < T; ++k) row[k] = row[k] / sum;
      }
      __syncthreads();
      // O_h = P V_h into the Q columns of head h (every score of head h is already formed)
      for (int i = tid; i < T * hd; i += nt) {
        const int q = i / hd, j = i - q * hd;
        float acc = 0.f;
        for (int k = 0; k < T; ++k) acc = fmaf(P[q * ldp + k], V[k * ldx + c0 + j], acc);
        Q[q * ldx + c0 + j] = acc;
      }
      __syncthreads();
    }
    // a = O Wo + x
    for (int i = tid; i < TD; i += nt) {
      const int t = i / D, d = i - t * D;
      const float* o = Q + t * ldx;
      float acc = 0.f;
      for (int k = 0; k < D; ++k) acc = fmaf(o[k], __ldg(Wo + (int64_t)k * D + d), acc);
      X[t * ldx + d] = acc + X[t * ldx + d];
    }
    __syncthreads();
    rms_rows(X, Xn, P, rms_ffn, T, D, ldx);
    // FFN: the 4D hidden in four column chunks of D (into Q); the output chain continues across chunks (in Kt)
    for (int c = 0; c < 4; ++c) {
      for (int i = tid; i < TD; i += nt) {
        const int t = i / D, j = i - t * D;
        const float* x = Xn + t * ldx;
        const float* W = W1 + c * D + j;
        float acc = 0.f;
        for (int k = 0; k < D; ++k) acc = fmaf(x[k], __ldg(W + (int64_t)k * 4 * D), acc);
        Q[t * ldx + j] = gelu_erf(acc);
      }
      __syncthreads();
      for (int i = tid; i < TD; i += nt) {
        const int t = i / D, d = i - t * D;
        const float* hrow = Q + t * ldx;
        const float* W = W2 + (int64_t)c * D * D + d;
        float acc = c ? Kt[t * ldx + d] : 0.f;
        for (int j = 0; j < D; ++j) acc = fmaf(hrow[j], __ldg(W + (int64_t)j * D), acc);
        Kt[t * ldx + d] = acc;
      }
      __syncthreads();
    }
    for (int i = tid; i < TD; i += nt) {
      const int t = i / D, d = i - t * D;
      X[t * ldx + d] = X[t * ldx + d] + Kt[t * ldx + d];
    }
    __syncthreads();
    wl += layer_floats(D);
  }
  rms_rows(X, Xn, P, p.rms_last, T, D, ldx);
  float* out = p.S + s * TD;
  for (int i = tid; i < TD; i += nt) {
    const int t = i / D, d = i - t * D;
    out[i] = Xn[t * ldx + d];
  }
}

// ---- grid mode: every (user b, item n) pair -------------------------------------------------------------------
constexpr int TP_THREADS = 128;
constexpr int TP_ITEMS = 2 * TP_THREADS;   // two items per thread
constexpr int TP_KCH = 32;                 // Qi / Pi columns per staged chunk
constexpr int TP_MAXH2 = 64;
constexpr int TP_MAXH3 = 32;

struct PairArgs {
  const float* Qi;
  int64_t ldq, N;
  const float *S, *Vp, *Pu;
  const int32_t* lens;
  const float* Pi;
  int64_t ldpi;
  int T, D, H1, H2, H3;
  const float *W2, *b2, *W3, *b3, *w_out;
  float b_out;
  float* scores;
  int64_t lds;
};

struct PairLayout {
  int ld_su, ld_v, ld_p, pu_n;
  int64_t w2, w3, pu, su, vp, pm, tile, total;   // float offsets into shared memory
};

__host__ __device__ inline PairLayout pair_layout(int T, int D, int H1) {
  PairLayout L;
  L.ld_su = round_up(D, TP_KCH);      // zero padded to whole chunks: the float4 reads of a chunk stay in the row
  L.ld_v = round_up(H1, TP_KCH);
  L.ld_p = odd_ld(T);
  L.pu_n = round_up(H1, 4);
  L.w2 = 0;
  L.w3 = L.w2 + (int64_t)H1 * TP_MAXH2;
  L.pu = L.w3 + TP_MAXH2 * TP_MAXH3;
  L.su = L.pu + L.pu_n;
  L.vp = L.su + (int64_t)T * L.ld_su;
  L.pm = L.vp + (int64_t)T * L.ld_v;
  L.tile = L.pm + (int64_t)TP_ITEMS * L.ld_p;
  L.total = L.tile + 2 * TP_ITEMS * (TP_KCH + 1);
  return L;
}

// Per tile of TP_ITEMS items the staged chunks are the ceil(D/32) chunks of Qi, then the ceil(H1/32) chunks of Pi;
// the tiles of a block form one stream of chunks, chunk c+1 fetched with cp.async while chunk c is consumed.
// Logits and then softmax weights of the thread's two items live in its two rows of pm.
__global__ void __launch_bounds__(TP_THREADS) transformer_pair_kernel(const PairArgs a) {
  extern __shared__ float sm[];
  const PairLayout L = pair_layout(a.T, a.D, a.H1);
  float* w2 = sm + L.w2;
  float* w3 = sm + L.w3;
  float* pu = sm + L.pu;
  float* su = sm + L.su;
  float* vp = sm + L.vp;
  float* pm = sm + L.pm;
  float* tile = sm + L.tile;
  const int64_t b = blockIdx.y;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int T = a.T, D = a.D, H1 = a.H1;
  for (int i = tid; i < H1 * TP_MAXH2; i += TP_THREADS) {
    const int k = i / TP_MAXH2, j = i % TP_MAXH2;
    w2[i] = j < a.H2 ? a.W2[(size_t)k * a.H2 + j] : 0.f;
  }
  for (int i = tid; i < TP_MAXH2 * TP_MAXH3; i += TP_THREADS) {
    const int k = i / TP_MAXH3, j = i % TP_MAXH3;
    w3[i] = (a.H3 > 0 && k < a.H2 && j < a.H3) ? a.W3[(size_t)k * a.H3 + j] : 0.f;
  }
  for (int i = tid; i < H1; i += TP_THREADS) pu[i] = a.Pu[b * H1 + i];
  for (int i = tid; i < T * L.ld_su; i += TP_THREADS) {
    const int t = i / L.ld_su, d = i - t * L.ld_su;
    su[i] = d < D ? a.S[(b * T + t) * D + d] : 0.f;
  }
  for (int i = tid; i < T * L.ld_v; i += TP_THREADS) {
    const int t = i / L.ld_v, j = i - t * L.ld_v;
    vp[i] = j < H1 ? a.Vp[(b * T + t) * H1 + j] : 0.f;
  }
  __syncthreads();
  const int len = min(max(a.lens[b], 0), T);
  const int nk = len > 0 ? len : T;   // with no valid key every position takes part, each score shifted by -1e9
  const bool all_masked = len == 0;
  const int ncq = (D + TP_KCH - 1) / TP_KCH, nch = (H1 + TP_KCH - 1) / TP_KCH, nc = ncq + nch;
  const int64_t n_iters = a.N > (int64_t)blockIdx.x * TP_ITEMS
                              ? (a.N - (int64_t)blockIdx.x * TP_ITEMS + (int64_t)gridDim.x * TP_ITEMS - 1) /
                                    ((int64_t)gridDim.x * TP_ITEMS)
                              : 0;
  const int64_t n_chunks = n_iters * nc;
  auto fetch = [&](int64_t c) {
    const int64_t base = ((int64_t)blockIdx.x + (c / nc) * gridDim.x) * TP_ITEMS;
    const int ci = (int)(c % nc);
    const bool q = ci < ncq;
    const int kc = (q ? ci : ci - ncq) * TP_KCH;
    const int kw = min(TP_KCH, (q ? D : H1) - kc);
    const float* src = q ? a.Qi : a.Pi;
    const int64_t ld = q ? a.ldq : a.ldpi;
    float* dst = tile + (c & 1) * (TP_ITEMS * (TP_KCH + 1));
    for (int r = wid; r < TP_ITEMS; r += TP_THREADS / 32) {
      const int64_t n = base + r;
      float* d = dst + r * (TP_KCH + 1) + lane;
      if (n < a.N && lane < kw) {
        const uint32_t sa = (uint32_t)__cvta_generic_to_shared(d);
        asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(sa), "l"(src + n * ld + kc + lane) : "memory");
      } else {
        *d = 0.f;
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  // chunk c landed for every thread; returns its buffer
  auto stage = [&](int64_t c) -> const float* {
    if (c + 1 < n_chunks) {
      fetch(c + 1);            // the other buffer: freed by the barrier that ended the previous chunk
      asm volatile("cp.async.wait_group 1;" ::: "memory");
    } else {
      asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    return tile + (c & 1) * (TP_ITEMS * (TP_KCH + 1));
  };
  if (n_chunks > 0) fetch(0);
  float* p0 = pm + tid * L.ld_p;
  float* p1 = pm + (tid + TP_THREADS) * L.ld_p;
  for (int64_t it = 0; it < n_iters; ++it) {
    const int64_t base = ((int64_t)blockIdx.x + it * gridDim.x) * TP_ITEMS;
    // logits <q_n, S_u[t]>: one chain over d ascending per (item, t), continued across the Qi chunks
    for (int ci = 0; ci < ncq; ++ci) {
      const float* tb = stage(it * nc + ci);
      const int kc = ci * TP_KCH;
      float q0[TP_KCH], q1[TP_KCH];
#pragma unroll
      for (int d = 0; d < TP_KCH; ++d) {
        q0[d] = tb[tid * (TP_KCH + 1) + d];
        q1[d] = tb[(tid + TP_THREADS) * (TP_KCH + 1) + d];
      }
      for (int t = 0; t < nk; ++t) {
        float a0 = ci ? p0[t] : 0.f, a1 = ci ? p1[t] : 0.f;
        const float4* srow = reinterpret_cast<const float4*>(su + t * L.ld_su + kc);
#pragma unroll
        for (int d4 = 0; d4 < TP_KCH / 4; ++d4) {
          const float4 s = srow[d4];
          a0 = fmaf(q0[4 * d4 + 0], s.x, a0); a1 = fmaf(q1[4 * d4 + 0], s.x, a1);
          a0 = fmaf(q0[4 * d4 + 1], s.y, a0); a1 = fmaf(q1[4 * d4 + 1], s.y, a1);
          a0 = fmaf(q0[4 * d4 + 2], s.z, a0); a1 = fmaf(q1[4 * d4 + 2], s.z, a1);
          a0 = fmaf(q0[4 * d4 + 3], s.w, a0); a1 = fmaf(q1[4 * d4 + 3], s.w, a1);
        }
        p0[t] = a0;
        p1[t] = a1;
      }
      __syncthreads();   // chunk consumed: its buffer may be refilled
    }
    // masked softmax over the keys: max, expf, an ascending sum, a division (the thread's own rows)
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      float* pr = e ? p1 : p0;
      float mx = -INFINITY;
      for (int t = 0; t < nk; ++t) {
        float v = pr[t];
        if (all_masked) {
          v = v - MASK_NEG;
          pr[t] = v;
        }
        mx = fmaxf(mx, v);
      }
      float sum = 0.f;
      for (int t = 0; t < nk; ++t) {
        const float ex = expf(pr[t] - mx);
        pr[t] = ex;
        sum += ex;
      }
      for (int t = 0; t < nk; ++t) pr[t] = pr[t] / sum;
    }
    float h2[2][TP_MAXH2];
#pragma unroll
    for (int j = 0; j < TP_MAXH2; ++j) { h2[0][j] = 0.f; h2[1][j] = 0.f; }
    for (int ci = 0; ci < nch; ++ci) {
      const float* tbc = stage(it * nc + ncq + ci);
      float* t0 = const_cast<float*>(tbc) + tid * (TP_KCH + 1);
      float* t1 = const_cast<float*>(tbc) + (tid + TP_THREADS) * (TP_KCH + 1);
      const int kc = ci * TP_KCH;
      const int kw = min(TP_KCH, H1 - kc);
      // first layer: h1 = swish(Pu + Pi + sum_t p_t V'[t]), written over the thread's own rows of the chunk
#pragma unroll
      for (int half = 0; half < 2; ++half) {
        float m0[16], m1[16];
#pragma unroll
        for (int j = 0; j < 16; ++j) { m0[j] = 0.f; m1[j] = 0.f; }
        for (int t = 0; t < nk; ++t) {
          const float pa = p0[t], pb = p1[t];
          const float4* vr = reinterpret_cast<const float4*>(vp + t * L.ld_v + kc + 16 * half);
#pragma unroll
          for (int j4 = 0; j4 < 4; ++j4) {
            const float4 v = vr[j4];
            m0[4 * j4 + 0] = fmaf(pa, v.x, m0[4 * j4 + 0]); m1[4 * j4 + 0] = fmaf(pb, v.x, m1[4 * j4 + 0]);
            m0[4 * j4 + 1] = fmaf(pa, v.y, m0[4 * j4 + 1]); m1[4 * j4 + 1] = fmaf(pb, v.y, m1[4 * j4 + 1]);
            m0[4 * j4 + 2] = fmaf(pa, v.z, m0[4 * j4 + 2]); m1[4 * j4 + 2] = fmaf(pb, v.z, m1[4 * j4 + 2]);
            m0[4 * j4 + 3] = fmaf(pa, v.w, m0[4 * j4 + 3]); m1[4 * j4 + 3] = fmaf(pb, v.w, m1[4 * j4 + 3]);
          }
        }
#pragma unroll
        for (int j = 0; j < 16; ++j) {
          const int kk = 16 * half + j;
          if (kk < kw) {
            t0[kk] = swish(pu[kc + kk] + t0[kk] + m0[j]);
            t1[kk] = swish(pu[kc + kk] + t1[kk] + m1[j]);
          }
        }
      }
#pragma unroll 2
      for (int kk = 0; kk < kw; ++kk) {
        const float ha = t0[kk], hb = t1[kk];
        const float4* wrow = reinterpret_cast<const float4*>(w2 + (size_t)(kc + kk) * TP_MAXH2);
#pragma unroll
        for (int j4 = 0; j4 < TP_MAXH2 / 4; ++j4) {
          const float4 w = wrow[j4];
          h2[0][4 * j4 + 0] = fmaf(ha, w.x, h2[0][4 * j4 + 0]);
          h2[0][4 * j4 + 1] = fmaf(ha, w.y, h2[0][4 * j4 + 1]);
          h2[0][4 * j4 + 2] = fmaf(ha, w.z, h2[0][4 * j4 + 2]);
          h2[0][4 * j4 + 3] = fmaf(ha, w.w, h2[0][4 * j4 + 3]);
          h2[1][4 * j4 + 0] = fmaf(hb, w.x, h2[1][4 * j4 + 0]);
          h2[1][4 * j4 + 1] = fmaf(hb, w.y, h2[1][4 * j4 + 1]);
          h2[1][4 * j4 + 2] = fmaf(hb, w.z, h2[1][4 * j4 + 2]);
          h2[1][4 * j4 + 3] = fmaf(hb, w.w, h2[1][4 * j4 + 3]);
        }
      }
      __syncthreads();
    }
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int64_t n = base + tid + e * TP_THREADS;
      if (n >= a.N) continue;
      float out = a.b_out;
      if (a.H3 > 0) {
        float v[TP_MAXH2];
#pragma unroll
        for (int k = 0; k < TP_MAXH2; ++k) v[k] = k < a.H2 ? swish(h2[e][k] + __ldg(a.b2 + k)) : 0.f;
#pragma unroll 1
        for (int j = 0; j < a.H3; ++j) {
          float h3 = 0.f;
#pragma unroll
          for (int k = 0; k < TP_MAXH2; ++k) h3 = fmaf(v[k], w3[k * TP_MAXH3 + j], h3);
          out = fmaf(h3 + __ldg(a.b3 + j), __ldg(a.w_out + j), out);
        }
      } else {
#pragma unroll
        for (int j = 0; j < TP_MAXH2; ++j)
          if (j < a.H2) out = fmaf(h2[e][j] + __ldg(a.b2 + j), __ldg(a.w_out + j), out);
      }
      a.scores[b * a.lds + n] = out;
    }
  }
}

// ---- rows mode: one warp per (slot, item) row writes s_u = sum_t p_t S[slot, t] ---------------------------------
__global__ void __launch_bounds__(256)
    transformer_target_attention_kernel(const float* __restrict__ Qi, int64_t ldq, const float* __restrict__ S, int T,
                                        int D, const int32_t* __restrict__ lens, const int32_t* __restrict__ slot_of_row,
                                        const int64_t* __restrict__ items, int64_t n, int64_t grid_items,
                                        int64_t row_offset, float* __restrict__ out, int64_t ldo) {
  const int lane = threadIdx.x & 31;
  const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  for (int64_t r = w0; r < n; r += nw) {
    const int64_t slot = slot_of_row ? (int64_t)slot_of_row[r] : (row_offset + r) / grid_items;
    const int64_t item = items ? items[r] : (row_offset + r) % grid_items;
    const float* q = Qi + item * ldq;
    const float* s = S + slot * T * D;
    const int len = min(max(lens[slot], 0), T);
    const int nk = len > 0 ? len : T;
    // logits: lane owns keys t = lane and lane + 32
    float l[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) {
      const int t = lane + 32 * e;
      float acc = 0.f;
      if (t < nk) {
        const float* st = s + (int64_t)t * D;
        for (int d = 0; d < D; ++d) acc = fmaf(__ldg(q + d), __ldg(st + d), acc);
        if (len == 0) acc = acc - MASK_NEG;
      }
      l[e] = t < nk ? acc : -INFINITY;
    }
    const float mx = warp_max(fmaxf(l[0], l[1]));
    float ex[2];
#pragma unroll
    for (int e = 0; e < 2; ++e) ex[e] = lane + 32 * e < nk ? expf(l[e] - mx) : 0.f;
    const float sum = warp_sum(ex[0] + ex[1]);
    const float pw[2] = {ex[0] / sum, ex[1] / sum};
    float acc[TF_MAX_D / 32];
#pragma unroll
    for (int j = 0; j < TF_MAX_D / 32; ++j) acc[j] = 0.f;
    for (int t = 0; t < nk; ++t) {
      const float pt = __shfl_sync(0xffffffffu, t < 32 ? pw[0] : pw[1], t & 31);
      const float* st = s + (int64_t)t * D;
#pragma unroll
      for (int j = 0; j < TF_MAX_D / 32; ++j) {
        const int d = lane + 32 * j;
        if (d < D) acc[j] = fmaf(pt, __ldg(st + d), acc[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < TF_MAX_D / 32; ++j) {
      const int d = lane + 32 * j;
      if (d < D) out[r * ldo + d] = acc[j];
    }
  }
}

int check_tfm_shape(int32_t T, int32_t D, const char* who) {
  B200_REQUIRE(T >= 1 && T <= TF_MAX_T, "%s: sequence length %d outside [1, %d]", who, T, TF_MAX_T);
  B200_REQUIRE(D >= 1 && D <= TF_MAX_D, "%s: model width %d outside [1, %d]", who, D, TF_MAX_D);
  return 0;
}

int smem_optin(int& optin) {
  int dev = 0;
  B200_CUDA_OK(cudaGetDevice(&dev));
  B200_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  return 0;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200_transformer_encode(const int64_t* users, int64_t n_slots, const int32_t* lens, const int32_t* seqs,
                                       int64_t ld_seq, const float* G, int64_t ldg, int32_t Kp, const float* pos,
                                       int32_t Kpos, int32_t T, int32_t num_heads, int32_t n_layers, int32_t causal,
                                       const float* weights, const float* rms_last, float* S, void* stream) {
  const char* who = "b200_transformer_encode";
  B200_REQUIRE(users && lens && seqs && G && pos && weights && rms_last && S, "%s: null pointer", who);
  const int D = Kp + Kpos;
  B200_REQUIRE(Kp >= 1 && Kpos >= 1, "%s: item width %d and position width %d must be >= 1", who, Kp, Kpos);
  int rc = check_tfm_shape(T, D, who);
  if (rc != 0) return rc;
  B200_REQUIRE(n_layers >= 1 && n_layers <= TF_MAX_LAYERS, "%s: layer count %d outside [1, %d]", who, n_layers,
               TF_MAX_LAYERS);
  B200_REQUIRE(num_heads >= 1 && D % num_heads == 0, "%s: width %d is not a multiple of num_heads %d", who, D, num_heads);
  B200_REQUIRE(n_slots >= 0 && n_slots <= 0x7fffffff && ld_seq >= T && ldg >= Kp, "%s: bad shape", who);
  if (n_slots == 0) return 0;
  EncParams p;
  p.T = T; p.Kp = Kp; p.Kpos = Kpos; p.D = D; p.H = num_heads; p.L = n_layers; p.causal = causal ? 1 : 0;
  p.ldx = odd_ld(D); p.ldp = odd_ld(T);
  p.users = users; p.lens = lens; p.seqs = seqs; p.ld_seq = ld_seq; p.G = G; p.ldg = ldg; p.pos = pos;
  p.w = weights; p.rms_last = rms_last; p.S = S;
  const size_t smem = (size_t)enc_smem_floats(T, p.ldx, p.ldp) * sizeof(float);
  int optin = 0;
  rc = smem_optin(optin);
  if (rc != 0) return rc;
  B200_REQUIRE(smem <= (size_t)optin, "%s: one sequence needs %zu B of shared memory, the device allows %d", who, smem,
               optin);
  if (smem > 48 * 1024)
    B200_CUDA_OK(cudaFuncSetAttribute(transformer_encode_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  transformer_encode_kernel<<<(unsigned)n_slots, ENC_THREADS, smem, (cudaStream_t)stream>>>(p);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int64_t b200_transformer_pair_smem_bytes(int32_t T, int32_t D, int32_t H1) {
  if (T < 1 || D < 1 || H1 < 1) return -2;
  return pair_layout(T, D, H1).total * (int64_t)sizeof(float);
}

extern "C" int b200_transformer_pair_scores(const float* Qi, int64_t ldq, int64_t N, const float* S, const float* Vp,
                                            const float* Pu, const int32_t* lens, int64_t B, const float* Pi,
                                            int64_t ldpi, int32_t T, int32_t D, int32_t H1, int32_t H2, int32_t H3,
                                            const float* W2, const float* b2, const float* W3, const float* b3,
                                            const float* w_out, float b_out, float* scores, int64_t lds, void* stream) {
  const char* who = "b200_transformer_pair_scores";
  B200_REQUIRE(Qi && S && Vp && Pu && lens && Pi && W2 && b2 && w_out && scores, "%s: null pointer", who);
  int rc = check_tfm_shape(T, D, who);
  if (rc != 0) return rc;
  B200_REQUIRE(H1 >= 1 && H1 <= 256 && H2 >= 1 && H2 <= TP_MAXH2 && H3 >= 0 && H3 <= TP_MAXH3,
               "%s: unsupported layer sizes H=(%d,%d,%d)", who, H1, H2, H3);
  B200_REQUIRE(H3 == 0 || (W3 && b3), "%s: third layer weights missing", who);
  B200_REQUIRE(B >= 0 && B <= 65535 && N >= 0 && ldq >= D && ldpi >= H1 && lds >= N, "%s: bad shape", who);
  const size_t smem = (size_t)b200_transformer_pair_smem_bytes(T, D, H1);
  int optin = 0;
  rc = smem_optin(optin);
  if (rc != 0) return rc;
  B200_REQUIRE(smem <= (size_t)optin, "%s: T %d, D %d, H1 %d need %zu B of shared memory, the device allows %d", who, T,
               D, H1, smem, optin);
  if (B == 0 || N == 0) return 0;
  PairArgs a;
  a.Qi = Qi; a.ldq = ldq; a.N = N; a.S = S; a.Vp = Vp; a.Pu = Pu; a.lens = lens; a.Pi = Pi; a.ldpi = ldpi;
  a.T = T; a.D = D; a.H1 = H1; a.H2 = H2; a.H3 = H3; a.W2 = W2; a.b2 = b2; a.W3 = W3; a.b3 = b3; a.w_out = w_out;
  a.b_out = b_out; a.scores = scores; a.lds = lds;
  if (smem > 48 * 1024)
    B200_CUDA_OK(cudaFuncSetAttribute(transformer_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t cap = (int64_t)(num_sms() > 0 ? num_sms() : 132) * 2;
  const unsigned gx = (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(N, TP_ITEMS), std::max<int64_t>(1, cap / B)));
  transformer_pair_kernel<<<dim3(gx, (unsigned)B), TP_THREADS, smem, (cudaStream_t)stream>>>(a);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_transformer_target_attention(const float* Qi, int64_t ldq, const float* S, int32_t T, int32_t D,
                                                 const int32_t* lens, const int32_t* slot_of_row, const int64_t* items,
                                                 int64_t n, int64_t grid_items, int64_t row_offset, float* out,
                                                 int64_t ldo, void* stream) {
  const char* who = "b200_transformer_target_attention";
  B200_REQUIRE(Qi && S && lens && out, "%s: null pointer", who);
  int rc = check_tfm_shape(T, D, who);
  if (rc != 0) return rc;
  B200_REQUIRE((slot_of_row != nullptr) == (items != nullptr) && (items != nullptr || grid_items > 0),
               "%s: give slot_of_row and items, or grid_items > 0", who);
  B200_REQUIRE(n >= 0 && ldq >= D && ldo >= D && row_offset >= 0, "%s: bad shape", who);
  if (n == 0) return 0;
  const int64_t blocks = std::min<int64_t>(ceil_div64(n, 8), (int64_t)(num_sms() > 0 ? num_sms() : 132) * 16);
  transformer_target_attention_kernel<<<(unsigned)blocks, 256, 0, (cudaStream_t)stream>>>(
      Qi, ldq, S, T, D, lens, slot_of_row, items, n, grid_items, row_offset, out, ldo);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
