// K2 — behaviour-sequence kernels: DIN attention and YouTubeRanking sequence pooling.
//
// Replaces
//   din_attention        libreco/layers/attention.py:28-64   (+ the lookups of din.py:236-250)
//   seq_embeds_pooling   libreco/layers/embedding.py:54-85   (youtube_ranking.py:188-199)
// Sequences come from the per-user cache the reference keeps on the host
// (recent_seqs / recent_seq_lens, libreco/batch/sequence.py:75-91, prediction/preprocess.py:109-118):
// row r uses the sequence of user users[r] or — all-items scoring — users[(r + off) / grid].
// The [B*N, T] repeat of the reference is never materialised.
//
// One warp per row.  DIN: the attention MLP input [q, k, q-k, q*k] W1 is re-associated per row as
//   h_j(t) = c_j + sum_c k_c(t) * M[c][j],   M[c][j] = (W1k - W1d)[c][j] + q_c * W1p[c][j],
//   c_j    = b1_j + sum_c q_c * (W1q + W1d)[c][j]
// (W1q/W1k/W1d/W1p = the four K'-row blocks of the Dense(16) kernel), so the per-key work is one
// K' x 16 mat-vec held in registers; a 16-value butterfly reduction needs 16 shuffles.
#include <algorithm>
#include "common.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace seq {

constexpr int HID = 16;      // attention.py:47  Dense(16)
constexpr int MAX_TK = 4;    // K' <= 128
constexpr int MAX_T = 256;   // sequence length limit

__device__ __forceinline__ int64_t seq_row_of(const int64_t* users, int64_t r, int64_t grid, int64_t off) {
  return grid > 0 ? users[(r + off) / grid] : users[r];
}

__global__ void __launch_bounds__(256)
seq_pool_kernel(const float* __restrict__ E, int64_t lde, int d, int64_t pad_index,
                const int32_t* __restrict__ seqs, int64_t ld_seq, const int32_t* __restrict__ lens, int T,
                const int64_t* __restrict__ users, int64_t R, int64_t grid, int64_t off,
                float* __restrict__ out, int64_t ld_out) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  const int64_t sr = seq_row_of(users, r, grid, off);
  const int32_t* s = seqs + sr * ld_seq;
  const float len = (float)lens[sr];
  const float inv = len > 0.f ? 1.0f / sqrtf(len) : 0.f;          // tf.div_no_nan
  for (int k0 = 0; k0 < d; k0 += 32) {
    const int k = k0 + lane;
    float acc = 0.f;
    for (int t = 0; t < T; ++t) {
      const int32_t it = __ldg(s + t);
      if (it != pad_index && k < d) acc += __ldg(E + (int64_t)it * lde + k);   // pad row reads as zero
    }
    if (k < d) out[r * ld_out + k] = acc * inv;
  }
}

// backward of seq_pool: g[seq_t, :] += dout[r, :] / sqrt(len) for every non-pad position (float atomics)
__global__ void __launch_bounds__(256)
seq_pool_backward_kernel(const float* __restrict__ dout, int64_t ld_dout, int d, int64_t pad_index,
                         const int32_t* __restrict__ seqs, int64_t ld_seq, const int32_t* __restrict__ lens, int T,
                         const int64_t* __restrict__ users, int64_t R, float* __restrict__ g, int64_t ldg) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  const int64_t sr = seq_row_of(users, r, 0, 0);
  const int32_t* s = seqs + sr * ld_seq;
  const float len = (float)lens[sr];
  if (!(len > 0.f)) return;                                        // div_no_nan: the output (and its gradient) is 0
  const float inv = 1.0f / sqrtf(len);
  for (int k0 = 0; k0 < d; k0 += 32) {
    const int k = k0 + lane;
    if (k >= d) continue;
    const float v = dout[r * ld_dout + k] * inv;
    for (int t = 0; t < T; ++t) {
      const int32_t it = __ldg(s + t);
      if (it != pad_index) atomicAdd(g + (int64_t)it * ldg + k, v);
    }
  }
}

struct AttW {
  const float* k1;   // [4K', 16] row-major (Dense(16) kernel; rows: q | k | q-k | q*k)
  const float* b1;   // [16]
  const float* k2;   // [16]      Dense(1) kernel
  float b2;
};

__global__ void __launch_bounds__(128)
din_attention_kernel(const float* __restrict__ G, int64_t ldg, int Kp, const int64_t* __restrict__ items,
                     const int32_t* __restrict__ seqs, int64_t ld_seq, const int32_t* __restrict__ lens, int T,
                     const int64_t* __restrict__ users, int64_t R, int64_t grid, int64_t off, AttW w,
                     float* __restrict__ out, int64_t ld_out) {
  __shared__ float s_att[4][MAX_T];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * 4 + wid;
  if (r >= R) return;
  const int64_t sr = seq_row_of(users, r, grid, off);
  const int64_t item = grid > 0 ? (r + off) % grid : items[r];
  const int32_t* s = seqs + sr * ld_seq;
  const int len = min(max(lens[sr], 0), T);
  const int TK = (Kp + 31) / 32;
  // query row and the per-row matrix M (registers)
  float q[MAX_TK];
  float M[MAX_TK][HID];
  float cpart[HID];
#pragma unroll
  for (int j = 0; j < HID; ++j) cpart[j] = 0.f;
#pragma unroll
  for (int t = 0; t < MAX_TK; ++t) {
    const int c = lane + t * 32;
    q[t] = 0.f;
    if (t < TK && c < Kp) {
      q[t] = __ldg(G + item * ldg + c);
#pragma unroll
      for (int j = 0; j < HID; ++j) {
        const float wq = __ldg(w.k1 + (int64_t)c * HID + j);
        const float wk = __ldg(w.k1 + (int64_t)(Kp + c) * HID + j);
        const float wd = __ldg(w.k1 + (int64_t)(2 * Kp + c) * HID + j);
        const float wp = __ldg(w.k1 + (int64_t)(3 * Kp + c) * HID + j);
        M[t][j] = (wk - wd) + q[t] * wp;
        cpart[j] = fmaf(q[t], wq + wd, cpart[j]);
      }
    } else {
#pragma unroll
      for (int j = 0; j < HID; ++j) M[t][j] = 0.f;
    }
  }
  // c_j: full warp sums (once per row)
#pragma unroll
  for (int j = 0; j < HID; ++j) cpart[j] = warp_sum(cpart[j]) + __ldg(w.b1 + j);
  const float scale = rsqrtf((float)Kp);
  float amax = -3.0e38f;
  for (int t = 0; t < len; ++t) {
    const int64_t key = __ldg(s + t);
    float part[HID];
#pragma unroll
    for (int j = 0; j < HID; ++j) part[j] = 0.f;
#pragma unroll
    for (int tt = 0; tt < MAX_TK; ++tt) {
      const int c = lane + tt * 32;
      if (tt < TK && c < Kp) {
        const float kv = __ldg(G + key * ldg + c);
#pragma unroll
        for (int j = 0; j < HID; ++j) part[j] = fmaf(kv, M[tt][j], part[j]);
      }
    }
    // butterfly: after the stage with offset o each lane keeps half of its values
    // 16 -> 8 -> 4 -> 2 -> 1 values, 15 shuffles, then one more across the last pair
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const bool up = lane & 16;
      const float send = up ? part[j] : part[j + 8];
      const float recv = __shfl_xor_sync(0xffffffffu, send, 16);
      part[j] = (up ? part[j + 8] : part[j]) + recv;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const bool up = lane & 8;
      const float send = up ? part[j] : part[j + 4];
      const float recv = __shfl_xor_sync(0xffffffffu, send, 8);
      part[j] = (up ? part[j + 4] : part[j]) + recv;
    }
#pragma unroll
    for (int j = 0; j < 2; ++j) {
      const bool up = lane & 4;
      const float send = up ? part[j] : part[j + 2];
      const float recv = __shfl_xor_sync(0xffffffffu, send, 4);
      part[j] = (up ? part[j + 2] : part[j]) + recv;
    }
    {
      const bool up = lane & 2;
      const float send = up ? part[0] : part[1];
      const float recv = __shfl_xor_sync(0xffffffffu, send, 2);
      part[0] = (up ? part[1] : part[0]) + recv;
    }
    part[0] += __shfl_xor_sync(0xffffffffu, part[0], 1);
    // lane now holds the full sum of hidden unit j(lane)
    const int j = ((lane >> 4) & 1) * 8 + ((lane >> 3) & 1) * 4 + ((lane >> 2) & 1) * 2 + ((lane >> 1) & 1);
    const float hj = 1.0f / (1.0f + expf(-(part[0] + cpart[j])));
    float a = hj * __ldg(w.k2 + j);
    a = warp_sum(a) * 0.5f;                       // every j is held by two lanes
    a = (a + w.b2) * scale;
    if (lane == 0) s_att[wid][t] = a;
    amax = fmaxf(amax, a);
  }
  __syncwarp();
  // softmax over the unmasked positions (masked logits are -2^32+1: exp underflows to exactly 0)
  float den = 0.f;
  for (int t = lane; t < len; t += 32) den += expf(s_att[wid][t] - amax);
  den = warp_sum(den);
  float acc[MAX_TK];
#pragma unroll
  for (int tt = 0; tt < MAX_TK; ++tt) acc[tt] = 0.f;
  for (int t = 0; t < len; ++t) {
    const int64_t key = __ldg(s + t);
    const float p = expf(s_att[wid][t] - amax) / den;
#pragma unroll
    for (int tt = 0; tt < MAX_TK; ++tt) {
      const int c = lane + tt * 32;
      if (tt < TK && c < Kp) acc[tt] = fmaf(p, __ldg(G + key * ldg + c), acc[tt]);
    }
  }
#pragma unroll
  for (int tt = 0; tt < MAX_TK; ++tt) {
    const int c = lane + tt * 32;
    if (tt < TK && c < Kp) out[r * ld_out + c] = acc[tt];
  }
}

// tf_attention (use_tf_attention=True; libreco/layers/attention.py:5-25 = tf.keras.layers.Attention(
// use_scale=False) on [query] x keys with the sequence mask): a_t = <q, k_t>, masked positions get
// -1e9 (their softmax weight underflows to exactly 0), out = sum_t softmax(a)_t k_t.  One warp per row.
__global__ void __launch_bounds__(128)
dot_attention_kernel(const float* __restrict__ G, int64_t ldg, int Kp, const int64_t* __restrict__ items,
                     const int32_t* __restrict__ seqs, int64_t ld_seq, const int32_t* __restrict__ lens, int T,
                     const int64_t* __restrict__ users, int64_t R, int64_t grid, int64_t off,
                     float* __restrict__ out, int64_t ld_out) {
  __shared__ float s_att[4][MAX_T];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r = (int64_t)blockIdx.x * 4 + wid;
  if (r >= R) return;
  const int64_t sr = seq_row_of(users, r, grid, off);
  const int64_t item = grid > 0 ? (r + off) % grid : items[r];
  const int32_t* s = seqs + sr * ld_seq;
  const int len = min(max(lens[sr], 0), T);
  const int TK = (Kp + 31) / 32;
  float q[MAX_TK];
#pragma unroll
  for (int t = 0; t < MAX_TK; ++t) {
    const int c = lane + t * 32;
    q[t] = (t < TK && c < Kp) ? __ldg(G + item * ldg + c) : 0.f;
  }
  float amax = -3.0e38f;
  for (int t = 0; t < len; ++t) {
    const int64_t key = __ldg(s + t);
    float a = 0.f;
#pragma unroll
    for (int tt = 0; tt < MAX_TK; ++tt) {
      const int c = lane + tt * 32;
      if (tt < TK && c < Kp) a = fmaf(q[tt], __ldg(G + key * ldg + c), a);
    }
    a = warp_sum(a);
    if (lane == 0) s_att[wid][t] = a;
    amax = fmaxf(amax, a);
  }
  __syncwarp();
  float den = 0.f;
  for (int t = lane; t < len; t += 32) den += expf(s_att[wid][t] - amax);
  den = warp_sum(den);
  float acc[MAX_TK];
#pragma unroll
  for (int tt = 0; tt < MAX_TK; ++tt) acc[tt] = 0.f;
  for (int t = 0; t < len; ++t) {
    const int64_t key = __ldg(s + t);
    const float p = expf(s_att[wid][t] - amax) / den;
#pragma unroll
    for (int tt = 0; tt < MAX_TK; ++tt) {
      const int c = lane + tt * 32;
      if (tt < TK && c < Kp) acc[tt] = fmaf(p, __ldg(G + key * ldg + c), acc[tt]);
    }
  }
#pragma unroll
  for (int tt = 0; tt < MAX_TK; ++tt) {
    const int c = lane + tt * 32;
    if (tt < TK && c < Kp) out[r * ld_out + c] = acc[tt];
  }
}

// ---- DIN all-items scoring, hoisted (SURVEY.md 8d "a7 DIN all-items": per user one GEMM
// [N, K'] x [K', 16 len] on the tensor cores instead of N x len re-associated mat-vecs) -------------
// For ONE user the keys k_t are fixed and only the query q_n = G[n] varies:
//   z[t][j](n) = <q_n, A_t[:, j]> + c_t[j],  A_t[c][j] = (W1q + W1d)[c][j] + k_t[c] W1p[c][j],
//   c_t[j] = b1[j] + sum_c k_t[c] (W1k - W1d)[c][j]
// din_user_weights builds Wt [16 len, K'] (row (t, j) = A_t[:, j]) and the bias [16 len]; the GEMM runs
// on b200_linear_*; din_attention_hoisted turns Z [N, 16 len] into the attention output [N, K'].
__global__ void __launch_bounds__(128)
din_user_weights_kernel(const float* __restrict__ G, int64_t ldg, int Kp, const int32_t* __restrict__ seq, int len,
                        const float* __restrict__ k1, const float* __restrict__ b1, float* __restrict__ Wt,
                        int64_t ldw, float* __restrict__ bias) {
  __shared__ float red[4];
  const int row = blockIdx.x;                 // (t, j)
  const int t = row / HID, j = row % HID;
  if (t >= len) return;
  const float* key = G + (int64_t)seq[t] * ldg;
  float part = 0.f;
  for (int c = threadIdx.x; c < Kp; c += blockDim.x) {
    const float kv = __ldg(key + c);
    const float wq = __ldg(k1 + (int64_t)c * HID + j);
    const float wk = __ldg(k1 + (int64_t)(Kp + c) * HID + j);
    const float wd = __ldg(k1 + (int64_t)(2 * Kp + c) * HID + j);
    const float wp = __ldg(k1 + (int64_t)(3 * Kp + c) * HID + j);
    Wt[(int64_t)row * ldw + c] = (wq + wd) + kv * wp;
    part = fmaf(kv, wk - wd, part);
  }
  part = warp_sum(part);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = part;
  __syncthreads();
  if (threadIdx.x == 0) bias[row] = red[0] + red[1] + red[2] + red[3] + __ldg(b1 + j);
}

// one warp per item: scores a_t from Z (two sequence positions per 32-lane load), softmax over the
// len positions, out = sum_t p_t k_t  (attention.py:49-64; len == 0 -> zeros)
__global__ void __launch_bounds__(128)
din_attention_hoisted_kernel(const float* __restrict__ Z, int64_t ldz, int64_t N, const float* __restrict__ G,
                             int64_t ldg, int Kp, const int32_t* __restrict__ seq, int len,
                             const float* __restrict__ k2, float b2, float* __restrict__ out, int64_t ld_out) {
  __shared__ float s_att[4][MAX_T];
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t n = (int64_t)blockIdx.x * 4 + wid;
  if (n >= N) return;
  const float scale = rsqrtf((float)Kp);
  const float w2 = __ldg(k2 + (lane & 15));
  const float* z = Z + n * ldz;
  float amax = -3.0e38f;
  for (int t0 = 0; t0 < len; t0 += 2) {
    const int t = t0 + (lane >> 4);
    float v = 0.f;
    if (t < len) v = w2 / (1.0f + expf(-__ldg(z + t * HID + (lane & 15))));
    v += __shfl_xor_sync(0xffffffffu, v, 8);
    v += __shfl_xor_sync(0xffffffffu, v, 4);
    v += __shfl_xor_sync(0xffffffffu, v, 2);
    v += __shfl_xor_sync(0xffffffffu, v, 1);
    const float a = (v + b2) * scale;
    if ((lane & 15) == 0 && t < len) s_att[wid][t] = a;
  }
  __syncwarp();
  for (int t = lane; t < len; t += 32) amax = fmaxf(amax, s_att[wid][t]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
  float den = 0.f;
  for (int t = lane; t < len; t += 32) den += expf(s_att[wid][t] - amax);
  den = warp_sum(den);
  const int TK = (Kp + 31) / 32;
  float acc[MAX_TK];
#pragma unroll
  for (int tt = 0; tt < MAX_TK; ++tt) acc[tt] = 0.f;
  for (int t = 0; t < len; ++t) {
    const float p = expf(s_att[wid][t] - amax) / den;
    const float* key = G + (int64_t)__ldg(seq + t) * ldg;
#pragma unroll
    for (int tt = 0; tt < MAX_TK; ++tt) {
      const int c = lane + tt * 32;
      if (tt < TK && c < Kp) acc[tt] = fmaf(p, __ldg(key + c), acc[tt]);
    }
  }
#pragma unroll
  for (int tt = 0; tt < MAX_TK; ++tt) {
    const int c = lane + tt * 32;
    if (tt < TK && c < Kp) out[n * ld_out + c] = acc[tt];
  }
}


// DIN all-items, second half: A[n, t] = Dense(1)(sigmoid(Dense(16)(...))) WITHOUT its bias, written by the fused
// GEMM epilogue (b200_linear_tf32x3_sigmoid_dot).  One warp per item: lane t owns position t (two rounds for
// T <= 64), softmax over the len positions, out = sum_t p_t k_t with the user's keys staged ONCE per CTA in
// shared memory (they are the same for every item) and p_t broadcast by shuffle.
__global__ void __launch_bounds__(256)
din_attention_from_logits_kernel(const float* __restrict__ A, int64_t lda, int64_t N, const float* __restrict__ G,
                                 int64_t ldg, int Kp, const int32_t* __restrict__ seq, int len, float b2,
                                 float* __restrict__ out, int64_t ld_out) {
  extern __shared__ float s_keys[];                      // [len][Kp]
  for (int i = threadIdx.x; i < len * Kp; i += blockDim.x)
    s_keys[i] = __ldg(G + (int64_t)__ldg(seq + i / Kp) * ldg + (i % Kp));
  __syncthreads();
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float scale = rsqrtf((float)Kp);
  const int TK = (Kp + 31) / 32;
  for (int64_t n = (int64_t)blockIdx.x * (blockDim.x >> 5) + wid; n < N; n += (int64_t)gridDim.x * (blockDim.x >> 5)) {
    const float* a = A + n * lda;
    const float a0 = lane < len ? (__ldg(a + lane) + b2) * scale : -3.0e38f;
    const float a1 = lane + 32 < len ? (__ldg(a + lane + 32) + b2) * scale : -3.0e38f;
    float amax = fmaxf(a0, a1);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    float e0 = lane < len ? expf(a0 - amax) : 0.f;
    float e1 = lane + 32 < len ? expf(a1 - amax) : 0.f;
    const float den = warp_sum(e0 + e1);
    e0 /= den;
    e1 /= den;
    float acc[MAX_TK];
#pragma unroll
    for (int tt = 0; tt < MAX_TK; ++tt) acc[tt] = 0.f;
    for (int t = 0; t < len; ++t) {
      const float p = __shfl_sync(0xffffffffu, t < 32 ? e0 : e1, t & 31);
#pragma unroll
      for (int tt = 0; tt < MAX_TK; ++tt) {
        const int c = lane + tt * 32;
        if (tt < TK && c < Kp) acc[tt] = fmaf(p, s_keys[t * Kp + c], acc[tt]);
      }
    }
#pragma unroll
    for (int tt = 0; tt < MAX_TK; ++tt) {
      const int c = lane + tt * 32;
      if (tt < TK && c < Kp) out[n * ld_out + c] = acc[tt];
    }
  }
}


// DIN all-items, hoisted form, second kernel — v2.  The first version (one warp per item, two positions per 32-lane
// load, a 4-step shuffle tree per pair of positions, softmax weights recomputed by every lane) was instruction
// bound: 3660 warp instructions per item, issue slots 84 % busy (profiles/r02_din_attention_ncu.txt).  Here lane t
// OWNS positions t and t + 32: it reads the 16 pre-activations of a position as four 16-byte loads (consecutive
// lanes = consecutive 64 bytes), does the 16 sigmoids and the Dense(1) dot in registers — no shuffles —, the softmax
// is one max / one sum over the warp, and the weighted key sum reads the user's keys from shared memory (staged once
// per CTA, they are the same for every item) with p_t broadcast by shuffle.
template <int TKC>
__global__ void __launch_bounds__(256)
din_attention_hoisted_v2_kernel(const float* __restrict__ Z, int64_t ldz, int64_t N, const float* __restrict__ G,
                                int64_t ldg, int Kp, const int32_t* __restrict__ seq, int len,
                                const float* __restrict__ k2, float b2, float* __restrict__ out, int64_t ld_out) {
  extern __shared__ float s_keys[];                      // [len][Kp]
  for (int i = threadIdx.x; i < len * Kp; i += blockDim.x)
    s_keys[i] = __ldg(G + (int64_t)__ldg(seq + i / Kp) * ldg + (i % Kp));
  __syncthreads();
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const float scale = rsqrtf((float)Kp);
  float w2[HID];
#pragma unroll
  for (int j = 0; j < HID; ++j) w2[j] = __ldg(k2 + j);
  const int wpb = blockDim.x >> 5;
  for (int64_t n = (int64_t)blockIdx.x * wpb + wid; n < N; n += (int64_t)gridDim.x * wpb) {
    const float4* z4 = reinterpret_cast<const float4*>(Z + n * ldz);
    float a[2];
#pragma unroll
    for (int rnd = 0; rnd < 2; ++rnd) {
      const int t = lane + rnd * 32;
      a[rnd] = -3.0e38f;
      if (t < len) {
        float4 v[HID / 4];
#pragma unroll
        for (int q = 0; q < HID / 4; ++q) v[q] = __ldg(z4 + t * (HID / 4) + q);
        float d = 0.f;
#pragma unroll
        for (int q = 0; q < HID / 4; ++q) {
          d = fmaf(w2[4 * q + 0], __frcp_rn(1.0f + expf(-v[q].x)), d);
          d = fmaf(w2[4 * q + 1], __frcp_rn(1.0f + expf(-v[q].y)), d);
          d = fmaf(w2[4 * q + 2], __frcp_rn(1.0f + expf(-v[q].z)), d);
          d = fmaf(w2[4 * q + 3], __frcp_rn(1.0f + expf(-v[q].w)), d);
        }
        a[rnd] = (d + b2) * scale;
      }
    }
    float amax = fmaxf(a[0], a[1]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    float e0 = lane < len ? expf(a[0] - amax) : 0.f;
    float e1 = lane + 32 < len ? expf(a[1] - amax) : 0.f;
    const float den = warp_sum(e0 + e1);
    e0 /= den;
    e1 /= den;
    float acc[TKC];
#pragma unroll
    for (int tt = 0; tt < TKC; ++tt) acc[tt] = 0.f;
    const int l0 = min(len, 32);
    for (int t = 0; t < l0; ++t) {
      const float p = __shfl_sync(0xffffffffu, e0, t);
#pragma unroll
      for (int tt = 0; tt < TKC; ++tt) {
        const int c = lane + tt * 32;
        if (c < Kp) acc[tt] = fmaf(p, s_keys[t * Kp + c], acc[tt]);
      }
    }
    for (int t = 32; t < len; ++t) {
      const float p = __shfl_sync(0xffffffffu, e1, t - 32);
#pragma unroll
      for (int tt = 0; tt < TKC; ++tt) {
        const int c = lane + tt * 32;
        if (c < Kp) acc[tt] = fmaf(p, s_keys[t * Kp + c], acc[tt]);
      }
    }
#pragma unroll
    for (int tt = 0; tt < TKC; ++tt) {
      const int c = lane + tt * 32;
      if (c < Kp) out[n * ld_out + c] = acc[tt];
    }
  }
}


// ---- DIN attention backward (training of DIN, SURVEY 8f-1): gradient of out[r] = sum_t p_t k_t with
// p = softmax_t((Dense1(sigmoid(Dense16([q, k_t, q - k_t, q * k_t]))) ) * rsqrt(K')) w.r.t. the item feature rows
// (q = G[item], k_t = G[seq_t]) and the attention weights.  One warp per row, lanes own feature columns; the forward
// quantities are recomputed (h_t kept in shared memory), the weight gradient uses
//     sum_t dz_t (x) [q, k_t, q - k_t, q * k_t] = [q (x) A, B, q (x) A - B, q * B],  A = sum_t dz_t, B = sum_t k_t (x) dz_t
// so a row costs 4 K' x 16 shared-memory accumulations instead of that per position; persistent CTAs flush their
// [4 K', 16] accumulator with one global atomic per element at the end.
constexpr int BWD_T = 64;        // positions per row this kernel keeps (sequence lengths above fall outside training use)
template <int TKC>
__global__ void __launch_bounds__(128)
din_attention_backward_kernel(const float* __restrict__ G, int64_t ldg, int Kp, const int64_t* __restrict__ items,
                              const int32_t* __restrict__ seqs, int64_t ld_seq, const int32_t* __restrict__ lens, int T,
                              const int64_t* __restrict__ users, int64_t R, AttW w, const float* __restrict__ dout,
                              int64_t ld_dout, float* __restrict__ dG, int64_t ld_dg, float* __restrict__ g_k1,
                              float* __restrict__ g_b1, float* __restrict__ g_k2, float* __restrict__ g_b2) {
  extern __shared__ float bsm[];
  float* sW = bsm;                                        // [4 Kp][HID]
  float* sh_all = sW + 4 * Kp * HID;                      // [4 warps][BWD_T][HID]
  float* sa_all = sh_all + 4 * BWD_T * HID;               // [4][BWD_T]  logits, then p
  float* sdp_all = sa_all + 4 * BWD_T;                    // [4][BWD_T]  <dout, k_t>
  for (int i = threadIdx.x; i < 4 * Kp * HID; i += blockDim.x) sW[i] = 0.f;
  __syncthreads();
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sh = sh_all + wid * BWD_T * HID;
  float* sa = sa_all + wid * BWD_T;
  float* sdp = sdp_all + wid * BWD_T;
  const float scale = rsqrtf((float)Kp);
  float k2r[HID], gk2[HID], gb1[HID];
  float gb2 = 0.f;
#pragma unroll
  for (int j = 0; j < HID; ++j) { k2r[j] = __ldg(w.k2 + j); gk2[j] = 0.f; gb1[j] = 0.f; }
  for (int64_t r = (int64_t)blockIdx.x * 4 + wid; r < R; r += (int64_t)gridDim.x * 4) {
    const int64_t sr = seq_row_of(users, r, 0, 0);
    const int64_t item = items[r];
    const int32_t* sq = seqs + sr * ld_seq;
    const int len = min(min(max(lens[sr], 0), T), BWD_T);
    if (len == 0) continue;                               // forward output is 0: no gradient
    float q[TKC], dy[TKC], M[TKC][HID], cpart[HID];
#pragma unroll
    for (int j = 0; j < HID; ++j) cpart[j] = 0.f;
#pragma unroll
    for (int tt = 0; tt < TKC; ++tt) {
      const int c = lane + tt * 32;
      q[tt] = 0.f; dy[tt] = 0.f;
      if (c < Kp) {
        q[tt] = __ldg(G + item * ldg + c);
        dy[tt] = __ldg(dout + r * ld_dout + c);
#pragma unroll
        for (int j = 0; j < HID; ++j) {
          const float wq = __ldg(w.k1 + (int64_t)c * HID + j);
          const float wk = __ldg(w.k1 + (int64_t)(Kp + c) * HID + j);
          const float wd = __ldg(w.k1 + (int64_t)(2 * Kp + c) * HID + j);
          const float wp = __ldg(w.k1 + (int64_t)(3 * Kp + c) * HID + j);
          M[tt][j] = (wk - wd) + q[tt] * wp;
          cpart[j] = fmaf(q[tt], wq + wd, cpart[j]);
        }
      } else {
#pragma unroll
        for (int j = 0; j < HID; ++j) M[tt][j] = 0.f;
      }
    }
#pragma unroll
    for (int j = 0; j < HID; ++j) cpart[j] = warp_sum(cpart[j]) + __ldg(w.b1 + j);
    // ---- forward recompute: h_t, logits, <dout, k_t>
    float amax = -3.0e38f;
    for (int t = 0; t < len; ++t) {
      const int64_t key = __ldg(sq + t);
      float part[HID];
      float dp = 0.f;
#pragma unroll
      for (int j = 0; j < HID; ++j) part[j] = 0.f;
#pragma unroll
      for (int tt = 0; tt < TKC; ++tt) {
        const int c = lane + tt * 32;
        if (c < Kp) {
          const float kv = __ldg(G + key * ldg + c);
          dp = fmaf(dy[tt], kv, dp);
#pragma unroll
          for (int j = 0; j < HID; ++j) part[j] = fmaf(kv, M[tt][j], part[j]);
        }
      }
      dp = warp_sum(dp);
      float a = 0.f;
#pragma unroll
      for (int j = 0; j < HID; ++j) {
        const float z = warp_sum(part[j]) + cpart[j];
        const float hj = 1.0f / (1.0f + expf(-z));
        if (lane == j) sh[t * HID + j] = hj;
        a = fmaf(hj, k2r[j], a);
      }
      a = (a + w.b2) * scale;
      if (lane == 0) { sa[t] = a; sdp[t] = dp; }
      amax = fmaxf(amax, a);
    }
    __syncwarp();
    float den = 0.f;
    for (int t = lane; t < len; t += 32) den += expf(sa[t] - amax);
    den = warp_sum(den);
    float S = 0.f;
    for (int t = lane; t < len; t += 32) {
      const float pt = expf(sa[t] - amax) / den;
      S = fmaf(pt, sdp[t], S);
      sa[t] = pt;                                          // logits -> probabilities
    }
    S = warp_sum(S);
    __syncwarp();
    // ---- backward over the positions
    float A[HID], B[TKC][HID];
#pragma unroll
    for (int j = 0; j < HID; ++j) A[j] = 0.f;
#pragma unroll
    for (int tt = 0; tt < TKC; ++tt)
#pragma unroll
      for (int j = 0; j < HID; ++j) B[tt][j] = 0.f;
    for (int t = 0; t < len; ++t) {
      const int64_t key = __ldg(sq + t);
      const float pt = sa[t];
      const float da = scale * pt * (sdp[t] - S);          // d loss / d (Dense1 output of position t)
      gb2 += da;
      float dz[HID];
#pragma unroll
      for (int j = 0; j < HID; ++j) {
        const float hj = sh[t * HID + j];
        gk2[j] = fmaf(da, hj, gk2[j]);
        dz[j] = da * k2r[j] * hj * (1.0f - hj);
        A[j] += dz[j];
      }
#pragma unroll
      for (int tt = 0; tt < TKC; ++tt) {
        const int c = lane + tt * 32;
        if (c < Kp) {
          const float kv = __ldg(G + key * ldg + c);
          float dk = pt * dy[tt];
#pragma unroll
          for (int j = 0; j < HID; ++j) {
            dk = fmaf(M[tt][j], dz[j], dk);
            B[tt][j] = fmaf(kv, dz[j], B[tt][j]);
          }
          atomicAdd(dG + key * ld_dg + c, dk);
        }
      }
    }
    // ---- query gradient, weight gradients of this row
#pragma unroll
    for (int j = 0; j < HID; ++j) gb1[j] += A[j];
#pragma unroll
    for (int tt = 0; tt < TKC; ++tt) {
      const int c = lane + tt * 32;
      if (c < Kp) {
        float dq = 0.f;
#pragma unroll
        for (int j = 0; j < HID; ++j) {
          const float wq = __ldg(w.k1 + (int64_t)c * HID + j);
          const float wd = __ldg(w.k1 + (int64_t)(2 * Kp + c) * HID + j);
          const float wp = __ldg(w.k1 + (int64_t)(3 * Kp + c) * HID + j);
          dq = fmaf(wq + wd, A[j], dq);
          dq = fmaf(wp, B[tt][j], dq);
          const float qa = q[tt] * A[j];
          atomicAdd(sW + (0 * Kp + c) * HID + j, qa);
          atomicAdd(sW + (1 * Kp + c) * HID + j, B[tt][j]);
          atomicAdd(sW + (2 * Kp + c) * HID + j, qa - B[tt][j]);
          atomicAdd(sW + (3 * Kp + c) * HID + j, q[tt] * B[tt][j]);
        }
        atomicAdd(dG + item * ld_dg + c, dq);
      }
    }
    __syncwarp();
  }
  // every lane holds the same gk2 / gb1 / gb2 (computed redundantly): lane j publishes element j
#pragma unroll
  for (int j = 0; j < HID; ++j) {
    if (lane == j) { atomicAdd(g_k2 + j, gk2[j]); atomicAdd(g_b1 + j, gb1[j]); }
  }
  if (lane == 0) atomicAdd(g_b2, gb2);
  __syncthreads();
  for (int i = threadIdx.x; i < 4 * Kp * HID; i += blockDim.x) {
    const float v = sW[i];
    if (v != 0.f) atomicAdd(g_k1 + i, v);
  }
}


// ---- din_attention, v2 (T <= 64, K' % 4 == 0): the per-row matrix M[c][j] = (Wk - Wd)[c][j] + q_c Wp[c][j] goes to
// SHARED memory (K' x 16 floats per warp) and lane t OWNS position t (and t + 32): it streams its key row in
// 16-byte pieces and does the 16 dot products against M with broadcast shared-memory reads — 16 FMAs per loaded
// element, no shuffle butterflies (the first version: K'/32 x 16 FMAs and 31 shuffles + selects per position for the
// whole warp).  Softmax = one max / one sum over the warp; the weighted key sum reads each key row once more,
// coalesced, with p_t broadcast by shuffle.
template <int TKC>
__global__ void __launch_bounds__(128)
din_attention_v2_kernel(const float* __restrict__ G, int64_t ldg, int Kp, const int64_t* __restrict__ items,
                        const int32_t* __restrict__ seqs, int64_t ld_seq, const int32_t* __restrict__ lens, int T,
                        const int64_t* __restrict__ users, int64_t R, int64_t grid, int64_t off, AttW w,
                        float* __restrict__ out, int64_t ld_out) {
  extern __shared__ float sM_all[];                       // [4 warps][Kp][HID]
  const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float* sM = sM_all + (size_t)wid * Kp * HID;
  const float scale = rsqrtf((float)Kp);
  float k2r[HID];
#pragma unroll
  for (int j = 0; j < HID; ++j) k2r[j] = __ldg(w.k2 + j);
  for (int64_t r = (int64_t)blockIdx.x * 4 + wid; r < R; r += (int64_t)gridDim.x * 4) {
    const int64_t sr = seq_row_of(users, r, grid, off);
    const int64_t item = grid > 0 ? (r + off) % grid : items[r];
    const int32_t* sq = seqs + sr * ld_seq;
    const int len = min(max(lens[sr], 0), T);
    // ---- M (shared) and c_j = <q, Wq + Wd> + b1 (every lane)
    float cpart[HID];
#pragma unroll
    for (int j = 0; j < HID; ++j) cpart[j] = 0.f;
    __syncwarp();                                          // the previous row's readers of sM are done
#pragma unroll
    for (int tt = 0; tt < TKC; ++tt) {
      const int c = lane + tt * 32;
      if (c < Kp) {
        const float qc = __ldg(G + item * ldg + c);
        const float4* wq4 = reinterpret_cast<const float4*>(w.k1 + (int64_t)c * HID);
        const float4* wk4 = reinterpret_cast<const float4*>(w.k1 + (int64_t)(Kp + c) * HID);
        const float4* wd4 = reinterpret_cast<const float4*>(w.k1 + (int64_t)(2 * Kp + c) * HID);
        const float4* wp4 = reinterpret_cast<const float4*>(w.k1 + (int64_t)(3 * Kp + c) * HID);
#pragma unroll
        for (int j4 = 0; j4 < HID / 4; ++j4) {
          const float4 a = __ldg(wq4 + j4), b = __ldg(wk4 + j4), d = __ldg(wd4 + j4), e = __ldg(wp4 + j4);
          float4 m;
          m.x = (b.x - d.x) + qc * e.x; m.y = (b.y - d.y) + qc * e.y;
          m.z = (b.z - d.z) + qc * e.z; m.w = (b.w - d.w) + qc * e.w;
          reinterpret_cast<float4*>(sM + c * HID)[j4] = m;
          cpart[4 * j4 + 0] = fmaf(qc, a.x + d.x, cpart[4 * j4 + 0]);
          cpart[4 * j4 + 1] = fmaf(qc, a.y + d.y, cpart[4 * j4 + 1]);
          cpart[4 * j4 + 2] = fmaf(qc, a.z + d.z, cpart[4 * j4 + 2]);
          cpart[4 * j4 + 3] = fmaf(qc, a.w + d.w, cpart[4 * j4 + 3]);
        }
      }
    }
#pragma unroll
    for (int j = 0; j < HID; ++j) cpart[j] = warp_sum(cpart[j]) + __ldg(w.b1 + j);
    __syncwarp();
    // ---- logits: lane t owns positions t and t + 32
    float a[2];
#pragma unroll
    for (int rnd = 0; rnd < 2; ++rnd) {
      const int t = lane + rnd * 32;
      a[rnd] = -3.0e38f;
      if (t < len) {
        const float4* k4 = reinterpret_cast<const float4*>(G + (int64_t)__ldg(sq + t) * ldg);
        float z[HID];
#pragma unroll
        for (int j = 0; j < HID; ++j) z[j] = cpart[j];
        for (int c4 = 0; c4 < Kp / 4; ++c4) {
          const float4 kv = __ldg(k4 + c4);
          const float kk[4] = {kv.x, kv.y, kv.z, kv.w};
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float4* m4 = reinterpret_cast<const float4*>(sM + (c4 * 4 + i) * HID);
#pragma unroll
            for (int j4 = 0; j4 < HID / 4; ++j4) {
              const float4 m = m4[j4];                    // same address in every lane: a broadcast
              z[4 * j4 + 0] = fmaf(kk[i], m.x, z[4 * j4 + 0]);
              z[4 * j4 + 1] = fmaf(kk[i], m.y, z[4 * j4 + 1]);
              z[4 * j4 + 2] = fmaf(kk[i], m.z, z[4 * j4 + 2]);
              z[4 * j4 + 3] = fmaf(kk[i], m.w, z[4 * j4 + 3]);
            }
          }
        }
        float d = 0.f;
#pragma unroll
        for (int j = 0; j < HID; ++j) d = fmaf(k2r[j], __frcp_rn(1.0f + expf(-z[j])), d);
        a[rnd] = (d + w.b2) * scale;
      }
    }
    float amax = fmaxf(a[0], a[1]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
    float e0 = lane < len ? expf(a[0] - amax) : 0.f;
    float e1 = lane + 32 < len ? expf(a[1] - amax) : 0.f;
    const float den = warp_sum(e0 + e1);
    if (len > 0) { e0 /= den; e1 /= den; }
    float acc[TKC];
#pragma unroll
    for (int tt = 0; tt < TKC; ++tt) acc[tt] = 0.f;
    for (int t = 0; t < len; ++t) {
      const float pt = __shfl_sync(0xffffffffu, t < 32 ? e0 : e1, t & 31);
      const float* key = G + (int64_t)__ldg(sq + t) * ldg;
#pragma unroll
      for (int tt = 0; tt < TKC; ++tt) {
        const int c = lane + tt * 32;
        if (c < Kp) acc[tt] = fmaf(pt, __ldg(key + c), acc[tt]);
      }
    }
#pragma unroll
    for (int tt = 0; tt < TKC; ++tt) {
      const int c = lane + tt * 32;
      if (c < Kp) out[r * ld_out + c] = acc[tt];
    }
  }
}

}  // namespace seq
}  // namespace b200

using namespace b200;
using namespace b200::seq;

static int g_din_v2 = 1;     // b200_din_attention_tune: 1 = lane-owns-position kernel where eligible (default), 0 = first version

extern "C" int b200_din_attention_tune(int32_t use_v2) {
  g_din_v2 = use_v2 ? 1 : 0;
  return 0;
}

extern "C" int b200_din_user_weights(const float* G, int64_t ldg, int32_t Kp, const int32_t* seq, int32_t len,
                                     const float* k1, const float* b1, float* Wt, int64_t ldw, float* bias,
                                     void* stream) {
  B200_REQUIRE(G && seq && k1 && b1 && Wt && bias, "b200_din_user_weights: null pointer");
  B200_REQUIRE(Kp >= 1 && ldw >= Kp && len >= 0 && len <= MAX_T, "b200_din_user_weights: bad shape");
  if (len == 0) return 0;
  din_user_weights_kernel<<<(unsigned)(len * HID), 128, 0, (cudaStream_t)stream>>>(G, ldg, Kp, seq, len, k1, b1, Wt,
                                                                                  ldw, bias);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_din_attention_hoisted(const float* Z, int64_t ldz, int64_t N, const float* G, int64_t ldg,
                                          int32_t Kp, const int32_t* seq, int32_t len, const float* k2, float b2,
                                          float* out, int64_t ld_out, void* stream) {
  B200_REQUIRE(G && seq && k2 && out && (Z || len == 0), "b200_din_attention_hoisted: null pointer");
  B200_REQUIRE(Kp >= 1 && Kp <= 32 * MAX_TK && len >= 0 && len <= MAX_T, "b200_din_attention_hoisted: bad shape");
  if (N == 0) return 0;
  const bool z_ok = Z && (ldz % 4 == 0) && ((reinterpret_cast<uintptr_t>(Z) & 15) == 0);
  if (len >= 1 && len <= 64 && z_ok && (size_t)len * Kp * 4 <= 48 * 1024 && N >= 1024) {
    const size_t smem = (size_t)len * Kp * 4;
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div64(N, 8), (int64_t)std::max(1, num_sms()) * 8);
    cudaStream_t st = (cudaStream_t)stream;
    switch ((Kp + 31) / 32) {
      case 1: din_attention_hoisted_v2_kernel<1><<<blocks, 256, smem, st>>>(Z, ldz, N, G, ldg, Kp, seq, len, k2, b2, out, ld_out); break;
      case 2: din_attention_hoisted_v2_kernel<2><<<blocks, 256, smem, st>>>(Z, ldz, N, G, ldg, Kp, seq, len, k2, b2, out, ld_out); break;
      case 3: din_attention_hoisted_v2_kernel<3><<<blocks, 256, smem, st>>>(Z, ldz, N, G, ldg, Kp, seq, len, k2, b2, out, ld_out); break;
      default: din_attention_hoisted_v2_kernel<4><<<blocks, 256, smem, st>>>(Z, ldz, N, G, ldg, Kp, seq, len, k2, b2, out, ld_out); break;
    }
    B200_CUDA_OK(cudaGetLastError());
    count_launch();
    return 0;
  }
  din_attention_hoisted_kernel<<<(unsigned)ceil_div64(N, 4), 128, 0, (cudaStream_t)stream>>>(
      Z, ldz, N, G, ldg, Kp, seq, len, k2, b2, out, ld_out);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_din_attention_from_logits(const float* A, int64_t lda, int64_t N, const float* G, int64_t ldg,
                                              int32_t Kp, const int32_t* seq, int32_t len, float b2, float* out,
                                              int64_t ld_out, void* stream) {
  B200_REQUIRE(A && G && seq && out, "b200_din_attention_from_logits: null pointer");
  B200_REQUIRE(Kp >= 1 && Kp <= 32 * MAX_TK && len >= 1 && len <= 64 && len <= MAX_T,
               "b200_din_attention_from_logits: bad shape");
  if (N == 0) return 0;
  const size_t smem = (size_t)len * Kp * 4;
  B200_REQUIRE(smem <= 48 * 1024, "b200_din_attention_from_logits: keys do not fit shared memory");
  const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div64(N, 8), (int64_t)std::max(1, num_sms()) * 8);
  din_attention_from_logits_kernel<<<blocks, 256, smem, (cudaStream_t)stream>>>(A, lda, N, G, ldg, Kp, seq, len, b2, out,
                                                                               ld_out);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_din_attention_backward(const float* G, int64_t ldg, int32_t Kp, const int64_t* items,
                                           const int32_t* seqs, int64_t ld_seq, const int32_t* lens, int32_t T,
                                           const int64_t* users, int64_t R, const float* k1, const float* b1,
                                           const float* k2, float b2, const float* dout, int64_t ld_dout, float* dG,
                                           int64_t ld_dg, float* g_k1, float* g_b1, float* g_k2, float* g_b2,
                                           void* stream) {
  B200_REQUIRE(G && items && seqs && lens && users && k1 && b1 && k2 && dout && dG && g_k1 && g_b1 && g_k2 && g_b2,
               "b200_din_attention_backward: null pointer");
  B200_REQUIRE(Kp >= 1 && Kp <= 32 * MAX_TK, "b200_din_attention_backward: feature width %d outside [1, %d]", Kp, 32 * MAX_TK);
  B200_REQUIRE(T >= 1 && T <= BWD_T, "b200_din_attention_backward: sequence length %d outside [1, %d]", T, BWD_T);
  if (R == 0) return 0;
  AttW w{k1, b1, k2, b2};
  const size_t smem = ((size_t)4 * Kp * HID + (size_t)4 * BWD_T * HID + (size_t)8 * BWD_T) * 4;
  const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div64(R, 4), (int64_t)std::max(1, num_sms()) * 4);
  cudaStream_t st = (cudaStream_t)stream;
  auto launch = [&](auto kern) -> int {
    B200_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<blocks, 128, smem, st>>>(G, ldg, Kp, items, seqs, ld_seq, lens, T, users, R, w, dout, ld_dout, dG, ld_dg, g_k1,
                                    g_b1, g_k2, g_b2);
    return 0;
  };
  int rc;
  switch ((Kp + 31) / 32) {
    case 1: rc = launch(din_attention_backward_kernel<1>); break;
    case 2: rc = launch(din_attention_backward_kernel<2>); break;
    case 3: rc = launch(din_attention_backward_kernel<3>); break;
    default: rc = launch(din_attention_backward_kernel<4>); break;
  }
  if (rc) return rc;
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_seq_pool(const float* E, int64_t lde, int32_t d, int64_t pad_index,
                             const int32_t* seqs, int64_t ld_seq, const int32_t* lens, int32_t T,
                             const int64_t* users, int64_t R, int64_t grid_items, int64_t row_offset,
                             float* out, int64_t ld_out, void* stream) {
  B200_REQUIRE(E && seqs && lens && users && out, "b200_seq_pool: null pointer");
  if (R == 0) return 0;
  seq_pool_kernel<<<(unsigned)ceil_div64(R * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      E, lde, d, pad_index, seqs, ld_seq, lens, T, users, R, grid_items, row_offset, out, ld_out);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_seq_pool_backward(const float* dout, int64_t ld_dout, int32_t d, int64_t pad_index,
                                      const int32_t* seqs, int64_t ld_seq, const int32_t* lens, int32_t T,
                                      const int64_t* users, int64_t R, float* g_embeds, int64_t ld_g,
                                      void* stream) {
  B200_REQUIRE(dout && seqs && lens && users && g_embeds, "b200_seq_pool_backward: null pointer");
  if (R == 0) return 0;
  seq_pool_backward_kernel<<<(unsigned)ceil_div64(R * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      dout, ld_dout, d, pad_index, seqs, ld_seq, lens, T, users, R, g_embeds, ld_g);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_din_attention(const float* G, int64_t ldg, int32_t Kp, const int64_t* items,
                                  const int32_t* seqs, int64_t ld_seq, const int32_t* lens, int32_t T,
                                  const int64_t* users, int64_t R, int64_t grid_items,
                                  int64_t row_offset, const float* k1, const float* b1,
                                  const float* k2, float b2, float* out, int64_t ld_out, void* stream) {
  B200_REQUIRE(G && seqs && lens && users && out, "b200_din_attention: null pointer");
  B200_REQUIRE(grid_items > 0 || items, "b200_din_attention: item ids missing");
  B200_REQUIRE(Kp >= 1 && Kp <= 32 * MAX_TK, "b200_din_attention: feature width %d outside [1, %d]", Kp, 32 * MAX_TK);
  B200_REQUIRE(T >= 1 && T <= MAX_T, "b200_din_attention: sequence length %d outside [1, %d]", T, MAX_T);
  if (R == 0) return 0;
  if (k1 == nullptr) {   // use_tf_attention=True: plain dot-product attention, no learned weights
    dot_attention_kernel<<<(unsigned)ceil_div64(R, 4), 128, 0, (cudaStream_t)stream>>>(
        G, ldg, Kp, items, seqs, ld_seq, lens, T, users, R, grid_items, row_offset, out, ld_out);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
  }
  B200_REQUIRE(b1 && k2, "b200_din_attention: attention MLP weights missing");
  AttW w; w.k1 = k1; w.b1 = b1; w.k2 = k2; w.b2 = b2;
  const bool v2_ok = g_din_v2 && T <= 64 && Kp % 4 == 0 && ldg % 4 == 0 && ((reinterpret_cast<uintptr_t>(G) & 15) == 0) &&
                     ((reinterpret_cast<uintptr_t>(k1) & 15) == 0);
  if (v2_ok) {
    const size_t smem = (size_t)4 * Kp * HID * 4;
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div64(R, 4), (int64_t)std::max(1, num_sms()) * 16);
    cudaStream_t st = (cudaStream_t)stream;
    switch ((Kp + 31) / 32) {
      case 1: din_attention_v2_kernel<1><<<blocks, 128, smem, st>>>(G, ldg, Kp, items, seqs, ld_seq, lens, T, users, R, grid_items, row_offset, w, out, ld_out); break;
      case 2: din_attention_v2_kernel<2><<<blocks, 128, smem, st>>>(G, ldg, Kp, items, seqs, ld_seq, lens, T, users, R, grid_items, row_offset, w, out, ld_out); break;
      case 3: din_attention_v2_kernel<3><<<blocks, 128, smem, st>>>(G, ldg, Kp, items, seqs, ld_seq, lens, T, users, R, grid_items, row_offset, w, out, ld_out); break;
      default: din_attention_v2_kernel<4><<<blocks, 128, smem, st>>>(G, ldg, Kp, items, seqs, ld_seq, lens, T, users, R, grid_items, row_offset, w, out, ld_out); break;
    }
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    return 0;
  }
  din_attention_kernel<<<(unsigned)ceil_div64(R, 4), 128, 0, (cudaStream_t)stream>>>(
      G, ldg, Kp, items, seqs, ld_seq, lens, T, users, R, grid_items, row_offset, w, out, ld_out);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
