// SIM inference (libreco/algorithms/sim.py:193-304, soft search): the second stage only, which is what the reference
// serves (sim.py:206-207).
//
// Gp = combine_seq_features(concat) Wp [N+1, K] (sim.py:197-199) is the item table every attention reads.  For a
// (user, item n) pair with q = Gp[n]:
//   GSU (sim.py:264-286): s_t = q . Gp[long_t] for t < long_len, -1e9 for the other positions; the search_topk
//       largest, equal scores resolving to the lower position (tf.math.top_k);
//   ESU (sim.py:288-299): multi-head attention of Qp[n] = q Wq over the selected keys Kl = Gp[long] Wk and values
//       Vl = Gp[long] Wv (scale 1/sqrt(hd)), then Wo;
//   short (sim.py:301-304): Keras dot-product attention of q over Gp[short], no scale.
// Hidden logits are fl32(logit - 1e9), as Keras adds the mask; with no valid key the weights are the softmax of those
// rounded values, uniform whenever |logit| < 32.
//
// The rows kernel's GSU (scores, warp top-k, compaction) is sim::gsu_select of sim_gsu.cuh, which the training GSU
// kernel (sim_train.cu) calls too.  Both modes compute the GSU scores with the same chain,
// acc = fmaf(q[d], Gp[t][d], acc) over d ascending from 0, on the same Gp, so they select the same positions.
//   * b200_sim_attention (rows mode): one warp per (slot, item) row writes [long_out || short_out] into the sequence
//     block of the concat the library's dense layers read.
//   * b200_sim_pair_scores (grid mode): one thread per (slot, item) pair, the first MLP layer re-associated as
//     relu(Pu[b] + Pi[n] + [o || s] W_att) with W_att = [Wo W1_long ; W1_short], then the small layers and the head.
#include <math.h>

#include <algorithm>
#include <climits>

#include "../../include/b200reco.h"
#include "common.cuh"
#include "sim_gsu.cuh"

namespace b200 {
namespace {

constexpr int SIM_MAX_L = sim::MAX_L;
constexpr int SIM_MAX_S = sim::MAX_S;
constexpr int SIM_MAX_TOPK = sim::MAX_TOPK;
constexpr int SIM_MAX_K = sim::MAX_K;
constexpr float MASK_NEG = sim::MASK_NEG;

__host__ __device__ inline int64_t round_up64(int64_t n, int64_t m) { return (n + m - 1) / m * m; }

// ---- rows mode: one warp per (slot, item) row ----------------------------------------------------------------
struct RowsArgs {
  const float *Gp, *Qp;
  int64_t ldg, ldq;
  int K, H, L, S, topk;
  const int32_t *long_seqs, *long_lens, *short_seqs, *short_lens;
  int64_t ld_long, ld_short;
  const float *Kl, *Vl, *Wo;
  const int32_t* slot_of_row;
  const int64_t* items;
  int64_t n, grid_items, row_offset;
  float* out;
  int64_t ldo;
  int32_t* gsu_pos;
};

constexpr int ROWS_THREADS = 256;

__global__ void __launch_bounds__(ROWS_THREADS) sim_attention_kernel(const __grid_constant__ RowsArgs a) {
  __shared__ int sel_sm[ROWS_THREADS / 32][SIM_MAX_TOPK];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int K = a.K, L = a.L, S = a.S, k = a.topk, hd = a.K / a.H;
  const float scale = 1.0f / sqrtf((float)hd);
  for (int64_t r = w0; r < a.n; r += nw) {
    const int64_t slot = a.slot_of_row ? (int64_t)a.slot_of_row[r] : (a.row_offset + r) / a.grid_items;
    const int64_t item = a.items ? a.items[r] : (a.row_offset + r) % a.grid_items;
    const float* q = a.Gp + item * a.ldg;
    const float* qp = a.Qp + item * a.ldq;
    const int32_t* ls = a.long_seqs + slot * a.ld_long;
    const int32_t* ss = a.short_seqs + slot * a.ld_short;
    const int llen = min(max(a.long_lens[slot], 0), L), slen = min(max(a.short_lens[slot], 0), S);
    const float* kl = a.Kl + slot * L * K;
    const float* vl = a.Vl + slot * L * K;
    const int pi = sim::gsu_select(a.Gp, a.ldg, q, ls, llen, K, L, k, sel_sm[wib], lane);
    if (a.gsu_pos && lane < k) a.gsu_pos[r * k + lane] = pi;
    // ESU: lane i owns the i-th selected key for the logits, lanes own columns d = lane, lane + 32 for the mix
    float o[2] = {0.f, 0.f};
    for (int h = 0; h < a.H; ++h) {
      const int d0 = h * hd;
      float v = -INFINITY;
      if (lane < k) {
        const float* kr = kl + (int64_t)pi * K;
        float acc = 0.f;
        for (int d = d0; d < d0 + hd; ++d) acc = fmaf(__ldg(qp + d), __ldg(kr + d), acc);
        v = acc * scale;
        if (pi >= llen) v = v - MASK_NEG;
      }
      const float mx = warp_max(v);
      const float e = lane < k ? expf(v - mx) : 0.f;
      const float p = e / warp_sum(e);
      for (int i = 0; i < k; ++i) {
        const float pv = __shfl_sync(0xffffffffu, p, i);
        const int pt = __shfl_sync(0xffffffffu, pi, i);
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int d = lane + 32 * c;
          if (d >= d0 && d < d0 + hd) o[c] = fmaf(pv, __ldg(vl + (int64_t)pt * K + d), o[c]);
        }
      }
    }
    float lo[2] = {0.f, 0.f};
    for (int d = 0; d < K; ++d) {
      const float od = __shfl_sync(0xffffffffu, d < 32 ? o[0] : o[1], d & 31);
#pragma unroll
      for (int c = 0; c < 2; ++c)
        if (lane + 32 * c < K) lo[c] = fmaf(od, __ldg(a.Wo + (int64_t)d * K + lane + 32 * c), lo[c]);
    }
    // short attention: lane owns positions s = lane, lane + 32
    float sv[2];
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int s = lane + 32 * c;
      float v = -INFINITY;
      if (s < S) {
        const float* g = a.Gp + (int64_t)__ldg(ss + s) * a.ldg;
        float acc = 0.f;
        for (int d = 0; d < K; ++d) acc = fmaf(__ldg(q + d), __ldg(g + d), acc);
        v = s < slen ? acc : acc - MASK_NEG;
      }
      sv[c] = v;
    }
    const float smx = warp_max(fmaxf(sv[0], sv[1]));
    const float e0 = lane < S ? expf(sv[0] - smx) : 0.f, e1 = lane + 32 < S ? expf(sv[1] - smx) : 0.f;
    const float ssum = warp_sum(e0 + e1);
    float so[2] = {0.f, 0.f};
    for (int s = 0; s < S; ++s) {
      const float es = __shfl_sync(0xffffffffu, s < 32 ? e0 : e1, s & 31);
      const float* g = a.Gp + (int64_t)__ldg(ss + s) * a.ldg;
#pragma unroll
      for (int c = 0; c < 2; ++c)
        if (lane + 32 * c < K) so[c] = fmaf(es, __ldg(g + lane + 32 * c), so[c]);
    }
    float* out = a.out + r * a.ldo;
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const int d = lane + 32 * c;
      if (d < K) {
        out[d] = lo[c];
        out[K + d] = so[c] / ssum;
      }
    }
  }
}

// ---- grid mode: one thread per (slot b, item n) pair --------------------------------------------------------
constexpr int SP_THREADS = 256;
constexpr int SP_MAXH1 = 256;
constexpr int SP_MAXH2 = 128;
constexpr int SP_MAXH3 = 64;

struct PairArgs {
  const float *GpT, *QpT;   // [K, ldt]: column n is item n's Gp / Qp row (coalesced per-thread loads)
  int64_t ldt, N;
  const float* Gp;
  int64_t ldg;
  const int32_t *long_seqs, *long_lens, *short_seqs, *short_lens;
  int64_t ld_long, ld_short;
  const float *Kl, *Vl, *Pu, *PiT;
  int64_t ldpi;
  int K, H, L, S, topk, H1, H2, H3;
  const float *Watt, *W2, *b2, *W3, *b3, *w_out;
  float b_out;
  float* scores;
  int64_t lds;
};

// Shared memory (float offsets): W_att [2KP, h1p], W2 [h1p, h2p], W3 [h2p, H3], Pu [h1p], the slot's long rows of Gp
// [L, KP] (read as broadcasts), Kl / Vl [L, KP+1] (read at each thread's own positions: odd stride), Gp[short] [S, KP],
// then per thread: the selection's scores and positions [topk] and x = [o || s] [2KP], each strided by the block size.
struct PairLayout {
  int kp, ldk, h1p, h2p;
  int64_t watt, w2, w3, pu, gl, kl, vl, gs, selv, seli, x, total;
};

__host__ __device__ inline PairLayout pair_layout(int K, int L, int S, int topk, int H1, int H2, int H3) {
  PairLayout P;
  P.kp = (int)round_up64(K, 16);
  P.ldk = P.kp + 1;
  P.h1p = (int)round_up64(H1, 32);
  P.h2p = (int)round_up64(H2, 16);
  P.watt = 0;
  P.w2 = P.watt + 2 * (int64_t)P.kp * P.h1p;
  P.w3 = P.w2 + (int64_t)P.h1p * P.h2p;
  P.pu = P.w3 + (int64_t)P.h2p * H3;
  P.gl = P.pu + P.h1p;
  P.kl = P.gl + (int64_t)L * P.kp;
  P.vl = P.kl + round_up64((int64_t)L * P.ldk, 4);
  P.gs = P.vl + round_up64((int64_t)L * P.ldk, 4);
  P.selv = P.gs + (int64_t)S * P.kp;
  P.seli = P.selv + (int64_t)topk * SP_THREADS;
  P.x = P.seli + (int64_t)topk * SP_THREADS;
  P.total = P.x + 2 * (int64_t)P.kp * SP_THREADS;
  return P;
}

template <int KP>
__device__ __forceinline__ float dot_row(const float (&q)[KP], const float* g) {
  float acc = 0.f;
#pragma unroll
  for (int d4 = 0; d4 < KP / 4; ++d4) {
    const float4 v = reinterpret_cast<const float4*>(g)[d4];
    acc = fmaf(q[4 * d4 + 0], v.x, acc);
    acc = fmaf(q[4 * d4 + 1], v.y, acc);
    acc = fmaf(q[4 * d4 + 2], v.z, acc);
    acc = fmaf(q[4 * d4 + 3], v.w, acc);
  }
  return acc;
}

template <int KP>
__global__ void __launch_bounds__(SP_THREADS, 1) sim_pair_kernel(const __grid_constant__ PairArgs a) {
  extern __shared__ __align__(16) float sm[];
  const int K = a.K, L = a.L, S = a.S, k = a.topk, H1 = a.H1, H2 = a.H2, H3 = a.H3;
  const PairLayout P = pair_layout(K, L, S, k, H1, H2, H3);
  float* watt = sm + P.watt;
  float* w2 = sm + P.w2;
  float* w3 = sm + P.w3;
  float* pu = sm + P.pu;
  float* gl = sm + P.gl;
  float* kl = sm + P.kl;
  float* vl = sm + P.vl;
  float* gs = sm + P.gs;
  const int tid = threadIdx.x, h1p = P.h1p, h2p = P.h2p, ldk = P.ldk;
  const int64_t b = blockIdx.y;
  for (int i = tid; i < 2 * KP * h1p; i += SP_THREADS) {
    const int c = i / h1p, j = i - c * h1p, d = c % KP;
    watt[i] = (d < K && j < H1) ? __ldg(a.Watt + (int64_t)((c / KP) * K + d) * H1 + j) : 0.f;
  }
  for (int i = tid; i < h1p * h2p; i += SP_THREADS) {
    const int kk = i / h2p, j = i - kk * h2p;
    w2[i] = (kk < H1 && j < H2) ? __ldg(a.W2 + (int64_t)kk * H2 + j) : 0.f;
  }
  for (int i = tid; i < h2p * H3; i += SP_THREADS) {
    const int kk = i / H3;
    w3[i] = kk < H2 ? __ldg(a.W3 + i) : 0.f;
  }
  for (int j = tid; j < h1p; j += SP_THREADS) pu[j] = j < H1 ? __ldg(a.Pu + b * H1 + j) : 0.f;
  const int32_t* ls = a.long_seqs + b * a.ld_long;
  const int32_t* ss = a.short_seqs + b * a.ld_short;
  for (int i = tid; i < L * KP; i += SP_THREADS) {
    const int t = i / KP, d = i - t * KP;
    gl[i] = d < K ? __ldg(a.Gp + (int64_t)__ldg(ls + t) * a.ldg + d) : 0.f;
    kl[t * ldk + d] = d < K ? __ldg(a.Kl + (b * L + t) * K + d) : 0.f;
    vl[t * ldk + d] = d < K ? __ldg(a.Vl + (b * L + t) * K + d) : 0.f;
  }
  for (int i = tid; i < S * KP; i += SP_THREADS) {
    const int s = i / KP, d = i - s * KP;
    gs[i] = d < K ? __ldg(a.Gp + (int64_t)__ldg(ss + s) * a.ldg + d) : 0.f;
  }
  __syncthreads();
  const int llen = min(max(a.long_lens[b], 0), L), slen = min(max(a.short_lens[b], 0), S);
  const int H = a.H, hd = K / H;
  const float scale = 1.0f / sqrtf((float)hd);
  float* selv = sm + P.selv + tid;                           // element i at selv[i * SP_THREADS]
  int* seli = reinterpret_cast<int*>(sm + P.seli) + tid;
  float* x = sm + P.x + tid;
  constexpr int TS = SP_THREADS;
  for (int64_t n = (int64_t)blockIdx.x * TS + tid; n - tid < a.N; n += (int64_t)gridDim.x * TS) {
    if (n >= a.N) continue;   // no barrier below: a thread past the end only skips its pair
    float q[KP];
#pragma unroll
    for (int d = 0; d < KP; ++d) q[d] = d < K ? __ldg(a.GpT + d * a.ldt + n) : 0.f;
    // short attention: max of the logits, then exp, sum and the weighted rows in ascending s; s = (sum e_s g_s) / sum
    {
      float mx = -INFINITY;
      for (int s = 0; s < S; ++s) {
        float v = dot_row<KP>(q, gs + s * KP);
        if (s >= slen) v = v - MASK_NEG;
        mx = fmaxf(mx, v);
      }
      float acc[KP];
#pragma unroll
      for (int d = 0; d < KP; ++d) acc[d] = 0.f;
      float sum = 0.f;
      for (int s = 0; s < S; ++s) {
        const float* g = gs + s * KP;
        float v = dot_row<KP>(q, g);
        if (s >= slen) v = v - MASK_NEG;
        const float e = expf(v - mx);
        sum += e;
#pragma unroll
        for (int d = 0; d < KP; ++d) acc[d] = fmaf(e, g[d], acc[d]);
      }
#pragma unroll
      for (int d = 0; d < KP; ++d) x[(KP + d) * TS] = acc[d] / sum;
    }
    // GSU: running top-k over t ascending; the worst member (lowest score, then highest position) is replaced by a
    // strictly larger score, so equal scores keep the lower position
    {
      float wv = INFINITY;
      int wt = -1, wslot = 0, filled = 0;
      for (int t = 0; t < L; ++t) {
        float s;
        if (t < llen) {
          s = dot_row<KP>(q, gl + t * KP);
          if (s != s) s = -INFINITY;
        } else {
          if (filled == k && wv >= -MASK_NEG) break;   // every later position scores -1e9 and loses the tie
          s = -MASK_NEG;
        }
        if (filled < k) {
          selv[filled * TS] = s;
          seli[filled * TS] = t;
          ++filled;
          if (filled < k) continue;
        } else if (s > wv) {
          selv[wslot * TS] = s;
          seli[wslot * TS] = t;
        } else {
          continue;
        }
        wv = INFINITY;
        wt = -1;
        for (int i = 0; i < k; ++i) {
          const float v = selv[i * TS];
          const int ti = seli[i * TS];
          if (v < wv || (v == wv && ti > wt)) {
            wv = v;
            wt = ti;
            wslot = i;
          }
        }
      }
    }
    // ESU: Qp[n] into x[0, KP), each head's output written over its own query columns once its logits are formed
#pragma unroll
    for (int d = 0; d < KP; ++d) x[d * TS] = d < K ? __ldg(a.QpT + d * a.ldt + n) : 0.f;
    for (int h = 0; h < H; ++h) {
      const int d0 = h * hd;
      float mx = -INFINITY;
      for (int i = 0; i < k; ++i) {
        const int p = seli[i * TS];
        const float* kr = kl + p * ldk;
        float acc = 0.f;
        for (int d = d0; d < d0 + hd; ++d) acc = fmaf(x[d * TS], kr[d], acc);
        float v = acc * scale;
        if (p >= llen) v = v - MASK_NEG;
        selv[i * TS] = v;
        mx = fmaxf(mx, v);
      }
      float sum = 0.f;
      for (int i = 0; i < k; ++i) {
        const float e = expf(selv[i * TS] - mx);
        selv[i * TS] = e;
        sum += e;
      }
      for (int i = 0; i < k; ++i) selv[i * TS] = selv[i * TS] / sum;
      for (int d = d0; d < d0 + hd; ++d) {
        float acc = 0.f;
        for (int i = 0; i < k; ++i) acc = fmaf(selv[i * TS], vl[seli[i * TS] * ldk + d], acc);
        x[d * TS] = acc;
      }
    }
    // first layer in 32-column chunks: h1 = relu(Pu + Pi + [o || s] W_att), straight into the second layer
    float h2[SP_MAXH2];
#pragma unroll
    for (int j = 0; j < SP_MAXH2; ++j) h2[j] = 0.f;
    for (int kc = 0; kc < H1; kc += 32) {
      float m[32];
#pragma unroll
      for (int j = 0; j < 32; ++j) m[j] = 0.f;
      for (int c = 0; c < 2 * KP; ++c) {
        const float xv = x[c * TS];
        const float4* wr = reinterpret_cast<const float4*>(watt + c * h1p + kc);
#pragma unroll
        for (int j4 = 0; j4 < 8; ++j4) {
          const float4 w = wr[j4];
          m[4 * j4 + 0] = fmaf(xv, w.x, m[4 * j4 + 0]);
          m[4 * j4 + 1] = fmaf(xv, w.y, m[4 * j4 + 1]);
          m[4 * j4 + 2] = fmaf(xv, w.z, m[4 * j4 + 2]);
          m[4 * j4 + 3] = fmaf(xv, w.w, m[4 * j4 + 3]);
        }
      }
#pragma unroll
      for (int jj = 0; jj < 32; ++jj) {
        const int kk = kc + jj;
        if (kk < H1) {
          const float hv = fmaxf(pu[kk] + __ldg(a.PiT + kk * a.ldpi + n) + m[jj], 0.f);
          const float4* wr = reinterpret_cast<const float4*>(w2 + kk * h2p);
#pragma unroll
          for (int j16 = 0; j16 < SP_MAXH2 / 16; ++j16) {
            if (16 * j16 < H2) {
#pragma unroll
              for (int j4 = 0; j4 < 4; ++j4) {
                const float4 w = wr[4 * j16 + j4];
                const int j = 16 * j16 + 4 * j4;
                h2[j + 0] = fmaf(hv, w.x, h2[j + 0]);
                h2[j + 1] = fmaf(hv, w.y, h2[j + 1]);
                h2[j + 2] = fmaf(hv, w.z, h2[j + 2]);
                h2[j + 3] = fmaf(hv, w.w, h2[j + 3]);
              }
            }
          }
        }
      }
    }
    float out = a.b_out;
    if (H3 > 0) {
#pragma unroll
      for (int j = 0; j < SP_MAXH2; ++j) h2[j] = j < H2 ? fmaxf(h2[j] + __ldg(a.b2 + j), 0.f) : 0.f;
#pragma unroll 1
      for (int j = 0; j < H3; ++j) {
        float h3 = 0.f;
#pragma unroll
        for (int j16 = 0; j16 < SP_MAXH2 / 16; ++j16) {
          if (16 * j16 < H2) {
#pragma unroll
            for (int i = 0; i < 16; ++i) h3 = fmaf(h2[16 * j16 + i], w3[(16 * j16 + i) * H3 + j], h3);
          }
        }
        out = fmaf(h3 + __ldg(a.b3 + j), __ldg(a.w_out + j), out);
      }
    } else {
#pragma unroll
      for (int j = 0; j < SP_MAXH2; ++j)
        if (j < H2) out = fmaf(h2[j] + __ldg(a.b2 + j), __ldg(a.w_out + j), out);
    }
    a.scores[b * a.lds + n] = out;
  }
}

int check_sim_shape(int32_t K, int32_t H, int32_t L, int32_t S, int32_t topk, const char* who) {
  B200_REQUIRE(K >= 1 && K <= SIM_MAX_K, "%s: embed size %d outside [1, %d]", who, K, SIM_MAX_K);
  B200_REQUIRE(H >= 1 && K % H == 0, "%s: embed size %d is not a multiple of num_heads %d", who, K, H);
  B200_REQUIRE(L >= 1 && L <= SIM_MAX_L, "%s: long sequence length %d outside [1, %d]", who, L, SIM_MAX_L);
  B200_REQUIRE(S >= 1 && S <= SIM_MAX_S, "%s: short sequence length %d outside [1, %d]", who, S, SIM_MAX_S);
  B200_REQUIRE(topk >= 1 && topk <= std::min(SIM_MAX_TOPK, (int)L), "%s: search_topk %d outside [1, min(%d, %d)]",
               who, topk, SIM_MAX_TOPK, L);
  return 0;
}

int pair_mlp_ok(int32_t H1, int32_t H2, int32_t H3) {
  return H1 >= 1 && H1 <= SP_MAXH1 && H2 >= 1 && H2 <= SP_MAXH2 && H3 >= 0 && H3 <= SP_MAXH3;
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200_sim_attention(const float* Gp, int64_t ldg, const float* Qp, int64_t ldq, int32_t K, int32_t H,
                                  const int32_t* long_seqs, int64_t ld_long, const int32_t* long_lens, const float* Kl,
                                  const float* Vl, int32_t L, const int32_t* short_seqs, int64_t ld_short,
                                  const int32_t* short_lens, int32_t S, int32_t topk, const float* Wo,
                                  const int32_t* slot_of_row, const int64_t* items, int64_t n, int64_t grid_items,
                                  int64_t row_offset, float* out, int64_t ldo, int32_t* gsu_pos, void* stream) {
  const char* who = "b200_sim_attention";
  int rc = check_sim_shape(K, H, L, S, topk, who);
  if (rc != 0) return rc;
  B200_REQUIRE(Gp && Qp && long_seqs && long_lens && Kl && Vl && short_seqs && short_lens && Wo && out,
               "%s: null pointer", who);
  B200_REQUIRE((slot_of_row != nullptr) == (items != nullptr) && (items != nullptr || grid_items > 0),
               "%s: give slot_of_row and items, or grid_items > 0", who);
  B200_REQUIRE(n >= 0 && ldg >= K && ldq >= K && ld_long >= L && ld_short >= S && ldo >= 2 * K && row_offset >= 0,
               "%s: bad shape", who);
  if (n == 0) return 0;
  RowsArgs a;
  a.Gp = Gp; a.Qp = Qp; a.ldg = ldg; a.ldq = ldq; a.K = K; a.H = H; a.L = L; a.S = S; a.topk = topk;
  a.long_seqs = long_seqs; a.long_lens = long_lens; a.short_seqs = short_seqs; a.short_lens = short_lens;
  a.ld_long = ld_long; a.ld_short = ld_short; a.Kl = Kl; a.Vl = Vl; a.Wo = Wo; a.slot_of_row = slot_of_row;
  a.items = items; a.n = n; a.grid_items = grid_items; a.row_offset = row_offset; a.out = out; a.ldo = ldo;
  a.gsu_pos = gsu_pos;
  const int64_t blocks = std::min<int64_t>(ceil_div64(n, ROWS_THREADS / 32), (int64_t)(num_sms() > 0 ? num_sms() : 132) * 16);
  sim_attention_kernel<<<(unsigned)blocks, ROWS_THREADS, 0, (cudaStream_t)stream>>>(a);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int64_t b200_sim_pair_smem_bytes(int32_t K, int32_t L, int32_t S, int32_t topk, int32_t H1, int32_t H2,
                                            int32_t H3) {
  if (K < 1 || K > SIM_MAX_K || L < 1 || S < 1 || topk < 1 || !pair_mlp_ok(H1, H2, H3)) return -2;
  return pair_layout(K, L, S, topk, H1, H2, H3).total * (int64_t)sizeof(float);
}

template <int KP>
static int launch_pair(const PairArgs& a, size_t smem, int64_t B, cudaStream_t st) {
  if (smem > 48 * 1024)
    B200_CUDA_OK(cudaFuncSetAttribute(sim_pair_kernel<KP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t cap = num_sms() > 0 ? num_sms() : 132;
  const unsigned gx = (unsigned)std::max<int64_t>(1, std::min<int64_t>(ceil_div64(a.N, SP_THREADS), std::max<int64_t>(1, cap / B)));
  sim_pair_kernel<KP><<<dim3(gx, (unsigned)B), SP_THREADS, smem, st>>>(a);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_sim_pair_scores(const float* GpT, const float* QpT, int64_t ldt, int64_t N, const float* Gp,
                                    int64_t ldg, const int32_t* long_seqs, int64_t ld_long, const int32_t* long_lens,
                                    const int32_t* short_seqs, int64_t ld_short, const int32_t* short_lens,
                                    const float* Kl, const float* Vl, const float* Pu, int64_t B, const float* PiT,
                                    int64_t ldpi, int32_t K, int32_t H, int32_t L, int32_t S, int32_t topk, int32_t H1,
                                    int32_t H2, int32_t H3, const float* W_att, const float* W2, const float* b2,
                                    const float* W3, const float* b3, const float* w_out, float b_out, float* scores,
                                    int64_t lds, void* stream) {
  const char* who = "b200_sim_pair_scores";
  int rc = check_sim_shape(K, H, L, S, topk, who);
  if (rc != 0) return rc;
  B200_REQUIRE(pair_mlp_ok(H1, H2, H3), "%s: unsupported layer sizes H=(%d,%d,%d), supported <= (%d,%d,%d)", who, H1,
               H2, H3, SP_MAXH1, SP_MAXH2, SP_MAXH3);
  B200_REQUIRE(GpT && QpT && Gp && long_seqs && long_lens && short_seqs && short_lens && Kl && Vl && Pu && PiT &&
                   W_att && W2 && b2 && w_out && scores,
               "%s: null pointer", who);
  B200_REQUIRE(H3 == 0 || (W3 && b3), "%s: third layer weights missing", who);
  B200_REQUIRE(B >= 0 && B <= 65535 && N >= 0 && ldt >= N && ldg >= K && ld_long >= L && ld_short >= S && ldpi >= N &&
                   lds >= N,
               "%s: bad shape", who);
  const size_t smem = (size_t)b200_sim_pair_smem_bytes(K, L, S, topk, H1, H2, H3);
  int dev = 0, optin = 0;
  B200_CUDA_OK(cudaGetDevice(&dev));
  B200_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  B200_REQUIRE(smem <= (size_t)optin, "%s: K %d, L %d, S %d, topk %d, H=(%d,%d,%d) need %zu B of shared memory, the "
               "device allows %d", who, K, L, S, topk, H1, H2, H3, smem, optin);
  if (B == 0 || N == 0) return 0;
  PairArgs a;
  a.GpT = GpT; a.QpT = QpT; a.ldt = ldt; a.N = N; a.Gp = Gp; a.ldg = ldg; a.long_seqs = long_seqs;
  a.long_lens = long_lens; a.short_seqs = short_seqs; a.short_lens = short_lens; a.ld_long = ld_long;
  a.ld_short = ld_short; a.Kl = Kl; a.Vl = Vl; a.Pu = Pu; a.PiT = PiT; a.ldpi = ldpi; a.K = K; a.H = H; a.L = L;
  a.S = S; a.topk = topk; a.H1 = H1; a.H2 = H2; a.H3 = H3; a.Watt = W_att; a.W2 = W2; a.b2 = b2; a.W3 = W3; a.b3 = b3;
  a.w_out = w_out; a.b_out = b_out; a.scores = scores; a.lds = lds;
  const cudaStream_t st = (cudaStream_t)stream;
  switch ((K + 15) / 16) {
    case 1: return launch_pair<16>(a, smem, B, st);
    case 2: return launch_pair<32>(a, smem, B, st);
    case 3: return launch_pair<48>(a, smem, B, st);
    default: return launch_pair<64>(a, smem, B, st);
  }
}
