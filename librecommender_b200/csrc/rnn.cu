// RNN4Rec inference: the recurrent user encoder (libreco/algorithms/rnn4rec.py:151-237, layers/recurrent.py:4-63).
//
// The user vector of RNN4Rec is tf_dense(embed_size)(rnn(seq_embeds[seq])): b200_rnn_encode computes the rnn part
// for every slot and the Dense head runs on the dense-layer kernels.  One CTA owns a tile of users and runs every
// step of every layer for it: the step loop is outermost (a wavefront over the layers), so only each layer's state
// [tile, H] lives on chip and neither the gathered input rows nor an intermediate layer's outputs reach HBM.  The
// loop runs to the longest len of the tile, not to T.  Layer weights are read from global memory (through L1 / L2)
// at every step: a GRU with H = 256 is 1.5 MB, so no form of the kernel assumes they fit in shared memory.
//
// Work item = (hidden unit j, group of RNN_UPT users): the thread runs the unit's G gate columns for its users, each
// pre-activation one fmaf chain over the input index ascending (x part) and one over the state index (h part).
// Nothing a user computes reads another user's data, so a user's bits do not depend on the tile it shares, on n or
// on the call.
#include <math.h>

#include <algorithm>

#include "../../include/b200reco.h"
#include "common.cuh"

namespace b200 {
namespace {

constexpr int RNN_MAX_T = 128;
constexpr int RNN_MAX_DIM = 256;
constexpr int RNN_MAX_LAYERS = 4;
constexpr int RNN_THREADS = 128;
constexpr int RNN_UPT = 8;          // users per work item
constexpr int RNN_MAX_TILE = 64;
constexpr float RNN_LN_EPS = 1e-3f;  // Keras LayerNormalization default

enum CellKind { GRU_RESET_AFTER = 0, GRU_RESET_BEFORE = 1, LSTM = 2 };
enum CellAct { ACT_TANH = 0, ACT_LN_TANH = 1 };

__host__ __device__ inline int odd_ld(int n) { return n | 1; }
__host__ __device__ inline int cell_gates(int kind) { return kind == LSTM ? 4 : 3; }

// floats of one packed layer: W [in, G*H], U [H, G*H], bx [G*H], bh [G*H], gamma [H], beta [H]
__host__ __device__ inline int64_t rnn_layer_floats(int kind, int in, int H) {
  const int64_t GH = (int64_t)cell_gates(kind) * H;
  return (int64_t)in * GH + (int64_t)H * GH + 2 * GH + 2 * (int64_t)H;
}

__device__ __forceinline__ float sigmoid_f(float x) { return 1.0f / (1.0f + expf(-x)); }

struct RnnParams {
  int T, in0, L, tile, Hmax;
  int kind[RNN_MAX_LAYERS], H[RNN_MAX_LAYERS], act[RNN_MAX_LAYERS], in[RNN_MAX_LAYERS];
  int64_t woff[RNN_MAX_LAYERS];
  // float offsets into shared memory of [tile, odd_ld(.)] blocks (-1: absent)
  int s_h[RNN_MAX_LAYERS], s_c[RNN_MAX_LAYERS], s_y[RNN_MAX_LAYERS];
  int s_x0, s_hn, s_z, s_rh, s_st, s_len;
  const int64_t* users;
  int64_t n;
  const int32_t* lens;
  const int32_t* seqs;
  int64_t ld_seq;
  const float* X;
  int64_t ldx;
  const float* w;
  float* out;
  int64_t ldo;
  float* sv[RNN_MAX_LAYERS][6];   // training forward only: the saved tensors of each layer (SV_*), rows s * T + t
};

// What the training forward saves per layer, row s * T + t for t < len (rows t >= len are 0): the state before the
// step, the layer output, the post-activation gates, one cell-specific block, and with layer norm x^ and rstd.
enum SavedTensor { SV_HP = 0, SV_Y = 1, SV_G = 2, SV_X = 3, SV_XH = 4, SV_RS = 5 };

// acc[g][v] = sum_k xs[v * ldxs + k] * W[k * ldw + col[g]], one chain per (g, v) over k ascending
template <int NG>
__device__ __forceinline__ void chain(float (&acc)[NG][RNN_UPT], const float* __restrict__ W, int ldw, const int (&col)[NG],
                                      const float* xs, int ldxs, int nk) {
#pragma unroll
  for (int g = 0; g < NG; ++g)
#pragma unroll
    for (int v = 0; v < RNN_UPT; ++v) acc[g][v] = 0.f;
  for (int k = 0; k < nk; ++k) {
    float w[NG];
#pragma unroll
    for (int g = 0; g < NG; ++g) w[g] = __ldg(W + (int64_t)k * ldw + col[g]);
#pragma unroll
    for (int v = 0; v < RNN_UPT; ++v) {
      const float x = xs[v * ldxs + k];
#pragma unroll
      for (int g = 0; g < NG; ++g) acc[g][v] = fmaf(x, w[g], acc[g][v]);
    }
  }
}

__device__ __forceinline__ float cell_act(int act, float x) { return act == ACT_TANH ? tanhf(x) : x; }

// One step of layer l for every active user of the tile: new states into hn (and c in place).  GRU reset-before
// runs in two passes because its candidate chain reads r o h of every unit.  SAVE (the training forward) also
// writes h_{t-1}, the gates and the cell-specific block (LSTM c_t, Keras GRU U_c h + bh_c, TF1 GRU r o h_{t-1}).
template <bool SAVE>
__device__ void layer_step(const RnnParams& p, float* sm, int l, int t, const float* xin, int ldin) {
  const int kind = p.kind[l], H = p.H[l], act = p.act[l], in = p.in[l], tid = threadIdx.x;
  const int G = cell_gates(kind), GH = G * H, ldh = odd_ld(H), lds = odd_ld(p.Hmax);
  const float* W = p.w + p.woff[l];
  const float* U = W + (int64_t)in * GH;
  const float* bx = U + (int64_t)H * GH;
  const float* bh = bx + GH;
  const int* slen = reinterpret_cast<const int*>(sm + p.s_len);
  float* h = sm + p.s_h[l];
  float* hn = sm + p.s_hn;
  const int items = H * (p.tile / RNN_UPT);
  if (kind == LSTM) {
    float* c = sm + p.s_c[l];
    for (int it = tid; it < items; it += blockDim.x) {
      const int j = it % H, u0 = (it / H) * RNN_UPT;
      const int col[4] = {j, H + j, 2 * H + j, 3 * H + j};
      float ax[4][RNN_UPT], ah[4][RNN_UPT];
      chain<4>(ax, W, GH, col, xin + u0 * ldin, ldin, in);
      chain<4>(ah, U, GH, col, h + u0 * ldh, ldh, H);
      float b[4], r[4];
#pragma unroll
      for (int g = 0; g < 4; ++g) { b[g] = __ldg(bx + col[g]); r[g] = __ldg(bh + col[g]); }
#pragma unroll
      for (int v = 0; v < RNN_UPT; ++v) {
        const int u = u0 + v;
        if (t >= slen[u]) continue;
        const float ig = sigmoid_f((ax[0][v] + b[0]) + (ah[0][v] + r[0]));
        const float fg = sigmoid_f((ax[1][v] + b[1]) + (ah[1][v] + r[1]));
        const float gg = cell_act(act, (ax[2][v] + b[2]) + (ah[2][v] + r[2]));
        const float og = sigmoid_f((ax[3][v] + b[3]) + (ah[3][v] + r[3]));
        const float cn = fg * c[u * ldh + j] + ig * gg;
        c[u * ldh + j] = cn;
        hn[u * lds + j] = og * cell_act(act, cn);
        if constexpr (SAVE) {
          const int64_t row = ((int64_t)blockIdx.x * p.tile + u) * p.T + t;
          float* g = p.sv[l][SV_G] + row * GH;
          g[j] = ig; g[H + j] = fg; g[2 * H + j] = gg; g[3 * H + j] = og;
          p.sv[l][SV_X][row * H + j] = cn;
          p.sv[l][SV_HP][row * H + j] = h[u * ldh + j];
        }
      }
    }
  } else if (kind == GRU_RESET_AFTER) {
    for (int it = tid; it < items; it += blockDim.x) {
      const int j = it % H, u0 = (it / H) * RNN_UPT;
      const int col[3] = {j, H + j, 2 * H + j};
      float ax[3][RNN_UPT], ah[3][RNN_UPT];
      chain<3>(ax, W, GH, col, xin + u0 * ldin, ldin, in);
      chain<3>(ah, U, GH, col, h + u0 * ldh, ldh, H);
      float b[3], r[3];
#pragma unroll
      for (int g = 0; g < 3; ++g) { b[g] = __ldg(bx + col[g]); r[g] = __ldg(bh + col[g]); }
#pragma unroll
      for (int v = 0; v < RNN_UPT; ++v) {
        const int u = u0 + v;
        if (t >= slen[u]) continue;
        const float z = sigmoid_f((ax[0][v] + b[0]) + (ah[0][v] + r[0]));
        const float rg = sigmoid_f((ax[1][v] + b[1]) + (ah[1][v] + r[1]));
        const float hh = cell_act(act, (ax[2][v] + b[2]) + rg * (ah[2][v] + r[2]));
        hn[u * lds + j] = z * h[u * ldh + j] + (1.0f - z) * hh;
        if constexpr (SAVE) {
          const int64_t row = ((int64_t)blockIdx.x * p.tile + u) * p.T + t;
          float* g = p.sv[l][SV_G] + row * GH;
          g[j] = z; g[H + j] = rg; g[2 * H + j] = hh;
          p.sv[l][SV_X][row * H + j] = ah[2][v] + r[2];
          p.sv[l][SV_HP][row * H + j] = h[u * ldh + j];
        }
      }
    }
  } else {   // GRU_RESET_BEFORE: z, r and the x part of the candidate; then the candidate over r o h
    float* zb = sm + p.s_z;
    float* rh = sm + p.s_rh;
    for (int it = tid; it < items; it += blockDim.x) {
      const int j = it % H, u0 = (it / H) * RNN_UPT;
      const int col[3] = {j, H + j, 2 * H + j};
      const int colzr[2] = {j, H + j};
      float ax[3][RNN_UPT], ah[2][RNN_UPT];
      chain<3>(ax, W, GH, col, xin + u0 * ldin, ldin, in);
      chain<2>(ah, U, GH, colzr, h + u0 * ldh, ldh, H);
      float b[3], r[2];
#pragma unroll
      for (int g = 0; g < 3; ++g) b[g] = __ldg(bx + col[g]);
#pragma unroll
      for (int g = 0; g < 2; ++g) r[g] = __ldg(bh + col[g]);
#pragma unroll
      for (int v = 0; v < RNN_UPT; ++v) {
        const int u = u0 + v;
        const float z = sigmoid_f((ax[0][v] + b[0]) + (ah[0][v] + r[0]));
        const float rg = sigmoid_f((ax[1][v] + b[1]) + (ah[1][v] + r[1]));
        zb[u * lds + j] = z;
        rh[u * lds + j] = rg * h[u * ldh + j];
        hn[u * lds + j] = ax[2][v] + b[2];
        if constexpr (SAVE) {
          if (t < slen[u]) {
            const int64_t row = ((int64_t)blockIdx.x * p.tile + u) * p.T + t;
            p.sv[l][SV_G][row * GH + H + j] = rg;
            p.sv[l][SV_X][row * H + j] = rh[u * lds + j];
            p.sv[l][SV_HP][row * H + j] = h[u * ldh + j];
          }
        }
      }
    }
    __syncthreads();
    for (int it = tid; it < items; it += blockDim.x) {
      const int j = it % H, u0 = (it / H) * RNN_UPT;
      const int col[1] = {2 * H + j};
      float ac[1][RNN_UPT];
      chain<1>(ac, U, GH, col, rh + u0 * lds, lds, H);
      const float r = __ldg(bh + col[0]);
#pragma unroll
      for (int v = 0; v < RNN_UPT; ++v) {
        const int u = u0 + v;
        if (t >= slen[u]) continue;
        const float cc = cell_act(act, hn[u * lds + j] + (ac[0][v] + r));
        const float z = zb[u * lds + j];
        hn[u * lds + j] = z * h[u * ldh + j] + (1.0f - z) * cc;
        if constexpr (SAVE) {
          const int64_t row = ((int64_t)blockIdx.x * p.tile + u) * p.T + t;
          p.sv[l][SV_G][row * GH + j] = z;
          p.sv[l][SV_G][row * GH + 2 * H + j] = cc;
        }
      }
    }
  }
  __syncthreads();
  for (int i = tid; i < p.tile * H; i += blockDim.x) {
    const int u = i / H, j = i - u * H;
    if (t < slen[u]) h[u * ldh + j] = hn[u * lds + j];
  }
  __syncthreads();
}

// y = tanh((h - mean) * rsqrt(var + 1e-3) * gamma + beta) per user row (Keras LayerNormalization, then tanh);
// mean and var are ascending sums divided by H
__device__ void layer_norm_tanh(const RnnParams& p, float* sm, int l) {
  const int H = p.H[l], ldh = odd_ld(H), tid = threadIdx.x;
  const float* h = sm + p.s_h[l];
  float* y = sm + p.s_y[l];
  float* st = sm + p.s_st;
  const float* gb = p.w + p.woff[l] + rnn_layer_floats(p.kind[l], p.in[l], H) - 2 * H;
  for (int u = tid; u < p.tile; u += blockDim.x) {
    const float* x = h + u * ldh;
    float s = 0.f;
    for (int j = 0; j < H; ++j) s += x[j];
    const float mean = s / (float)H;
    float q = 0.f;
    for (int j = 0; j < H; ++j) {
      const float d = x[j] - mean;
      q = fmaf(d, d, q);
    }
    st[2 * u] = mean;
    st[2 * u + 1] = rsqrtf(q / (float)H + RNN_LN_EPS);
  }
  __syncthreads();
  for (int i = tid; i < p.tile * H; i += blockDim.x) {
    const int u = i / H, j = i - u * H;
    y[u * ldh + j] = tanhf((h[u * ldh + j] - st[2 * u]) * st[2 * u + 1] * __ldg(gb + j) + __ldg(gb + H + j));
  }
  __syncthreads();
}

// SAVE: the layer output of step t (h_t, or tanh(LN(h_t)) with x^ = (h_t - mean) rstd and rstd) for t < len
__device__ void save_outputs(const RnnParams& p, const float* sm, int l, int t) {
  const int H = p.H[l], ldh = odd_ld(H);
  const bool ln = p.act[l] == ACT_LN_TANH;
  const int* slen = reinterpret_cast<const int*>(sm + p.s_len);
  const float* h = sm + p.s_h[l];
  const float* st = sm + p.s_st;
  for (int i = threadIdx.x; i < p.tile * H; i += blockDim.x) {
    const int u = i / H, j = i - u * H;
    if (t >= slen[u]) continue;
    const int64_t row = ((int64_t)blockIdx.x * p.tile + u) * p.T + t;
    p.sv[l][SV_Y][row * H + j] = ln ? sm[p.s_y[l] + u * ldh + j] : h[u * ldh + j];
    if (ln) {
      p.sv[l][SV_XH][row * H + j] = (h[u * ldh + j] - st[2 * u]) * st[2 * u + 1];
      if (j == 0) p.sv[l][SV_RS][row] = st[2 * u + 1];
    }
  }
}

// SAVE: rows t >= len of every saved tensor are written as 0
__device__ void save_zero_tail(const RnnParams& p, const float* sm) {
  const int* slen = reinterpret_cast<const int*>(sm + p.s_len);
  const int64_t s0 = (int64_t)blockIdx.x * p.tile;
  for (int l = 0; l < p.L; ++l) {
    const int H = p.H[l], GH = cell_gates(p.kind[l]) * H;
    const bool ln = p.act[l] == ACT_LN_TANH;
    for (int u = 0; u < p.tile; ++u) {
      if (s0 + u >= p.n) break;
      const int64_t r0 = (s0 + u) * p.T + slen[u], nr = p.T - slen[u];
      for (int64_t i = threadIdx.x; i < nr * H; i += blockDim.x) {
        p.sv[l][SV_HP][r0 * H + i] = 0.f;
        p.sv[l][SV_Y][r0 * H + i] = 0.f;
        p.sv[l][SV_X][r0 * H + i] = 0.f;
        if (ln) p.sv[l][SV_XH][r0 * H + i] = 0.f;
      }
      for (int64_t i = threadIdx.x; i < nr * GH; i += blockDim.x) p.sv[l][SV_G][r0 * GH + i] = 0.f;
      if (ln)
        for (int64_t i = threadIdx.x; i < nr; i += blockDim.x) p.sv[l][SV_RS][r0 + i] = 0.f;
    }
  }
}

template <bool SAVE>
__global__ void __launch_bounds__(RNN_THREADS) rnn_encode_kernel(const __grid_constant__ RnnParams p) {
  extern __shared__ float sm[];
  const int tid = threadIdx.x, nt = blockDim.x;
  const int64_t s0 = (int64_t)blockIdx.x * p.tile;
  int* slen = reinterpret_cast<int*>(sm + p.s_len);
  int64_t* srow = reinterpret_cast<int64_t*>(sm + p.s_len + 2 * p.tile);   // 8-byte aligned by the host layout
  for (int u = tid; u < p.tile; u += nt) {
    const int64_t s = s0 + u;
    const int64_t row = s < p.n ? p.users[s] : 0;
    srow[u] = row;
    slen[u] = s < p.n ? min(max(p.lens[row], 0), p.T) : 0;
  }
  // zero state, and a zero input row for users that never gather one
  const int ld0 = odd_ld(p.in0);
  for (int i = tid; i < p.tile * ld0; i += nt) sm[p.s_x0 + i] = 0.f;
  for (int l = 0; l < p.L; ++l) {
    const int n = p.tile * odd_ld(p.H[l]);
    for (int i = tid; i < n; i += nt) {
      sm[p.s_h[l] + i] = 0.f;
      if (p.s_c[l] >= 0) sm[p.s_c[l] + i] = 0.f;
      if (p.s_y[l] >= 0) sm[p.s_y[l] + i] = 0.f;
    }
  }
  __syncthreads();
  int steps = 0;
  for (int u = 0; u < p.tile; ++u) steps = max(steps, slen[u]);
  for (int t = 0; t < steps; ++t) {
    for (int i = tid; i < p.tile * p.in0; i += nt) {
      const int u = i / p.in0, k = i - u * p.in0;
      if (t < slen[u]) {
        const int64_t item = __ldg(p.seqs + srow[u] * p.ld_seq + t);
        sm[p.s_x0 + u * ld0 + k] = __ldg(p.X + item * p.ldx + k);
      }
    }
    __syncthreads();
    const float* xin = sm + p.s_x0;
    int ldin = ld0;
    for (int l = 0; l < p.L; ++l) {
      layer_step<SAVE>(p, sm, l, t, xin, ldin);
      if (l + 1 < p.L) {
        if (p.act[l] == ACT_LN_TANH) {
          layer_norm_tanh(p, sm, l);
          xin = sm + p.s_y[l];
        } else {
          xin = sm + p.s_h[l];
        }
        ldin = odd_ld(p.H[l]);
      } else if constexpr (SAVE) {
        if (p.act[l] == ACT_LN_TANH) layer_norm_tanh(p, sm, l);
      }
      if constexpr (SAVE) save_outputs(p, sm, l, t);
    }
  }
  if constexpr (SAVE) save_zero_tail(p, sm);
  // output[:, -1] = the last layer's state after step len - 1 (after its LayerNorm and tanh when it has them)
  const int Lz = p.L - 1, H = p.H[Lz], ldh = odd_ld(H);
  const float* res = sm + p.s_h[Lz];
  if (p.act[Lz] == ACT_LN_TANH) {
    layer_norm_tanh(p, sm, Lz);
    res = sm + p.s_y[Lz];
  }
  for (int i = tid; i < p.tile * H; i += nt) {
    const int u = i / H, j = i - u * H;
    if (s0 + u < p.n) p.out[(s0 + u) * p.ldo + j] = res[u * ldh + j];
  }
}

// shared-memory layout of a tile; returns the float count
int64_t rnn_layout(RnnParams& p, int tile) {
  int64_t off = 0;
  auto take = [&](int64_t floats) { const int64_t o = off; off += floats; return (int)o; };
  p.tile = tile;
  p.s_x0 = take((int64_t)tile * odd_ld(p.in0));
  for (int l = 0; l < p.L; ++l) {
    const int64_t blk = (int64_t)tile * odd_ld(p.H[l]);
    p.s_h[l] = take(blk);
    p.s_c[l] = p.kind[l] == LSTM ? take(blk) : -1;
    p.s_y[l] = p.act[l] == ACT_LN_TANH ? take(blk) : -1;
  }
  const int64_t scr = (int64_t)tile * odd_ld(p.Hmax);
  p.s_hn = take(scr);
  p.s_z = take(scr);
  p.s_rh = take(scr);
  p.s_st = take(2 * (int64_t)tile);
  off += off & 1;                    // the int64 row ids below are 8-byte aligned
  p.s_len = take(2 * (int64_t)tile + 2 * (int64_t)tile);   // int32 lens (padded to 2 tile floats), int64 rows
  return off;
}

// ---- training: the backward through time of one layer ----------------------------------------------------------
// One CTA owns a tile of users and runs the layer's steps in reverse from the tile's longest len.  dh (and dc) stay
// in shared memory; at step t < len the incoming dY_t is added (through the LN + tanh backward for a layer-norm
// layer), the gate pre-activation gradients are formed and written as dGx (x part) and dGh (h part, Keras GRU only:
// the two differ in the candidate block, scaled by r), and dh_{t-1} = direct terms + dGh_t U^T is one ascending fmaf
// chain per (unit, user) over U's row, read through L1 / L2.  The dense products over all rows (dW, dU, dX, the
// bias, gamma and beta sums) run on the dense kernels outside.  No atomics: a user's rows depend on its own data.
struct RnnBwdParams {
  int T, tile, kind, H, GH, act, ldg;
  int s_dh, s_dc, s_dd, s_q, s_g, s_st, s_len;
  const int64_t* users;
  int64_t n;
  const int32_t* lens;
  const float* U;
  const float* gamma;   // gamma [H], beta [H] (layer norm)
  const float* dout;    // top layer: the head gradient [n, lddo], added at step len - 1
  int64_t lddo;
  const float* dy;      // lower layer: dX of the layer above [n * T, H]
  const float* sv[6];
  float* dgx;
  float* dgh;
  float* dln;           // layer norm: dLN = dy (1 - y^2) and dLN x^, rows [n * T, H]
  float* dlnx;
};

int64_t rnn_bwd_layout(RnnBwdParams& p, int tile) {
  int64_t off = 0;
  auto take = [&](int64_t floats) { const int64_t o = off; off += floats; return (int)o; };
  const int64_t blk = (int64_t)tile * odd_ld(p.H);
  p.tile = tile;
  p.ldg = odd_ld(p.GH);
  p.s_dh = take(blk);
  p.s_dc = take(blk);
  p.s_dd = take(blk);
  p.s_q = take(blk);
  p.s_g = take((int64_t)tile * p.ldg);
  p.s_st = take(2 * (int64_t)tile);
  p.s_len = take(tile);
  return off;
}

// acc[v] = sum_{c < nc} g[(u0 + v) * ldg + c] * ur[c], one chain per user over c ascending
__device__ __forceinline__ void row_chain(float (&acc)[RNN_UPT], const float* g, int ldg, const float* __restrict__ ur,
                                          int nc) {
#pragma unroll
  for (int v = 0; v < RNN_UPT; ++v) acc[v] = 0.f;
  for (int c = 0; c < nc; ++c) {
    const float w = __ldg(ur + c);
#pragma unroll
    for (int v = 0; v < RNN_UPT; ++v) acc[v] = fmaf(g[v * ldg + c], w, acc[v]);
  }
}

__global__ void __launch_bounds__(RNN_THREADS) rnn_backward_kernel(const __grid_constant__ RnnBwdParams p) {
  extern __shared__ float sm[];
  const int tid = threadIdx.x, nt = blockDim.x, H = p.H, GH = p.GH, ldh = odd_ld(H), ldg = p.ldg, T = p.T;
  const bool ln = p.act == ACT_LN_TANH;
  const int64_t s0 = (int64_t)blockIdx.x * p.tile;
  int* slen = reinterpret_cast<int*>(sm + p.s_len);
  float *dh = sm + p.s_dh, *dc = sm + p.s_dc, *dd = sm + p.s_dd, *q = sm + p.s_q, *sg = sm + p.s_g, *st = sm + p.s_st;
  for (int u = tid; u < p.tile; u += nt) {
    const int64_t s = s0 + u;
    slen[u] = s < p.n ? min(max(p.lens[p.users[s]], 0), T) : 0;
  }
  for (int i = tid; i < p.tile * ldh; i += nt) { dh[i] = 0.f; dc[i] = 0.f; }
  __syncthreads();
  // rows t >= len of every output are 0
  for (int u = 0; u < p.tile; ++u) {
    if (s0 + u >= p.n) break;
    const int64_t r0 = (s0 + u) * T + slen[u], nr = T - slen[u];
    for (int64_t i = tid; i < nr * GH; i += nt) {
      p.dgx[r0 * GH + i] = 0.f;
      if (p.dgh) p.dgh[r0 * GH + i] = 0.f;
    }
    if (ln)
      for (int64_t i = tid; i < nr * H; i += nt) { p.dln[r0 * H + i] = 0.f; p.dlnx[r0 * H + i] = 0.f; }
  }
  __syncthreads();
  // a len-0 user of the top layer-norm layer outputs tanh(beta) (h = 0): its dLN goes to row t = 0 (x^ = 0)
  if (ln && p.dout) {
    for (int i = tid; i < p.tile * H; i += nt) {
      const int u = i / H, j = i - u * H;
      const int64_t s = s0 + u;
      if (s >= p.n || slen[u] != 0) continue;
      const float y = tanhf(__ldg(p.gamma + H + j));
      p.dln[s * T * H + j] = p.dout[s * p.lddo + j] * (1.0f - y * y);
    }
  }
  int steps = 0;
  for (int u = 0; u < p.tile; ++u) steps = max(steps, slen[u]);
  const float* Sg = p.sv[SV_G];
  const float* Sx = p.sv[SV_X];
  const float* Shp = p.sv[SV_HP];
  const int items = H * (p.tile / RNN_UPT);
  for (int t = steps - 1; t >= 0; --t) {
    // 1. dh += dY_t (through the LN + tanh backward)
    for (int i = tid; i < p.tile * H; i += nt) {
      const int u = i / H, j = i - u * H;
      if (t >= slen[u]) continue;
      const int64_t s = s0 + u, row = s * T + t;
      const float add = p.dy ? p.dy[row * H + j] : (t == slen[u] - 1 ? p.dout[s * p.lddo + j] : 0.f);
      if (ln) {
        const float y = p.sv[SV_Y][row * H + j], xh = p.sv[SV_XH][row * H + j];
        const float dl = add * (1.0f - y * y);
        p.dln[row * H + j] = dl;
        p.dlnx[row * H + j] = dl * xh;
        q[u * ldh + j] = dl * __ldg(p.gamma + j);
      } else {
        dh[u * ldh + j] += add;
      }
    }
    __syncthreads();
    if (ln) {
      for (int u = tid; u < p.tile; u += nt) {
        if (t >= slen[u]) continue;
        const float* xh = p.sv[SV_XH] + ((s0 + u) * T + t) * H;
        float a = 0.f, b = 0.f;
        for (int j = 0; j < H; ++j) {
          a += q[u * ldh + j];
          b = fmaf(q[u * ldh + j], xh[j], b);
        }
        st[2 * u] = a / (float)H;
        st[2 * u + 1] = b / (float)H;
      }
      __syncthreads();
      for (int i = tid; i < p.tile * H; i += nt) {
        const int u = i / H, j = i - u * H;
        if (t >= slen[u]) continue;
        const int64_t row = (s0 + u) * T + t;
        const float xh = p.sv[SV_XH][row * H + j];
        dh[u * ldh + j] += p.sv[SV_RS][row] * (q[u * ldh + j] - st[2 * u] - xh * st[2 * u + 1]);
      }
      __syncthreads();
    }
    // 2. the cell: gate pre-activation gradients, the direct terms of dh_{t-1} (and dc_{t-1})
    int nc = GH;
    if (p.kind == LSTM) {
      for (int i = tid; i < p.tile * H; i += nt) {
        const int u = i / H, j = i - u * H;
        float* gs = sg + u * ldg;
        if (t >= slen[u]) {
          for (int g = 0; g < 4; ++g) gs[g * H + j] = 0.f;
          continue;
        }
        const int64_t row = (s0 + u) * T + t;
        const float* G = Sg + row * GH;
        const float ig = G[j], fg = G[H + j], gg = G[2 * H + j], og = G[3 * H + j];
        const float c1 = Sx[row * H + j], c0 = t ? Sx[(row - 1) * H + j] : 0.f;
        const float tc = cell_act(p.act, c1);
        const float dhv = dh[u * ldh + j];
        const float dcv = dc[u * ldh + j] + dhv * og * (p.act == ACT_TANH ? 1.0f - tc * tc : 1.0f);
        const float di = dcv * gg * ig * (1.0f - ig);
        const float df = dcv * c0 * fg * (1.0f - fg);
        const float dg = dcv * ig * (p.act == ACT_TANH ? 1.0f - gg * gg : 1.0f);
        const float dov = dhv * tc * og * (1.0f - og);
        dc[u * ldh + j] = dcv * fg;
        float* dG = p.dgx + row * GH;
        dG[j] = di; dG[H + j] = df; dG[2 * H + j] = dg; dG[3 * H + j] = dov;
        gs[j] = di; gs[H + j] = df; gs[2 * H + j] = dg; gs[3 * H + j] = dov;
        dd[u * ldh + j] = 0.f;
      }
    } else if (p.kind == GRU_RESET_AFTER) {
      for (int i = tid; i < p.tile * H; i += nt) {
        const int u = i / H, j = i - u * H;
        float* gs = sg + u * ldg;
        if (t >= slen[u]) {
          for (int g = 0; g < 3; ++g) gs[g * H + j] = 0.f;
          continue;
        }
        const int64_t row = (s0 + u) * T + t;
        const float* G = Sg + row * GH;
        const float z = G[j], r = G[H + j], hh = G[2 * H + j];
        const float hp = Shp[row * H + j], dhv = dh[u * ldh + j];
        const float dn = dhv * (1.0f - z) * (p.act == ACT_TANH ? 1.0f - hh * hh : 1.0f);
        const float dz = dhv * (hp - hh) * z * (1.0f - z);
        const float dr = dn * Sx[row * H + j] * r * (1.0f - r);
        float* dG = p.dgx + row * GH;
        float* dU = p.dgh + row * GH;
        dG[j] = dz; dG[H + j] = dr; dG[2 * H + j] = dn;
        dU[j] = dz; dU[H + j] = dr; dU[2 * H + j] = dn * r;
        gs[j] = dz; gs[H + j] = dr; gs[2 * H + j] = dn * r;
        dd[u * ldh + j] = dhv * z;
      }
    } else {   // GRU_RESET_BEFORE: z and the candidate first; r needs d(r o h) = dc U_c^T of every unit
      for (int i = tid; i < p.tile * H; i += nt) {
        const int u = i / H, j = i - u * H;
        float* gs = sg + u * ldg;
        if (t >= slen[u]) {
          for (int g = 0; g < 3; ++g) gs[g * H + j] = 0.f;
          continue;
        }
        const int64_t row = (s0 + u) * T + t;
        const float* G = Sg + row * GH;
        const float z = G[j], cc = G[2 * H + j];
        const float hp = Shp[row * H + j], dhv = dh[u * ldh + j];
        const float dn = dhv * (1.0f - z) * (p.act == ACT_TANH ? 1.0f - cc * cc : 1.0f);
        const float dz = dhv * (hp - cc) * z * (1.0f - z);
        float* dG = p.dgx + row * GH;
        dG[j] = dz; dG[2 * H + j] = dn;
        gs[j] = dz; gs[2 * H + j] = dn;
      }
      __syncthreads();
      for (int it = tid; it < items; it += nt) {
        const int j = it % H, u0 = (it / H) * RNN_UPT;
        float acc[RNN_UPT];
        row_chain(acc, sg + u0 * ldg + 2 * H, ldg, p.U + (int64_t)j * GH + 2 * H, H);
#pragma unroll
        for (int v = 0; v < RNN_UPT; ++v) {
          const int u = u0 + v;
          if (t >= slen[u]) continue;
          const int64_t row = (s0 + u) * T + t;
          const float z = Sg[row * GH + j], r = Sg[row * GH + H + j];
          const float dr = acc[v] * Shp[row * H + j] * r * (1.0f - r);
          p.dgx[row * GH + H + j] = dr;
          sg[u * ldg + H + j] = dr;
          dd[u * ldh + j] = dh[u * ldh + j] * z + acc[v] * r;
        }
      }
      nc = 2 * H;
    }
    __syncthreads();
    // 3. dh_{t-1} = direct + dGh_t U^T
    for (int it = tid; it < items; it += nt) {
      const int j = it % H, u0 = (it / H) * RNN_UPT;
      float acc[RNN_UPT];
      row_chain(acc, sg + u0 * ldg, ldg, p.U + (int64_t)j * GH, nc);
#pragma unroll
      for (int v = 0; v < RNN_UPT; ++v) {
        const int u = u0 + v;
        if (t < slen[u]) dh[u * ldh + j] = dd[u * ldh + j] + acc[v];
      }
    }
    __syncthreads();
  }
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int64_t b200_rnn_layer_floats(int32_t cell_kind, int32_t in_dim, int32_t hidden) {
  if (cell_kind < 0 || cell_kind > 2 || in_dim < 1 || hidden < 1) return -2;
  return rnn_layer_floats(cell_kind, in_dim, hidden);
}

// the checks, weight offsets and launch shared by b200_rnn_encode and b200_rnn_train_forward
static int rnn_encode_launch(const char* who, bool save, float* const* saved, const int64_t* users, int64_t n,
                             const int32_t* lens, const int32_t* seqs, int64_t ld_seq, int32_t T, const float* X,
                             int64_t ldx, int32_t in_dim, int32_t n_layers, const int32_t* cell_kinds,
                             const int32_t* hidden, const int32_t* acts, const float* weights, float* out, int64_t ldo,
                             void* stream) {
  B200_REQUIRE(T >= 1 && T <= RNN_MAX_T, "%s: sequence length %d outside [1, %d]", who, T, RNN_MAX_T);
  B200_REQUIRE(in_dim >= 1 && in_dim <= RNN_MAX_DIM, "%s: input width %d outside [1, %d]", who, in_dim, RNN_MAX_DIM);
  B200_REQUIRE(n_layers >= 1 && n_layers <= RNN_MAX_LAYERS, "%s: layer count %d outside [1, %d]", who, n_layers,
               RNN_MAX_LAYERS);
  B200_REQUIRE(cell_kinds && hidden && acts, "%s: null layer description", who);
  RnnParams p;
  p.T = T; p.in0 = in_dim; p.L = n_layers; p.Hmax = 1;
  int64_t woff = 0;
  for (int l = 0; l < n_layers; ++l) {
    B200_REQUIRE(cell_kinds[l] >= 0 && cell_kinds[l] <= 2, "%s: layer %d has unknown cell kind %d", who, l,
                 cell_kinds[l]);
    B200_REQUIRE(hidden[l] >= 1 && hidden[l] <= RNN_MAX_DIM, "%s: layer %d hidden size %d outside [1, %d]", who, l,
                 hidden[l], RNN_MAX_DIM);
    B200_REQUIRE(acts[l] == ACT_TANH || acts[l] == ACT_LN_TANH, "%s: layer %d has unknown activation %d", who, l,
                 acts[l]);
    p.kind[l] = cell_kinds[l]; p.H[l] = hidden[l]; p.act[l] = acts[l];
    p.in[l] = l ? hidden[l - 1] : in_dim;
    p.woff[l] = woff;
    woff += rnn_layer_floats(p.kind[l], p.in[l], p.H[l]);
    p.Hmax = std::max(p.Hmax, p.H[l]);
  }
  B200_REQUIRE(n >= 0 && n <= (int64_t)0x7fffffff * 8, "%s: bad slot count %lld", who, (long long)n);
  if (n == 0) return 0;
  B200_REQUIRE(users && lens && seqs && X && weights && out, "%s: null pointer", who);
  B200_REQUIRE(ld_seq >= T && ldx >= in_dim && ldo >= hidden[n_layers - 1], "%s: bad leading dimension", who);
  p.users = users; p.n = n; p.lens = lens; p.seqs = seqs; p.ld_seq = ld_seq; p.X = X; p.ldx = ldx; p.w = weights;
  p.out = out; p.ldo = ldo;
  for (int l = 0; l < RNN_MAX_LAYERS; ++l)
    for (int k = 0; k < 6; ++k) p.sv[l][k] = nullptr;
  if (save) {
    B200_REQUIRE(saved, "%s: null saved-tensor table", who);
    for (int l = 0; l < n_layers; ++l)
      for (int k = 0; k < 6; ++k) {
        p.sv[l][k] = saved[6 * l + k];
        B200_REQUIRE(p.sv[l][k] || (k >= SV_XH && acts[l] != ACT_LN_TANH), "%s: layer %d saved tensor %d is null",
                     who, l, k);
      }
  }
  int dev = 0, optin = 0;
  B200_CUDA_OK(cudaGetDevice(&dev));
  B200_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  // the largest tile (a multiple of RNN_UPT) within 96 KB, so that two CTAs share an SM; at least one work group
  int tile = RNN_MAX_TILE;
  while (tile > RNN_UPT && rnn_layout(p, tile) * (int64_t)sizeof(float) > 96 * 1024) tile -= RNN_UPT;
  const size_t smem = (size_t)rnn_layout(p, tile) * sizeof(float);
  B200_REQUIRE(smem <= (size_t)optin, "%s: a tile of %d users needs %zu B of shared memory, the device allows %d", who,
               tile, smem, optin);
  auto kernel = save ? rnn_encode_kernel<true> : rnn_encode_kernel<false>;
  if (smem > 48 * 1024)
    B200_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  kernel<<<(unsigned)ceil_div64(n, tile), RNN_THREADS, smem, (cudaStream_t)stream>>>(p);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_rnn_encode(const int64_t* users, int64_t n, const int32_t* lens, const int32_t* seqs,
                               int64_t ld_seq, int32_t T, const float* X, int64_t ldx, int32_t in_dim,
                               int32_t n_layers, const int32_t* cell_kinds, const int32_t* hidden,
                               const int32_t* acts, const float* weights, float* out, int64_t ldo, void* stream) {
  return rnn_encode_launch("b200_rnn_encode", false, nullptr, users, n, lens, seqs, ld_seq, T, X, ldx, in_dim,
                           n_layers, cell_kinds, hidden, acts, weights, out, ldo, stream);
}

extern "C" int b200_rnn_train_forward(const int64_t* users, int64_t n, const int32_t* lens, const int32_t* seqs,
                                      int64_t ld_seq, int32_t T, const float* X, int64_t ldx, int32_t in_dim,
                                      int32_t n_layers, const int32_t* cell_kinds, const int32_t* hidden,
                                      const int32_t* acts, const float* weights, float* out, int64_t ldo,
                                      float* const* saved, void* stream) {
  return rnn_encode_launch("b200_rnn_train_forward", true, saved, users, n, lens, seqs, ld_seq, T, X, ldx, in_dim,
                           n_layers, cell_kinds, hidden, acts, weights, out, ldo, stream);
}

extern "C" int b200_rnn_backward(const int64_t* users, int64_t n, const int32_t* lens, int32_t T, int32_t cell_kind,
                                 int32_t in_dim, int32_t hidden, int32_t act, const float* layer_weights,
                                 const float* dout, int64_t lddo, const float* dy, const float* const* saved,
                                 float* dgx, float* dgh, float* dln, float* dlnx, void* stream) {
  const char* who = "b200_rnn_backward";
  B200_REQUIRE(T >= 1 && T <= RNN_MAX_T, "%s: sequence length %d outside [1, %d]", who, T, RNN_MAX_T);
  B200_REQUIRE(in_dim >= 1 && in_dim <= RNN_MAX_DIM, "%s: input width %d outside [1, %d]", who, in_dim, RNN_MAX_DIM);
  B200_REQUIRE(hidden >= 1 && hidden <= RNN_MAX_DIM, "%s: hidden size %d outside [1, %d]", who, hidden, RNN_MAX_DIM);
  B200_REQUIRE(cell_kind >= 0 && cell_kind <= 2, "%s: unknown cell kind %d", who, cell_kind);
  B200_REQUIRE(act == ACT_TANH || act == ACT_LN_TANH, "%s: unknown activation %d", who, act);
  B200_REQUIRE(n >= 0 && n <= (int64_t)0x7fffffff * 8, "%s: bad slot count %lld", who, (long long)n);
  if (n == 0) return 0;
  const bool ln = act == ACT_LN_TANH;
  B200_REQUIRE(users && lens && layer_weights && saved && dgx, "%s: null pointer", who);
  B200_REQUIRE((dout == nullptr) != (dy == nullptr), "%s: give exactly one of dout (top layer) and dy", who);
  B200_REQUIRE(!dout || lddo >= hidden, "%s: bad leading dimension", who);
  B200_REQUIRE(cell_kind != GRU_RESET_AFTER || dgh, "%s: the Keras GRU needs dgh", who);
  for (int k = 0; k < 6; ++k)
    B200_REQUIRE(saved[k] || (k >= SV_XH && !ln), "%s: saved tensor %d is null", who, k);
  B200_REQUIRE(!ln || (dln && dlnx), "%s: a layer-norm layer needs dln and dlnx", who);
  RnnBwdParams p;
  p.T = T; p.kind = cell_kind; p.H = hidden; p.GH = cell_gates(cell_kind) * hidden; p.act = act;
  p.users = users; p.n = n; p.lens = lens;
  p.U = layer_weights + (int64_t)in_dim * p.GH;
  p.gamma = layer_weights + rnn_layer_floats(cell_kind, in_dim, hidden) - 2 * hidden;
  p.dout = dout; p.lddo = lddo; p.dy = dy;
  for (int k = 0; k < 6; ++k) p.sv[k] = saved[k];
  p.dgx = dgx; p.dgh = cell_kind == GRU_RESET_AFTER ? dgh : nullptr; p.dln = dln; p.dlnx = dlnx;
  int dev = 0, optin = 0;
  B200_CUDA_OK(cudaGetDevice(&dev));
  B200_CUDA_OK(cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev));
  int tile = RNN_MAX_TILE;
  while (tile > RNN_UPT && rnn_bwd_layout(p, tile) * (int64_t)sizeof(float) > 96 * 1024) tile -= RNN_UPT;
  const size_t smem = (size_t)rnn_bwd_layout(p, tile) * sizeof(float);
  B200_REQUIRE(smem <= (size_t)optin, "%s: a tile of %d users needs %zu B of shared memory, the device allows %d", who,
               tile, smem, optin);
  if (smem > 48 * 1024)
    B200_CUDA_OK(cudaFuncSetAttribute(rnn_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  rnn_backward_kernel<<<(unsigned)ceil_div64(n, tile), RNN_THREADS, smem, (cudaStream_t)stream>>>(p);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
