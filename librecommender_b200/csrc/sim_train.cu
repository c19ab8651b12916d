// SIM training (libreco/algorithms/sim.py:193-304, training mode): the kernels the step needs besides the shared
// dense, batch-norm, loss and Adam kernels.  Every row carries its own long sequence (the collator's per-sample
// dual sequences), so here the slot is the row.
//   * b200_sim_gsu_forward: one warp per row selects the GSU positions with sim::gsu_select, the very code of the
//     inference rows kernel (same fmaf chain, same (score desc, position asc) warp top-k), and sums the first stage's
//     pooled rows Gp[long_t], t < long_len, right after the score pass has brought them into L1.
//   * b200_sim_esu_forward / _backward: one warp per (row, head), a lane per selected key; the query attends over
//     its k <= 32 selected keys.  Hidden keys (sel_pos >= long_len) get probability exactly 0 and exact-zero
//     gradient rows.  No atomics: repeated calls give identical bits.
//   * b200_sim_long_backward: the pooled and selected-row gradients into dGp (float atomics, as the DIN attention
//     backward and b200_scatter_add_rows).
#include <math.h>

#include <algorithm>

#include "../../include/b200reco.h"
#include "common.cuh"
#include "sim_gsu.cuh"

namespace b200 {
namespace {

constexpr int TRAIN_THREADS = 256;

int64_t warp_blocks(int64_t warps) {
  return std::min<int64_t>(ceil_div64(warps, TRAIN_THREADS / 32), (int64_t)(num_sms() > 0 ? num_sms() : 132) * 16);
}

int check_long(int32_t K, int32_t L, int32_t topk, const char* who) {
  B200_REQUIRE(K >= 1 && K <= sim::MAX_K, "%s: embed size %d outside [1, %d]", who, K, sim::MAX_K);
  B200_REQUIRE(L >= 1 && L <= sim::MAX_L, "%s: long sequence length %d outside [1, %d]", who, L, sim::MAX_L);
  B200_REQUIRE(topk >= 1 && topk <= std::min(sim::MAX_TOPK, (int)L), "%s: search_topk %d outside [1, min(%d, %d)]",
               who, topk, sim::MAX_TOPK, L);
  return 0;
}

int check_esu(int32_t K, int32_t H, int32_t topk, const char* who) {
  B200_REQUIRE(K >= 1 && K <= sim::MAX_K, "%s: embed size %d outside [1, %d]", who, K, sim::MAX_K);
  B200_REQUIRE(H >= 1 && K % H == 0, "%s: embed size %d is not a multiple of num_heads %d", who, K, H);
  B200_REQUIRE(topk >= 1 && topk <= sim::MAX_TOPK, "%s: search_topk %d outside [1, %d]", who, topk, sim::MAX_TOPK);
  return 0;
}

// ---- GSU + first-stage pooling: one warp per row --------------------------------------------------------------
struct GsuArgs {
  const float* Gp;
  int64_t ldg;
  int K, L, topk;
  const int64_t* items;
  const int32_t *long_seqs, *long_lens;
  int64_t ld_long, R;
  int32_t* sel_pos;
  float* pooled;
  int64_t ldp;
};

__global__ void __launch_bounds__(TRAIN_THREADS) sim_gsu_train_kernel(const __grid_constant__ GsuArgs a) {
  __shared__ int sel_sm[TRAIN_THREADS / 32][sim::MAX_TOPK];
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int K = a.K, L = a.L, k = a.topk;
  for (int64_t r = w0; r < a.R; r += nw) {
    const float* q = a.Gp + a.items[r] * a.ldg;
    const int32_t* ls = a.long_seqs + r * a.ld_long;
    const int llen = min(max(a.long_lens[r], 0), L);
    const int pi = sim::gsu_select(a.Gp, a.ldg, q, ls, llen, K, L, k, sel_sm[wib], lane);
    if (lane < k) a.sel_pos[r * k + lane] = pi;
    // pooled: lanes own columns d = lane, lane + 32; t ascending
    float p0 = 0.f, p1 = 0.f;
    for (int t = 0; t < llen; ++t) {
      const float* g = a.Gp + (int64_t)__ldg(ls + t) * a.ldg;
      if (lane < K) p0 += __ldg(g + lane);
      if (lane + 32 < K) p1 += __ldg(g + lane + 32);
    }
    float* out = a.pooled + r * a.ldp;
    if (lane < K) out[lane] = p0;
    if (lane + 32 < K) out[lane + 32] = p1;
  }
}

// ---- ESU: one warp per (row, head) ------------------------------------------------------------------------------
struct EsuArgs {
  const float *Q, *Ks, *Vs;
  int64_t ldq, ldkv;
  const int32_t *sel_pos, *long_lens;
  int64_t R;
  int K, H, topk;
  float scale;
  float *O, *P;
  int64_t ldo;
  const float* dO;
  int64_t lddo;
  float *dQ, *dKs, *dVs;
  int64_t lddq, lddkv;
};

// lane i < k: whether selected key i is visible (sel_pos < max(long_len, 1))
__device__ __forceinline__ bool esu_visible(const EsuArgs& a, int64_t r, int lane) {
  return lane < a.topk && __ldg(a.sel_pos + r * a.topk + lane) < max(__ldg(a.long_lens + r), 1);
}

__global__ void __launch_bounds__(TRAIN_THREADS) sim_esu_forward_kernel(const __grid_constant__ EsuArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int k = a.topk, hd = a.K / a.H;
  for (int64_t w = w0; w < a.R * a.H; w += nw) {
    const int64_t r = w / a.H;
    const int d0 = (int)(w - r * a.H) * hd;
    const float* q = a.Q + r * a.ldq + d0;
    const int64_t kr = r * k;
    const bool vis = esu_visible(a, r, lane);
    float v = -INFINITY;
    if (vis) {
      const float* kk = a.Ks + (kr + lane) * a.ldkv + d0;
      float acc = 0.f;
      for (int d = 0; d < hd; ++d) acc = fmaf(__ldg(q + d), __ldg(kk + d), acc);
      v = acc * a.scale;
    }
    const float mx = warp_max(v);
    const float e = vis ? expf(v - mx) : 0.f;
    const float p = e / warp_sum(e);
    if (lane < k) a.P[w * k + lane] = p;
    // o: lanes own the head's columns c = lane, lane + 32; i ascending
#pragma unroll
    for (int c0 = 0; c0 < 64; c0 += 32) {
      const int c = c0 + lane;
      float acc = 0.f;
      for (int i = 0; i < k; ++i) {
        const float pv = __shfl_sync(0xffffffffu, p, i);
        if (c < hd) acc = fmaf(pv, __ldg(a.Vs + (kr + i) * a.ldkv + d0 + c), acc);
      }
      if (c < hd) a.O[r * a.ldo + d0 + c] = acc;
    }
  }
}

// dp_i = <dO_h, V_i>, ds_i = p_i (dp_i - sum_j p_j dp_j); dQ_h = scale sum_i ds_i K_i, dK_i = scale ds_i q_h,
// dV_i = p_i dO_h; hidden keys' rows written as exact zeros.
__global__ void __launch_bounds__(TRAIN_THREADS) sim_esu_backward_kernel(const __grid_constant__ EsuArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int k = a.topk, hd = a.K / a.H;
  for (int64_t w = w0; w < a.R * a.H; w += nw) {
    const int64_t r = w / a.H;
    const int d0 = (int)(w - r * a.H) * hd;
    const float* q = a.Q + r * a.ldq + d0;
    const float* dO = a.dO + r * a.lddo + d0;
    const int64_t kr = r * k;
    const bool vis = esu_visible(a, r, lane);
    const float p = vis ? __ldg(a.P + w * k + lane) : 0.f;
    float dp = 0.f;
    if (vis) {
      const float* vv = a.Vs + (kr + lane) * a.ldkv + d0;
      for (int d = 0; d < hd; ++d) dp = fmaf(__ldg(dO + d), __ldg(vv + d), dp);
    }
    const float tot = warp_sum(p * dp);
    const float ds = vis ? p * (dp - tot) : 0.f;
    const float dss = ds * a.scale;
#pragma unroll
    for (int c0 = 0; c0 < 64; c0 += 32) {
      const int c = c0 + lane;
      const float qc = c < hd ? __ldg(q + c) : 0.f;
      const float oc = c < hd ? __ldg(dO + c) : 0.f;
      float acc = 0.f;
      for (int i = 0; i < k; ++i) {
        const float dsi = __shfl_sync(0xffffffffu, ds, i);
        const float dssi = __shfl_sync(0xffffffffu, dss, i);
        const float pi = __shfl_sync(0xffffffffu, p, i);
        const int vi = __shfl_sync(0xffffffffu, (int)vis, i);
        if (c < hd) {
          acc = fmaf(dsi, __ldg(a.Ks + (kr + i) * a.ldkv + d0 + c), acc);
          a.dKs[(kr + i) * a.lddkv + d0 + c] = vi ? dssi * qc : 0.f;
          a.dVs[(kr + i) * a.lddkv + d0 + c] = vi ? pi * oc : 0.f;
        }
      }
      if (c < hd) a.dQ[r * a.lddq + d0 + c] = acc * a.scale;
    }
  }
}

// ---- gradients into dGp: pooled rows (t < long_len) and the selected rows ------------------------------------
struct LongBwdArgs {
  const int32_t *long_seqs, *long_lens, *sel_pos;
  int64_t ld_long, R;
  int K, L, topk;
  const float *dpooled, *dXsel;
  int64_t ldp, ldx;
  float* dGp;
  int64_t ldg;
};

__global__ void __launch_bounds__(TRAIN_THREADS) sim_long_backward_kernel(const __grid_constant__ LongBwdArgs a) {
  const int lane = threadIdx.x & 31;
  const int64_t w0 = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t nw = ((int64_t)gridDim.x * blockDim.x) >> 5;
  const int K = a.K, L = a.L, k = a.topk;
  const bool c0 = lane < K, c1 = lane + 32 < K;
  for (int64_t r = w0; r < a.R; r += nw) {
    const int32_t* ls = a.long_seqs + r * a.ld_long;
    const int llen = min(max(a.long_lens[r], 0), L);
    const float* dp = a.dpooled + r * a.ldp;
    const float g0 = c0 ? __ldg(dp + lane) : 0.f, g1 = c1 ? __ldg(dp + lane + 32) : 0.f;
    for (int t = 0; t < llen; ++t) {
      float* row = a.dGp + (int64_t)__ldg(ls + t) * a.ldg;
      if (c0) atomicAdd(row + lane, g0);
      if (c1) atomicAdd(row + lane + 32, g1);
    }
    for (int i = 0; i < k; ++i) {
      const int pos = min(max(__ldg(a.sel_pos + r * k + i), 0), L - 1);
      float* row = a.dGp + (int64_t)__ldg(ls + pos) * a.ldg;
      const float* dx = a.dXsel + (r * k + i) * a.ldx;
      if (c0) atomicAdd(row + lane, __ldg(dx + lane));
      if (c1) atomicAdd(row + lane + 32, __ldg(dx + lane + 32));
    }
  }
}

}  // namespace
}  // namespace b200

using namespace b200;

extern "C" int b200_sim_gsu_forward(const float* Gp, int64_t ldg, int32_t K, const int64_t* items,
                                    const int32_t* long_seqs, int64_t ld_long, const int32_t* long_lens, int32_t L,
                                    int32_t topk, int64_t R, int32_t* sel_pos, float* pooled, int64_t ldp,
                                    void* stream) {
  const char* who = "b200_sim_gsu_forward";
  int rc = check_long(K, L, topk, who);
  if (rc != 0) return rc;
  B200_REQUIRE(Gp && items && long_seqs && long_lens && sel_pos && pooled, "%s: null pointer", who);
  B200_REQUIRE(R >= 0 && ldg >= K && ld_long >= L && ldp >= K, "%s: bad shape", who);
  if (R == 0) return 0;
  GsuArgs a;
  a.Gp = Gp; a.ldg = ldg; a.K = K; a.L = L; a.topk = topk; a.items = items; a.long_seqs = long_seqs;
  a.long_lens = long_lens; a.ld_long = ld_long; a.R = R; a.sel_pos = sel_pos; a.pooled = pooled; a.ldp = ldp;
  sim_gsu_train_kernel<<<(unsigned)warp_blocks(R), TRAIN_THREADS, 0, (cudaStream_t)stream>>>(a);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

static int esu_launch(bool backward, const EsuArgs& a, cudaStream_t st) {
  if (a.R == 0) return 0;
  const unsigned blocks = (unsigned)warp_blocks(a.R * a.H);
  if (backward)
    sim_esu_backward_kernel<<<blocks, TRAIN_THREADS, 0, st>>>(a);
  else
    sim_esu_forward_kernel<<<blocks, TRAIN_THREADS, 0, st>>>(a);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_sim_esu_forward(const float* Q, int64_t ldq, const float* Ksel, const float* Vsel, int64_t ldkv,
                                    const int32_t* sel_pos, const int32_t* long_lens, int64_t R, int32_t K, int32_t H,
                                    int32_t topk, float* O, int64_t ldo, float* P, void* stream) {
  const char* who = "b200_sim_esu_forward";
  int rc = check_esu(K, H, topk, who);
  if (rc != 0) return rc;
  B200_REQUIRE(Q && Ksel && Vsel && sel_pos && long_lens && O && P, "%s: null pointer", who);
  B200_REQUIRE(R >= 0 && ldq >= K && ldkv >= K && ldo >= K, "%s: bad shape", who);
  EsuArgs a = {};
  a.Q = Q; a.Ks = Ksel; a.Vs = Vsel; a.ldq = ldq; a.ldkv = ldkv; a.sel_pos = sel_pos; a.long_lens = long_lens;
  a.R = R; a.K = K; a.H = H; a.topk = topk; a.scale = 1.0f / sqrtf((float)(K / H)); a.O = O; a.P = P; a.ldo = ldo;
  return esu_launch(false, a, (cudaStream_t)stream);
}

extern "C" int b200_sim_esu_backward(const float* Q, int64_t ldq, const float* Ksel, const float* Vsel, int64_t ldkv,
                                     const int32_t* sel_pos, const int32_t* long_lens, int64_t R, int32_t K, int32_t H,
                                     int32_t topk, const float* P, const float* dO, int64_t lddo, float* dQ,
                                     int64_t lddq, float* dKsel, float* dVsel, int64_t lddkv, void* stream) {
  const char* who = "b200_sim_esu_backward";
  int rc = check_esu(K, H, topk, who);
  if (rc != 0) return rc;
  B200_REQUIRE(Q && Ksel && Vsel && sel_pos && long_lens && P && dO && dQ && dKsel && dVsel, "%s: null pointer", who);
  B200_REQUIRE(R >= 0 && ldq >= K && ldkv >= K && lddo >= K && lddq >= K && lddkv >= K, "%s: bad shape", who);
  EsuArgs a = {};
  a.Q = Q; a.Ks = Ksel; a.Vs = Vsel; a.ldq = ldq; a.ldkv = ldkv; a.sel_pos = sel_pos; a.long_lens = long_lens;
  a.R = R; a.K = K; a.H = H; a.topk = topk; a.scale = 1.0f / sqrtf((float)(K / H)); a.P = const_cast<float*>(P);
  a.dO = dO; a.lddo = lddo; a.dQ = dQ; a.lddq = lddq; a.dKs = dKsel; a.dVs = dVsel; a.lddkv = lddkv;
  return esu_launch(true, a, (cudaStream_t)stream);
}

extern "C" int b200_sim_long_backward(const int32_t* long_seqs, int64_t ld_long, const int32_t* long_lens, int32_t L,
                                      const int32_t* sel_pos, int32_t topk, int64_t R, int32_t K,
                                      const float* dpooled, int64_t ldp, const float* dXsel, int64_t ldx, float* dGp,
                                      int64_t ldg, void* stream) {
  const char* who = "b200_sim_long_backward";
  int rc = check_long(K, L, topk, who);
  if (rc != 0) return rc;
  B200_REQUIRE(long_seqs && long_lens && sel_pos && dpooled && dXsel && dGp, "%s: null pointer", who);
  B200_REQUIRE(R >= 0 && ld_long >= L && ldp >= K && ldx >= K && ldg >= K, "%s: bad shape", who);
  if (R == 0) return 0;
  LongBwdArgs a;
  a.long_seqs = long_seqs; a.long_lens = long_lens; a.sel_pos = sel_pos; a.ld_long = ld_long; a.R = R; a.K = K;
  a.L = L; a.topk = topk; a.dpooled = dpooled; a.dXsel = dXsel; a.ldp = ldp; a.ldx = ldx; a.dGp = dGp; a.ldg = ldg;
  sim_long_backward_kernel<<<(unsigned)warp_blocks(R), TRAIN_THREADS, 0, (cudaStream_t)stream>>>(a);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
