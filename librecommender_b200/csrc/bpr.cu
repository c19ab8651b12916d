// BPR training — one epoch of libreco/algorithms/_bpr.pyx bpr_update (:30-110) on the device.
//
// Tables U [n_users, D] and I [n_items, D], D = embed_size + 1 (the last column is the item bias; U's last column
// is 1 and never written).  For every sample s = (u, p) in the given order, with a negative n:
//   diff = sum_{j<D} U[u,j] (I[p,j] - I[n,j]),  g = 1 / (1 + exp(diff))
//   grad_u = g (I[p] - I[n]) - reg U[u],  grad_p = g U[u] - reg I[p],  grad_n = -g U[u] - reg I[n]
// and the optimizer step on every updated element (gradient ascent):
//   sgd      (_bpr_update_sgd, :116-190)       w += lr grad
//   momentum (_bpr_update_momentum, :196-280)  v = momentum v + lr grad;  w += v
//   adam     (_bpr_update_adam, :286-399)      m = rho1 m + (1-rho1) grad;  h = rho2 h + (1-rho2) grad^2;
//                                              w += lr (m / (1-rho1^epoch)) / (sqrt(h / (1-rho2^epoch)) + 1e-8)
// with the caller's epoch in the bias correction, as the reference has it.
//
// Negatives (unless the caller injects items_neg): uniform over the items the user did not consume, like the
// reference's rejection loop (:150-155), drawn with ONE Philox4x32-10 draw keyed by (seed, epoch, sample index):
// r = bounded(., n_items - c_u), then the r-th unconsumed item is r + k, where k is the number of row entries with
// row[j] - j <= r (binary search on the sorted, duplicate-free CSR row).  A user whose row holds every item has
// no negative: the sample is skipped (neg_out = -1); the host rejects such input first.  All three gradients come
// from the values before the sample, as in the reference; when a negative equals the positive (possible only if the
// positive is not in the user's row) both deltas land on the row, where the reference applies them one after another.
//
// Layout: one group of G lanes (a power of two, sized from D) per sample; lane l owns elements l + G k of every
// row, the dot product is a shuffle tree inside the group.  Groups walk the samples in order with a grid stride,
// so about max_inflight consecutive samples are in flight.  Tables and optimizer state are read with plain loads
// (never the read-only path: another group's adds must be visible) and updated by red.global.add.f32 of deltas,
// so concurrent samples on the same row lose no update (a read may be stale).  max_inflight = 1 is the serial
// schedule: each element is read and written by one lane, so program order puts every read after the previous
// sample's adds — deterministic, and the sequential semantics of the reference.  fp32 SIMT.
#include <math.h>

#include "common.cuh"
#include "philox.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace bpr {

constexpr int MAX_EMBED = 128;
constexpr int THREADS = 256;
// the default schedule keeps this many warps' worth of groups per SM in flight: on the C5-like graph 16 reach at least
// 92 % of the full-occupancy rate, and on C1 Adam loses quality at full occupancy (DESIGN.md §4, "BPR training")
constexpr int DEFAULT_WARPS_PER_SM = 16;

enum { SGD = 0, MOMENTUM = 1, ADAM = 2 };

struct Args {
  const int32_t* users;
  const int32_t* items_pos;
  int64_t n;
  const int64_t* indptr;
  const int32_t* indices;
  int64_t n_items;
  float* U;
  float* I;
  float* us1;   // momentum: velocity; adam: first moment
  float* is1;
  float* us2;   // adam: second moment
  float* is2;
  int D;
  float lr, reg, momentum, rho1, rho2, c1, c2;   // c1, c2: 1 - rho^epoch
  uint32_t ctr_w, k0, k1;                         // Philox counter word 3 and keys of this epoch
  const int32_t* items_neg;
  int32_t* neg_out;
  int64_t groups;
};

// lanes per sample: the smallest power of two giving at most 4 elements per lane, at most a warp
__host__ __device__ inline int group_lanes(int D) {
  int g = 1;
  while (g < 32 && g * 4 < D) g <<= 1;
  return g;
}

__device__ __forceinline__ void red_add(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

__device__ __forceinline__ int32_t draw_negative(const Args& a, int64_t s, int32_t u) {
  const int64_t beg = __ldg(a.indptr + u), c = __ldg(a.indptr + u + 1) - beg;
  const int64_t m = a.n_items - c;
  if (m <= 0) return -1;
  U4 ctr;
  ctr.x = (uint32_t)s; ctr.y = (uint32_t)((uint64_t)s >> 32); ctr.z = 0u; ctr.w = a.ctr_w;
  const U4 r = philox4x32_10(ctr, a.k0, a.k1);
  const int64_t rank = bounded(r.x, r.y, m);
  // k = #{j : row[j] - j <= rank}; row[j] - j is non-decreasing on a sorted duplicate-free row
  int64_t lo = 0, hi = c;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if ((int64_t)__ldg(a.indices + beg + mid) - mid > rank) hi = mid; else lo = mid + 1;
  }
  return (int32_t)(rank + lo);
}

template <int G, int E, int OPT>
__global__ void __launch_bounds__(THREADS) bpr_epoch_kernel(const Args a) {
  const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
  if (gid >= a.groups) return;
  const int lane = threadIdx.x & 31;
  const int sub = lane & (G - 1);
  const unsigned mask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << (lane & ~(G - 1)));
  const int D = a.D;
  for (int64_t s = gid; s < a.n; s += a.groups) {
    const int32_t u = __ldg(a.users + s), p = __ldg(a.items_pos + s);
    const int32_t n = a.items_neg ? __ldg(a.items_neg + s) : draw_negative(a, s, u);
    if (a.neg_out && sub == 0) a.neg_out[s] = n;
    if (n < 0) continue;
    float* Uu = a.U + (int64_t)u * D;
    float* Ip = a.I + (int64_t)p * D;
    float* In = a.I + (int64_t)n * D;
    float uu[E], pp[E], nn[E];
    float part = 0.f;
#pragma unroll
    for (int k = 0; k < E; ++k) {
      const int j = sub + G * k;
      uu[k] = pp[k] = nn[k] = 0.f;
      if (j < D) {
        uu[k] = Uu[j];
        pp[k] = Ip[j];
        nn[k] = In[j];
      }
      part += uu[k] * (pp[k] - nn[k]);
    }
#pragma unroll
    for (int o = G / 2; o > 0; o >>= 1) part += __shfl_xor_sync(mask, part, o, G);
    const float g = 1.f / (1.f + expf(part));
#pragma unroll
    for (int k = 0; k < E; ++k) {
      const int j = sub + G * k;
      if (j >= D) continue;
      const bool user_col = j < D - 1;
      const float gu = g * (pp[k] - nn[k]) - a.reg * uu[k];
      const float gp = g * uu[k] - a.reg * pp[k];
      const float gn = -g * uu[k] - a.reg * nn[k];
      if (OPT == SGD) {
        if (user_col) red_add(Uu + j, a.lr * gu);
        red_add(Ip + j, a.lr * gp);
        red_add(In + j, a.lr * gn);
      } else if (OPT == MOMENTUM) {
        float* Vu = a.us1 + (Uu - a.U) + j;
        float* Vp = a.is1 + (Ip - a.I) + j;
        float* Vn = a.is1 + (In - a.I) + j;
        if (user_col) {
          const float v0 = *Vu, v = a.momentum * v0 + a.lr * gu;
          red_add(Vu, v - v0);
          red_add(Uu + j, v);
        }
        const float vp0 = *Vp, vp = a.momentum * vp0 + a.lr * gp;
        const float vn0 = *Vn, vn = a.momentum * vn0 + a.lr * gn;
        red_add(Vp, vp - vp0);
        red_add(Ip + j, vp);
        red_add(Vn, vn - vn0);
        red_add(In + j, vn);
      } else {
        const int64_t ou = (Uu - a.U) + j, op = (Ip - a.I) + j, on = (In - a.I) + j;
        auto step = [&](float* M, float* H, float* W, float grad) {
          const float m0 = *M, h0 = *H;
          const float m = a.rho1 * m0 + (1.f - a.rho1) * grad;
          const float h = a.rho2 * h0 + (1.f - a.rho2) * (grad * grad);
          red_add(M, m - m0);
          red_add(H, h - h0);
          red_add(W, a.lr * (m / a.c1) / (sqrtf(h / a.c2) + 1e-8f));
        };
        if (user_col) step(a.us1 + ou, a.us2 + ou, Uu + j, gu);
        step(a.is1 + op, a.is2 + op, Ip + j, gp);
        step(a.is1 + on, a.is2 + on, In + j, gn);
      }
    }
  }
}

template <int G, int E>
static const void* pick(int opt) {
  if (opt == SGD) return (const void*)bpr_epoch_kernel<G, E, SGD>;
  if (opt == MOMENTUM) return (const void*)bpr_epoch_kernel<G, E, MOMENTUM>;
  return (const void*)bpr_epoch_kernel<G, E, ADAM>;
}

static const void* kernel_for(int D, int opt) {
  switch (group_lanes(D)) {
    case 1: return pick<1, 4>(opt);
    case 2: return pick<2, 4>(opt);
    case 4: return pick<4, 4>(opt);
    case 8: return pick<8, 4>(opt);
    case 16: return pick<16, 4>(opt);
    default: return pick<32, 5>(opt);    // D <= 129 = 32 * 4 + 1
  }
}

}  // namespace bpr
}  // namespace b200

using namespace b200;
using namespace b200::bpr;

extern "C" int64_t b200_bpr_default_inflight(int32_t embed_size) {
  if (embed_size < 1 || embed_size > MAX_EMBED) return 0;
  const int sms = num_sms();
  return (int64_t)(sms > 0 ? sms : 1) * DEFAULT_WARPS_PER_SM * (32 / group_lanes(embed_size + 1));
}

extern "C" int b200_bpr_update(int32_t optimizer, const int32_t* users, const int32_t* items_pos, int64_t n,
                               const int64_t* indptr, const int32_t* indices, int64_t n_users, int64_t n_items,
                               float* U, float* I, int32_t embed_size, float* u_state1, float* i_state1,
                               float* u_state2, float* i_state2, float lr, float reg, float momentum, float rho1,
                               float rho2, int32_t epoch, uint64_t seed, const int32_t* items_neg, int32_t* neg_out,
                               int64_t max_inflight, void* stream) {
  B200_REQUIRE(embed_size >= 1 && embed_size <= MAX_EMBED, "b200_bpr_update: embed size %d outside [1, %d]",
               embed_size, MAX_EMBED);
  B200_REQUIRE(optimizer >= SGD && optimizer <= ADAM, "b200_bpr_update: unknown optimizer %d", optimizer);
  B200_REQUIRE(n >= 0 && n_users >= 1 && n_items >= 1 && max_inflight >= 0, "b200_bpr_update: bad sizes");
  B200_REQUIRE(n_users < (1ll << 31) && n_items < (1ll << 31), "b200_bpr_update: more than 2^31 rows");
  B200_REQUIRE(users && items_pos && indptr && indices && U && I, "b200_bpr_update: null pointer");
  B200_REQUIRE(optimizer != MOMENTUM || (u_state1 && i_state1), "b200_bpr_update: momentum needs both velocities");
  B200_REQUIRE(optimizer != ADAM || (u_state1 && i_state1 && u_state2 && i_state2),
               "b200_bpr_update: adam needs both moments of both tables");
  B200_REQUIRE(optimizer != ADAM || epoch >= 1, "b200_bpr_update: adam needs epoch >= 1, got %d", epoch);
  if (n == 0) return 0;
  const int D = embed_size + 1, G = group_lanes(D);
  int64_t groups = max_inflight > 0 ? max_inflight : b200_bpr_default_inflight(embed_size);
  if (groups > n) groups = n;
  Args a;
  a.users = users; a.items_pos = items_pos; a.n = n; a.indptr = indptr; a.indices = indices; a.n_items = n_items;
  a.U = U; a.I = I; a.us1 = u_state1; a.is1 = i_state1; a.us2 = u_state2; a.is2 = i_state2; a.D = D;
  a.lr = lr; a.reg = reg; a.momentum = momentum; a.rho1 = rho1; a.rho2 = rho2;
  a.c1 = optimizer == ADAM ? (float)(1.0 - pow((double)rho1, (double)epoch)) : 1.f;
  a.c2 = optimizer == ADAM ? (float)(1.0 - pow((double)rho2, (double)epoch)) : 1.f;
  const uint64_t ep = (uint64_t)(int64_t)epoch;
  a.ctr_w = (uint32_t)ep; a.k0 = (uint32_t)seed; a.k1 = (uint32_t)(seed >> 32) ^ (uint32_t)(ep >> 32);
  a.items_neg = items_neg; a.neg_out = neg_out; a.groups = groups;
  const int64_t threads = groups * G;
  const int block = (int)(threads < THREADS ? threads : THREADS);
  const void* fn = kernel_for(D, optimizer);
  void* params[] = {&a};
  B200_CUDA_OK(cudaLaunchKernel(fn, dim3((unsigned)ceil_div64(threads, block)), dim3(block), params, 0,
                                (cudaStream_t)stream));
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
