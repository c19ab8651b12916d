// The SIM general search unit (libreco/algorithms/sim.py:264-286), shared by the inference rows kernel (sim.cu) and
// the training GSU kernel (sim_train.cu) so that both select the same positions bit for bit.
#pragma once

#include <climits>

#include "common.cuh"

namespace b200 {
namespace sim {

constexpr int MAX_L = 256;
constexpr int MAX_S = 64;
constexpr int MAX_TOPK = 32;
constexpr int MAX_K = 64;
constexpr float MASK_NEG = 1.0e9f;

// One warp, one row: s_t = q . Gp[ls[t]] as acc = fmaf(q[d], Gp[ls[t]][d], acc) over d ascending (NaN -> -inf) for
// t < llen, -1e9 for llen <= t < L; then k rounds of a warp arg-max over (score desc, position asc) among the
// positions not yet taken.  Returns lane i < k's selected position in ascending order (0 on the other lanes);
// sel (the warp's [MAX_TOPK] shared slots) is scratch.
__device__ __forceinline__ int gsu_select(const float* Gp, int64_t ldg, const float* q, const int32_t* ls, int llen,
                                          int K, int L, int k, int* sel, int lane) {
  // GSU scores: lane owns positions t = lane + 32 j
  float sc[MAX_L / 32];
#pragma unroll
  for (int j = 0; j < MAX_L / 32; ++j) {
    const int t = lane + 32 * j;
    float s = -MASK_NEG;
    if (t < llen) {
      const float* g = Gp + (int64_t)__ldg(ls + t) * ldg;
      float acc = 0.f;
      for (int d = 0; d < K; ++d) acc = fmaf(__ldg(q + d), __ldg(g + d), acc);
      s = acc != acc ? -INFINITY : acc;
    }
    sc[j] = s;
  }
  // top-k: k rounds of a warp arg-max over (score desc, position asc) among the positions not yet taken
  uint32_t selm = 0;
  for (int i = 0; i < k; ++i) {
    float bv = -INFINITY;
    int bt = INT_MAX;
#pragma unroll
    for (int j = 0; j < MAX_L / 32; ++j) {
      const int t = lane + 32 * j;
      if (t < L && !((selm >> j) & 1u) && (sc[j] > bv || (sc[j] == bv && t < bt))) {
        bv = sc[j];
        bt = t;
      }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      const float ov = __shfl_xor_sync(0xffffffffu, bv, off);
      const int ot = __shfl_xor_sync(0xffffffffu, bt, off);
      if (ov > bv || (ov == bv && ot < bt)) {
        bv = ov;
        bt = ot;
      }
    }
    if ((bt & 31) == lane) selm |= 1u << (bt >> 5);
  }
  // the selected positions in ascending order
  int cnt = 0;
#pragma unroll
  for (int j = 0; j < MAX_L / 32; ++j) {
    const bool mine = (selm >> j) & 1u;
    const uint32_t ball = __ballot_sync(0xffffffffu, mine);
    if (mine) sel[cnt + __popc(ball & ((1u << lane) - 1u))] = lane + 32 * j;
    cnt += __popc(ball);
  }
  __syncwarp();
  const int pi = lane < k ? sel[lane] : 0;
  __syncwarp();
  return pi;
}

}  // namespace sim
}  // namespace b200
