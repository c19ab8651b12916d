// Swing — the item-item swing scores of recfarm (rust/src/graph.rs:147-234) on the device.  The neighbourhood
// recommend / predict of rust/src/swing.rs:153-240 over the resulting table is neighbours.cu's.
//
// Scores.  R is the user x item interaction CSR (rows sorted, duplicate-free), R^T its item x user CSR.
// w_u = 1 / sqrt(|I_u|) in fp32 (IEEE sqrt, correctly rounded reciprocal).  For a target item i and every pair of its
// users u < v (positions in row i of R^T), C = I_u ∩ I_v (i included), and the pair's term
// (w_u * w_v) * (alpha + (|C| - 1))^-1 is added to score_i[j] for every j in C, j != i.  The term is the reference's
// fp32 expression rounding for rounding; only the order of the sums differs (atomics).
//
// Layout.  A task is (item, outer position range [pb, pe), slot).  A persistent CTA takes tasks heavy first from an
// atomic counter.  For each outer user u it marks I_u in a shared-memory bitmap of the catalogue; then each warp takes
// one v > u, probes I_v against the bitmap 32 entries at a time and counts |C| with ballot / popc; when |C| >= 2 it
// adds the term to the CTA's accumulator row at every common j != i.  The accumulator row is in shared memory when
// 4 n_items bytes fit beside the bitmap, otherwise one global row per resident CTA.  Every add is a CAS loop on the
// entry's bit pattern with a plain fp32 add (add_first_touch), so subnormal terms are kept, as in the reference, and
// the one add that finds the pattern 0 (every term is > 0) appends the id to the CTA's touched list.  Clearing,
// counting and selection therefore cost the row's nonzeros, never n_items.
//
// Heavy items.  An item whose pair count exceeds the piece size is split into pieces of its outer range.  Each piece
// flushes its touched entries into a global row of the item's split slot (again add_first_touch), and a
// finalize kernel selects from that row.  At most kSlots split items are in flight per round; rounds run back to
// back, each with an even share of the unsplit items.
//
// Selection.  Per item the nonzero count is the touched count.  The top top_k entries by (score desc, id asc) are
// neighbours.cuh's exact radix select on (score bits << 32 | ~id) (scores are positive, so their bits order as floats).
#include "common.cuh"
#include "neighbours.cuh"
#include "../../include/b200reco.h"

#include <vector>

namespace b200 {
namespace swing {

using namespace nbr;

constexpr int64_t kMinPiecePairs = 1 << 15;   // an item with more pairs than max(this, total / (8 CTAs)) is split

struct Graph {
  const int64_t* user_ptr; const int32_t* user_items;
  const int64_t* item_ptr; const int32_t* item_users;
};

__device__ __forceinline__ float pair_term(float wu, float wv, float alpha, int cnt) {
  // graph.rs:185-186: user_weights[u] * user_weights[v] * (alpha + k).recip(), k = |C| - 1, all fp32
  return __fmul_rn(__fmul_rn(wu, wv), __frcp_rn(__fadd_rn(alpha, (float)(cnt - 1))));
}

// *p += v for v > 0 and *p >= 0, with a plain (non-flushing) fp32 add; true for the one add that found *p == +0.
// A float atomicAdd would not do: on global memory it flushes subnormals to zero (ATOM.ADD.F32.FTZ), so a subnormal
// term (alpha above about 4e37) would leave the entry at 0 and every later add would look like a first touch.
__device__ __forceinline__ bool add_first_touch(float* p, float v) {
  unsigned* q = reinterpret_cast<unsigned*>(p);
  unsigned old = *q;
  for (;;) {
    const unsigned prev = atomicCAS(q, old, __float_as_uint(__fadd_rn(__uint_as_float(old), v)));
    if (prev == old) return old == 0u;
    old = prev;
  }
}

__global__ void user_weights_kernel(const int64_t* __restrict__ user_ptr, int64_t n_users, float* __restrict__ w) {
  const int64_t u = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (u < n_users) w[u] = __frcp_rn(__fsqrt_rn((float)(user_ptr[u + 1] - user_ptr[u])));
}

__global__ void __launch_bounds__(THREADS) swing_scores_kernel(
    Graph g, const float* __restrict__ w, float alpha, int64_t n_items, int top_k, int sort_cap, int smem_acc,
    const Task* __restrict__ tasks, int n_tasks, unsigned* __restrict__ task_counter, float* __restrict__ acc_g,
    int32_t* __restrict__ tl_g, float* __restrict__ split_rows, int32_t* __restrict__ split_tl,
    unsigned long long* __restrict__ split_n, int32_t* __restrict__ nbr_ids, float* __restrict__ nbr_scores,
    int64_t* __restrict__ nbr_count) {
  extern __shared__ __align__(16) unsigned char smem[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem);
  uint32_t* bm = reinterpret_cast<uint32_t*>(keys + sort_cap);
  const int64_t bm_words = (n_items + 31) / 32;
  float* acc = smem_acc ? reinterpret_cast<float*>(bm + bm_words) : acc_g + (int64_t)blockIdx.x * n_items;
  int32_t* tl = tl_g + (int64_t)blockIdx.x * n_items;
  __shared__ int s_task;
  __shared__ unsigned long long s_ntl;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int64_t e = tid; e < bm_words; e += THREADS) bm[e] = 0u;
  if (smem_acc)
    for (int64_t e = tid; e < n_items; e += THREADS) acc[e] = 0.f;
  if (tid == 0) s_ntl = 0;
  __syncthreads();
  for (;;) {
    if (tid == 0) s_task = (int)atomicAdd(task_counter, 1u);
    __syncthreads();
    const int t = s_task;
    if (t >= n_tasks) break;
    const Task task = tasks[t];
    const int32_t i = task.item;
    const int64_t i0 = g.item_ptr[i];
    const int d = (int)(g.item_ptr[i + 1] - i0);
    const int32_t* users = g.item_users + i0;
    for (int p = task.pb; p < task.pe && p < d - 1; ++p) {
      const int32_t u = users[p];
      const int64_t a0 = g.user_ptr[u], a1 = g.user_ptr[u + 1];
      for (int64_t e = a0 + tid; e < a1; e += THREADS) {
        const int32_t j = g.user_items[e];
        atomicOr(&bm[j >> 5], 1u << (j & 31));
      }
      __syncthreads();
      const float wu = w[u];
      for (int q = p + 1 + warp; q < d; q += WARPS) {
        const int32_t v = users[q];
        const int64_t b0 = g.user_ptr[v], b1 = g.user_ptr[v + 1];
        int cnt = 0;
        for (int64_t e = b0; e < b1; e += 32) {
          bool hit = false;
          if (e + lane < b1) {
            const int32_t j = g.user_items[e + lane];
            hit = (bm[j >> 5] >> (j & 31)) & 1u;
          }
          cnt += __popc(__ballot_sync(0xffffffffu, hit));
        }
        if (cnt < 2) continue;              // C = {i}: nothing to add to
        const float term = pair_term(wu, w[v], alpha, cnt);
        if (term == 0.f) continue;          // an underflowed term leaves every score as it is
        for (int64_t e = b0 + lane; e < b1; e += 32) {
          const int32_t j = g.user_items[e];
          if (j != i && ((bm[j >> 5] >> (j & 31)) & 1u)) {
            if (add_first_touch(&acc[j], term)) tl[atomicAdd(&s_ntl, 1ull)] = j;
          }
        }
      }
      __syncthreads();
      for (int64_t e = a0 + tid; e < a1; e += THREADS) bm[g.user_items[e] >> 5] = 0u;
      __syncthreads();
    }
    const int64_t T = (int64_t)s_ntl;
    if (task.slot < 0) {
      if (tid == 0) nbr_count[i] = T;
      select_topk<false>([acc](int32_t j) { return acc[j]; }, tl, T, top_k, sort_cap, keys,
                         nbr_ids + (int64_t)i * top_k, nbr_scores + (int64_t)i * top_k);
    } else {
      float* row = split_rows + (int64_t)task.slot * n_items;
      int32_t* stl = split_tl + (int64_t)task.slot * n_items;
      for (int64_t e = tid; e < T; e += THREADS) {
        const int32_t j = tl[e];
        if (add_first_touch(&row[j], acc[j])) stl[atomicAdd(&split_n[task.slot], 1ull)] = j;
      }
      __syncthreads();
    }
    for (int64_t e = tid; e < T; e += THREADS) acc[tl[e]] = 0.f;
    if (tid == 0) s_ntl = 0;
    __syncthreads();
  }
}

// one CTA per split slot in use: select from the slot's row, then clear the row for the next round
__global__ void __launch_bounds__(THREADS) swing_split_finalize_kernel(
    const int32_t* __restrict__ slot_item, int top_k, int sort_cap, int64_t n_items, float* __restrict__ split_rows,
    const int32_t* __restrict__ split_tl, unsigned long long* __restrict__ split_n, int32_t* __restrict__ nbr_ids,
    float* __restrict__ nbr_scores, int64_t* __restrict__ nbr_count) {
  extern __shared__ __align__(16) unsigned char smem[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem);
  const int s = blockIdx.x;
  const int32_t i = slot_item[s];
  float* row = split_rows + (int64_t)s * n_items;
  const int32_t* stl = split_tl + (int64_t)s * n_items;
  const int64_t T = (int64_t)split_n[s];
  if (threadIdx.x == 0) nbr_count[i] = T;
  select_topk<false>([row](int32_t j) { return row[j]; }, stl, T, top_k, sort_cap, keys,
                     nbr_ids + (int64_t)i * top_k, nbr_scores + (int64_t)i * top_k);
  for (int64_t e = threadIdx.x; e < T; e += THREADS) row[stl[e]] = 0.f;
  if (threadIdx.x == 0) split_n[s] = 0;
}

// ---------------------------------------------------------------------------------------------------------------
// shared memory: [sort keys u64 sort_cap][bitmap u32 (n_items + 31) / 32][acc f32 n_items (shared path)]
Plan make_plan(int64_t n_items, int top_k) {
  return nbr::make_plan(swing_scores_kernel, n_items, top_k, sizeof(float), (size_t)(n_items + 31) / 32 * 4);
}

// the workspace: the user weights, then the scheduler's pieces
Workspace<float> carve(unsigned char* ws, int64_t n_users, int64_t n_items, const Plan& p) {
  return Workspace<float>(ws, round256((size_t)n_users * 4), n_items, p);
}

}  // namespace swing
}  // namespace b200

using namespace b200;
using namespace b200::swing;

extern "C" int b200_swing_scores_workspace_bytes(int64_t n_users, int64_t n_items, int32_t top_k, size_t* bytes) {
  B200_REQUIRE(bytes, "b200_swing_scores_workspace_bytes: null pointer");
  B200_REQUIRE(n_users >= 0 && n_items >= 1 && n_items < (1ll << 31) && n_users < (1ll << 31),
               "b200_swing_scores: bad shape");
  B200_REQUIRE(top_k >= 1 && top_k <= kMaxTopK, "b200_swing_scores: top_k %d outside [1, %d]", top_k, kMaxTopK);
  const Plan p = make_plan(n_items, top_k);
  B200_REQUIRE(p.ctas > 0, "b200_swing_scores: a %lld-item bitmap does not fit in shared memory",
               (long long)n_items);
  *bytes = carve(nullptr, n_users, n_items, p).bytes;
  return 0;
}

extern "C" int b200_swing_scores(const int64_t* user_ptr, const int32_t* user_items, int64_t n_users,
                                 const int64_t* item_ptr, const int32_t* item_users, int64_t n_items, float alpha,
                                 int32_t top_k, int32_t* nbr_ids, float* nbr_scores, int64_t* nbr_count,
                                 void* workspace, size_t workspace_bytes, void* stream_) {
  B200_REQUIRE(user_ptr && item_ptr && nbr_ids && nbr_scores && nbr_count && workspace,
               "b200_swing_scores: null pointer");
  size_t need = 0;
  if (int rc = b200_swing_scores_workspace_bytes(n_users, n_items, top_k, &need)) return rc;
  B200_REQUIRE(workspace_bytes >= need, "b200_swing_scores: workspace %zu < %zu bytes", workspace_bytes, need);
  B200_REQUIRE(alpha >= 0.f && alpha <= 3.4028235e38f, "b200_swing_scores: alpha must be finite and >= 0");
  cudaStream_t stream = (cudaStream_t)stream_;
  const Plan p = make_plan(n_items, top_k);
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  const Workspace<float> W = carve(ws, n_users, n_items, p);
  float* w = reinterpret_cast<float*>(ws);

  B200_CUDA_OK(cudaMemsetAsync(nbr_ids, 0xff, (size_t)n_items * top_k * 4, stream));
  B200_CUDA_OK(cudaMemsetAsync(nbr_scores, 0, (size_t)n_items * top_k * 4, stream));
  B200_CUDA_OK(cudaMemsetAsync(nbr_count, 0, (size_t)n_items * 8, stream));

  // plan the tasks on the host from the item degrees
  std::vector<int64_t> iptr(n_items + 1);
  B200_CUDA_OK(cudaMemcpyAsync(iptr.data(), item_ptr, (n_items + 1) * 8, cudaMemcpyDeviceToHost, stream));
  B200_CUDA_OK(cudaStreamSynchronize(stream));
  B200_REQUIRE(iptr[0] == 0, "b200_swing_scores: item_ptr[0] != 0");
  std::vector<int64_t> pairs(n_items);
  bool any_pair = false;
  for (int64_t i = 0; i < n_items; ++i) {
    const int64_t d = iptr[i + 1] - iptr[i];
    B200_REQUIRE(d >= 0 && d <= n_users, "b200_swing_scores: item %lld has a bad degree", (long long)i);
    pairs[i] = d * (d - 1) / 2;
    any_pair |= pairs[i] > 0;
  }
  if (!any_pair) return 0;

  B200_REQUIRE(n_users > 0, "b200_swing_scores: no users");
  user_weights_kernel<<<(unsigned)ceil_div64(n_users, 256), 256, 0, stream>>>(user_ptr, n_users, w);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());

  const Graph g{user_ptr, user_items, item_ptr, item_users};
  // contiguous outer ranges of about pairs / n_pieces pairs each (position q pairs with d - 1 - q users)
  auto cut = [&](int32_t i, int64_t d, int64_t n_pieces, int32_t slot, std::vector<Task>& tasks) {
    int64_t acc_pairs = 0, k = 1;
    int pb = 0;
    for (int q = 0; q < d - 1; ++q) {
      acc_pairs += d - 1 - q;
      if (acc_pairs * n_pieces >= k * pairs[i] || q == d - 2) {
        tasks.push_back(Task{i, pb, q + 1, slot});
        pb = q + 1;
        ++k;
      }
    }
  };
  auto scores = [&](int n_tasks) {
    swing_scores_kernel<<<p.ctas, THREADS, p.smem, stream>>>(
        g, w, alpha, n_items, top_k, p.sort_cap, p.smem_acc ? 1 : 0, W.tasks, n_tasks, W.counter, W.acc, W.tl,
        W.split_rows, W.split_tl, W.split_n, nbr_ids, nbr_scores, nbr_count);
  };
  auto finalize = [&](unsigned n_slots) {
    swing_split_finalize_kernel<<<n_slots, THREADS, (size_t)p.sort_cap * 8, stream>>>(
        W.slot_item, top_k, p.sort_cap, n_items, W.split_rows, W.split_tl, W.split_n, nbr_ids, nbr_scores, nbr_count);
  };
  return run_rounds(iptr, pairs, kMinPiecePairs, p, W, stream, cut, scores, finalize);
}

extern "C" int b200_swing_plan(int64_t n_items, int32_t top_k, int32_t* smem_acc, int32_t* ctas) {
  B200_REQUIRE(smem_acc && ctas, "b200_swing_plan: null pointer");
  B200_REQUIRE(n_items >= 1 && top_k >= 1 && top_k <= kMaxTopK, "b200_swing_plan: bad shape");
  const Plan p = make_plan(n_items, top_k);
  *smem_acc = p.smem_acc ? 1 : 0;
  *ctas = p.ctas;
  return 0;
}
