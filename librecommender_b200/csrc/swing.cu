// Swing — the item-item swing scores of recfarm (rust/src/graph.rs:147-234) and the neighbourhood recommend /
// predict of rust/src/swing.rs:153-240 and rust/src/inference.rs:11-96, on the device.
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
#include "philox.cuh"
#include "../../include/b200reco.h"

#include <algorithm>
#include <vector>

namespace b200 {
namespace swing {

using namespace nbr;

constexpr int64_t kMinPiecePairs = 1 << 15;   // an item with more pairs than max(this, total / (8 CTAs)) is split

struct Graph {
  const int64_t* user_ptr; const int32_t* user_items;
  const int64_t* item_ptr; const int32_t* item_users;
};

struct Plan {
  bool smem_acc;
  int ctas;
  size_t smem;       // dynamic shared memory of the scores kernel
  int sort_cap;      // power of two >= top_k
  int64_t bm_words;
};

// shared memory: [sort keys u64 sort_cap][bitmap u32 bm_words][acc f32 n_items (smem path)]
__host__ inline size_t smem_bytes(int64_t n_items, int sort_cap, bool smem_acc) {
  const int64_t bm_words = (n_items + 31) / 32;
  return (size_t)sort_cap * 8 + (size_t)bm_words * 4 + (smem_acc ? (size_t)n_items * 4 : 0);
}

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

__global__ void __launch_bounds__(THREADS) swing_recommend_kernel(
    const int64_t* __restrict__ user_ptr, const int32_t* __restrict__ user_items, const float* __restrict__ labels,
    int64_t n_users, const int32_t* __restrict__ nbr_ids, const float* __restrict__ nbr_scores,
    const int64_t* __restrict__ nbr_count, int64_t n_items, int top_k, const int64_t* __restrict__ cons_ptr,
    const int32_t* __restrict__ cons_idx, int filter, const int64_t* __restrict__ users, float* __restrict__ scores,
    int64_t ld, int64_t* __restrict__ counts) {
  const int64_t r = blockIdx.x;
  const int64_t u = users[r];
  recommend_row(u, n_users, n_items, cons_ptr, cons_idx, filter, scores + r * ld, counts + r,
                [&](uint32_t* row, unsigned long long* cand) {
    const int64_t a0 = user_ptr[u], len = user_ptr[u + 1] - a0;
    for (int64_t t = threadIdx.x; t < len * top_k; t += THREADS) {
      const int64_t e = a0 + t / top_k;
      const int s = (int)(t % top_k);
      const int32_t i = user_items[e];
      if (s >= nbr_count[i]) continue;
      const int32_t j = nbr_ids[(int64_t)i * top_k + s];
      // swing.rs:213-218: item_scores[j] += i_j_swing_score * i_label
      add_candidate(row, j, __fmul_rn(nbr_scores[(int64_t)i * top_k + s], labels[e]), cand);
    }
  });
}

// random_rec: a row with more than n_rec candidates gets a uniform key in [1, 2) per candidate, keyed by
// (seed, user, item), so its top n_rec by key is a uniform draw of n_rec distinct candidates
__global__ void __launch_bounds__(THREADS) swing_random_keys_kernel(float* __restrict__ scores, int64_t ld,
                                                                    int64_t n_items, const int64_t* __restrict__ users,
                                                                    const int64_t* __restrict__ counts, int n_rec,
                                                                    uint32_t k0, uint32_t k1) {
  const int64_t r = blockIdx.x;
  if (counts[r] <= n_rec) return;
  uint32_t* row = reinterpret_cast<uint32_t*>(scores + r * ld);
  const uint64_t u = (uint64_t)users[r];
  for (int64_t n = threadIdx.x; n < n_items; n += THREADS) {
    if (row[n] == kRemovedBits) continue;
    U4 c;
    c.x = (uint32_t)n; c.y = (uint32_t)u; c.z = (uint32_t)(u >> 32); c.w = 0x53574e47u;
    row[n] = 0x3f800000u | (philox4x32_10(c, k0, k1).x >> 9);
  }
}

// ---------------------------------------------------------------------------------------------------------------
Plan make_plan(int64_t n_items, int top_k) {
  Plan p;
  p.sort_cap = pow2_ceil(top_k);
  p.bm_words = (n_items + 31) / 32;
  int dev = 0, optin = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  const size_t reserve = 2048;     // the kernel's static shared memory
  p.smem_acc = smem_bytes(n_items, p.sort_cap, true) + reserve <= (size_t)optin;
  p.smem = smem_bytes(n_items, p.sort_cap, p.smem_acc);
  p.ctas = 0;
  if (p.smem + reserve > (size_t)optin) return p;
  if (cudaFuncSetAttribute(swing_scores_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem) !=
      cudaSuccess)
    return p;
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, swing_scores_kernel, THREADS, p.smem) != cudaSuccess)
    return p;
  if (!p.smem_acc) per_sm = std::min(per_sm, kMaxGlobalCtasPerSm);
  p.ctas = per_sm * num_sms();
  return p;
}

struct Layout {
  size_t w, counter, tasks, slot_item, tl, acc, split_rows, split_tl, split_n, total;
};

Layout layout(int64_t n_users, int64_t n_items, const Plan& p) {
  Layout L;
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t at = off; off += (bytes + 255) & ~(size_t)255; return at; };
  L.w = take((size_t)n_users * 4);
  L.counter = take(4);
  L.tasks = take(((size_t)n_items + (size_t)kSlots * kMaxPieces) * sizeof(Task));
  L.slot_item = take((size_t)kSlots * 4);
  L.tl = take((size_t)p.ctas * n_items * 4);
  L.acc = take(p.smem_acc ? 0 : (size_t)p.ctas * n_items * 4);
  L.split_rows = take((size_t)kSlots * n_items * 4);
  L.split_tl = take((size_t)kSlots * n_items * 4);
  L.split_n = take((size_t)kSlots * 8);
  L.total = off;
  return L;
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
  *bytes = layout(n_users, n_items, p).total;
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
  const Layout L = layout(n_users, n_items, p);
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  float* w = reinterpret_cast<float*>(ws + L.w);
  unsigned* counter = reinterpret_cast<unsigned*>(ws + L.counter);
  Task* tasks_d = reinterpret_cast<Task*>(ws + L.tasks);
  int32_t* slot_item_d = reinterpret_cast<int32_t*>(ws + L.slot_item);
  int32_t* tl = reinterpret_cast<int32_t*>(ws + L.tl);
  float* acc = p.smem_acc ? nullptr : reinterpret_cast<float*>(ws + L.acc);
  float* split_rows = reinterpret_cast<float*>(ws + L.split_rows);
  int32_t* split_tl = reinterpret_cast<int32_t*>(ws + L.split_tl);
  unsigned long long* split_n = reinterpret_cast<unsigned long long*>(ws + L.split_n);

  B200_CUDA_OK(cudaMemsetAsync(nbr_ids, 0xff, (size_t)n_items * top_k * 4, stream));
  B200_CUDA_OK(cudaMemsetAsync(nbr_scores, 0, (size_t)n_items * top_k * 4, stream));
  B200_CUDA_OK(cudaMemsetAsync(nbr_count, 0, (size_t)n_items * 8, stream));

  // plan the tasks on the host from the item degrees
  std::vector<int64_t> iptr(n_items + 1);
  B200_CUDA_OK(cudaMemcpyAsync(iptr.data(), item_ptr, (n_items + 1) * 8, cudaMemcpyDeviceToHost, stream));
  B200_CUDA_OK(cudaStreamSynchronize(stream));
  B200_REQUIRE(iptr[0] == 0, "b200_swing_scores: item_ptr[0] != 0");
  std::vector<int64_t> pairs(n_items);
  int64_t total = 0;
  for (int64_t i = 0; i < n_items; ++i) {
    const int64_t d = iptr[i + 1] - iptr[i];
    B200_REQUIRE(d >= 0 && d <= n_users, "b200_swing_scores: item %lld has a bad degree", (long long)i);
    pairs[i] = d * (d - 1) / 2;
    total += pairs[i];
  }
  if (total == 0) return 0;
  const int64_t piece = std::max(kMinPiecePairs, total / ((int64_t)p.ctas * 8));
  std::vector<int32_t> whole, split;
  for (int64_t i = 0; i < n_items; ++i) {
    if (pairs[i] == 0) continue;
    (pairs[i] > piece ? split : whole).push_back((int32_t)i);
  }
  auto heavier = [&](int32_t a, int32_t b) { return pairs[a] != pairs[b] ? pairs[a] > pairs[b] : a < b; };
  std::sort(whole.begin(), whole.end(), heavier);
  std::sort(split.begin(), split.end(), heavier);

  B200_REQUIRE(n_users > 0, "b200_swing_scores: no users");
  user_weights_kernel<<<(unsigned)ceil_div64(n_users, 256), 256, 0, stream>>>(user_ptr, n_users, w);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  if (!p.smem_acc) B200_CUDA_OK(cudaMemsetAsync(acc, 0, (size_t)p.ctas * n_items * 4, stream));
  B200_CUDA_OK(cudaMemsetAsync(split_rows, 0, (size_t)kSlots * n_items * 4, stream));
  B200_CUDA_OK(cudaMemsetAsync(split_n, 0, (size_t)kSlots * 8, stream));

  const Graph g{user_ptr, user_items, item_ptr, item_users};
  const int64_t rounds = std::max<int64_t>(1, ceil_div64((int64_t)split.size(), kSlots));
  std::vector<Task> tasks;
  std::vector<int32_t> slot_item;
  for (int64_t r = 0; r < rounds; ++r) {
    tasks.clear();
    slot_item.clear();
    for (int64_t s = r * kSlots; s < (int64_t)split.size() && s < (r + 1) * kSlots; ++s) {
      const int32_t i = split[s];
      const int d = (int)(iptr[i + 1] - iptr[i]);
      const int64_t n_pieces = std::min<int64_t>(kMaxPieces, ceil_div64(pairs[i], piece));
      const int32_t slot = (int32_t)slot_item.size();
      slot_item.push_back(i);
      // contiguous outer ranges of about pairs / n_pieces pairs each (position p pairs with d - 1 - p users)
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
    }
    for (size_t t = (size_t)r; t < whole.size(); t += (size_t)rounds) tasks.push_back(Task{whole[t], 0, (int32_t)(iptr[whole[t] + 1] - iptr[whole[t]]), -1});
    if (tasks.empty()) continue;
    B200_CUDA_OK(cudaMemcpyAsync(tasks_d, tasks.data(), tasks.size() * sizeof(Task), cudaMemcpyHostToDevice, stream));
    B200_CUDA_OK(cudaMemsetAsync(counter, 0, 4, stream));
    swing_scores_kernel<<<p.ctas, THREADS, p.smem, stream>>>(
        g, w, alpha, n_items, top_k, p.sort_cap, p.smem_acc ? 1 : 0, tasks_d, (int)tasks.size(), counter, acc, tl,
        split_rows, split_tl, split_n, nbr_ids, nbr_scores, nbr_count);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    if (!slot_item.empty()) {
      B200_CUDA_OK(cudaMemcpyAsync(slot_item_d, slot_item.data(), slot_item.size() * 4, cudaMemcpyHostToDevice,
                                   stream));
      const size_t fsmem = (size_t)p.sort_cap * 8;
      B200_CUDA_OK(cudaFuncSetAttribute(swing_split_finalize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                        (int)fsmem));
      swing_split_finalize_kernel<<<(unsigned)slot_item.size(), THREADS, fsmem, stream>>>(
          slot_item_d, top_k, p.sort_cap, n_items, split_rows, split_tl, split_n, nbr_ids, nbr_scores, nbr_count);
      count_launch();
      B200_CUDA_OK(cudaGetLastError());
    }
  }
  // the host task vectors are released on return: wait for the last upload to have been read
  B200_CUDA_OK(cudaStreamSynchronize(stream));
  return 0;
}

extern "C" int b200_swing_plan(int64_t n_items, int32_t top_k, int32_t* smem_acc, int32_t* ctas) {
  B200_REQUIRE(smem_acc && ctas, "b200_swing_plan: null pointer");
  B200_REQUIRE(n_items >= 1 && top_k >= 1 && top_k <= kMaxTopK, "b200_swing_plan: bad shape");
  const Plan p = make_plan(n_items, top_k);
  *smem_acc = p.smem_acc ? 1 : 0;
  *ctas = p.ctas;
  return 0;
}

extern "C" int b200_swing_recommend(const int64_t* user_ptr, const int32_t* user_items, const float* user_labels,
                                    int64_t n_users, const int32_t* nbr_ids, const float* nbr_scores,
                                    const int64_t* nbr_count, int64_t n_items, int32_t top_k,
                                    const int64_t* consumed_ptr, const int32_t* consumed_idx, int32_t filter_consumed,
                                    const int64_t* users, int64_t B, float* scores, int64_t ld, int64_t* counts,
                                    void* stream) {
  B200_REQUIRE(user_ptr && user_items && user_labels && nbr_ids && nbr_scores && nbr_count && users && scores &&
               counts, "b200_swing_recommend: null pointer");
  B200_REQUIRE(!filter_consumed || consumed_ptr, "b200_swing_recommend: filtering needs the consumed CSR");
  B200_REQUIRE(B >= 0 && B <= 0x7fffffff && n_items >= 1 && ld >= n_items && n_users >= 0,
               "b200_swing_recommend: bad shape");
  B200_REQUIRE(top_k >= 1 && top_k <= kMaxTopK, "b200_swing_recommend: bad top_k");
  if (B == 0) return 0;
  swing_recommend_kernel<<<(unsigned)B, THREADS, 0, (cudaStream_t)stream>>>(
      user_ptr, user_items, user_labels, n_users, nbr_ids, nbr_scores, nbr_count, n_items, top_k, consumed_ptr,
      consumed_idx, filter_consumed, users, scores, ld, counts);
  count_launch();
  return check_cuda(cudaGetLastError(), "swing_recommend_kernel");
}

extern "C" int b200_swing_random_keys(float* scores, int64_t ld, int64_t B, int64_t n_items, const int64_t* users,
                                      const int64_t* counts, int32_t n_rec, uint64_t seed, void* stream) {
  B200_REQUIRE(scores && users && counts, "b200_swing_random_keys: null pointer");
  B200_REQUIRE(B >= 0 && B <= 0x7fffffff && n_items >= 1 && ld >= n_items && n_rec >= 1,
               "b200_swing_random_keys: bad shape");
  if (B == 0) return 0;
  swing_random_keys_kernel<<<(unsigned)B, THREADS, 0, (cudaStream_t)stream>>>(
      scores, ld, n_items, users, counts, n_rec, (uint32_t)seed, (uint32_t)(seed >> 32));
  count_launch();
  return check_cuda(cudaGetLastError(), "swing_random_keys_kernel");
}

extern "C" int b200_swing_predict(const int64_t* user_ptr, const int32_t* user_items, int64_t n_users,
                                  const int32_t* nbr_ids, const float* nbr_scores, const int64_t* nbr_count,
                                  int64_t n_items, int32_t top_k, const int64_t* users, const int64_t* items,
                                  int64_t n, float default_pred, float* out, void* stream) {
  B200_REQUIRE(user_ptr && nbr_ids && nbr_scores && nbr_count && users && items && out,
               "b200_swing_predict: null pointer");
  B200_REQUIRE(n >= 0 && n_items >= 1 && n_users >= 0 && top_k >= 1 && top_k <= kMaxTopK,
               "b200_swing_predict: bad shape");
  if (n == 0) return 0;
  // the mean swing score of the item's first top_k neighbours that row u of R holds: compute_pred "ranking"
  neighbour_predict_kernel<false><<<(unsigned)ceil_div64(n, WARPS), THREADS, 0, (cudaStream_t)stream>>>(
      user_ptr, user_items, nullptr, n_users, nbr_ids, nbr_scores, nbr_count, n_items, top_k, users, items, n,
      default_pred, out);
  count_launch();
  return check_cuda(cudaGetLastError(), "neighbour_predict_kernel");
}
