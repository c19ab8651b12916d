// Serving a neighbour table (Swing's, ItemCF's or UserCF's: nbr_ids / nbr_scores [n, top_k], nbr_count [n]), the
// neighbourhood recommend / predict of recfarm's rust/src/swing.rs, item_cf.rs, user_cf.rs and inference.rs.
//
// Recommend.  One CTA per user fills its dense score row with REMOVED, marks the consumed items when filtering, adds
// every term through add_candidate (the add that finds REMOVED counts a candidate), and restores the marks; the
// library's b200_topk_rows ranks the rows.  random_rec gives each candidate of a row with more than n_rec of them a
// Philox key, so the top n_rec are a uniform draw.  Predict: one warp per (row, query).
#include "common.cuh"
#include "neighbours.cuh"
#include "philox.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace nbr {

constexpr uint32_t kFiltered = 0xfffffffeu;   // recommend: a consumed item while filtering (restored to REMOVED)

// recommend: row[j] += v in a dense score row whose untouched entries hold kRemovedBits and whose filtered entries
// hold kFiltered.  The add that finds kRemovedBits stores v itself and counts one more candidate in *cand.
__device__ __forceinline__ void add_candidate(uint32_t* row, int32_t j, float v, unsigned long long* cand) {
  uint32_t old = row[j];
  for (;;) {
    if (old == kFiltered) return;
    const float nv = old == kRemovedBits ? v : __fadd_rn(__uint_as_float(old), v);
    const uint32_t prev = atomicCAS(&row[j], old, __float_as_uint(nv));
    if (prev == old) {
      if (old == kRemovedBits) atomicAdd(cand, 1ull);
      return;
    }
    old = prev;
  }
}

// recommend: fill row r (user u) of scores [B, ld] with kRemovedBits, mark u's consumed items kFiltered when
// filtering, let `accumulate(row, &cand)` add the user's terms through add_candidate, restore the filtered entries
// to kRemovedBits and write the number of candidates (entries that got a term) to *count.  A user outside
// [0, n_users) gets an all-REMOVED row and count 0.  Every thread of the CTA calls it.
template <typename Accumulate>
__device__ void recommend_row(int64_t u, int64_t n_users, int64_t n_items, const int64_t* cons_ptr,
                              const int32_t* cons_idx, int filter, float* scores_row, int64_t* count,
                              Accumulate accumulate) {
  __shared__ unsigned long long s_cand;
  uint32_t* row = reinterpret_cast<uint32_t*>(scores_row);
  for (int64_t n = threadIdx.x; n < n_items; n += blockDim.x) row[n] = kRemovedBits;
  if (threadIdx.x == 0) s_cand = 0;
  const bool known = u >= 0 && u < n_users;
  const bool filt = known && filter && cons_ptr != nullptr;
  __syncthreads();
  if (filt) {
    for (int64_t e = cons_ptr[u] + threadIdx.x; e < cons_ptr[u + 1]; e += blockDim.x) {
      const int32_t c = cons_idx[e];
      if (c >= 0 && c < n_items) row[c] = kFiltered;
    }
    __syncthreads();
  }
  if (known) accumulate(row, &s_cand);
  __syncthreads();
  if (filt) {
    for (int64_t e = cons_ptr[u] + threadIdx.x; e < cons_ptr[u + 1]; e += blockDim.x) {
      const int32_t c = cons_idx[e];
      if (c >= 0 && c < n_items) row[c] = kRemovedBits;
    }
  }
  if (threadIdx.x == 0) *count = (int64_t)s_cand;
}

// One CTA per user u = users[r].  Item-based (Swing, ItemCF): each (i, label) of row u of R and each of item i's
// first min(top_k, nbr_count[i]) neighbours (j, s) add s * label at j.  User-based (UserCF): each of u's first
// min(top_k, nbr_count[u]) neighbours (v, sim) gets a warp, whose lanes add sim * label at each (i, label) of row v.
template <bool kUserBased>
__global__ void __launch_bounds__(THREADS) neighbour_recommend_kernel(
    const int64_t* __restrict__ user_ptr, const int32_t* __restrict__ user_items, const float* __restrict__ labels,
    int64_t n_users, const int32_t* __restrict__ nbr_ids, const float* __restrict__ nbr_scores,
    const int64_t* __restrict__ nbr_count, int64_t n_items, int top_k, const int64_t* __restrict__ cons_ptr,
    const int32_t* __restrict__ cons_idx, int filter, const int64_t* __restrict__ users, float* __restrict__ scores,
    int64_t ld, int64_t* __restrict__ counts) {
  const int64_t r = blockIdx.x;
  const int64_t u = users[r];
  recommend_row(u, n_users, n_items, cons_ptr, cons_idx, filter, scores + r * ld, counts + r,
                [&](uint32_t* row, unsigned long long* cand) {
    if constexpr (kUserBased) {
      const int kk = (int)min((int64_t)top_k, nbr_count[u]);
      const int lane = threadIdx.x & 31;
      for (int s = threadIdx.x >> 5; s < kk; s += WARPS) {
        const int32_t v = nbr_ids[u * top_k + s];
        const float sim = nbr_scores[u * top_k + s];
        for (int64_t e = user_ptr[v] + lane; e < user_ptr[v + 1]; e += 32)
          add_candidate(row, user_items[e], __fmul_rn(sim, labels[e]), cand);   // user_cf.rs: u_v_sim * v_i_score
      }
    } else {
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
    }
  });
}

// random_rec: a row with more than n_rec candidates gets a uniform key in [1, 2) per candidate, keyed by
// (seed, user, item), so its top n_rec by key is a uniform draw of n_rec distinct candidates
__global__ void __launch_bounds__(THREADS) neighbour_random_keys_kernel(
    float* __restrict__ scores, int64_t ld, int64_t n_items, const int64_t* __restrict__ users,
    const int64_t* __restrict__ counts, int n_rec, uint32_t k0, uint32_t k1) {
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

// One warp per (row r, query q): the first min(top_k, nbr_count[q]) neighbours of q, intersected with row r of a
// sorted CSR (ptr / idx, and labels for kRating), recfarm's compute_pred (inference.rs:48-71):
//   ranking: sum of the intersected neighbours' scores / their number;
//   rating:  sum over them of label * sim / (sum of their sims), each term as written (a zero sum gives NaN or inf).
// default_pred for an id outside range or an empty intersection.
template <bool kRating>
__global__ void __launch_bounds__(THREADS) neighbour_predict_kernel(
    const int64_t* __restrict__ ptr, const int32_t* __restrict__ idx, const float* __restrict__ labels,
    int64_t n_rows, const int32_t* __restrict__ nbr_ids, const float* __restrict__ nbr_scores,
    const int64_t* __restrict__ nbr_count, int64_t n_queries, int top_k, const int64_t* __restrict__ rows,
    const int64_t* __restrict__ queries, int64_t n, float default_pred, float* __restrict__ out) {
  const int64_t r = ((int64_t)blockIdx.x * THREADS + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const int64_t u = rows[r], i = queries[r];
  if (u < 0 || u >= n_rows || i < 0 || i >= n_queries) {
    if (lane == 0) out[r] = default_pred;
    return;
  }
  const int kk = (int)min((int64_t)top_k, nbr_count[i]);
  const int64_t a0 = ptr[u], a1 = ptr[u + 1];
  float sum = 0.f;
  int hits = 0;
  for (int s = lane; s < kk && a1 > a0; s += 32) {
    const int32_t j = nbr_ids[i * top_k + s];
    int64_t lo = a0, hi = a1;          // row u is sorted: lower bound of j
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (idx[mid] < j) lo = mid + 1; else hi = mid;
    }
    if (lo < a1 && idx[lo] == j) {
      sum += nbr_scores[i * top_k + s];
      ++hits;
    }
  }
  sum = warp_sum(sum);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) hits += __shfl_xor_sync(0xffffffffu, hits, o);
  if (!kRating) {
    if (lane == 0) out[r] = hits ? __fdiv_rn(sum, (float)hits) : default_pred;
    return;
  }
  if (!hits) {
    if (lane == 0) out[r] = default_pred;
    return;
  }
  float acc = 0.f;                   // rating: a second pass over the hits, once their sum of sims is known
  for (int s = lane; s < kk; s += 32) {
    const int32_t j = nbr_ids[i * top_k + s];
    int64_t lo = a0, hi = a1;
    while (lo < hi) {
      const int64_t mid = (lo + hi) >> 1;
      if (idx[mid] < j) lo = mid + 1; else hi = mid;
    }
    if (lo < a1 && idx[lo] == j) acc += __fdiv_rn(__fmul_rn(labels[lo], nbr_scores[i * top_k + s]), sum);
  }
  acc = warp_sum(acc);
  if (lane == 0) out[r] = acc;
}

}  // namespace nbr
}  // namespace b200

using namespace b200;
using namespace b200::nbr;

extern "C" int b200_nbr_recommend(const int64_t* user_ptr, const int32_t* user_items, const float* user_labels,
                                  int64_t n_users, const int32_t* nbr_ids, const float* nbr_scores,
                                  const int64_t* nbr_count, int64_t n_items, int32_t top_k, int32_t user_based,
                                  const int64_t* consumed_ptr, const int32_t* consumed_idx, int32_t filter_consumed,
                                  const int64_t* users, int64_t B, float* scores, int64_t ld, int64_t* counts,
                                  void* stream) {
  B200_REQUIRE(user_ptr && user_items && user_labels && nbr_ids && nbr_scores && nbr_count && users && scores &&
               counts, "b200_nbr_recommend: null pointer");
  B200_REQUIRE(!filter_consumed || consumed_ptr, "b200_nbr_recommend: filtering needs the consumed CSR");
  B200_REQUIRE(B >= 0 && B <= 0x7fffffff && n_items >= 1 && ld >= n_items && n_users >= 0,
               "b200_nbr_recommend: bad shape");
  B200_REQUIRE(top_k >= 1 && top_k <= kMaxTopK, "b200_nbr_recommend: bad top_k");
  if (B == 0) return 0;
  auto kernel = user_based ? neighbour_recommend_kernel<true> : neighbour_recommend_kernel<false>;
  kernel<<<(unsigned)B, THREADS, 0, (cudaStream_t)stream>>>(
      user_ptr, user_items, user_labels, n_users, nbr_ids, nbr_scores, nbr_count, n_items, top_k, consumed_ptr,
      consumed_idx, filter_consumed, users, scores, ld, counts);
  count_launch();
  return check_cuda(cudaGetLastError(), "neighbour_recommend_kernel");
}

extern "C" int b200_nbr_random_keys(float* scores, int64_t ld, int64_t B, int64_t n_items, const int64_t* users,
                                    const int64_t* counts, int32_t n_rec, uint64_t seed, void* stream) {
  B200_REQUIRE(scores && users && counts, "b200_nbr_random_keys: null pointer");
  B200_REQUIRE(B >= 0 && B <= 0x7fffffff && n_items >= 1 && ld >= n_items && n_rec >= 1,
               "b200_nbr_random_keys: bad shape");
  if (B == 0) return 0;
  neighbour_random_keys_kernel<<<(unsigned)B, THREADS, 0, (cudaStream_t)stream>>>(
      scores, ld, n_items, users, counts, n_rec, (uint32_t)seed, (uint32_t)(seed >> 32));
  count_launch();
  return check_cuda(cudaGetLastError(), "neighbour_random_keys_kernel");
}

extern "C" int b200_nbr_predict(const int64_t* ptr, const int32_t* idx, const float* labels, int64_t n_rows,
                                const int32_t* nbr_ids, const float* nbr_scores, const int64_t* nbr_count,
                                int64_t n_queries, int32_t top_k, const int64_t* rows, const int64_t* queries,
                                int64_t n, int32_t task, float default_pred, float* out, void* stream) {
  B200_REQUIRE(ptr && (labels || task == 1) && nbr_ids && nbr_scores && nbr_count && rows && queries && out,
               "b200_nbr_predict: null pointer");
  B200_REQUIRE(n >= 0 && n_queries >= 1 && n_rows >= 0 && top_k >= 1 && top_k <= kMaxTopK,
               "b200_nbr_predict: bad shape");
  B200_REQUIRE(task == 0 || task == 1, "b200_nbr_predict: task %d is neither 0 (rating) nor 1 (ranking)", task);
  if (n == 0) return 0;
  auto kernel = task == 0 ? neighbour_predict_kernel<true> : neighbour_predict_kernel<false>;
  kernel<<<(unsigned)ceil_div64(n, WARPS), THREADS, 0, (cudaStream_t)stream>>>(
      ptr, idx, labels, n_rows, nbr_ids, nbr_scores, nbr_count, n_queries, top_k, rows, queries, n, default_pred,
      out);
  count_launch();
  return check_cuda(cudaGetLastError(), "neighbour_predict_kernel");
}
