// Device code shared by the neighbourhood engines (swing.cu, cf.cu): per-target accumulator rows with a first-touch
// list, heavy targets split over CTAs into global split rows, the exact radix select of a row's top k, and the
// serving pieces (candidate accumulation of recommend, predict over a neighbour table).
//
// Accumulator rows.  A persistent CTA owns one row of n_targets entries, in shared memory when it fits and otherwise
// one global row per resident CTA.  The add that finds an entry untouched appends its id to the CTA's touched list,
// so clearing, counting and selection cost the row's touched entries, never n_targets.  A target too heavy for one
// CTA is cut into pieces (tasks with slot >= 0); each piece flushes its touched entries into the global row of the
// target's split slot, with its own touched list, and a finalize kernel selects from that row.
#pragma once
#include "common.cuh"

namespace b200 {
namespace nbr {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int kMaxTopK = 4096;
constexpr int kSlots = 64;                    // split targets in flight per round
constexpr int kMaxPieces = 1024;              // pieces per split target
constexpr int kMaxGlobalCtasPerSm = 4;        // global accumulator rows: bound their number
constexpr uint32_t kFiltered = 0xfffffffeu;   // recommend: a consumed item while filtering (restored to REMOVED)

// target row `item`, its entry / outer position range [pb, pe), and its split slot (-1: the whole target)
struct Task { int32_t item, pb, pe, slot; };

__host__ __device__ inline int pow2_ceil(int x) { int p = 1; while (p < x) p <<= 1; return p; }

// The 32 high bits of a selection key.  kSigned = false: the value's bits, for values >= +0 (Swing's scores).
// kSigned = true: an order-preserving map of every non-NaN float (-0.0 just below +0.0), for values of any sign.
template <bool kSigned>
__device__ __forceinline__ uint32_t value_bits(float v) {
  const uint32_t b = __float_as_uint(v);
  return kSigned ? ((b & 0x80000000u) ? ~b : (b | 0x80000000u)) : b;
}
template <bool kSigned>
__device__ __forceinline__ float bits_value(uint32_t k) {
  return __uint_as_float(kSigned ? ((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k) : k);
}

// Top min(T, top_k) of the T touched entries `tl` of a row into out_ids / out_scores (padded with -1 / 0), sorted by
// (value desc, id asc), where value_of(j) is entry j's value.  An exact 64-bit radix select on
// (value_bits << 32 | ~id), whose keys are distinct, then a bitonic sort in shared memory of at most top_k keys.
// Every thread of the CTA calls it; ends with a __syncthreads.
template <bool kSigned, typename ValueOf>
__device__ void select_topk(ValueOf value_of, const int32_t* tl, int64_t T, int top_k, int sort_cap,
                            unsigned long long* keys, int32_t* out_ids, float* out_scores) {
  __shared__ int hist[256];
  __shared__ unsigned long long s_prefix;
  __shared__ int s_need, s_n;
  const int tid = threadIdx.x;
  auto key_of = [value_of](int32_t j) -> unsigned long long {
    return ((unsigned long long)value_bits<kSigned>(value_of(j)) << 32) | (unsigned long long)(~(uint32_t)j);
  };
  unsigned long long thr = 0;
  if (T > top_k) {
    unsigned long long prefix = 0, mask = 0;
    int need = top_k;
    for (int shift = 56; shift >= 0; shift -= 8) {
      for (int b = tid; b < 256; b += blockDim.x) hist[b] = 0;
      __syncthreads();
      for (int64_t e = tid; e < T; e += blockDim.x) {
        const unsigned long long k = key_of(tl[e]);
        if ((k & mask) == prefix) atomicAdd(&hist[(k >> shift) & 255], 1);
      }
      __syncthreads();
      if (tid == 0) {
        int cum = 0, b = 255;
        for (; b > 0; --b) {
          if (cum + hist[b] >= need) break;
          cum += hist[b];
        }
        s_need = need - cum;
        s_prefix = prefix | ((unsigned long long)b << shift);
      }
      __syncthreads();
      need = s_need;
      prefix = s_prefix;
      mask |= 255ull << shift;
      __syncthreads();
    }
    thr = prefix;   // the top_k-th key itself: keys are distinct, so exactly top_k are >= thr
  }
  if (tid == 0) s_n = 0;
  for (int e = tid; e < sort_cap; e += blockDim.x) keys[e] = 0ull;
  __syncthreads();
  for (int64_t e = tid; e < T; e += blockDim.x) {
    const unsigned long long k = key_of(tl[e]);
    if (k >= thr) keys[atomicAdd(&s_n, 1)] = k;
  }
  __syncthreads();
  const int n = s_n;
  const int len = pow2_ceil(n);
  for (int k = 2; k <= len; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int t = tid; t < len; t += blockDim.x) {
        const int p = t ^ j;
        if (p > t) {
          const unsigned long long a = keys[t], b = keys[p];
          if (((t & k) == 0) ? (a < b) : (a > b)) { keys[t] = b; keys[p] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int s = tid; s < top_k; s += blockDim.x) {
    if (s < n) {
      out_ids[s] = (int32_t)~(uint32_t)(keys[s] & 0xffffffffull);
      out_scores[s] = bits_value<kSigned>((uint32_t)(keys[s] >> 32));
    } else {
      out_ids[s] = -1;
      out_scores[s] = 0.f;
    }
  }
  __syncthreads();
}

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
