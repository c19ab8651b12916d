// K7 — on-device negative sampler (the "fast mode" of SURVEY.md §7.2-1).
//
// Replaces, in distribution and in the rejection rules, the host samplers of
// libreco/sampling/negatives.py:17-82 used by BaseCollator.sample_neg_items
// (libreco/batch/collators.py:138-166).  The reference draws from numpy's PCG64 / Python's
// Mersenne Twister — sequential generators; bit-exact reproduction of those streams is the
// PARITY mode and stays on the host (librecommender_b200/sampling.py).  This kernel uses a
// counter-based generator (Philox4x32-10) so that every (sample, attempt) is independent and the
// result is a pure function of (seed, step, index): oracle/sampling.py restates it bit-exactly.
//
//   mode 0 "random"     (negatives.py:17-31): uniform over items; a draw equal to ITS OWN positive is
//                        re-drawn, at most `tolerance` times.
//   mode 1 "unconsumed" (negatives.py:55-82): additionally rejects items the user consumed (binary
//                        search in the per-user SORTED consumed list) and negatives already drawn for
//                        the same positive; after `tolerance` failures the consumed test is dropped
//                        for another `tolerance` tries, then the draw is accepted (same relaxation).
//   mode 2 "popular"    (negatives.py:34-43): inverse-CDF draw from p ~ freq^0.75 (cdf given),
//                        one re-draw when equal to the positive.
// Layout: negatives of positive j are out[j*num_neg : (j+1)*num_neg] (collators.py:231-232).
// Also here: the per-sample history windows (b200_interacted_seqs, SIM's b200_interacted_dual_seqs) and the unique
// candidate sampler of the sampled-class losses (b200_unique_candidates, training/tf_trainer.py:162-245).
#include "common.cuh"
#include "philox.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace sampler {

__device__ __forceinline__ bool in_sorted(const int32_t* __restrict__ a, int64_t beg, int64_t end, int32_t v) {
  while (beg < end) {
    const int64_t mid = (beg + end) >> 1;
    const int32_t x = __ldg(a + mid);
    if (x == v) return true;
    if (x < v) beg = mid + 1; else end = mid;
  }
  return false;
}

__device__ __forceinline__ int64_t draw(int mode, const float* __restrict__ cdf, int64_t n_items,
                                        uint64_t seed, uint64_t step, uint64_t index, uint32_t attempt) {
  U4 c;
  c.x = (uint32_t)index; c.y = (uint32_t)(index >> 32); c.z = attempt; c.w = (uint32_t)step;
  const U4 r = philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32));
  if (mode != 2) return bounded(r.x, r.y, n_items);
  // inverse CDF: first index whose cdf >= u, u in [0,1) with 24 random bits
  const float u = (float)(r.x >> 8) * (1.0f / 16777216.0f);
  int64_t lo = 0, hi = n_items - 1;
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (__ldg(cdf + mid) > u) hi = mid; else lo = mid + 1;
  }
  return lo;
}

__global__ void sample_negatives_kernel(const int64_t* __restrict__ users,
                                        const int64_t* __restrict__ items_pos, int64_t n_pos,
                                        int num_neg, int64_t n_items, int mode, int tolerance,
                                        uint64_t seed, uint64_t step,
                                        const int64_t* __restrict__ indptr,
                                        const int32_t* __restrict__ idx_sorted, int64_t n_users,
                                        const float* __restrict__ cdf, int64_t* __restrict__ out) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_pos) return;
  const int64_t pos = items_pos[j];
  int64_t beg = 0, end = 0;
  if (mode == 1) {
    const int64_t u = users[j];
    if (u >= 0 && u < n_users) { beg = indptr[u]; end = indptr[u + 1]; }
  }
  int64_t* o = out + j * num_neg;
  for (int t = 0; t < num_neg; ++t) {
    const uint64_t index = (uint64_t)(j * num_neg + t);
    uint32_t attempt = 0;
    int64_t n = draw(mode, cdf, n_items, seed, step, index, attempt++);
    if (mode == 0) {
      for (int a = 0; a < tolerance && n == pos; ++a) n = draw(mode, cdf, n_items, seed, step, index, attempt++);
    } else if (mode == 2) {
      if (n == pos) n = draw(mode, cdf, n_items, seed, step, index, attempt++);
    } else {
      bool ok = false;
      for (int a = 0; a < tolerance; ++a) {
        bool dup = false;
        for (int s = 0; s < t; ++s) dup |= (o[s] == n);
        if (n != pos && !dup && !in_sorted(idx_sorted, beg, end, (int32_t)n)) { ok = true; break; }
        n = draw(mode, cdf, n_items, seed, step, index, attempt++);
      }
      if (!ok) {
        for (int a = 0; a < tolerance; ++a) {
          bool dup = false;
          for (int s = 0; s < t; ++s) dup |= (o[s] == n);
          if (n != pos && !dup) break;
          n = draw(mode, cdf, n_items, seed, step, index, attempt++);
        }
      }
    }
    o[t] = n;
  }
}

// ---- per-sample behaviour sequences at collate time (libreco/batch/sequence.py:33-71, mode "recent")
// One warp per sample.  position = FIRST occurrence of the item in the user's time-ordered consumed
// list (list.index); an item the user never consumed (a sampled negative) takes a random position
// (random.randrange(0, len) in the reference: `rand_pos` carries that stream in parity mode, else
// Philox(seed, step, j)).  seq = consumed[max(0, position - L) : position], padded with pad_index;
// len = min(position, L), 1 when position == 0 (reference :56-58).
// One warp per sample: the sample's position in its user's list and the list's bounds [beg, beg + clen).
__device__ __forceinline__ int64_t interacted_position(const int64_t* __restrict__ indptr,
                                                       const int32_t* __restrict__ idx, int64_t n_users,
                                                       const int64_t* __restrict__ users,
                                                       const int64_t* __restrict__ items, int64_t j,
                                                       const int64_t* __restrict__ rand_pos, uint64_t seed,
                                                       uint64_t step, int lane, int64_t& beg) {
  const int64_t u = users[j];
  int64_t end = 0;
  beg = 0;
  if (u >= 0 && u < n_users) { beg = indptr[u]; end = indptr[u + 1]; }
  const int64_t clen = end - beg;
  const int64_t item = items[j];
  int64_t pos = -1;
  for (int64_t base = 0; base < clen && pos < 0; base += 32) {
    const bool in = base + lane < clen;
    const bool hit = in && (int64_t)__ldg(idx + beg + base + lane) == item;
    const unsigned m = __ballot_sync(0xffffffffu, hit);
    if (m) pos = base + (__ffs(m) - 1);
  }
  if (pos < 0) {
    if (clen == 0) pos = 0;
    else if (rand_pos) pos = min(max(rand_pos[j], (int64_t)0), clen - 1);
    else {
      U4 c;
      c.x = (uint32_t)j; c.y = (uint32_t)((uint64_t)j >> 32); c.z = 0x5e9u; c.w = (uint32_t)step;
      const U4 r = philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32));
      pos = bounded(r.x, r.y, clen);
    }
  }
  return pos;
}

__global__ void interacted_seqs_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ idx,
                                       int64_t n_users, const int64_t* __restrict__ users,
                                       const int64_t* __restrict__ items, int64_t n, int L, int32_t pad_index,
                                       const int64_t* __restrict__ rand_pos, uint64_t seed, uint64_t step,
                                       int32_t* __restrict__ seqs, int32_t* __restrict__ lens) {
  const int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= n) return;
  int64_t beg;
  const int64_t pos = interacted_position(indptr, idx, n_users, users, items, j, rand_pos, seed, step, lane, beg);
  const int64_t count = pos < L ? pos : L;
  const int64_t start = pos - count;
  for (int t = lane; t < L; t += 32)
    seqs[j * L + t] = t < count ? __ldg(idx + beg + start + t) : pad_index;
  if (lane == 0) lens[j] = pos == 0 ? 1 : (int32_t)count;
}

// ---- SIM's per-sample dual sequences at collate time (libreco/batch/sequence.py:94-147, called from
// batch/collators.py:114-116).  Same position rule as above.  With p the position: short = consumed[p - s : p],
// s = min(p, S); long = the up to L items before the short window, consumed[p - s - l : p - s], l = min(p - S, L)
// when p > S and 0 otherwise.  Both padded with pad_index; each length is max(count, 1) (position 0 gives two
// all-pad rows of length 1, 1 <= p <= S an all-pad long row of length 1).
__global__ void interacted_dual_seqs_kernel(const int64_t* __restrict__ indptr, const int32_t* __restrict__ idx,
                                            int64_t n_users, const int64_t* __restrict__ users,
                                            const int64_t* __restrict__ items, int64_t n, int L, int S,
                                            int32_t pad_index, const int64_t* __restrict__ rand_pos, uint64_t seed,
                                            uint64_t step, int32_t* __restrict__ long_seqs,
                                            int32_t* __restrict__ long_lens, int32_t* __restrict__ short_seqs,
                                            int32_t* __restrict__ short_lens) {
  const int64_t j = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (j >= n) return;
  int64_t beg;
  const int64_t pos = interacted_position(indptr, idx, n_users, users, items, j, rand_pos, seed, step, lane, beg);
  const int64_t s_cnt = pos < S ? pos : S;
  const int64_t l_cnt = pos <= S ? 0 : (pos - S < L ? pos - S : L);
  const int64_t s_start = pos - s_cnt, l_start = s_start - l_cnt;
  for (int t = lane; t < L; t += 32)
    long_seqs[j * L + t] = t < l_cnt ? __ldg(idx + beg + l_start + t) : pad_index;
  for (int t = lane; t < S; t += 32)
    short_seqs[j * S + t] = t < s_cnt ? __ldg(idx + beg + s_start + t) : pad_index;
  if (lane == 0) {
    long_lens[j] = l_cnt > 0 ? (int32_t)l_cnt : 1;
    short_lens[j] = s_cnt > 0 ? (int32_t)s_cnt : 1;
  }
}

// ---- unique candidate sampler of the sampled-class losses (YouTubeRetrieval training): TensorFlow's
// uniform_candidate_sampler / log_uniform_candidate_sampler with unique=True (range_sampler.cc SampleBatch...):
// draws with replacement, keeps the FIRST occurrence of every id until S distinct ids are held, num_tries = the
// number of draws taken.  Draw j is Philox(seed, step, j); the result is that sequential process over the draw
// stream.  One CTA: a round draws j = base .. base + blockDim - 1, every draw claims its id in owner[] with
// atomicMin(j) (the lowest draw index of the round wins a tie, an id owned by an earlier round keeps its owner),
// a draw is fresh iff it owns its id, and a block scan over the fresh flags gives the output ranks in draw order.
// owner[] (one uint32 per item, 0xFFFFFFFF = free) is left free again by walking the S kept ids and the last
// round's draws after the stop: O(S) per call, never O(n_items).
constexpr int UNIQ_THREADS = 1024;
constexpr uint32_t UNIQ_FREE = 0xFFFFFFFFu;
constexpr uint32_t UNIQ_MAX_DRAWS = 1u << 31;

__device__ __forceinline__ int64_t candidate(int kind, int64_t n_items, double log_range, uint64_t seed,
                                             uint64_t step, uint32_t j) {
  U4 c;
  c.x = j; c.y = 0u; c.z = 0xca7du; c.w = (uint32_t)step;
  const U4 r = philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32));
  if (kind == 0) return bounded(r.x, r.y, n_items);
  // LogUniformSampler::Sample: (int64)exp(u * log1p(range)) - 1, then % range; u = 53 random bits in [0, 1)
  const double u = (double)((((uint64_t)r.z << 32) | r.w) >> 11) * 0x1.0p-53;
  const int64_t v = (int64_t)exp(u * log_range) - 1;
  return v % n_items;
}

__global__ void __launch_bounds__(UNIQ_THREADS)
unique_candidates_kernel(int kind, int64_t n_items, int S, uint64_t seed, const int64_t* __restrict__ step_dev,
                         uint32_t* __restrict__ owner, int64_t* __restrict__ out, int64_t* __restrict__ num_tries) {
  __shared__ int warp_cnt[UNIQ_THREADS / 32];
  __shared__ uint32_t s_stop;
  const uint64_t step = (uint64_t)*step_dev;
  const double log_range = log1p((double)n_items);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  int have = 0;                      // ids kept before the current round (block-uniform)
  uint32_t stop, j;
  int64_t id;
  if (tid == 0) s_stop = 0u;
  for (uint32_t base = 0;; base += UNIQ_THREADS) {
    j = base + tid;
    id = candidate(kind, n_items, log_range, seed, step, j);
    atomicMin(owner + id, j);
    __syncthreads();
    const bool fresh = __ldcg(owner + id) == j;          // L2 read: the atomics bypass L1
    const unsigned m = __ballot_sync(0xffffffffu, fresh);
    if (lane == 0) warp_cnt[warp] = __popc(m);
    __syncthreads();
    int before = 0, total = 0;
    for (int w = 0; w < UNIQ_THREADS / 32; ++w) {
      const int c = warp_cnt[w];
      total += c;
      before += w < warp ? c : 0;
    }
    const int rank = have + before + __popc(m & ((1u << lane) - 1u));
    if (fresh && rank < S) out[rank] = id;
    if (fresh && rank == S - 1) s_stop = j + 1u;
    const bool last = have + total >= S || base + UNIQ_THREADS >= UNIQ_MAX_DRAWS;
    have = min(have + total, S);
    __syncthreads();
    if (last) {
      stop = s_stop ? s_stop : base + UNIQ_THREADS;
      break;
    }
  }
  if (tid == 0) *num_tries = (int64_t)stop;
  // free the owner slots again: draws of the last round after the stop, then every kept id
  if (j >= stop) owner[id] = UNIQ_FREE;
  for (int i = tid; i < have; i += UNIQ_THREADS) owner[out[i]] = UNIQ_FREE;
}

}  // namespace sampler
}  // namespace b200

using namespace b200;

extern "C" size_t b200_unique_candidates_workspace_bytes(int64_t n_items) {
  return n_items > 0 ? (size_t)n_items * sizeof(uint32_t) : 0;
}

extern "C" int b200_unique_candidates(int32_t kind, int64_t n_items, int32_t num_sampled, uint64_t seed,
                                      const int64_t* step_dev, void* workspace, size_t workspace_bytes, int64_t* out,
                                      int64_t* num_tries, void* stream) {
  B200_REQUIRE(kind == 0 || kind == 1, "b200_unique_candidates: kind must be 0 (uniform) or 1 (log-uniform)");
  B200_REQUIRE(n_items >= 1 && n_items < ((int64_t)1 << 31), "b200_unique_candidates: n_items %lld outside [1, 2^31)",
               (long long)n_items);
  B200_REQUIRE(num_sampled >= 1 && num_sampled <= B200_UNIQUE_MAX_SAMPLED && num_sampled <= n_items,
               "b200_unique_candidates: num_sampled %d outside [1, min(n_items, %d)]", num_sampled,
               B200_UNIQUE_MAX_SAMPLED);
  B200_REQUIRE(step_dev && out && num_tries && workspace, "b200_unique_candidates: null pointer");
  B200_REQUIRE(workspace_bytes >= b200_unique_candidates_workspace_bytes(n_items),
               "b200_unique_candidates: workspace too small");
  sampler::unique_candidates_kernel<<<1, sampler::UNIQ_THREADS, 0, (cudaStream_t)stream>>>(
      kind, n_items, num_sampled, seed, step_dev, (uint32_t*)workspace, out, num_tries);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_interacted_seqs(const int64_t* indptr, const int32_t* idx, int64_t n_users,
                                    const int64_t* users, const int64_t* items, int64_t n,
                                    int32_t max_seq_len, int32_t pad_index, const int64_t* rand_pos,
                                    uint64_t seed, uint64_t step, int32_t* seqs, int32_t* lens, void* stream) {
  B200_REQUIRE(indptr && idx && users && items && seqs && lens, "b200_interacted_seqs: null pointer");
  B200_REQUIRE(max_seq_len >= 1, "b200_interacted_seqs: max_seq_len must be positive");
  if (n == 0) return 0;
  sampler::interacted_seqs_kernel<<<(unsigned)ceil_div64(n * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      indptr, idx, n_users, users, items, n, max_seq_len, pad_index, rand_pos, seed, step, seqs, lens);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_interacted_dual_seqs(const int64_t* indptr, const int32_t* idx, int64_t n_users,
                                         const int64_t* users, const int64_t* items, int64_t n, int32_t long_max_len,
                                         int32_t short_max_len, int32_t pad_index, const int64_t* rand_pos,
                                         uint64_t seed, uint64_t step, int32_t* long_seqs, int32_t* long_lens,
                                         int32_t* short_seqs, int32_t* short_lens, void* stream) {
  B200_REQUIRE(indptr && idx && users && items && long_seqs && long_lens && short_seqs && short_lens,
               "b200_interacted_dual_seqs: null pointer");
  B200_REQUIRE(long_max_len >= 1 && short_max_len >= 1, "b200_interacted_dual_seqs: lengths must be positive");
  if (n == 0) return 0;
  sampler::interacted_dual_seqs_kernel<<<(unsigned)ceil_div64(n * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      indptr, idx, n_users, users, items, n, long_max_len, short_max_len, pad_index, rand_pos, seed, step, long_seqs,
      long_lens, short_seqs, short_lens);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_sample_negatives(const int64_t* users, const int64_t* items_pos, int64_t n_pos,
                                     int32_t num_neg, int64_t n_items, int32_t mode,
                                     int32_t tolerance, uint64_t seed, uint64_t step,
                                     const int64_t* indptr, const int32_t* idx_sorted,
                                     int64_t n_users, const float* cdf, int64_t* out, void* stream) {
  B200_REQUIRE(items_pos && out, "b200_sample_negatives: null pointer");
  B200_REQUIRE(mode >= 0 && mode <= 2, "b200_sample_negatives: unknown mode %d", mode);
  B200_REQUIRE(mode != 1 || (users && indptr && idx_sorted), "unconsumed sampler needs users + sorted consumed CSR");
  B200_REQUIRE(mode != 2 || cdf, "popular sampler needs the cdf");
  B200_REQUIRE(num_neg >= 1 && n_items >= 2, "b200_sample_negatives: bad num_neg / n_items");
  if (n_pos == 0) return 0;
  sampler::sample_negatives_kernel<<<(unsigned)ceil_div64(n_pos, 128), 128, 0, (cudaStream_t)stream>>>(
      users, items_pos, n_pos, num_neg, n_items, mode, tolerance, seed, step, indptr, idx_sorted,
      n_users, cdf, out);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
