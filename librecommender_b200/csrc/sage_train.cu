// GraphSage training — the device pieces of the reference's GraphCollator (libreco/batch/collators.py:338-386) and
// of the backward of the non-DGL GraphSageModel encoder (libreco/algorithms/torch_modules/graphsage_module.py:82-140).
//
//   b200_sage_aggregate_backward  backward of b200_sage_aggregate in mean mode (no weights): dout[r] = d loss /
//                                 d [h_self | mean_nb] of row r; dout[r, :d] is added into the self row and
//                                 dout[r, d:] / len into each neighbour row of r.  One group of G lanes per row, plain
//                                 read-modify-write adds: every target row must belong to one row r (the sampler's
//                                 layout, num_neighbors consecutive neighbour rows per node), so no float atomics and
//                                 the result does not depend on the schedule.
//   b200_sage_walk_pairs          pairs_from_random_walk (libreco/sampling/random_walks.py:21-41) for a batch of start
//                                 items drawn on the device.  Three launches: per (start, slot) pair counts, a
//                                 one-block exclusive scan, and the fill that replays the same draws into the offsets.
//   b200_sage_i2i_negatives       negatives_from_random with items (libreco/sampling/negatives.py:17-31): uniform, a
//                                 draw equal to the sample's item or its positive is drawn again, at most `tolerance`
//                                 times.
//
// Draws are Philox4x32-10 keyed by (seed lo, seed hi ^ step hi) with counter (index, sub-index, step lo, tag):
//   start item i:                   (i, 0xFFFFFFFF, step, TAG_START), bounded over n_items of words x, y;
//   one-walk t of walk w of start i: (i, w * walk_length + t, step, TAG_WALK), words x, y pick the consumer, z, w the
//                                    consumer's item (the one_walk of csrc/sage.cu);
//   negative k, attempt a:          (k, a, step, TAG_NEG) with k = j * num_neg + t.
#include "common.cuh"
#include "philox.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace sage_train {

constexpr int THREADS = 256;
constexpr int MAX_D = 128;
constexpr int MAX_WALKS = 1024;
constexpr int MAX_WALK_LEN = 1024;
constexpr int SCAN_THREADS = 1024;
enum : uint32_t { TAG_START = 0x5a6e0001u, TAG_WALK = 0x5a6e0002u, TAG_NEG = 0x5a6e0003u };

__device__ __forceinline__ U4 keyed(uint32_t a, uint32_t b, uint32_t tag, uint64_t seed, uint64_t step) {
  U4 c;
  c.x = a; c.y = b; c.z = (uint32_t)step; c.w = tag;
  return philox4x32_10(c, (uint32_t)seed, (uint32_t)(seed >> 32) ^ (uint32_t)(step >> 32));
}

// ---- aggregation backward ------------------------------------------------------------------------------------------
template <int G, int PER>
__global__ void __launch_bounds__(THREADS) aggregate_backward_kernel(
    const float* __restrict__ dout, int64_t ldo, const int32_t* __restrict__ self_idx, int64_t n,
    float* __restrict__ dS, int64_t lds, const int32_t* __restrict__ nb_idx, const int64_t* __restrict__ nb_offsets,
    const int32_t* __restrict__ nb_lens, int stride, int d, float* __restrict__ dN, int64_t ldn) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
  const int t = threadIdx.x % G;
  if (r >= n) return;
  const float* g = dout + r * ldo;
  const int64_t sr = self_idx ? (int64_t)self_idx[r] : r;
  if (sr >= 0) {
    float* s = dS + sr * lds;
    for (int k = t; k < d; k += G) s[k] += g[k];
  }
  int64_t start, len;
  if (nb_offsets) { start = nb_offsets[r]; len = nb_lens ? (int64_t)nb_lens[r] : nb_offsets[r + 1] - start; }
  else { start = r * stride; len = nb_lens ? (int64_t)nb_lens[r] : stride; }
  if (len <= 0) return;
  const float inv_len = 1.f / (float)len;       // the forward's factor: mean = sum * (1 / len)
  float gm[PER];
#pragma unroll
  for (int c = 0; c < PER; ++c) {
    const int k = t + c * G;
    gm[c] = k < d ? g[d + k] * inv_len : 0.f;
  }
  for (int64_t j = start; j < start + len; ++j) {
    const int64_t nr = nb_idx ? (int64_t)nb_idx[j] : j;
    if (nr < 0) continue;
    float* row = dN + nr * ldn;
#pragma unroll
    for (int c = 0; c < PER; ++c) {
      const int k = t + c * G;
      if (k < d) row[k] += gm[c];
    }
  }
}

template <int G, int PER>
int launch_aggregate_backward(const float* dout, int64_t ldo, const int32_t* self_idx, int64_t n, float* dS,
                              int64_t lds, const int32_t* nb_idx, const int64_t* nb_offsets, const int32_t* nb_lens,
                              int stride, int d, float* dN, int64_t ldn, cudaStream_t st) {
  aggregate_backward_kernel<G, PER><<<(unsigned)ceil_div64(n * G, THREADS), THREADS, 0, st>>>(
      dout, ldo, self_idx, n, dS, lds, nb_idx, nb_offsets, nb_lens, stride, d, dN, ldn);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

// ---- random-walk pairs ---------------------------------------------------------------------------------------------
struct Graph {
  const int64_t* item_ptr; const int32_t* item_users;
  const int64_t* user_ptr; const int32_t* user_items;
};

__device__ __forceinline__ int32_t one_walk(const Graph& g, int32_t v, const U4& r) {
  const int64_t i0 = g.item_ptr[v];
  const int32_t u = g.item_users[i0 + bounded(r.x, r.y, g.item_ptr[v + 1] - i0)];
  const int64_t u0 = g.user_ptr[u];
  return g.user_items[u0 + bounded(r.z, r.w, g.user_ptr[u + 1] - u0)];
}

__device__ __forceinline__ bool has_no_neighbor(const Graph& g, int32_t v) {
  for (int64_t e = g.item_ptr[v]; e < g.item_ptr[v + 1]; ++e) {
    const int32_t u = g.item_users[e];
    if (g.user_ptr[u + 1] - g.user_ptr[u] > 1) return false;
  }
  return true;
}

// slot 0 of start i: the (v, v) pair of an item without neighbours; slot 1 + w: walk w.  fill == false: counts[q] =
// the pairs of slot q; fill == true: the pairs written from offsets[q].
template <bool FILL>
__global__ void __launch_bounds__(THREADS) walk_pairs_kernel(Graph g, int64_t n_items, int64_t n_starts,
                                                             int num_walks, int walk_len, int focus_start,
                                                             uint64_t seed, uint64_t step, int32_t* __restrict__ starts,
                                                             int64_t* __restrict__ counts,
                                                             const int64_t* __restrict__ offsets,
                                                             int32_t* __restrict__ items,
                                                             int32_t* __restrict__ items_pos) {
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int slots = num_walks + 1;
  if (q >= n_starts * slots) return;
  const int64_t i = q / slots;
  const int slot = (int)(q % slots);
  int32_t v;
  if (FILL) {
    v = starts[i];
  } else {
    const U4 r = keyed((uint32_t)i, 0xFFFFFFFFu, TAG_START, seed, step);
    v = (int32_t)bounded(r.x, r.y, n_items);
    if (slot == 0) starts[i] = v;
  }
  int64_t o = FILL ? offsets[q] : 0;
  if (slot == 0) {
    const bool lonely = has_no_neighbor(g, v);
    if (FILL) { if (lonely) { items[o] = v; items_pos[o] = v; } }
    else counts[q] = lonely ? 1 : 0;
    return;
  }
  const int w = slot - 1;
  int32_t cur = v;
  int64_t c = 0;
  for (int t = 0; t < walk_len; ++t) {
    const int32_t nxt = one_walk(g, cur, keyed((uint32_t)i, (uint32_t)(w * walk_len + t), TAG_WALK, seed, step));
    const int32_t from = focus_start ? v : cur;
    if (nxt != from) {
      if (FILL) { items[o + c] = from; items_pos[o + c] = nxt; }
      ++c;
    }
    cur = nxt;
  }
  if (!FILL) counts[q] = c;
}

// exclusive prefix sum of counts[0..n) into offsets[0..n], offsets[n] = the total; one block, a serial chunk per thread
__global__ void __launch_bounds__(SCAN_THREADS) exclusive_scan_kernel(const int64_t* __restrict__ counts, int64_t n,
                                                                      int64_t* __restrict__ offsets) {
  __shared__ int64_t part[SCAN_THREADS];
  const int tid = threadIdx.x;
  const int64_t chunk = (n + SCAN_THREADS - 1) / SCAN_THREADS;
  const int64_t b = tid * chunk, e = b + chunk < n ? b + chunk : n;
  int64_t s = 0;
  for (int64_t k = b; k < e; ++k) s += counts[k];
  part[tid] = s;
  __syncthreads();
  for (int off = 1; off < SCAN_THREADS; off <<= 1) {      // Hillis-Steele inclusive scan of the chunk sums
    const int64_t x = tid >= off ? part[tid - off] : 0;
    __syncthreads();
    part[tid] += x;
    __syncthreads();
  }
  int64_t run = part[tid] - s;
  for (int64_t k = b; k < e; ++k) { offsets[k] = run; run += counts[k]; }
  if (tid == SCAN_THREADS - 1) offsets[n] = part[tid];
}

// ---- i2i negatives -------------------------------------------------------------------------------------------------
__global__ void i2i_negatives_kernel(const int32_t* __restrict__ items, const int32_t* __restrict__ items_pos,
                                     int64_t n, int num_neg, int64_t n_items, int tolerance, uint64_t seed,
                                     uint64_t step, int32_t* __restrict__ out) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n * num_neg) return;
  const int64_t j = k / num_neg;
  const int32_t a = items[j], p = items_pos[j];
  uint32_t attempt = 0;
  U4 r = keyed((uint32_t)k, attempt++, TAG_NEG, seed, step);
  int32_t x = (int32_t)bounded(r.x, r.y, n_items);
  for (int t = 0; t < tolerance && (x == a || x == p); ++t) {
    r = keyed((uint32_t)k, attempt++, TAG_NEG, seed, step);
    x = (int32_t)bounded(r.x, r.y, n_items);
  }
  out[k] = x;
}

}  // namespace sage_train
}  // namespace b200

using namespace b200;
using namespace b200::sage_train;

extern "C" int b200_sage_aggregate_backward(const float* dout, int64_t ldo, const int32_t* self_idx, int64_t n_rows,
                                            float* dS, int64_t lds, const int32_t* nb_idx,
                                            const int64_t* nb_offsets, const int32_t* nb_lens, int32_t nb_stride,
                                            int32_t d, float* dN, int64_t ldn, void* stream) {
  B200_REQUIRE(dout && dS && dN, "b200_sage_aggregate_backward: null pointer");
  B200_REQUIRE(d >= 1 && d <= MAX_D, "b200_sage_aggregate_backward: d %d outside [1, %d]", d, MAX_D);
  B200_REQUIRE(n_rows >= 0 && lds >= d && ldn >= d && ldo >= 2 * d, "b200_sage_aggregate_backward: bad sizes");
  B200_REQUIRE(nb_offsets || nb_stride >= 0, "b200_sage_aggregate_backward: give nb_offsets or nb_stride >= 0");
  if (n_rows == 0) return 0;
  const cudaStream_t st = (cudaStream_t)stream;
#define B200_SAGE_AGG_BW(G, PER) \
  launch_aggregate_backward<G, PER>(dout, ldo, self_idx, n_rows, dS, lds, nb_idx, nb_offsets, nb_lens, nb_stride, d, \
                                    dN, ldn, st)
  if (d <= 8) return B200_SAGE_AGG_BW(8, 1);
  if (d <= 16) return B200_SAGE_AGG_BW(16, 1);
  if (d <= 32) return B200_SAGE_AGG_BW(32, 1);
  if (d <= 64) return B200_SAGE_AGG_BW(32, 2);
  return B200_SAGE_AGG_BW(32, 4);
#undef B200_SAGE_AGG_BW
}

extern "C" int b200_sage_walk_pairs(const int64_t* item_ptr, const int32_t* item_users, const int64_t* user_ptr,
                                    const int32_t* user_items, int64_t n_items, int64_t n_starts, int32_t num_walks,
                                    int32_t walk_length, int32_t focus_start, uint64_t seed, uint64_t step,
                                    int32_t* starts, int64_t* counts, int64_t* offsets, int32_t* items,
                                    int32_t* items_pos, void* stream) {
  B200_REQUIRE(item_ptr && item_users && user_ptr && user_items && starts,
               "b200_sage_walk_pairs: null pointer");
  B200_REQUIRE(n_items >= 1 && n_items < ((int64_t)1 << 31) && n_starts >= 0 && n_starts < ((int64_t)1 << 31),
               "b200_sage_walk_pairs: bad n_items / n_starts");
  B200_REQUIRE(num_walks >= 1 && num_walks <= MAX_WALKS && walk_length >= 1 && walk_length <= MAX_WALK_LEN,
               "b200_sage_walk_pairs: num_walks / walk_length outside [1, %d] / [1, %d]", MAX_WALKS, MAX_WALK_LEN);
  const bool fill = items != nullptr;
  B200_REQUIRE(fill ? (items_pos && offsets) : (counts && offsets),
               "b200_sage_walk_pairs: give counts + offsets (count pass) or offsets + items + items_pos (fill pass)");
  if (n_starts == 0) {
    if (!fill) B200_CUDA_OK(cudaMemsetAsync(offsets, 0, sizeof(int64_t), (cudaStream_t)stream));
    return 0;
  }
  const cudaStream_t st = (cudaStream_t)stream;
  Graph g{item_ptr, item_users, user_ptr, user_items};
  const int64_t slots = n_starts * (num_walks + 1);
  const unsigned grid = (unsigned)ceil_div64(slots, THREADS);
  if (fill) {
    walk_pairs_kernel<true><<<grid, THREADS, 0, st>>>(g, n_items, n_starts, num_walks, walk_length, focus_start,
                                                      seed, step, starts, nullptr, offsets, items, items_pos);
    count_launch();
  } else {
    walk_pairs_kernel<false><<<grid, THREADS, 0, st>>>(g, n_items, n_starts, num_walks, walk_length, focus_start,
                                                       seed, step, starts, counts, nullptr, nullptr, nullptr);
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    exclusive_scan_kernel<<<1, SCAN_THREADS, 0, st>>>(counts, slots, offsets);
    count_launch();
  }
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_sage_i2i_negatives(const int32_t* items, const int32_t* items_pos, int64_t n, int32_t num_neg,
                                       int64_t n_items, int32_t tolerance, uint64_t seed, uint64_t step, int32_t* out,
                                       void* stream) {
  B200_REQUIRE(items && items_pos && out, "b200_sage_i2i_negatives: null pointer");
  B200_REQUIRE(num_neg >= 1 && n_items >= 2 && n_items < ((int64_t)1 << 31) && n >= 0 && tolerance >= 0,
               "b200_sage_i2i_negatives: bad num_neg / n_items / n / tolerance");
  if (n == 0) return 0;
  i2i_negatives_kernel<<<(unsigned)ceil_div64(n * num_neg, THREADS), THREADS, 0, (cudaStream_t)stream>>>(
      items, items_pos, n, num_neg, n_items, tolerance, seed, step, out);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
