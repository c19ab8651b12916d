// GraphSage / PinSage inference — the neighbour sampling of libreco/graph/neighbor_walk.py:25-75 and
// libreco/sampling/random_walks.py:16-147 on the device, and the per-layer aggregation of the item encoders
// (libreco/algorithms/torch_modules/graphsage_module.py:106-151, pinsage_module.py:63-98).
//
// The graph is two CSRs kept as the reference's dicts hold them, list order and multiplicity included:
// item_consumed (users of each item) and user_consumed (items of each user).  A one-walk from item v draws a
// consumer u of v, then an item of u, each uniformly over list positions (random.choice), so repeated entries count.
//
// Sampling is per level.  The level-0 nodes are the caller's roots; level l+1 is the flattened [n_l, num_neighbors]
// output of level l, every slot sampled again, duplicates included (sample_graphsage / sample_pinsage).  A node is
// named by (root, level, path): path is its slot index inside its root's padded subtree, path' = path * nn + j.
// Every draw is Philox4x32-10 with key (seed lo, seed hi) and counter (root, path, level << 24 | draw, tag), so a
// node's neighbours do not depend on how roots are batched.  An index in [0, n) is bounded() of philox.cuh over a
// 64-bit word: words x, y pick the consumer, z, w the consumer's item.
//
//   b200_sage_neighbors     (bipartite_neighbors) num_neighbors slots per node.  Slot j has 12 keyed attempts
//                           a = 0..11 (counter path = the slot's own path, draw = a): attempt 0 if it is neither
//                           the node nor a neighbour taken so far; else the first of 1..5 that is neither; else the first of 6..10 that is not the
//                           node; else attempt 11.  One warp per node: the 12 attempts of a slot run on 12 lanes.
//   b200_pinsage_neighbors  (bipartite_neighbors_with_weights, items_pos = None) num_walks walks of up to walk_len
//                           one-walks; step s > 0 of walk w continues when the termination word of draw
//                           w * walk_len + s is >= cont_threshold = ceil(termination_prob 2^32) (random.random() >=
//                           termination_prob).  A node whose every consumer consumed one item only
//                           (has_no_neighbor) gives [node] with weight 1.  Visits equal to the node are removed
//                           unless all are, which gives [node].  The top num_neighbors distinct visits by count,
//                           ties by first visit in walk order (Counter.most_common), weight count / kept total.
//                           One warp per node, the visits in shared memory.
//   b200_sage_aggregate     out[r] = [S[self r], sum_j w_j N[nb j]] over row r's neighbour rows: the concat the
//                           w_linears read, mean (embedding_bag "mean") or per-neighbour weights ("sum").
//
// A padded slot past a node's length holds id -1 and weight 0; a node id < 0 (such a slot sampled again) gives
// length 0.  Envelope: num_neighbors 1..32, num_walks * walk_len 1..256, d 1..128.  fp32 SIMT.
#include "common.cuh"
#include "philox.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace sage {

constexpr int THREADS = 256;
constexpr int MAX_NEIGHBORS = 32;
constexpr int MAX_VISITS = 256;
constexpr int MAX_D = 128;
constexpr int ATTEMPTS = 12;     // 1 + tolerance 5 + tolerance 5 + 1 (random_walks.py:48-71)
enum : uint32_t { TAG_SAGE = 0u, TAG_PIN_STEP = 1u, TAG_PIN_STOP = 2u };

struct Graph {
  const int64_t* item_ptr; const int32_t* item_users;   // item_consumed
  const int64_t* user_ptr; const int32_t* user_items;   // user_consumed
};

__device__ __forceinline__ U4 draw(uint32_t root, uint32_t path, int level, uint32_t idx, uint32_t tag,
                                   uint32_t k0, uint32_t k1) {
  U4 c;
  c.x = root; c.y = path; c.z = ((uint32_t)level << 24) | idx; c.w = tag;
  return philox4x32_10(c, k0, k1);
}

// bipartite_one_walk: item v -> consumer of v -> item of that consumer
__device__ __forceinline__ int32_t one_walk(const Graph& g, int32_t v, const U4& r) {
  const int64_t i0 = g.item_ptr[v];
  const int32_t u = g.item_users[i0 + bounded(r.x, r.y, g.item_ptr[v + 1] - i0)];
  const int64_t u0 = g.user_ptr[u];
  return g.user_items[u0 + bounded(r.z, r.w, g.user_ptr[u + 1] - u0)];
}

// (root, path) of padded node r of a level whose nodes are `per_root` per root
__device__ __forceinline__ void node_key(const int32_t* roots, int64_t r, int64_t per_root, uint32_t* root,
                                         uint32_t* path) {
  *root = (uint32_t)roots[r / per_root];
  *path = (uint32_t)(r % per_root);
}

__global__ void __launch_bounds__(THREADS) sage_neighbors_kernel(Graph g, const int32_t* __restrict__ roots,
                                                                 const int32_t* __restrict__ nodes, int64_t n,
                                                                 int64_t per_root, int level, int nn, uint32_t k0,
                                                                 uint32_t k1, int32_t* __restrict__ out) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const int32_t v = nodes[r];
  if (v < 0) {
    if (lane < nn) out[r * nn + lane] = -1;
    return;
  }
  uint32_t root, path;
  node_key(roots, r, per_root, &root, &path);
  const uint32_t child0 = path * (uint32_t)nn;
  int32_t mine = -1;                       // lane j: the neighbour taken for slot j
  for (int j = 0; j < nn; ++j) {
    int32_t cand = -1;
    bool self = true, dup = false;
    if (lane < ATTEMPTS) {
      cand = one_walk(g, v, draw(root, child0 + j, level, (uint32_t)lane, TAG_SAGE, k0, k1));
      self = cand == v;
    }
    for (int s = 0; s < j; ++s) dup |= __shfl_sync(0xffffffffu, mine, s) == cand;
    const unsigned ok = __ballot_sync(0xffffffffu, lane < ATTEMPTS && !self && !dup);
    const unsigned not_self = __ballot_sync(0xffffffffu, lane < ATTEMPTS && !self);
    int pick;
    if (ok & 1u) pick = 0;
    else if (ok & 0x3Eu) pick = __ffs(ok & 0x3Eu) - 1;
    else if (not_self & 0x7C0u) pick = __ffs(not_self & 0x7C0u) - 1;
    else pick = ATTEMPTS - 1;
    const int32_t taken = __shfl_sync(0xffffffffu, cand, pick);
    if (lane == j) mine = taken;
  }
  if (lane < nn) out[r * nn + lane] = mine;
}

__global__ void __launch_bounds__(THREADS) pinsage_neighbors_kernel(
    Graph g, const int32_t* __restrict__ roots, const int32_t* __restrict__ nodes, int64_t n, int64_t per_root,
    int level, int nn, int num_walks, int walk_len, uint64_t cont_threshold, uint32_t k0, uint32_t k1,
    int32_t* __restrict__ out_ids, float* __restrict__ out_w, int32_t* __restrict__ out_len) {
  __shared__ int32_t visits_s[THREADS / 32][MAX_VISITS];
  __shared__ int32_t count_s[THREADS / 32][MAX_VISITS];
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  int32_t* visits = visits_s[threadIdx.x >> 5];
  int32_t* counts = count_s[threadIdx.x >> 5];
  const int32_t v = nodes[r];
  for (int j = lane; j < nn; j += 32) { out_ids[r * nn + j] = -1; out_w[r * nn + j] = 0.f; }
  if (v < 0) {
    if (lane == 0) out_len[r] = 0;
    return;
  }
  // has_no_neighbor: every consumer of v consumed one item only
  bool lonely = true;
  const int64_t e1 = g.item_ptr[v + 1];
  for (int64_t e0 = g.item_ptr[v]; e0 < e1 && lonely; e0 += 32) {
    const int64_t e = e0 + lane;
    bool multi = false;
    if (e < e1) { const int32_t u = g.item_users[e]; multi = g.user_ptr[u + 1] - g.user_ptr[u] > 1; }
    lonely = !__any_sync(0xffffffffu, multi);
  }
  if (lonely) {
    if (lane == 0) { out_ids[r * nn] = v; out_w[r * nn] = 1.f; out_len[r] = 1; }
    return;
  }
  uint32_t root, path;
  node_key(roots, r, per_root, &root, &path);
  const int V = num_walks * walk_len;
  for (int w = lane; w < num_walks; w += 32) {
    int32_t cur = v;
    bool alive = true;
    for (int s = 0; s < walk_len; ++s) {
      const uint32_t idx = (uint32_t)(w * walk_len + s);
      if (alive && s > 0) alive = draw(root, path, level, idx, TAG_PIN_STOP, k0, k1).x >= cont_threshold;
      if (alive) cur = one_walk(g, cur, draw(root, path, level, idx, TAG_PIN_STEP, k0, k1));
      visits[idx] = alive ? cur : -1;
    }
  }
  __syncwarp();
  // at the first visit of every distinct neighbour its count, elsewhere 0; the target node is not a neighbour
  constexpr int PER = MAX_VISITS / 32;
  int cnt[PER];
  int distinct = 0;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int p = lane + 32 * i;
    cnt[i] = 0;
    const int32_t x = p < V ? visits[p] : -1;
    if (x >= 0 && x != v) {
      int c = 0;
      for (int q = 0; q < V; ++q) {
        if (visits[q] == x) {
          if (q < p) { c = 0; break; }
          ++c;
        }
      }
      cnt[i] = c;
    }
    if (p < MAX_VISITS) counts[p] = cnt[i];
    distinct += cnt[i] > 0;
  }
  __syncwarp();
  for (int o = 16; o > 0; o >>= 1) distinct += __shfl_xor_sync(0xffffffffu, distinct, o);
  if (distinct == 0) {                     // every visit is the target (remove_target_node)
    if (lane == 0) { out_ids[r * nn] = v; out_w[r * nn] = 1.f; out_len[r] = 1; }
    return;
  }
  // rank of a distinct neighbour: count descending, then first visit ascending (a stable sort by count)
  int rank[PER];
  int total = 0;
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    const int p = lane + 32 * i, c = cnt[i];
    rank[i] = nn;
    if (c <= 0) continue;
    int k = 0;
    for (int q = 0; q < V && k < nn; ++q) {
      const int cq = counts[q];
      k += cq > c || (cq == c && q < p);
    }
    rank[i] = k;
    if (k < nn) total += c;
  }
  for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
#pragma unroll
  for (int i = 0; i < PER; ++i) {
    if (rank[i] >= nn) continue;
    out_ids[r * nn + rank[i]] = visits[lane + 32 * i];
    out_w[r * nn + rank[i]] = __fdiv_rn((float)cnt[i], (float)total);
  }
  if (lane == 0) out_len[r] = distinct < nn ? distinct : nn;
}

// G lanes per row (a power of two <= 32); lane t of a group covers columns t, t + G, ..., PER of them
template <int G, int PER>
__global__ void __launch_bounds__(THREADS) aggregate_kernel(
    const float* __restrict__ S, int64_t lds, const int32_t* __restrict__ self_idx, int64_t n,
    const float* __restrict__ N, int64_t ldn, const int32_t* __restrict__ nb_idx,
    const int64_t* __restrict__ nb_offsets, const int32_t* __restrict__ nb_lens, int stride,
    const float* __restrict__ nb_w, int d, float* __restrict__ out, int64_t ldo) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
  const int t = threadIdx.x % G;
  if (r >= n) return;
  const int64_t sr = self_idx ? (int64_t)self_idx[r] : r;
  float* o = out + r * ldo;
  for (int k = t; k < d; k += G) o[k] = sr >= 0 ? S[sr * lds + k] : 0.f;
  int64_t start, len;
  if (nb_offsets) { start = nb_offsets[r]; len = nb_lens ? (int64_t)nb_lens[r] : nb_offsets[r + 1] - start; }
  else { start = r * stride; len = nb_lens ? (int64_t)nb_lens[r] : stride; }
  float acc[PER];
#pragma unroll
  for (int c = 0; c < PER; ++c) acc[c] = 0.f;
  for (int64_t j = start; j < start + len; ++j) {
    const int64_t nr = nb_idx ? (int64_t)nb_idx[j] : j;
    const float w = nb_w ? nb_w[j] : 1.f;
    const float* row = N + nr * ldn;
#pragma unroll
    for (int c = 0; c < PER; ++c) {
      const int k = t + c * G;
      if (k < d) acc[c] = nb_w ? fmaf(w, row[k], acc[c]) : acc[c] + row[k];
    }
  }
  const float inv_len = len > 0 ? 1.f / (float)len : 0.f;
#pragma unroll
  for (int c = 0; c < PER; ++c) {
    const int k = t + c * G;
    if (k < d) o[d + k] = nb_w ? acc[c] : acc[c] * inv_len;
  }
}

template <int G, int PER>
int launch_aggregate(const float* S, int64_t lds, const int32_t* self_idx, int64_t n, const float* N, int64_t ldn,
                     const int32_t* nb_idx, const int64_t* nb_offsets, const int32_t* nb_lens, int stride,
                     const float* nb_w, int d, float* out, int64_t ldo, cudaStream_t st) {
  aggregate_kernel<G, PER><<<(unsigned)ceil_div64(n * G, THREADS), THREADS, 0, st>>>(
      S, lds, self_idx, n, N, ldn, nb_idx, nb_offsets, nb_lens, stride, nb_w, d, out, ldo);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

}  // namespace sage
}  // namespace b200

using namespace b200;
using namespace b200::sage;

static int check_graph(const int64_t* item_ptr, const int32_t* item_users, const int64_t* user_ptr,
                       const int32_t* user_items, const int32_t* roots, const int32_t* nodes, int64_t n,
                       int64_t per_root, int32_t level, int32_t nn, const char* fn) {
  B200_REQUIRE(item_ptr && item_users && user_ptr && user_items && roots && nodes, "%s: null pointer", fn);
  B200_REQUIRE(nn >= 1 && nn <= MAX_NEIGHBORS, "%s: num_neighbors %d outside [1, %d]", fn, nn, MAX_NEIGHBORS);
  B200_REQUIRE(level >= 0 && level < 8 && n >= 0 && per_root >= 1 && n % per_root == 0 && per_root <= (1 << 20),
               "%s: bad level / node count", fn);
  return 0;
}

extern "C" int b200_sage_neighbors(const int64_t* item_ptr, const int32_t* item_users, const int64_t* user_ptr,
                                   const int32_t* user_items, const int32_t* roots, const int32_t* nodes, int64_t n,
                                   int64_t per_root, int32_t level, int32_t num_neighbors, uint64_t seed,
                                   int32_t* out, void* stream) {
  const int rc = check_graph(item_ptr, item_users, user_ptr, user_items, roots, nodes, n, per_root, level,
                             num_neighbors, "b200_sage_neighbors");
  if (rc) return rc;
  B200_REQUIRE(out, "b200_sage_neighbors: null pointer");
  if (n == 0) return 0;
  Graph g{item_ptr, item_users, user_ptr, user_items};
  sage_neighbors_kernel<<<(unsigned)ceil_div64(n * 32, THREADS), THREADS, 0, (cudaStream_t)stream>>>(
      g, roots, nodes, n, per_root, level, num_neighbors, (uint32_t)seed, (uint32_t)(seed >> 32), out);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_pinsage_neighbors(const int64_t* item_ptr, const int32_t* item_users, const int64_t* user_ptr,
                                      const int32_t* user_items, const int32_t* roots, const int32_t* nodes,
                                      int64_t n, int64_t per_root, int32_t level, int32_t num_neighbors,
                                      int32_t num_walks, int32_t walk_len, uint64_t cont_threshold, uint64_t seed,
                                      int32_t* out_ids, float* out_weights, int32_t* out_lens, void* stream) {
  const int rc = check_graph(item_ptr, item_users, user_ptr, user_items, roots, nodes, n, per_root, level,
                             num_neighbors, "b200_pinsage_neighbors");
  if (rc) return rc;
  B200_REQUIRE(out_ids && out_weights && out_lens, "b200_pinsage_neighbors: null pointer");
  B200_REQUIRE(num_walks >= 1 && walk_len >= 1 && (int64_t)num_walks * walk_len <= MAX_VISITS,
               "b200_pinsage_neighbors: num_walks * walk_len outside [1, %d]", MAX_VISITS);
  B200_REQUIRE(cont_threshold <= (1ull << 32), "b200_pinsage_neighbors: cont_threshold above 2^32");
  if (n == 0) return 0;
  Graph g{item_ptr, item_users, user_ptr, user_items};
  pinsage_neighbors_kernel<<<(unsigned)ceil_div64(n * 32, THREADS), THREADS, 0, (cudaStream_t)stream>>>(
      g, roots, nodes, n, per_root, level, num_neighbors, num_walks, walk_len, cont_threshold, (uint32_t)seed,
      (uint32_t)(seed >> 32), out_ids, out_weights, out_lens);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_sage_aggregate(const float* S, int64_t lds, const int32_t* self_idx, int64_t n_rows,
                                   const float* N, int64_t ldn, const int32_t* nb_idx, const int64_t* nb_offsets,
                                   const int32_t* nb_lens, int32_t nb_stride, const float* nb_weights, int32_t d,
                                   float* out, int64_t ldo, void* stream) {
  B200_REQUIRE(S && N && out, "b200_sage_aggregate: null pointer");
  B200_REQUIRE(d >= 1 && d <= MAX_D, "b200_sage_aggregate: d %d outside [1, %d]", d, MAX_D);
  B200_REQUIRE(n_rows >= 0 && lds >= d && ldn >= d && ldo >= 2 * d, "b200_sage_aggregate: bad sizes");
  B200_REQUIRE(nb_offsets || nb_stride >= 0, "b200_sage_aggregate: give nb_offsets or nb_stride >= 0");
  if (n_rows == 0) return 0;
  const cudaStream_t st = (cudaStream_t)stream;
#define B200_SAGE_AGG(G, PER) \
  launch_aggregate<G, PER>(S, lds, self_idx, n_rows, N, ldn, nb_idx, nb_offsets, nb_lens, nb_stride, nb_weights, d, \
                           out, ldo, st)
  if (d <= 8) return B200_SAGE_AGG(8, 1);
  if (d <= 16) return B200_SAGE_AGG(16, 1);
  if (d <= 32) return B200_SAGE_AGG(32, 1);
  if (d <= 64) return B200_SAGE_AGG(32, 2);
  return B200_SAGE_AGG(32, 4);
#undef B200_SAGE_AGG
}
