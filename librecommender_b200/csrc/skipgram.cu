// Skip-gram training — what gensim's Word2Vec(sg=1) does for libreco's Item2Vec and DeepWalk
// (libreco/bases/gensim_base.py:65-70, algorithms/item2vec.py:70-83, algorithms/deepwalk.py:96-126), on the device.
//
// A corpus is a sentence CSR: indptr int64 [S+1], tokens int32 (item ids), at most 10 000 tokens per sentence.
// Per epoch (pass p, counted from 1; pass 0 is DeepWalk's vocabulary walk set):
//   b200_skipgram_subsample  keep raw token t with probability min(1, p_w) (the caller's per-item threshold
//                            keep_thr[w] = round(min(1, p_w) 2^32), one Philox draw keyed by (seed, p, t)), and
//                            compact each sentence's kept tokens in place: slot q = indptr[s] + k holds the k-th
//                            kept token of sentence s; kept_sent[q] = s, or -1 past kept_len[s].
//   b200_skipgram_epoch      for every kept centre i of every sentence, in order: b_i = bounded(Philox(seed, p, q_i),
//                            window); contexts j in [i - window + b_i, i + window - b_i], j != i, j inner.  Pair
//                            (i, j) with h = syn0[w_j]: hierarchical softmax over w_i's Huffman path (when hs), then
//                            syn0[w_j] += work; negative sampling (target w_i label 1, then `negative` draws from
//                            the unigram^0.75 table, a draw equal to w_i skipped) then syn0[w_j] += work.  A target
//                            with |f| >= 6 is skipped; g = (label - sigmoid(f)) alpha (HS: label = 1 - code); the
//                            target row gets g h at once, work += g row.  alpha decays linearly per sentence from
//                            its raw offset.  sigmoid is the exact logistic.
//   b200_item_walks          DeepWalk's corpus: n_walks rounds, one walk from every item per round; each step picks
//                            uniformly among the node's out-edges (a CSR kept with multiplicity), one Philox draw
//                            keyed by (seed, p, walk, step); a walk stops at walk_length tokens or at a sink.
//
// Layout (as csrc/bpr.cu): one group of G lanes per centre token, G the smallest power of two giving at most 4
// elements per lane; the dot product is a shuffle tree inside the group.  Groups walk the compacted slots in order
// with a grid stride, so about max_inflight consecutive centres are in flight.  Tables are read with plain loads
// (never the read-only path: other groups' adds must be visible) and updated by red.global.add.f32 of deltas.
// max_inflight = 1 is the serial schedule: every element is read and written by one lane, so program order puts
// every read after the previous update — deterministic, and the sequential semantics.  fp32 SIMT.
#include <math.h>

#include "common.cuh"
#include "philox.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace skipgram {

constexpr int MAX_EMBED = 128;
constexpr int MAX_WINDOW = 4096;
constexpr int MAX_NEGATIVE = 16;
constexpr int64_t MAX_SENTENCE = 10000;
constexpr int THREADS = 256;
constexpr float MAX_EXP = 6.f;
// the default schedule keeps this many warps' worth of groups per SM in flight, and at most 1/DEFAULT_CORPUS_SHARE of the
// epoch's slots (DESIGN.md §4, "Skip-gram training").  Every DeepWalk pair updates the top rows of the Huffman tree, so
// on a small corpus a large share in flight makes those updates stale: on C1 (64 k walk tokens) recall@10 fell from
// 0.0242 at 64 centres in flight to 0.0199 at 16 896
constexpr int DEFAULT_WARPS_PER_SM = 16;
constexpr int64_t DEFAULT_CORPUS_SHARE = 256;

// Philox counter word 2: stream tag in the top bits, a sub-index below
enum : uint32_t { TAG_KEEP = 0u, TAG_WINDOW = 1u, TAG_NEG = 2u, TAG_WALK = 3u };

__device__ __forceinline__ U4 draw(uint64_t pos, uint32_t tag, uint32_t sub, uint32_t ctr_w, uint32_t k0,
                                   uint32_t k1) {
  U4 c;
  c.x = (uint32_t)pos; c.y = (uint32_t)(pos >> 32); c.z = (tag << 28) | sub; c.w = ctr_w;
  return philox4x32_10(c, k0, k1);
}

__host__ __device__ inline int group_lanes(int d) {
  int g = 1;
  while (g < 32 && g * 4 < d) g <<= 1;
  return g;
}

__device__ __forceinline__ void red_add(float* p, float v) {
  asm volatile("red.global.add.f32 [%0], %1;" ::"l"(p), "f"(v) : "memory");
}

// ---- subsample + per-sentence compaction: one warp per sentence -------------------------------------------------
__global__ void __launch_bounds__(THREADS) subsample_kernel(
    const int64_t* __restrict__ indptr, const int32_t* __restrict__ tokens, int64_t n_sent,
    const uint64_t* __restrict__ keep_thr, uint32_t ctr_w, uint32_t k0, uint32_t k1, int32_t* kept_tokens,
    int32_t* kept_sent, int32_t* kept_len, uint8_t* keep_out) {
  const int64_t s = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (s >= n_sent) return;
  const int64_t beg = indptr[s], end = indptr[s + 1];
  int64_t out = beg;
  for (int64_t base = beg; base < end; base += 32) {
    const int64_t t = base + lane;
    bool keep = false;
    int32_t w = 0;
    if (t < end) {
      w = tokens[t];
      const U4 r = draw((uint64_t)t, TAG_KEEP, 0u, ctr_w, k0, k1);
      keep = (uint64_t)r.x < keep_thr[w];
      if (keep_out) keep_out[t] = keep ? 1 : 0;
    }
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const int64_t q = out + __popc(m & ((1u << lane) - 1u));
      kept_tokens[q] = w;
      kept_sent[q] = (int32_t)s;
    }
    out += __popc(m);
  }
  for (int64_t q = out + lane; q < end; q += 32) kept_sent[q] = -1;
  if (lane == 0) kept_len[s] = (int32_t)(out - beg);
}

// ---- the epoch -------------------------------------------------------------------------------------------------
struct Args {
  const int64_t* indptr;
  const int32_t* kept_tokens;
  const int32_t* kept_sent;
  const int32_t* kept_len;
  int64_t n_slots;
  float* syn0;
  float* syn1neg;
  float* syn1;
  int d;
  const int64_t* hs_ptr;
  const int32_t* hs_points;
  const int8_t* hs_codes;
  const uint32_t* neg_cum;
  const int32_t* neg_items;
  const int32_t* neg_guide;
  int64_t vocab;
  uint32_t cum_last;
  int64_t guide_step;
  int window, negative;
  double alpha0, min_alpha, words_before, inv_words_total;
  uint32_t ctr_w, k0, k1;
  int32_t* window_out;
  int32_t* neg_out;
  int64_t groups;
};

__device__ __forceinline__ float sigmoid(float f) { return 1.f / (1.f + expf(-f)); }

// bisect_left(cum, r) over the vocabulary, started from the guide bucket of r; returns the item id
__device__ __forceinline__ int32_t negative_item(const Args& a, uint64_t q, int off, int dd) {
  const U4 r4 = draw(q, TAG_NEG, ((uint32_t)(off + a.window) << 4) | (uint32_t)dd, a.ctr_w, a.k0, a.k1);
  const uint32_t r = (uint32_t)bounded(r4.x, r4.y, (int64_t)a.cum_last);
  const int64_t b = (int64_t)r / a.guide_step;
  int64_t lo = a.neg_guide[b], hi = a.neg_guide[b + 1];
  while (lo < hi) {
    const int64_t mid = (lo + hi) >> 1;
    if (a.neg_cum[mid] < r) lo = mid + 1; else hi = mid;
  }
  return a.neg_items[lo];
}

template <int G, int E, bool HS>
__global__ void __launch_bounds__(THREADS) epoch_kernel(const Args a) {
  const int64_t gid = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) / G;
  if (gid >= a.groups) return;
  const int lane = threadIdx.x & 31;
  const int sub = lane & (G - 1);
  const unsigned mask = G == 32 ? 0xffffffffu : (((1u << G) - 1u) << (lane & ~(G - 1)));
  const int d = a.d;
  for (int64_t q = gid; q < a.n_slots; q += a.groups) {
    const int32_t s = a.kept_sent[q];
    if (s < 0) continue;
    const int64_t beg = a.indptr[s];
    const int n = a.kept_len[s];
    const int i = (int)(q - beg);
    const U4 rw = draw((uint64_t)q, TAG_WINDOW, 0u, a.ctr_w, a.k0, a.k1);
    const int b = (int)bounded(rw.x, rw.y, (int64_t)a.window);
    if (a.window_out && sub == 0) a.window_out[q] = b;
    const double prog = fmin(1.0, (a.words_before + (double)beg) * a.inv_words_total);
    const float alpha = (float)(a.alpha0 - (a.alpha0 - a.min_alpha) * prog);
    const int32_t wi = a.kept_tokens[q];
    const int reach = a.window - b;
    const int jlo = max(0, i - reach), jhi = min(n - 1, i + reach);
    for (int j = jlo; j <= jhi; ++j) {
      if (j == i) continue;
      const int32_t wj = a.kept_tokens[beg + j];
      float* h0 = a.syn0 + (int64_t)wj * d;
      float h[E], work[E];
#pragma unroll
      for (int k = 0; k < E; ++k) {
        const int c = sub + G * k;
        h[k] = c < d ? h0[c] : 0.f;
        work[k] = 0.f;
      }
      auto train = [&](float* row, float label_or_code, bool is_hs) {
        float rr[E], part = 0.f;
#pragma unroll
        for (int k = 0; k < E; ++k) {
          const int c = sub + G * k;
          rr[k] = c < d ? row[c] : 0.f;
          part += h[k] * rr[k];
        }
#pragma unroll
        for (int o = G / 2; o > 0; o >>= 1) part += __shfl_xor_sync(mask, part, o, G);
        if (part <= -MAX_EXP || part >= MAX_EXP) return;
        const float label = is_hs ? 1.f - label_or_code : label_or_code;
        const float g = (label - sigmoid(part)) * alpha;
#pragma unroll
        for (int k = 0; k < E; ++k) {
          const int c = sub + G * k;
          work[k] += g * rr[k];
          if (c < d) red_add(row + c, g * h[k]);
        }
      };
      if (HS) {
        const int64_t pb = a.hs_ptr[wi], pe = a.hs_ptr[wi + 1];
        for (int64_t p = pb; p < pe; ++p)
          train(a.syn1 + (int64_t)a.hs_points[p] * d, (float)a.hs_codes[p], true);
#pragma unroll
        for (int k = 0; k < E; ++k) {
          const int c = sub + G * k;
          if (c < d) red_add(h0 + c, work[k]);
          h[k] += work[k];
          work[k] = 0.f;
        }
      }
      for (int dd = 0; dd <= a.negative; ++dd) {
        int32_t target = wi;
        if (dd > 0) {
          target = negative_item(a, (uint64_t)q, j - i, dd - 1);
          if (a.neg_out && sub == 0)
            a.neg_out[(q * (2 * a.window + 1) + (j - i + a.window)) * a.negative + (dd - 1)] = target;
          if (target == wi) continue;
        }
        train(a.syn1neg + (int64_t)target * d, dd == 0 ? 1.f : 0.f, false);
      }
#pragma unroll
      for (int k = 0; k < E; ++k) {
        const int c = sub + G * k;
        if (c < d) red_add(h0 + c, work[k]);
      }
    }
  }
}

template <bool HS>
static const void* kernel_for(int d) {
  switch (group_lanes(d)) {
    case 1: return (const void*)epoch_kernel<1, 4, HS>;
    case 2: return (const void*)epoch_kernel<2, 4, HS>;
    case 4: return (const void*)epoch_kernel<4, 4, HS>;
    case 8: return (const void*)epoch_kernel<8, 4, HS>;
    case 16: return (const void*)epoch_kernel<16, 4, HS>;
    default: return (const void*)epoch_kernel<32, 4, HS>;
  }
}

// ---- item walks: one thread per walk ---------------------------------------------------------------------------
__global__ void __launch_bounds__(THREADS) walk_kernel(
    const int64_t* __restrict__ g_indptr, const int32_t* __restrict__ g_dst, int64_t n_items, int64_t n_walks_total,
    int walk_length, uint32_t ctr_w, uint32_t k0, uint32_t k1, int64_t* lengths, const int64_t* __restrict__ indptr,
    int32_t* tokens) {
  const int64_t w = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (w >= n_walks_total) return;
  int32_t cur = (int32_t)(w % n_items);
  int32_t* out = tokens ? tokens + indptr[w] : nullptr;
  if (out) out[0] = cur;
  int len = 1;
  for (; len < walk_length; ++len) {
    const int64_t beg = g_indptr[cur], deg = g_indptr[cur + 1] - beg;
    if (deg == 0) break;
    const U4 r = draw((uint64_t)w, TAG_WALK, (uint32_t)len, ctr_w, k0, k1);
    cur = g_dst[beg + bounded(r.x, r.y, deg)];
    if (out) out[len] = cur;
  }
  if (lengths) lengths[w] = len;
}

inline void keys(uint64_t seed, int64_t pass, uint32_t* ctr_w, uint32_t* k0, uint32_t* k1) {
  const uint64_t p = (uint64_t)pass;
  *ctr_w = (uint32_t)p; *k0 = (uint32_t)seed; *k1 = (uint32_t)(seed >> 32) ^ (uint32_t)(p >> 32);
}

}  // namespace skipgram
}  // namespace b200

using namespace b200;
using namespace b200::skipgram;

extern "C" int64_t b200_skipgram_default_inflight(int32_t d) {
  if (d < 1 || d > MAX_EMBED) return 0;
  const int sms = num_sms();
  return (int64_t)(sms > 0 ? sms : 1) * DEFAULT_WARPS_PER_SM * (32 / group_lanes(d));
}

extern "C" int b200_skipgram_subsample(const int64_t* indptr, const int32_t* tokens, int64_t n_sentences,
                                       int64_t n_items, const uint64_t* keep_thr, uint64_t seed, int64_t pass,
                                       int32_t* kept_tokens, int32_t* kept_sent, int32_t* kept_len,
                                       uint8_t* keep_out, void* stream) {
  B200_REQUIRE(n_sentences >= 0 && n_items >= 1 && n_items < (1ll << 31) && n_sentences < (1ll << 31),
               "b200_skipgram_subsample: bad sizes");
  B200_REQUIRE(indptr && tokens && keep_thr && kept_tokens && kept_sent && kept_len,
               "b200_skipgram_subsample: null pointer");
  if (n_sentences == 0) return 0;
  uint32_t cw, k0, k1;
  keys(seed, pass, &cw, &k0, &k1);
  const int64_t threads = n_sentences * 32;
  subsample_kernel<<<(unsigned)ceil_div64(threads, THREADS), THREADS, 0, (cudaStream_t)stream>>>(
      indptr, tokens, n_sentences, keep_thr, cw, k0, k1, kept_tokens, kept_sent, kept_len, keep_out);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_skipgram_epoch(const int64_t* indptr, int64_t n_sentences, const int32_t* kept_tokens,
                                   const int32_t* kept_sent, const int32_t* kept_len, int64_t n_tokens, int64_t n_items, float* syn0,
                                   float* syn1neg, float* syn1, int32_t d, int32_t hs, const int64_t* hs_ptr,
                                   const int32_t* hs_points, const int8_t* hs_codes, const uint32_t* neg_cum,
                                   const int32_t* neg_items, int64_t vocab_size, uint32_t cum_last,
                                   const int32_t* neg_guide, int64_t guide_buckets, int32_t window, int32_t negative, double alpha0,
                                   double min_alpha, double words_before, double words_total, uint64_t seed,
                                   int64_t pass, int32_t* window_out, int32_t* neg_out, int64_t max_inflight,
                                   void* stream) {
  B200_REQUIRE(d >= 1 && d <= MAX_EMBED, "b200_skipgram_epoch: embed size %d outside [1, %d]", d, MAX_EMBED);
  B200_REQUIRE(window >= 1 && window <= MAX_WINDOW, "b200_skipgram_epoch: window %d outside [1, %d]", window,
               MAX_WINDOW);
  B200_REQUIRE(negative >= 1 && negative <= MAX_NEGATIVE, "b200_skipgram_epoch: negative %d outside [1, %d]",
               negative, MAX_NEGATIVE);
  B200_REQUIRE(hs == 0 || hs == 1, "b200_skipgram_epoch: hs must be 0 or 1, got %d", hs);
  B200_REQUIRE(n_sentences >= 0 && n_sentences < (1ll << 31) && n_items >= 1 && n_items < (1ll << 31) &&
               n_tokens >= 0 && vocab_size >= 1 && vocab_size <= n_items && cum_last >= 1 &&
               guide_buckets >= 1 && max_inflight >= 0 && words_total > 0.0, "b200_skipgram_epoch: bad sizes");
  B200_REQUIRE(indptr && kept_tokens && kept_sent && kept_len && syn0 && syn1neg && neg_cum && neg_items &&
               neg_guide, "b200_skipgram_epoch: null pointer");
  B200_REQUIRE(!hs || (syn1 && hs_ptr && hs_points && hs_codes),
               "b200_skipgram_epoch: hierarchical softmax needs syn1, hs_ptr, hs_points and hs_codes");
  if (n_sentences == 0 || n_tokens == 0) return 0;
  Args a;
  a.indptr = indptr; a.kept_tokens = kept_tokens; a.kept_sent = kept_sent; a.kept_len = kept_len;
  a.n_slots = n_tokens; a.syn0 = syn0; a.syn1neg = syn1neg; a.syn1 = syn1; a.d = d;
  a.hs_ptr = hs_ptr; a.hs_points = hs_points; a.hs_codes = hs_codes;
  a.neg_cum = neg_cum; a.neg_items = neg_items; a.neg_guide = neg_guide; a.vocab = vocab_size;
  a.cum_last = cum_last; a.guide_step = ((int64_t)cum_last + guide_buckets - 1) / guide_buckets;
  a.window = window; a.negative = negative;
  a.alpha0 = alpha0; a.min_alpha = min_alpha; a.words_before = words_before; a.inv_words_total = 1.0 / words_total;
  keys(seed, pass, &a.ctr_w, &a.k0, &a.k1);
  a.window_out = window_out; a.neg_out = neg_out;
  const int G = group_lanes(d);
  int64_t groups = max_inflight;
  if (groups == 0) {
    groups = b200_skipgram_default_inflight(d);
    const int64_t share = n_tokens / DEFAULT_CORPUS_SHARE;
    if (groups > share) groups = share > 0 ? share : 1;
  }
  if (groups > n_tokens) groups = n_tokens;
  a.groups = groups;
  const int64_t threads = groups * G;
  const int block = (int)(threads < THREADS ? threads : THREADS);
  const void* fn = hs ? kernel_for<true>(d) : kernel_for<false>(d);
  void* params[] = {&a};
  B200_CUDA_OK(cudaLaunchKernel(fn, dim3((unsigned)ceil_div64(threads, block)), dim3(block), params, 0,
                                (cudaStream_t)stream));
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_item_walks(const int64_t* graph_indptr, const int32_t* graph_dst, int64_t n_items,
                               int32_t n_walks, int32_t walk_length, uint64_t seed, int64_t pass, int64_t* lengths,
                               const int64_t* indptr, int32_t* tokens, void* stream) {
  B200_REQUIRE(n_items >= 1 && n_items < (1ll << 31) && n_walks >= 0 && walk_length >= 1 &&
               walk_length <= MAX_SENTENCE && (int64_t)n_walks * n_items < (1ll << 31),
               "b200_item_walks: bad sizes");
  B200_REQUIRE(graph_indptr && graph_dst, "b200_item_walks: null pointer");
  B200_REQUIRE((lengths != nullptr) != (tokens != nullptr), "b200_item_walks: pass exactly one of lengths, tokens");
  B200_REQUIRE(!tokens || indptr, "b200_item_walks: tokens needs indptr");
  const int64_t total = (int64_t)n_walks * n_items;
  if (total == 0) return 0;
  uint32_t cw, k0, k1;
  keys(seed, pass, &cw, &k0, &k1);
  walk_kernel<<<(unsigned)ceil_div64(total, THREADS), THREADS, 0, (cudaStream_t)stream>>>(
      graph_indptr, graph_dst, n_items, total, walk_length, cw, k0, k1, lengths, indptr, tokens);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
