// K5 — masked per-row top-K (stand-alone).
//
// Replaces libreco/recommendation/ranking.py:10-78 (rank_recommendations: filter_items,
// partition_select, argsort) for a materialised score matrix [B, N] in HBM.
//
// Algorithm: exact 3-pass MSD radix select (11+11+10 bits) on an order-preserving uint32 image
// of the fp32 score, multi-CTA per row (grid = chunks x rows, per-row global histogram, the last
// CTA of a row resolves the digit), then a count / collect pair that takes every element above
// the K-th key plus the lowest-id ties, and a per-row bitonic sort by (score desc, id asc).
// The key (float_to_key, common.cuh) makes -0.0 equal to +0.0, every NaN the largest value and the
// REMOVED pattern written by mask_consumed_kernel the smallest.
// HBM-bound integer/byte work: 5 coalesced sweeps over the row, no tensor cores.
#include "common.cuh"
#include "../../include/b200reco.h"

namespace b200 {

constexpr int kTopkThreads = 256;
constexpr int kTopkChunk = 8192;  // elements of one row handled by one CTA
constexpr int kBins = 2048;
constexpr int kMaxK = 4096;

struct RowState {
  uint32_t prefix;    // digits resolved so far (after pass 2: the K-th largest key)
  uint32_t k_rem;     // rank still to resolve inside the prefix (after pass 2: ties to take)
};

struct TopkWorkspace {
  uint32_t* hist;      // [B, kBins]
  uint32_t* done;      // [B]
  RowState* state;     // [B]
  uint32_t* chunk_gt;  // [B, C]  count, then exclusive offset
  uint32_t* chunk_eq;  // [B, C]
  uint32_t* sel_key;   // [B, K]
  int32_t* sel_id;     // [B, K]
};

static size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

static size_t carve(TopkWorkspace* w, char* base, int64_t B, int64_t C, int32_t K) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = base ? base + off : nullptr;
    off += align_up(bytes, 256);
    return p;
  };
  w->hist = (uint32_t*)take((size_t)B * kBins * 4);
  w->done = (uint32_t*)take((size_t)B * 4);
  w->state = (RowState*)take((size_t)B * sizeof(RowState));
  w->chunk_gt = (uint32_t*)take((size_t)B * C * 4);
  w->chunk_eq = (uint32_t*)take((size_t)B * C * 4);
  w->sel_key = (uint32_t*)take((size_t)B * K * 4);
  w->sel_id = (int32_t*)take((size_t)B * K * 4);
  return off;
}

// ------------------------------------------------------------------------------------------
// consumed mask (ranking.py:38, :59-61)
// ------------------------------------------------------------------------------------------
__global__ void mask_consumed_kernel(float* __restrict__ scores, int64_t ld,
                                     const int64_t* __restrict__ user_ids, int64_t B, int64_t N,
                                     int32_t K, const int64_t* __restrict__ indptr,
                                     const int32_t* __restrict__ idx, int64_t n_users) {
  const int64_t row = blockIdx.x;
  const int64_t u = user_ids[row];
  if (u < 0 || u >= n_users) return;
  const int64_t beg = indptr[u], end = indptr[u + 1];
  const int64_t c = end - beg;
  if (c <= 0 || (int64_t)K + c > N) return;  // "cannot filter" branch: leave the row untouched
  // removed, not -inf: a consumed item must rank below every real score, -inf and NaN included
  float* s = scores + row * ld;
  const float removed = __uint_as_float(kRemovedBits);
  for (int64_t j = beg + threadIdx.x; j < end; j += blockDim.x) {
    const int32_t it = idx[j];
    if (it >= 0 && it < N) s[it] = removed;
  }
}

// ------------------------------------------------------------------------------------------
// radix histogram passes
// ------------------------------------------------------------------------------------------
template <int PASS>
__device__ __forceinline__ bool key_bin(uint32_t key, uint32_t prefix, uint32_t& bin) {
  if (PASS == 0) { bin = key >> 21; return true; }
  if (PASS == 1) { bin = (key >> 10) & 0x7ffu; return (key >> 21) == prefix; }
  bin = key & 0x3ffu; return (key >> 10) == prefix;
}

template <int PASS>
__global__ void __launch_bounds__(kTopkThreads)
radix_hist_kernel(const float* __restrict__ scores, int64_t ld, int64_t N, int32_t K,
                  TopkWorkspace w) {
  __shared__ uint32_t sh[kBins];
  __shared__ uint32_t warp_tot[kTopkThreads / 32];
  __shared__ int is_last;
  const int tid = threadIdx.x;
  const int64_t row = blockIdx.y;
  for (int b = tid; b < kBins; b += kTopkThreads) sh[b] = 0;
  __syncthreads();
  const uint32_t prefix = (PASS == 0) ? 0u : w.state[row].prefix;
  const float* s = scores + row * ld;
  const int64_t beg = (int64_t)blockIdx.x * kTopkChunk;
  const int64_t end = min(beg + (int64_t)kTopkChunk, N);
#pragma unroll 8
  for (int64_t i = beg + tid; i < end; i += kTopkThreads) {
    uint32_t bin;
    if (key_bin<PASS>(float_to_key(__ldg(s + i)), prefix, bin)) atomicAdd(&sh[bin], 1u);
  }
  __syncthreads();
  uint32_t* gh = w.hist + row * kBins;
  for (int b = tid; b < kBins; b += kTopkThreads) {
    const uint32_t c = sh[b];
    if (c) atomicAdd(&gh[b], c);
  }
  __threadfence();
  __syncthreads();
  if (tid == 0) {
    const uint32_t ticket = atomicAdd(&w.done[row], 1u);
    is_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // resolve this pass's digit: largest bin whose suffix count reaches k_rem
  const uint32_t k_rem = (PASS == 0) ? (uint32_t)K : w.state[row].k_rem;
  uint32_t mine[8];
  uint32_t v = 0;
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    mine[j] = __ldcg(&gh[tid * 8 + j]);
    v += mine[j];
  }
  // inclusive suffix scan across the block (thread t owns bins [8t, 8t+8))
  uint32_t incl = v;
  const int lane = tid & 31, wid = tid >> 5;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_down_sync(0xffffffffu, incl, o);
    if (lane + o < 32) incl += t;
  }
  if (lane == 0) warp_tot[wid] = incl;
  __syncthreads();
  uint32_t add = 0;
  for (int w2 = wid + 1; w2 < kTopkThreads / 32; ++w2) add += warp_tot[w2];
  incl += add;
  const uint32_t excl = incl - v;  // count in bins above this thread's range
  if (excl < k_rem && k_rem <= incl) {
    uint32_t c = excl;
#pragma unroll
    for (int j = 7; j >= 0; --j) {
      if (c + mine[j] >= k_rem) {
        const uint32_t bin = tid * 8 + j;
        RowState st;
        st.prefix = (PASS == 0) ? bin : (PASS == 1 ? ((prefix << 11) | bin) : ((prefix << 10) | bin));
        st.k_rem = k_rem - c;
        w.state[row] = st;
        break;
      }
      c += mine[j];
    }
  }
  __syncthreads();
  for (int b = tid; b < kBins; b += kTopkThreads) gh[b] = 0;
  if (tid == 0) w.done[row] = 0;
}

// ------------------------------------------------------------------------------------------
// count (> kth, == kth) per chunk; the last CTA of the row turns counts into exclusive offsets
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTopkThreads)
count_kernel(const float* __restrict__ scores, int64_t ld, int64_t N, TopkWorkspace w, int64_t C) {
  __shared__ uint32_t s_gt, s_eq;
  __shared__ int is_last;
  const int tid = threadIdx.x;
  const int64_t row = blockIdx.y;
  if (tid == 0) { s_gt = 0; s_eq = 0; }
  __syncthreads();
  const uint32_t kth = w.state[row].prefix;
  const float* s = scores + row * ld;
  const int64_t beg = (int64_t)blockIdx.x * kTopkChunk;
  const int64_t end = min(beg + (int64_t)kTopkChunk, N);
  uint32_t gt = 0, eq = 0;
#pragma unroll 8
  for (int64_t i = beg + tid; i < end; i += kTopkThreads) {
    const uint32_t key = float_to_key(__ldg(s + i));
    gt += key > kth;
    eq += key == kth;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    gt += __shfl_xor_sync(0xffffffffu, gt, o);
    eq += __shfl_xor_sync(0xffffffffu, eq, o);
  }
  if ((tid & 31) == 0) { atomicAdd(&s_gt, gt); atomicAdd(&s_eq, eq); }
  __syncthreads();
  if (tid == 0) {
    w.chunk_gt[row * C + blockIdx.x] = s_gt;
    w.chunk_eq[row * C + blockIdx.x] = s_eq;
    __threadfence();
    const uint32_t ticket = atomicAdd(&w.done[row], 1u);
    is_last = (ticket == gridDim.x - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (tid == 0) {  // C is small (N / 8192); a serial exclusive scan is fine
    uint32_t a = 0, b = 0;
    for (int64_t c = 0; c < C; ++c) {
      const uint32_t g = __ldcg(&w.chunk_gt[row * C + c]);
      const uint32_t e = __ldcg(&w.chunk_eq[row * C + c]);
      w.chunk_gt[row * C + c] = a;
      w.chunk_eq[row * C + c] = b;
      a += g;
      b += e;
    }
    w.done[row] = 0;
  }
}

// ------------------------------------------------------------------------------------------
// collect: everything above the K-th key, plus the first k_rem ties in item-id order
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kTopkThreads)
collect_kernel(const float* __restrict__ scores, int64_t ld, int64_t N, int32_t K,
               TopkWorkspace w, int64_t C) {
  __shared__ uint32_t s_gt_pos;
  __shared__ uint32_t s_warp[kTopkThreads / 32];
  __shared__ uint32_t s_base;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  const int64_t row = blockIdx.y;
  const RowState st = w.state[row];
  const uint32_t kth = st.prefix;
  const uint32_t ties_to_take = st.k_rem;
  const uint32_t total_gt = (uint32_t)K - ties_to_take;
  const uint32_t gt_off = w.chunk_gt[row * C + blockIdx.x];
  const uint32_t eq_off = w.chunk_eq[row * C + blockIdx.x];
  if (tid == 0) { s_gt_pos = 0; s_base = 0; }
  __syncthreads();
  const float* s = scores + row * ld;
  uint32_t* okey = w.sel_key + row * K;
  int32_t* oid = w.sel_id + row * K;
  const int64_t beg = (int64_t)blockIdx.x * kTopkChunk;
  const int64_t end = min(beg + (int64_t)kTopkChunk, N);
  const bool want_ties = eq_off < ties_to_take;
  for (int64_t i0 = beg; i0 < end; i0 += kTopkThreads) {
    const int64_t i = i0 + tid;
    uint32_t key = 0;
    bool valid = i < end;
    if (valid) key = float_to_key(__ldg(s + i));
    if (valid && key > kth) {
      const uint32_t p = gt_off + atomicAdd(&s_gt_pos, 1u);
      okey[p] = key;
      oid[p] = (int32_t)i;
    }
    if (want_ties) {  // block-ordered rank of ties (uniform branch)
      const bool is_eq = valid && key == kth;
      const uint32_t bal = __ballot_sync(0xffffffffu, is_eq);
      const uint32_t before = __popc(bal & ((1u << lane) - 1u));
      if (lane == 0) s_warp[wid] = __popc(bal);
      __syncthreads();
      uint32_t wbase = 0, tot = 0;
      for (int w2 = 0; w2 < kTopkThreads / 32; ++w2) {
        const uint32_t c = s_warp[w2];
        if (w2 < wid) wbase += c;
        tot += c;
      }
      const uint32_t rank = eq_off + s_base + wbase + before;
      if (is_eq && rank < ties_to_take) {
        okey[total_gt + rank] = key;
        oid[total_gt + rank] = (int32_t)i;
      }
      __syncthreads();
      if (tid == 0) s_base += tot;
      __syncthreads();
    }
  }
}

// ------------------------------------------------------------------------------------------
// per-row sort of the K selected entries: (score desc, id asc)
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024)
sort_rows_kernel(TopkWorkspace w, int32_t K, int32_t P /*pow2 >= K*/, int64_t* __restrict__ out_ids,
                 float* __restrict__ out_scores) {
  extern __shared__ unsigned long long sm[];
  const int64_t row = blockIdx.x;
  const uint32_t* key = w.sel_key + row * K;
  const int32_t* id = w.sel_id + row * K;
  for (int i = threadIdx.x; i < P; i += blockDim.x) {
    unsigned long long c = 0ull;
    if (i < K) c = ((unsigned long long)key[i] << 32) | (unsigned long long)(~(uint32_t)id[i]);
    sm[i] = c;
  }
  __syncthreads();
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < P; i += blockDim.x) {
        const int ixj = i ^ j;
        if (ixj > i) {
          const unsigned long long a = sm[i], b = sm[ixj];
          const bool desc = ((i & k) == 0);  // descending overall
          if (desc ? (a < b) : (a > b)) { sm[i] = b; sm[ixj] = a; }
        }
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < K; i += blockDim.x) {
    const unsigned long long c = sm[i];
    out_ids[row * K + i] = (int64_t)(~(uint32_t)(c & 0xffffffffull));
    if (out_scores) out_scores[row * K + i] = key_to_float((uint32_t)(c >> 32));
  }
}

}  // namespace b200

using namespace b200;

extern "C" int b200_mask_consumed(float* scores, int64_t ld, const int64_t* user_ids, int64_t B,
                                  int64_t N, int32_t K, const int64_t* indptr, const int32_t* idx,
                                  int64_t n_users, void* stream) {
  B200_REQUIRE(scores && user_ids && indptr, "b200_mask_consumed: null pointer");
  if (B == 0) return 0;
  mask_consumed_kernel<<<(unsigned)B, 128, 0, (cudaStream_t)stream>>>(scores, ld, user_ids, B, N, K,
                                                                      indptr, idx, n_users);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_topk_rows_workspace_bytes(int64_t B, int64_t N, int32_t K, size_t* bytes) {
  B200_REQUIRE(bytes, "null bytes pointer");
  B200_REQUIRE(B >= 0 && N >= 1 && K >= 1, "bad shape B=%lld N=%lld K=%d", (long long)B, (long long)N, K);
  TopkWorkspace w;
  *bytes = carve(&w, nullptr, B, ceil_div64(N, kTopkChunk), K) + 256;
  return 0;
}

// one launch group over at most 65535 rows (gridDim.y limit)
static int topk_rows_chunk(const float* scores, int64_t ld, int64_t B, int64_t N, int32_t K,
                           int64_t* out_ids, float* out_scores, void* workspace,
                           size_t workspace_bytes, cudaStream_t stream) {
  const int64_t C = ceil_div64(N, kTopkChunk);
  TopkWorkspace w;
  char* base = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  const size_t need = carve(&w, base, B, C, K);
  B200_REQUIRE(need + 256 <= workspace_bytes, "b200_topk_rows: workspace too small (%zu < %zu)",
               workspace_bytes, need + 256);
  // hist + done must start zeroed (each pass leaves them zeroed again)
  B200_CUDA_OK(cudaMemsetAsync(w.hist, 0, (size_t)B * kBins * 4, stream));
  B200_CUDA_OK(cudaMemsetAsync(w.done, 0, (size_t)B * 4, stream));
  dim3 grid((unsigned)C, (unsigned)B);
  radix_hist_kernel<0><<<grid, kTopkThreads, 0, stream>>>(scores, ld, N, K, w);
  radix_hist_kernel<1><<<grid, kTopkThreads, 0, stream>>>(scores, ld, N, K, w);
  radix_hist_kernel<2><<<grid, kTopkThreads, 0, stream>>>(scores, ld, N, K, w);
  count_kernel<<<grid, kTopkThreads, 0, stream>>>(scores, ld, N, w, C);
  collect_kernel<<<grid, kTopkThreads, 0, stream>>>(scores, ld, N, K, w, C);
  int P = 1;
  while (P < K) P <<= 1;
  const int threads = P / 2 < 32 ? 32 : (P / 2 > 1024 ? 1024 : P / 2);
  sort_rows_kernel<<<(unsigned)B, threads, (size_t)P * 8, stream>>>(w, K, P, out_ids, out_scores);
  count_launch(6);
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_topk_rows(const float* scores, int64_t ld, int64_t B, int64_t N, int32_t K,
                              int64_t* out_ids, float* out_scores, void* workspace,
                              size_t workspace_bytes, void* stream_) {
  B200_REQUIRE(scores && out_ids && workspace, "b200_topk_rows: null pointer");
  B200_REQUIRE(K >= 1 && K <= kMaxK, "b200_topk_rows: n_rec %d outside [1, %d]", K, kMaxK);
  B200_REQUIRE((int64_t)K <= N, "`n_rec` %d exceeds num of items %lld", K, (long long)N);
  B200_REQUIRE(N < (1ll << 31), "b200_topk_rows: N must be < 2^31");
  // any number of rows: groups of <= 65535 rows run back to back on the stream and share the workspace
  const int64_t kRows = 65535;
  for (int64_t r0 = 0; r0 < B; r0 += kRows) {
    const int64_t b = B - r0 < kRows ? B - r0 : kRows;
    if (int rc = topk_rows_chunk(scores + r0 * ld, ld, b, N, K, out_ids + r0 * K,
                                 out_scores ? out_scores + r0 * K : nullptr, workspace, workspace_bytes,
                                 (cudaStream_t)stream_))
      return rc;
  }
  return 0;
}
