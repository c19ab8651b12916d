// UserCF / ItemCF — recfarm's cosine similarities (rust/src/similarities.rs) on the device.  The neighbourhood
// recommend / predict of rust/src/item_cf.rs and user_cf.rs over the resulting table is neighbours.cu's.
//
// Similarities.  The "sim side" S is the n_x x n_y CSR whose rows are compared (item_interactions for ItemCF,
// user_interactions for UserCF) and the "middle" M = S^T.  sq[x] = sum of r^2 over row x of S in fp32, in row order
// (compute_sum_squares).  For a target row x1, every entry (p, r1) of S's row x1 and every x2 != x1 of M's row p add
// r1 * r[x2, p] to prod[x2] and 1 to count[x2].  Every x2 with count >= min_common is kept, cosine 0 included, with
// cosine = 0 if prod, sq1 or sq2 is 0, else prod / (sqrt(sq1) * sqrt(sq2)) in fp32 (compute_cosine).  Only the order
// of the prod sum differs from the reference (atomics).
//
// Layout.  A task is (target x1, entry range [pb, pe) of its row, slot).  Persistent CTAs take tasks heavy first.
// Middle rows of up to kLongRow entries are walked one warp each, longer ones by the whole CTA.  The accumulator row
// (neighbours.cuh) holds one 64-bit entry per x2, count << 32 | prod bits, updated by one CAS with a plain fp32 add
// (no flush of subnormal products, as in the reference); the add that finds the entry 0 appends x2 to the touched
// list.  The row is in shared memory when 8 n_x bytes fit, otherwise one global row per resident CTA.  A target whose
// work (the sum of its middle rows' lengths) exceeds the piece size is cut into pieces of equal entry counts, merged
// in a global split row of its slot, and finalized by its own kernel.
//
// Selection.  The touched list is compacted to the kept entries (count >= min_common), their cosine written over
// their prod; the kept count is the row's count and its top k_sim by (cosine desc, id asc) are neighbours.cuh's
// radix select on order-preserving keys, so negative cosines rank last and ties go to the smaller id.
#include "common.cuh"
#include "neighbours.cuh"
#include "../../include/b200reco.h"

#include <vector>

namespace b200 {
namespace cf {

using namespace nbr;

constexpr int kLongRow = 256;                 // a middle row longer than this is walked by the whole CTA
constexpr int64_t kMinPieceWork = 1 << 16;    // a target with more work than max(this, total / (8 CTAs)) is split

struct Csr { const int64_t* ptr; const int32_t* idx; const float* val; };

// *p += (c, v) on a packed (count << 32 | prod bits) entry with a plain fp32 add; true for the add that found 0
__device__ __forceinline__ bool add_packed(unsigned long long* p, uint32_t c, float v) {
  unsigned long long old = *p;
  for (;;) {
    const unsigned long long nv = ((unsigned long long)((uint32_t)(old >> 32) + c) << 32) |
                                  __float_as_uint(__fadd_rn(__uint_as_float((uint32_t)old), v));
    const unsigned long long prev = atomicCAS(p, old, nv);
    if (prev == old) return old == 0ull;
    old = prev;
  }
}

// similarities.rs:22-29, in that expression order
__device__ __forceinline__ float cosine(float prod, float sq1, float sq2) {
  if (prod == 0.f || sq1 == 0.f || sq2 == 0.f) return 0.f;
  return __fdiv_rn(prod, __fmul_rn(__fsqrt_rn(sq1), __fsqrt_rn(sq2)));
}

// sq[x] (similarities.rs:13-20) and the work of target x: the summed length of the middle rows it walks
__global__ void sum_squares_kernel(Csr s, const int64_t* __restrict__ mid_ptr, int64_t n_x, float* __restrict__ sq,
                                   int64_t* __restrict__ work) {
  const int64_t x = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (x >= n_x) return;
  float ss = 0.f;
  int64_t w = 0;
  for (int64_t e = s.ptr[x]; e < s.ptr[x + 1]; ++e) {
    ss = __fadd_rn(ss, __fmul_rn(s.val[e], s.val[e]));
    const int32_t p = s.idx[e];
    w += mid_ptr[p + 1] - mid_ptr[p];
  }
  sq[x] = ss;
  work[x] = w;
}

// Compact the T touched entries `tl` of row `acc` to the kept ones (count >= min_common), in place and in any order,
// with their cosine bits over their prod bits; dropped entries are cleared.  Returns the kept count.  Every thread
// of the CTA calls it.
__device__ __forceinline__ int64_t keep_cosines(unsigned long long* acc, int32_t* tl, int64_t T, float sq1,
                                                const float* __restrict__ sq, int64_t min_common) {
  __shared__ unsigned long long s_kept;
  if (threadIdx.x == 0) s_kept = 0;
  __syncthreads();
  for (int64_t base = 0; base < T; base += THREADS) {
    const int64_t e = base + threadIdx.x;
    const int32_t j = e < T ? tl[e] : -1;
    __syncthreads();     // the chunk is read before any write: writes land below the kept count, <= base + THREADS
    if (j >= 0) {
      const unsigned long long a = acc[j];
      if ((int64_t)(a >> 32) >= min_common) {
        const float c = cosine(__uint_as_float((uint32_t)a), sq1, sq[j]);
        acc[j] = (a & 0xffffffff00000000ull) | __float_as_uint(c);
        tl[atomicAdd(&s_kept, 1ull)] = j;
      } else {
        acc[j] = 0ull;
      }
    }
  }
  __syncthreads();
  return (int64_t)s_kept;
}

__device__ __forceinline__ float entry_value(const unsigned long long* acc, int32_t j) {
  return __uint_as_float((uint32_t)acc[j]);
}

__global__ void __launch_bounds__(THREADS) cf_cosine_kernel(
    Csr s, Csr m, const float* __restrict__ sq, int64_t n_x, int64_t min_common, int top_k, int sort_cap,
    int smem_acc, const Task* __restrict__ tasks, int n_tasks, unsigned* __restrict__ task_counter,
    unsigned long long* __restrict__ acc_g, int32_t* __restrict__ tl_g, unsigned long long* __restrict__ split_rows,
    int32_t* __restrict__ split_tl, unsigned long long* __restrict__ split_n, int32_t* __restrict__ nbr_ids,
    float* __restrict__ nbr_scores, int64_t* __restrict__ nbr_count) {
  extern __shared__ __align__(16) unsigned char smem[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem);
  unsigned long long* acc = smem_acc ? keys + sort_cap : acc_g + (int64_t)blockIdx.x * n_x;
  int32_t* tl = tl_g + (int64_t)blockIdx.x * n_x;
  __shared__ int s_task;
  __shared__ unsigned long long s_ntl;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if (smem_acc)
    for (int64_t e = tid; e < n_x; e += THREADS) acc[e] = 0ull;
  if (tid == 0) s_ntl = 0;
  __syncthreads();
  for (;;) {
    if (tid == 0) s_task = (int)atomicAdd(task_counter, 1u);
    __syncthreads();
    const int t = s_task;
    if (t >= n_tasks) break;
    const Task task = tasks[t];
    const int32_t x1 = task.item;
    const int64_t e0 = s.ptr[x1] + task.pb, e1 = s.ptr[x1] + task.pe;
    auto add = [&](int64_t q, float r1) {
      const int32_t x2 = m.idx[q];
      if (x2 != x1 && add_packed(&acc[x2], 1u, __fmul_rn(r1, m.val[q]))) tl[atomicAdd(&s_ntl, 1ull)] = x2;
    };
    for (int64_t e = e0 + warp; e < e1; e += WARPS) {       // short middle rows: one warp each
      const int32_t p = s.idx[e];
      const int64_t b0 = m.ptr[p], b1 = m.ptr[p + 1];
      if (b1 - b0 > kLongRow) continue;
      const float r1 = s.val[e];
      for (int64_t q = b0 + lane; q < b1; q += 32) add(q, r1);
    }
    for (int64_t e = e0; e < e1; ++e) {                      // long middle rows: the whole CTA
      const int32_t p = s.idx[e];
      const int64_t b0 = m.ptr[p], b1 = m.ptr[p + 1];
      if (b1 - b0 <= kLongRow) continue;
      const float r1 = s.val[e];
      for (int64_t q = b0 + tid; q < b1; q += THREADS) add(q, r1);
    }
    __syncthreads();
    const int64_t T = (int64_t)s_ntl;
    if (task.slot < 0) {
      const int64_t kept = keep_cosines(acc, tl, T, sq[x1], sq, min_common);
      if (tid == 0) nbr_count[x1] = kept;
      select_topk<true>([acc](int32_t j) { return entry_value(acc, j); }, tl, kept, top_k, sort_cap, keys,
                        nbr_ids + (int64_t)x1 * top_k, nbr_scores + (int64_t)x1 * top_k);
      for (int64_t e = tid; e < kept; e += THREADS) acc[tl[e]] = 0ull;
    } else {
      unsigned long long* row = split_rows + (int64_t)task.slot * n_x;
      int32_t* stl = split_tl + (int64_t)task.slot * n_x;
      for (int64_t e = tid; e < T; e += THREADS) {
        const int32_t j = tl[e];
        const unsigned long long a = acc[j];
        if (add_packed(&row[j], (uint32_t)(a >> 32), __uint_as_float((uint32_t)a)))
          stl[atomicAdd(&split_n[task.slot], 1ull)] = j;
      }
      __syncthreads();
      for (int64_t e = tid; e < T; e += THREADS) acc[tl[e]] = 0ull;
    }
    if (tid == 0) s_ntl = 0;
    __syncthreads();
  }
}

// one CTA per split slot in use: keep, select from the slot's row, then clear the row for the next round
__global__ void __launch_bounds__(THREADS, 1) cf_split_finalize_kernel(
    const int32_t* __restrict__ slot_item, const float* __restrict__ sq, int64_t min_common, int top_k, int sort_cap,
    int64_t n_x, unsigned long long* __restrict__ split_rows, int32_t* __restrict__ split_tl,
    unsigned long long* __restrict__ split_n, int32_t* __restrict__ nbr_ids, float* __restrict__ nbr_scores,
    int64_t* __restrict__ nbr_count) {
  extern __shared__ __align__(16) unsigned char smem[];
  unsigned long long* keys = reinterpret_cast<unsigned long long*>(smem);
  const int s = blockIdx.x;
  const int32_t x1 = slot_item[s];
  unsigned long long* row = split_rows + (int64_t)s * n_x;
  int32_t* stl = split_tl + (int64_t)s * n_x;
  const int64_t kept = keep_cosines(row, stl, (int64_t)split_n[s], sq[x1], sq, min_common);
  if (threadIdx.x == 0) nbr_count[x1] = kept;
  select_topk<true>([row](int32_t j) { return entry_value(row, j); }, stl, kept, top_k, sort_cap, keys,
                    nbr_ids + (int64_t)x1 * top_k, nbr_scores + (int64_t)x1 * top_k);
  for (int64_t e = threadIdx.x; e < kept; e += THREADS) row[stl[e]] = 0ull;
  if (threadIdx.x == 0) split_n[s] = 0;
}

// ---------------------------------------------------------------------------------------------------------------
// shared memory: [sort keys u64 sort_cap][acc u64 n_x (shared path)]
Plan make_plan(int64_t n_x, int k_sim) {
  return nbr::make_plan(cf_cosine_kernel, n_x, k_sim, sizeof(unsigned long long), 0);
}

// the workspace: sq and the per-target work, then the scheduler's pieces
Workspace<unsigned long long> carve(unsigned char* ws, int64_t n_x, const Plan& p) {
  return Workspace<unsigned long long>(ws, round256((size_t)n_x * 4) + round256((size_t)n_x * 8), n_x, p);
}

}  // namespace cf
}  // namespace b200

using namespace b200;
using namespace b200::cf;

extern "C" int b200_cf_cosine_workspace_bytes(int64_t n_x, int32_t k_sim, size_t* bytes) {
  B200_REQUIRE(bytes, "b200_cf_cosine_workspace_bytes: null pointer");
  B200_REQUIRE(n_x >= 1 && n_x < (1ll << 31), "b200_cf_cosine: bad shape");
  B200_REQUIRE(k_sim >= 1 && k_sim <= kMaxTopK, "b200_cf_cosine: k_sim %d outside [1, %d]", k_sim, kMaxTopK);
  const Plan p = make_plan(n_x, k_sim);
  B200_REQUIRE(p.ctas > 0, "b200_cf_cosine: no resident CTA for %lld rows", (long long)n_x);
  *bytes = carve(nullptr, n_x, p).bytes;
  return 0;
}

extern "C" int b200_cf_plan(int64_t n_x, int32_t k_sim, int32_t* smem_acc, int32_t* ctas) {
  B200_REQUIRE(smem_acc && ctas, "b200_cf_plan: null pointer");
  B200_REQUIRE(n_x >= 1 && n_x < (1ll << 31) && k_sim >= 1 && k_sim <= kMaxTopK, "b200_cf_plan: bad shape");
  const Plan p = make_plan(n_x, k_sim);
  *smem_acc = p.smem_acc ? 1 : 0;
  *ctas = p.ctas;
  return 0;
}

extern "C" int b200_cf_cosine(const int64_t* sim_ptr, const int32_t* sim_idx, const float* sim_val, int64_t n_x,
                              const int64_t* mid_ptr, const int32_t* mid_idx, const float* mid_val, int64_t n_y,
                              int64_t min_common, int32_t k_sim, int32_t* nbr_ids, float* nbr_scores,
                              int64_t* nbr_count, void* workspace, size_t workspace_bytes, void* stream_) {
  B200_REQUIRE(sim_ptr && mid_ptr && nbr_ids && nbr_scores && nbr_count && workspace, "b200_cf_cosine: null pointer");
  size_t need = 0;
  if (int rc = b200_cf_cosine_workspace_bytes(n_x, k_sim, &need)) return rc;
  B200_REQUIRE(workspace_bytes >= need, "b200_cf_cosine: workspace %zu < %zu bytes", workspace_bytes, need);
  B200_REQUIRE(n_y >= 0 && n_y < (1ll << 31), "b200_cf_cosine: bad shape");
  B200_REQUIRE(min_common >= 1, "b200_cf_cosine: min_common must be >= 1");
  cudaStream_t stream = (cudaStream_t)stream_;
  const Plan p = make_plan(n_x, k_sim);
  unsigned char* ws = static_cast<unsigned char*>(workspace);
  const Workspace<unsigned long long> W = carve(ws, n_x, p);
  float* sq = reinterpret_cast<float*>(ws);
  int64_t* work_d = reinterpret_cast<int64_t*>(ws + round256((size_t)n_x * 4));

  B200_CUDA_OK(cudaMemsetAsync(nbr_ids, 0xff, (size_t)n_x * k_sim * 4, stream));
  B200_CUDA_OK(cudaMemsetAsync(nbr_scores, 0, (size_t)n_x * k_sim * 4, stream));
  B200_CUDA_OK(cudaMemsetAsync(nbr_count, 0, (size_t)n_x * 8, stream));

  const Csr s{sim_ptr, sim_idx, sim_val}, m{mid_ptr, mid_idx, mid_val};
  sum_squares_kernel<<<(unsigned)ceil_div64(n_x, 256), 256, 0, stream>>>(s, mid_ptr, n_x, sq, work_d);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());

  // plan the tasks on the host from the per-target work and row lengths
  std::vector<int64_t> sptr(n_x + 1), work(n_x);
  B200_CUDA_OK(cudaMemcpyAsync(sptr.data(), sim_ptr, (n_x + 1) * 8, cudaMemcpyDeviceToHost, stream));
  B200_CUDA_OK(cudaMemcpyAsync(work.data(), work_d, n_x * 8, cudaMemcpyDeviceToHost, stream));
  B200_CUDA_OK(cudaStreamSynchronize(stream));
  B200_REQUIRE(sptr[0] == 0, "b200_cf_cosine: sim_ptr[0] != 0");
  for (int64_t x = 0; x < n_x; ++x) {
    const int64_t d = sptr[x + 1] - sptr[x];
    B200_REQUIRE(d >= 0 && d <= n_y, "b200_cf_cosine: row %lld has a bad length", (long long)x);
  }

  auto cut = [](int32_t x, int64_t d, int64_t n_pieces, int32_t slot, std::vector<Task>& tasks) {
    n_pieces = std::min(n_pieces, d);
    for (int64_t q = 0; q < n_pieces; ++q)      // equal entry counts
      tasks.push_back(Task{x, (int32_t)(d * q / n_pieces), (int32_t)(d * (q + 1) / n_pieces), slot});
  };
  auto scores = [&](int n_tasks) {
    cf_cosine_kernel<<<p.ctas, THREADS, p.smem, stream>>>(
        s, m, sq, n_x, min_common, k_sim, p.sort_cap, p.smem_acc ? 1 : 0, W.tasks, n_tasks, W.counter, W.acc, W.tl,
        W.split_rows, W.split_tl, W.split_n, nbr_ids, nbr_scores, nbr_count);
  };
  auto finalize = [&](unsigned n_slots) {
    cf_split_finalize_kernel<<<n_slots, THREADS, (size_t)p.sort_cap * 8, stream>>>(
        W.slot_item, sq, min_common, k_sim, p.sort_cap, n_x, W.split_rows, W.split_tl, W.split_n, nbr_ids,
        nbr_scores, nbr_count);
  };
  return run_rounds(sptr, work, kMinPieceWork, p, W, stream, cut, scores, finalize);
}
