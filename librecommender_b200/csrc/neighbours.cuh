// What the scoring of the neighbourhood engines (swing.cu, cf.cu) shares: per-target accumulator rows with a
// first-touch list, heavy targets split over CTAs into global split rows, the exact radix select of a row's top k, and
// on the host the plan, the workspace and the rounds of tasks that drive a scores kernel.  Serving a neighbour table
// (recommend, predict) is neighbours.cu.
//
// Accumulator rows.  A persistent CTA owns one row of n_targets entries, in shared memory when it fits and otherwise
// one global row per resident CTA.  The add that finds an entry untouched appends its id to the CTA's touched list,
// so clearing, counting and selection cost the row's touched entries, never n_targets.  A target too heavy for one
// CTA is cut into pieces (tasks with slot >= 0); each piece flushes its touched entries into the global row of the
// target's split slot, with its own touched list, and a finalize kernel selects from that row.
#pragma once
#include "common.cuh"

#include <algorithm>
#include <vector>

namespace b200 {
namespace nbr {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int kMaxTopK = 4096;
constexpr int kSlots = 64;                    // split targets in flight per round
constexpr int kMaxPieces = 1024;              // pieces per split target
constexpr int kMaxGlobalCtasPerSm = 4;        // global accumulator rows: bound their number

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

// ---- host: the plan, the workspace and the rounds of a scores kernel ------------------------------------------------

struct Plan {
  bool smem_acc;     // the accumulator rows are in shared memory, else one global row per resident CTA
  int ctas;          // resident CTAs of the scores kernel; 0 when its shared memory cannot fit
  size_t smem;       // its dynamic shared memory
  int sort_cap;      // power of two >= top_k
};

// The plan of `kernel` over rows of n accumulator entries of entry_bytes each.  Dynamic shared memory:
// [sort keys u64 sort_cap][extra_smem bytes of the engine's][acc entry_bytes * n (shared path)].
template <typename Kernel>
Plan make_plan(Kernel kernel, int64_t n, int top_k, size_t entry_bytes, size_t extra_smem) {
  Plan p;
  p.sort_cap = pow2_ceil(top_k);
  int dev = 0, optin = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  const size_t reserve = 2048;     // the kernel's static shared memory
  const size_t base = (size_t)p.sort_cap * 8 + extra_smem, acc = (size_t)n * entry_bytes;
  p.smem_acc = base + acc + reserve <= (size_t)optin;
  p.smem = base + (p.smem_acc ? acc : 0);
  p.ctas = 0;
  if (p.smem + reserve > (size_t)optin) return p;     // extra_smem alone does not fit (Swing's bitmap)
  if (cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)p.smem) != cudaSuccess) return p;
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, THREADS, p.smem) != cudaSuccess) return p;
  if (!p.smem_acc) per_sm = std::min(per_sm, kMaxGlobalCtasPerSm);
  p.ctas = per_sm * num_sms();
  return p;
}

inline size_t round256(size_t bytes) { return (bytes + 255) & ~(size_t)255; }

// A scores call's workspace: the engine's own arrays (`prefix` bytes at its start), then the scheduler's pieces, each
// rounded to 256 B on its own.  Entry is the accumulator entry.  With ws == nullptr only `bytes` is meaningful.
template <typename Entry>
struct Workspace {
  unsigned* counter;                  // the task counter of a round
  Task* tasks;                        // a round's tasks
  int32_t* slot_item;                 // the target of each split slot in use
  int32_t* tl;                        // one touched list of n per resident CTA
  Entry* acc;                         // one accumulator row of n per resident CTA; nullptr on the shared path
  Entry* split_rows;                  // per split slot: a row of n, its touched list and its touched count
  int32_t* split_tl;
  unsigned long long* split_n;
  size_t bytes;                       // the whole workspace, prefix included

  Workspace(unsigned char* ws, size_t prefix, int64_t n, const Plan& p) {
    size_t off = prefix;
    auto take = [&](size_t b) {
      const size_t at = off;
      off += round256(b);
      return ws ? static_cast<void*>(ws + at) : nullptr;
    };
    counter = static_cast<unsigned*>(take(4));
    tasks = static_cast<Task*>(take(((size_t)n + (size_t)kSlots * kMaxPieces) * sizeof(Task)));
    slot_item = static_cast<int32_t*>(take((size_t)kSlots * 4));
    tl = static_cast<int32_t*>(take((size_t)p.ctas * n * 4));
    acc = static_cast<Entry*>(take(p.smem_acc ? 0 : (size_t)p.ctas * n * sizeof(Entry)));
    if (p.smem_acc) acc = nullptr;
    split_rows = static_cast<Entry*>(take((size_t)kSlots * n * sizeof(Entry)));
    split_tl = static_cast<int32_t*>(take((size_t)kSlots * n * 4));
    split_n = static_cast<unsigned long long*>(take((size_t)kSlots * 8));
    bytes = off;
  }
};

// Runs the scores kernel over the n targets with weight[x] > 0 (row x of the host row pointers ptr holds
// ptr[x + 1] - ptr[x] entries), heaviest first, ties to the smaller id.  A target of more than one entry whose
// weight exceeds the piece size max(min_piece, total weight / (8 resident CTAs)) is split:
// cut(x, entries, n_pieces, slot, tasks) appends its pieces, n_pieces = min(kMaxPieces, ceil(weight / piece)).
// Each round gives up to kSlots split targets a slot, split targets first, then takes an even, strided share of the
// whole targets; a round without tasks is skipped.  scores(n_tasks) launches the scores kernel on the round's
// uploaded tasks, finalize(n_slots) the split finalize kernel over its slots.  Synchronises `stream` once at the end.
template <typename Entry, typename Cut, typename Scores, typename Finalize>
int run_rounds(const std::vector<int64_t>& ptr, const std::vector<int64_t>& weight, int64_t min_piece,
               const Plan& p, const Workspace<Entry>& w, cudaStream_t stream, Cut cut, Scores scores,
               Finalize finalize) {
  const int64_t n = (int64_t)weight.size();
  int64_t total = 0;
  for (int64_t x = 0; x < n; ++x) total += weight[x];
  if (total == 0) return 0;
  const int64_t piece = std::max(min_piece, total / ((int64_t)p.ctas * 8));
  std::vector<int32_t> whole, split;
  for (int64_t x = 0; x < n; ++x) {
    if (weight[x] == 0) continue;
    (weight[x] > piece && ptr[x + 1] - ptr[x] > 1 ? split : whole).push_back((int32_t)x);
  }
  auto heavier = [&](int32_t a, int32_t b) { return weight[a] != weight[b] ? weight[a] > weight[b] : a < b; };
  std::sort(whole.begin(), whole.end(), heavier);
  std::sort(split.begin(), split.end(), heavier);

  if (!p.smem_acc) B200_CUDA_OK(cudaMemsetAsync(w.acc, 0, (size_t)p.ctas * n * sizeof(Entry), stream));
  B200_CUDA_OK(cudaMemsetAsync(w.split_rows, 0, (size_t)kSlots * n * sizeof(Entry), stream));
  B200_CUDA_OK(cudaMemsetAsync(w.split_n, 0, (size_t)kSlots * 8, stream));

  const int64_t rounds = std::max<int64_t>(1, ceil_div64((int64_t)split.size(), kSlots));
  std::vector<Task> tasks;
  std::vector<int32_t> slot_item;
  for (int64_t r = 0; r < rounds; ++r) {
    tasks.clear();
    slot_item.clear();
    for (int64_t s = r * kSlots; s < (int64_t)split.size() && s < (r + 1) * kSlots; ++s) {
      const int32_t x = split[s];
      cut(x, ptr[x + 1] - ptr[x], std::min<int64_t>(kMaxPieces, ceil_div64(weight[x], piece)),
          (int32_t)slot_item.size(), tasks);
      slot_item.push_back(x);
    }
    for (size_t t = (size_t)r; t < whole.size(); t += (size_t)rounds)
      tasks.push_back(Task{whole[t], 0, (int32_t)(ptr[whole[t] + 1] - ptr[whole[t]]), -1});
    if (tasks.empty()) continue;
    B200_CUDA_OK(cudaMemcpyAsync(w.tasks, tasks.data(), tasks.size() * sizeof(Task), cudaMemcpyHostToDevice, stream));
    B200_CUDA_OK(cudaMemsetAsync(w.counter, 0, 4, stream));
    scores((int)tasks.size());
    count_launch();
    B200_CUDA_OK(cudaGetLastError());
    if (!slot_item.empty()) {
      B200_CUDA_OK(cudaMemcpyAsync(w.slot_item, slot_item.data(), slot_item.size() * 4, cudaMemcpyHostToDevice,
                                   stream));
      finalize((unsigned)slot_item.size());
      count_launch();
      B200_CUDA_OK(cudaGetLastError());
    }
  }
  // the host task vectors are released on return: wait for the last upload to have been read
  B200_CUDA_OK(cudaStreamSynchronize(stream));
  return 0;
}

}  // namespace nbr
}  // namespace b200
