// K4 — fused user x all-items scoring + consumed filter + top-K on the Hopper tensor cores (wgmma).
//
// Replaces recommend_from_embedding + rank_recommendations
// (libreco/recommendation/recommend.py:57-78, ranking.py:10-78) without ever materialising
// the [B, N] score matrix.
//
// Pipeline (all on one stream, no host sync):
//   prep_items   (once per item table)  fp32 [N,d] -> fp16 [N_pad, d_pad] (K-major, zero padded),
//                                        scaled by a power of two so that max ||I_i|| is in [64,128)
//   prep_users   gather U[user_ids] -> fp16 [B_pad, d_pad], every row scaled by its own power of
//                two (row norm in [64,128)); per-row error bound eps, k_row
//   sweep<PRE>   tensor-core pass over every pre_stride-th item tile that only records, per user row, the
//                maximum coarse score of each sampled 128-item block (one coalesced store per
//                tile, no divergence); guess_kernel turns the block maxima into a SPECULATIVE
//                per-row threshold (the pre_k-th largest block maximum, pre_k from a failure budget).
//   sweep<MAIN>  persistent wgmma kernel over all item tiles: TMA -> smem (SWIZZLE_128B, multi-stage
//                ring, item tiles shared by a 2-CTA cluster through TMA multicast) -> wgmma (fp16 in,
//                fp32 accumulate in registers, 128x256 tile = two warpgroups x 64 user rows) -> the
//                same warpgroups keep, per user row, every item whose COARSE score is >= tau.  tau starts at the speculative value and
//                is only ever raised by a rigorous bound: (k_row-th best coarse score counted so
//                far in the row's global histogram) - 2*eps.
//   finalize     per row: exact k_row-th coarse score c_k over the union of the lists; checks that
//                the speculative threshold did not exceed c_k - 2*eps (otherwise the row is
//                flagged); cuts at c_k - 2*eps, drops consumed items, EXACT fp32 re-score
//                (sequential fma = the library's exact-score definition), sorts by
//                (score desc, id asc), emits K ids.  One warp per row (finalize_warp_kernel); rows
//                outside its envelope are deferred to one CTA per row (finalize_kernel).
//
// Coarse scores live in a SCALED domain: coarse(u, i) ~ s_u * s_i * <u, i> with s_u, s_i powers of
// two (exact scalings), so the fp16 operands keep 11 significant bits whatever the magnitude of the
// embeddings; every threshold of a row (tau, eps, R, histogram range) is in that row's scaled units.
//
// Exactness argument: |coarse - s_u s_i exact| <= eps for every (user, item) (fp16 rounding of both
// operands, |delta| <= 2^-11 each, plus an absolute term that covers fp16 subnormals even if the
// tensor core flushed them, plus a generous accumulation term).  Let c_k be the k-th
// largest coarse score.  Every item of the exact top-k has coarse >= c_k - 2 eps.  The lists hold
// every item with coarse >= T, T = the largest threshold ever used for the row; finalize proves
// T <= c_k - 2 eps (rigorous raises satisfy it by construction, the speculative start value is
// checked explicitly), so the candidate set contains the exact top-k; the order is decided on
// exact fp32 scores only.  k_row = K + c_u (c_u = consumed count, duplicates included) when the
// reference's filter rule applies (ranking.py:38), so removing consumed candidates still leaves
// the exact top-K.  Rows that cannot be bounded (k_row too large, failed speculation, too many
// near-ties) are flagged in row_status and re-run by the caller on the exact materialised path.
#include <cmath>
#include <type_traits>
#include "common.cuh"
#include "ptx_sm90.cuh"
#include "../../include/b200reco.h"
#include <cuda_fp16.h>

namespace b200 {
namespace tc {

constexpr int TM = 128;        // users per tile (two wgmma M = 64 warpgroups)
constexpr int TN = 256;        // items per tile (wgmma N)
constexpr int KBLK = 64;       // fp16 per 128-byte swizzled row
constexpr int CAPG_MAX = 256;  // candidate GROUP records per (row, list), upper limit (runtime capg <= this)
constexpr int GW = 8;          // a record = the 8 coarse scores of one 8-column group + its first item id ...
constexpr int REC = 12;        // ... in 12 words (48 bytes: two 16-byte score halves, the id, padding)
constexpr int NB = 1024;       // bins of the per-row global coarse-score histogram
constexpr int STEP = 64;       // accumulator columns per epilogue vote
// Every (row, item split) has two candidate lists, one per 128-column half of the item tiles:
// n_lists = 2 * n_splits.  The pre-pass records one block maximum per row and half (block = 128 items).
constexpr int W_PRE = 2;
constexpr int KROW_MAX = 288;  // fast-path limit for k_row = K + c_u
constexpr int MAX_KB = 4;      // d_pad <= 256
// Speculation defaults (b200_recommend_embed_speculation): the pre-pass visits every PRE_STRIDE-th item
// tile of a split, and a row's speculative threshold fails with probability at most PRE_DELTA (DESIGN §4).
constexpr int PRE_STRIDE = 8;
constexpr double PRE_DELTA = 1e-5;
// items allowed for inside the 2 eps band below c_k when the speculative rank is chosen (DESIGN §4)
constexpr int PRE_TIE_ALLOWANCE = 16;
constexpr int A_KB_BYTES = TM * KBLK * 2;   // 16 KB
constexpr int B_KB_BYTES = TN * KBLK * 2;   // 32 KB
constexpr int MAXU = 3072;                  // finalize: collected elements per row (union of the lists)
constexpr int MAXC = 2048;                  // finalize: candidates per row after the c_k - 2 eps cut
constexpr int FIN_THREADS = 256;
// |coarse - exact| <= ERR_COEF * ||u|| * ||i|| (+ absolute subnormal term, + accumulation slack):
// fp16 x fp16 products, both operands rounded to nearest: (1 + 2^-11)^2 - 1 = 2^-10 (1 + 2^-12)
constexpr float ERR_COEF = 0.00097705f;

constexpr int SWEEP_CONSUMER_WARPS = 8;   // two warpgroups: wgmma M = 64 user rows each
constexpr int WARP_TMA = SWEEP_CONSUMER_WARPS;   // first warp of the producer warpgroup
// registers are handed out per warpgroup: the producer warpgroup gives most of its share to the two
// consumer warpgroups (128 accumulator registers per thread plus the epilogue state, no spills)
constexpr int SWEEP_THREADS = 32 * (SWEEP_CONSUMER_WARPS + 4);
constexpr int SWEEP_PRODUCER_REGS = 40, SWEEP_CONSUMER_REGS = 232;

struct CatalogHeader {   // first 256 bytes of the catalog buffer (device)
  uint32_t max_norm_bits;  // max_i ||I_i||_2 of the UNSCALED rows (fp32 bits; non-negative so uint order == float order)
  int32_t d, d_pad;
  int64_t N, N_pad;
  float scale;             // power of two applied to every item row before the fp16 rounding
  float max_norm_scaled;   // scale * max norm (rounded up), in [64, 128) unless the table is all zero
};

struct RowMeta {
  float eps2;       // 2 * eps                                   (scaled units of the row)
  float R;          // |coarse score| <= R for every item (Cauchy-Schwarz on the row norms)
  float scale;      // s_u * s_i: coarse ~ scale * exact
  int32_t k_row;    // K (+ consumed count when the filter applies)
  int32_t pre_k;    // rank of the block maximum used as speculative threshold
  int32_t active;   // 0: pad row (never collects)
  int32_t apply;    // consumed filter applies
  int32_t capped;   // k_row was capped below K + c_u: finalize must verify the result a posteriori
};


struct SweepParams {
  int64_t N;
  int32_t B_pad, m_tiles, n_splits, tiles_per_split, total_tiles, KB, nstage;
  int32_t kb_stages;          // 1: a ring stage holds ONE 64-wide k-block of an item tile (d_pad > 128), 0: the whole tile
  int32_t n_pre_tiles;        // sampled tiles per split in the pre-pass
  int32_t pre_stride;         // the pre-pass visits every pre_stride-th tile of a split
  int32_t capg, trig;         // records per list / uncounted records that trigger a compaction
  int32_t ablate;             // diagnostics only (b200_recommend_embed_debug): 0 = normal operation
  uint32_t hint_ns;           // suspend-time hint of the mbarrier waits
  const RowMeta* meta;        // [B_pad]
  uint32_t* row_tau_key;      // [B_pad]  running max of tau (order-preserving key)
  int32_t* row_status;        // [B_pad]  1 = needs the exact path
  uint32_t* ghist;            // [B_pad][NB]  coarse-score histogram of every counted candidate
  float* cand_r;              // [W*n_splits][B_pad][capg][REC]  group records: 8 coarse scores + first item id
  int32_t* cand_cnt;          // [W*n_splits][B_pad]            records per list
  float* blockmax;            // [W_PRE*n_splits][n_pre_tiles][B_pad]   (pre-pass output)
};

// ------------------------------------------------------------------------------------------
// prep kernels
// ------------------------------------------------------------------------------------------
// power of two s with s * nrm in [64, 128) (1 for a zero / non-finite norm)
__device__ __forceinline__ float pow2_scale_for(float nrm) {
  if (!(nrm > 0.f) || !(nrm < 3.0e38f)) return 1.f;
  int x;
  frexpf(nrm, &x);                 // nrm = m * 2^x, m in [0.5, 1)
  int e = 7 - x;                   // m * 2^7 in [64, 128)
  e = max(-120, min(120, e));
  return ldexpf(1.f, e);
}

__global__ void item_norm_kernel(const float* __restrict__ I, int64_t ldi, int64_t N, int d,
                                 CatalogHeader* hdr) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= N) return;
  float ss = 0.f;
  for (int k = lane; k < d; k += 32) {
    const float v = __ldg(I + row * ldi + k);
    ss = fmaf(v, v, ss);
  }
  ss = warp_sum(ss);
  if (lane == 0) atomicMax(&hdr->max_norm_bits, __float_as_uint(sqrtf(ss) * 1.0001f));  // round up a little
}

__global__ void item_scale_kernel(CatalogHeader* hdr) {
  const float mx = __uint_as_float(hdr->max_norm_bits);
  const float s = pow2_scale_for(mx);
  hdr->scale = s;
  hdr->max_norm_scaled = mx * s;
}

__global__ void prep_items_kernel(const float* __restrict__ I, int64_t ldi, int64_t N, int d,
                                  int d_pad, int64_t N_pad, __half* __restrict__ out,
                                  const CatalogHeader* __restrict__ hdr) {
  // one warp per item row
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= N_pad) return;
  const float s = hdr->scale;
  for (int k = lane; k < d_pad; k += 32) {
    float v = 0.f;
    if (row < N && k < d) v = __ldg(I + row * ldi + k) * s;
    out[row * d_pad + k] = __float2half_rn(v);
  }
}

struct PreRank {   // speculative rank pre_k of every k_row (rank_table on the host)
  int32_t k[KROW_MAX + 1];
};

__global__ void prep_users_kernel(const float* __restrict__ U, int64_t ldu,
                                  const int64_t* __restrict__ user_ids, int64_t B, int B_pad, int d,
                                  int d_pad, int K, int64_t N, int filter, const __grid_constant__ PreRank pre_rank,
                                  const int64_t* __restrict__ indptr, int64_t n_users,
                                  const CatalogHeader* __restrict__ hdr,
                                  __half* __restrict__ A, RowMeta* __restrict__ meta,
                                  uint32_t* __restrict__ row_tau_key, int32_t* __restrict__ row_status) {
  const int64_t row = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (row >= B_pad) return;
  const bool real = row < B;
  const int64_t u = real ? user_ids[row] : 0;
  float ss = 0.f;
  for (int k = lane; k < d; k += 32) {
    const float v = real ? __ldg(U + u * ldu + k) : 0.f;
    ss = fmaf(v, v, ss);
  }
  ss = warp_sum(ss);
  const float nrm = sqrtf(ss) * 1.0001f;
  const float su = pow2_scale_for(nrm);
  for (int k = lane; k < d_pad; k += 32) {
    float v = 0.f;
    if (real && k < d) v = __ldg(U + u * ldu + k) * su;      // exact scaling, then one fp16 rounding
    A[row * d_pad + k] = __float2half_rn(v);
  }
  if (lane == 0) {
    RowMeta m;
    const float nu = nrm * su, ni = hdr->max_norm_scaled;    // scaled norms (< 128 each)
    // relative part (operand rounding + fp32 accumulation slack) + absolute part: an operand below
    // the fp16 normal range is off by at most 2^-25 (rounded) resp. 2^-14 (if the tensor core
    // flushed subnormals); sum_k |x_k| * 2^-14 <= sqrt(d) * ||x|| * 2^-14 for both operands
    const float coef = ERR_COEF + (float)d_pad * 2.4e-7f;
    const float abs_term = sqrtf((float)d_pad) * 6.2e-5f * (nu + ni);
    m.eps2 = 2.f * (coef * nu * ni + abs_term) + 1e-30f;
    m.R = 1.02f * nu * ni + 1e-30f;
    m.scale = su * hdr->scale;
    int64_t c = 0;
    if (real && filter && indptr && u >= 0 && u < n_users) c = indptr[u + 1] - indptr[u];
    const bool apply = c > 0 && (int64_t)K + c <= N;
    // k_row = K + c_u guarantees K survivors after the consumed filter.  Heavy users would need
    // lists longer than the kernel keeps: their k_row is capped and finalize_kernel verifies the
    // result instead (the K-th surviving exact score must beat everything that was not collected).
    const int64_t k_full = (int64_t)K + (apply ? c : 0);
    const int64_t k_row = min(k_full, (int64_t)KROW_MAX);
    m.apply = apply;
    m.capped = k_row < k_full;
    m.k_row = (int32_t)k_row;
    // speculative threshold = pre_k-th largest SAMPLED block maximum
    m.pre_k = pre_rank.k[m.k_row];
    m.active = real;
    meta[row] = m;
    row_tau_key[row] = 0u;  // below every finite float
    row_status[row] = 0;
  }
}

// ------------------------------------------------------------------------------------------
// sweep kernel
// ------------------------------------------------------------------------------------------
struct SweepSmem {
  uint64_t full[8];
  uint64_t empty[8];
  uint64_t a_full;
  uint64_t a_empty;
};

__device__ __forceinline__ int score_bin(float s, float R, float inv_w) {
  const float t = (s + R) * inv_w;
  return (int)fminf(fmaxf(t, 0.f), (float)(NB - 1));
}

// Warp-cooperative compaction of one candidate list of one row (rare in the main pass: the
// speculative threshold keeps the lists short; this is the rigorous safety net and the normal
// mode when no pre-pass ran).  A list holds GROUP records (8 scores + first item id, REC words).
//  1. every element >= tau_old of every record pushed since the previous compaction is counted
//     ONCE into the row's global coarse-score histogram (shared by all lists / CTAs of the row);
//  2. the histogram is read back: the highest bin whose suffix count reaches k gives a rigorous
//     lower bound of the k-th largest coarse score over everything counted so far
//     (counts are a subset of the items at or above each edge), tau = edge - eps2;
//  3. the list is rewritten keeping the records whose maximum is >= tau.
// Records live in registers (CAPG_MAX/32 per lane).  Returns the new count; *tau_out = new tau.
__device__ __noinline__ int compact_row(float* __restrict__ ls, int n,
                                           int n_counted, int k, float eps2, float R, float tau_old,
                                           uint32_t* __restrict__ gh, int lane, int32_t n_items,
                                           float* tau_out) {
  const float inv_w = (float)NB / (2.f * R);
  constexpr int PER = CAPG_MAX / 32;
  float4 e0[PER], e1[PER];
  int32_t bs[PER];
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int i = j * 32 + lane;
    e0[j] = e1[j] = make_float4(0.f, 0.f, 0.f, 0.f);
    bs[j] = 0;
    if (i < n) {
      e0[j] = *reinterpret_cast<const float4*>(ls + (size_t)i * REC);
      e1[j] = *reinterpret_cast<const float4*>(ls + (size_t)i * REC + 4);
      bs[j] = reinterpret_cast<const int32_t*>(ls)[(size_t)i * REC + 8];
    }
  }
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int i = j * 32 + lane;
    if (i >= n_counted && i < n) {
      const float v[GW] = {e0[j].x, e0[j].y, e0[j].z, e0[j].w, e1[j].x, e1[j].y, e1[j].z, e1[j].w};
#pragma unroll
      for (int q = 0; q < GW; ++q)   // zero-padded item rows (id >= N) are not items: never counted
        if (v[q] >= tau_old && bs[j] + q < n_items) atomicAdd(gh + score_bin(v[q], R, inv_w), 1u);
    }
  }
  __threadfence();
  __syncwarp();
  // lane l owns bins [32 l, 32 l + 32); lane 31 holds the top of the range
  uint32_t mine[32], tot = 0;
#pragma unroll
  for (int q4 = 0; q4 < 8; ++q4) {
    const uint4 h = __ldcg(reinterpret_cast<const uint4*>(gh + lane * 32) + q4);
    mine[q4 * 4 + 0] = h.x; mine[q4 * 4 + 1] = h.y; mine[q4 * 4 + 2] = h.z; mine[q4 * 4 + 3] = h.w;
    tot += h.x + h.y + h.z + h.w;
  }
  uint32_t incl = tot;
#pragma unroll
  for (int o = 1; o < 32; o <<= 1) {
    const uint32_t t = __shfl_down_sync(0xffffffffu, incl, o);
    if (lane + o < 32) incl += t;
  }
  const uint32_t excl = incl - tot;
  const bool owner = excl < (uint32_t)k && (uint32_t)k <= incl;
  int f_bin = -1;
  if (owner) {
    uint32_t c = excl;
#pragma unroll
    for (int b = 31; b >= 0; --b) {
      c += mine[b];
      if (c >= (uint32_t)k) { f_bin = lane * 32 + b; break; }
    }
  }
  const uint32_t bal = __ballot_sync(0xffffffffu, owner);
  float tau = tau_old;
  if (bal) {
    f_bin = __shfl_sync(0xffffffffu, f_bin, __ffs(bal) - 1);
    const float edge = -R + (float)f_bin * (2.f * R / (float)NB) - 1e-6f * R;
    tau = fmaxf(tau, edge - eps2);
  }
  *tau_out = tau;
  int w = 0;
#pragma unroll
  for (int j = 0; j < PER; ++j) {
    const int i = j * 32 + lane;
    const float m = fmaxf(fmaxf(fmaxf(e0[j].x, e0[j].y), fmaxf(e0[j].z, e0[j].w)),
                          fmaxf(fmaxf(e1[j].x, e1[j].y), fmaxf(e1[j].z, e1[j].w)));
    const bool keep = (i < n) && (m >= tau);
    const uint32_t kb = __ballot_sync(0xffffffffu, keep);
    if (keep) {
      const int pos = w + __popc(kb & ((1u << lane) - 1u));
      *reinterpret_cast<float4*>(ls + (size_t)pos * REC) = e0[j];
      *reinterpret_cast<float4*>(ls + (size_t)pos * REC + 4) = e1[j];
      reinterpret_cast<int32_t*>(ls)[(size_t)pos * REC + 8] = bs[j];
    }
    w += __popc(kb);
  }
  __syncwarp();
  return w;
}

// CL = CTAs per thread-block cluster (1 or 2).  With CL = 2 the two CTAs of a cluster work on two
// ADJACENT user tiles of the SAME item split in lock step: every item tile is fetched from L2 once
// per cluster — each CTA loads half of it and the TMA multicasts that half into both CTAs' shared
// memory — which halves the L2 -> SM traffic of the item table (the pass is L2-bandwidth bound
// otherwise).  NH = MMA organisation of an item tile (1: one N=256 wgmma chain; 2: two N=128 chains into
// separate accumulators, the epilogue of the first runs while the tensor core computes the second;
// 3: the same two N=128 groups pipelined across item tiles, so every half-tile epilogue of the main
// pass runs while the tensor core computes the other half, see the main pass).
// EPI = record stores of a hot 64-column step: 3 divergent per-group branches (the quad maximum by
// shuffles), 5 quad masks (one bit per (group, row) slot, one warp-uniform branch per slot).
//
// Threads: warpgroups 0 and 1 issue the wgmma of user rows [64 g, 64 g + 64) of the tile and run the
// epilogue on the accumulator registers; one lane of warpgroup 2 is the TMA producer.  In the m64nN fragment, lane
// (4 quad + tq) of warp w holds rows 16 w + quad and 16 w + quad + 8, columns 8 j + 2 tq + {0, 1}:
// the 8 columns of a group are spread over the 4 lanes of a quad, which write the 48-byte record
// together (8 bytes each, the id from lane tq = 0).
// Lane tq of a quad also owns one (row, list) pair — row quad + 8 (tq >> 1), list tq & 1 — for
// the warp-wide bookkeeping (compaction votes, list lengths, pre-pass maxima).
template <class T>
__device__ __forceinline__ T sel22(T const (&c)[2][2], int rs, int j) {
  return rs ? (j ? c[1][1] : c[1][0]) : (j ? c[0][1] : c[0][0]);
}
template <class T>
__device__ __forceinline__ void set22(T (&c)[2][2], int rs, int j, T v) {
  if (rs) { if (j) c[1][1] = v; else c[1][0] = v; } else { if (j) c[0][1] = v; else c[0][0] = v; }
}

template <bool PRE, int EPI, int CL, int NH>
__global__ void __launch_bounds__(SWEEP_THREADS, 1)
sweep_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
             const __grid_constant__ CUtensorMap tmBh, const SweepParams p) {
  extern __shared__ uint8_t smem_raw[];
  // 1024-byte alignment for SWIZZLE_128B tiles
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  uint8_t* smemA = smem;                                  // KB * 16 KB
  uint8_t* smemB = smem + (size_t)p.KB * A_KB_BYTES;      // nstage * KB * 32 KB
  SweepSmem* ss = (SweepSmem*)(smemB + (size_t)p.nstage * (p.kb_stages ? 1 : p.KB) * B_KB_BYTES);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  // work units: (item split, user tile); a cluster takes CL adjacent user tiles of one split
  const int crank = CL > 1 ? (int)ptx::cluster_ctarank() : 0;
  const int cid = (int)blockIdx.x / CL, n_clusters = (int)gridDim.x / CL;
  const int m_groups = p.m_tiles / CL;                    // host guarantees m_tiles % CL == 0
  const int n_units = m_groups * p.n_splits;              // units per cluster-rank
  const int STRIDE = PRE ? p.pre_stride : 1;
  constexpr uint16_t CL_MASK = (uint16_t)((1u << CL) - 1u);

  if (threadIdx.x == 0) {
    // a shared-memory stage is written by the multicasts of all CL producers and may be refilled only
    // when every consumer warp of all CL CTAs has finished its MMAs on it
    for (int s = 0; s < p.nstage; ++s) {
      ptx::mbar_init(&ss->full[s], 1);
      ptx::mbar_init(&ss->empty[s], SWEEP_CONSUMER_WARPS * CL);
    }
    ptx::mbar_init(&ss->a_full, 1);
    ptx::mbar_init(&ss->a_empty, SWEEP_CONSUMER_WARPS);
    ptx::fence_barrier_init();
    ptx::prefetch_tensormap(&tmA);
    ptx::prefetch_tensormap(&tmB);
  }
  __syncthreads();
  if (CL > 1) ptx::cluster_sync_all();     // the peer's barriers exist before anything is multicast to them

  if (warp >= WARP_TMA) {
    ptx::setmaxnreg_dec<SWEEP_PRODUCER_REGS>();
    // ===================== TMA producer (one lane of the last warpgroup) =====================
    if (warp == WARP_TMA && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      uint32_t uiter = 0;
      for (int unit = cid; unit < n_units; unit += n_clusters, ++uiter) {
        const int split = unit / m_groups, m = (unit % m_groups) * CL + crank;
        const int t0 = split * p.tiles_per_split;
        const int t1 = min(t0 + p.tiles_per_split, p.total_tiles);
        ptx::mbar_wait_hint(&ss->a_empty, (uiter & 1) ^ 1, p.hint_ns);
        ptx::mbar_arrive_expect_tx(&ss->a_full, (uint32_t)(p.KB * A_KB_BYTES));
        for (int kb = 0; kb < p.KB; ++kb)
          ptx::tma_load_2d(smemA + (size_t)kb * A_KB_BYTES, &tmA, &ss->a_full, kb * KBLK, m * TM);
        for (int t = t0; t < t1; t += STRIDE) {
          if (p.kb_stages) {
            // wide embeddings (d_pad > 128): one ring stage per 64-wide k-block, consumed block by block
            for (int kb = 0; kb < p.KB; ++kb) {
              ptx::mbar_wait_hint(&ss->empty[stage], phase ^ 1, p.hint_ns);
              ptx::mbar_arrive_expect_tx(&ss->full[stage], (uint32_t)B_KB_BYTES);
              uint8_t* dst = smemB + (size_t)stage * B_KB_BYTES;
              if (CL == 1) {
                ptx::tma_load_2d(dst, &tmB, &ss->full[stage], kb * KBLK, t * TN);
              } else {
                ptx::tma_load_2d_multicast(dst + (size_t)crank * (B_KB_BYTES / CL), &tmBh, &ss->full[stage], kb * KBLK,
                                           t * TN + crank * (TN / CL), CL_MASK);
              }
              if (++stage == p.nstage) { stage = 0; phase ^= 1; }
            }
            continue;
          }
          ptx::mbar_wait_hint(&ss->empty[stage], phase ^ 1, p.hint_ns);
          // the whole tile lands in THIS CTA's stage: its own share plus the peers' multicast shares
          ptx::mbar_arrive_expect_tx(&ss->full[stage], (uint32_t)(p.KB * B_KB_BYTES));
          uint8_t* dst = smemB + (size_t)stage * p.KB * B_KB_BYTES;
          for (int kb = 0; kb < p.KB; ++kb) {
            if (CL == 1) {
              ptx::tma_load_2d(dst + (size_t)kb * B_KB_BYTES, &tmB, &ss->full[stage], kb * KBLK, t * TN);
            } else {   // rows [crank * TN/CL, +TN/CL) of the tile, delivered to every CTA of the cluster
              ptx::tma_load_2d_multicast(dst + (size_t)kb * B_KB_BYTES + (size_t)crank * (B_KB_BYTES / CL), &tmBh,
                                         &ss->full[stage], kb * KBLK, t * TN + crank * (TN / CL), CL_MASK);
            }
          }
          if (++stage == p.nstage) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    ptx::setmaxnreg_inc<SWEEP_CONSUMER_REGS>();
    // ===================== MMA + epilogue: 2 warpgroups x 64 user rows ==========
    constexpr bool PIPE = NH == 3;          // two N=128 groups pipelined across item tiles (main pass only)
    static_assert(!(PRE && PIPE), "the pre-pass runs the unpipelined two-group organisation");
    constexpr int NG = NH == 1 ? 1 : 2;     // MMA groups (accumulators) per item tile
    constexpr int NC = TN / NG;             // accumulator columns per MMA group
    const int g = warp >> 2;
    const int quad = lane >> 2, tq = lane & 3;
    const int my_rs = tq >> 1, my_j = tq & 1;          // the (row, list) pair this lane reports
    const int trow0 = 64 * g + 16 * (warp & 3) + quad;   // rows trow0 and trow0 + 8 of the tile
    const float pinf = __int_as_float(0x7f800000);
    const float ninf = __int_as_float(0xff800000);
    const uint32_t a_addr = ptx::smem_u32(smemA) + (uint32_t)(g * 64 * KBLK * 2);
    const uint32_t b_addr = ptx::smem_u32(smemB);
    float acc[NG][NC / 2];
    int stage = 0;
    uint32_t phase = 0;

    // hand a stage back: one arrival per consumer warp on the stage's barrier in every CTA of the cluster
    auto release = [&]() {
      __syncwarp();
      if (lane == 0) {
        if (CL == 1) ptx::mbar_arrive(&ss->empty[stage]);
        else
#pragma unroll
          for (int c = 0; c < CL; ++c) ptx::mbar_arrive_cluster(&ss->empty[stage], (uint32_t)c);
      }
      if (++stage == p.nstage) { stage = 0; phase ^= 1; }
    };
    // the four k16 MMAs of one 64-wide k-block; the first k-block of a tile starts the accumulator
    auto mma_kblock = [&](float (&d)[NC / 2], uint64_t da, uint64_t db, bool first) {
      if (first) {
        if (NG == 1) ptx::wgmma_f16_n256_first(*reinterpret_cast<float(*)[128]>(&d[0]), da, db);
        else ptx::wgmma_f16_n128_first(*reinterpret_cast<float(*)[64]>(&d[0]), da, db);
      }
#pragma unroll
      for (int k4 = first ? 1 : 0; k4 < KBLK / 16; ++k4) {
        // advance 16 fp16 = 32 bytes inside the 128-byte swizzled row: +2 in the >>4 field
        if (NG == 1) ptx::wgmma_f16_n256(*reinterpret_cast<float(*)[128]>(&d[0]), da + 2 * k4, db + 2 * k4);
        else ptx::wgmma_f16_n128(*reinterpret_cast<float(*)[64]>(&d[0]), da + 2 * k4, db + 2 * k4);
      }
    };
    // MMAs of column group hh of the item tile in (whole-tile) stage st, as one commit group
    auto issue_group = [&](float (&d)[NC / 2], int hh, int st) {
      const uint32_t b_hh = b_addr + (uint32_t)(st * p.KB * B_KB_BYTES + hh * NC * KBLK * 2);
      mma_kblock(d, ptx::wgmma_desc_sw128_kmajor(a_addr), ptx::wgmma_desc_sw128_kmajor(b_hh), true);
#pragma unroll 1
      for (int kb = 1; kb < p.KB; ++kb)
        mma_kblock(d, ptx::wgmma_desc_sw128_kmajor(a_addr + (uint32_t)(kb * A_KB_BYTES)),
                   ptx::wgmma_desc_sw128_kmajor(b_hh + (uint32_t)(kb * B_KB_BYTES)), false);
      ptx::wgmma_commit();
    };
    // every MMA group of one item tile; `epi(acc_group, column offset)` runs as soon as its group is done
    auto tile_mma = [&](auto&& epi) {
      if (NH == 1 && p.kb_stages) {
        // k-block stages: the accumulator of the tile is built block by block, every stage is handed back
        // as soon as its MMAs are complete
        auto kblock_stage = [&](int kb, bool first) {
          ptx::mbar_wait_hint(&ss->full[stage], phase, p.hint_ns);
          ptx::wgmma_fence();
          mma_kblock(acc[0], ptx::wgmma_desc_sw128_kmajor(a_addr + (uint32_t)(kb * A_KB_BYTES)),
                     ptx::wgmma_desc_sw128_kmajor(b_addr + (uint32_t)(stage * B_KB_BYTES)), first);
          ptx::wgmma_commit();
          ptx::wgmma_wait<0>(acc[0]);
          release();
        };
        kblock_stage(0, true);
#pragma unroll 1
        for (int kb = 1; kb < p.KB; ++kb) kblock_stage(kb, false);
        epi(acc[0], std::integral_constant<int, 0>{});
        return;
      }
      ptx::mbar_wait_hint(&ss->full[stage], phase, p.hint_ns);
      ptx::wgmma_fence();
#pragma unroll
      for (int hh = 0; hh < NG; ++hh) issue_group(acc[hh], hh, stage);
      if (NG == 2) {
        ptx::wgmma_wait<1>(acc[0]);
        epi(acc[0], std::integral_constant<int, 0>{});
        ptx::wgmma_wait<0>(acc[NG - 1]);
        release();
        epi(acc[NG - 1], std::integral_constant<int, NC>{});
      } else {
        ptx::wgmma_wait<0>(acc[0]);
        release();
        epi(acc[0], std::integral_constant<int, 0>{});
      }
    };

    uint32_t uiter = 0;
    for (int unit = cid; unit < n_units; unit += n_clusters, ++uiter) {
      const int split = unit / m_groups, m = (unit % m_groups) * CL + crank;
      const int t0 = split * p.tiles_per_split;
      const int t1 = min(t0 + p.tiles_per_split, p.total_tiles);
      const int grow0 = m * TM + trow0;                 // global rows grow0 (rs = 0) and grow0 + 8 (rs = 1)
      const int list_base = split * 2;                  // list j = column half j of the tile
      ptx::mbar_wait_hint(&ss->a_full, uiter & 1, p.hint_ns);

      if (PRE) {
        // ---- pre-pass: per sampled tile the maximum coarse score of each row and 128-column half ----
        float* bm = p.blockmax + (int64_t)(list_base + my_j) * p.n_pre_tiles * p.B_pad + grow0 + 8 * my_rs;
        int ti = 0;
        for (int t = t0; t < t1; t += STRIDE, ++ti) {
          float mx[2][2] = {{ninf, ninf}, {ninf, ninf}};
          tile_mma([&](auto& d, auto c0) {
            constexpr int COL0 = decltype(c0)::value;
#pragma unroll
            for (int jj = 0; jj < NC / 8; ++jj) {
              const int j = (COL0 + 8 * jj) >= TN / 2;
#pragma unroll
              for (int rs = 0; rs < 2; ++rs) {
                const float v = fmaxf(d[4 * jj + 2 * rs], d[4 * jj + 2 * rs + 1]);
                if (j) mx[rs][1] = fmaxf(mx[rs][1], v); else mx[rs][0] = fmaxf(mx[rs][0], v);
              }
            }
          });
#pragma unroll
          for (int rs = 0; rs < 2; ++rs)
#pragma unroll
            for (int j = 0; j < 2; ++j) {
              mx[rs][j] = fmaxf(mx[rs][j], __shfl_xor_sync(0xffffffffu, mx[rs][j], 1));
              mx[rs][j] = fmaxf(mx[rs][j], __shfl_xor_sync(0xffffffffu, mx[rs][j], 2));
            }
          float tm = my_rs ? (my_j ? mx[1][1] : mx[1][0]) : (my_j ? mx[0][1] : mx[0][0]);
          // tiles that contain zero-padded item rows would bias the estimate: drop them
          if ((int64_t)(t + 1) * TN > p.N) tm = ninf;
          bm[(int64_t)ti * p.B_pad] = tm;
        }
        for (; ti < p.n_pre_tiles; ++ti) bm[(int64_t)ti * p.B_pad] = ninf;   // short last split
      } else {
        // ---- main pass ----
        float tau[2];
        int n_counted[2][2] = {{0, 0}, {0, 0}};
        // lp(rs, j): first record of the (row, list), computed rather than held (registers are scarce);
        // rp: where its next record goes (records = (rp - lp) / REC)
        float* rp[2][2];
        const int64_t cap_words = (int64_t)p.capg * REC;
        auto lp = [&](int rs, int j) {
          return p.cand_r + ((int64_t)(list_base + j) * p.B_pad + grow0 + 8 * rs) * cap_words;
        };
#pragma unroll
        for (int rs = 0; rs < 2; ++rs) {
          const int grow = grow0 + 8 * rs;
          tau[rs] = p.meta[grow].active ? ninf : pinf;
          if (tau[rs] == ninf) {  // speculative start value (guess_kernel) / bounds published by other lists
            const uint32_t gk = __ldcg(p.row_tau_key + grow);
            if (gk != 0u) tau[rs] = key_to_float(gk);
          }
          if (p.ablate >= 1) tau[rs] = pinf;   // diagnostics: nothing is ever collected (cold path only)
#pragma unroll
          for (int j = 0; j < 2; ++j) rp[rs][j] = lp(rs, j);
        }
        auto records = [&](int rs, int j) { return (int)(sel22(rp, rs, j) - lp(rs, j)) / REC; };

        // Zero-padded item rows of the last tile (ids >= N, coarse score exactly 0) may be collected when
        // tau <= 0; compact_row and finalize_kernel ignore ids >= N, so the sweep needs no tail code.
        bool hot = false;   // warp-uniform: some step of the current tile stored records
        // epilogue of the MMA group at column offset c0 of item tile t: records of its hot groups
        auto epilogue = [&](auto& d, auto c0, int t) {
            constexpr int COL0 = decltype(c0)::value;
            if (p.ablate >= 2) return;   // diagnostics: MMAs and stage releases only
#pragma unroll
            for (int s = 0; s < NC / STEP; ++s) {
              // one warp vote per 64-column step: a cold step (the common case) costs its max tree only.
              // pm = the lane's maximum of each (group, row) slot; the group maximum reaches tau exactly
              // when the pair maximum of some lane of the quad does
              float pm[8][2];
              float m0 = ninf, m1 = ninf;
#pragma unroll
              for (int jl = 0; jl < 8; ++jl) {
                const int jj = 8 * s + jl;
                pm[jl][0] = fmaxf(d[4 * jj + 0], d[4 * jj + 1]);
                pm[jl][1] = fmaxf(d[4 * jj + 2], d[4 * jj + 3]);
                m0 = fmaxf(m0, pm[jl][0]);
                m1 = fmaxf(m1, pm[jl][1]);
              }
              if (!__any_sync(0xffffffffu, m0 >= tau[0] || m1 >= tau[1])) continue;
              hot = true;   // some slot of the warp reaches tau: records are stored
              // Slots are visited group by group, row by row, so every list receives its records in
              // column order whichever variant runs.
              if (EPI == 5) {
                // one ballot per (group, row) slot: bits 4 q .. 4 q + 3 are the lanes of quad q, so the slot
                // is live in the warp iff its ballot is non-zero, and quad q stores iff its nibble is
                uint32_t bal[8][2];
#pragma unroll
                for (int jl = 0; jl < 8; ++jl)
#pragma unroll
                  for (int rs = 0; rs < 2; ++rs) bal[jl][rs] = __ballot_sync(0xffffffffu, pm[jl][rs] >= tau[rs]);
                const uint32_t qmask = 0xfu << (4 * quad);
                // two-level slot tests: a hot step usually holds one or two slots, so test the four
                // slots of a group pair only when the pair has one (4 + 4 uniform tests instead of 16)
#pragma unroll
                for (int jp = 0; jp < 4; ++jp) {
                  // warp-uniform: no slot in groups 2 jp, 2 jp + 1
                  if (!(bal[2 * jp][0] | bal[2 * jp][1] | bal[2 * jp + 1][0] | bal[2 * jp + 1][1])) continue;
#pragma unroll
                for (int jl = 2 * jp; jl < 2 * jp + 2; ++jl) {
                  const int jj = 8 * s + jl;
                  const int col = COL0 + 8 * jj;
#pragma unroll
                  for (int rs = 0; rs < 2; ++rs) {
                    if (!bal[jl][rs]) continue;   // warp-uniform: no quad of the warp has this slot
                    const uint32_t mine = bal[jl][rs] & qmask;
                    float*& r = col >= TN / 2 ? rp[rs][1] : rp[rs][0];
                    // predicated stores (not a branch on the lane's bit, which the compiler would merge
                    // with the uniform test above into one divergent branch per slot)
                    asm volatile(
                        "{\n\t.reg .pred p, q;\n\t"
                        "setp.ne.u32 p, %0, 0;\n\t"
                        "setp.eq.and.u32 q, %5, 0, p;\n\t"
                        "@p st.global.v2.f32 [%1], {%2, %3};\n\t"
                        "@q st.global.b32 [%4], %6;\n\t}"
                        ::"r"(mine), "l"(r + 2 * tq), "f"(d[4 * jj + 2 * rs]), "f"(d[4 * jj + 2 * rs + 1]),
                        "l"(r + 8), "r"(tq), "r"(t * TN + col)
                        : "memory");
                    r += mine ? REC : 0;
                  }
                }
                }
              } else {
#pragma unroll
                for (int jl = 0; jl < 8; ++jl) {
                  const int jj = 8 * s + jl;
                  const int col = COL0 + 8 * jj;
#pragma unroll
                  for (int rs = 0; rs < 2; ++rs) {
                    float gm = pm[jl][rs];
                    gm = fmaxf(gm, __shfl_xor_sync(0xffffffffu, gm, 1));
                    gm = fmaxf(gm, __shfl_xor_sync(0xffffffffu, gm, 2));
                    if (gm >= tau[rs]) {
                      float*& r = col >= TN / 2 ? rp[rs][1] : rp[rs][0];
                      *reinterpret_cast<float2*>(r + 2 * tq) = make_float2(d[4 * jj + 2 * rs], d[4 * jj + 2 * rs + 1]);
                      if (tq == 0) reinterpret_cast<int32_t*>(r)[8] = t * TN + col;
                      r += REC;
                    }
                  }
                }
              }
            }
        };
        // the lane's (row, list) is due for a compaction once it holds `extra` more records
        auto compaction_due = [&](int extra) {
          const int mc = records(my_rs, my_j) + extra, mn = sel22(n_counted, my_rs, my_j);
          return (mc - mn > p.trig) || (mc > p.capg - 24);
        };
        // one overflow / compaction check per TILE, after all of the tile's records
        auto check = [&]() {
          if (!hot) return;
          const int mc = records(my_rs, my_j), mn = sel22(n_counted, my_rs, my_j);
          uint32_t need = __ballot_sync(0xffffffffu, compaction_due(0));
          while (need) {
            const int src = __ffs(need) - 1;
            need &= need - 1;
            const int s_cnt = __shfl_sync(0xffffffffu, mc, src);
            const int s_cntd = __shfl_sync(0xffffffffu, mn, src);
            const float s_tau = __shfl_sync(0xffffffffu, my_rs ? tau[1] : tau[0], src);
            const int sq = src >> 2, srs = (src >> 1) & 1, sj = src & 1;
            const int sgrow = grow0 - quad + sq + 8 * srs;
            const RowMeta sm = p.meta[sgrow];
            float new_tau;
            const int w = compact_row(p.cand_r + ((int64_t)(list_base + sj) * p.B_pad + sgrow) * cap_words, s_cnt, s_cntd,
                                      sm.k_row, sm.eps2, sm.R, s_tau, p.ghist + (int64_t)sgrow * NB, lane, (int32_t)p.N,
                                      &new_tau);
            if (quad == sq) {
              set22(rp, srs, sj, lp(srs, sj) + (size_t)w * REC);
              set22(n_counted, srs, sj, w);
              // also pick up what other lists of this row published meanwhile
              float nt = fmaxf(new_tau, key_to_float(max(__ldcg(p.row_tau_key + sgrow), 1u)));
              if (lane == src) atomicMax(p.row_tau_key + sgrow, float_to_key(new_tau));
              if (w > p.capg - 32) {  // too many near-ties to bound: hand the row to the exact path
                nt = pinf;
                set22(rp, srs, sj, lp(srs, sj));
                set22(n_counted, srs, sj, 0);
                if (lane == src) p.row_status[sgrow] = 1;
              }
              if (srs) tau[1] = nt; else tau[0] = nt;
            }
          }
        };

        if constexpr (!PIPE) {
          for (int t = t0; t < t1; ++t) {
            hot = false;
            tile_mma([&](auto& d, auto c0) { epilogue(d, c0, t); });
            check();
          }
        } else {
          // Two N=128 groups per tile (G0 / G1 = columns [0, 128) / [128, 256); group h feeds list h only,
          // so every list still receives its records in column order), pipelined across the unit's tiles.
          // Steady state of tile t:
          //   wait full(t+1); issue G0(t+1) | wait<1>: G1(t) done, release stage(t) | epilogue G1(t)
          //   issue G1(t+1) | wait<1>: G0(t+1) done | epilogue G0(t+1)
          // so each half-tile epilogue runs while the tensor core computes the other half.
          //  - Every group is its own commit group and its first MMA writes the accumulator, so wait<1>
          //    means "all but the newest group are complete".
          //  - Two ring stages are held at once: stage(t) until G1(t) completes, then stage(t+1).
          //    release() hands stage(t) back exactly once per warp, to every CTA of the cluster, right after
          //    G1(t) completes (nstage >= 2 whenever a stage holds a whole tile, d_pad <= 128).
          //  - compact_row is __noinline__ and register-hungry: no wgmma may be in flight and no accumulator
          //    live across it (ptxas would serialise every wgmma of the kernel, or spill).  So before G0(t+1)
          //    is issued the warpgroup decides from the worst case whether the check of tile t can compact:
          //    list 0 has all of tile t's records, list 1 gets at most TN / 2 / GW = 16 more.  If it can
          //    (rare), the pipeline drains (wait<0>, epilogue G1(t), check) and restarts at t+1; otherwise
          //    the check provably finds nothing to do and is skipped.  Either way it sits where the
          //    unpipelined organisations have it, after all of tile t's records and before any of t+1's, so
          //    lists and thresholds evolve exactly as there.  The vote is warpgroup-wide (named barrier 1 + g)
          //    because wgmma issue and wait are warpgroup-collective.
          //  - The user tile changes at unit boundaries: the last tile of a unit always drains, so nothing
          //    is issued into the next unit and every MMA of the unit is complete before a_empty.
          constexpr int MAX_TILE_RECORDS = TN / 2 / GW;   // records one tile adds to one (row, list)
          // (every split has at least one tile)
          ptx::mbar_wait_hint(&ss->full[stage], phase, p.hint_ns);
          ptx::wgmma_fence();
          issue_group(acc[0], 0, stage);
          // the loop leaves only through the drain branch (after wait<0>): ptxas then sees that no group is
          // pending at the end of the unit (otherwise it serialises every wgmma of the kernel, C7514)
          for (int t = t0;; ++t) {
            // here G0(t) is issued into `stage`, no other group is pending
            ptx::wgmma_fence();
            issue_group(acc[1], 1, stage);
            ptx::wgmma_wait<1>(acc[0]);
            hot = false;
            epilogue(acc[0], std::integral_constant<int, 0>{}, t);
            const bool due = compaction_due(my_j ? MAX_TILE_RECORDS : 0);
            const bool drain = t + 1 == t1 ||
                __any_sync(0xffffffffu, g ? ptx::named_bar_any<2, 128>(due) : ptx::named_bar_any<1, 128>(due));
            if (!drain) {
              const int nst = stage + 1 == p.nstage ? 0 : stage + 1;
              ptx::mbar_wait_hint(&ss->full[nst], nst ? phase : phase ^ 1, p.hint_ns);
              ptx::wgmma_fence();
              issue_group(acc[0], 0, nst);
              ptx::wgmma_wait<1>(acc[1]);
              release();
              epilogue(acc[1], std::integral_constant<int, NC>{}, t);
            } else {
              ptx::wgmma_wait<0>(acc[1]);
              release();
              epilogue(acc[1], std::integral_constant<int, NC>{}, t);
              check();
              if (t + 1 == t1) break;
              // restart the pipeline at t + 1
              ptx::mbar_wait_hint(&ss->full[stage], phase, p.hint_ns);
              ptx::wgmma_fence();
              issue_group(acc[0], 0, stage);
            }
          }
        }
        p.cand_cnt[(int64_t)(list_base + my_j) * p.B_pad + grow0 + 8 * my_rs] = records(my_rs, my_j);
      }
      // the user tile is reusable once every consumer warp's last MMA of the unit is complete
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&ss->a_empty);
    }
  }
  __syncthreads();
  if (CL > 1) ptx::cluster_sync_all();     // no CTA leaves while a peer may still multicast to it
}

// ------------------------------------------------------------------------------------------
// guess kernel: speculative threshold = pre_k-th largest sampled block maximum of the row.
// One CTA per 32 consecutive rows: lane = row, the 8 warps stride the block index, so every load
// of blockmax[i][row0..row0+31] is one coalesced 128-byte request; per-row 4 x 8-bit radix select
// on shared-memory histograms.
// ------------------------------------------------------------------------------------------
constexpr int GUESS_THREADS = 256;
__global__ void __launch_bounds__(GUESS_THREADS)
guess_kernel(const float* __restrict__ blockmax, int n_vals /* lists * n_pre_tiles */, int B_pad,
             const RowMeta* __restrict__ meta, uint32_t* __restrict__ row_tau_key,
             uint32_t* __restrict__ guess_key) {
  __shared__ uint32_t hist[32][256 + 1];      // +1: rows land in different banks
  __shared__ uint32_t s_prefix[32], s_krem[32], s_ok[32];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int row = blockIdx.x * 32 + lane;
  const RowMeta m = meta[row];
  if (wid == 0) { s_prefix[lane] = 0; s_krem[lane] = (uint32_t)m.pre_k; s_ok[lane] = m.active != 0; }
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    for (int i = threadIdx.x; i < 32 * 257; i += GUESS_THREADS) (&hist[0][0])[i] = 0;
    __syncthreads();
    const uint32_t prefix = s_prefix[lane];
    for (int i = wid; i < n_vals; i += GUESS_THREADS / 32) {
      const float v = blockmax[(int64_t)i * B_pad + row];
      const uint32_t key = float_to_key(v);
      if (v > -3.0e38f && (pass == 0 || (key >> (shift + 8)) == prefix))
        atomicAdd(&hist[lane][(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    // digit resolution: warp w resolves rows w, w+8, w+16, w+24; lane l owns bins [8l, 8l+8)
    for (int rr = wid; rr < 32; rr += GUESS_THREADS / 32) {
      uint32_t mine[8], tot = 0;
#pragma unroll
      for (int b = 0; b < 8; ++b) { mine[b] = hist[rr][lane * 8 + b]; tot += mine[b]; }
      uint32_t incl = tot;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_down_sync(0xffffffffu, incl, o);
        if (lane + o < 32) incl += t;
      }
      const uint32_t excl = incl - tot;
      const uint32_t krem = s_krem[rr];
      const uint32_t total = __shfl_sync(0xffffffffu, incl, 0);
      if (excl < krem && krem <= incl) {
        uint32_t c = excl;
#pragma unroll
        for (int b = 7; b >= 0; --b) {
          if (c + mine[b] >= krem) {
            s_prefix[rr] = (s_prefix[rr] << 8) | (uint32_t)(lane * 8 + b);
            s_krem[rr] = krem - c;
            break;
          }
          c += mine[b];
        }
      }
      if (lane == 0 && total < krem) s_ok[rr] = 0;   // fewer than pre_k sampled blocks: no speculation
    }
    __syncthreads();
  }
  if (wid == 0) {
    const uint32_t key = s_ok[lane] ? s_prefix[lane] : 0u;   // 0 = no speculation for this row
    row_tau_key[row] = key;
    guess_key[row] = key;
  }
}

// ------------------------------------------------------------------------------------------
// finalize: one warp per user row (finalize_warp_kernel), rows outside its envelope deferred to
// one CTA per row (finalize_kernel)
// ------------------------------------------------------------------------------------------
struct FinalizeParams {
  int64_t B, N;
  int32_t B_pad, n_lists, K, d, capg;
  int32_t defer_all;               // diagnostics (b200_recommend_embed_debug level 3): every row takes finalize_kernel
  const RowMeta* meta;
  const int32_t* row_status;       // [B_pad] status after the sweep (0, or 1 = list overflow)
  int32_t* out_status;             // [B] final row_status of the call, written once per row by one of the kernels
  int32_t* defer_count;            // rows handed from finalize_warp_kernel to finalize_kernel ...
  int32_t* defer_rows;             // ... and their indices [B_pad]
  int32_t* flagged;                // rows of the call whose final status is not 0 (only finalize_kernel flags)
  const uint32_t* row_tau_key;     // [B_pad] final threshold of the row (speculative start or rigorous raises)
  const uint32_t* tau_guess_key;   // [B_pad] speculative threshold used by the main pass (0 = none)
  const float* cand_r;
  const int32_t* cand_cnt;
  const float* U; int64_t ldu;
  const float* I; int64_t ldi;
  const int64_t* user_ids;
  const int64_t* indptr; const int32_t* idx;
  int64_t* out_ids;    // [B, K]
  float* out_scores;   // [B, K] or null
};

// not inlined: inside finalize_kernel's row loop ptxas spills it
__device__ __noinline__ void finalize_row(const FinalizeParams& p, const int64_t row) {
  __shared__ uint32_t hist[256];
  __shared__ uint32_t s_prefix, s_krem;
  __shared__ uint32_t s_wtot[FIN_THREADS / 32];
  __shared__ int s_nu, s_nc;
  __shared__ float u_s[MAXU];                      // union of the lists: coarse scores ...
  __shared__ int32_t u_id[MAXU];                   // ... and item ids (later: the candidate ids)
  __shared__ unsigned long long c_sort[MAXC];      // first the consumed hash set (int32 x 4096), then sort keys
  __shared__ float urow[MAX_KB * KBLK];
  int32_t* htab = reinterpret_cast<int32_t*>(c_sort);
  const int tid = threadIdx.x;
  int64_t* oid = p.out_ids + row * p.K;
  float* osc = p.out_scores ? p.out_scores + row * p.K : nullptr;
  const RowMeta meta = p.meta[row];
  // row_status codes (non-zero = re-run on the exact path): 1 sweep overflow, 2 too few collected,
  // 3 failed speculation, 4 candidate set outside [K, MAXC], 5 capped row not provable
  auto give_up = [&](int code) {   // code 0 only for a row the sweep flagged: the status is never 0
    if (tid == 0) {
      p.out_status[row] = code ? code : p.row_status[row];
      atomicAdd(p.flagged, 1);
    }
    for (int i = tid; i < p.K; i += FIN_THREADS) { oid[i] = -1; if (osc) osc[i] = 0.f; }
  };
  if (p.row_status[row] != 0) { give_up(0); return; }
  // ---- gather: every element of every group record that is >= the row's final threshold.
  // (every exact top-k_row item has coarse >= c_k - 2 eps >= that threshold, see the header)
  const uint32_t tk = p.row_tau_key[row];
  const float low = tk ? key_to_float(tk) : __int_as_float(0xff800000);
  if (tid == 0) { s_nu = 0; s_nc = 0; }
  // list lengths first (one parallel round of loads), their exclusive prefix, then ONE parallel round
  // over all group records of the row: thread <-> record, so the number of dependent global round
  // trips does not grow with the number of lists
  int* s_cnt = reinterpret_cast<int*>(c_sort);          // c_sort is free until the hash set is built
  int* s_off = s_cnt + p.n_lists;                       // [n_lists + 1]
  for (int s = tid; s < p.n_lists; s += FIN_THREADS) s_cnt[s] = p.cand_cnt[(int64_t)s * p.B_pad + row];
  __syncthreads();
  if (tid < 32) {   // warp 0: chunked scan of the list lengths
    const int per = (p.n_lists + 31) / 32;
    const int b = min(tid * per, p.n_lists), e = min(b + per, p.n_lists);
    int sum = 0;
    for (int s = b; s < e; ++s) sum += s_cnt[s];
    int incl = sum;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (tid >= o) incl += t;
    }
    int run = incl - sum;
    for (int s = b; s < e; ++s) { s_off[s] = run; run += s_cnt[s]; }
    if (tid == 31) s_off[p.n_lists] = incl;
  }
  __syncthreads();
  {
    const int lane = tid & 31;
    const int total = s_off[p.n_lists];
    constexpr int UN = 3;                                // records in flight per thread
    for (int g0 = 0; g0 < total; g0 += FIN_THREADS * UN) {   // block-uniform trip count
      float4 a[UN], b[UN];
      int base[UN];
      bool ok[UN];
#pragma unroll
      for (int q = 0; q < UN; ++q) {
        const int g = g0 + q * FIN_THREADS + tid;
        ok[q] = g < total;
        a[q] = b[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        base[q] = 0;
        if (ok[q]) {
          int lo = 0, hi = p.n_lists - 1;                // last list whose first record is <= g
          while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (s_off[mid] <= g) lo = mid; else hi = mid - 1;
          }
          const int j = g - s_off[lo];
          const int64_t slot = (int64_t)lo * p.B_pad + row;
          const float4* ls = reinterpret_cast<const float4*>(p.cand_r + (slot * (int64_t)p.capg + j) * REC);
          a[q] = __ldcs(ls);
          b[q] = __ldcs(ls + 1);
          base[q] = __ldcs(reinterpret_cast<const int32_t*>(ls + 2));
        }
      }
#pragma unroll
      for (int q = 0; q < UN; ++q) {
        const float v[8] = {a[q].x, a[q].y, a[q].z, a[q].w, b[q].x, b[q].y, b[q].z, b[q].w};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const bool hit = ok[q] && v[e] >= low && (int64_t)(base[q] + e) < p.N;   // never a zero-padded item row
          const unsigned m = __ballot_sync(0xffffffffu, hit);
          if (m) {   // one shared-memory atomic per warp and element slot
            int pos0 = 0;
            if (lane == 0) pos0 = atomicAdd(&s_nu, __popc(m));
            pos0 = __shfl_sync(0xffffffffu, pos0, 0);
            const int pos = pos0 + __popc(m & ((1u << lane) - 1u));
            if (hit && pos < MAXU) { u_s[pos] = v[e]; u_id[pos] = base[q] + e; }
          }
        }
      }
    }
  }
  __syncthreads();
  const int nu = s_nu;
  if (nu < meta.k_row) { give_up(2); return; }
  const bool in_smem = nu <= MAXU;   // common case; otherwise (no speculation, small catalogue) stream from HBM
  // visit every collected element (score, id): from shared memory, or again from the lists
  auto for_each = [&](auto&& f) {
    if (in_smem) {
      for (int i = tid; i < nu; i += FIN_THREADS) f(u_s[i], u_id[i]);
    } else {
      for (int s = 0; s < p.n_lists; ++s) {
        const int64_t slot = (int64_t)s * p.B_pad + row;
        const int n = p.cand_cnt[slot];
        const float* ls = p.cand_r + slot * (int64_t)(p.capg * REC);
        for (int i = tid; i < n * GW; i += FIN_THREADS) {
          const float v = ls[(i / GW) * REC + (i % GW)];
          const int32_t id = reinterpret_cast<const int32_t*>(ls)[(i / GW) * REC + 8] + (i % GW);
          if (v >= low && (int64_t)id < p.N) f(v, id);
        }
      }
    }
  };
  // ---- exact k_row-th largest coarse score of the union (4 x 8-bit radix select)
  uint32_t prefix = 0, krem = (uint32_t)meta.k_row;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    hist[tid] = 0;
    __syncthreads();
    for_each([&](float v, int32_t) {
      const uint32_t key = float_to_key(v);
      if (pass == 0 || (key >> (shift + 8)) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
    });
    __syncthreads();
    {
      // parallel resolution of the digit: thread t owns bin t, suffix sums by warp scan + warp totals
      const int lane = tid & 31, wid = tid >> 5;
      const uint32_t v = hist[tid];
      uint32_t incl = v;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) {
        const uint32_t t = __shfl_down_sync(0xffffffffu, incl, o);
        if (lane + o < 32) incl += t;
      }
      if (lane == 0) s_wtot[wid] = incl;
      __syncthreads();
      uint32_t above = 0;
      for (int w2 = wid + 1; w2 < FIN_THREADS / 32; ++w2) above += s_wtot[w2];
      incl += above;                       // count in bins >= tid
      const uint32_t excl = incl - v;      // count in bins >  tid
      if (excl < krem && krem <= incl) {
        s_prefix = (prefix << 8) | (uint32_t)tid;
        s_krem = krem - excl;
      }
    }
    __syncthreads();
    prefix = s_prefix;
    krem = s_krem;
    __syncthreads();
  }
  const float thr = key_to_float(prefix) - meta.eps2;
  {
    // The main pass started from a speculative threshold: the lists are complete only above it.
    // Every exact top-k_row item has coarse >= thr, so the guess must not exceed thr.
    const uint32_t gk = p.tau_guess_key[row];
    if (gk != 0u && key_to_float(gk) > thr) { give_up(3); return; }
  }
  // ---- candidates: elements >= thr (ids only from here on)
  if (in_smem) {   // compact in place: read everything first, then write
    int my_keep[MAXU / FIN_THREADS];
#pragma unroll
    for (int t = 0; t < MAXU / FIN_THREADS; ++t) {
      const int i = tid + t * FIN_THREADS;
      my_keep[t] = (i < nu && u_s[i] >= thr) ? u_id[i] : -1;
    }
    __syncthreads();
#pragma unroll
    for (int t = 0; t < MAXU / FIN_THREADS; ++t) {
      if (my_keep[t] >= 0) {
        const int pos = atomicAdd(&s_nc, 1);
        if (pos < MAXC) u_id[pos] = my_keep[t];
      }
    }
  } else {
    __syncthreads();
    for_each([&](float v, int32_t id) {
      if (v >= thr) {
        const int pos = atomicAdd(&s_nc, 1);
        if (pos < MAXC) u_id[pos] = id;
      }
    });
  }
  for (int i = tid; i < 2 * MAXC; i += FIN_THREADS) htab[i] = -1;
  __syncthreads();
  const int nc = s_nc;
  int32_t* c_id = u_id;
  if (nc > MAXC || nc < p.K) { give_up(4); return; }  // cannot bound (dense near-ties) -> exact path
  const int64_t u = p.user_ids[row];
  // ---- consumed filter through a hash set of candidate ids
  if (meta.apply) {
    for (int i = tid; i < nc; i += FIN_THREADS) {
      uint32_t h = ((uint32_t)c_id[i] * 2654435761u) & (2 * MAXC - 1);
      while (atomicCAS(&htab[h], -1, i) != -1) h = (h + 1) & (2 * MAXC - 1);
    }
    __syncthreads();
    const int64_t beg = p.indptr[u], end = p.indptr[u + 1];
    for (int64_t j = beg + tid; j < end; j += FIN_THREADS) {
      const int32_t it = p.idx[j];
      uint32_t h = ((uint32_t)it * 2654435761u) & (2 * MAXC - 1);
      while (true) {
        const int32_t e = htab[h];
        if (e < 0) break;
        if (c_id[e] == it || c_id[e] == ~it) { c_id[e] = ~it; break; }  // mark removed (negative)
        h = (h + 1) & (2 * MAXC - 1);
      }
    }
  }
  for (int k = tid; k < p.d; k += FIN_THREADS) urow[k] = __ldg(p.U + u * p.ldu + k);
  __syncthreads();   // the hash set is dead from here on: its storage becomes the sort buffer
  // ---- exact fp32 re-score: acc = fma(u[k], i[k], acc), k ascending
  const bool vec4 = (p.d % 4 == 0) && (p.ldi % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.I) & 15) == 0);
  int P = 1;
  while (P < nc) P <<= 1;
  unsigned long long mine[MAXC / FIN_THREADS];
#pragma unroll
  for (int t = 0; t < MAXC / FIN_THREADS; ++t) {
    const int i = tid + t * FIN_THREADS;
    unsigned long long comp = 0ull;
    if (i < nc && c_id[i] >= 0) {
      const float* it = p.I + (int64_t)c_id[i] * p.ldi;
      float acc = 0.f;
      if (vec4) {   // 16-byte loads; the fma chain stays sequential in k (exact-score definition)
        const float4* it4 = reinterpret_cast<const float4*>(it);
#pragma unroll 8
        for (int k4 = 0; k4 < p.d / 4; ++k4) {   // loads are independent of the fma chain: keep 8 in flight
          const float4 x = __ldg(it4 + k4);
          acc = fmaf(urow[4 * k4 + 0], x.x, acc);
          acc = fmaf(urow[4 * k4 + 1], x.y, acc);
          acc = fmaf(urow[4 * k4 + 2], x.z, acc);
          acc = fmaf(urow[4 * k4 + 3], x.w, acc);
        }
      } else {
        for (int k = 0; k < p.d; ++k) acc = fmaf(urow[k], __ldg(it + k), acc);
      }
      comp = ((unsigned long long)float_to_key(acc) << 32) | (unsigned long long)(~(uint32_t)c_id[i]);
    }
    mine[t] = comp;
  }
  __syncthreads();
  if (P <= 2 * FIN_THREADS) {
    // common case (<= 512 candidates): bitonic network over keys held in REGISTERS (element
    // e = tid + t * 256).  Partners inside the thread (j >= 256) are exchanged directly, partners
    // inside the warp (j < 32) with shuffles; only the stages with 32 <= j < 256 go through shared
    // memory (double-buffered: one barrier per such stage instead of one per stage).
    // two instantiations: one element per thread (<= 256 candidates, the usual case: k_row ~ 150) and two
    auto bitonic_regs = [&](auto ec) {
      constexpr int EPT = decltype(ec)::value;
      unsigned long long x[EPT];
#pragma unroll
      for (int t = 0; t < EPT; ++t) x[t] = mine[t];
      int buf = 0;
#pragma unroll 1
      for (int k = 2; k <= P; k <<= 1) {
#pragma unroll 1
        for (int j = k >> 1; j > 0; j >>= 1) {
          if (EPT == 2 && j >= FIN_THREADS) {   // only k = 512, j = 256: elements tid and tid + 256, descending
            const unsigned long long a = x[0], b = x[EPT - 1];
            x[0] = a > b ? a : b;
            x[EPT - 1] = a > b ? b : a;
            continue;
          }
          unsigned long long y[EPT];
          if (j >= 32) {
            unsigned long long* sb = c_sort + buf * (EPT * FIN_THREADS);
#pragma unroll
            for (int t = 0; t < EPT; ++t) sb[t * FIN_THREADS + tid] = x[t];
            __syncthreads();
#pragma unroll
            for (int t = 0; t < EPT; ++t) y[t] = sb[t * FIN_THREADS + (tid ^ j)];
            buf ^= 1;
          } else {
#pragma unroll
            for (int t = 0; t < EPT; ++t) y[t] = __shfl_xor_sync(0xffffffffu, x[t], j);
          }
#pragma unroll
          for (int t = 0; t < EPT; ++t) {
            const int e = tid + t * FIN_THREADS;
            const bool take_max = (((e & k) == 0) == ((e & j) == 0));   // descending blocks keep the max first
            x[t] = take_max ? (x[t] > y[t] ? x[t] : y[t]) : (x[t] < y[t] ? x[t] : y[t]);
          }
        }
      }
      __syncthreads();
#pragma unroll
      for (int t = 0; t < EPT; ++t) c_sort[t * FIN_THREADS + tid] = x[t];
      __syncthreads();
    };
    if (P <= FIN_THREADS) bitonic_regs(std::integral_constant<int, 1>{});
    else bitonic_regs(std::integral_constant<int, 2>{});
  } else {
#pragma unroll
    for (int t = 0; t < MAXC / FIN_THREADS; ++t) {
      const int i = tid + t * FIN_THREADS;
      if (i < P) c_sort[i] = mine[t];
    }
    __syncthreads();
    for (int k = 2; k <= P; k <<= 1) {
      for (int j = k >> 1; j > 0; j >>= 1) {
        for (int i = tid; i < P; i += FIN_THREADS) {
          const int ixj = i ^ j;
          if (ixj > i) {
            const unsigned long long a = c_sort[i], b = c_sort[ixj];
            const bool desc = ((i & k) == 0);
            if (desc ? (a < b) : (a > b)) { c_sort[i] = b; c_sort[ixj] = a; }
          }
        }
        __syncthreads();
      }
    }
  }
  {
    // Survivors: fewer than K (possible when k_row was capped), or — capped rows — a K-th exact
    // score that an uncollected item could still beat.  Uncollected items have coarse < thr, hence
    // exact < thr + eps = c_k - eps; the row is only accepted if the K-th survivor is above that.
    const unsigned long long kth = c_sort[p.K - 1];
    const bool short_row = kth == 0ull;
    // exact scores are unscaled: bring the K-th one into the row's coarse (scaled) units first
    const bool unsafe = meta.capped && key_to_float((uint32_t)(kth >> 32)) * meta.scale < thr + 0.5f * meta.eps2;
    if (short_row || unsafe) { __syncthreads(); give_up(5); return; }
  }
  for (int i = tid; i < p.K; i += FIN_THREADS) {
    const unsigned long long c = c_sort[i];
    oid[i] = (int64_t)(~(uint32_t)(c & 0xffffffffull));
    if (osc) osc[i] = key_to_float((uint32_t)(c >> 32));
  }
  if (tid == 0) p.out_status[row] = 0;
}

// The rows finalize_warp_kernel deferred (rare at the bench shape), over a fixed grid: the count is
// only known on the device.
constexpr int FIN_CTAS_PER_SM = 3;
__global__ void __launch_bounds__(FIN_THREADS)
finalize_kernel(const FinalizeParams p) {
  const int n = *p.defer_count;
#pragma unroll 1
  for (int i = blockIdx.x; i < n; i += gridDim.x) {
    finalize_row(p, p.defer_rows[i]);
    __syncthreads();   // the next row reuses the shared memory
  }
}

// One warp per row, no block barriers: the same steps as finalize_row on a per-warp buffer, for the
// rows that fit it (at the bench shape all but a handful).  It only ever completes rows with status 0:
// a row that would give up, or does not fit (more than WCAP collected elements, more than WSORT
// candidates, a capped k_row), is appended to the deferred list and finalize_kernel redoes it from
// scratch, so every give-up code and output comes from the block kernel.
constexpr int FINW_WARPS = 4;      // warps (rows) per CTA
constexpr int FINW_CTAS_PER_SM = 8;
constexpr int WCAP = 512;          // collected elements per row (measured at the bench shape: DESIGN §4)
constexpr int WSORT = 256;         // candidates per row (sort keys in FinWarpSmem::s)
struct FinWarpSmem {
  float4 urow[MAX_KB * KBLK / 4];  // the user row (fp32, unscaled)
  float s[WCAP];                   // collected coarse scores; after the cut: the hash set, then the sort keys
  int32_t id[WCAP];                // collected item ids; after the cut: candidate ids (~id = consumed)
  uint32_t hist[256];
};
static_assert(WCAP >= 2 * WSORT, "the hash set (2 WSORT slots) and the sort keys live in FinWarpSmem::s");

__global__ void __launch_bounds__(FINW_WARPS * 32, FINW_CTAS_PER_SM)
finalize_warp_kernel(const FinalizeParams p) {
  __shared__ FinWarpSmem smem[FINW_WARPS];
  const int lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * FINW_WARPS + (threadIdx.x >> 5);
  if (row >= p.B) return;
  FinWarpSmem& sm = smem[threadIdx.x >> 5];
  const unsigned lt = (1u << lane) - 1u;
  // ---- every independent load of the row at once
  const int32_t st = p.row_status[row];
  const RowMeta meta = p.meta[row];
  const uint32_t tk = p.row_tau_key[row], gk = p.tau_guess_key[row];
  const int64_t u = p.user_ids[row];
  auto defer = [&]() { if (lane == 0) p.defer_rows[atomicAdd(p.defer_count, 1)] = (int32_t)row; };
  if (st != 0 || meta.capped || p.defer_all) { defer(); return; }
  int64_t beg = 0, end = 0;
  if (meta.apply) { beg = p.indptr[u]; end = p.indptr[u + 1]; }
  float* urow = reinterpret_cast<float*>(sm.urow);
  for (int k = lane; k < p.d; k += 32) urow[k] = __ldg(p.U + u * p.ldu + k);   // needed only by the re-score
  // ---- gather every element >= the row's final threshold (ids < N) into the warp's buffer
  const float low = tk ? key_to_float(tk) : __int_as_float(0xff800000);
  int nu = 0;
  for (int s0 = 0; s0 < p.n_lists; s0 += 32) {
    const int c = s0 + lane < p.n_lists ? p.cand_cnt[(int64_t)(s0 + lane) * p.B_pad + row] : 0;
    int incl = c;   // records of lists s0 .. s0 + lane
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, o);
      if (lane >= o) incl += t;
    }
    const int total = __shfl_sync(0xffffffffu, incl, 31);
    constexpr int UN = 4;   // records in flight per lane
    for (int g0 = 0; g0 < total; g0 += 32 * UN) {
      float4 a[UN], b[UN];
      int base[UN];
#pragma unroll
      for (int q = 0; q < UN; ++q) {
        const int g = g0 + q * 32 + lane;
        int lo = 0, hi = 31;   // first lane (list) whose inclusive count exceeds g
#pragma unroll
        for (int it = 0; it < 5; ++it) {
          const int mid = (lo + hi) >> 1;
          if (__shfl_sync(0xffffffffu, incl, mid) <= g) lo = mid + 1; else hi = mid;
        }
        const int j = g - (__shfl_sync(0xffffffffu, incl, lo) - __shfl_sync(0xffffffffu, c, lo));
        a[q] = b[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        base[q] = 0;
        if (g < total) {
          const int64_t slot = (int64_t)(s0 + lo) * p.B_pad + row;
          const float4* ls = reinterpret_cast<const float4*>(p.cand_r + (slot * (int64_t)p.capg + j) * REC);
          a[q] = __ldcs(ls);
          b[q] = __ldcs(ls + 1);
          base[q] = __ldcs(reinterpret_cast<const int32_t*>(ls + 2));
        }
      }
#pragma unroll
      for (int q = 0; q < UN; ++q) {
        const bool ok = g0 + q * 32 + lane < total;
        const float v[8] = {a[q].x, a[q].y, a[q].z, a[q].w, b[q].x, b[q].y, b[q].z, b[q].w};
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const bool hit = ok && v[e] >= low && (int64_t)(base[q] + e) < p.N;   // never a zero-padded item row
          const unsigned m = __ballot_sync(0xffffffffu, hit);
          const int pos = nu + __popc(m & lt);
          if (hit && pos < WCAP) { sm.s[pos] = v[e]; sm.id[pos] = base[q] + e; }
          nu += __popc(m);
        }
      }
    }
  }
  if (nu < meta.k_row || nu > WCAP) { defer(); return; }
  __syncwarp();
  // ---- exact k_row-th largest coarse score of the buffer: 4 x 8-bit radix select, per-warp histogram
  uint32_t prefix = 0, krem = (uint32_t)meta.k_row;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    reinterpret_cast<uint4*>(sm.hist)[2 * lane] = make_uint4(0u, 0u, 0u, 0u);
    reinterpret_cast<uint4*>(sm.hist)[2 * lane + 1] = make_uint4(0u, 0u, 0u, 0u);
    __syncwarp();
    for (int i = lane; i < nu; i += 32) {
      const uint32_t key = float_to_key(sm.s[i]);
      if (pass == 0 || (key >> (shift + 8)) == prefix) atomicAdd(&sm.hist[(key >> shift) & 255u], 1u);
    }
    __syncwarp();
    // lane l owns bins [8 l, 8 l + 8); suffix counts over the lanes above
    uint32_t mine[8], tot = 0;
    const uint4 h0 = reinterpret_cast<const uint4*>(sm.hist)[2 * lane];
    const uint4 h1 = reinterpret_cast<const uint4*>(sm.hist)[2 * lane + 1];
    mine[0] = h0.x; mine[1] = h0.y; mine[2] = h0.z; mine[3] = h0.w;
    mine[4] = h1.x; mine[5] = h1.y; mine[6] = h1.z; mine[7] = h1.w;
#pragma unroll
    for (int b = 0; b < 8; ++b) tot += mine[b];
    uint32_t incl = tot;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const uint32_t t = __shfl_down_sync(0xffffffffu, incl, o);
      if (lane + o < 32) incl += t;
    }
    const uint32_t excl = incl - tot;   // count in the bins of the lanes above
    uint32_t np = 0, nk = 0;
    const bool owner = excl < krem && krem <= incl;
    if (owner) {
      uint32_t c = excl;
#pragma unroll
      for (int b = 7; b >= 0; --b) {
        if (c + mine[b] >= krem) { np = (prefix << 8) | (uint32_t)(lane * 8 + b); nk = krem - c; break; }
        c += mine[b];
      }
    }
    const int src = __ffs(__ballot_sync(0xffffffffu, owner)) - 1;
    prefix = __shfl_sync(0xffffffffu, np, src);
    krem = __shfl_sync(0xffffffffu, nk, src);
    __syncwarp();   // every lane has read the histogram before the next pass clears it
  }
  const float thr = key_to_float(prefix) - meta.eps2;
  // the speculative threshold must not exceed thr (see finalize_row)
  if (gk != 0u && key_to_float(gk) > thr) { defer(); return; }
  // ---- candidates: elements >= thr, compacted in place (a chunk is read before any of it is written)
  int nc = 0;
  for (int i0 = 0; i0 < nu; i0 += 32) {
    const int i = i0 + lane;
    const bool keep = i < nu && sm.s[i] >= thr;
    const int32_t id = i < nu ? sm.id[i] : 0;
    const unsigned m = __ballot_sync(0xffffffffu, keep);
    __syncwarp();
    const int pos = nc + __popc(m & lt);
    if (keep && pos < WSORT) sm.id[pos] = id;
    nc += __popc(m);
  }
  if (nc > WSORT || nc < p.K) { defer(); return; }
  int32_t* c_id = sm.id;
  // ---- consumed filter through a hash set of candidate slots (in s, dead after the cut)
  if (meta.apply) {
    int32_t* htab = reinterpret_cast<int32_t*>(sm.s);
    for (int i = lane; i < 2 * WSORT; i += 32) htab[i] = -1;
    __syncwarp();
    for (int i = lane; i < nc; i += 32) {
      uint32_t h = ((uint32_t)c_id[i] * 2654435761u) & (2 * WSORT - 1);
      while (atomicCAS(&htab[h], -1, i) != -1) h = (h + 1) & (2 * WSORT - 1);
    }
    __syncwarp();
    for (int64_t j = beg + lane; j < end; j += 32) {
      const int32_t it = p.idx[j];
      uint32_t h = ((uint32_t)it * 2654435761u) & (2 * WSORT - 1);
      while (true) {
        const int32_t e = htab[h];
        if (e < 0) break;
        if (c_id[e] == it || c_id[e] == ~it) { c_id[e] = ~it; break; }  // mark removed (negative)
        h = (h + 1) & (2 * WSORT - 1);
      }
    }
  }
  __syncwarp();   // the hash set is dead from here on: its storage holds the sort keys
  // ---- exact fp32 re-score, one lane per candidate: acc = fma(u[k], i[k], acc), k ascending
  unsigned long long* skey = reinterpret_cast<unsigned long long*>(sm.s);
  const bool vec4 = (p.d % 4 == 0) && (p.ldi % 4 == 0) && ((reinterpret_cast<uintptr_t>(p.I) & 15) == 0);
#pragma unroll 1
  for (int i = lane; i < WSORT; i += 32) {
    unsigned long long comp = 0ull;
    if (i < nc && c_id[i] >= 0) {
      const float* it = p.I + (int64_t)c_id[i] * p.ldi;
      float acc = 0.f;
      if (vec4) {   // 16-byte loads; the fma chain stays sequential in k (exact-score definition)
        const float4* it4 = reinterpret_cast<const float4*>(it);
#pragma unroll 8
        for (int k4 = 0; k4 < p.d / 4; ++k4) {
          const float4 x = __ldg(it4 + k4);
          const float4 w = sm.urow[k4];
          acc = fmaf(w.x, x.x, acc);
          acc = fmaf(w.y, x.y, acc);
          acc = fmaf(w.z, x.z, acc);
          acc = fmaf(w.w, x.w, acc);
        }
      } else {
        for (int k = 0; k < p.d; ++k) acc = fmaf(urow[k], __ldg(it + k), acc);
      }
      comp = ((unsigned long long)float_to_key(acc) << 32) | (unsigned long long)(~(uint32_t)c_id[i]);
    }
    skey[i] = comp;
  }
  __syncwarp();
  // ---- bitonic sort (descending) of the first P keys in shared memory: stages with j >= 32 pair
  // elements of one lane, stages with j < 32 run on shuffles, one element per lane at a time
  int P = 32;
  while (P < nc) P <<= 1;
  for (int k = 2; k <= P; k <<= 1) {
    for (int j = k >> 1; j >= 32; j >>= 1) {
      for (int q = lane; q < P / 2; q += 32) {
        const int e = ((q & ~(j - 1)) << 1) | (q & (j - 1));   // the pair (e, e + j), bit j of e clear
        const unsigned long long a = skey[e], b = skey[e + j];
        if ((e & k) == 0 ? a < b : a > b) { skey[e] = b; skey[e + j] = a; }
      }
      __syncwarp();
    }
    for (int e = lane; e < P; e += 32) {
      unsigned long long x = skey[e];
      for (int j = min(k >> 1, 16); j > 0; j >>= 1) {
        const unsigned long long y = __shfl_xor_sync(0xffffffffu, x, j);
        const bool take_max = ((e & k) == 0) == ((e & j) == 0);
        x = take_max ? (x > y ? x : y) : (x < y ? x : y);
      }
      skey[e] = x;
    }
    __syncwarp();
  }
  // fewer than K survivors: finalize_kernel flags the row (code 5)
  if (skey[p.K - 1] == 0ull) { defer(); return; }
  int64_t* oid = p.out_ids + row * p.K;
  float* osc = p.out_scores ? p.out_scores + row * p.K : nullptr;
  for (int e = lane; e < p.K; e += 32) {
    const unsigned long long c = skey[e];
    oid[e] = (int64_t)(~(uint32_t)(c & 0xffffffffull));
    if (osc) osc[e] = key_to_float((uint32_t)(c >> 32));
  }
  if (lane == 0) p.out_status[row] = 0;
}

// ------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (fn) return fn;
  void* p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) != cudaSuccess ||
      q != cudaDriverEntryPointSuccess)
    return nullptr;
  fn = (EncodeTiledFn)p;
  return fn;
}

// fp16 [rows, d_pad] row-major, box = [KBLK, box_rows], SWIZZLE_128B
static int make_tmap(CUtensorMap* m, const void* base, int64_t rows, int d_pad, int box_rows) {
  EncodeTiledFn enc = get_encode_fn();
  B200_REQUIRE(enc, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {(cuuint64_t)d_pad, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)d_pad * 2};
  cuuint32_t box[2] = {(cuuint32_t)KBLK, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), dims, strides,
                   box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return 0;
}

static inline int pad_to(int64_t x, int m) { return (int)((x + m - 1) / m * m); }
static inline size_t al256(size_t x) { return (x + 255) & ~(size_t)255; }


// ---- tuning knobs (defaults compiled in; b200_recommend_embed_tune overrides them per process) ----
static int g_epi = 5;              // record stores of a hot epilogue step: 5 quad masks (measured best on H100), 3 divergent group tests
static int g_cluster = 2;          // 2 = pairs of user tiles share every item tile through TMA multicast, 1 = off
static int g_nh = 1;               // MMA organisation of an item tile (1 x N=256, measured best on H100; 2 x N=128, epilogue of
                                   // the first overlaps the second; 3 = 2 x N=128 pipelined across tiles)
static int g_ablate = 0;           // b200_recommend_embed_debug
static int g_defer_all = 0;        // b200_recommend_embed_debug level 3
static int g_hint_ns = 20000;      // suspend-time hint of the mbarrier waits in the sweep kernels
static int g_pre_stride = PRE_STRIDE;   // b200_recommend_embed_speculation
static double g_pre_delta = PRE_DELTA;
static float g_pre_coef = 0.f;     // non-zero: linear speculative rank pre_k = margin + coef * f * k_row (A/B runs, tests)
static int g_pre_margin = 12;      // its additive part (b200_recommend_embed_debug)

struct Plan {
  int B_pad, d_pad, KB, m_tiles, total_tiles, n_splits, tiles_per_split, nstage, n_pre_tiles, kb_stages;
  int W, n_lists, capg, trig;
  int CL, NH;        // CTAs per cluster (TMA multicast of the item tiles), MMA groups per item tile
  bool use_pre;
  int pre_stride;    // the pre-pass visits every pre_stride-th item tile of a split
  int pre_sampled;   // item tiles the pre-pass visits (f = pre_sampled / total_tiles)
  int64_t N_pad;
  size_t smem_bytes;
  // workspace offsets
  size_t off_A, off_meta, off_tau, off_guess, off_status, off_cnt, off_defer, off_flag, off_hist, off_cs, off_bm, total;
};

static int make_plan(int64_t B, int64_t N, int d, Plan* pl) {
  pl->d_pad = pad_to(d, KBLK);
  pl->KB = pl->d_pad / KBLK;
  B200_REQUIRE(pl->KB >= 1 && pl->KB <= MAX_KB, "fused scorer supports embed width <= %d (got %d)",
               MAX_KB * KBLK, d);
  // clusters of 2 CTAs take two adjacent user tiles: worth it from two user tiles on (B > 128)
  pl->CL = (g_cluster == 2 && B > TM) ? 2 : 1;
  // d_pad <= 128: a ring stage = one whole 256-item tile (KB k-blocks); wider embeddings: one k-block per stage
  // (a whole tile of d_pad = 256 is 128 KB: two of them do not fit beside the 64 KB user tile)
  pl->kb_stages = pl->KB > 2;
  // the pipelined organisation holds two whole-tile stages at once: k-block stages run one N=256 group
  pl->NH = (g_nh == 3 && pl->kb_stages) ? 1 : g_nh;
  pl->B_pad = pad_to(B, TM * pl->CL);
  pl->N_pad = (N + TN - 1) / TN * TN;
  pl->m_tiles = pl->B_pad / TM;
  pl->total_tiles = (int)(pl->N_pad / TN);
  pl->W = 2;
  // item splits: minimise makespan = waves * (tiles per split + per-unit overhead)
  const int ovh = 12;
  long best = -1;
  int bestS = 1;
  // without a device (plan and workspace queries only) the plan is the one of a 132-SM H100 SXM
  const int sms = num_sms() > 0 ? num_sms() : 132;
  const int maxS = pl->total_tiles < 2 * sms ? pl->total_tiles : 2 * sms;
  for (int S = 1; S <= maxS; ++S) {
    const long units = (long)pl->m_tiles * S;
    const long waves = (units + sms - 1) / sms;
    const long tps = (pl->total_tiles + S - 1) / S;
    const long cost = waves * (tps + ovh);
    if (best < 0 || cost < best) { best = cost; bestS = S; }
  }
  pl->tiles_per_split = (pl->total_tiles + bestS - 1) / bestS;
  pl->n_splits = (pl->total_tiles + pl->tiles_per_split - 1) / pl->tiles_per_split;
  pl->pre_stride = g_pre_stride;
  pl->n_pre_tiles = (pl->tiles_per_split + pl->pre_stride - 1) / pl->pre_stride;
  pl->n_lists = pl->W * pl->n_splits;
  // speculation needs enough sampled blocks per row to take a stable order statistic
  pl->use_pre = (long)W_PRE * pl->n_splits * pl->n_pre_tiles >= 256;
  pl->pre_sampled = 0;   // every pre_stride-th tile of every split
  for (int sp = 0; sp < pl->n_splits; ++sp) {
    const int t0 = sp * pl->tiles_per_split;
    const int t1 = t0 + pl->tiles_per_split < pl->total_tiles ? t0 + pl->tiles_per_split : pl->total_tiles;
    pl->pre_sampled += (t1 - t0 + pl->pre_stride - 1) / pl->pre_stride;
  }
  // With the speculative threshold a few times k_row candidates per row (<= ~1500 at k_row = 288 under
  // the linear rule's defaults) are spread over the lists; the lists are sized for that and the
  // compaction runs only when a list is about to overflow (the speculation was far off).
  pl->capg = (pl->use_pre && pl->n_lists >= 16) ? 128 : CAPG_MAX;
  pl->trig = pl->use_pre ? pl->capg : 96;
  const size_t budget = 227 * 1024 - 1024 /*align*/ - sizeof(SweepSmem) - (size_t)pl->KB * A_KB_BYTES;
  B200_REQUIRE(!pl->kb_stages || pl->NH == 1, "the two-MMA-group organisation supports embed width <= 128 only");
  const size_t stage_bytes = pl->kb_stages ? (size_t)B_KB_BYTES : (size_t)pl->KB * B_KB_BYTES;
  int ns = (int)(budget / stage_bytes);
  if (ns > (pl->kb_stages ? 8 : 6)) ns = pl->kb_stages ? 8 : 6;
  B200_REQUIRE(ns >= 2, "not enough shared memory for the item pipeline");
  pl->nstage = ns;
  pl->smem_bytes = 1024 + (size_t)pl->KB * A_KB_BYTES + (size_t)ns * stage_bytes + sizeof(SweepSmem);
  size_t off = 0;
  pl->off_A = off; off += al256((size_t)pl->B_pad * pl->d_pad * 2);
  pl->off_meta = off; off += al256((size_t)pl->B_pad * sizeof(RowMeta));
  pl->off_tau = off; off += al256((size_t)pl->B_pad * 4);
  pl->off_guess = off; off += al256((size_t)pl->B_pad * 4);
  pl->off_status = off; off += al256((size_t)pl->B_pad * 4);
  pl->off_cnt = off; off += al256((size_t)pl->n_lists * pl->B_pad * 4);
  pl->off_defer = off; off += al256((size_t)(1 + pl->B_pad) * 4);   // count, then the rows finalize_kernel redoes
  pl->off_flag = off; off += al256(4);                              // rows with a non-zero status
  pl->off_hist = off; off += al256((size_t)pl->B_pad * NB * 4);
  pl->off_cs = off; off += al256((size_t)pl->n_lists * pl->B_pad * pl->capg * REC * 4);
  pl->off_bm = off; off += al256((size_t)W_PRE * pl->n_splits * pl->n_pre_tiles * pl->B_pad * 4);
  pl->total = off + 256;
  return 0;
}

// Smallest r with P[Binomial(n, f) >= r] <= delta (n + 1 when no r <= n qualifies).
static int binomial_rank(int n, double f, double delta) {
  if (f >= 1.0) return n + 1;
  const double log_odds = std::log(f) - std::log1p(-f);
  double log_pmf = n * std::log1p(-f);   // log P[X = 0]
  double cdf = 0.0;
  for (int r = 0; r < n; ++r) {
    cdf += std::exp(log_pmf);
    if (1.0 - cdf <= delta) return r + 1;   // P[X >= r + 1] = 1 - P[X <= r]
    log_pmf += std::log((double)(n - r) / (double)(r + 1)) + log_odds;
  }
  return n + 1;
}

// Speculative rank pre_k of every k_row for the plan's sampled fraction f, under the active rule.
// Failure budget (default): speculation fails exactly when at least pre_k sampled block maxima exceed
// c_k - 2 eps, and each such block holds a sampled item with coarse >= c_k - 2 eps.  About
// n = k_row + PRE_TIE_ALLOWANCE items lie that high; when the item order does not depend on the scores,
// the number of them in the sampled tiles is about Binomial(n, f), so pre_k = the smallest r with
// P[Binomial(n, f) >= r] <= delta keeps the rate of failed rows (status 3, repaired on the exact path)
// near delta.  Linear rule (a non-zero rank coefficient): pre_k = margin + ceil(coef * f * k_row).
static void rank_table(const Plan& pl, int32_t* out) {
  thread_local int32_t tab[KROW_MAX + 1];
  thread_local double key_f = -1.0, key_delta = -1.0;
  const double f = (double)pl.pre_sampled / (double)pl.total_tiles;
  if (g_pre_coef != 0.f) {
    const float pre_scale = g_pre_coef * (float)pl.pre_sampled / (float)pl.total_tiles;
    for (int k = 0; k <= KROW_MAX; ++k) out[k] = g_pre_margin + (int32_t)ceilf(pre_scale * (float)k);
    return;
  }
  if (f != key_f || g_pre_delta != key_delta) {   // recomputed only when the plan's f or delta changes
    for (int k = 0; k <= KROW_MAX; ++k) tab[k] = binomial_rank(k + PRE_TIE_ALLOWANCE, f, g_pre_delta);
    key_f = f;
    key_delta = g_pre_delta;
  }
  memcpy(out, tab, sizeof(tab));
}

template <bool PRE, int EPI, int CL, int NH>
static int launch_sweep(int grid, const Plan& pl, cudaStream_t stream, const CUtensorMap& tmA,
                        const CUtensorMap& tmB, const CUtensorMap& tmBh, const SweepParams& sp) {
  static bool attr_set = false;
  if (!attr_set) {
    B200_CUDA_OK(cudaFuncSetAttribute(sweep_kernel<PRE, EPI, CL, NH>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                      227 * 1024));
    attr_set = true;
  }
  cudaLaunchConfig_t cfg;
  memset(&cfg, 0, sizeof(cfg));
  cfg.gridDim = dim3((unsigned)grid, 1, 1);
  cfg.blockDim = dim3((unsigned)SWEEP_THREADS, 1, 1);
  cfg.dynamicSmemBytes = pl.smem_bytes;
  cfg.stream = stream;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension;
  at[0].val.clusterDim.x = CL; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at;
  cfg.numAttrs = 1;
  B200_CUDA_OK(cudaLaunchKernelEx(&cfg, sweep_kernel<PRE, EPI, CL, NH>, tmA, tmB, tmBh, sp));
  count_launch();
  return 0;
}

// organisation = (record stores EPI, cluster size CL, MMA organisation NH); the default is (5, 2, 1)
static int launch_pre_dispatch(int grid, const Plan& pl, cudaStream_t stream, const CUtensorMap& tmA,
                               const CUtensorMap& tmB, const CUtensorMap& tmBh, const SweepParams& sp) {
  // the pre-pass stores no records: one epilogue; the pipelined organisation (NH = 3) runs its pre-pass on
  // the unpipelined two-group kernel
  if (pl.CL == 2) {
    if (pl.NH == 1) return launch_sweep<true, 3, 2, 1>(grid, pl, stream, tmA, tmB, tmBh, sp);
    return launch_sweep<true, 3, 2, 2>(grid, pl, stream, tmA, tmB, tmBh, sp);
  }
  if (pl.NH == 1) return launch_sweep<true, 3, 1, 1>(grid, pl, stream, tmA, tmB, tmBh, sp);
  return launch_sweep<true, 3, 1, 2>(grid, pl, stream, tmA, tmB, tmBh, sp);
}

static int launch_main_dispatch(int grid, const Plan& pl, int epi, cudaStream_t stream, const CUtensorMap& tmA,
                                const CUtensorMap& tmB, const CUtensorMap& tmBh, const SweepParams& sp) {
#define B200_SWEEP(E_, C_, N_) return launch_sweep<false, E_, C_, N_>(grid, pl, stream, tmA, tmB, tmBh, sp)
  if (epi == 5) {
    if (pl.CL == 2) { if (pl.NH == 3) B200_SWEEP(5, 2, 3); if (pl.NH == 2) B200_SWEEP(5, 2, 2); B200_SWEEP(5, 2, 1); }
    if (pl.NH == 3) B200_SWEEP(5, 1, 3);
    if (pl.NH == 2) B200_SWEEP(5, 1, 2);
    B200_SWEEP(5, 1, 1);
  }
  if (pl.CL == 2) { if (pl.NH == 3) B200_SWEEP(3, 2, 3); if (pl.NH == 2) B200_SWEEP(3, 2, 2); B200_SWEEP(3, 2, 1); }
  if (pl.NH == 3) B200_SWEEP(3, 1, 3);
  if (pl.NH == 2) B200_SWEEP(3, 1, 2);
  B200_SWEEP(3, 1, 1);
#undef B200_SWEEP
}

}  // namespace tc
}  // namespace b200

using namespace b200;
using namespace b200::tc;

extern "C" int b200_embed_catalog_bytes(int64_t N, int32_t d, size_t* bytes) {
  B200_REQUIRE(bytes && N >= 1 && d >= 1, "b200_embed_catalog_bytes: bad arguments");
  const int d_pad = pad_to(d, KBLK);
  const int64_t N_pad = (N + TN - 1) / TN * TN;
  *bytes = 256 + (size_t)N_pad * d_pad * 2 + 1024;
  return 0;
}

extern "C" int b200_embed_catalog_prepare(const float* I, int64_t ldi, int64_t N, int32_t d,
                                          void* catalog, size_t bytes, void* stream_) {
  B200_REQUIRE(I && catalog, "b200_embed_catalog_prepare: null pointer");
  size_t need;
  if (int rc = b200_embed_catalog_bytes(N, d, &need)) return rc;
  B200_REQUIRE(bytes >= need, "catalog buffer too small (%zu < %zu)", bytes, need);
  B200_REQUIRE(((uintptr_t)catalog & 255) == 0, "catalog buffer must be 256-byte aligned");
  cudaStream_t stream = (cudaStream_t)stream_;
  const int d_pad = pad_to(d, KBLK);
  const int64_t N_pad = (N + TN - 1) / TN * TN;
  CatalogHeader h;
  memset(&h, 0, sizeof(h));
  h.d = d; h.d_pad = d_pad; h.N = N; h.N_pad = N_pad; h.scale = 1.f;
  B200_CUDA_OK(cudaMemcpyAsync(catalog, &h, sizeof(h), cudaMemcpyHostToDevice, stream));
  __half* tab = (__half*)((char*)catalog + 256);
  // pass 1: max row norm -> power-of-two scale; pass 2: scaled fp16 copy
  item_norm_kernel<<<(unsigned)ceil_div64(N * 32, 256), 256, 0, stream>>>(I, ldi, N, d, (CatalogHeader*)catalog);
  item_scale_kernel<<<1, 1, 0, stream>>>((CatalogHeader*)catalog);
  prep_items_kernel<<<(unsigned)ceil_div64(N_pad * 32, 256), 256, 0, stream>>>(
      I, ldi, N, d, d_pad, N_pad, tab, (const CatalogHeader*)catalog);
  count_launch(3);
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_recommend_embed_tune(int32_t epilogue_warps_per_quadrant, float pre_rank_coef) {
  if (epilogue_warps_per_quadrant != 0) {   // organisation code: 100 * cluster size + 10 * MMA organisation + epilogue variant
    const int code = epilogue_warps_per_quadrant % 1000;
    const int cl = (code / 100) % 10, nh = (code / 10) % 10, epi = code % 10;
    B200_REQUIRE((cl == 1 || cl == 2) && (nh >= 1 && nh <= 3) && (epi == 3 || epi == 5),
                 "b200_recommend_embed_tune: code = 100 * cluster (1|2) + 10 * MMA groups (1|2, 3 = 2 pipelined) "
                 "+ record stores (3|5)");
    g_cluster = cl; g_nh = nh; g_epi = epi;
  }
  if (pre_rank_coef != 0.f) {
    B200_REQUIRE(pre_rank_coef >= 1.0f && pre_rank_coef <= 16.f,
                 "b200_recommend_embed_tune: rank coefficient out of [1, 16]");
    g_pre_coef = pre_rank_coef;
  }
  return 0;
}

extern "C" int b200_recommend_embed_speculation(int32_t pre_stride, float delta) {
  B200_REQUIRE((pre_stride == 0 || (pre_stride >= 2 && pre_stride <= 32)) &&
                   (delta == 0.f || (delta >= 1e-9f && delta <= 1e-2f)),
               "b200_recommend_embed_speculation: stride 0 or 2..32, failure budget 0 or [1e-9, 1e-2]");
  g_pre_stride = pre_stride ? pre_stride : PRE_STRIDE;
  g_pre_delta = delta != 0.f ? (double)delta : PRE_DELTA;
  g_pre_coef = 0.f;   // the failure-budget rule
  return 0;
}

// Diagnostics (profiling only; results are WRONG while level 1 or 2 is set): 1 = the main pass collects
// nothing (cold epilogue steps only), 2 = the main pass runs no epilogue at all (wait, MMA, release).
// Level 3 (results unchanged) = finalize_warp_kernel defers every row to finalize_kernel, so that both
// finalize paths can be run and compared on the same sweep output.
extern "C" int b200_recommend_embed_debug(int32_t ablate_level) {
  // levels >= 100: suspend-time hint (ns) of the mbarrier waits of the sweep kernels = level - 100
  // levels -1 .. -64: additive margin of the linear speculative rank (pre_k = margin + coef * f * k_row) = -level
  if (ablate_level < 0 && ablate_level >= -64) { g_pre_margin = -ablate_level; return 0; }
  if (ablate_level >= 100) { g_hint_ns = ablate_level - 100; return 0; }
  B200_REQUIRE(ablate_level >= 0 && ablate_level <= 3, "b200_recommend_embed_debug: level 0..3 (or 100 + hint ns)");
  g_ablate = ablate_level <= 2 ? ablate_level : 0;
  g_defer_all = ablate_level == 3;
  return 0;
}

extern "C" int b200_recommend_embed_plan(int64_t B, int64_t N, int32_t d, int32_t K, int32_t* out,
                                         int32_t n_out) {
  B200_REQUIRE(out && n_out >= 8 && B >= 1 && N >= 1 && d >= 1 && K >= 1,
               "b200_recommend_embed_plan: bad arguments");
  Plan pl;
  if (int rc = make_plan(B, N, d, &pl)) return rc;
  out[0] = pl.use_pre ? 1 : 0; out[1] = pl.n_splits; out[2] = pl.tiles_per_split; out[3] = pl.m_tiles;
  out[4] = pl.n_pre_tiles; out[5] = pl.nstage; out[6] = pl.CL * 10 + pl.NH; out[7] = pl.capg;
  if (n_out >= 10) { out[8] = pl.pre_stride; out[9] = pl.pre_sampled; }
  if (n_out >= 10 + KROW_MAX + 1) rank_table(pl, out + 10);
  return 0;
}

extern "C" int b200_recommend_embed_workspace_bytes(int64_t B, int64_t N, int32_t d, int32_t K,
                                                    size_t* bytes) {
  B200_REQUIRE(bytes && B >= 1 && N >= 1 && d >= 1 && K >= 1, "bad arguments");
  Plan pl;
  if (int rc = make_plan(B, N, d, &pl)) return rc;
  *bytes = pl.total;
  return 0;
}

extern "C" int b200_recommend_embed(const float* U, int64_t ldu, const int64_t* user_ids, int64_t B,
                                    const float* I, int64_t ldi, int64_t N, int32_t d,
                                    const void* catalog, const int64_t* indptr, const int32_t* idx,
                                    int64_t n_users, int32_t filter, int32_t K, int64_t* out_ids,
                                    float* out_scores, int32_t* row_status, void* workspace,
                                    size_t workspace_bytes, void* stream_, void* ev_sweep_start,
                                    void* ev_sweep_stop, int32_t* n_flagged) {
  B200_REQUIRE(U && user_ids && I && catalog && out_ids && row_status && workspace,
               "b200_recommend_embed: null pointer");
  B200_REQUIRE((int64_t)K <= N, "`n_rec` %d exceeds num of items %lld", K, (long long)N);
  B200_REQUIRE(K <= KROW_MAX, "b200_recommend_embed: n_rec %d above the fused-path limit %d", K, KROW_MAX);
  B200_REQUIRE(N < (1ll << 31) - TN, "N too large");
  if (B == 0) return 0;
  cudaStream_t stream = (cudaStream_t)stream_;
  Plan pl;
  if (int rc = make_plan(B, N, d, &pl)) return rc;
  B200_REQUIRE(workspace_bytes >= pl.total, "workspace too small (%zu < %zu)", workspace_bytes, pl.total);
  char* ws = (char*)(((uintptr_t)workspace + 255) & ~(uintptr_t)255);
  __half* A = (__half*)(ws + pl.off_A);
  RowMeta* meta = (RowMeta*)(ws + pl.off_meta);
  uint32_t* tau = (uint32_t*)(ws + pl.off_tau);
  uint32_t* guess = (uint32_t*)(ws + pl.off_guess);
  int32_t* status = (int32_t*)(ws + pl.off_status);
  int32_t* cnt = (int32_t*)(ws + pl.off_cnt);
  int32_t* defer = (int32_t*)(ws + pl.off_defer);
  int32_t* flagged = (int32_t*)(ws + pl.off_flag);
  uint32_t* ghist = (uint32_t*)(ws + pl.off_hist);
  float* cand_r = (float*)(ws + pl.off_cs);
  float* bm = (float*)(ws + pl.off_bm);
  const CatalogHeader* hdr = (const CatalogHeader*)catalog;
  const __half* Ih = (const __half*)((const char*)catalog + 256);

  PreRank pre_rank;
  rank_table(pl, pre_rank.k);
  prep_users_kernel<<<(unsigned)ceil_div64((int64_t)pl.B_pad * 32, 256), 256, 0, stream>>>(
      U, ldu, user_ids, B, pl.B_pad, d, pl.d_pad, K, N, filter, pre_rank, indptr, n_users, hdr, A, meta,
      tau, status);
  count_launch();
  // cnt, the deferred-row list, the flagged-row count and ghist are adjacent in the workspace: one memset
  B200_CUDA_OK(cudaMemsetAsync(cnt, 0, (pl.off_cs - pl.off_cnt), stream));

  CUtensorMap tmA, tmB, tmBh;
  if (int rc = make_tmap(&tmA, A, pl.B_pad, pl.d_pad, TM)) return rc;
  if (int rc = make_tmap(&tmB, Ih, pl.N_pad, pl.d_pad, TN)) return rc;
  if (int rc = make_tmap(&tmBh, Ih, pl.N_pad, pl.d_pad, TN / 2)) return rc;   // per-CTA share of a tile (cluster of 2)

  SweepParams sp;
  sp.N = N; sp.B_pad = pl.B_pad; sp.m_tiles = pl.m_tiles; sp.n_splits = pl.n_splits;
  sp.tiles_per_split = pl.tiles_per_split; sp.total_tiles = pl.total_tiles; sp.KB = pl.KB;
  sp.nstage = pl.nstage; sp.kb_stages = pl.kb_stages; sp.n_pre_tiles = pl.n_pre_tiles;
  sp.pre_stride = pl.pre_stride; sp.capg = pl.capg; sp.trig = pl.trig;
  sp.meta = meta; sp.row_tau_key = tau;
  sp.row_status = status; sp.ghist = ghist; sp.cand_r = cand_r; sp.cand_cnt = cnt;
  sp.blockmax = bm; sp.ablate = g_ablate; sp.hint_ns = (uint32_t)g_hint_ns;
  const int n_units = pl.m_tiles * pl.n_splits;
  const int sm_count = num_sms();
  int grid = n_units < sm_count ? n_units : sm_count;
  grid -= grid % pl.CL;                                    // whole clusters

  if (ev_sweep_start) B200_CUDA_OK(cudaEventRecord((cudaEvent_t)ev_sweep_start, stream));
  if (pl.use_pre) {
    if (int rc = launch_pre_dispatch(grid, pl, stream, tmA, tmB, tmBh, sp)) return rc;
    guess_kernel<<<(unsigned)(pl.B_pad / 32), GUESS_THREADS, 0, stream>>>(
        bm, W_PRE * pl.n_splits * pl.n_pre_tiles, pl.B_pad, meta, tau, guess);
    count_launch();
  } else {
    B200_CUDA_OK(cudaMemsetAsync(guess, 0, (size_t)pl.B_pad * 4, stream));
  }
  if (int rc = launch_main_dispatch(grid, pl, g_epi, stream, tmA, tmB, tmBh, sp)) return rc;
  if (ev_sweep_stop) B200_CUDA_OK(cudaEventRecord((cudaEvent_t)ev_sweep_stop, stream));

  FinalizeParams fp;
  fp.B = B; fp.N = N; fp.B_pad = pl.B_pad; fp.n_lists = pl.n_lists; fp.K = K; fp.d = d; fp.capg = pl.capg;
  fp.defer_all = g_defer_all;
  fp.meta = meta; fp.row_status = status; fp.out_status = row_status; fp.defer_count = defer;
  fp.defer_rows = defer + 1; fp.flagged = flagged; fp.row_tau_key = tau; fp.tau_guess_key = guess;
  fp.cand_r = cand_r; fp.cand_cnt = cnt;
  fp.U = U; fp.ldu = ldu; fp.I = I; fp.ldi = ldi; fp.user_ids = user_ids; fp.indptr = indptr;
  fp.idx = idx; fp.out_ids = out_ids; fp.out_scores = out_scores;
  // every row writes its row_status once: 0 from the warp kernel, or any code from the block kernel
  finalize_warp_kernel<<<(unsigned)ceil_div64(B, FINW_WARPS), FINW_WARPS * 32, 0, stream>>>(fp);
  const int64_t fin_grid = (int64_t)FIN_CTAS_PER_SM * (sm_count > 0 ? sm_count : 132);
  finalize_kernel<<<(unsigned)(B < fin_grid ? B : fin_grid), FIN_THREADS, 0, stream>>>(fp);
  count_launch(2);
  if (n_flagged)   // stream-ordered: a caller can wait for this call alone, not for what it enqueues next
    B200_CUDA_OK(cudaMemcpyAsync(n_flagged, flagged, sizeof(int32_t), cudaMemcpyDefault, stream));
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
