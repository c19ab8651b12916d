// K1, bulk-copy staged variant — the embedding gather of the feature models
// (libreco/layers/embedding.py:4-23, libreco/tfops/features.py:6-44,121-148) as a persistent,
// warp-specialised kernel whose row gathers run on the TMA engine:
//
//   producer warp : for a batch of RB rows resolves the (2 + F_s + F_d) source rows of every output
//                   row (ids -> unique tables -> offsets into the shared tables; all index loads of a
//                   batch are in flight together), then issues ONE `cp.async.bulk` (UBLKCP, 4K bytes)
//                   per gathered embedding row straight into the stage's shared-memory image of the
//                   concatenated row [F][K]; completion is counted in bytes on the stage's mbarrier.
//                   Nothing is held in registers while the copies fly: the ring of NSTAGE stages keeps
//                   NSTAGE * RB * F row reads outstanding per CTA (the kernel is HBM/L2-latency bound
//                   on random 4K-byte rows, so the bytes in flight are what matters).
//   consumer warps: one per row of the batch: FM sums (sum_f e, sum_f e^2) with 16-byte shared-memory
//                   reads and a warp-shuffle reduction over the field groups, linear term, fused FM
//                   head; the deep / tower input row is written back with ONE bulk store
//                   (shared -> global, F*K*4 contiguous bytes) — or not at all when only the fused
//                   head is wanted ([B, F, K] never touches HBM).
//
// Eligible when K % 4 == 0, K <= 32 and all tables are 16-byte aligned; b200_feat_forward falls
// back to the register kernels of feat.cu otherwise.
#include "common.cuh"
#include "feat_common.cuh"
#include "ptx_sm90.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace feat {

constexpr int FT_MAX_RB = 8;
constexpr int FT_NSTAGE = 3;
constexpr int FT_MAX_FJ = (2 + 2 * B200_MAX_FIELDS + 31) / 32;   // fields per producer lane (upper bound)

struct FtOut {
  float* concat; int64_t ld_concat;
  float* pw; int64_t ld_pw;
  float* lin;
  float* fm_out;
  float* ssum; float* sqsum; int64_t ld_s;
};
struct FtHead {
  const float* lin_kernel; float lin_bias;
  const float* bn_scale; const float* bn_shift; const float* pw_kernel; float pw_bias;
};

__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               ::"r"(ptx::smem_u32(smem_dst)), "l"(gsrc), "r"(bytes), "r"(ptx::smem_u32(bar))
               : "memory");
}
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;"
               ::"l"(gdst), "r"(ptx::smem_u32(smem_src)), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void bulk_wait_read0() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }

template <int K4>
__global__ void __launch_bounds__(32 * (1 + FT_MAX_RB))
feat_forward_tma_kernel(const b200_feat_layout L, const b200_feat_tables T, const int64_t* __restrict__ users,
                        const int64_t* __restrict__ items, int64_t R, int64_t grid_items, int64_t row_offset,
                        FtOut o, FtHead h, int RB) {
  constexpr int K = K4 * 4;
  extern __shared__ uint8_t ft_smem_raw[];
  uint8_t* base = (uint8_t*)(((uintptr_t)ft_smem_raw + 127) & ~(uintptr_t)127);
  const int n_id = ((L.id_mask & 1) ? 1 : 0) + ((L.id_mask & 2) ? 1 : 0);
  const int F = n_id + L.n_sparse + L.n_dense;
  const int first_dense = n_id + L.n_sparse;
  const size_t row_bytes = (size_t)F * K * 4;
  const size_t aux_bytes = ((size_t)F * 4 * 2 + 15) & ~(size_t)15;        // xs[F], lw[F] per row
  const size_t stage_bytes = (size_t)RB * (row_bytes + aux_bytes);
  uint64_t* full = (uint64_t*)(base + FT_NSTAGE * stage_bytes);
  uint64_t* empty = full + FT_NSTAGE;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const bool want_lin = (o.lin != nullptr) || (o.fm_out != nullptr);

  if (threadIdx.x == 0) {
    for (int s = 0; s < FT_NSTAGE; ++s) { ptx::mbar_init(&full[s], 32); ptx::mbar_init(&empty[s], RB); }
    ptx::fence_barrier_init();
  }
  __syncthreads();
  const int64_t n_batches = (R + RB - 1) / RB;

  if (warp == 0) {
    // ===================== producer =====================
    int stage = 0;
    uint32_t phase = 0;
    for (int64_t b = blockIdx.x; b < n_batches; b += gridDim.x) {
      ptx::mbar_wait(&empty[stage], phase ^ 1);
      uint8_t* st = base + (size_t)stage * stage_bytes;
      uint32_t tx = 0;
      for (int i = 0; i < RB; ++i) {
        const int64_t r = b * RB + i;
        if (r >= R) break;
        int64_t u, it;
        if (grid_items > 0) { const int64_t rg = r + row_offset; u = users[rg / grid_items]; it = rg % grid_items; }
        else { u = users[r]; it = items[r]; }
        float* rows = (float*)(st + (size_t)i * (row_bytes + aux_bytes));
        float* xs = (float*)((uint8_t*)rows + row_bytes);
        float* lw = xs + F;
        // pass 1: resolve every source row of this lane's fields (all index loads in flight together)
        const float* src[FT_MAX_FJ];
        float x[FT_MAX_FJ], lv[FT_MAX_FJ];
#pragma unroll
        for (int j = 0; j < FT_MAX_FJ; ++j) {
          const int f = lane + 32 * j;
          src[j] = nullptr; x[j] = 1.f; lv[j] = 0.f;
          if (f < F) {
            if (f < n_id) {
              const bool is_user = (L.id_mask & 1) && f == 0;
              src[j] = is_user ? T.user_embeds + u * K : T.item_embeds + it * K;
              if (want_lin) lv[j] = is_user ? __ldg(T.user_linear + u) : __ldg(T.item_linear + it);
            } else if (f < first_dense) {
              const int32_t idx = sparse_index(L, r, u, it, f - n_id);
              src[j] = T.sparse_embeds + (int64_t)idx * K;
              if (want_lin) lv[j] = __ldg(T.sparse_linear + idx);
            } else {
              const int fd = f - first_dense;
              x[j] = dense_value(L, r, u, it, fd);
              src[j] = T.dense_embeds + (int64_t)L.dense_embed_row[fd] * K;
              if (want_lin) lv[j] = __ldg(T.dense_linear + L.dense_embed_row[fd]) * x[j];
            }
            if (want_lin) lv[j] *= h.lin_kernel[f];
          }
        }
        // pass 2: one bulk copy per gathered row; the scale / linear contribution go to the aux arrays
#pragma unroll
        for (int j = 0; j < FT_MAX_FJ; ++j) {
          const int f = lane + 32 * j;
          if (f < F) {
            bulk_g2s(rows + (size_t)f * K, src[j], (uint32_t)(K * 4), &full[stage]);
            xs[f] = x[j];
            lw[f] = lv[j];
            tx += (uint32_t)(K * 4);
          }
        }
      }
      // lanes 1..31 arrive; lane 0 arrives WITH the byte count of the whole warp (the transaction count
      // may run negative until then, the phase cannot complete before all 32 arrivals)
      const uint32_t tx_all = __reduce_add_sync(0xffffffffu, tx);
      if (lane == 0) ptx::mbar_arrive_expect_tx(&full[stage], tx_all);
      else ptx::mbar_arrive(&full[stage]);
      if (++stage == FT_NSTAGE) { stage = 0; phase ^= 1; }
    }
  } else if (warp <= RB) {
    // ===================== consumers: warp w <-> row w - 1 of every batch =====================
    const int i = warp - 1;
    constexpr int G = 32 / K4;                 // field groups per warp
    const int fg = lane / K4, q = lane % K4;
    int stage = 0;
    uint32_t phase = 0;
    for (int64_t b = blockIdx.x; b < n_batches; b += gridDim.x) {
      ptx::mbar_wait(&full[stage], phase);
      const int64_t r = b * RB + i;
      uint8_t* st = base + (size_t)stage * stage_bytes;
      if (r < R) {
        float* rows = (float*)(st + (size_t)i * (row_bytes + aux_bytes));
        const float* xs = (const float*)((uint8_t*)rows + row_bytes);
        const float* lw = xs + F;
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s;
        for (int f = fg; f < F; f += G) {
          float4 v = *reinterpret_cast<const float4*>(rows + (size_t)f * K + 4 * q);
          if (f >= first_dense) {               // dense field: value * embedding row (features.py:121-148)
            const float xv = xs[f];
            v.x *= xv; v.y *= xv; v.z *= xv; v.w *= xv;
            if (o.concat) *reinterpret_cast<float4*>(rows + (size_t)f * K + 4 * q) = v;
          }
          s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
          s2.x = fmaf(v.x, v.x, s2.x); s2.y = fmaf(v.y, v.y, s2.y);
          s2.z = fmaf(v.z, v.z, s2.z); s2.w = fmaf(v.w, v.w, s2.w);
        }
        float lin_acc = 0.f;
        if (want_lin) {
          for (int f = lane; f < F; f += 32) lin_acc += lw[f];
          lin_acc = warp_sum(lin_acc) + h.lin_bias;
        }
        if (o.concat) {   // the [F][K] image in shared memory IS the concatenated row: one bulk store
          asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
          __syncwarp();
          if (lane == 0) {
            bulk_s2g(o.concat + r * o.ld_concat, rows, (uint32_t)row_bytes);
            bulk_commit();
          }
        }
        if (o.pw || o.fm_out || o.ssum) {
          // reduce over the G field groups (lanes with equal q): xor-shuffles over the group bits
#pragma unroll
          for (int off = K4; off < 32; off <<= 1) {
            s.x += __shfl_xor_sync(0xffffffffu, s.x, off); s.y += __shfl_xor_sync(0xffffffffu, s.y, off);
            s.z += __shfl_xor_sync(0xffffffffu, s.z, off); s.w += __shfl_xor_sync(0xffffffffu, s.w, off);
            s2.x += __shfl_xor_sync(0xffffffffu, s2.x, off); s2.y += __shfl_xor_sync(0xffffffffu, s2.y, off);
            s2.z += __shfl_xor_sync(0xffffffffu, s2.z, off); s2.w += __shfl_xor_sync(0xffffffffu, s2.w, off);
          }
          float head_acc = 0.f;
          const float sv[4] = {s.x, s.y, s.z, s.w}, s2v[4] = {s2.x, s2.y, s2.z, s2.w};
#pragma unroll
          for (int c = 0; c < 4; ++c) {
            const int k = 4 * q + c;
            const float pw = 0.5f * (sv[c] * sv[c] - s2v[c]);
            if (fg == 0) {
              if (o.pw) o.pw[r * o.ld_pw + k] = pw;
              if (o.ssum) { o.ssum[r * o.ld_s + k] = sv[c]; o.sqsum[r * o.ld_s + k] = s2v[c]; }
              if (o.fm_out) {
                const float z = h.bn_scale ? fmaf(pw, h.bn_scale[k], h.bn_shift[k]) : pw;
                head_acc = fmaf(z, h.pw_kernel[k], head_acc);
              }
            }
          }
          if (o.fm_out) {
            head_acc = warp_sum(head_acc) + h.pw_bias;     // lanes with fg != 0 contribute 0
            if (lane == 0) o.fm_out[r] = lin_acc + (head_acc > 0.f ? head_acc : expm1f(head_acc));
          }
        }
        if (o.lin && lane == 0) o.lin[r] = lin_acc;
        if (o.concat && lane == 0) bulk_wait_read0();   // the stage may be refilled once the store has READ it
      }
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&empty[stage]);
      if (++stage == FT_NSTAGE) { stage = 0; phase ^= 1; }
    }
    if (o.concat && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // stores landed
  }
}

// returns 1 when the staged kernel was launched, 0 when the shape is not eligible, < 0 on error
int launch_feat_forward_tma(const b200_feat_layout* L, const b200_feat_tables* T, const int64_t* users,
                            const int64_t* items, int64_t R, int64_t grid_items, int64_t row_offset,
                            float* concat, int64_t ld_concat, float* pw, int64_t ld_pw, float* lin,
                            float* fm_out, const float* lin_kernel, float lin_bias, const float* bn_scale,
                            const float* bn_shift, const float* pw_kernel, float pw_bias, float* ssum,
                            float* sqsum, int64_t ld_s, cudaStream_t stream) {
  const int K = L->embed_size;
  if (K % 4 != 0 || K > 32 || R < 2048) return 0;
  const int n_id = ((L->id_mask & 1) ? 1 : 0) + ((L->id_mask & 2) ? 1 : 0);
  const int F = n_id + L->n_sparse + L->n_dense;
  if (F < 1 || F > 32 * FT_MAX_FJ) return 0;
  const size_t row_bytes = (size_t)F * K * 4;
  const size_t aux_bytes = ((size_t)F * 4 * 2 + 15) & ~(size_t)15;
  // rows per stage: as many as fit ~100 KB for the 3-stage ring (two CTAs per SM), at most 8
  int RB = FT_MAX_RB;
  while (RB > 1 && FT_NSTAGE * RB * (row_bytes + aux_bytes) > 100 * 1024) RB >>= 1;
  const size_t smem = 128 + FT_NSTAGE * RB * (row_bytes + aux_bytes) + 2 * FT_NSTAGE * 8 + 64;
  if (smem > 220 * 1024) return 0;
  FtOut o; o.concat = concat; o.ld_concat = ld_concat; o.pw = pw; o.ld_pw = ld_pw; o.lin = lin; o.fm_out = fm_out;
  o.ssum = ssum; o.sqsum = sqsum; o.ld_s = ld_s;
  FtHead h; h.lin_kernel = lin_kernel; h.lin_bias = lin_bias; h.bn_scale = bn_scale; h.bn_shift = bn_shift;
  h.pw_kernel = pw_kernel; h.pw_bias = pw_bias;
  const int sm_count = num_sms();
  B200_REQUIRE(sm_count > 0, "no CUDA device");
  const int ctas_per_sm = smem <= 110 * 1024 ? 2 : 1;
  const int64_t n_batches = (R + RB - 1) / RB;
  const int64_t want = (int64_t)sm_count * ctas_per_sm;
  const unsigned grid = (unsigned)(n_batches < want ? n_batches : want);
  const unsigned threads = 32 * (1 + RB);
#define FT_LAUNCH(K4)                                                                                          \
  {                                                                                                            \
    static bool attr = false;                                                                                  \
    if (!attr) {                                                                                               \
      B200_CUDA_OK(cudaFuncSetAttribute(feat_forward_tma_kernel<K4>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                        220 * 1024));                                                          \
      attr = true;                                                                                             \
    }                                                                                                          \
    feat_forward_tma_kernel<K4><<<grid, threads, smem, stream>>>(*L, *T, users, items, R, grid_items, row_offset, \
                                                                 o, h, RB);                                    \
  }
  switch (K / 4) {
    case 1: FT_LAUNCH(1); break;
    case 2: FT_LAUNCH(2); break;
    case 4: FT_LAUNCH(4); break;
    case 8: FT_LAUNCH(8); break;
    default: return 0;        // K = 12, 20, 24, 28: 32 / K4 is not integral -> register kernel
  }
#undef FT_LAUNCH
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 1;
}

}  // namespace feat
}  // namespace b200
