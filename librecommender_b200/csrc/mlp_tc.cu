// Dense layer on the Hopper tensor cores (wgmma) with fp32-level accuracy: Y = act(X Wt^T + b).
//
// Replaces tf_dense (reference libreco/layers/dense.py:52-80, BN folded by the caller) for the MLP
// tails of DeepFM / DIN / YouTubeRanking / TwoTower when the layer is large enough to be
// compute-bound on the SIMT path (b200_linear_f32).  The reference computes these layers in fp32
// (TensorFlow MatMul); a plain tf32 or bf16 tensor-core GEMM would miss the 1e-5 parity bar, so
// the operands are split  x = hi + lo  (hi = top 11 mantissa bits, lo = next 11) and three
// wgmma tf32 products are accumulated:  hi*hi + lo*hi + hi*lo  (truncation keeps 10 explicit
// mantissa bits, |lo| < 2^-10 |x|: the dropped lo*lo term is < 2^-20 |x||w| and the two truncated
// cross terms add < 2^-20 each; tests/test_tf32x3_model_cpu.py).  Both hi and lo are written
// explicitly (hi in place of the loaded tile), so the result does not depend on how the tensor core
// treats the 13 low mantissa bits of an fp32 container.  The dominant hi*hi products and the
// 2^-11-times smaller cross products go to SEPARATE wgmma accumulators, and both are promoted to
// fp32 registers (round-to-nearest adds) every GC k-chunks, so no accumulator runs over many MMAs.
// Unlike b200_linear_f32 it does not carry +-inf inputs through: the lo part of +-inf is inf - inf = NaN, so
// an output that b200_linear_f32 gives as +-inf comes out NaN here (finite inputs only).
//
// One persistent CTA per SM, warp-specialised:
//   warpgroups 0-1  split the landed tiles into hi / lo, issue the wgmma of rows [64 g, 64 g + 64) of
//                   the 128-row tile, promote, and run the bias / ReLU / store epilogue
//   warp 8          TMA producer: X tile [128 x 32 fp32] and Wt tile [n_pad x 32 fp32] per k-chunk
//                   (the weight tiles arrive pre-split when the caller made a split copy)
#include <type_traits>
#include "common.cuh"
#include "ptx_sm90.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace mlp {

constexpr int TM = 128;          // rows per tile (two wgmma M = 64 warpgroups)
constexpr int KC = 32;           // fp32 per k-chunk = one 128-byte swizzled row
constexpr int GC = 2;            // k-chunks per accumulator group (promotion interval = 64 k)
constexpr int NMAX = 128;        // output columns per CTA (grid.y covers wider layers)
constexpr int MAXSTAGE = 4;
constexpr int CONSUMER_THREADS = 256;
constexpr int THREADS = CONSUMER_THREADS + 128;   // + the producer warpgroup
constexpr int PRODUCER_REGS = 40, CONSUMER_REGS = 232;
constexpr int A_BYTES = TM * KC * 4;   // 16 KB

struct Params {
  int64_t R;
  int64_t ldy;
  const float* bias;
  float* Y;
  const float* dot_w;     // fused DIN epilogue: 16 weights of the Dense(1) on sigmoid(Dense(16)) (NULL = plain layer)
  int din, dout, n_pad, act;
  int n_tiles, n_chunks, nstage;
  int n_chunks_total;      // split-K: CTA z takes k-chunks [z * n_chunks, min((z + 1) * n_chunks, n_chunks_total))
  int64_t split_stride;    //          and writes its partial product to Y + z * split_stride (no bias / ReLU)
};

struct Smem {
  uint64_t full[MAXSTAGE], empty[MAXSTAGE];
  float bias_s[NMAX];      // bias of this CTA's column block (0 past dout / without bias)
};

__device__ __forceinline__ float hi_part(float x) { return __uint_as_float(__float_as_uint(x) & 0xffffe000u); }

// x -> (hi, lo): hi keeps the 10 explicit mantissa bits of tf32, lo = x - hi (exact in fp32).
__device__ __forceinline__ void split4(float4* hi, float4* lo) {
  const float4 v = *hi;
  const float4 h = make_float4(hi_part(v.x), hi_part(v.y), hi_part(v.z), hi_part(v.w));
  *hi = h;
  *lo = make_float4(v.x - h.x, v.y - h.y, v.z - h.z, v.w - h.w);
}

// weights: explicit hi / lo copies, made once per layer (b200_linear_tf32x3_split_weights)
__global__ void split_weights_kernel(const float* __restrict__ W, int64_t ldw, int din, int dout, int64_t ld,
                                     float* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)dout * ld) return;
  const int r = (int)(i / ld), c = (int)(i % ld);
  const float x = c < din ? W[(int64_t)r * ldw + c] : 0.f;
  const float h = hi_part(x);
  out[i] = h;
  out[(int64_t)dout * ld + i] = x - h;
}

// D (+)= A B^T for one k8 step at N = NP
template <int NP>
__device__ __forceinline__ void mma_tf32(float (&d)[NP / 2], uint64_t da, uint64_t db, bool first) {
  if constexpr (NP == 32) { if (first) ptx::wgmma_tf32_n32_first(d, da, db); else ptx::wgmma_tf32_n32(d, da, db); }
  if constexpr (NP == 64) { if (first) ptx::wgmma_tf32_n64_first(d, da, db); else ptx::wgmma_tf32_n64(d, da, db); }
  if constexpr (NP == 96) { if (first) ptx::wgmma_tf32_n96_first(d, da, db); else ptx::wgmma_tf32_n96(d, da, db); }
  if constexpr (NP == 128) { if (first) ptx::wgmma_tf32_n128_first(d, da, db); else ptx::wgmma_tf32_n128(d, da, db); }
}

// WSPLIT: tmW / tmWlo address the pre-split weight copies; otherwise the consumers also split the
// weight tile of every stage (self-contained call, more shared-memory traffic).  NP = n_pad.
template <bool WSPLIT, bool DOT, int NP>
__global__ void __launch_bounds__(THREADS, 1)
linear_tf32x3_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW,
                     const __grid_constant__ CUtensorMap tmWlo, const Params p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = (uint8_t*)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
  constexpr int b_bytes = NP * KC * 4;
  constexpr int stage_bytes = 2 * A_BYTES + 2 * b_bytes;
  Smem* ss = (Smem*)(smem + (size_t)p.nstage * stage_bytes);

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int col0 = blockIdx.y * NMAX;
  const int kc_base = blockIdx.z * p.n_chunks;
  const int kc_count = min(p.n_chunks, p.n_chunks_total - kc_base);

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.nstage; ++s) {
      ptx::mbar_init(&ss->full[s], 1);
      ptx::mbar_init(&ss->empty[s], CONSUMER_THREADS / 32);
    }
    ptx::fence_barrier_init();
    ptx::prefetch_tensormap(&tmX);
    ptx::prefetch_tensormap(&tmW);
  }
  if (threadIdx.x < NMAX) {
    const int c = threadIdx.x;
    ss->bias_s[c] = (p.bias && col0 + c < p.dout) ? __ldg(p.bias + col0 + c) : 0.f;
  }
  __syncthreads();

  if (threadIdx.x >= CONSUMER_THREADS) {
    ptx::setmaxnreg_dec<PRODUCER_REGS>();
    // ===================== TMA producer =====================
    if (threadIdx.x == CONSUMER_THREADS) {
      int stage = 0;
      uint32_t phase = 0;
      for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
        for (int kc = 0; kc < kc_count; ++kc) {
          ptx::mbar_wait(&ss->empty[stage], phase ^ 1);
          ptx::mbar_arrive_expect_tx(&ss->full[stage], (uint32_t)(A_BYTES + (WSPLIT ? 2 : 1) * b_bytes));
          uint8_t* st = smem + (size_t)stage * stage_bytes;
          const int kx = (kc_base + kc) * KC;
          ptx::tma_load_2d(st, &tmX, &ss->full[stage], kx, tile * TM);
          ptx::tma_load_2d(st + 2 * A_BYTES, &tmW, &ss->full[stage], kx, col0);
          if (WSPLIT) ptx::tma_load_2d(st + 2 * A_BYTES + b_bytes, &tmWlo, &ss->full[stage], kx, col0);
          if (++stage == p.nstage) { stage = 0; phase ^= 1; }
        }
      }
    }
    return;
  }

  // ===================== consumers: split, MMA, promote, epilogue =====================
  ptx::setmaxnreg_inc<CONSUMER_REGS>();
  const int t = threadIdx.x;                 // 0..255
  const int g = warp >> 2;
  const int quad = lane >> 2, tq = lane & 3;
  const int trow0 = 64 * g + 16 * (warp & 3) + quad;   // rows trow0 and trow0 + 8 of the tile
  const uint32_t s_addr = ptx::smem_u32(smem);
  int stage = 0;
  uint32_t phase = 0;
  float acc_main[NP / 2], acc_corr[NP / 2];
  for (int tile = blockIdx.x; tile < p.n_tiles; tile += gridDim.x) {
    float y[NP / 2];
#pragma unroll
    for (int i = 0; i < NP / 2; ++i) y[i] = 0.f;
    for (int kc = 0; kc < kc_count; ++kc) {
      const int gpos = kc % GC;
      ptx::mbar_wait(&ss->full[stage], phase);
      uint8_t* st = smem + (size_t)stage * stage_bytes;
#pragma unroll
      for (int j = 0; j < A_BYTES / 16 / CONSUMER_THREADS; ++j)
        split4((float4*)st + t + j * CONSUMER_THREADS, (float4*)(st + A_BYTES) + t + j * CONSUMER_THREADS);
      if (!WSPLIT)
        for (int j = t; j < b_bytes / 16; j += CONSUMER_THREADS)
          split4((float4*)(st + 2 * A_BYTES) + j, (float4*)(st + 2 * A_BYTES + b_bytes) + j);
      ptx::fence_proxy_async_smem();         // generic-proxy writes -> visible to the tensor core
      ptx::named_bar_sync(1, CONSUMER_THREADS);
      ptx::wgmma_fence();
      const uint32_t sa = s_addr + (uint32_t)(stage * stage_bytes) + (uint32_t)(g * 64 * KC * 4);
      const uint64_t a_hi = ptx::wgmma_desc_sw128_kmajor(sa);
      const uint64_t a_lo = ptx::wgmma_desc_sw128_kmajor(sa + A_BYTES);
      const uint64_t b_hi = ptx::wgmma_desc_sw128_kmajor(s_addr + (uint32_t)(stage * stage_bytes + 2 * A_BYTES));
      const uint64_t b_lo = ptx::wgmma_desc_sw128_kmajor(s_addr + (uint32_t)(stage * stage_bytes + 2 * A_BYTES + b_bytes));
#pragma unroll
      for (int k4 = 0; k4 < KC / 8; ++k4) {
        // 8 tf32 = 32 bytes per MMA inside the 128-byte swizzled row: +2 in the >>4 field
        const uint64_t o = (uint64_t)(k4 * 2);
        const bool first = gpos == 0 && k4 == 0;
        mma_tf32<NP>(acc_main, a_hi + o, b_hi + o, first);
        mma_tf32<NP>(acc_corr, a_lo + o, b_hi + o, first);
        mma_tf32<NP>(acc_corr, a_hi + o, b_lo + o, false);
      }
      ptx::wgmma_commit();
      ptx::wgmma_wait<0>(acc_main);
      ptx::wgmma_wait<0>(acc_corr);
      __syncwarp();
      if (lane == 0) ptx::mbar_arrive(&ss->empty[stage]);
      if (++stage == p.nstage) { stage = 0; phase ^= 1; }
      if (gpos == GC - 1 || kc == kc_count - 1) {
#pragma unroll
        for (int i = 0; i < NP / 2; ++i) y[i] = (y[i] + acc_corr[i]) + acc_main[i];   // correction first
      }
    }
    // fragment: y[4 j + 2 rs + e] = row trow0 + 8 rs, column 8 j + 2 tq + e
    const int ncol = min(p.dout - col0, NMAX);
#pragma unroll
    for (int rs = 0; rs < 2; ++rs) {
      const int64_t row = (int64_t)tile * TM + trow0 + 8 * rs;
      if (DOT) {
        // fused attention epilogue (DIN all-items): per group of 16 columns ONE output
        //   a[row, (col0 + 16 g) / 16] = sum_j dot_w[j] * sigmoid(y[16 g + j] + bias)
        // the [R, dout] pre-activations (16x the bytes) are never written
        float* yd = p.Y + row * p.ldy + col0 / 16;
#pragma unroll
        for (int gg = 0; gg < NP / 16; ++gg) {
          float a = 0.f;
#pragma unroll
          for (int h = 0; h < 2; ++h)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
              const int cj = 8 * h + 2 * tq + e;          // column inside the group of 16
              const float v = y[4 * (2 * gg + h) + 2 * rs + e] + ss->bias_s[16 * gg + cj];
              a = fmaf(__ldg(p.dot_w + cj), 1.0f / (1.0f + expf(-v)), a);
            }
          a += __shfl_xor_sync(0xffffffffu, a, 1);
          a += __shfl_xor_sync(0xffffffffu, a, 2);
          if (tq == 0 && gg * 16 < ncol && row < p.R) yd[gg] = a;
        }
      } else if (row < p.R) {
        float* yr = p.Y + (int64_t)blockIdx.z * p.split_stride + row * p.ldy + col0;
        const bool vec = ((p.ldy & 1) == 0) && ((((uintptr_t)p.Y) & 7) == 0);
#pragma unroll
        for (int j = 0; j < NP / 8; ++j) {
          const int c = 8 * j + 2 * tq;
          float o[2];
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const float v = y[4 * j + 2 * rs + e] + ss->bias_s[c + e];
            o[e] = apply_act(v, p.act);
          }
          if (vec && c + 1 < ncol) {
            *(float2*)(yr + c) = make_float2(o[0], o[1]);
          } else {
            if (c < ncol) yr[c] = o[0];
            if (c + 1 < ncol) yr[c + 1] = o[1];
          }
        }
      }
    }
  }
}


// split-K: Y[r, c] = act(sum_z part[z][r, c] + bias[c]) in a fixed order (deterministic)
__global__ void splitk_reduce_kernel(const float* __restrict__ part, int splits, int64_t R, int dout,
                                     const float* __restrict__ bias, int act, float* __restrict__ Y, int64_t ldy) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * dout) return;
  const int64_t r = i / dout;
  const int c = (int)(i % dout);
  float v = 0.f;
  for (int z = 0; z < splits; ++z) v += part[(int64_t)z * R * dout + i];
  if (bias) v += __ldg(bias + c);
  Y[r * ldy + c] = apply_act(v, act);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
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

// fp32 [rows, cols] row-major with leading dimension ld; box = [KC, box_rows], SWIZZLE_128B;
// out-of-range elements (k >= cols, row >= rows) read as zero
static int make_tmap_f32(CUtensorMap* m, const float* base, int64_t rows, int64_t cols, int64_t ld,
                         int box_rows) {
  EncodeTiledFn enc = encode_fn();
  B200_REQUIRE(enc, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)ld * 4};
  cuuint32_t box[2] = {(cuuint32_t)KC, (cuuint32_t)box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<float*>(base), dims, strides, box,
                   estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                   CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  B200_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return 0;
}

}  // namespace mlp
}  // namespace b200

extern "C" int64_t b200_linear_tf32x3_split_ld(int32_t din) { return ((int64_t)din + 3) / 4 * 4; }

extern "C" int b200_linear_tf32x3_split_weights(const float* Wt, int64_t ldw, int32_t din, int32_t dout,
                                                float* Wsplit, void* stream) {
  using namespace b200;
  using namespace b200::mlp;
  B200_REQUIRE(Wt && Wsplit && din > 0 && dout > 0 && ldw >= din, "bad arguments");
  const int64_t ld = b200_linear_tf32x3_split_ld(din);
  const int64_t n = (int64_t)dout * ld;
  split_weights_kernel<<<(unsigned)((n + 255) / 256), 256, 0, (cudaStream_t)stream>>>(Wt, ldw, din, dout, ld, Wsplit);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

static int launch_linear_tf32x3(const float* X, int64_t ldx, int64_t R, const float* Wt, int64_t ldw,
                                const float* Wsplit, const float* bias, int32_t din, int32_t dout,
                                int32_t act, const float* dot_w, float* Y, int64_t ldy, void* stream,
                                int splits = 1, float* workspace = nullptr);

extern "C" int b200_linear_tf32x3(const float* X, int64_t ldx, int64_t R, const float* Wt, int64_t ldw,
                                  const float* Wsplit, const float* bias, int32_t din, int32_t dout,
                                  int32_t act, float* Y, int64_t ldy, void* stream) {
  B200_REQUIRE(ldy >= dout, "leading dimension too small");
  return launch_linear_tf32x3(X, ldx, R, Wt, ldw, Wsplit, bias, din, dout, act, nullptr, Y, ldy, stream);
}

extern "C" int b200_linear_tf32x3_sigmoid_dot(const float* X, int64_t ldx, int64_t R, const float* Wt, int64_t ldw,
                                              const float* Wsplit, const float* bias, int32_t din, int32_t dout,
                                              const float* dot_w16, float* A, int64_t lda, void* stream) {
  B200_REQUIRE(dot_w16 && A, "b200_linear_tf32x3_sigmoid_dot: null pointer");
  B200_REQUIRE(dout % 16 == 0 && lda >= dout / 16, "b200_linear_tf32x3_sigmoid_dot: dout must be a multiple of 16, lda >= dout / 16");
  return launch_linear_tf32x3(X, ldx, R, Wt, ldw, Wsplit, bias, din, dout, 0, dot_w16, A, lda, stream);
}

extern "C" int b200_linear_tf32x3_splitk(const float* X, int64_t ldx, int64_t R, const float* Wt, int64_t ldw,
                                         const float* bias, int32_t din, int32_t dout, int32_t act, int32_t splits,
                                         float* workspace, size_t workspace_bytes, float* Y, int64_t ldy, void* stream) {
  B200_REQUIRE(splits >= 1 && splits <= 64, "b200_linear_tf32x3_splitk: splits outside [1, 64]");
  B200_REQUIRE(ldy >= dout, "leading dimension too small");
  B200_REQUIRE(splits == 1 || (workspace && workspace_bytes >= (size_t)splits * (size_t)R * (size_t)dout * 4),
               "b200_linear_tf32x3_splitk: workspace too small (splits * R * dout floats)");
  return launch_linear_tf32x3(X, ldx, R, Wt, ldw, nullptr, bias, din, dout, act, nullptr, Y, ldy, stream, splits,
                              workspace);
}

static int launch_linear_tf32x3(const float* X, int64_t ldx, int64_t R, const float* Wt, int64_t ldw,
                                const float* Wsplit, const float* bias, int32_t din, int32_t dout,
                                int32_t act, const float* dot_w, float* Y, int64_t ldy, void* stream,
                                int splits, float* workspace) {
  using namespace b200;
  using namespace b200::mlp;
  B200_REQUIRE(R >= 0 && din > 0 && dout > 0, "bad shape");
  B200_REQUIRE(act >= 0 && act <= 2, "b200_linear_tf32x3: activation code %d outside [0, 2]", act);
  B200_REQUIRE((ldx & 3) == 0 && ((uintptr_t)X & 15) == 0, "b200_linear_tf32x3 needs 16-byte aligned X rows (ldx % 4 == 0)");
  B200_REQUIRE(Wsplit ? (((uintptr_t)Wsplit & 15) == 0) : ((ldw & 3) == 0 && ((uintptr_t)Wt & 15) == 0),
               "b200_linear_tf32x3 needs 16-byte aligned weight rows (ldw % 4 == 0) or a split copy");
  B200_REQUIRE(ldx >= din && (Wsplit || ldw >= din), "leading dimension too small");
  if (R == 0) return 0;
  Params p;
  p.dot_w = dot_w;
  p.R = R;
  p.ldy = ldy;
  p.bias = bias;
  p.Y = Y;
  p.din = din;
  p.dout = dout;
  p.act = act;
  p.n_pad = dout >= NMAX ? NMAX : (dout + 31) / 32 * 32;
  p.n_tiles = (int)((R + TM - 1) / TM);
  p.n_chunks_total = (din + KC - 1) / KC;
  p.n_chunks = (p.n_chunks_total + splits - 1) / splits;
  splits = (p.n_chunks_total + p.n_chunks - 1) / p.n_chunks;        // no empty split
  p.split_stride = 0;
  if (splits > 1) {   // partial products [splits][R, dout] into the workspace, bias / activation in the reduction
    p.split_stride = R * (int64_t)dout;
    p.Y = workspace;
    p.ldy = dout;
    p.bias = nullptr;
    p.act = 0;
  }
  const int stage_bytes = 2 * A_BYTES + 2 * p.n_pad * KC * 4;
  p.nstage = min(MAXSTAGE, (200 * 1024) / stage_bytes);
  const size_t smem = (size_t)p.nstage * stage_bytes + sizeof(Smem) + 1024;

  CUtensorMap tmX, tmW, tmWlo;
  if (make_tmap_f32(&tmX, X, R, din, ldx, TM)) return 1;
  if (Wsplit) {
    const int64_t ld = b200_linear_tf32x3_split_ld(din);
    if (make_tmap_f32(&tmW, Wsplit, dout, din, ld, p.n_pad)) return 1;
    if (make_tmap_f32(&tmWlo, Wsplit + (int64_t)dout * ld, dout, din, ld, p.n_pad)) return 1;
  } else {
    if (make_tmap_f32(&tmW, Wt, dout, din, ldw, p.n_pad)) return 1;
    tmWlo = tmW;
  }

  const int sms = num_sms();
  B200_REQUIRE(sms > 0, "no CUDA device");
  const int gy = (dout + NMAX - 1) / NMAX;
  const int gx = max(1, min(p.n_tiles, sms / (gy * splits)));
  const dim3 grid(gx, gy, splits);
  cudaStream_t st = (cudaStream_t)stream;
  auto launch = [&](auto kernel) -> int {
    B200_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024));
    kernel<<<grid, THREADS, smem, st>>>(tmX, tmW, tmWlo, p);
    return 0;
  };
  auto by_width = [&](auto wsplit, auto dot) -> int {
    constexpr bool WS = decltype(wsplit)::value, DT = decltype(dot)::value;
    switch (p.n_pad) {
      case 32: return launch(linear_tf32x3_kernel<WS, DT, 32>);
      case 64: return launch(linear_tf32x3_kernel<WS, DT, 64>);
      case 96: return launch(linear_tf32x3_kernel<WS, DT, 96>);
      default: return launch(linear_tf32x3_kernel<WS, DT, 128>);
    }
  };
  using T = std::true_type;
  using F = std::false_type;
  int rc;
  if (dot_w) rc = Wsplit ? by_width(T{}, T{}) : by_width(F{}, T{});
  else rc = Wsplit ? by_width(T{}, F{}) : by_width(F{}, F{});
  if (rc) return rc;
  if (splits > 1) {
    const int64_t n = R * (int64_t)dout;
    splitk_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(workspace, splits, R, dout, bias, act, Y, ldy);
    count_launch();
  }
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}
