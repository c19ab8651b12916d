// ALS training — one half-epoch of the per-row least squares of libreco/algorithms/_als.pyx.
//
// Every row m of X [n_x, d] is solved against the fixed other-side table Y [n_y, d] given that side's CSR
// (indptr int64, indices int32, data float32).  A0 is the base matrix the host computes once per call
// (implicit: Y^T Y + reg I, explicit: reg I).
//
//   CG (_least_squares_cg, _als.pyx:167-268), warm-started from X[m], cg_steps iterations:
//     r  = -A0 x + sum (c - (c-1) y.x) y          (implicit)      r  = -A0 x + sum (r_ui - y.x) y   (explicit)
//     Ap =  A0 p + sum (c-1)(y.p) y               (implicit)      Ap =  A0 p + sum (y.p) y          (explicit)
//     with the reference's two absolute exits: rsold < 1e-10 leaves X[m] untouched, rsnew < 1e-10 breaks
//     after x and r are updated.
//   Direct (_least_squares, _als.pyx:96-164): A = A0 + sum w y y^T, b = sum c y (w = c-1 / 1), then a Cholesky
//     factorisation and two triangular solves in shared memory.  A pivot <= 0 or NaN at column j fails the row
//     with info = j+1 (LAPACK spotrf's test); the row is not written and the smallest failing row is recorded.
//
// Row classes (the plan is built on the device by the host, once per CSR):
//   short rows (nnz <= LONG_ROW):  CG — one warp per row, 8 rows per CTA, A0 in shared memory for the CTA.  A
//                                  row's Y slice is staged once in shared memory by cp.async when it fits
//                                  (stage_rows(d) rows), so the 1 + cg_steps passes read SMEM; longer short
//                                  rows read their Y rows through L2 in every pass.
//                                  Direct — one CTA per row, A accumulated in registers over staged Y tiles.
//   long rows (nnz > LONG_ROW):    fixed CHUNK-nnz pieces, one warp (CG) or CTA (direct) per piece, writing
//                                  partial sums; one small per-row kernel adds them in chunk order and does the
//                                  vector update (CG: one chunk + one update launch per pass for all long rows).
// Deterministic: no float atomics; every sum runs in a fixed order.  fp32 SIMT.
#include <type_traits>

#include "common.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace als {

constexpr int LONG_ROW = 2048;      // rows above this go to the chunked path
constexpr int CHUNK = 1024;         // nnz per chunk of a long row
constexpr int MAX_D = 128;
constexpr int CG_WARPS = 8;         // rows per CTA of the short-row CG kernel
constexpr int STAGE_FLOATS = 4096;  // per-warp Y staging buffer (16 KB)
constexpr int DIRECT_THREADS = 512;
constexpr int DIRECT_TILE = 32;     // Y rows per staged tile of the direct path

__host__ __device__ inline int stage_rows(int d) { return STAGE_FLOATS / d; }

__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
  const uint32_t s = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(s), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
  asm volatile("cp.async.commit_group;\ncp.async.wait_group 0;" ::: "memory");
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

struct Args {
  const int64_t* indptr;
  const int32_t* indices;
  const float* data;
  float* X;
  const float* Y;
  const float* A0;
  int d, implicit, cg_steps;
};

// a lane's share of a d-vector: elements lane + 32 t, t < T = ceil(d / 32) rounded up to 1, 2 or 4 (zero past d)
template <int T>
struct Vec {
  float v[T];
};

template <int T>
__device__ __forceinline__ float dot(const Vec<T>& a, const Vec<T>& b) {
  float s = 0.f;
#pragma unroll
  for (int t = 0; t < T; ++t) s = fmaf(a.v[t], b.v[t], s);
  return warp_sum(s);
}

template <int T>
__device__ __forceinline__ void load_vec(Vec<T>& o, const float* p, int d, int lane) {
#pragma unroll
  for (int t = 0; t < T; ++t) {
    const int j = lane + 32 * t;
    o.v[t] = j < d ? p[j] : 0.f;
  }
}

template <int T>
__device__ __forceinline__ void store_vec(float* p, const Vec<T>& o, int d, int lane) {
#pragma unroll
  for (int t = 0; t < T; ++t) {
    const int j = lane + 32 * t;
    if (j < d) p[j] = o.v[t];
  }
}

// o = s * (A0 v); A0 symmetric in shared memory, read by columns so that lanes hit distinct banks.  `buf` is the
// warp's d-float broadcast buffer.
template <int T>
__device__ __forceinline__ void symv(Vec<T>& o, const float* A0s, const Vec<T>& v, float s, float* buf, int d,
                                     int lane) {
  store_vec(buf, v, d, lane);
  __syncwarp();
#pragma unroll
  for (int t = 0; t < T; ++t) o.v[t] = 0.f;
  for (int k = 0; k < d; ++k) {
    const float vk = buf[k];
#pragma unroll
    for (int t = 0; t < T; ++t) {
      const int j = lane + 32 * t;
      if (j < d) o.v[t] = fmaf(A0s[k * d + j], vk, o.v[t]);
    }
  }
#pragma unroll
  for (int t = 0; t < T; ++t) o.v[t] *= s;
  __syncwarp();
}

// acc += sum over nnz [beg, end) of coef(y.v, value) * y, in nnz order.  phase 0 (residual) uses
// coef = c - (c-1) y.v (implicit) or r_ui - y.v; a CG step uses (c-1) y.v or y.v.  Y rows come from `stage`
// (row q of the slice at stage + q * d) when it is non-null, else from global memory.
template <int PHASE0, int T>
__device__ __forceinline__ void accumulate(const Args& a, int64_t beg, int64_t end, const float* stage,
                                           const Vec<T>& v, Vec<T>& acc, int lane) {
  const int d = a.d;
  constexpr int U = 8;   // nnz per group: their dot products share one shuffle tree
  int64_t i = beg;
  for (; i + U <= end; i += U) {
    Vec<T> y[U];
    float c[U], s[U];
#pragma unroll
    for (int u = 0; u < U; ++u) {
      const float* yr = stage ? stage + (i + u - beg) * d : a.Y + (int64_t)__ldg(a.indices + i + u) * d;
      load_vec(y[u], yr, d, lane);
      c[u] = __ldg(a.data + i + u);
      float p = 0.f;
#pragma unroll
      for (int t = 0; t < T; ++t) p = fmaf(y[u].v[t], v.v[t], p);
      s[u] = p;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
      for (int u = 0; u < U; ++u) s[u] += __shfl_xor_sync(0xffffffffu, s[u], o);
#pragma unroll
    for (int u = 0; u < U; ++u) {
      float w;
      if (PHASE0) w = a.implicit ? __fsub_rn(c[u], __fmul_rn(__fsub_rn(c[u], 1.f), s[u])) : __fsub_rn(c[u], s[u]);
      else w = a.implicit ? __fmul_rn(__fsub_rn(c[u], 1.f), s[u]) : s[u];
#pragma unroll
      for (int t = 0; t < T; ++t) acc.v[t] = fmaf(w, y[u].v[t], acc.v[t]);
    }
  }
  for (; i < end; ++i) {
    Vec<T> y;
    const float* yr = stage ? stage + (i - beg) * d : a.Y + (int64_t)__ldg(a.indices + i) * d;
    load_vec(y, yr, d, lane);
    const float c = __ldg(a.data + i);
    const float s = dot(y, v);
    float w;
    if (PHASE0) w = a.implicit ? __fsub_rn(c, __fmul_rn(__fsub_rn(c, 1.f), s)) : __fsub_rn(c, s);
    else w = a.implicit ? __fmul_rn(__fsub_rn(c, 1.f), s) : s;
#pragma unroll
    for (int t = 0; t < T; ++t) acc.v[t] = fmaf(w, y.v[t], acc.v[t]);
  }
}

__device__ __forceinline__ void stage_slice(const Args& a, int64_t beg, int64_t end, float* stage, int lane) {
  const int d = a.d;
  const int n = (int)(end - beg);
  if ((d & 3) == 0) {
    const int q = d >> 2;
    for (int e = lane; e < n * q; e += 32) {
      const int r = e / q, c = e - r * q;
      cp_async16(stage + r * d + c * 4, a.Y + (int64_t)__ldg(a.indices + beg + r) * d + c * 4);
    }
  } else {
    for (int e = lane; e < n * d; e += 32) {
      const int r = e / d, c = e - r * d;
      cp_async4(stage + r * d + c, a.Y + (int64_t)__ldg(a.indices + beg + r) * d + c);
    }
  }
  cp_async_wait_all();
  __syncwarp();
}

// x += ak p; r -= ak Ap; rsnew = r.r; returns true when the reference breaks (rsnew < 1e-10), else
// p = r + (rsnew / rsold) p and rsold = rsnew.
template <int T>
__device__ __forceinline__ bool cg_update(Vec<T>& x, Vec<T>& r, Vec<T>& p, const Vec<T>& Ap, float& rsold) {
  const float ak = rsold / dot(p, Ap);
#pragma unroll
  for (int t = 0; t < T; ++t) {
    x.v[t] = fmaf(ak, p.v[t], x.v[t]);
    r.v[t] = fmaf(-ak, Ap.v[t], r.v[t]);
  }
  const float rsnew = dot(r, r);
  if ((double)rsnew < 1e-10) return true;
  const float beta = rsnew / rsold;
#pragma unroll
  for (int t = 0; t < T; ++t) p.v[t] = fmaf(1.f, r.v[t], p.v[t] * beta);
  rsold = rsnew;
  return false;
}

__device__ __forceinline__ void load_A0(const float* A0, float* A0s, int d) {
  for (int e = threadIdx.x; e < d * d; e += blockDim.x) A0s[e] = A0[e];
  __syncthreads();
}

// ---- CG, short rows: one warp per row ------------------------------------------------------------------------
template <int T>
__global__ void __launch_bounds__(CG_WARPS * 32) cg_rows_kernel(Args a, const int32_t* __restrict__ rows,
                                                                int64_t n_rows) {
  extern __shared__ __align__(16) float smem[];
  const int d = a.d, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float* A0s = smem;
  float* stage = smem + ((d * d + 3) & ~3) + w * (STAGE_FLOATS + MAX_D);
  float* buf = stage + STAGE_FLOATS;
  load_A0(a.A0, A0s, d);
  const int64_t k = (int64_t)blockIdx.x * CG_WARPS + w;
  if (k >= n_rows) return;
  const int64_t m = rows[k];
  const int64_t beg = a.indptr[m], end = a.indptr[m + 1];
  const float* st = nullptr;
  if (end - beg <= stage_rows(d)) {
    stage_slice(a, beg, end, stage, lane);
    st = stage;
  }
  Vec<T> x, r, p, Ap;
  load_vec(x, a.X + m * d, d, lane);
  symv(r, A0s, x, -1.f, buf, d, lane);
  accumulate<1>(a, beg, end, st, x, r, lane);
  p = r;
  float rsold = dot(r, r);
  if ((double)rsold < 1e-10) return;
  for (int j = 0; j < a.cg_steps; ++j) {
    symv(Ap, A0s, p, 1.f, buf, d, lane);
    accumulate<0>(a, beg, end, st, p, Ap, lane);
    if (cg_update(x, r, p, Ap, rsold)) break;
  }
  store_vec(a.X + m * d, x, d, lane);
}

// ---- CG, long rows: chunk partials per pass, then one warp per row ---------------------------------------------
// per long row l the state block st + l * (3 d + 2): r[d], p[d], Ap[d], rsold, live (1.0 while iterating)
__host__ __device__ inline int64_t cg_state_floats(int d) { return 3 * (int64_t)d + 2; }

template <int T>
__global__ void cg_chunks_kernel(Args a, int phase0, const int32_t* __restrict__ chunk_long,
                                 const int32_t* __restrict__ long_rows, const int32_t* __restrict__ chunk_k,
                                 int64_t n_chunks, const float* __restrict__ st, float* __restrict__ partials) {
  const int64_t c = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (c >= n_chunks) return;
  const int d = a.d;
  const int l = chunk_long[c];
  const int64_t m = long_rows[l];
  const float* s = st + l * cg_state_floats(d);
  if (!phase0 && s[3 * d + 1] == 0.f) return;
  const int64_t beg = a.indptr[m] + (int64_t)chunk_k[c] * CHUNK;
  const int64_t end = min(beg + (int64_t)CHUNK, a.indptr[m + 1]);
  Vec<T> v, acc;
  load_vec(v, phase0 ? a.X + m * d : s + d, d, lane);
#pragma unroll
  for (int t = 0; t < T; ++t) acc.v[t] = 0.f;
  if (phase0) accumulate<1>(a, beg, end, nullptr, v, acc, lane);
  else accumulate<0>(a, beg, end, nullptr, v, acc, lane);
  store_vec(partials + c * d, acc, d, lane);
}

template <int T>
__global__ void __launch_bounds__(CG_WARPS * 32) cg_long_update_kernel(Args a, int phase0,
                                                                       const int32_t* __restrict__ long_rows,
                                                                       const int64_t* __restrict__ long_chunk_ptr,
                                                                       int64_t n_long, float* __restrict__ st,
                                                                       const float* __restrict__ partials) {
  extern __shared__ __align__(16) float smem[];
  const int d = a.d, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  float* A0s = smem;
  float* buf = smem + ((d * d + 3) & ~3) + w * MAX_D;
  load_A0(a.A0, A0s, d);
  const int64_t l = (int64_t)blockIdx.x * CG_WARPS + w;
  if (l >= n_long) return;
  const int64_t m = long_rows[l];
  float* s = st + l * cg_state_floats(d);
  if (!phase0 && s[3 * d + 1] == 0.f) return;
  Vec<T> x, r, p, Ap, part;
  load_vec(x, a.X + m * d, d, lane);
  if (phase0) {
    symv(r, A0s, x, -1.f, buf, d, lane);
#pragma unroll 1
    for (int64_t c = long_chunk_ptr[l]; c < long_chunk_ptr[l + 1]; ++c) {
      load_vec(part, partials + c * d, d, lane);
#pragma unroll
      for (int t = 0; t < T; ++t) r.v[t] += part.v[t];
    }
    const float rsold = dot(r, r);
    store_vec(s, r, d, lane);
    store_vec(s + d, r, d, lane);
    if (lane == 0) {
      s[3 * d] = rsold;
      s[3 * d + 1] = ((double)rsold < 1e-10 || a.cg_steps == 0) ? 0.f : 1.f;
    }
    return;
  }
  load_vec(r, s, d, lane);
  load_vec(p, s + d, d, lane);
  float rsold = s[3 * d];
  symv(Ap, A0s, p, 1.f, buf, d, lane);
#pragma unroll 1
  for (int64_t c = long_chunk_ptr[l]; c < long_chunk_ptr[l + 1]; ++c) {
    load_vec(part, partials + c * d, d, lane);
#pragma unroll
    for (int t = 0; t < T; ++t) Ap.v[t] += part.v[t];
  }
  const bool stop = cg_update(x, r, p, Ap, rsold);
  store_vec(a.X + m * d, x, d, lane);
  store_vec(s, r, d, lane);
  store_vec(s + d, p, d, lane);
  __syncwarp();
  if (lane == 0) {
    s[3 * d] = rsold;
    if (stop) s[3 * d + 1] = 0.f;
  }
}

// ---- direct: A = A0 + sum w y y^T, b = sum c y; one CTA per row (short) or per chunk (long) -------------------
// with R = DIRECT_THREADS / d threads per column, thread t < R d owns column k = t % d and the rows
// j = t / d + R q (q < Q, j < d) of the row-major d x d matrix, and b[t] for t < d.
struct Owner {
  int k, j0, R;
  __device__ Owner(int d) {
    R = DIRECT_THREADS / d;
    const int t = threadIdx.x;
    k = t < R * d ? t % d : 0;
    j0 = t < R * d ? t / d : d;   // idle threads own no row
  }
  __device__ __forceinline__ int row(int q) const { return j0 + R * q; }
};

template <int Q>
__device__ __forceinline__ void direct_accumulate(const Args& a, const Owner& o, int64_t beg, int64_t end,
                                                  float* tile, float* tile_c, float (&acc)[Q], float& bacc) {
  const int d = a.d, tid = threadIdx.x;
  for (int64_t t0 = beg; t0 < end; t0 += DIRECT_TILE) {
    const int n = (int)min((int64_t)DIRECT_TILE, end - t0);
    for (int e = tid; e < n * d; e += DIRECT_THREADS) {
      const int r = e / d, c = e - r * d;
      tile[e] = __ldg(a.Y + (int64_t)__ldg(a.indices + t0 + r) * d + c);
    }
    if (tid < n) tile_c[tid] = __ldg(a.data + t0 + tid);
    __syncthreads();
    for (int r = 0; r < n; ++r) {
      const float c = tile_c[r];
      const float* y = tile + r * d;
      const float wgt = __fsub_rn(c, 1.f);
      const float yk = y[o.k];
#pragma unroll
      for (int q = 0; q < Q; ++q) {
        const int j = o.row(q);
        if (j < d) {
          const float yj = y[j];
          // the reference adds temp * Y[i, :] to row j of A, temp = (c - 1) * Y[i, j] (implicit) or Y[i, j]
          acc[q] = a.implicit ? fmaf(__fmul_rn(wgt, yj), yk, acc[q]) : fmaf(yj, yk, acc[q]);
        }
      }
      if (tid < d) bacc = fmaf(c, y[tid], bacc);
    }
    __syncthreads();
  }
}

// Cholesky of the SPD d x d matrix A (row-major, shared memory), then L L^T x = b in place of b.  L is written to
// the lower triangle and L^T to the upper one, and `col` holds the current column of L, so that every inner loop
// walks a row (no bank conflicts).  Returns info (0, or j+1 at the first pivot <= 0 or NaN), uniform over the CTA.
__device__ int cholesky_solve(float* A, float* b, float* col, int d) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, n_warps = blockDim.x >> 5;
  for (int j = 0; j < d; ++j) {
    __syncthreads();
    const float piv = A[j * d + j];
    if (!(piv > 0.f)) return j + 1;
    const float ljj = sqrtf(piv);
    __syncthreads();
    for (int i = j + 1 + tid; i < d; i += blockDim.x) {
      const float v = A[i * d + j] / ljj;
      A[i * d + j] = v;
      A[j * d + i] = v;
      col[i] = v;
    }
    if (tid == 0) A[j * d + j] = ljj;
    __syncthreads();
    // trailing update of the lower triangle: one warp per row i, lanes over the columns k <= i
    for (int i = j + 1 + warp; i < d; i += n_warps) {
      const float lij = col[i];
      for (int k = j + 1 + lane; k <= i; k += 32) A[i * d + k] = fmaf(-lij, col[k], A[i * d + k]);
    }
  }
  __syncthreads();
  if (warp == 0) {   // forward L z = b, then backward L^T x = z; one warp, fixed-order lane sums
    for (int i = 0; i < d; ++i) {
      float s = 0.f;
      for (int k = lane; k < i; k += 32) s = fmaf(A[i * d + k], b[k], s);
      s = warp_sum(s);
      if (lane == 0) b[i] = (b[i] - s) / A[i * d + i];
      __syncwarp();
    }
    for (int i = d - 1; i >= 0; --i) {
      float s = 0.f;
      for (int k = i + 1 + lane; k < d; k += 32) s = fmaf(A[i * d + k], b[k], s);
      s = warp_sum(s);
      if (lane == 0) b[i] = (b[i] - s) / A[i * d + i];
      __syncwarp();
    }
  }
  __syncthreads();
  return 0;
}

__host__ __device__ inline int64_t direct_partial_floats(int d) { return (int64_t)d * d + d; }

// LONG = 0: rows[k] are short rows, built from the CSR.  LONG = 1: rows[k] are long rows, summed from chunk
// partials in chunk order.  CHUNKS = 1: one CTA per chunk of a long row writes its partial (no solve).
template <int Q, int MODE>
__global__ void __launch_bounds__(DIRECT_THREADS) direct_kernel(Args a, const int32_t* __restrict__ rows,
                                                                const int64_t* __restrict__ long_chunk_ptr,
                                                                const int32_t* __restrict__ chunk_long,
                                                                const int32_t* __restrict__ chunk_k,
                                                                float* __restrict__ partials,
                                                                unsigned long long* __restrict__ fail) {
  extern __shared__ __align__(16) float smem[];
  const int d = a.d, tid = threadIdx.x;
  float* As = smem;
  float* bs = As + d * d;
  float* tile = bs + MAX_D;
  float* tile_c = tile + DIRECT_TILE * d;
  float* col = tile_c + DIRECT_TILE;
  const Owner o(d);
  float acc[Q];
  float bacc = 0.f;
  const int64_t k = blockIdx.x;
  if (MODE == 2) {   // chunk partial of a long row
    const int64_t m = rows[chunk_long[k]];
    const int64_t beg = a.indptr[m] + (int64_t)chunk_k[k] * CHUNK;
    const int64_t end = min(beg + (int64_t)CHUNK, a.indptr[m + 1]);
#pragma unroll
    for (int q = 0; q < Q; ++q) acc[q] = 0.f;
    direct_accumulate<Q>(a, o, beg, end, tile, tile_c, acc, bacc);
    float* out = partials + k * direct_partial_floats(d);
#pragma unroll
    for (int q = 0; q < Q; ++q)
      if (o.row(q) < d) out[o.row(q) * d + o.k] = acc[q];
    if (tid < d) out[d * d + tid] = bacc;
    return;
  }
  const int64_t m = rows[k];
  if (MODE == 0) {
#pragma unroll
    for (int q = 0; q < Q; ++q) acc[q] = o.row(q) < d ? __ldg(a.A0 + o.row(q) * d + o.k) : 0.f;
    direct_accumulate<Q>(a, o, a.indptr[m], a.indptr[m + 1], tile, tile_c, acc, bacc);
#pragma unroll
    for (int q = 0; q < Q; ++q)
      if (o.row(q) < d) As[o.row(q) * d + o.k] = acc[q];
    if (tid < d) bs[tid] = bacc;
  } else {   // A0 + the chunk partials, in chunk order
    const int64_t c0 = long_chunk_ptr[k], c1 = long_chunk_ptr[k + 1];
    const int64_t stride = direct_partial_floats(d);
    for (int e = tid; e < d * d + d; e += DIRECT_THREADS) {
      float v = e < d * d ? __ldg(a.A0 + e) : 0.f;
      for (int64_t c = c0; c < c1; ++c) v += partials[c * stride + e];
      if (e < d * d) As[e] = v;
      else bs[e - d * d] = v;
    }
  }
  const int info = cholesky_solve(As, bs, col, d);
  if (info != 0) {
    if (tid == 0) atomicMin(fail, ((unsigned long long)m << 32) | (unsigned)info);
    return;
  }
  if (tid < d) a.X[m * d + tid] = bs[tid];
}

template <int Q>
static void launch_direct(const Args& a, const int32_t* short_rows, int64_t n_short, const int32_t* long_rows,
                          const int64_t* long_chunk_ptr, int64_t n_long, const int32_t* chunk_long,
                          const int32_t* chunk_k, int64_t n_chunks, float* partials, unsigned long long* fail,
                          size_t smem, cudaStream_t stream) {
  cudaFuncSetAttribute(direct_kernel<Q, 0>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaFuncSetAttribute(direct_kernel<Q, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  cudaFuncSetAttribute(direct_kernel<Q, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (n_short > 0) {
    direct_kernel<Q, 0><<<(unsigned)n_short, DIRECT_THREADS, smem, stream>>>(a, short_rows, nullptr, nullptr,
                                                                            nullptr, nullptr, fail);
    count_launch();
  }
  if (n_long > 0) {
    direct_kernel<Q, 2><<<(unsigned)n_chunks, DIRECT_THREADS, smem, stream>>>(a, long_rows, nullptr, chunk_long,
                                                                             chunk_k, partials, fail);
    direct_kernel<Q, 1><<<(unsigned)n_long, DIRECT_THREADS, smem, stream>>>(a, long_rows, long_chunk_ptr, nullptr,
                                                                           nullptr, partials, fail);
    count_launch(2);
  }
}

}  // namespace als
}  // namespace b200

using namespace b200;
using namespace b200::als;

extern "C" int b200_als_long_row_threshold(void) { return LONG_ROW; }
extern "C" int b200_als_chunk(void) { return CHUNK; }
extern "C" int b200_als_stage_rows(int32_t d) { return d >= 1 && d <= MAX_D ? stage_rows(d) : 0; }

extern "C" int b200_als_workspace_bytes(int32_t d, int32_t use_cg, int64_t n_long, int64_t n_chunks,
                                        size_t* bytes) {
  B200_REQUIRE(bytes, "b200_als_workspace_bytes: null pointer");
  B200_REQUIRE(d >= 1 && d <= MAX_D, "b200_als_workspace_bytes: embed size %d outside [1, %d]", d, MAX_D);
  B200_REQUIRE(n_long >= 0 && n_chunks >= 0, "b200_als_workspace_bytes: negative count");
  const int64_t floats = use_cg ? n_chunks * d + n_long * cg_state_floats(d) : n_chunks * direct_partial_floats(d);
  *bytes = (size_t)floats * 4 + 32;   // + the direct path's failure word, 16-byte aligned
  return 0;
}

static int check_args(const char* fn, const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_x,
                      float* X, const float* Y, int64_t n_y, int32_t d, const float* A0, const int32_t* short_rows,
                      int64_t n_short, const int32_t* long_rows, const int64_t* long_chunk_ptr, int64_t n_long,
                      const int32_t* chunk_long, const int32_t* chunk_k, int64_t n_chunks, void* workspace,
                      size_t workspace_bytes, int32_t use_cg) {
  B200_REQUIRE(d >= 1 && d <= MAX_D, "%s: embed size %d outside [1, %d]", fn, d, MAX_D);
  B200_REQUIRE(n_x >= 0 && n_y >= 0 && n_short >= 0 && n_long >= 0 && n_chunks >= 0 && n_short + n_long == n_x,
               "%s: bad row counts (n_x %lld, short %lld, long %lld)", fn, (long long)n_x, (long long)n_short,
               (long long)n_long);
  B200_REQUIRE(n_x < (1ll << 31) && n_y < (1ll << 31), "%s: more than 2^31 rows", fn);
  B200_REQUIRE(indptr && A0 && (n_x == 0 || X) && (n_short == 0 || short_rows), "%s: null pointer", fn);
  B200_REQUIRE(n_long == 0 || (long_rows && long_chunk_ptr && chunk_long && chunk_k && n_chunks > 0),
               "%s: long-row plan missing", fn);
  size_t need = 0;
  b200_als_workspace_bytes(d, use_cg, n_long, n_chunks, &need);
  B200_REQUIRE(workspace && workspace_bytes >= need && ((uintptr_t)workspace & 15) == 0,
               "%s: workspace needs %zu bytes, 16-byte aligned", fn, need);
  B200_REQUIRE(((uintptr_t)Y & 15) == 0 || (d & 3) != 0, "%s: Y must be 16-byte aligned", fn);
  (void)indices; (void)data;
  return 0;
}

template <int T>
static int launch_cg(const Args& a, const int32_t* short_rows, int64_t n_short, const int32_t* long_rows,
                     const int64_t* long_chunk_ptr, int64_t n_long, const int32_t* chunk_long, const int32_t* chunk_k,
                     int64_t n_chunks, float* workspace, cudaStream_t stream) {
  const int d = a.d, cg_steps = a.cg_steps;
  const int a0f = (d * d + 3) & ~3;
  if (n_short > 0) {
    const size_t smem = (size_t)(a0f + CG_WARPS * (STAGE_FLOATS + MAX_D)) * 4;
    B200_CUDA_OK(cudaFuncSetAttribute(cg_rows_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cg_rows_kernel<T><<<(unsigned)ceil_div64(n_short, CG_WARPS), CG_WARPS * 32, smem, stream>>>(a, short_rows, n_short);
    count_launch();
  }
  if (n_long > 0) {
    float* partials = workspace;
    float* st = partials + n_chunks * d;
    const size_t smem = (size_t)(a0f + CG_WARPS * MAX_D) * 4;
    B200_CUDA_OK(cudaFuncSetAttribute(cg_long_update_kernel<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    for (int pass = 0; pass <= cg_steps; ++pass) {
      const int phase0 = pass == 0;
      cg_chunks_kernel<T><<<(unsigned)ceil_div64(n_chunks * 32, 256), 256, 0, stream>>>(
          a, phase0, chunk_long, long_rows, chunk_k, n_chunks, st, partials);
      cg_long_update_kernel<T><<<(unsigned)ceil_div64(n_long, CG_WARPS), CG_WARPS * 32, smem, stream>>>(
          a, phase0, long_rows, long_chunk_ptr, n_long, st, partials);
      count_launch(2);
    }
  }
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_als_cg(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_x, float* X,
                           const float* Y, int64_t n_y, int32_t d, const float* A0, int32_t implicit,
                           int32_t cg_steps, const int32_t* short_rows, int64_t n_short, const int32_t* long_rows,
                           const int64_t* long_chunk_ptr, int64_t n_long, const int32_t* chunk_long,
                           const int32_t* chunk_k, int64_t n_chunks, void* workspace, size_t workspace_bytes,
                           void* stream_) {
  int rc = check_args("b200_als_cg", indptr, indices, data, n_x, X, Y, n_y, d, A0, short_rows, n_short, long_rows,
                      long_chunk_ptr, n_long, chunk_long, chunk_k, n_chunks, workspace, workspace_bytes, 1);
  if (rc) return rc;
  B200_REQUIRE(cg_steps >= 0, "b200_als_cg: cg_steps %d < 0", cg_steps);
  // with no step X is never written; the residual pass has no effect
  if (n_x == 0 || cg_steps == 0) return 0;
  cudaStream_t stream = (cudaStream_t)stream_;
  Args a{indptr, indices, data, X, Y, A0, d, implicit ? 1 : 0, cg_steps};
  if (d <= 32) return launch_cg<1>(a, short_rows, n_short, long_rows, long_chunk_ptr, n_long, chunk_long, chunk_k,
                                   n_chunks, (float*)workspace, stream);
  if (d <= 64) return launch_cg<2>(a, short_rows, n_short, long_rows, long_chunk_ptr, n_long, chunk_long, chunk_k,
                                   n_chunks, (float*)workspace, stream);
  return launch_cg<4>(a, short_rows, n_short, long_rows, long_chunk_ptr, n_long, chunk_long, chunk_k, n_chunks,
                      (float*)workspace, stream);
}

extern "C" int b200_als_direct(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_x,
                               float* X, const float* Y, int64_t n_y, int32_t d, const float* A0, int32_t implicit,
                               const int32_t* short_rows, int64_t n_short, const int32_t* long_rows,
                               const int64_t* long_chunk_ptr, int64_t n_long, const int32_t* chunk_long,
                               const int32_t* chunk_k, int64_t n_chunks, void* workspace, size_t workspace_bytes,
                               int64_t* fail_row, int32_t* fail_info, void* stream_) {
  int rc = check_args("b200_als_direct", indptr, indices, data, n_x, X, Y, n_y, d, A0, short_rows, n_short,
                      long_rows, long_chunk_ptr, n_long, chunk_long, chunk_k, n_chunks, workspace, workspace_bytes, 0);
  if (rc) return rc;
  B200_REQUIRE(fail_row && fail_info, "b200_als_direct: null failure output");
  *fail_row = -1;
  *fail_info = 0;
  if (n_x == 0) return 0;
  cudaStream_t stream = (cudaStream_t)stream_;
  Args a{indptr, indices, data, X, Y, A0, d, implicit ? 1 : 0, 0};
  float* partials = (float*)workspace;
  unsigned long long* fail =
      (unsigned long long*)((char*)workspace + (((size_t)n_chunks * direct_partial_floats(d) * 4 + 15) & ~(size_t)15));
  const unsigned long long none = ~0ull;
  B200_CUDA_OK(cudaMemcpyAsync(fail, &none, 8, cudaMemcpyHostToDevice, stream));
  const size_t smem = (size_t)(d * d + MAX_D + DIRECT_TILE * d + DIRECT_TILE + MAX_D) * 4;
  const int R = DIRECT_THREADS / d, Q = (d + R - 1) / R;
  auto go = [&](auto q) {
    launch_direct<decltype(q)::value>(a, short_rows, n_short, long_rows, long_chunk_ptr, n_long, chunk_long, chunk_k,
                                      n_chunks, partials, fail, smem, stream);
  };
  if (Q <= 1) go(std::integral_constant<int, 1>());
  else if (Q <= 2) go(std::integral_constant<int, 2>());
  else if (Q <= 8) go(std::integral_constant<int, 8>());
  else go(std::integral_constant<int, 32>());
  B200_CUDA_OK(cudaGetLastError());
  unsigned long long f = 0;
  B200_CUDA_OK(cudaMemcpyAsync(&f, fail, 8, cudaMemcpyDeviceToHost, stream));
  B200_CUDA_OK(cudaStreamSynchronize(stream));
  if (f != none) {
    *fail_row = (int64_t)(f >> 32);
    *fail_info = (int32_t)(f & 0xffffffffu);
  }
  return 0;
}
