// Training step of the FM-family feature models on the device (SURVEY.md §8f-1: "backward + optimizer
// for the gather path").  Follows the reference graph in TRAINING mode:
//   libreco/algorithms/fm.py:152-171      FM head: BN(pairwise, training=True) -> Dense(1, elu)
//   libreco/tfops/loss.py:14-18            mean sigmoid cross entropy (csrc/loss.cu gives d loss / d logit)
//   libreco/training/tf_trainer.py:112-123 tf.train.AdamOptimizer(lr, epsilon) + BN update ops
// Kernels:
//   bn_train            batch mean / biased variance per column (two-pass, deterministic), normalise,
//                       moving statistics with momentum (tf.layers.batch_normalization, eps 1e-3)
//   fm_head_forward     z = <y, pw_kernel> + b, logit = lin + elu(z)
//   fm_head_backward    d logit -> d pw [R,K] (through elu, Dense, BN with batch statistics) + the
//                       gradients of pw_kernel, pw_bias, gamma, beta (deterministic column reductions)
//   feat_backward       scatter-add of the field gradients into dense gradient buffers of the
//                       embedding / linear tables (float atomics), block-local accumulation for the
//                       variables every row touches (dense-field rows, Dense(1) kernel of the linear term)
//   adam_dense          TF-Adam over a whole variable: m, v decayed everywhere, var updated everywhere
//                       (what _apply_sparse_shared does for IndexedSlices gradients), gradient zeroed
#include <cooperative_groups.h>
#include "common.cuh"
#include "feat_common.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace train {

constexpr int RED_THREADS = 256;

__device__ __forceinline__ double block_sum_d(double v) {
  __shared__ double sh[RED_THREADS / 32];
  __syncthreads();                       // protect sh across consecutive calls
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < RED_THREADS / 32; ++i) s += sh[i];
  return s;
}

// one block per column: mean, biased variance (two passes), moving statistics
__global__ void __launch_bounds__(RED_THREADS)
bn_stats_kernel(const float* __restrict__ x, int64_t ld, int64_t R, float momentum, float* __restrict__ mean,
                float* __restrict__ var, float* __restrict__ moving_mean, float* __restrict__ moving_var) {
  const int k = blockIdx.x;
  double s = 0.0;
  for (int64_t r = threadIdx.x; r < R; r += RED_THREADS) s += (double)x[r * ld + k];
  const double mu = block_sum_d(s) / (double)R;
  double q = 0.0;
  for (int64_t r = threadIdx.x; r < R; r += RED_THREADS) { const double d = (double)x[r * ld + k] - mu; q += d * d; }
  const double v = block_sum_d(q) / (double)R;
  if (threadIdx.x == 0) {
    mean[k] = (float)mu;
    var[k] = (float)v;
    if (moving_mean) moving_mean[k] = momentum * moving_mean[k] + (1.f - momentum) * (float)mu;
    if (moving_var) moving_var[k] = momentum * moving_var[k] + (1.f - momentum) * (float)v;
  }
}

__global__ void bn_apply_kernel(const float* __restrict__ x, int64_t ldx, int64_t R, int K,
                                const float* __restrict__ mean, const float* __restrict__ var,
                                const float* __restrict__ gamma, const float* __restrict__ beta, float eps,
                                float* __restrict__ y, int64_t ldy) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R * K) return;
  const int64_t r = i / K;
  const int k = (int)(i % K);
  const float xh = (x[r * ldx + k] - mean[k]) * rsqrtf(var[k] + eps);
  y[r * ldy + k] = fmaf(xh, gamma[k], beta[k]);
}

// thread per row: z = <y, w> + b ; logit = lin + elu(z)
__global__ void fm_head_forward_kernel(const float* __restrict__ y, int64_t ldy, int64_t R, int K,
                                       const float* __restrict__ w, const float* __restrict__ b,
                                       const float* __restrict__ lin, const float* __restrict__ lin_bias,
                                       float* __restrict__ z_out, float* __restrict__ logit) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  float z = b ? __ldg(b) : 0.f;
  for (int k = 0; k < K; ++k) z = fmaf(y[r * ldy + k], __ldg(w + k), z);
  z_out[r] = z;
  logit[r] = lin[r] + (lin_bias ? __ldg(lin_bias) : 0.f) + (z > 0.f ? z : expm1f(z));
}

// stage 1 of the head backward: dz_r = dlogit_r * elu'(z_r); D = sum dz; T_k = sum_r dz_r * u[r,k]
// with u = xhat (BN) or pw (no BN).  One block per column k (+ one extra block for D).
__global__ void __launch_bounds__(RED_THREADS)
fm_head_reduce_kernel(const float* __restrict__ dlogit, const float* __restrict__ z,
                      const float* __restrict__ pw, int64_t ld, int64_t R, int K,
                      const float* __restrict__ mean, const float* __restrict__ var, float eps,
                      float* __restrict__ dz_out, double* __restrict__ red /* [K + 2]: T_k, D, sum dlogit */) {
  const int k = blockIdx.x;
  double s = 0.0;
  if (k == K + 1) {
    for (int64_t r = threadIdx.x; r < R; r += RED_THREADS) s += (double)dlogit[r];
  } else if (k == K) {
    for (int64_t r = threadIdx.x; r < R; r += RED_THREADS) {
      const float zz = z[r];
      const float d = dlogit[r] * (zz > 0.f ? 1.f : expf(zz));
      dz_out[r] = d;
      s += (double)d;
    }
  } else {
    const float mu = mean ? mean[k] : 0.f;
    const float inv = mean ? rsqrtf(var[k] + eps) : 1.f;
    for (int64_t r = threadIdx.x; r < R; r += RED_THREADS) {
      const float zz = z[r];
      const float d = dlogit[r] * (zz > 0.f ? 1.f : expf(zz));
      s += (double)d * (double)((pw[r * ld + k] - mu) * inv);
    }
  }
  const double tot = block_sum_d(s);
  if (threadIdx.x == 0) red[k] = tot;
}

// stage 2: d pw[r,k] and the parameter gradients (ADDED to the gradient buffers)
__global__ void fm_head_apply_kernel(const float* __restrict__ dz, const float* __restrict__ pw, int64_t ld,
                                     int64_t R, int K, const float* __restrict__ mean,
                                     const float* __restrict__ var, const float* __restrict__ gamma,
                                     const float* __restrict__ beta, float eps, const float* __restrict__ w,
                                     const double* __restrict__ red, float* __restrict__ dpw, int64_t ld_dpw,
                                     float* __restrict__ g_w, float* __restrict__ g_b,
                                     float* __restrict__ g_gamma, float* __restrict__ g_beta,
                                     float* __restrict__ g_lin_bias) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const double D = red[K];
  if (i < K) {   // parameter gradients, once
    const int k = (int)i;
    const double T = red[k];
    if (mean) {
      g_gamma[k] += (float)((double)w[k] * T);
      g_beta[k] += (float)((double)w[k] * D);
      g_w[k] += (float)((double)gamma[k] * T + (double)beta[k] * D);   // sum dz * y, y = gamma xhat + beta
    } else {
      g_w[k] += (float)T;
    }
    if (k == 0) {
      g_b[0] += (float)D;
      if (g_lin_bias) g_lin_bias[0] += (float)red[K + 1];   // d loss / d (bias of the linear term) = sum dlogit
    }
  }
  if (i >= R * K) return;
  const int64_t r = i / K;
  const int k = (int)(i % K);
  if (mean) {
    const float inv = rsqrtf(var[k] + eps);
    const float xh = (pw[r * ld + k] - mean[k]) * inv;
    const float invR = 1.f / (float)R;
    dpw[r * ld_dpw + k] = inv * w[k] * gamma[k] * (dz[r] - (float)D * invR - xh * (float)red[k] * invR);
  } else {
    dpw[r * ld_dpw + k] = dz[r] * w[k];
  }
}

struct Grads {
  float* user_embeds; float* item_embeds; float* sparse_embeds; float* dense_embeds;
  float* user_linear; float* item_linear; float* sparse_linear; float* dense_linear;
  float* lin_kernel;      // [2 + F_s + F_d]
};

// One sub-warp (lpr lanes) per row, lanes over K.  ge_f[k] = dpw[r,k] * (S[r,k] - e_f[k]) (+ dconcat).
// Shared accumulators for the variables every row touches.
__global__ void __launch_bounds__(256)
feat_backward_kernel(const b200_feat_layout L, const b200_feat_tables T, const int64_t* __restrict__ users,
                     const int64_t* __restrict__ items, int64_t R, const float* __restrict__ dpw, int64_t ld_dpw,
                     const float* __restrict__ S, int64_t ld_s, const float* __restrict__ dconcat,
                     int64_t ld_dc, const float* __restrict__ dlogit, const float* __restrict__ lin_kernel,
                     Grads G, int lpr) {
  extern __shared__ float sh[];
  const int K = L.embed_size;
  const int F = 2 + L.n_sparse + L.n_dense;
  float* sh_dense = sh;                          // [n_dense * K]
  float* sh_link = sh + L.n_dense * K;           // [F]      d lin_kernel
  float* sh_dlin = sh_link + F;                  // [n_dense] d dense_linear
  const int n_sh = L.n_dense * K + F + L.n_dense;
  for (int i = threadIdx.x; i < n_sh; i += blockDim.x) sh[i] = 0.f;
  __syncthreads();

  const int lane = threadIdx.x & 31;
  const int rows_per_warp = 32 / lpr;
  const int g = lane / lpr, li = lane % lpr;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int64_t r = warp * rows_per_warp + g;
  if (r < R) {
    const int64_t u = users[r], it = items[r];
    const float dl = dlogit ? dlogit[r] : 0.f;
    auto field_grad = [&](int f, const float* __restrict__ erow, float scale, float* __restrict__ gdst, float gscale) {
      // e_f = scale * erow ; d erow = gscale * ge
      for (int k = li; k < K; k += lpr) {
        const float e = __ldg(erow + k) * scale;
        float ge = dpw ? dpw[r * ld_dpw + k] * (S[r * ld_s + k] - e) : 0.f;
        if (dconcat) ge += dconcat[r * ld_dc + (int64_t)f * K + k];
        atomicAdd(gdst + k, ge * gscale);
      }
    };
    int fpos = 0;
    if (L.id_mask & 1) {
      field_grad(fpos, T.user_embeds + u * K, 1.f, G.user_embeds + u * K, 1.f);
      if (dlogit && li == 0) {
        atomicAdd(G.user_linear + u, dl * __ldg(lin_kernel + fpos));
        atomicAdd(sh_link + fpos, dl * __ldg(T.user_linear + u));
      }
      ++fpos;
    }
    if (L.id_mask & 2) {
      field_grad(fpos, T.item_embeds + it * K, 1.f, G.item_embeds + it * K, 1.f);
      if (dlogit && li == 0) {
        atomicAdd(G.item_linear + it, dl * __ldg(lin_kernel + fpos));
        atomicAdd(sh_link + fpos, dl * __ldg(T.item_linear + it));
      }
      ++fpos;
    }
    for (int f = 0; f < L.n_sparse; ++f) {
      const int32_t idx = feat::sparse_index(L, r, u, it, f);
      field_grad(fpos + f, T.sparse_embeds + (int64_t)idx * K, 1.f, G.sparse_embeds + (int64_t)idx * K, 1.f);
      if (dlogit && li == 0) {
        atomicAdd(G.sparse_linear + idx, dl * __ldg(lin_kernel + fpos + f));
        atomicAdd(sh_link + fpos + f, dl * __ldg(T.sparse_linear + idx));
      }
    }
    fpos += L.n_sparse;
    for (int f = 0; f < L.n_dense; ++f) {
      const float x = feat::dense_value(L, r, u, it, f);
      const int row = L.dense_embed_row[f];
      field_grad(fpos + f, T.dense_embeds + (int64_t)row * K, x, sh_dense + f * K, x);
      if (dlogit && li == 0) {
        atomicAdd(sh_dlin + f, dl * __ldg(lin_kernel + fpos + f) * x);
        atomicAdd(sh_link + fpos + f, dl * x * __ldg(T.dense_linear + row));
      }
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_sh; i += blockDim.x) {
    const float v = sh[i];
    if (v == 0.f) continue;
    if (i < L.n_dense * K) atomicAdd(G.dense_embeds + (int64_t)L.dense_embed_row[i / K] * K + (i % K), v);
    else if (i < L.n_dense * K + F) { if (G.lin_kernel) atomicAdd(G.lin_kernel + (i - L.n_dense * K), v); }
    else if (G.dense_linear) atomicAdd(G.dense_linear + L.dense_embed_row[i - L.n_dense * K - F], v);
  }
}

__global__ void adam_dense_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                                  float* __restrict__ g, int64_t n, float lr_t, float b1, float b2, float eps) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float gi = g[i];
  const float mi = b1 * m[i] + (1.f - b1) * gi;
  const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
  m[i] = mi;
  v[i] = vi;
  p[i] -= lr_t * mi / (sqrtf(vi) + eps);
  g[i] = 0.f;
}

// ---- generic pieces for the MLP tails (dense_nn in training mode, libreco/layers/dense.py:12-49) ----

// out[k] = sum_r (w ? w[r] : 1) * X[r,k] * (Y ? Y[r,k] : 1): 32 columns x 16 row lanes per CTA, a CLUSTER of
// COLRED_CL CTAs along the rows (thread-block cluster + distributed shared memory: CTA 0 adds the other CTAs'
// partial sums straight out of their shared memory, no global scratch, no atomics), 4 independent accumulators
// per thread, double accumulation, fixed reduction order (deterministic).  The first version ran ONE CTA per 32
// columns with a 1024-deep dependent loop: 155 us per call, 41 % of a DeepFM training step.
constexpr int COLRED_CL = 8;
constexpr int COLRED_TY = 16;
__global__ void __launch_bounds__(32 * COLRED_TY)
col_reduce_kernel(const float* __restrict__ X, int64_t ldx, int64_t R, int K, const float* __restrict__ w,
                  const float* __restrict__ Y, int64_t ldy, double* __restrict__ out_d, float* __restrict__ out_f) {
  namespace cg = cooperative_groups;
  __shared__ double sh[COLRED_TY][33];
  __shared__ double tot[32];
  cg::cluster_group cluster = cg::this_cluster();
  const int crank = (int)cluster.block_rank();          // position along the rows
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  const int k = blockIdx.x * 32 + tx;
  const int lanes = COLRED_CL * COLRED_TY;
  double a0 = 0.0, a1 = 0.0, a2 = 0.0, a3 = 0.0;
  if (k < K) {
    auto term = [&](int64_t r) -> double {
      double v = (double)X[r * ldx + k];
      if (Y) v *= (double)Y[r * ldy + k];
      if (w) v *= (double)w[r];
      return v;
    };
    int64_t r = crank * COLRED_TY + ty;
    for (; r + 3 * lanes < R; r += 4 * lanes) {
      const double v0 = term(r), v1 = term(r + lanes), v2 = term(r + 2 * lanes), v3 = term(r + 3 * lanes);
      a0 += v0; a1 += v1; a2 += v2; a3 += v3;
    }
    for (; r < R; r += lanes) a0 += term(r);
  }
  sh[ty][tx] = (a0 + a1) + (a2 + a3);
  __syncthreads();
  if (ty == 0) {
    double t = 0.0;
#pragma unroll
    for (int j = 0; j < COLRED_TY; ++j) t += sh[j][tx];
    tot[tx] = t;
  }
  cluster.sync();
  if (crank == 0 && ty == 0 && k < K) {
    double t = 0.0;
    for (int c = 0; c < COLRED_CL; ++c) t += *cluster.map_shared_rank(&tot[tx], c);
    if (out_d) out_d[k] = t;
    if (out_f) out_f[k] += (float)t;
  }
  cluster.sync();                                          // keep every CTA's shared memory alive until it was read
}

static int launch_col_reduce(const float* X, int64_t ldx, int64_t R, int K, const float* w, const float* Y, int64_t ldy,
                             double* out_d, float* out_f, cudaStream_t st) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)((K + 31) / 32), COLRED_CL, 1);
  cfg.blockDim = dim3(32 * COLRED_TY, 1, 1);
  cfg.dynamicSmemBytes = 0;
  cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = 1;
  attr[0].val.clusterDim.y = COLRED_CL;
  attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  B200_CUDA_OK(cudaLaunchKernelEx(&cfg, col_reduce_kernel, X, ldx, R, K, w, Y, ldy, out_d, out_f));
  return 0;
}

// BN backward with batch statistics.  s1 = sum dy, s2 = sum dy * x (workspace, doubles).
__global__ void bn_backward_apply_kernel(const float* __restrict__ dy, int64_t lddy, const float* __restrict__ x,
                                         int64_t ldx, int64_t R, int K, const float* __restrict__ mean,
                                         const float* __restrict__ var, const float* __restrict__ gamma, float eps,
                                         int relu_mask, const double* __restrict__ s1, const double* __restrict__ s2,
                                         float* __restrict__ dx, int64_t lddx, float* __restrict__ g_gamma,
                                         float* __restrict__ g_beta) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < K) {
    const int k = (int)i;
    const double inv = 1.0 / sqrt((double)var[k] + (double)eps);
    g_gamma[k] += (float)(inv * (s2[k] - (double)mean[k] * s1[k]));   // sum dy * xhat
    g_beta[k] += (float)s1[k];
  }
  if (i >= R * K) return;
  const int64_t r = i / K;
  const int k = (int)(i % K);
  const float inv = rsqrtf(var[k] + eps);
  const float xv = x[r * ldx + k];
  const float xh = (xv - mean[k]) * inv;
  const float T = inv * (float)(s2[k] - (double)mean[k] * s1[k]);
  const float invR = 1.f / (float)R;
  float d = gamma[k] * inv * (dy[r * lddy + k] - (float)s1[k] * invR - xh * T * invR);
  if (relu_mask && !(xv > 0.f)) d = 0.f;      // x = relu(h): pass the gradient only where h > 0
  dx[r * lddx + k] = d;
}

__global__ void relu_backward_kernel(const float* __restrict__ dy, const float* __restrict__ a, int64_t n,
                                     float* __restrict__ dx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dx[i] = a[i] > 0.f ? dy[i] : 0.f;
}

// DeepFM head (deepfm.py:172-173): logit = <[lin + lin_bias, pw, deep], w_out> + b_out
__global__ void deepfm_head_forward_kernel(const float* __restrict__ lin, const float* __restrict__ lin_bias,
                                           const float* __restrict__ pw, int64_t ldpw, int K,
                                           const float* __restrict__ deep, int64_t lddeep, int H,
                                           const float* __restrict__ w, const float* __restrict__ b, int64_t R,
                                           float* __restrict__ logit) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  float acc = (b ? __ldg(b) : 0.f) + (lin[r] + (lin_bias ? __ldg(lin_bias) : 0.f)) * __ldg(w);
  for (int k = 0; k < K; ++k) acc = fmaf(pw[r * ldpw + k], __ldg(w + 1 + k), acc);
  for (int j = 0; j < H; ++j) acc = fmaf(deep[r * lddeep + j], __ldg(w + 1 + K + j), acc);
  logit[r] = acc;
}

__global__ void deepfm_head_backward_kernel(const float* __restrict__ dlogit, const float* __restrict__ w, int K,
                                            int H, int64_t R, float* __restrict__ dlin, float* __restrict__ dpw,
                                            int64_t lddpw, float* __restrict__ ddeep, int64_t ldd) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int W = 1 + K + H;
  if (i >= R * W) return;
  const int64_t r = i / W;
  const int c = (int)(i % W);
  const float v = dlogit[r] * __ldg(w + c);
  if (c == 0) dlin[r] = v;
  else if (c <= K) dpw[r * lddpw + (c - 1)] = v;
  else ddeep[r * ldd + (c - 1 - K)] = v;
}


// backward of tf.linalg.l2_normalize (y = x rsqrt(max(|x|^2, 1e-12))): dx = r (dy - y <y, dy>) above the clamp
__global__ void l2_normalize_backward_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ dy,
                                             int64_t lddy, int64_t R, int d, float* __restrict__ dx, int64_t lddx) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  float ss = 0.f, xd = 0.f;
  for (int k = lane; k < d; k += 32) {
    const float v = x[r * ldx + k];
    ss = fmaf(v, v, ss);
    xd = fmaf(v, dy[r * lddy + k], xd);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    ss += __shfl_xor_sync(0xffffffffu, ss, o);
    xd += __shfl_xor_sync(0xffffffffu, xd, o);
  }
  const bool clamped = ss < 1e-12f;
  const float inv = rsqrtf(fmaxf(ss, 1e-12f));
  const float c = clamped ? 0.f : xd * inv * inv * inv;      // <y, dy> r / |x| ... = <x, dy> r^3
  for (int k = lane; k < d; k += 32) dx[r * lddx + k] = dy[r * lddy + k] * inv - x[r * ldx + k] * c;
}


// CUDA-graph friendly Adam: the step counter and the bias-corrected step size live on the device, so a captured
// training step can be replayed (a host-computed lr_t would be baked into the graph at capture time)
__global__ void adam_begin_step_kernel(long long* __restrict__ step, float lr, float b1, float b2, float decay_rate,
                                       long long decay_steps, float* __restrict__ lr_t) {
  const long long t = *step + 1;
  *step = t;
  // tf.train.exponential_decay(lr, global_step, decay_steps, decay_rate, staircase=True): global_step counts the
  // COMPLETED steps, i.e. t - 1 while step t runs (libreco/tfops/configs.py:38-45)
  double lr_now = (double)lr;
  if (decay_steps > 0) lr_now *= pow((double)decay_rate, (double)((t - 1) / decay_steps));
  *lr_t = (float)(lr_now * sqrt(1.0 - pow((double)b2, (double)t)) / (1.0 - pow((double)b1, (double)t)));
}

// y += alpha * x  (L2 regulariser: d (reg * sum w^2) / dw = 2 reg w added to the gradient buffers)
__global__ void axpy_kernel(float* __restrict__ y, const float* __restrict__ x, float alpha, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) y[i] = fmaf(alpha, x[i], y[i]);
}

__global__ void adam_dense_dev_kernel(float* __restrict__ p, float* __restrict__ m, float* __restrict__ v,
                                      float* __restrict__ g, int64_t n, const float* __restrict__ lr_t_dev, float b1,
                                      float b2, float eps) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float lr_t = __ldg(lr_t_dev);
  const float gi = g[i];
  const float mi = b1 * m[i] + (1.f - b1) * gi;
  const float vi = b2 * v[i] + (1.f - b2) * gi * gi;
  m[i] = mi;
  v[i] = vi;
  p[i] -= lr_t * mi / (sqrtf(vi) + eps);
  g[i] = 0.f;
}

}  // namespace train
}  // namespace b200

using namespace b200;
using namespace b200::train;

extern "C" int b200_col_reduce(const float* X, int64_t ldx, int64_t R, int32_t K, const float* wrow,
                               const float* Y, int64_t ldy, float* out, void* stream) {
  B200_REQUIRE(X && out && K > 0, "b200_col_reduce: bad arguments");
  if (R == 0) return 0;
  if (launch_col_reduce(X, ldx, R, K, wrow, Y, ldy, nullptr, out, (cudaStream_t)stream)) return 1;
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_bn_train_backward(const float* dy, int64_t lddy, const float* x, int64_t ldx, int64_t R,
                                      int32_t K, const float* batch_mean, const float* batch_var,
                                      const float* gamma, float eps, int32_t relu_mask, float* dx, int64_t lddx,
                                      float* g_gamma, float* g_beta, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  B200_REQUIRE(dy && x && batch_mean && batch_var && gamma && dx && g_gamma && g_beta, "b200_bn_train_backward: null pointer");
  B200_REQUIRE(workspace && workspace_bytes >= (size_t)K * 16, "workspace too small (need 16 bytes per column)");
  if (R == 0) return 0;                    // an empty batch adds nothing to g_gamma / g_beta
  cudaStream_t st = (cudaStream_t)stream;
  double* s1 = (double*)workspace;
  double* s2 = s1 + K;
  if (launch_col_reduce(dy, lddy, R, K, nullptr, nullptr, 0, s1, nullptr, st)) return 1;
  if (launch_col_reduce(dy, lddy, R, K, nullptr, x, ldx, s2, nullptr, st)) return 1;
  bn_backward_apply_kernel<<<(unsigned)ceil_div64(R * K, 256), 256, 0, st>>>(
      dy, lddy, x, ldx, R, K, batch_mean, batch_var, gamma, eps, relu_mask, s1, s2, dx, lddx, g_gamma, g_beta);
  B200_CUDA_OK(cudaGetLastError());
  count_launch(3);
  return 0;
}

extern "C" int b200_relu_backward(const float* dy, const float* a, int64_t n, float* dx, void* stream) {
  B200_REQUIRE(dy && a && dx, "b200_relu_backward: null pointer");
  if (n == 0) return 0;
  relu_backward_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(dy, a, n, dx);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_deepfm_head_forward(const float* lin, const float* lin_bias, const float* pw, int64_t ldpw,
                                        int32_t K, const float* deep, int64_t lddeep, int32_t H,
                                        const float* out_kernel, const float* out_bias, int64_t R, float* logit,
                                        void* stream) {
  B200_REQUIRE(lin && pw && deep && out_kernel && logit, "b200_deepfm_head_forward: null pointer");
  if (R == 0) return 0;
  deepfm_head_forward_kernel<<<(unsigned)ceil_div64(R, 256), 256, 0, (cudaStream_t)stream>>>(
      lin, lin_bias, pw, ldpw, K, deep, lddeep, H, out_kernel, out_bias, R, logit);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_deepfm_head_backward(const float* dlogit, const float* out_kernel, int32_t K, int32_t H,
                                         int64_t R, float* dlin, float* dpw, int64_t lddpw, float* ddeep,
                                         int64_t lddeep, void* stream) {
  B200_REQUIRE(dlogit && out_kernel && dlin && dpw && ddeep, "b200_deepfm_head_backward: null pointer");
  if (R == 0) return 0;
  deepfm_head_backward_kernel<<<(unsigned)ceil_div64(R * (1 + K + H), 256), 256, 0, (cudaStream_t)stream>>>(
      dlogit, out_kernel, K, H, R, dlin, dpw, lddpw, ddeep, lddeep);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_bn_train_forward(const float* x, int64_t ldx, int64_t R, int32_t K, const float* gamma,
                                     const float* beta, float eps, float momentum, float* y, int64_t ldy,
                                     float* batch_mean, float* batch_var, float* moving_mean,
                                     float* moving_var, void* stream) {
  B200_REQUIRE(x && gamma && beta && y && batch_mean && batch_var, "b200_bn_train_forward: null pointer");
  B200_REQUIRE(R > 0 && K > 0, "bad shape");
  cudaStream_t st = (cudaStream_t)stream;
  bn_stats_kernel<<<K, RED_THREADS, 0, st>>>(x, ldx, R, momentum, batch_mean, batch_var, moving_mean, moving_var);
  bn_apply_kernel<<<(unsigned)ceil_div64(R * K, 256), 256, 0, st>>>(x, ldx, R, K, batch_mean, batch_var, gamma, beta,
                                                                    eps, y, ldy);
  B200_CUDA_OK(cudaGetLastError());
  count_launch(2);
  return 0;
}

extern "C" int b200_fm_head_forward(const float* y, int64_t ldy, int64_t R, int32_t K, const float* pw_kernel,
                                    const float* pw_bias, const float* lin, const float* lin_bias, float* z,
                                    float* logit, void* stream) {
  B200_REQUIRE(y && pw_kernel && lin && z && logit, "b200_fm_head_forward: null pointer");
  if (R == 0) return 0;
  fm_head_forward_kernel<<<(unsigned)ceil_div64(R, 256), 256, 0, (cudaStream_t)stream>>>(
      y, ldy, R, K, pw_kernel, pw_bias, lin, lin_bias, z, logit);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" size_t b200_fm_head_backward_workspace_bytes(int64_t R, int32_t K) {
  return (size_t)R * 4 + (size_t)(K + 2) * 8 + 256;
}

extern "C" int b200_fm_head_backward(const float* dlogit, const float* z, const float* pw, int64_t ld, int64_t R,
                                     int32_t K, const float* batch_mean, const float* batch_var,
                                     const float* gamma, const float* beta, float eps, const float* pw_kernel,
                                     float* dpw, int64_t ld_dpw, float* g_pw_kernel, float* g_pw_bias,
                                     float* g_gamma, float* g_beta, float* g_lin_bias, void* workspace,
                                     size_t workspace_bytes, void* stream) {
  B200_REQUIRE(dlogit && z && pw && pw_kernel && dpw && g_pw_kernel && g_pw_bias, "b200_fm_head_backward: null pointer");
  B200_REQUIRE(!batch_mean || (batch_var && gamma && beta && g_gamma && g_beta), "BN arguments incomplete");
  B200_REQUIRE(workspace && workspace_bytes >= b200_fm_head_backward_workspace_bytes(R, K), "workspace too small");
  if (R == 0) return 0;                    // an empty batch adds nothing to the parameter gradients
  cudaStream_t st = (cudaStream_t)stream;
  double* red = (double*)workspace;                                   // 8-byte aligned start
  float* dz = (float*)((char*)workspace + (((size_t)(K + 2) * 8 + 255) / 256) * 256);
  fm_head_reduce_kernel<<<K + 2, RED_THREADS, 0, st>>>(dlogit, z, pw, ld, R, K, batch_mean, batch_var, eps, dz, red);
  fm_head_apply_kernel<<<(unsigned)ceil_div64(R * K, 256), 256, 0, st>>>(
      dz, pw, ld, R, K, batch_mean, batch_var, gamma, beta, eps, pw_kernel, red, dpw, ld_dpw, g_pw_kernel,
      g_pw_bias, g_gamma, g_beta, g_lin_bias);
  B200_CUDA_OK(cudaGetLastError());
  count_launch(2);
  return 0;
}

extern "C" int b200_feat_backward(const b200_feat_layout* layout, const b200_feat_tables* tables,
                                  const int64_t* users, const int64_t* items, int64_t R, const float* dpw,
                                  int64_t ld_dpw, const float* S, int64_t ld_s, const float* dconcat,
                                  int64_t ld_dconcat, const float* dlogit, const float* lin_kernel,
                                  float* g_user_embeds, float* g_item_embeds, float* g_sparse_embeds,
                                  float* g_dense_embeds, float* g_user_linear, float* g_item_linear,
                                  float* g_sparse_linear, float* g_dense_linear, float* g_lin_kernel,
                                  void* stream) {
  B200_REQUIRE(layout && tables && users && items, "b200_feat_backward: null pointer");
  B200_REQUIRE(!layout->sparse_rows && !layout->dense_rows, "explicit feature rows are not supported in training");
  B200_REQUIRE(dpw || dconcat, "nothing to propagate");
  B200_REQUIRE(!dpw || S, "the pairwise gradient needs the field sum S");
  B200_REQUIRE(!dlogit || (lin_kernel && g_lin_kernel), "linear-term gradient needs lin_kernel");
  // every field of the layout scatters into its table's gradient buffer (and its linear table's, with dlogit)
  const bool has_u = layout->id_mask & 1, has_i = layout->id_mask & 2;
  const bool has_s = layout->n_sparse > 0, has_d = layout->n_dense > 0;
  B200_REQUIRE(!has_u || g_user_embeds, "b200_feat_backward: the layout has user ids but g_user_embeds is null");
  B200_REQUIRE(!has_i || g_item_embeds, "b200_feat_backward: the layout has item ids but g_item_embeds is null");
  B200_REQUIRE(!has_s || g_sparse_embeds, "b200_feat_backward: the layout has sparse fields but g_sparse_embeds is null");
  B200_REQUIRE(!has_d || g_dense_embeds, "b200_feat_backward: the layout has dense fields but g_dense_embeds is null");
  if (dlogit) {
    B200_REQUIRE(!has_u || g_user_linear, "b200_feat_backward: dlogit given but g_user_linear is null");
    B200_REQUIRE(!has_i || g_item_linear, "b200_feat_backward: dlogit given but g_item_linear is null");
    B200_REQUIRE(!has_s || g_sparse_linear, "b200_feat_backward: dlogit given but g_sparse_linear is null");
    B200_REQUIRE(!has_d || g_dense_linear, "b200_feat_backward: dlogit given but g_dense_linear is null");
  }
  if (R == 0) return 0;
  const int K = layout->embed_size;
  int lpr = 1;
  while (lpr < K && lpr < 32) lpr <<= 1;
  Grads G{g_user_embeds, g_item_embeds, g_sparse_embeds, g_dense_embeds, g_user_linear,
          g_item_linear, g_sparse_linear, g_dense_linear, g_lin_kernel};
  const int F = 2 + layout->n_sparse + layout->n_dense;
  const size_t shm = (size_t)(layout->n_dense * K + F + layout->n_dense) * 4;
  const int64_t warps = ceil_div64(R, 32 / lpr);
  feat_backward_kernel<<<(unsigned)ceil_div64(warps * 32, 256), 256, shm, (cudaStream_t)stream>>>(
      *layout, *tables, users, items, R, dpw, ld_dpw, S, ld_s, dconcat, ld_dconcat, dlogit, lin_kernel, G, lpr);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_l2_normalize_backward(const float* x, int64_t ldx, const float* dy, int64_t lddy, int64_t R,
                                          int32_t d, float* dx, int64_t lddx, void* stream) {
  B200_REQUIRE(x && dy && dx, "b200_l2_normalize_backward: null pointer");
  if (R == 0) return 0;
  l2_normalize_backward_kernel<<<(unsigned)ceil_div64(R * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, ldx, dy, lddy, R,
                                                                                                   d, dx, lddx);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_adam_dense(float* param, float* m, float* v, float* grad, int64_t n, float lr, float beta1,
                               float beta2, float eps, int64_t step, void* stream) {
  B200_REQUIRE(param && m && v && grad, "b200_adam_dense: null pointer");
  B200_REQUIRE(step >= 1, "step counts from 1");
  if (n == 0) return 0;
  // tf.train.AdamOptimizer: lr_t = lr * sqrt(1 - beta2^t) / (1 - beta1^t)
  const double lr_t = (double)lr * sqrt(1.0 - pow((double)beta2, (double)step)) / (1.0 - pow((double)beta1, (double)step));
  adam_dense_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(param, m, v, grad, n, (float)lr_t,
                                                                                     beta1, beta2, eps);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_axpy(float* y, const float* x, float alpha, int64_t n, void* stream) {
  B200_REQUIRE(y && x, "b200_axpy: null pointer");
  if (n == 0) return 0;
  axpy_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(y, x, alpha, n);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_adam_begin_step(int64_t* step_dev, float lr, float beta1, float beta2, float decay_rate,
                                    int64_t decay_steps, float* lr_t_dev, void* stream) {
  B200_REQUIRE(step_dev && lr_t_dev, "b200_adam_begin_step: null pointer");
  adam_begin_step_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(reinterpret_cast<long long*>(step_dev), lr, beta1, beta2,
                                                            decay_rate, (long long)decay_steps, lr_t_dev);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}

extern "C" int b200_adam_dense_dev(float* param, float* m, float* v, float* grad, int64_t n, const float* lr_t_dev,
                                   float beta1, float beta2, float eps, void* stream) {
  B200_REQUIRE(param && m && v && grad && lr_t_dev, "b200_adam_dense_dev: null pointer");
  if (n == 0) return 0;
  adam_dense_dev_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, (cudaStream_t)stream>>>(param, m, v, grad, n, lr_t_dev,
                                                                                       beta1, beta2, eps);
  B200_CUDA_OK(cudaGetLastError());
  count_launch();
  return 0;
}
