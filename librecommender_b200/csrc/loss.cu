// Training losses of the hot path (SURVEY.md §8a row a13): value AND gradient w.r.t. the scores in
// one pass, deterministic two-stage reduction (no float atomics).
//
//   pointwise: reference libreco/torchops/loss.py:5-19 (binary_cross_entropy_loss, focal_loss),
//              libreco/tfops/loss.py:5-24,52-58 (sigmoid CE / focal / MSE of the TF models)
//   pairwise : torchops/loss.py:22-60 (bpr_loss, max_margin_loss, pairwise_bce_loss,
//              pairwise_focal_loss), tfops/loss.py:61-64 (max-margin of the TF two-tower models)
//   in-batch softmax: tfops/loss.py:67-71 + TwoTower.adjust_logits (algorithms/two_tower.py:458-479)
//   sampled softmax / NCE over sampled classes: training/tf_trainer.py:162-245 (YouTubeRetrieval;
//              tf.nn.sampled_softmax_loss / nce_loss with TensorFlow's expected counts)
#include "common.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace loss {

constexpr int THREADS = 256;
constexpr int MAX_BLOCKS = 1024;

__device__ __forceinline__ float softplus_neg_abs(float x) { return log1pf(__expf(-fabsf(x))); }
// numerically stable sigmoid cross entropy (same form torch and TF use): max(x,0) - x*y + log1p(e^-|x|)
__device__ __forceinline__ float bce(float x, float y) { return fmaxf(x, 0.f) - x * y + log1pf(expf(-fabsf(x))); }
__device__ __forceinline__ float sigmoidf(float x) {
  // stable on both tails
  if (x >= 0.f) return 1.f / (1.f + expf(-x));
  const float e = expf(x);
  return e / (1.f + e);
}

// focal(x, y) = w * (1 - p_t)^gamma * bce ; returns value, writes d/dx
__device__ __forceinline__ float focal(float x, float y, float alpha, float gamma, float* dx) {
  const float w = y * alpha + (1.f - y) * (1.f - alpha);
  const float p = sigmoidf(x);
  const float pt = y * p + (1.f - y) * (1.f - p);
  const float om = 1.f - pt;
  const float m = powf(om, gamma);
  const float b = bce(x, y);
  // d p_t / dx = (2y - 1) p (1 - p);  d m / dx = -gamma (1-p_t)^(gamma-1) d p_t/dx
  const float dpt = (2.f * y - 1.f) * p * (1.f - p);
  const float dm = (om > 0.f) ? -gamma * powf(om, gamma - 1.f) * dpt : 0.f;
  *dx = w * (dm * b + m * (p - y));
  return w * m * b;
}

__device__ __forceinline__ void block_sum_store(float v, double* partial) {
  __shared__ double sh[THREADS / 32];
  double d = (double)v;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = d;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
#pragma unroll
    for (int i = 0; i < THREADS / 32; ++i) s += sh[i];
    partial[blockIdx.x] = s;
  }
}

__global__ void __launch_bounds__(THREADS)
pointwise_kernel(const float* __restrict__ logits, const float* __restrict__ labels, int64_t n, int kind,
                 float alpha, float gamma, float inv_n, float* __restrict__ dlogits,
                 double* __restrict__ partial) {
  float acc = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * THREADS) {
    const float x = logits[i], y = labels[i];
    float v, g;
    if (kind == 0) { v = bce(x, y); g = sigmoidf(x) - y; }
    else if (kind == 1) { v = focal(x, y, alpha, gamma, &g); }
    else { const float d = x - y; v = d * d; g = 2.f * d; }
    acc += v;
    if (dlogits) dlogits[i] = g * inv_n;
  }
  block_sum_store(acc, partial);
}

// kind 0 bpr, 1 max_margin: one thread per positive with its `factor` negatives
__global__ void __launch_bounds__(THREADS)
pair_rank_kernel(const float* __restrict__ pos, int64_t n_pos, const float* __restrict__ neg, int factor,
                 int pos_repeated, int kind, float margin, float inv_n, float* __restrict__ dpos,
                 float* __restrict__ dneg, double* __restrict__ partial) {
  float acc = 0.f;
  for (int64_t j = (int64_t)blockIdx.x * THREADS + threadIdx.x; j < n_pos; j += (int64_t)gridDim.x * THREADS) {
    float gp_sum = 0.f;
    for (int f = 0; f < factor; ++f) {
      const int64_t e = j * factor + f;
      const float p = pos_repeated ? pos[e] : pos[j];
      const float d = p - neg[e];
      float v, gp;   // gp = d loss_e / d pos ; d/d neg = -gp
      if (kind == 0) {   // -log sigmoid(d)
        v = fmaxf(-d, 0.f) + softplus_neg_abs(d);
        gp = -sigmoidf(-d);
      } else {           // relu(margin - d); torch's clamp_min passes the gradient at the hinge t == 0
        const float t = margin - d;
        v = fmaxf(t, 0.f);
        gp = t >= 0.f ? -1.f : 0.f;
      }
      acc += v;
      if (dneg) dneg[e] = -gp * inv_n;
      if (dpos && pos_repeated) dpos[e] = gp * inv_n;
      gp_sum += gp;
    }
    if (dpos && !pos_repeated) dpos[j] = gp_sum * inv_n;
  }
  block_sum_store(acc, partial);
}

// kind 2 bce, 3 focal over the concatenation [pos with label 1, neg with label 0]
__global__ void __launch_bounds__(THREADS)
pair_class_kernel(const float* __restrict__ pos, int64_t n_pos, const float* __restrict__ neg, int64_t n_neg,
                  int kind, float alpha, float gamma, float scale, float* __restrict__ dpos,
                  float* __restrict__ dneg, double* __restrict__ partial) {
  float acc = 0.f;
  const int64_t n = n_pos + n_neg;
  for (int64_t i = (int64_t)blockIdx.x * THREADS + threadIdx.x; i < n; i += (int64_t)gridDim.x * THREADS) {
    const bool is_pos = i < n_pos;
    const float x = is_pos ? pos[i] : neg[i - n_pos];
    const float y = is_pos ? 1.f : 0.f;
    float v, g;
    if (kind == 2) { v = bce(x, y); g = sigmoidf(x) - y; }
    else { v = focal(x, y, alpha, gamma, &g); }
    acc += v;
    if (is_pos) { if (dpos) dpos[i] = g * scale; }
    else if (dneg) dneg[i - n_pos] = g * scale;
  }
  block_sum_store(acc, partial);
}

__global__ void final_sum_kernel(const double* __restrict__ partial, int nb, double scale, float* __restrict__ out) {
  __shared__ double sh[32];
  double d = 0.0;
  for (int i = threadIdx.x; i < nb; i += blockDim.x) d += partial[i];
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) d += __shfl_xor_sync(0xffffffffu, d, o);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = d;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int i = 0; i < (int)(blockDim.x >> 5); ++i) s += sh[i];
    *out = (float)(s * scale);
  }
}

// One warp per row of the in-batch logit matrix S[B, B] (already U I^T): logits = S / temperature
// - log(clip(correction[col], 1e-8, 1)); accidental hits (same item id, off-diagonal) -> float min;
// loss_row = logsumexp(row) - row[diag].  Optionally overwrites S with d(mean loss)/dS.
__global__ void __launch_bounds__(THREADS)
softmax_rows_kernel(float* __restrict__ S, int64_t lds, int B, float inv_temp, const float* __restrict__ correction,
                    const int64_t* __restrict__ item_ids, int write_grad, float inv_B, double* __restrict__ partial) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wpb = THREADS / 32;
  float acc = 0.f;
  for (int r = blockIdx.x * wpb + warp; r < B; r += gridDim.x * wpb) {
    float* row = S + (int64_t)r * lds;
    const int64_t my_item = item_ids ? item_ids[r] : 0;
    auto logit = [&](int c) -> float {
      float v = (inv_temp != 0.f) ? row[c] * inv_temp : 0.f;          // divide_no_nan
      if (correction) v -= logf(fminf(fmaxf(correction[c], 1e-8f), 1.f));
      if (item_ids && c != r && item_ids[c] == my_item) v = -3.402823466e38f;
      return v;
    };
    float mx = -3.402823466e38f;
    for (int c = lane; c < B; c += 32) mx = fmaxf(mx, logit(c));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float se = 0.f;
    for (int c = lane; c < B; c += 32) se += expf(logit(c) - mx);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) se += __shfl_xor_sync(0xffffffffu, se, o);
    const float lse = mx + logf(se);
    const float diag = logit(r);
    if (lane == 0) acc += lse - diag;
    if (write_grad) {
      __syncwarp();
      for (int c = lane; c < B; c += 32) {
        const float lg = logit(c);
        const bool masked = item_ids && c != r && item_ids[c] == my_item;
        float g = masked ? 0.f : (expf(lg - lse) - (c == r ? 1.f : 0.f)) * inv_temp * inv_B;
        row[c] = g;
      }
    }
  }
  block_sum_store(acc, partial);
}

// ---- sampled-class losses of YouTubeRetrieval (tf.nn.sampled_softmax_loss / tf.nn.nce_loss through
// _compute_sampled_logits, remove_accidental_hits=True, subtract_log_q=True) -----------------------------------
// TensorFlow's ExpectedCountHelper (range_sampler.cc) in float: p S when every draw was distinct, else
// -expm1(num_tries log1p(-p)); p = 1 / n_items (uniform, the sampler's float inv_range) or
// log((c + 2) / (c + 1)) / log1p(n_items) (log-uniform, double, then float).
__device__ __forceinline__ float expected_count(int sampler_kind, int64_t c, int64_t n_items, int S, int64_t tries) {
  const float p = sampler_kind == 0 ? (float)(1.0 / (double)n_items)
                                    : (float)(log((c + 2.0) / (c + 1.0)) / log1p((double)n_items));
  if (tries == (int64_t)S) return p * (float)S;
  return -expm1f((float)tries * log1pf(-p));
}

// adj[i] = bias[id] - log E(id) for the S sampled ids, then the B labels
__global__ void __launch_bounds__(THREADS)
sampled_adjust_kernel(const int64_t* __restrict__ sampled, int S, const int64_t* __restrict__ labels, int B,
                      const float* __restrict__ bias, int sampler_kind, int64_t n_items,
                      const int64_t* __restrict__ num_tries, float* __restrict__ adj) {
  const int i = blockIdx.x * THREADS + threadIdx.x;
  if (i >= S + B) return;
  const int64_t id = i < S ? sampled[i] : labels[i - S];
  adj[i] = bias[id] - logf(expected_count(sampler_kind, id, n_items, S, *num_tries));
}

// One warp per row r: z0 = true_dot[r] + adj[S + r] (the label, column 0), z_s = L[r, s] + adj[s]; a sampled id
// equal to the row's label is an accidental hit (TensorFlow adds -FLT_MAX: it contributes exactly nothing, so it
// is skipped here and its gradient is 0).  kind 0 softmax CE over [z0, z_s] (online max / sum per lane, merged in
// a fixed shuffle tree), kind 1 NCE: sigmoid CE(z0, 1) + sum_s sigmoid CE(z_s, 0).  L is overwritten with
// d(mean loss) / d z_s, dtrue[r] = d(mean loss) / d z0.
__global__ void __launch_bounds__(THREADS)
sampled_rows_kernel(float* __restrict__ L, int64_t ldl, int B, int S, int kind, const float* __restrict__ true_dot,
                    const int64_t* __restrict__ labels, const int64_t* __restrict__ sampled,
                    const float* __restrict__ adj, float inv_B, float* __restrict__ dtrue,
                    double* __restrict__ partial) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int wpb = THREADS / 32;
  float acc = 0.f;
  for (int r = blockIdx.x * wpb + warp; r < B; r += gridDim.x * wpb) {
    float* row = L + (int64_t)r * ldl;
    const int64_t lab = labels[r];
    const float z0 = true_dot[r] + adj[S + r];
    float loss, d0;
    if (kind == 0) {
      float m = z0, s = 0.f;
      for (int c = lane; c < S; c += 32) {
        if (sampled[c] == lab) continue;
        const float z = row[c] + adj[c];
        if (z > m) { s = s * expf(m - z) + 1.f; m = z; }
        else s += expf(z - m);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, m, o), s2 = __shfl_xor_sync(0xffffffffu, s, o);
        const float mm = fmaxf(m, m2);
        s = s * expf(m - mm) + s2 * expf(m2 - mm);
        m = mm;
      }
      const float lse = m + logf(s + expf(z0 - m));
      loss = lse - z0;
      d0 = (expf(z0 - lse) - 1.f) * inv_B;
      for (int c = lane; c < S; c += 32)
        row[c] = sampled[c] == lab ? 0.f : expf(row[c] + adj[c] - lse) * inv_B;
    } else {
      float ls = 0.f;
      for (int c = lane; c < S; c += 32) {
        if (sampled[c] == lab) { row[c] = 0.f; continue; }
        const float z = row[c] + adj[c];
        ls += bce(z, 0.f);
        row[c] = sigmoidf(z) * inv_B;
      }
      loss = warp_sum(ls) + bce(z0, 1.f);
      d0 = (sigmoidf(z0) - 1.f) * inv_B;
    }
    if (lane == 0) {
      acc += loss;
      dtrue[r] = d0;
    }
  }
  block_sum_store(acc, partial);
}

static inline int grid_for(int64_t n) {
  int64_t b = (n + THREADS - 1) / THREADS;
  if (b < 1) b = 1;
  if (b > MAX_BLOCKS) b = MAX_BLOCKS;
  return (int)b;
}

}  // namespace loss
}  // namespace b200

using namespace b200;
using namespace b200::loss;

extern "C" size_t b200_loss_workspace_bytes(void) { return (size_t)MAX_BLOCKS * sizeof(double); }

extern "C" int b200_pointwise_loss(const float* logits, const float* labels, int64_t n, int32_t kind,
                                   float alpha, float gamma, float* loss_out, float* dlogits,
                                   void* workspace, size_t workspace_bytes, void* stream) {
  B200_REQUIRE(n > 0, "empty batch");
  B200_REQUIRE(kind >= 0 && kind <= 2, "pointwise loss kind must be 0 (bce), 1 (focal) or 2 (mse)");
  B200_REQUIRE(workspace && workspace_bytes >= b200_loss_workspace_bytes(), "workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int g = grid_for(n);
  pointwise_kernel<<<g, THREADS, 0, st>>>(logits, labels, n, kind, alpha, gamma, 1.f / (float)n, dlogits,
                                          (double*)workspace);
  final_sum_kernel<<<1, 256, 0, st>>>((const double*)workspace, g, 1.0 / (double)n, loss_out);
  B200_CUDA_OK(cudaGetLastError());
  count_launch(2);
  return 0;
}

extern "C" int b200_pairwise_loss(const float* pos, int64_t n_pos, const float* neg, int64_t n_neg,
                                  int32_t kind, float margin, float alpha, float gamma, int32_t mean,
                                  float* loss_out, float* dpos, float* dneg, void* workspace,
                                  size_t workspace_bytes, void* stream) {
  B200_REQUIRE(n_pos > 0 && n_neg > 0, "empty batch");
  B200_REQUIRE(kind >= 0 && kind <= 3, "pairwise loss kind must be 0 (bpr), 1 (max_margin), 2 (bce), 3 (focal)");
  B200_REQUIRE(workspace && workspace_bytes >= b200_loss_workspace_bytes(), "workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  if (kind <= 1) {
    // positives either already repeated (n_pos == n_neg) or broadcast over n_neg / n_pos negatives
    // (compute_pair_scores, torchops/loss.py:63-90)
    B200_REQUIRE(n_neg % n_pos == 0, "negatives length %lld is not a multiple of positives length %lld",
                 (long long)n_neg, (long long)n_pos);
    const int factor = (int)(n_neg / n_pos);
    const int g = grid_for(n_pos);
    pair_rank_kernel<<<g, THREADS, 0, st>>>(pos, n_pos, neg, factor, 0, kind, margin, 1.f / (float)n_neg, dpos,
                                            dneg, (double*)workspace);
    final_sum_kernel<<<1, 256, 0, st>>>((const double*)workspace, g, 1.0 / (double)n_neg, loss_out);
  } else {
    const int64_t n = n_pos + n_neg;
    const int g = grid_for(n);
    const double scale = mean ? 1.0 / (double)n : 1.0;
    pair_class_kernel<<<g, THREADS, 0, st>>>(pos, n_pos, neg, n_neg, kind, alpha, gamma, (float)scale, dpos, dneg,
                                             (double*)workspace);
    final_sum_kernel<<<1, 256, 0, st>>>((const double*)workspace, g, scale, loss_out);
  }
  B200_CUDA_OK(cudaGetLastError());
  count_launch(2);
  return 0;
}

extern "C" int b200_softmax_inbatch_loss(float* S, int64_t lds, int32_t B, float temperature,
                                         const float* correction, const int64_t* item_ids,
                                         int32_t write_grad, float* loss_out, void* workspace,
                                         size_t workspace_bytes, void* stream) {
  B200_REQUIRE(B > 0 && lds >= B, "bad shape");
  B200_REQUIRE(workspace && workspace_bytes >= b200_loss_workspace_bytes(), "workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int wpb = THREADS / 32;
  int g = (B + wpb - 1) / wpb;
  if (g > MAX_BLOCKS) g = MAX_BLOCKS;
  const float inv_temp = temperature != 0.f ? 1.f / temperature : 0.f;
  softmax_rows_kernel<<<g, THREADS, 0, st>>>(S, lds, B, inv_temp, correction, item_ids, write_grad,
                                             1.f / (float)B, (double*)workspace);
  final_sum_kernel<<<1, 256, 0, st>>>((const double*)workspace, g, 1.0 / (double)B, loss_out);
  B200_CUDA_OK(cudaGetLastError());
  count_launch(2);
  return 0;
}

extern "C" size_t b200_sampled_class_loss_workspace_bytes(int32_t B, int32_t S) {
  return b200_loss_workspace_bytes() + (size_t)(B > 0 ? B : 0) * 4 + (size_t)(S > 0 ? S : 0) * 4;
}

extern "C" int b200_sampled_class_loss(int32_t loss_kind, float* logits, int64_t ld, int32_t B, int32_t S,
                                       const float* true_dot, const int64_t* labels, const int64_t* sampled,
                                       const float* bias, int32_t sampler_kind, int64_t n_items,
                                       const int64_t* num_tries, float* loss_out, float* dtrue, void* workspace,
                                       size_t workspace_bytes, void* stream) {
  B200_REQUIRE(loss_kind == 0 || loss_kind == 1, "b200_sampled_class_loss: loss kind must be 0 (softmax) or 1 (nce)");
  B200_REQUIRE(sampler_kind == 0 || sampler_kind == 1,
               "b200_sampled_class_loss: sampler kind must be 0 (uniform) or 1 (log-uniform)");
  B200_REQUIRE(B >= 1 && S >= 1 && S <= B200_UNIQUE_MAX_SAMPLED && ld >= S && n_items >= S,
               "b200_sampled_class_loss: bad shape B %d, S %d, ld %lld, n_items %lld", B, S, (long long)ld,
               (long long)n_items);
  B200_REQUIRE(logits && true_dot && labels && sampled && bias && num_tries && loss_out && dtrue,
               "b200_sampled_class_loss: null pointer");
  B200_REQUIRE(workspace && workspace_bytes >= b200_sampled_class_loss_workspace_bytes(B, S),
               "b200_sampled_class_loss: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  double* partial = (double*)workspace;
  float* adj = (float*)((char*)workspace + b200_loss_workspace_bytes());
  sampled_adjust_kernel<<<(unsigned)ceil_div64((int64_t)S + B, THREADS), THREADS, 0, st>>>(
      sampled, S, labels, B, bias, sampler_kind, n_items, num_tries, adj);
  const int wpb = THREADS / 32;
  int g = (B + wpb - 1) / wpb;
  if (g > MAX_BLOCKS) g = MAX_BLOCKS;
  sampled_rows_kernel<<<g, THREADS, 0, st>>>(logits, ld, B, S, loss_kind, true_dot, labels, sampled, adj,
                                             1.f / (float)B, dtrue, partial);
  final_sum_kernel<<<1, 256, 0, st>>>(partial, g, 1.0 / (double)B, loss_out);
  B200_CUDA_OK(cudaGetLastError());
  count_launch(3);
  return 0;
}
