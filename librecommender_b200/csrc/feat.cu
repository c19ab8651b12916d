// K1 — fused multi-field embedding gather + FM pairwise interaction + linear term, and the small
// dense kernels of the FM / DeepFM / MLP heads (K3, fp32).
//
// Replaces, for inference rows:
//   embedding_lookup / compute_sparse_feats / compute_dense_feats
//       (libreco/layers/embedding.py:4-23, libreco/tfops/features.py:6-44,121-148)
//   the feed construction of predict_tf_feat / process_tf_feat
//       (libreco/prediction/predict.py:43-92, libreco/recommendation/preprocess.py:104-212):
//       per-row feature indices are read IN THE KERNEL from the per-user / per-item unique tables
//       (data_info.user_sparse_unique, item_sparse_unique, ...) — the [B*N, F] feed is never built
//   FM head    (libreco/algorithms/fm.py:152-171)
//   DeepFM head (libreco/algorithms/deepfm.py:155-174) through b200_linear_f32 + b200_concat_dense
//
// HBM-bound gather: per row (2+F_s) random reads of 4K (+4) bytes.  One sub-warp of
// lpr = min(32, pow2 >= K) lanes per row, lanes stride the embedding width; field indices are
// loaded cooperatively and broadcast by shuffle, 4 gathers in flight.
#include <algorithm>
#include "common.cuh"
#include "feat_common.cuh"
#include "../../include/b200reco.h"

namespace b200 {
namespace feat {

// feat_tma.cu: persistent bulk-copy staged gather (1 = launched, 0 = shape not eligible, < 0 = error)
int launch_feat_forward_tma(const b200_feat_layout* L, const b200_feat_tables* T, const int64_t* users,
                            const int64_t* items, int64_t R, int64_t grid_items, int64_t row_offset,
                            float* concat, int64_t ld_concat, float* pw, int64_t ld_pw, float* lin,
                            float* fm_out, const float* lin_kernel, float lin_bias, const float* bn_scale,
                            const float* bn_shift, const float* pw_kernel, float pw_bias, float* ssum,
                            float* sqsum, int64_t ld_s, cudaStream_t stream);

constexpr int MAX_T = 8;   // K <= 256

struct Out {
  float* concat; int64_t ld_concat;   // [R, F*K]  (deep / tower input) or null
  float* pw; int64_t ld_pw;           // [R, K]    FM pairwise term or null
  float* lin;                         // [R]       Dense1(linear features) incl. bias, or null
  float* fm_out;                      // [R]       full FM logit, or null
  float* ssum; float* sqsum; int64_t ld_s;   // [R, K] sum_f e and sum_f e^2 (hoisted all-items scoring), or null
};

struct Head {           // weights of the heads that can be fused here
  const float* lin_kernel;   // [2+F_s+F_d]   Dense(1) on the concatenated linear features
  float lin_bias;
  const float* bn_scale;     // [K] folded BN of the FM pairwise term (or null)
  const float* bn_shift;     // [K]
  const float* pw_kernel;    // [K]  Dense(1, elu) on the pairwise term
  float pw_bias;
};

__global__ void __launch_bounds__(256)
feat_forward_kernel(const b200_feat_layout L, const b200_feat_tables T, const int64_t* __restrict__ users,
                    const int64_t* __restrict__ items, int64_t R, int64_t grid_items,
                    int64_t row_offset, Out o, Head h, int lpr, int Tn) {
  const int lane = threadIdx.x & 31;
  const int rows_per_warp = 32 / lpr;
  const int64_t warp = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int g = lane / lpr, li = lane % lpr;
  const int64_t r = warp * rows_per_warp + g;
  const int gbase = g * lpr;
  const uint32_t gmask = (lpr == 32) ? 0xffffffffu : (((1u << lpr) - 1u) << gbase);
  if (r >= R) return;
  // row -> (user, item): explicit pairs, or the implicit grid "user r / N  x  item r % N"
  int64_t u, it;
  if (grid_items > 0) { const int64_t rg = r + row_offset; u = users[rg / grid_items]; it = rg % grid_items; }
  else { u = users[r]; it = items[r]; }
  const int K = L.embed_size;

  float s[MAX_T], s2[MAX_T];
#pragma unroll
  for (int t = 0; t < MAX_T; ++t) { s[t] = 0.f; s2[t] = 0.f; }
  float lin_acc = 0.f;

  int fpos = 0;   // position of the next field inside the concatenated row
  auto add_field = [&](int f, const float* __restrict__ rowp, float scale) {
#pragma unroll
    for (int t = 0; t < MAX_T; ++t) {
      const int k = li + t * lpr;
      if (t < Tn && k < K) {
        const float e = __ldg(rowp + k) * scale;
        s[t] += e;
        s2[t] = fmaf(e, e, s2[t]);
        if (o.concat) o.concat[r * o.ld_concat + (int64_t)f * K + k] = e;
      }
    }
  };
  // user / item id embeddings (fields 0, 1; a tower keeps only its own side)
  const bool want_lin = (o.lin != nullptr) || (o.fm_out != nullptr);
  if (L.id_mask & 1) {
    add_field(fpos, T.user_embeds + u * K, 1.f);
    if (want_lin && li == 0) lin_acc = fmaf(__ldg(T.user_linear + u), h.lin_kernel[fpos], lin_acc);
    ++fpos;
  }
  if (L.id_mask & 2) {
    add_field(fpos, T.item_embeds + it * K, 1.f);
    if (want_lin && li == 0) lin_acc = fmaf(__ldg(T.item_linear + it), h.lin_kernel[fpos], lin_acc);
    ++fpos;
  }
  // sparse fields: indices loaded cooperatively (lpr at a time), rows gathered 4 at a time
  for (int f0 = 0; f0 < L.n_sparse; f0 += lpr) {
    const int f = f0 + li;
    int32_t idx = 0;
    if (f < L.n_sparse) {
      idx = sparse_index(L, r, u, it, f);
      if (want_lin) lin_acc = fmaf(__ldg(T.sparse_linear + idx), h.lin_kernel[fpos + f], lin_acc);
    }
    const int cnt = min(lpr, L.n_sparse - f0);
    if (Tn == 1) {
      // common case K <= 32: one element per lane and field -> issue 8 row gathers before using them
      const bool kok = li < K;
      for (int q0 = 0; q0 < cnt; q0 += 8) {
        float e[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int32_t ix = __shfl_sync(gmask, idx, gbase + min(q0 + u, cnt - 1));
          e[u] = (kok && q0 + u < cnt) ? __ldg(T.sparse_embeds + (int64_t)ix * K + li) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          if (q0 + u < cnt) {
            s[0] += e[u];
            s2[0] = fmaf(e[u], e[u], s2[0]);
            if (o.concat && kok) o.concat[r * o.ld_concat + (int64_t)(fpos + f0 + q0 + u) * K + li] = e[u];
          }
        }
      }
    } else {
      for (int q = 0; q < cnt; ++q) {
        const int32_t ix = __shfl_sync(gmask, idx, gbase + q);
        add_field(fpos + f0 + q, T.sparse_embeds + (int64_t)ix * K, 1.f);
      }
    }
  }
  fpos += L.n_sparse;
  // dense fields: value * embedding row of the field
  for (int f0 = 0; f0 < L.n_dense; f0 += lpr) {
    const int f = f0 + li;
    float x = 0.f;
    if (f < L.n_dense) {
      x = dense_value(L, r, u, it, f);
      if (want_lin) lin_acc = fmaf(__ldg(T.dense_linear + L.dense_embed_row[f]) * x, h.lin_kernel[fpos + f], lin_acc);
    }
    const int cnt = min(lpr, L.n_dense - f0);
    for (int q = 0; q < cnt; ++q) {
      const float xv = __shfl_sync(gmask, x, gbase + q);
      add_field(fpos + f0 + q, T.dense_embeds + (int64_t)L.dense_embed_row[f0 + q] * K, xv);
    }
  }
  // epilogue: pairwise term, linear term, FM logit
  float head_acc = 0.f;
#pragma unroll
  for (int t = 0; t < MAX_T; ++t) {
    const int k = li + t * lpr;
    if (t < Tn && k < K) {
      const float pw = 0.5f * (s[t] * s[t] - s2[t]);
      if (o.pw) o.pw[r * o.ld_pw + k] = pw;
      if (o.ssum) { o.ssum[r * o.ld_s + k] = s[t]; o.sqsum[r * o.ld_s + k] = s2[t]; }
      if (o.fm_out) {
        const float z = h.bn_scale ? fmaf(pw, h.bn_scale[k], h.bn_shift[k]) : pw;
        head_acc = fmaf(z, h.pw_kernel[k], head_acc);
      }
    }
  }
  if (want_lin) lin_acc = subwarp_sum(lin_acc, lpr, gmask) + h.lin_bias;
  if (o.fm_out) {
    head_acc = subwarp_sum(head_acc, lpr, gmask) + h.pw_bias;
    const float elu = head_acc > 0.f ? head_acc : expm1f(head_acc);
    if (li == 0) o.fm_out[r] = lin_acc + elu;
  }
  if (o.lin && li == 0) o.lin[r] = lin_acc;
}

// ---- fast path for K % 4 == 0, K <= 32: one warp per row, ONE LANE PER FIELD.
// Every lane gathers whole embedding rows of its fields (K/4 16-byte loads, several fields in
// flight), accumulates its private sum / sum of squares over its fields and writes its slice of the
// concatenated row (consecutive lanes = consecutive fields = fully coalesced stores); the cross-lane
// reduction over fields happens once per row.
template <int K4>
__global__ void __launch_bounds__(256, (K4 <= 4 ? 3 : 2))
feat_forward_lanefield_kernel(const b200_feat_layout L, const b200_feat_tables T,
                              const int64_t* __restrict__ users, const int64_t* __restrict__ items,
                              int64_t R, int64_t grid_items, int64_t row_offset, Out o, Head h) {
  constexpr int K = K4 * 4;
  constexpr int MAXJ = 4;                      // fields per lane and chunk (128 fields per chunk)
  const int lane = threadIdx.x & 31;
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  if (r >= R) return;
  int64_t u, it;
  if (grid_items > 0) { const int64_t rg = r + row_offset; u = users[rg / grid_items]; it = rg % grid_items; }
  else { u = users[r]; it = items[r]; }
  const int n_id = ((L.id_mask & 1) ? 1 : 0) + ((L.id_mask & 2) ? 1 : 0);
  const int F = n_id + L.n_sparse + L.n_dense;
  const bool want_lin = (o.lin != nullptr) || (o.fm_out != nullptr);
  float4 s[K4], s2[K4];
#pragma unroll
  for (int q = 0; q < K4; ++q) { s[q] = make_float4(0.f, 0.f, 0.f, 0.f); s2[q] = s[q]; }
  float lin_acc = 0.f;
  for (int f0 = 0; f0 < F; f0 += 32 * MAXJ) {
    // phase 1: resolve the source row of EVERY field of this lane (all index loads of the chunk in
    // flight together: one dependent round trip instead of one per pair of fields)
    const float4* src[MAXJ];
    float scale[MAXJ];
    bool valid[MAXJ];
#pragma unroll
    for (int j = 0; j < MAXJ; ++j) {
      const int f = f0 + j * 32 + lane;
      valid[j] = f < F;
      scale[j] = 1.f;
      const float* rowp = T.user_embeds;       // placeholder for invalid lanes
      float lw = 0.f;
      if (valid[j]) {
        if (f < n_id) {
          const bool is_user = (L.id_mask & 1) && f == 0;
          rowp = is_user ? T.user_embeds + u * K : T.item_embeds + it * K;
          if (want_lin) lw = is_user ? __ldg(T.user_linear + u) : __ldg(T.item_linear + it);
        } else if (f < n_id + L.n_sparse) {
          const int32_t idx = sparse_index(L, r, u, it, f - n_id);
          rowp = T.sparse_embeds + (int64_t)idx * K;
          if (want_lin) lw = __ldg(T.sparse_linear + idx);
        } else {
          const int fd = f - n_id - L.n_sparse;
          const float x = dense_value(L, r, u, it, fd);
          rowp = T.dense_embeds + (int64_t)L.dense_embed_row[fd] * K;
          scale[j] = x;
          if (want_lin) lw = __ldg(T.dense_linear + L.dense_embed_row[fd]) * x;
        }
        if (want_lin) lin_acc = fmaf(lw, h.lin_kernel[f], lin_acc);
      }
      src[j] = reinterpret_cast<const float4*>(rowp);
    }
    // phase 2: the row gathers, two fields (2 x K4 16-byte loads) in flight per lane
#pragma unroll
    for (int j0 = 0; j0 < MAXJ; j0 += 2) {
      float4 e[2][K4];
#pragma unroll
      for (int jj = 0; jj < 2; ++jj)
#pragma unroll
        for (int q = 0; q < K4; ++q)
          e[jj][q] = valid[j0 + jj] ? __ldg(src[j0 + jj] + q) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
      for (int jj = 0; jj < 2; ++jj) {
        const int j = j0 + jj;
        if (!valid[j]) continue;
        const int f = f0 + j * 32 + lane;
#pragma unroll
        for (int q = 0; q < K4; ++q) {
          float4 v = e[jj][q];
          v.x *= scale[j]; v.y *= scale[j]; v.z *= scale[j]; v.w *= scale[j];
          s[q].x += v.x; s[q].y += v.y; s[q].z += v.z; s[q].w += v.w;
          s2[q].x = fmaf(v.x, v.x, s2[q].x); s2[q].y = fmaf(v.y, v.y, s2[q].y);
          s2[q].z = fmaf(v.z, v.z, s2[q].z); s2[q].w = fmaf(v.w, v.w, s2[q].w);
          if (o.concat) *(reinterpret_cast<float4*>(o.concat + r * o.ld_concat + (int64_t)f * K) + q) = v;
        }
      }
    }
  }
  if (!o.pw && !o.fm_out && !o.lin && !o.ssum) return;
  // one reduction over the 32 lanes (= over the fields) per row
  float head_acc = 0.f;
#pragma unroll
  for (int q = 0; q < K4; ++q) {
    float sv[4] = {s[q].x, s[q].y, s[q].z, s[q].w};
    float s2v[4] = {s2[q].x, s2[q].y, s2[q].z, s2[q].w};
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const float a = warp_sum(sv[c]);
      const float b = warp_sum(s2v[c]);
      const float pw = 0.5f * (a * a - b);
      const int k = q * 4 + c;
      if (o.pw && lane == 0) o.pw[r * o.ld_pw + k] = pw;
      if (o.ssum && lane == 0) { o.ssum[r * o.ld_s + k] = a; o.sqsum[r * o.ld_s + k] = b; }
      if (o.fm_out) {
        const float z = h.bn_scale ? fmaf(pw, h.bn_scale[k], h.bn_shift[k]) : pw;
        head_acc = fmaf(z, h.pw_kernel[k], head_acc);
      }
    }
  }
  if (want_lin) lin_acc = warp_sum(lin_acc) + h.lin_bias;
  if (o.fm_out && lane == 0) {
    head_acc += h.pw_bias;
    o.fm_out[r] = lin_acc + (head_acc > 0.f ? head_acc : expm1f(head_acc));
  }
  if (o.lin && lane == 0) o.lin[r] = lin_acc;
}

// ---- fast path for K in {4, 8, 16, 32}: one warp per row, K/4 LANES PER FIELD (a "field group" of 32/(K/4)
// fields per warp instruction).  Every warp-level load reads 32/(K/4) whole embedding rows with 16 B per lane
// (one L1 wavefront per 128 B instead of one per lane), every warp-level store writes 512 contiguous bytes of
// the concatenated row, and the field sums need log2(32/(K/4)) shuffle steps on 8 values instead of a 32-lane
// reduction of 2K values.  Field metadata (side, column, head weight) is staged once per block in shared
// memory — indexing the by-value layout struct with a per-lane field number serialises in the constant cache.
// U steps are resolved (index loads) and then gathered together: U row reads in flight per lane.
// Measured ceiling for this access pattern (tools/ubench/gather.cu): 64-B random rows 2.7 TB/s from HBM,
// 5.7 TB/s when the table mostly fits the 126 MB L2.
template <int K4>
__global__ void __launch_bounds__(256, 3)
feat_forward_fieldgroup_kernel(const b200_feat_layout L, const b200_feat_tables T,
                               const int64_t* __restrict__ users, const int64_t* __restrict__ items,
                               int64_t R, int64_t grid_items, int64_t row_offset, Out o, Head h) {
  constexpr int K = K4 * 4;
  constexpr int FPW = 32 / K4;                 // fields per warp instruction
  constexpr int U = 8;                         // steps in flight
  constexpr int MAXF = 2 + 2 * B200_MAX_FIELDS;
  __shared__ int32_t sh_code[MAXF];            // kind | column << 3
  __shared__ int32_t sh_drow[MAXF];            // dense fields: row of dense_embeds / dense_linear
  __shared__ float sh_link[MAXF];              // Dense(1) weight of the field's linear feature
  const int n_id = ((L.id_mask & 1) ? 1 : 0) + ((L.id_mask & 2) ? 1 : 0);
  const int F = n_id + L.n_sparse + L.n_dense;
  const bool want_lin = (o.lin != nullptr) || (o.fm_out != nullptr);
  for (int f = threadIdx.x; f < F; f += blockDim.x) {
    int kind, col = 0, drow = 0;
    if (f < n_id) kind = ((L.id_mask & 1) && f == 0) ? 0 : 1;
    else if (f < n_id + L.n_sparse) {
      const int fs = f - n_id;
      if (L.sparse_rows) { kind = 4; col = fs; }
      else { kind = L.sparse_side[fs] == 0 ? 2 : 3; col = L.sparse_col[fs]; }
    } else {
      const int fd = f - n_id - L.n_sparse;
      drow = L.dense_embed_row[fd];
      if (L.dense_rows) { kind = 7; col = fd; }
      else { kind = L.dense_side[fd] == 0 ? 5 : 6; col = L.dense_col[fd]; }
    }
    sh_code[f] = kind | (col << 3);
    sh_drow[f] = drow;
    sh_link[f] = want_lin ? h.lin_kernel[f] : 0.f;
  }
  __syncthreads();
  const int lane = threadIdx.x & 31;
  const int fg = lane / K4, q = lane % K4;
  const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  for (int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); r < R; r += n_warps) {
    int64_t u, it;
    if (grid_items > 0) { const int64_t rg = r + row_offset; u = users[rg / grid_items]; it = rg % grid_items; }
    else { u = users[r]; it = items[r]; }
    float4 s = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s;
    float lin_acc = 0.f;
    for (int f0 = 0; f0 < F; f0 += FPW * U) {
      const float4* src[U];
      float scale[U];
      // phase 1: source row of this lane's field in each of the U steps (the index loads go out together)
#pragma unroll
      for (int j = 0; j < U; ++j) {
        const int f = f0 + j * FPW + fg;
        src[j] = nullptr;
        scale[j] = 1.f;
        if (f < F) {
          const int code = sh_code[f];
          const int kind = code & 7, col = code >> 3;
          const float* rowp;
          float lw = 0.f;
          if (kind < 2) {
            rowp = kind == 0 ? T.user_embeds + u * K : T.item_embeds + it * K;
            if (want_lin) lw = kind == 0 ? __ldg(T.user_linear + u) : __ldg(T.item_linear + it);
          } else if (kind < 5) {
            const int32_t* ip = kind == 2 ? L.user_sparse_unique + u * L.ld_us + col
                              : kind == 3 ? L.item_sparse_unique + it * L.ld_is + col
                                          : L.sparse_rows + r * L.ld_sparse_rows + col;
            const int32_t idx = __ldg(ip);
            rowp = T.sparse_embeds + (int64_t)idx * K;
            if (want_lin) lw = __ldg(T.sparse_linear + idx);
          } else {
            const float* xp = kind == 5 ? L.user_dense_unique + u * L.ld_ud + col
                            : kind == 6 ? L.item_dense_unique + it * L.ld_id + col
                                        : L.dense_rows + r * L.ld_dense_rows + col;
            const float x = __ldg(xp);
            const int drow = sh_drow[f];
            rowp = T.dense_embeds + (int64_t)drow * K;
            scale[j] = x;
            if (want_lin) lw = __ldg(T.dense_linear + drow) * x;
          }
          if (want_lin && q == 0) lin_acc = fmaf(lw, sh_link[f], lin_acc);
          src[j] = reinterpret_cast<const float4*>(rowp) + q;
        }
      }
      // phase 2: U row reads in flight (16 B per lane, K/4 lanes per row)
      float4 e[U];
#pragma unroll
      for (int j = 0; j < U; ++j) e[j] = src[j] ? __ldg(src[j]) : make_float4(0.f, 0.f, 0.f, 0.f);
      // phase 3: sums + the concatenated row
#pragma unroll
      for (int j = 0; j < U; ++j) {
        if (!src[j]) continue;
        float4 v = e[j];
        v.x *= scale[j]; v.y *= scale[j]; v.z *= scale[j]; v.w *= scale[j];
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        s2.x = fmaf(v.x, v.x, s2.x); s2.y = fmaf(v.y, v.y, s2.y);
        s2.z = fmaf(v.z, v.z, s2.z); s2.w = fmaf(v.w, v.w, s2.w);
        if (o.concat) {
          const int f = f0 + j * FPW + fg;
          *reinterpret_cast<float4*>(o.concat + r * o.ld_concat + (int64_t)f * K + q * 4) = v;
        }
      }
    }
    if (!o.pw && !o.fm_out && !o.lin && !o.ssum) continue;
    // sum over the field groups: lanes with equal q hold the same 4 embedding columns
#pragma unroll
    for (int off = K4; off < 32; off <<= 1) {
      s.x += __shfl_xor_sync(0xffffffffu, s.x, off); s.y += __shfl_xor_sync(0xffffffffu, s.y, off);
      s.z += __shfl_xor_sync(0xffffffffu, s.z, off); s.w += __shfl_xor_sync(0xffffffffu, s.w, off);
      s2.x += __shfl_xor_sync(0xffffffffu, s2.x, off); s2.y += __shfl_xor_sync(0xffffffffu, s2.y, off);
      s2.z += __shfl_xor_sync(0xffffffffu, s2.z, off); s2.w += __shfl_xor_sync(0xffffffffu, s2.w, off);
    }
    const float sv[4] = {s.x, s.y, s.z, s.w};
    const float s2v[4] = {s2.x, s2.y, s2.z, s2.w};
    float head_acc = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int k = q * 4 + c;
      const float pw = 0.5f * (sv[c] * sv[c] - s2v[c]);
      if (fg == 0) {
        if (o.pw) o.pw[r * o.ld_pw + k] = pw;
        if (o.ssum) { o.ssum[r * o.ld_s + k] = sv[c]; o.sqsum[r * o.ld_s + k] = s2v[c]; }
      }
      if (o.fm_out) {
        const float z = h.bn_scale ? fmaf(pw, h.bn_scale[k], h.bn_shift[k]) : pw;
        head_acc = fmaf(z, h.pw_kernel[k], head_acc);
      }
    }
    if (want_lin) lin_acc = warp_sum(lin_acc) + h.lin_bias;
    if (o.fm_out) {
#pragma unroll
      for (int off = 1; off < K4; off <<= 1) head_acc += __shfl_xor_sync(0xffffffffu, head_acc, off);
      head_acc += h.pw_bias;
      if (lane == 0) o.fm_out[r] = lin_acc + (head_acc > 0.f ? head_acc : expm1f(head_acc));
    }
    if (o.lin && lane == 0) o.lin[r] = lin_acc;
  }
}

// ---- software-pipelined register gather (default for >= 4096 rows, K in {4, 8, 16, 32}, <= 16 steps per row):
// the field-group layout with (a) the index loads of the NEXT batch of 8 steps issued while the row gathers of the
// current batch are in flight — the dependent chain ids -> feature index -> embedding row costs one memory round
// trip per batch instead of two (ncu of the unpipelined kernel: 68 % of the stall cycles long-scoreboard, DRAM at
// 18 %) — and (b) the per-(lane, step) field metadata decoded ONCE into registers: a step whose 32/K4 fields are
// all sparse ("pure", warp-uniform) is a load of the packed column, one 64-bit multiply-add and the gather.
template <int K4>
__global__ void __launch_bounds__(256, 2)
feat_forward_pipe_kernel(const b200_feat_layout L, const b200_feat_tables T,
                         const int64_t* __restrict__ users, const int64_t* __restrict__ items,
                         int64_t R, int64_t grid_items, int64_t row_offset, Out o, Head h, int NS) {
  constexpr int K = K4 * 4;
  constexpr int FPW = 32 / K4;
  constexpr int U = 8;                          // steps per batch
  constexpr int MAXF = 2 + 2 * B200_MAX_FIELDS;
  __shared__ int32_t sh_code[MAXF];
  __shared__ int32_t sh_drow[MAXF];
  __shared__ float sh_link[MAXF + 32];
  const int lane = threadIdx.x & 31;
  const int fg = lane / K4, q = lane % K4;
  const int n_id = ((L.id_mask & 1) ? 1 : 0) + ((L.id_mask & 2) ? 1 : 0);
  const int F = n_id + L.n_sparse + L.n_dense;
  const bool want_lin = (o.lin != nullptr) || (o.fm_out != nullptr);
  for (int f = threadIdx.x; f < NS * FPW; f += blockDim.x) {
    if (f >= F) { sh_link[f] = 0.f; continue; }
    int kind, col = 0, drow = 0;
    if (f < n_id) kind = ((L.id_mask & 1) && f == 0) ? 0 : 1;
    else if (f < n_id + L.n_sparse) {
      const int fs = f - n_id;
      kind = L.sparse_side[fs] == 0 ? 2 : 3;
      col = L.sparse_col[fs];
    } else {
      const int fd = f - n_id - L.n_sparse;
      drow = L.dense_embed_row[fd];
      kind = L.dense_side[fd] == 0 ? 5 : 6;
      col = L.dense_col[fd];
    }
    sh_code[f] = kind | (col << 3);
    sh_drow[f] = drow;
    sh_link[f] = want_lin ? h.lin_kernel[f] : 0.f;
  }
  __syncthreads();
  const float* my_link = sh_link + fg;          // + j * FPW per step

  uint32_t colpack[4] = {0u, 0u, 0u, 0u};       // column of (lane, step j) in its side's unique table, 8 bits each
  uint32_t side_mask = 0, pure = 0;
#pragma unroll
  for (int j = 0; j < 2 * U; ++j) {
    const int f = j * FPW + fg;
    bool sparse_f = false;
    if (j < NS && f < F) {
      const int code = sh_code[f];
      const int kind = code & 7, col = code >> 3;
      if (kind == 2 || kind == 3) {
        sparse_f = true;
        colpack[j / 4] |= (uint32_t)col << (8 * (j % 4));
        if (kind == 3) side_mask |= 1u << j;
      }
    }
    if (__all_sync(0xffffffffu, sparse_f)) pure |= 1u << j;
  }
  const float4* tbl_q = reinterpret_cast<const float4*>(T.sparse_embeds) + q;

  auto load_ids = [&](int64_t r, int64_t& u, int64_t& it) {
    u = 0; it = 0;
    if (r < R) {
      if (grid_items > 0) { const int64_t rg = r + row_offset; u = users[rg / grid_items]; it = rg % grid_items; }
      else { u = users[r]; it = items[r]; }
    }
  };
  // index (sparse) / value bits (dense) of the 8 steps [J0, J0 + 8) of the row with ids (u, it)
  auto load_indices = [&](int32_t (&raw)[U], const int J0, int64_t u, int64_t it) {
    const int32_t* pu = L.user_sparse_unique + u * L.ld_us;
    const int32_t* pi = L.item_sparse_unique + it * L.ld_is;
#pragma unroll
    for (int jj = 0; jj < U; ++jj) {
      const int j = J0 + jj;
      raw[jj] = 0;
      if (j >= NS) continue;
      const int col = (colpack[j / 4] >> (8 * (j % 4))) & 255u;
      if ((pure >> j) & 1u) {
        raw[jj] = __ldg((((side_mask >> j) & 1u) ? pi : pu) + col);
      } else {
        const int f = j * FPW + fg;
        if (f < F) {
          const int code = sh_code[f];
          const int kind = code & 7;
          if (kind == 2 || kind == 3) raw[jj] = __ldg((kind == 3 ? pi : pu) + col);
          else if (kind >= 5) {
            const int dcol = code >> 3;
            const float* xp = kind == 5 ? L.user_dense_unique + u * L.ld_ud + dcol : L.item_dense_unique + it * L.ld_id + dcol;
            raw[jj] = __float_as_int(__ldg(xp));
          }
        }
      }
    }
  };

  float4 s, s2;
  float lin_acc;
  float4 e[U];
  float lw[U];
  // phase A: row gathers (+ linear weights) of the steps [J0, J0 + 8) from their indices
  auto gather = [&](const int32_t (&raw)[U], const int J0, int64_t u, int64_t it) {
#pragma unroll
    for (int jj = 0; jj < U; ++jj) {
      const int j = J0 + jj;
      e[jj] = make_float4(0.f, 0.f, 0.f, 0.f);
      lw[jj] = 0.f;
      if (j >= NS) continue;
      if ((pure >> j) & 1u) {
        e[jj] = __ldg(tbl_q + (int64_t)raw[jj] * K4);
        if (want_lin) lw[jj] = __ldg(T.sparse_linear + raw[jj]);
      } else {
        const int f = j * FPW + fg;
        if (f < F) {
          const int kind = sh_code[f] & 7;
          if (kind < 2) {
            e[jj] = __ldg(reinterpret_cast<const float4*>(kind == 0 ? T.user_embeds + u * K : T.item_embeds + it * K) + q);
            if (want_lin) lw[jj] = kind == 0 ? __ldg(T.user_linear + u) : __ldg(T.item_linear + it);
          } else if (kind < 5) {
            e[jj] = __ldg(tbl_q + (int64_t)raw[jj] * K4);
            if (want_lin) lw[jj] = __ldg(T.sparse_linear + raw[jj]);
          } else {
            const int drow = sh_drow[f];
            e[jj] = __ldg(reinterpret_cast<const float4*>(T.dense_embeds + (int64_t)drow * K) + q);
            if (want_lin) lw[jj] = __ldg(T.dense_linear + drow);
          }
        }
      }
    }
  };
  // phase C: sums, linear term, concatenated row
  auto consume = [&](const int32_t (&raw)[U], const int J0, float* crow) {
#pragma unroll
    for (int jj = 0; jj < U; ++jj) {
      const int j = J0 + jj;
      if (j >= NS) continue;
      const bool is_pure = (pure >> j) & 1u;
      const int f = j * FPW + fg;
      if (!is_pure && f >= F) continue;
      float4 v = e[jj];
      float l = lw[jj];
      if (!is_pure && (sh_code[f] & 7) >= 5) {
        const float sc = __int_as_float(raw[jj]);
        v.x *= sc; v.y *= sc; v.z *= sc; v.w *= sc;
        l *= sc;
      }
      if (want_lin) lin_acc = fmaf(l, my_link[j * FPW], lin_acc);
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
      s2.x = fmaf(v.x, v.x, s2.x); s2.y = fmaf(v.y, v.y, s2.y);
      s2.z = fmaf(v.z, v.z, s2.z); s2.w = fmaf(v.w, v.w, s2.w);
      if (crow) *reinterpret_cast<float4*>(crow + j * 128) = v;
    }
  };

  const int64_t n_warps = (int64_t)gridDim.x * (blockDim.x >> 5);
  int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  int64_t u, it, un, itn, un2, itn2;      // ids of the current row, the next one and the one after
  load_ids(r, u, it);
  load_ids(r + n_warps, un, itn);
  load_ids(r + 2 * n_warps, un2, itn2);
  int32_t rawA[U], rawB[U];
  if (r < R) load_indices(rawA, 0, u, it);
  const bool two = NS > U;
  for (; r < R; r += n_warps) {
    const bool has_next = r + n_warps < R;
    s = make_float4(0.f, 0.f, 0.f, 0.f);
    s2 = s;
    lin_acc = 0.f;
    float* crow = o.concat ? o.concat + r * o.ld_concat + lane * 4 : nullptr;   // + j * 128 floats per step
    // ---- batch 0: gathers of steps 0..7 | indices of the next batch | consume
    gather(rawA, 0, u, it);
    if (two) load_indices(rawB, U, u, it);
    else if (has_next) load_indices(rawB, 0, un, itn);
    consume(rawA, 0, crow);
    if (two) {
      // ---- batch 1: gathers of steps 8..15 | indices of the next row's first batch | consume
      gather(rawB, U, u, it);
      if (has_next) load_indices(rawA, 0, un, itn);
      consume(rawB, U, crow);
    } else {
#pragma unroll
      for (int jj = 0; jj < U; ++jj) rawA[jj] = rawB[jj];
    }
    u = un; it = itn; un = un2; itn = itn2;
    load_ids(r + 3 * n_warps, un2, itn2);
    if (!o.pw && !o.fm_out && !o.lin && !o.ssum) continue;
#pragma unroll
    for (int off = K4; off < 32; off <<= 1) {
      s.x += __shfl_xor_sync(0xffffffffu, s.x, off); s.y += __shfl_xor_sync(0xffffffffu, s.y, off);
      s.z += __shfl_xor_sync(0xffffffffu, s.z, off); s.w += __shfl_xor_sync(0xffffffffu, s.w, off);
      s2.x += __shfl_xor_sync(0xffffffffu, s2.x, off); s2.y += __shfl_xor_sync(0xffffffffu, s2.y, off);
      s2.z += __shfl_xor_sync(0xffffffffu, s2.z, off); s2.w += __shfl_xor_sync(0xffffffffu, s2.w, off);
      lin_acc += __shfl_xor_sync(0xffffffffu, lin_acc, off);     // the K4 lanes of a field hold copies
    }
    lin_acc += h.lin_bias;
    const float sv[4] = {s.x, s.y, s.z, s.w};
    const float s2v[4] = {s2.x, s2.y, s2.z, s2.w};
    float head_acc = 0.f;
#pragma unroll
    for (int c = 0; c < 4; ++c) {
      const int kk = q * 4 + c;
      const float pw = 0.5f * (sv[c] * sv[c] - s2v[c]);
      if (fg == 0) {
        if (o.pw) o.pw[r * o.ld_pw + kk] = pw;
        if (o.ssum) { o.ssum[r * o.ld_s + kk] = sv[c]; o.sqsum[r * o.ld_s + kk] = s2v[c]; }
      }
      if (o.fm_out) {
        const float z = h.bn_scale ? fmaf(pw, h.bn_scale[kk], h.bn_shift[kk]) : pw;
        head_acc = fmaf(z, h.pw_kernel[kk], head_acc);
      }
    }
    if (o.fm_out) {
#pragma unroll
      for (int off = 1; off < K4; off <<= 1) head_acc += __shfl_xor_sync(0xffffffffu, head_acc, off);
      head_acc += h.pw_bias;
      if (lane == 0) o.fm_out[r] = lin_acc + (head_acc > 0.f ? head_acc : expm1f(head_acc));
    }
    if (o.lin && lane == 0) o.lin[r] = lin_acc;
  }
}

// ---- large row counts, K in {4, 8, 16, 32}: the field-group layout above with the row gathers staged through
// shared memory by cp.async (LDGSTS, 16 B per lane — the SAME request pattern as the register gather, but the
// landing zone is shared memory instead of registers, so a warp keeps TWO whole rows of gathers in flight and the
// index loads of a third).  ncu of the register kernel (profiles/r02_feat_fieldgroup_ncu.txt): 12 of 18 stall
// cycles per issue are long-scoreboard, issue slots 33 % busy, DRAM 18 % — latency bound on the dependent chain
// ids -> feature index -> embedding row.  Pipeline per warp, rows k = 0, 1, ...:
//     iteration k:  G(k+1) address generation from the indices loaded one iteration ago + cp.async of every field
//                   I(k+2) index loads into registers          (ids of row k+3 prefetched)
//                   wait for the copies of row k, consume them from shared memory (every lane reads back exactly
//                   the 16 bytes it copied itself: no cross-lane hand-off), sums, concat store, row outputs
// One UBLKCP bulk copy per 64-byte row was measured 5.7x slower than register gathers (feat_tma.cu): the bulk-copy
// engine is the wrong tool for rows this small; LDGSTS keeps the LSU's 8-rows-per-instruction coalescing.
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* gsrc) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 16;" ::"r"(d), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

constexpr int ASYNC_MAXS = 16;   // steps (warp-level gathers) per row the staged kernel holds in registers

__device__ __forceinline__ void cp_async4(void* smem_dst, const void* gsrc) {
  const uint32_t d = (uint32_t)__cvta_generic_to_shared(smem_dst);
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gsrc) : "memory");
}

template <int K4>
__global__ void __launch_bounds__(256, 2)
feat_forward_async_kernel(const b200_feat_layout L, const b200_feat_tables T,
                          const int64_t* __restrict__ users, const int64_t* __restrict__ items,
                          int64_t R, int64_t grid_items, int64_t row_offset, Out o, Head h, int NS) {
  constexpr int K = K4 * 4;
  constexpr int FPW = 32 / K4;
  constexpr int MAXS = ASYNC_MAXS;
  extern __shared__ float4 dyn_smem[];
  const int wpb = blockDim.x >> 5;
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int fg = lane / K4, q = lane % K4;
  const int n_id = ((L.id_mask & 1) ? 1 : 0) + ((L.id_mask & 2) ? 1 : 0);
  const int F = n_id + L.n_sparse + L.n_dense;
  const bool want_lin = (o.lin != nullptr) || (o.fm_out != nullptr);
  // dynamic shared memory: [wpb][2][NS][32] float4 rings | [wpb][2][NS*FPW] scales | [wpb][2][NS*FPW] linear
  // weights | code[F] | drow[F] | link[NS*FPW]
  float4* ring = dyn_smem + (size_t)wib * 2 * NS * 32 + lane;          // this lane's 16-byte column of the ring
  float* aux = reinterpret_cast<float*>(dyn_smem + (size_t)wpb * 2 * NS * 32);
  float* sx = aux + (size_t)wib * 2 * NS * FPW + fg;                   // this lane's field column
  float* slw = aux + (size_t)(wpb + wib) * 2 * NS * FPW + fg;
  int32_t* sh_code = reinterpret_cast<int32_t*>(aux + (size_t)2 * wpb * 2 * NS * FPW);
  int32_t* sh_drow = sh_code + F;
  float* sh_link = reinterpret_cast<float*>(sh_drow + F);              // [NS * FPW], 0 past F
  for (int f = threadIdx.x; f < NS * FPW; f += blockDim.x) {
    if (f >= F) { sh_link[f] = 0.f; continue; }
    int kind, col = 0, drow = 0;
    if (f < n_id) kind = ((L.id_mask & 1) && f == 0) ? 0 : 1;
    else if (f < n_id + L.n_sparse) {
      const int fs = f - n_id;
      kind = L.sparse_side[fs] == 0 ? 2 : 3;
      col = L.sparse_col[fs];
    } else {
      const int fd = f - n_id - L.n_sparse;
      drow = L.dense_embed_row[fd];
      kind = L.dense_side[fd] == 0 ? 5 : 6;
      col = L.dense_col[fd];
    }
    sh_code[f] = kind | (col << 3);
    sh_drow[f] = drow;
    sh_link[f] = want_lin ? h.lin_kernel[f] : 0.f;
  }
  __syncthreads();
  const float* my_link = sh_link + fg;                                 // + j * FPW per step

  // ---- per-lane step descriptors (the field of (lane, step j) is the same for every row): a step whose 32/K4
  // fields are ALL sparse ("pure", warp-uniform) needs only its column in the side's unique table (8 bits,
  // packed four to a register) and one side bit; mixed steps (ids, dense fields, the ragged last step) take the
  // generic path through the shared-memory metadata.
  uint32_t colpack[MAXS / 4];
  uint32_t side_mask = 0, pure = 0;
#pragma unroll
  for (int j = 0; j < MAXS / 4; ++j) colpack[j] = 0;
#pragma unroll
  for (int j = 0; j < MAXS; ++j) {
    const int f = j * FPW + fg;
    bool sparse_f = false;
    if (j < NS && f < F) {
      const int code = sh_code[f];
      const int kind = code & 7, col = code >> 3;
      if (kind == 2 || kind == 3) {
        sparse_f = true;
        colpack[j / 4] |= (uint32_t)col << (8 * (j % 4));
        if (kind == 3) side_mask |= 1u << j;
      }
    }
    if (__all_sync(0xffffffffu, sparse_f)) pure |= 1u << j;
  }
  const float* tbl_q = T.sparse_embeds + q * 4;

  const int64_t n_warps = (int64_t)gridDim.x * wpb;
  const int64_t w0 = (int64_t)blockIdx.x * wpb + wib;
  auto load_ids = [&](int64_t r, int64_t& u, int64_t& it) {
    u = 0; it = 0;
    if (r < R) {
      if (grid_items > 0) { const int64_t rg = r + row_offset; u = users[rg / grid_items]; it = rg % grid_items; }
      else { u = users[r]; it = items[r]; }
    }
  };
  int32_t raw[MAXS];
  // I: feature index (sparse) / value bits (dense) of every step of a row with ids (u, it)
  auto load_indices = [&](int64_t u, int64_t it) {
    const int32_t* pu = L.user_sparse_unique + u * L.ld_us;
    const int32_t* pi = L.item_sparse_unique + it * L.ld_is;
#pragma unroll
    for (int j = 0; j < MAXS; ++j) {
      if (j >= NS) continue;
      const int col = (colpack[j / 4] >> (8 * (j % 4))) & 255u;
      if ((pure >> j) & 1u) {
        raw[j] = __ldg((((side_mask >> j) & 1u) ? pi : pu) + col);
      } else {
        raw[j] = 0;
        const int f = j * FPW + fg;
        if (f < F) {
          const int code = sh_code[f];
          const int kind = code & 7;
          if (kind == 2 || kind == 3) raw[j] = __ldg((kind == 3 ? pi : pu) + col);
          else if (kind >= 5) {
            const int dcol = code >> 3;
            const float* xp = kind == 5 ? L.user_dense_unique + u * L.ld_ud + dcol : L.item_dense_unique + it * L.ld_id + dcol;
            raw[j] = __float_as_int(__ldg(xp));
          }
        }
      }
    }
  };

  int64_t ua, ita, ub, itb, uc, itc;       // ids of rows k+1, k+2, k+3
  load_ids(w0, ua, ita);
  load_ids(w0 + n_warps, ub, itb);
  load_ids(w0 + 2 * n_warps, uc, itc);
  if (w0 < R) load_indices(ua, ita);
  for (int64_t k = -1;; ++k) {
    const int64_t r_cur = w0 + k * n_warps, r_nx = r_cur + n_warps, r_nx2 = r_nx + n_warps;
    if (k >= 0 && r_cur >= R) break;
    __syncwarp();
    const int nb = (int)((k + 1) & 1);
    // ---- G(k+1): addresses from raw[], asynchronous copies (rows AND linear weights) into buffer nb
    if (r_nx < R) {
      float4* dst = ring + (size_t)nb * NS * 32;
      float* dlw = slw + (size_t)nb * NS * FPW;
      float* dsx = sx + (size_t)nb * NS * FPW;
#pragma unroll
      for (int j = 0; j < MAXS; ++j) {
        if (j >= NS) continue;
        if ((pure >> j) & 1u) {
          cp_async16(dst + j * 32, tbl_q + (int64_t)raw[j] * K);
          if (want_lin && q == 0) cp_async4(dlw + j * FPW, T.sparse_linear + raw[j]);
        } else {
          const int f = j * FPW + fg;
          if (f < F) {
            const int kind = sh_code[f] & 7;
            const float* rowp;
            float scale = 1.f;
            if (kind < 2) {
              rowp = kind == 0 ? T.user_embeds + ua * K : T.item_embeds + ita * K;
              if (want_lin && q == 0) cp_async4(dlw + j * FPW, kind == 0 ? T.user_linear + ua : T.item_linear + ita);
            } else if (kind < 5) {
              rowp = T.sparse_embeds + (int64_t)raw[j] * K;
              if (want_lin && q == 0) cp_async4(dlw + j * FPW, T.sparse_linear + raw[j]);
            } else {
              const int drow = sh_drow[f];
              scale = __int_as_float(raw[j]);
              rowp = T.dense_embeds + (int64_t)drow * K;
              if (want_lin && q == 0) dlw[j * FPW] = __ldg(T.dense_linear + drow) * scale;
            }
            cp_async16(dst + j * 32, rowp + q * 4);
            if (q == 0) dsx[j * FPW] = scale;
          }
        }
      }
    }
    cp_async_commit();
    // ---- I(k+2) and the ids of row k+3
    if (r_nx2 < R) load_indices(ub, itb);
    ua = ub; ita = itb; ub = uc; itb = itc;
    load_ids(r_nx2 + 2 * n_warps, uc, itc);
    // ---- row k has landed (everything but the newest group)
    cp_async_wait<1>();
    if (k >= 0) {
      __syncwarp();          // scales / linear weights of the quad's lane 0 are read by all its lanes
      const int cb = (int)(k & 1);
      const int64_t r = r_cur;
      const float4* src = ring + (size_t)cb * NS * 32;
      const float* csx = sx + (size_t)cb * NS * FPW;
      const float* clw = slw + (size_t)cb * NS * FPW;
      float* crow = o.concat ? o.concat + r * o.ld_concat + lane * 4 : nullptr;   // + j * 128 floats per step
      float4 s = make_float4(0.f, 0.f, 0.f, 0.f), s2 = s;
      float lin_acc = 0.f;
#pragma unroll
      for (int j = 0; j < MAXS; ++j) {
        if (j >= NS) continue;
        const bool is_pure = (pure >> j) & 1u;
        if (!is_pure && j * FPW + fg >= F) continue;
        float4 v = src[j * 32];
        if (!is_pure) {
          const float sc = csx[j * FPW];
          v.x *= sc; v.y *= sc; v.z *= sc; v.w *= sc;
        }
        if (want_lin) lin_acc = fmaf(clw[j * FPW], my_link[j * FPW], lin_acc);   // same value in the K4 lanes of a field
        s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
        s2.x = fmaf(v.x, v.x, s2.x); s2.y = fmaf(v.y, v.y, s2.y);
        s2.z = fmaf(v.z, v.z, s2.z); s2.w = fmaf(v.w, v.w, s2.w);
        if (crow) *reinterpret_cast<float4*>(crow + j * 128) = v;
      }
      if (o.pw || o.fm_out || o.lin || o.ssum) {
#pragma unroll
        for (int off = K4; off < 32; off <<= 1) {
          s.x += __shfl_xor_sync(0xffffffffu, s.x, off); s.y += __shfl_xor_sync(0xffffffffu, s.y, off);
          s.z += __shfl_xor_sync(0xffffffffu, s.z, off); s.w += __shfl_xor_sync(0xffffffffu, s.w, off);
          s2.x += __shfl_xor_sync(0xffffffffu, s2.x, off); s2.y += __shfl_xor_sync(0xffffffffu, s2.y, off);
          s2.z += __shfl_xor_sync(0xffffffffu, s2.z, off); s2.w += __shfl_xor_sync(0xffffffffu, s2.w, off);
          lin_acc += __shfl_xor_sync(0xffffffffu, lin_acc, off);       // over the field groups (q lanes hold copies)
        }
        lin_acc += h.lin_bias;
        const float sv[4] = {s.x, s.y, s.z, s.w};
        const float s2v[4] = {s2.x, s2.y, s2.z, s2.w};
        float head_acc = 0.f;
#pragma unroll
        for (int c = 0; c < 4; ++c) {
          const int kk = q * 4 + c;
          const float pw = 0.5f * (sv[c] * sv[c] - s2v[c]);
          if (fg == 0) {
            if (o.pw) o.pw[r * o.ld_pw + kk] = pw;
            if (o.ssum) { o.ssum[r * o.ld_s + kk] = sv[c]; o.sqsum[r * o.ld_s + kk] = s2v[c]; }
          }
          if (o.fm_out) {
            const float z = h.bn_scale ? fmaf(pw, h.bn_scale[kk], h.bn_shift[kk]) : pw;
            head_acc = fmaf(z, h.pw_kernel[kk], head_acc);
          }
        }
        if (o.fm_out) {
#pragma unroll
          for (int off = 1; off < K4; off <<= 1) head_acc += __shfl_xor_sync(0xffffffffu, head_acc, off);
          head_acc += h.pw_bias;
          if (lane == 0) o.fm_out[r] = lin_acc + (head_acc > 0.f ? head_acc : expm1f(head_acc));
        }
        if (o.lin && lane == 0) o.lin[r] = lin_acc;
      }
    }
    if (r_nx >= R) { cp_async_wait<0>(); break; }
  }
}

// y[r, n] = act(sum_k x[r,k] * Wt[n,k] + b[n]) — 64x64x16 register-tiled SIMT GEMM (fp32, exact fma chain);
// act: 0 none, 1 relu, 2 swish (apply_act)
constexpr int LM = 64, LN = 64, LK = 16;
__global__ void __launch_bounds__(256)
linear_f32_kernel(const float* __restrict__ X, int64_t ldx, int64_t R, const float* __restrict__ Wt,
                  int64_t ldw, const float* __restrict__ bias, int din, int dout, int act,
                  float* __restrict__ Y, int64_t ldy) {
  __shared__ float Xs[LK][LM + 4];
  __shared__ float Ws[LK][LN + 4];
  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  const int64_t m0 = (int64_t)blockIdx.y * LM;
  const int n0 = blockIdx.x * LN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  const int lrow = tid >> 2, lk = (tid & 3) * 4;   // 64 rows x 16 k, 4 consecutive k per thread
  for (int k0 = 0; k0 < din; k0 += LK) {
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int k = k0 + lk + q;
      float a = 0.f, b = 0.f;
      if (k < din) {
        if (m0 + lrow < R) a = __ldg(X + (m0 + lrow) * ldx + k);
        if (n0 + lrow < dout) b = __ldg(Wt + (int64_t)(n0 + lrow) * ldw + k);
      }
      Xs[lk + q][lrow] = a;
      Ws[lk + q][lrow] = b;
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < LK; ++k) {
      float a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = Xs[k][ty + 16 * i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = Ws[k][tx + 16 * j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t r = m0 + ty + 16 * i;
    if (r >= R) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx + 16 * j;
      if (n < dout) {
        float v = acc[i][j] + (bias ? bias[n] : 0.f);
        Y[r * ldy + n] = apply_act(v, act);
      }
    }
  }
}

// out[r] = b + sum over up to 3 row-blocks of <block[r,:], w_block>  (the Dense(1) on a concat)
__global__ void concat_dense_kernel(const float* __restrict__ a, int64_t lda, int na,
                                    const float* __restrict__ b, int64_t ldb, int nb,
                                    const float* __restrict__ c, int64_t ldc, int nc,
                                    const float* __restrict__ w, float bias, int64_t R,
                                    float* __restrict__ out) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  float acc = 0.f;
  for (int k = lane; k < na; k += 32) acc = fmaf(a[r * lda + k], w[k], acc);
  for (int k = lane; k < nb; k += 32) acc = fmaf(b[r * ldb + k], w[na + k], acc);
  for (int k = lane; k < nc; k += 32) acc = fmaf(c[r * ldc + k], w[na + nb + k], acc);
  acc = warp_sum(acc);
  if (lane == 0) out[r] = acc + bias;
}

// row-wise L2 normalisation (libreco/layers/normalization.py:32-44, tf.linalg.l2_normalize)
__global__ void l2_normalize_kernel(float* __restrict__ x, int64_t ld, int64_t R, int d) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  float ss = 0.f;
  for (int k = lane; k < d; k += 32) { const float v = x[r * ld + k]; ss = fmaf(v, v, ss); }
  ss = warp_sum(ss);
  const float inv = rsqrtf(fmaxf(ss, 1e-12f));
  for (int k = lane; k < d; k += 32) x[r * ld + k] *= inv;
}

}  // namespace feat
}  // namespace b200

using namespace b200;
using namespace b200::feat;

static int g_feat_kernel = 0;   // b200_feat_forward_tune bit 1: 0 = field-group kernel (default), 1 = lane-per-field kernel (A/B)
static int g_feat_no_async = 0; // b200_feat_forward_tune bit 2: 1 = neither the pipelined nor the cp.async staged kernel (A/B)
static int g_feat_async = 0;    // bit 3: 1 = the cp.async staged kernel instead of the software-pipelined register kernel
static int g_feat_tma = 0;   // b200_feat_forward_tune: 1 = bulk-copy (TMA) staged kernel where eligible, 0 = register kernels
                             // (default: one UBLKCP per 64-byte row measured 5.7x SLOWER than the register gather, profiles/)

extern "C" int b200_feat_forward_tune(int32_t use_tma_staging) {
  g_feat_tma = (use_tma_staging & 1) ? 1 : 0;
  g_feat_kernel = (use_tma_staging & 2) ? 1 : 0;
  g_feat_no_async = (use_tma_staging & 4) ? 1 : 0;
  g_feat_async = (use_tma_staging & 8) ? 1 : 0;
  return 0;
}

extern "C" int b200_feat_forward(const b200_feat_layout* L, const b200_feat_tables* T,
                                 const int64_t* users, const int64_t* items, int64_t R,
                                 int64_t grid_items, int64_t row_offset, float* concat, int64_t ld_concat, float* pw,
                                 int64_t ld_pw, float* lin, float* fm_out, const float* lin_kernel,
                                 float lin_bias, const float* bn_scale, const float* bn_shift,
                                 const float* pw_kernel, float pw_bias, float* ssum, float* sqsum,
                                 int64_t ld_s, void* stream) {
  // an empty batch may come with null id arrays (an empty torch tensor has no storage)
  B200_REQUIRE(L && T && (users || R == 0), "b200_feat_forward: null pointer");
  B200_REQUIRE(grid_items > 0 || items || R == 0, "b200_feat_forward: item ids missing");
  B200_REQUIRE(L->embed_size >= 1 && L->embed_size <= 32 * MAX_T, "embed size %d outside [1, %d]",
               L->embed_size, 32 * MAX_T);
  B200_REQUIRE(L->n_sparse <= B200_MAX_FIELDS && L->n_dense <= B200_MAX_FIELDS, "too many feature fields");
  B200_REQUIRE((lin == nullptr && fm_out == nullptr) || lin_kernel, "linear head weights missing");
  B200_REQUIRE(fm_out == nullptr || pw_kernel, "FM head weights missing");
  if (R == 0) return 0;
  int lpr = 1;
  while (lpr < L->embed_size && lpr < 32) lpr <<= 1;
  const int Tn = (L->embed_size + lpr - 1) / lpr;
  Out o; o.concat = concat; o.ld_concat = ld_concat; o.pw = pw; o.ld_pw = ld_pw; o.lin = lin; o.fm_out = fm_out;
  o.ssum = ssum; o.sqsum = sqsum; o.ld_s = ld_s;
  B200_REQUIRE((ssum == nullptr) == (sqsum == nullptr), "b200_feat_forward: ssum and sqsum go together");
  Head h; h.lin_kernel = lin_kernel; h.lin_bias = lin_bias; h.bn_scale = bn_scale; h.bn_shift = bn_shift;
  h.pw_kernel = pw_kernel; h.pw_bias = pw_bias;
  auto al16 = [](const void* p) { return p == nullptr || (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  const int K = L->embed_size;
  const bool fast = K % 4 == 0 && K <= 32 && al16(T->user_embeds) && al16(T->item_embeds) &&
                    al16(T->sparse_embeds) && al16(T->dense_embeds) && al16(concat) && (ld_concat % 4 == 0);
  if (fast && g_feat_tma) {
    // large row counts: TMA-staged persistent kernel (many more row reads in flight per SM)
    const int rc = launch_feat_forward_tma(L, T, users, items, R, grid_items, row_offset, concat, ld_concat, pw, ld_pw,
                                           lin, fm_out, lin_kernel, lin_bias, bn_scale, bn_shift, pw_kernel, pw_bias,
                                           ssum, sqsum, ld_s, (cudaStream_t)stream);
    if (rc < 0) return rc;
    if (rc == 1) return 0;
  }
  const int K4v = K / 4;
  const bool group_ok = fast && g_feat_kernel == 0 && (K4v == 1 || K4v == 2 || K4v == 4 || K4v == 8);
  const bool staged_ok = group_ok && !g_feat_no_async && R >= 4096 && !L->sparse_rows && !L->dense_rows;
  if (staged_ok && !g_feat_async) {
    // software-pipelined register gather (default for large row counts)
    const int FPW = 32 / K4v;
    const int n_id = ((L->id_mask & 1) ? 1 : 0) + ((L->id_mask & 2) ? 1 : 0);
    const int NS = (n_id + L->n_sparse + L->n_dense + FPW - 1) / FPW;
    if (NS <= 16) {
      const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div64(R, 8), (int64_t)std::max(1, num_sms()) * 2);
      cudaStream_t st = (cudaStream_t)stream;
      switch (K4v) {
        case 1: feat_forward_pipe_kernel<1><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h, NS); break;
        case 2: feat_forward_pipe_kernel<2><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h, NS); break;
        case 4: feat_forward_pipe_kernel<4><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h, NS); break;
        default: feat_forward_pipe_kernel<8><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h, NS); break;
      }
      count_launch();
      B200_CUDA_OK(cudaGetLastError());
      return 0;
    }
  }
  if (staged_ok && g_feat_async) {
    // cp.async staged kernel: two rows of gathers in flight per warp; warps per CTA and CTAs per SM chosen so
    // that the rings fill the SM's shared memory
    const int FPW = 32 / K4v;
    const int n_id = ((L->id_mask & 1) ? 1 : 0) + ((L->id_mask & 2) ? 1 : 0);
    const int F = n_id + L->n_sparse + L->n_dense;
    const int NS = (F + FPW - 1) / FPW;
    if (NS <= ASYNC_MAXS) {
      const size_t per_warp = (size_t)2 * NS * 512 + (size_t)2 * 2 * NS * FPW * 4;   // rings + scales + linear weights
      const size_t meta = (size_t)F * 8 + (size_t)NS * FPW * 4;
      int best_w = 0, best_wpb = 0, best_nb = 0;
      for (int wpb = 8; wpb >= 2; --wpb) {
        const size_t per_block = wpb * per_warp + meta + 1024;
        int nb = (int)((size_t)(228 * 1024) / per_block);
        nb = std::min(nb, 16 / wpb);             // ~126 registers per thread: 16 warps per SM
        if (nb * wpb > best_w) { best_w = nb * wpb; best_wpb = wpb; best_nb = nb; }
      }
      if (best_w >= 8) {
        const size_t dyn = best_wpb * per_warp + meta;
        const int64_t blocks_needed = ceil_div64(R, best_wpb);
        const unsigned blocks = (unsigned)std::min<int64_t>(blocks_needed, (int64_t)std::max(1, num_sms()) * best_nb);
        cudaStream_t st = (cudaStream_t)stream;
        auto launch = [&](auto kern) -> int {
          B200_CUDA_OK(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)dyn));
          kern<<<blocks, best_wpb * 32, dyn, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h, NS);
          return 0;
        };
        int rc;
        switch (K4v) {
          case 1: rc = launch(feat_forward_async_kernel<1>); break;
          case 2: rc = launch(feat_forward_async_kernel<2>); break;
          case 4: rc = launch(feat_forward_async_kernel<4>); break;
          default: rc = launch(feat_forward_async_kernel<8>); break;
        }
        if (rc) return rc;
        count_launch();
        B200_CUDA_OK(cudaGetLastError());
        return 0;
      }
    }
  }
  if (group_ok) {
    // field-group kernel: persistent over rows (the per-block metadata staging is paid once per CTA)
    const unsigned blocks = (unsigned)std::min<int64_t>(ceil_div64(R, 8), (int64_t)std::max(1, num_sms()) * 3);
    cudaStream_t st = (cudaStream_t)stream;
    switch (K4v) {
      case 1: feat_forward_fieldgroup_kernel<1><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h); break;
      case 2: feat_forward_fieldgroup_kernel<2><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h); break;
      case 4: feat_forward_fieldgroup_kernel<4><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h); break;
      default: feat_forward_fieldgroup_kernel<8><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h); break;
    }
  } else if (fast) {
    const unsigned blocks = (unsigned)ceil_div64(R * 32, 256);
    cudaStream_t st = (cudaStream_t)stream;
    switch (K / 4) {
      case 1: feat_forward_lanefield_kernel<1><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h); break;
      case 2: feat_forward_lanefield_kernel<2><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h); break;
      case 3: feat_forward_lanefield_kernel<3><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h); break;
      case 4: feat_forward_lanefield_kernel<4><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h); break;
      case 5: feat_forward_lanefield_kernel<5><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h); break;
      case 6: feat_forward_lanefield_kernel<6><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h); break;
      case 7: feat_forward_lanefield_kernel<7><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h); break;
      default: feat_forward_lanefield_kernel<8><<<blocks, 256, 0, st>>>(*L, *T, users, items, R, grid_items, row_offset, o, h); break;
    }
  } else {
    const int64_t warps = ceil_div64(R, 32 / lpr);
    feat_forward_kernel<<<(unsigned)ceil_div64(warps * 32, 256), 256, 0, (cudaStream_t)stream>>>(
        *L, *T, users, items, R, grid_items, row_offset, o, h, lpr, Tn);
  }
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

// multi_sparse_alone (reference libreco/tfops/features.py:87-118): one warp per row, lanes over K
__global__ void multi_sparse_combine_kernel(const float* __restrict__ table, int64_t ld, int K,
                                            const int32_t* __restrict__ idx, int64_t ld_idx, int len, int64_t n,
                                            int32_t oov, int combiner, float* __restrict__ out, int64_t ld_out) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  int cnt = 0;
  for (int t = 0; t < len; ++t) cnt += (idx[r * ld_idx + t] != oov);
  float div = 1.f;
  if (combiner == 1) div = (float)cnt;
  else if (combiner == 2) div = sqrtf((float)cnt);
  for (int k = lane; k < K; k += 32) {
    float acc = 0.f;
    for (int t = 0; t < len; ++t) {
      const int32_t ix = idx[r * ld_idx + t];
      if (ix != oov) acc += __ldg(table + (int64_t)ix * ld + k);   // oov row counts as the zero vector
    }
    out[r * ld_out + k] = (combiner == 0) ? acc : (div != 0.f ? acc / div : 0.f);   // div_no_nan
  }
}

extern "C" int b200_multi_sparse_combine(const float* table, int64_t ld, int32_t K, const int32_t* idx,
                                         int64_t ld_idx, int32_t len, int64_t n, int32_t oov,
                                         int32_t combiner, float* out, int64_t ld_out, void* stream) {
  B200_REQUIRE(table && idx && out, "b200_multi_sparse_combine: null pointer");
  B200_REQUIRE(combiner >= 0 && combiner <= 2, "combiner must be 0 (sum), 1 (mean) or 2 (sqrtn)");
  B200_REQUIRE(K >= 1 && len >= 1, "bad shape");
  if (n == 0) return 0;
  multi_sparse_combine_kernel<<<(unsigned)ceil_div64(n * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      table, ld, K, idx, ld_idx, len, n, oov, combiner, out, ld_out);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

// plain row gather / scatter-add for row-sharded tables (SURVEY.md 8e row 2): one sub-warp per row
__global__ void gather_rows_kernel(const float* __restrict__ table, int64_t ld, int d, const int64_t* __restrict__ idx,
                                   int64_t n, float* __restrict__ out, int64_t ld_out) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  const float* src = table + idx[r] * ld;
  for (int k = lane; k < d; k += 32) out[r * ld_out + k] = __ldg(src + k);
}

__global__ void scatter_add_rows_kernel(float* __restrict__ table, int64_t ld, int d, const int64_t* __restrict__ idx,
                                        int64_t n, const float* __restrict__ rows, int64_t ld_rows) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= n) return;
  float* dst = table + idx[r] * ld;
  for (int k = lane; k < d; k += 32) atomicAdd(dst + k, rows[r * ld_rows + k]);
}

extern "C" int b200_gather_rows(const float* table, int64_t ld, int32_t d, const int64_t* idx, int64_t n,
                                float* out, int64_t ld_out, void* stream) {
  if (n == 0) return 0;      // empty requests carry null pointers (a rank that asked for nothing)
  B200_REQUIRE(table && idx && out && d > 0, "b200_gather_rows: bad arguments");
  gather_rows_kernel<<<(unsigned)ceil_div64(n * 32, 256), 256, 0, (cudaStream_t)stream>>>(table, ld, d, idx, n, out, ld_out);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_scatter_add_rows(float* table, int64_t ld, int32_t d, const int64_t* idx, int64_t n,
                                     const float* rows, int64_t ld_rows, void* stream) {
  if (n == 0) return 0;
  B200_REQUIRE(table && idx && rows && d > 0, "b200_scatter_add_rows: bad arguments");
  scatter_add_rows_kernel<<<(unsigned)ceil_div64(n * 32, 256), 256, 0, (cudaStream_t)stream>>>(table, ld, d, idx, n, rows,
                                                                                           ld_rows);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_linear_f32(const float* X, int64_t ldx, int64_t R, const float* Wt, int64_t ldw,
                               const float* bias, int32_t din, int32_t dout, int32_t act, float* Y,
                               int64_t ldy, void* stream) {
  B200_REQUIRE(X && Wt && Y, "b200_linear_f32: null pointer");
  B200_REQUIRE(act >= 0 && act <= 2, "b200_linear_f32: activation code %d outside [0, 2]", act);
  B200_REQUIRE(R >= 0 && din > 0 && dout > 0, "b200_linear_f32: bad shape (R %lld, din %d, dout %d)", (long long)R,
               din, dout);
  // ldy < dout would overlap output rows; ldx / ldw < din would read the next row's elements
  B200_REQUIRE(ldx >= din && ldw >= din && ldy >= dout, "b200_linear_f32: leading dimension too small");
  if (R == 0) return 0;
  const int64_t gy = ceil_div64(R, LM);
  B200_REQUIRE(gy <= 65535 * 32ll, "b200_linear_f32: too many rows");
  // grid.y limit: process in slabs of 65535 row tiles
  for (int64_t y0 = 0; y0 < gy; y0 += 65535) {
    const int64_t ny = min((int64_t)65535, gy - y0);
    const int64_t r0 = y0 * LM;
    dim3 grid((unsigned)ceil_div64(dout, LN), (unsigned)ny);
    linear_f32_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(X + r0 * ldx, ldx, R - r0, Wt, ldw, bias, din,
                                                              dout, act, Y + r0 * ldy, ldy);
    count_launch();
  }
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_concat_dense(const float* a, int64_t lda, int32_t na, const float* b, int64_t ldb,
                                 int32_t nb, const float* c, int64_t ldc, int32_t nc, const float* w,
                                 float bias, int64_t R, float* out, void* stream) {
  B200_REQUIRE(w && out && (na == 0 || a) && (nb == 0 || b) && (nc == 0 || c), "b200_concat_dense: null pointer");
  if (R == 0) return 0;
  concat_dense_kernel<<<(unsigned)ceil_div64(R * 32, 256), 256, 0, (cudaStream_t)stream>>>(
      a, lda, na, b, ldb, nb, c, ldc, nc, w, bias, R, out);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}

extern "C" int b200_l2_normalize_rows(float* x, int64_t ld, int64_t R, int32_t d, void* stream) {
  B200_REQUIRE(x, "b200_l2_normalize_rows: null pointer");
  if (R == 0) return 0;
  l2_normalize_kernel<<<(unsigned)ceil_div64(R * 32, 256), 256, 0, (cudaStream_t)stream>>>(x, ld, R, d);
  count_launch();
  B200_CUDA_OK(cudaGetLastError());
  return 0;
}
