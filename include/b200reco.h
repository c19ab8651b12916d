/*
 * b200reco.h — C-ABI of librecommender_b200 (sm_90a only).
 *
 * The reference (massquantity/LibRecommender @ 7463d9d) has no FFI on this path:
 * its seams are Python callables (SURVEY.md §8b).  Each entry point below names
 * the reference function whose arithmetic it replaces; the Python shims in
 * librecommender_b200/ keep the reference signatures and call these through
 * ctypes.  Conventions:
 *   - every function returns 0 on success, <0 on error; b200_last_error() gives
 *     the message for the calling thread;
 *   - pointers are DEVICE pointers unless the name ends in _host / says host;
 *   - no ownership transfer: all buffers (incl. workspaces sized by the
 *     *_workspace_bytes queries) are allocated by the caller;
 *   - stream-ordered on `stream` (a cudaStream_t passed as void*), re-entrant,
 *     no global state except the launch counter.
 */
#ifndef B200RECO_H_
#define B200RECO_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200RECO_VERSION 100

int b200_version(void);
const char* b200_last_error(void);
/* number of kernels this library has launched in this process (bench.py: gpu_launches) */
unsigned long long b200_launch_count(void);

/* ---- a0: user_consumed -> CSR ---------------------------------------------------------
 * Replaces recfarm.build_consumed_unique (rust/src/utils.rs:8-35) as used by
 * libreco/data/consumed.py:7-19: interactions are grouped per user in arrival order and
 * CONSECUTIVE repeats are dropped.  HOST function (all pointers host).
 * indptr_host[n_users+1], idx_host capacity n; *nnz_host receives the kept count. */
int b200_build_consumed_csr_host(const int64_t* user_indices_host, const int64_t* item_indices_host,
                                 int64_t n, int64_t n_users, int64_t* indptr_host,
                                 int32_t* idx_host, int64_t* nnz_host);

/* ---- a2: rank_recommendations (libreco/recommendation/ranking.py:10-78) ----------------
 * b200_mask_consumed: filter_items (:59-61) under the rule of :38 — row r (user user_ids[r])
 * is masked iff c_u > 0 and K + c_u <= N, c_u = indptr[u+1]-indptr[u] (duplicates counted);
 * users >= n_users (OOV) are never masked; ids outside [0, N) are skipped.  Masked scores are
 * overwritten with the REMOVED bit pattern 0xffffffff (a NaN no arithmetic produces), which
 * b200_topk_rows ranks below every score, -inf and NaN included. */
int b200_mask_consumed(float* scores, int64_t ld, const int64_t* user_ids, int64_t B, int64_t N,
                       int32_t K, const int64_t* indptr, const int32_t* idx, int64_t n_users,
                       void* stream);

/* b200_topk_rows: partition_select + argsort (:48-49,:76-78): per row the K largest scores,
 * sorted by (score desc, item id asc) where -0.0 == +0.0, every NaN ranks above +inf and REMOVED
 * below -inf.  out_ids int64 [B,K]; out_scores float [B,K] or NULL: the selected scores, with
 * -0.0 written as +0.0 and a NaN as 0x7fffffff.  K <= 4096 and K <= N. */
int b200_topk_rows_workspace_bytes(int64_t B, int64_t N, int32_t K, size_t* bytes);
int b200_topk_rows(const float* scores, int64_t ld, int64_t B, int64_t N, int32_t K,
                   int64_t* out_ids, float* out_scores, void* workspace, size_t workspace_bytes,
                   void* stream);

/* ---- a1: recommend_from_embedding (libreco/recommendation/recommend.py:57-78) ----------
 * scores[r, n] = sum_k U[user_ids[r], k] * I[n, k], fp32, one accumulator per output,
 * fused-multiply-add in increasing k (the library's exact-score definition). */
int b200_score_rows_f32(const float* U, int64_t ldu, const int64_t* user_ids, int64_t B,
                        const float* I, int64_t ldi, int64_t N, int32_t d, float* scores,
                        int64_t lds, void* stream);

/* ---- a1+a2 fused: recommend_from_embedding + rank_recommendations on the tensor cores -----
 * (recommend.py:57-78 + ranking.py:10-78, never materialising [B,N]).
 * catalog: device buffer prepared ONCE per item table (fp16 K-major copy scaled by a power of two
 * so that the largest row norm lies in [64, 128), + that norm).
 * Result per row: the K best non-consumed items by EXACT fp32 score (same definition as
 * b200_score_rows_f32), sorted (score desc, id asc).  row_status[r] (device int32[B]) = 1 marks a
 * row the fused path could not prove exact (failed threshold speculation, too many near-ties, or a
 * heavy user whose capped candidate budget did not suffice): its out_ids are -1 and the caller
 * re-runs it through b200_score_rows_f32 + b200_mask_consumed + b200_topk_rows.
 * row_status codes: 1 sweep list overflow, 2 too few collected, 3 failed speculation, 4 candidate
 * set outside [K, 2048], 5 capped row not provable.
 * Limits: d <= 256, K <= 288.
 * b200_recommend_embed_plan reports how a call of that shape will run: out[0] = 1 when the
 * speculative pre-pass (sweep<PRE> + guess_kernel) is used, out[1] item splits, out[2] item tiles
 * per split, out[3] user tiles, out[4] sampled tiles per split, out[5] TMA stages, out[6] = 10 x CTAs
 * per cluster (2: every item tile is fetched from L2 once per pair of user tiles and TMA-multicast to
 * both CTAs) + MMA groups per item tile, out[7] records per candidate list (n_out >= 8).
 * b200_recommend_embed_tune (process-wide, not thread-safe; 0 keeps a value): organisation code =
 * 100 x cluster size (1|2) + 10 x MMA groups per tile (1|2) + epilogue variant (3: divergent per-lane
 * group tests, 5: one warp vote per 64-column step + quad-mask record stores; default 215), and the rank
 * coefficient c of the speculative threshold (about c * k_row items are expected above it). */
int b200_recommend_embed_tune(int32_t organisation_code, float pre_rank_coef);
/* profiling diagnostics only (results are wrong while level > 0): ablate parts of the main pass
 * (1: nothing is collected, cold epilogue steps only; 2: no epilogue at all, MMAs and stage releases only) */
int b200_recommend_embed_debug(int32_t ablate_level);
int b200_recommend_embed_plan(int64_t B, int64_t N, int32_t d, int32_t K, int32_t* out, int32_t n_out);
int b200_embed_catalog_bytes(int64_t N, int32_t d, size_t* bytes);
int b200_embed_catalog_prepare(const float* I, int64_t ldi, int64_t N, int32_t d, void* catalog,
                               size_t bytes, void* stream);
int b200_recommend_embed_workspace_bytes(int64_t B, int64_t N, int32_t d, int32_t K, size_t* bytes);
int b200_recommend_embed(const float* U, int64_t ldu, const int64_t* user_ids, int64_t B,
                         const float* I, int64_t ldi, int64_t N, int32_t d, const void* catalog,
                         const int64_t* indptr, const int32_t* idx, int64_t n_users, int32_t filter,
                         int32_t K, int64_t* out_ids, float* out_scores, int32_t* row_status,
                         void* workspace, size_t workspace_bytes, void* stream,
                         void* ev_sweep_start /* cudaEvent_t or NULL: recorded on `stream` */,
                         void* ev_sweep_stop  /* just before / after the wgmma sweep kernels */);

/* ---- 8e row 2: row-sharded embedding table over NVLink peer memory ------------------------
 * (the reference has ONE table, libreco/layers/embedding.py:16-23; here row r lives on GPU r % G at
 * slot r / G).  shards: HOST array of n_ranks DEVICE pointers, shards[g] = GPU g's shard
 * [ceil(n_rows / G), ld] as mapped into this process (symmetric / peer-mapped allocation; for
 * n_ranks == 1 an ordinary device pointer).  One kernel does the gather AND the exchange:
 *   gather:      out[i, :d] = shards[ids[i] % G][(ids[i] / G) * ld + :d]        (peer loads)
 *   scatter_add: shards[ids[i] % G][(ids[i] / G) * ld + :d] += rows[i, :d]      (peer float atomics)
 * The caller orders the kernels against the owners' updates (stream-ordered barrier on the symmetric
 * memory signal pads).  n_ranks <= 16. */
int b200_peer_gather_rows(const void* const* shards, int32_t n_ranks, int64_t ld, int32_t d,
                          const int64_t* ids, int64_t n, float* out, int64_t ld_out, void* stream);
int b200_peer_scatter_add_rows(void* const* shards, int32_t n_ranks, int64_t ld, int32_t d,
                               const int64_t* ids, int64_t n, const float* rows, int64_t ld_rows,
                               void* stream);

/* ---- a10: LightGCN propagation (libreco/algorithms/torch_modules/lightgcn_module.py:66-88) -
 * out[r,:] = sum_j val[j] * E[col[j],:] over the CSR row r (fma in CSR order), optionally fused with
 * the layer-mean: acc = (acc_init ? E[r,:] : acc[r,:]) + out[r,:], then acc /= final_div if > 0.
 * Rows longer than b200_spmm_long_row_threshold() nnz must be listed in long_rows and split into
 * chunks of b200_spmm_chunk() nnz: chunk c covers nnz [indptr[row] + chunk_k[c]*chunk, ...) of
 * row chunk_row[c]; long_chunk_ptr[n_long+1] delimits each long row's chunks; partials is a
 * caller-provided float [n_chunks, d] scratch.  Deterministic (no float atomics).  d <= 256. */
int b200_spmm_long_row_threshold(void);
int b200_spmm_chunk(void);
int b200_spmm_csr(const int64_t* indptr, const int32_t* col, const float* val, int64_t n_rows,
                  const float* E, int64_t ld_e, int32_t d, float* out, int64_t ld_out, float* acc,
                  int64_t ld_acc, int32_t acc_init, float final_div, const int32_t* long_rows,
                  const int64_t* long_chunk_ptr, int64_t n_long, const int32_t* chunk_row,
                  const int32_t* chunk_k, int64_t n_chunks, float* partials, void* stream);

/* ---- a4/a5/a6: feature models (FM, DeepFM, towers) -------------------------------------
 * Layout of the per-row features, as the reference's DataInfo provides them
 * (libreco/data/data_info.py:107-158, libreco/prediction/preprocess.py:15-57):
 * sparse field f of a row comes either from an explicit matrix sparse_rows[r, f] or — when
 * sparse_rows is NULL — from the unique table of its side: user_sparse_unique[user, col] /
 * item_sparse_unique[item, col].  Same for dense fields.  All indices are global offsets into the
 * ONE shared sparse table (libreco/feature/sparse.py:106-119,165-168). */
#define B200_MAX_FIELDS 128
typedef struct {
  int32_t embed_size, n_sparse, n_dense;
  int32_t id_mask;                      /* bit0: user-id embedding is a field, bit1: item-id embedding
                                           (3 for FM/DeepFM/DIN rows, 1 / 2 for the TwoTower towers) */
  int32_t dense_embed_row[B200_MAX_FIELDS]; /* row of dense_embeds / dense_linear used by dense field f */
  int32_t sparse_side[B200_MAX_FIELDS]; /* 0 = user side, 1 = item side */
  int32_t sparse_col[B200_MAX_FIELDS];  /* column inside that side's unique table */
  int32_t dense_side[B200_MAX_FIELDS];
  int32_t dense_col[B200_MAX_FIELDS];
  const int32_t* user_sparse_unique; int64_t ld_us;  /* [n_users+1, F_us] */
  const int32_t* item_sparse_unique; int64_t ld_is;  /* [n_items+1, F_is] */
  const float* user_dense_unique; int64_t ld_ud;
  const float* item_dense_unique; int64_t ld_id;
  const int32_t* sparse_rows; int64_t ld_sparse_rows; /* explicit [R, n_sparse] or NULL */
  const float* dense_rows; int64_t ld_dense_rows;     /* explicit [R, n_dense] or NULL */
} b200_feat_layout;

typedef struct {       /* TF scope "embedding" (SURVEY.md Appendix C), fp32, row-major */
  const float* user_embeds;   /* [n_users+1, K] */
  const float* item_embeds;   /* [n_items+1, K] */
  const float* sparse_embeds; /* [V_s, K] */
  const float* dense_embeds;  /* [F_d, K] */
  const float* user_linear;   /* [n_users+1] (FM / DeepFM only, else NULL) */
  const float* item_linear;   /* [n_items+1] */
  const float* sparse_linear; /* [V_s] */
  const float* dense_linear;  /* [F_d] */
} b200_feat_tables;

/* One pass over R rows: row r = (users[r], items[r]), or with grid_items > 0 the implicit grid
 * (users[(r + row_offset) / grid_items], item (r + row_offset) % grid_items) used by all-items
 * scoring (outputs are indexed by the local r).  Any output may be NULL:
 *   concat [R, (2+F_s+F_d)*K]  concatenated field embeddings (deep / tower input)
 *   pw     [R, K]              0.5((sum_f e)^2 - sum_f e^2)            (fm.py:158-161)
 *   lin    [R]                 Dense1(concat of linear features) + bias (fm.py:156)
 *   fm_out [R]                 lin + elu(Dense1(BN(pw)))               (fm.py:165-170); BN folded
 *                              to scale/shift (inference), bn_scale NULL = use_bn False */
/* process-wide switch (A/B measurements, tests).  bit 0: 1 = the bulk-copy (TMA) staged persistent gather for
 * eligible shapes (K % 4 == 0, K <= 32, >= 2048 rows), 0 = the register-gather kernels only.
 * bit 1: 1 = the older lane-per-field register kernel instead of the field-group kernel (K in {4,8,16,32}).
 * bit 2: 1 = plain field-group kernel also for >= 4096 rows (default there: its software-pipelined variant).
 * bit 3: 1 = the cp.async (LDGSTS) shared-memory staged variant instead of the software-pipelined one. */
int b200_feat_forward_tune(int32_t use_tma_staging);
int b200_feat_forward(const b200_feat_layout* layout, const b200_feat_tables* tables,
                      const int64_t* users, const int64_t* items, int64_t R, int64_t grid_items,
                      int64_t row_offset, float* concat, int64_t ld_concat, float* pw, int64_t ld_pw, float* lin,
                      float* fm_out, const float* lin_kernel, float lin_bias, const float* bn_scale,
                      const float* bn_shift, const float* pw_kernel, float pw_bias,
                      float* ssum /* [R,K] sum_f e, or NULL */, float* sqsum /* [R,K] sum_f e^2 */,
                      int64_t ld_s, void* stream);

/* Hoisted all-items scoring (SURVEY.md §7.2-4): everything that depends on the user only or on the
 * item only is computed once (b200_feat_forward over the user-side / item-side fields: S = sum e,
 * Q = sum e^2, the linear partial, and for DeepFM the first MLP layer's partial products Pu, Pi);
 * a (user, item) pair then costs K adds for the FM term and the SMALL layers of the MLP:
 *   pw = 0.5((Su+Si)^2 - (Qu+Qi)),  lin = lu + li + lin_bias
 *   FM     (fm.py:158-170):      out = lin + elu(<bn(pw), pw_kernel> + pw_bias)
 *   DeepFM (deepfm.py:160-173):  h1 = relu(Pu[b] + Pi[n]); h2 = relu(h1 W2 + b2); deep = h2 W3 + b3
 *                                (or deep = h1 W2 + b2 with two layers); out = <[lin, pw, deep], w_out> + b_out
 * scores[b, n] for every b < B, n < N.  H1 <= 256, H2 <= 64, H3 <= 32; W2 [H1,H2], W3 [H2,H3] row-major. */
int b200_fm_pair_scores(const float* Su, const float* Qu, const float* lu, int64_t B, const float* Si,
                        const float* Qi, const float* li, int64_t N, int32_t K, float lin_bias,
                        const float* bn_scale, const float* bn_shift, const float* pw_kernel,
                        float pw_bias, float* scores, int64_t lds, void* stream);
int b200_deepfm_pair_scores(const float* Su, const float* Qu, const float* lu, const float* Pu, int64_t B,
                            const float* Si, const float* Qi, const float* li, const float* Pi,
                            int64_t N, int32_t K, int32_t H1, int32_t H2, int32_t H3, float lin_bias,
                            const float* W2, const float* b2, const float* W3, const float* b3,
                            const float* w_out, float b_out, float* scores, int64_t lds, void* stream);

/* multi_sparse_combine_embedding / multi_sparse_alone (libreco/tfops/features.py:47-118): the
 * `len` sub-columns of one multi-sparse field (idx[r, 0..len)) pooled into one row:
 * out[r] = sum_{t: idx != oov} table[idx[r,t]] / {1 | count | sqrt(count)} (combiner 0 sum, 1 mean,
 * 2 sqrtn; division is div_no_nan).  K = 1 with ld = 1 pools the 1-D linear table.  Run once per
 * (field, side) over the unique table: the pooled rows are appended to the shared sparse table and
 * the field becomes an ordinary single-index field of b200_feat_forward. */
int b200_multi_sparse_combine(const float* table, int64_t ld, int32_t K, const int32_t* idx, int64_t ld_idx,
                              int32_t len, int64_t n, int32_t oov, int32_t combiner, float* out,
                              int64_t ld_out, void* stream);

/* Row gather / scatter-add on ONE rank's slice of a row-sharded embedding table (SURVEY.md 8e row 2:
 * tables larger than one GPU; the exchange of indices and rows is torch.distributed all-to-all,
 * librecommender_b200/parallel.py::RowShardedTable).  out[r] = table[idx[r]]; table[idx[r]] += rows[r]. */
int b200_gather_rows(const float* table, int64_t ld, int32_t d, const int64_t* idx, int64_t n, float* out,
                     int64_t ld_out, void* stream);
int b200_scatter_add_rows(float* table, int64_t ld, int32_t d, const int64_t* idx, int64_t n,
                          const float* rows, int64_t ld_rows, void* stream);

/* Y = act(X Wt^T + b): tf_dense (libreco/layers/dense.py:52-80) with BN folded by the caller.
 * Wt is the TRANSPOSED kernel [dout, din]; fp32 SIMT (exact fma chain in k). */
int b200_linear_f32(const float* X, int64_t ldx, int64_t R, const float* Wt, int64_t ldw,
                    const float* bias, int32_t din, int32_t dout, int32_t relu, float* Y,
                    int64_t ldy, void* stream);

/* Same contract as b200_linear_f32 on the tensor cores (wgmma): operands split x = hi + lo into
 * two tf32 values, three tf32 products (hi*hi + lo*hi + hi*lo) in separate main / correction
 * accumulators promoted to fp32 registers every 64 k: fp32-level accuracy, not tf32-level.
 * Requires 16-byte aligned X rows (ldx % 4 == 0).  Wsplit (optional, NULL allowed): the layer's
 * weights pre-split once by b200_linear_tf32x3_split_weights — 2 * dout * split_ld(din) floats —
 * which removes the per-tile weight splitting from the kernel; without it Wt rows must be 16-byte
 * aligned too.  Callers use b200_linear_f32 for shapes that do not qualify. */
int64_t b200_linear_tf32x3_split_ld(int32_t din);
int b200_linear_tf32x3_split_weights(const float* Wt, int64_t ldw, int32_t din, int32_t dout, float* Wsplit,
                                     void* stream);
int b200_linear_tf32x3(const float* X, int64_t ldx, int64_t R, const float* Wt, int64_t ldw,
                       const float* Wsplit, const float* bias, int32_t din, int32_t dout, int32_t relu,
                       float* Y, int64_t ldy, void* stream);

/* Split-K form for products with few output tiles and a long reduction (the weight gradients dWt = dY^T X of
 * the training steps: 1792 x 128 outputs over 8192 rows = 14 tiles): `splits` CTAs along the reduction per
 * output tile write partial products into workspace (splits * R * dout floats), a second kernel adds them in a
 * fixed order (+ bias, ReLU).  splits == 1 is b200_linear_tf32x3 without a pre-split weight copy. */
int b200_linear_tf32x3_splitk(const float* X, int64_t ldx, int64_t R, const float* Wt, int64_t ldw, const float* bias,
                              int32_t din, int32_t dout, int32_t relu, int32_t splits, float* workspace,
                              size_t workspace_bytes, float* Y, int64_t ldy, void* stream);

/* ---- training step of the FM-family models (SURVEY.md 8f-1; reference graph in training mode:
 * libreco/algorithms/fm.py:152-171, tf.layers.batch_normalization(training=True),
 * libreco/training/tf_trainer.py:112-123 tf.train.AdamOptimizer + BN update ops) --------------- */

/* y = gamma * (x - mean_batch) / sqrt(var_batch + eps) + beta over the R rows of x [R, K]; the batch
 * variance is the biased one (tf.nn.moments); moving_* (nullable) are updated with `momentum`. */
int b200_bn_train_forward(const float* x, int64_t ldx, int64_t R, int32_t K, const float* gamma,
                          const float* beta, float eps, float momentum, float* y, int64_t ldy,
                          float* batch_mean, float* batch_var, float* moving_mean, float* moving_var,
                          void* stream);

/* z = <y, pw_kernel> + pw_bias; logit = lin + lin_bias + elu(z)   (fm.py:156,169-170).  The two
 * biases are DEVICE scalars (trainable variables; NULL = 0): no host round trip per step. */
int b200_fm_head_forward(const float* y, int64_t ldy, int64_t R, int32_t K, const float* pw_kernel,
                         const float* pw_bias, const float* lin, const float* lin_bias, float* z,
                         float* logit, void* stream);

/* d loss / d logit -> d loss / d pw [R, K] through elu, Dense(1) and (batch_mean != NULL) the batch-norm
 * with batch statistics; ADDS the gradients of pw_kernel [K], pw_bias [1], gamma / beta [K] and
 * (nullable) the bias of the linear term to the given buffers.  Deterministic. */
size_t b200_fm_head_backward_workspace_bytes(int64_t R, int32_t K);
int b200_fm_head_backward(const float* dlogit, const float* z, const float* pw, int64_t ld, int64_t R,
                          int32_t K, const float* batch_mean, const float* batch_var, const float* gamma,
                          const float* beta, float eps, const float* pw_kernel, float* dpw, int64_t ld_dpw,
                          float* g_pw_kernel, float* g_pw_bias, float* g_gamma, float* g_beta,
                          float* g_lin_bias, void* workspace, size_t workspace_bytes, void* stream);

/* Backward of b200_feat_forward: for every row and field f, d e_f = dpw[r] * (S[r] - e_f) (FM pairwise
 * term; S = sum_f e from the forward) + dconcat[r, f*K..] (deep input; nullable), scatter-ADDED into
 * dense gradient buffers shaped like the tables; with dlogit: the linear-feature gradients
 * (g_*_linear, g_lin_kernel [2+F_s+F_d]).  Float atomics (summation order is not fixed). */
int b200_feat_backward(const b200_feat_layout* layout, const b200_feat_tables* tables, const int64_t* users,
                       const int64_t* items, int64_t R, const float* dpw, int64_t ld_dpw, const float* S,
                       int64_t ld_s, const float* dconcat, int64_t ld_dconcat, const float* dlogit,
                       const float* lin_kernel, float* g_user_embeds, float* g_item_embeds,
                       float* g_sparse_embeds, float* g_dense_embeds, float* g_user_linear,
                       float* g_item_linear, float* g_sparse_linear, float* g_dense_linear,
                       float* g_lin_kernel, void* stream);

/* Pieces of dense_nn in training mode (libreco/layers/dense.py:12-49) and of the DeepFM head
 * (algorithms/deepfm.py:172-173).  The Dense layers themselves run on b200_linear_*:
 * dX = dY Wk^T and dWt = dY^T X are calls of the same kernel on transposed views. */

/* out[k] += sum_r (wrow ? wrow[r] : 1) * X[r,k] * (Y ? Y[r,k] : 1)   (bias gradients, weighted column
 * sums of the head); double accumulation, deterministic. */
int b200_col_reduce(const float* X, int64_t ldx, int64_t R, int32_t K, const float* wrow, const float* Y,
                    int64_t ldy, float* out, void* stream);

/* Backward of b200_bn_train_forward (batch statistics): dx, and g_gamma / g_beta ADDED.  relu_mask != 0:
 * x is a ReLU output and the result is additionally masked with x > 0 (Dense -> ReLU -> BN blocks).
 * workspace: 16 bytes per column. */
int b200_bn_train_backward(const float* dy, int64_t lddy, const float* x, int64_t ldx, int64_t R, int32_t K,
                           const float* batch_mean, const float* batch_var, const float* gamma, float eps,
                           int32_t relu_mask, float* dx, int64_t lddx, float* g_gamma, float* g_beta,
                           void* workspace, size_t workspace_bytes, void* stream);
int b200_relu_backward(const float* dy, const float* a, int64_t n, float* dx, void* stream);

/* logit = <[lin + lin_bias, pw[0..K), deep[0..H)], out_kernel> + out_bias (biases: device scalars or NULL);
 * backward: dlin = dlogit * w[0], dpw = dlogit * w[1..K], ddeep = dlogit * w[1+K..]. */
int b200_deepfm_head_forward(const float* lin, const float* lin_bias, const float* pw, int64_t ldpw, int32_t K,
                             const float* deep, int64_t lddeep, int32_t H, const float* out_kernel,
                             const float* out_bias, int64_t R, float* logit, void* stream);
int b200_deepfm_head_backward(const float* dlogit, const float* out_kernel, int32_t K, int32_t H, int64_t R,
                              float* dlin, float* dpw, int64_t lddpw, float* ddeep, int64_t lddeep,
                              void* stream);

/* Backward of b200_l2_normalize_rows: x = the rows BEFORE normalisation, dy = gradient of the
 * normalised rows; dx may alias dy. */
int b200_l2_normalize_backward(const float* x, int64_t ldx, const float* dy, int64_t lddy, int64_t R, int32_t d,
                               float* dx, int64_t lddx, void* stream);

/* tf.train.AdamOptimizer over a WHOLE variable (what _apply_sparse_shared does for embedding
 * variables: m, v decayed everywhere, every row updated): lr_t = lr sqrt(1-b2^t)/(1-b1^t),
 * m = b1 m + (1-b1) g, v = b2 v + (1-b2) g^2, param -= lr_t m / (sqrt(v) + eps); grad is zeroed. */
int b200_adam_dense(float* param, float* m, float* v, float* grad, int64_t n, float lr, float beta1,
                    float beta2, float eps, int64_t step, void* stream);

/* The same update for a CAPTURED (CUDA graph) training step: b200_adam_begin_step increments the device step
 * counter and writes lr_t = lr sqrt(1-b2^t)/(1-b1^t) (double arithmetic) to lr_t_dev once per step;
 * b200_adam_dense_dev reads it — nothing about the step number is baked into the launch parameters.
 * decay_steps > 0: lr is first multiplied by decay_rate ^ floor((t - 1) / decay_steps) (lr_decay=True:
 * tf.train.exponential_decay, staircase, libreco/tfops/configs.py:38-45). */
int b200_adam_begin_step(int64_t* step_dev, float lr, float beta1, float beta2, float decay_rate, int64_t decay_steps,
                         float* lr_t_dev, void* stream);
/* y += alpha * x — the L2 regulariser's gradient 2 reg w (tf.keras.regularizers.l2, tfops/configs.py:20-26). */
int b200_axpy(float* y, const float* x, float alpha, int64_t n, void* stream);
int b200_adam_dense_dev(float* param, float* m, float* v, float* grad, int64_t n, const float* lr_t_dev, float beta1,
                        float beta2, float eps, void* stream);

/* ---- training losses (SURVEY.md 8a row a13): value + gradient w.r.t. the scores in one pass ------
 * All reductions are two-stage and deterministic.  `workspace` >= b200_loss_workspace_bytes().
 * `loss_out` is a device scalar.  Gradient outputs may be NULL. */
size_t b200_loss_workspace_bytes(void);

/* mean over n of: kind 0 sigmoid cross entropy (torchops/loss.py:5-6, tfops/loss.py:14-18),
 * 1 focal (torchops/loss.py:10-19, tfops/loss.py:52-58), 2 squared error (tfops/loss.py:5-8).
 * dlogits[i] = d loss / d logits[i]. */
int b200_pointwise_loss(const float* logits, const float* labels, int64_t n, int32_t kind, float alpha,
                        float gamma, float* loss_out, float* dlogits, void* workspace,
                        size_t workspace_bytes, void* stream);

/* kind 0 bpr = -mean log sigmoid(pos - neg) (torchops/loss.py:22-24), 1 max-margin
 * mean relu(margin - (pos - neg)) (:27-30, tfops/loss.py:61-64): n_neg must be a multiple of n_pos,
 * negatives of positive j are neg[j*f .. (j+1)*f) (compute_pair_scores, :63-90), dpos has n_pos entries.
 * kind 2 / 3 = sigmoid CE / focal over [pos (label 1), neg (label 0)] (:33-60), mean or sum. */
int b200_pairwise_loss(const float* pos, int64_t n_pos, const float* neg, int64_t n_neg, int32_t kind,
                       float margin, float alpha, float gamma, int32_t mean, float* loss_out, float* dpos,
                       float* dneg, void* workspace, size_t workspace_bytes, void* stream);

/* In-batch sampled softmax of the two-tower models (tfops/loss.py:67-71, TwoTower.adjust_logits
 * algorithms/two_tower.py:458-479).  S[B, B] holds U I^T on entry; logits = S / temperature
 * - log(clip(correction[col], 1e-8, 1)) (correction may be NULL); when item_ids is given,
 * off-diagonal columns carrying the row's own item id are masked with FLT_MIN-like padding.
 * loss = mean_r (logsumexp(row r) - logit[r, r]).  write_grad: S is overwritten by d loss / d S. */
int b200_softmax_inbatch_loss(float* S, int64_t lds, int32_t B, float temperature, const float* correction,
                              const int64_t* item_ids, int32_t write_grad, float* loss_out, void* workspace,
                              size_t workspace_bytes, void* stream);

/* Sampled-class losses of YouTubeRetrieval training (tf.nn.sampled_softmax_loss / tf.nn.nce_loss, reference
 * libreco/training/tf_trainer.py:162-235; TensorFlow's _compute_sampled_logits with remove_accidental_hits=True and
 * subtract_log_q=True).  logits [B, ld] holds U W_s^T (the S sampled classes) on entry, true_dot[B] = <u_r, w_label>.
 *   z0 = true_dot[r] + bias[label] - log E(label),  z_s = logits[r, s] + bias[id_s] - log E(id_s),
 * E = TensorFlow's expected count in float: p S if *num_tries == S, else -expm1(num_tries log1p(-p)), with p = 1/n_items
 * (sampler_kind 0, uniform) or log((c+2)/(c+1)) / log1p(n_items) (1, log-uniform).  A sampled id equal to the row's
 * label is an accidental hit and contributes exactly nothing.  loss_kind 0: softmax CE over [z0, z_s..] with the
 * label in column 0; 1 (NCE): sigmoid CE(z0, 1) + sum_s sigmoid CE(z_s, 0).  *loss_out = mean over the B rows
 * (device scalar; deterministic two-stage reduction); logits is overwritten with d loss / d z_s and dtrue[r] =
 * d loss / d z0.  num_tries: device scalar (b200_unique_candidates).  1 <= S <= min(n_items, 65536), ld >= S;
 * workspace >= b200_sampled_class_loss_workspace_bytes(B, S). */
size_t b200_sampled_class_loss_workspace_bytes(int32_t B, int32_t S);
int b200_sampled_class_loss(int32_t loss_kind, float* logits, int64_t ld, int32_t B, int32_t S, const float* true_dot,
                            const int64_t* labels, const int64_t* sampled, const float* bias, int32_t sampler_kind,
                            int64_t n_items, const int64_t* num_tries, float* loss_out, float* dtrue, void* workspace,
                            size_t workspace_bytes, void* stream);

/* out[r] = bias + <[a[r,:na], b[r,:nb], c[r,:nc]], w>: Dense(1) on a concatenation
 * (deepfm.py:172-173; the final Dense(1) of DIN / YouTubeRanking). */
int b200_concat_dense(const float* a, int64_t lda, int32_t na, const float* b, int64_t ldb, int32_t nb,
                      const float* c, int64_t ldc, int32_t nc, const float* w, float bias, int64_t R,
                      float* out, void* stream);

/* x[r,:] /= sqrt(max(sum x^2, 1e-12)) — normalize_embeds (libreco/layers/normalization.py:32-44) */
int b200_l2_normalize_rows(float* x, int64_t ld, int64_t R, int32_t d, void* stream);

/* ---- a7/a8: behaviour sequences (DIN attention, YouTubeRanking pooling) -------------------
 * Sequences live in a per-user table seqs[n_users+1, T] (pad index = n_items) with lens[n_users+1]
 * (libreco/batch/sequence.py:75-91); row r reads the row of users[r], or with grid_items > 0 of
 * users[(r + row_offset) / grid_items] (item = (r + row_offset) % grid_items) — the reference's
 * np.repeat(seqs, n_items) (prediction/preprocess.py:109-118) is never built.
 * b200_seq_pool:      out[r,:d] = sum_t E[seq_t,:] / sqrt(len), entries equal to pad_index read as 0
 *                     (libreco/layers/embedding.py:54-85).
 * b200_din_attention: G = item feature table [n_items+1, Kp] (combine_seq_features, concat mode,
 *                     libreco/tfops/features.py:165-218); out[r,:Kp] = softmax_t(Dense1(sigmoid(
 *                     Dense16([q,k,q-k,q*k]))) * rsqrt(Kp), t < len) weighted sum of the keys
 *                     (libreco/layers/attention.py:45-64).  k1 [4Kp,16], b1 [16], k2 [16], b2.
 *                     k1 == NULL selects the reference's use_tf_attention=True variant
 *                     (attention.py:5-25: dot-product scores <q, k_t>, masked softmax, no weights).
 *                     Kp <= 128, T <= 256. */
int b200_seq_pool(const float* E, int64_t lde, int32_t d, int64_t pad_index, const int32_t* seqs,
                  int64_t ld_seq, const int32_t* lens, int32_t T, const int64_t* users, int64_t R,
                  int64_t grid_items, int64_t row_offset, float* out, int64_t ld_out, void* stream);
/* Backward of b200_seq_pool (training of the sequence models): g_embeds[seq_t, :d] += dout[r, :d] / sqrt(len)
 * for every non-pad position of row r's sequence (row of users[r] in seqs / lens); float atomics. */
int b200_seq_pool_backward(const float* dout, int64_t ld_dout, int32_t d, int64_t pad_index, const int32_t* seqs,
                           int64_t ld_seq, const int32_t* lens, int32_t T, const int64_t* users, int64_t R,
                           float* g_embeds, int64_t ld_g, void* stream);
int b200_din_attention(const float* G, int64_t ldg, int32_t Kp, const int64_t* items,
                       const int32_t* seqs, int64_t ld_seq, const int32_t* lens, int32_t T,
                       const int64_t* users, int64_t R, int64_t grid_items, int64_t row_offset,
                       const float* k1, const float* b1, const float* k2, float b2, float* out,
                       int64_t ld_out, void* stream);
/* process-wide A/B switch (tests, measurements): 1 = the lane-owns-position kernel for T <= 64 and K' % 4 == 0
 * (default), 0 = the first version everywhere. */
int b200_din_attention_tune(int32_t use_v2);

/* Backward of b200_din_attention (paper attention, explicit pairs: row r = (items[r], sequence row users[r])):
 * dout [R, Kp] = gradient of the attention output.  ADDS (float atomics) the gradient of the item feature rows
 * into dG [n_items+1, Kp] (query row and every non-masked key row) and the gradients of the attention weights
 * into g_k1 [4Kp, 16], g_b1 [16], g_k2 [16], g_b2 [1].  T <= 64; rows with length 0 contribute nothing. */
int b200_din_attention_backward(const float* G, int64_t ldg, int32_t Kp, const int64_t* items, const int32_t* seqs,
                                int64_t ld_seq, const int32_t* lens, int32_t T, const int64_t* users, int64_t R,
                                const float* k1, const float* b1, const float* k2, float b2, const float* dout,
                                int64_t ld_dout, float* dG, int64_t ld_dg, float* g_k1, float* g_b1, float* g_k2,
                                float* g_b2, void* stream);

/* NGCF layer pieces (libreco/algorithms/torch_modules/ngcf_module.py:100-121; SURVEY.md 8f-4): the
 * propagation L E is b200_spmm_csr, the two Dense products are b200_linear_*; these are the
 * element-wise parts: out = a * b, and out[r] = normalize_2(leaky_relu(self[r] + pair[r], slope)). */
int b200_mul_elementwise(const float* a, const float* b, int64_t n, float* out, void* stream);
int b200_ngcf_combine(const float* self_part, int64_t lda, const float* pair_part, int64_t ldb, int64_t R,
                      int32_t d, float negative_slope, float* out, int64_t ld_out, void* stream);

/* DIN all-items scoring, hoisted per user (SURVEY.md 8d row "a7 DIN all-items"): the keys of ONE
 * user (item ids seq[0..len) of the behaviour sequence, rows of the item feature table G [*, Kp]) turn
 * the attention MLP's Dense(16) into a plain GEMM over the candidate items:
 *   b200_din_user_weights      -> Wt [16 len, Kp], bias [16 len]  (row t*16+j)
 *   Z = b200_linear_*(G[:N], Wt, bias)                             [N, 16 len]
 *   b200_din_attention_hoisted -> out[n] = sum_t softmax_t((<k2, sigmoid(Z[n, t, :])> + b2) / sqrt(Kp)) k_t
 * (attention.py:28-64; len == 0 -> zeros). */
int b200_din_user_weights(const float* G, int64_t ldg, int32_t Kp, const int32_t* seq, int32_t len,
                          const float* k1, const float* b1, float* Wt, int64_t ldw, float* bias, void* stream);
int b200_din_attention_hoisted(const float* Z, int64_t ldz, int64_t N, const float* G, int64_t ldg, int32_t Kp,
                               const int32_t* seq, int32_t len, const float* k2, float b2, float* out,
                               int64_t ld_out, void* stream);

/* The same per-user product with the attention's tail FUSED into the GEMM epilogue (DIN all-items):
 * A[r, g] = sum_{j<16} dot_w16[j] * sigmoid((X Wt^T + bias)[r, 16 g + j]), g < dout / 16 — the [R, dout]
 * pre-activations (16x the bytes of A) are never written.  Then b200_din_attention_from_logits:
 * out[n, :Kp] = sum_t softmax_t((A[n, t] + b2) * rsqrt(Kp)) * G[seq[t], :Kp], t < len (1 <= len <= 64). */
int b200_linear_tf32x3_sigmoid_dot(const float* X, int64_t ldx, int64_t R, const float* Wt, int64_t ldw,
                                   const float* Wsplit, const float* bias, int32_t din, int32_t dout,
                                   const float* dot_w16, float* A, int64_t lda, void* stream);
int b200_din_attention_from_logits(const float* A, int64_t lda, int64_t N, const float* G, int64_t ldg, int32_t Kp,
                                   const int32_t* seq, int32_t len, float b2, float* out, int64_t ld_out,
                                   void* stream);

/* ---- a12: negative sampling (libreco/sampling/negatives.py:17-82; collators.py:138-166) ---
 * Counter-based (Philox4x32-10) device sampler; result = f(seed, step, index) only.
 * mode 0 random, 1 unconsumed (needs users + per-user SORTED consumed CSR), 2 popular (needs the
 * cdf of p ~ freq^0.75).  out[j*num_neg + t] = t-th negative of positive j.  The bit-exact
 * reproduction of the reference's numpy / Mersenne streams is the host parity mode
 * (librecommender_b200/sampling.py). */
int b200_sample_negatives(const int64_t* users, const int64_t* items_pos, int64_t n_pos,
                          int32_t num_neg, int64_t n_items, int32_t mode, int32_t tolerance,
                          uint64_t seed, uint64_t step, const int64_t* indptr,
                          const int32_t* idx_sorted, int64_t n_users, const float* cdf, int64_t* out,
                          void* stream);

/* Unique candidate sampler of the sampled-class losses: TensorFlow's uniform_candidate_sampler (kind 0) /
 * log_uniform_candidate_sampler (kind 1) with unique=True.  Draws with replacement and keeps first occurrences
 * until it holds num_sampled = S distinct ids: out[0..S) = those ids in draw order, *num_tries (device int64) =
 * the number of draws taken.  Draw j = Philox4x32-10(seed, step, j) with step = *step_dev (a DEVICE counter, e.g.
 * the Adam step of b200_adam_begin_step, so a captured CUDA graph draws fresh candidates on every replay);
 * uniform: the bounded 64-bit draw of b200_sample_negatives; log-uniform: (int64)exp(u log1p(n_items)) - 1, then
 * % n_items, u = 53 random bits in [0, 1).  The result equals the sequential process over that draw stream.  One
 * launch, no host round trip.  workspace: b200_unique_candidates_workspace_bytes(n_items) bytes, filled with 0xFF
 * before the FIRST call; every call leaves it that way again (O(S) work).  Envelope: 1 <= n_items < 2^31,
 * 1 <= S <= min(n_items, 65536); anything else returns -2 before launching. */
#define B200_UNIQUE_MAX_SAMPLED 65536
size_t b200_unique_candidates_workspace_bytes(int64_t n_items);
int b200_unique_candidates(int32_t kind, int64_t n_items, int32_t num_sampled, uint64_t seed, const int64_t* step_dev,
                           void* workspace, size_t workspace_bytes, int64_t* out, int64_t* num_tries, void* stream);

/* a11: per-sample behaviour sequences at collate time (libreco/batch/sequence.py:33-71, mode
 * "recent"; called from batch/collators.py:207-222).  consumed CSR in ARRIVAL order.  position =
 * first occurrence of items[j] in the user's list; for items the user never consumed (sampled
 * negatives) position = rand_pos[j] (the reference's random.randrange stream, parity mode) or a
 * Philox draw when rand_pos is NULL.  seqs int32[n, max_seq_len] (padded with pad_index), lens int32[n]. */
int b200_interacted_seqs(const int64_t* indptr, const int32_t* idx, int64_t n_users, const int64_t* users,
                         const int64_t* items, int64_t n, int32_t max_seq_len, int32_t pad_index,
                         const int64_t* rand_pos, uint64_t seed, uint64_t step, int32_t* seqs,
                         int32_t* lens, void* stream);

/* ---- AutoInt inference (libreco/algorithms/autoint.py:146-168, layers/attention.py:67-138) -------
 * X [F, K] = the pair's field embeddings [user, item, sparse.., dense..] (the b200_feat_forward concat).
 * For each layer l (D = num_heads * hd_l; weights packed per layer as Wq [K, D], Wk [K, D], Wv [K, D],
 * Wo [D, K], row-major, columns head-major h * hd + j as _split_heads lays them out):
 *   Q = X Wq, K = X Wk, V = X Wv;  O_h = softmax_rows(Q_h K_h^T / sqrt(hd_l)) V_h;  Y = concat_h(O_h) Wo;
 *   X = X + Y (use_residual) or X = Y.
 * logit = <flatten(X), w_out [F*K]> + b_out.  Wv is the EFFECTIVE value map (the TF < 2.10 graph applies its
 * value Dense to the projected keys, attention.py:104-106: Wv = Wk Wv').  Every dot product is one fmaf chain
 * over an ascending index, the softmax is max, expf(x - max), an ascending sum, then a division, so both
 * entry points give bit-identical logits for the same pair.
 * Supported: 2 <= F <= 130, 1 <= K <= 64, 1 <= n_layers <= 4, num_heads * hd_l <= 64; anything else
 * returns -2 before launching.  head_dims_host: HOST array [n_layers].
 * b200_autoint_rows: out[r] for X = rows of the materialised concat X [R, ldx].
 * b200_autoint_grid: scores[b * ld_scores + n] for every b < B, n < N; field f of pair (b, n) reads
 *   Xu[b, s*K..] with s = field_map[f] when field_map[f] >= 0, else Xi[n, s*K..] with s = -1 - field_map[f]
 *   (field_map: device int32 [F]); the [B*N, F*K] concat is never built. */
int b200_autoint_rows(const float* X, int64_t ldx, int64_t R, int32_t F, int32_t K, int32_t num_heads,
                      int32_t n_layers, const int32_t* head_dims_host, const float* weights, const float* w_out,
                      float b_out, int32_t use_residual, float* out, void* stream);
int b200_autoint_grid(const float* Xu, int64_t ldu, int64_t B, const float* Xi, int64_t ldi, int64_t N,
                      const int32_t* field_map, int32_t F, int32_t K, int32_t num_heads, int32_t n_layers,
                      const int32_t* head_dims_host, const float* weights, const float* w_out, float b_out,
                      int32_t use_residual, float* scores, int64_t ld_scores, void* stream);

/* ---- AutoInt training: the attention core of one layer (layers/attention.py:67-125) ----------------
 * Q, K, V, O: [R*F, ld] row-major, row r*F + f = field f of batch row r, columns head-major (h * hd + j).
 * Per (row r, head h):  S = scale * Q_h K_h^T [F, F],  P = softmax_rows(S),  O_h = P V_h,
 * lse[(r * H + h) * F + f] = log sum_g exp(S_fg)  (float [R, H, F]).  P itself is never stored.
 * The backward recomputes P from Q, K and lse and WRITES (does not add)
 *   dV_h = P^T dO_h,  dS = P o (dO_h V_h^T - rowsum(dO_h o O_h)),  dQ_h = scale dS K_h,  dK_h = scale dS^T Q_h
 * into dQ, dK, dV [R*F, ldg].  One warp owns one (row, head) and accumulates on chip: no atomics, and two
 * identical calls give identical bits.
 * Supported: 2 <= F <= 130, num_heads >= 1, head_dim >= 1, num_heads * head_dim <= 64, every stride >= that
 * product, a finite scale; anything else returns -2 before launching. */
int b200_autoint_attention_forward(const float* Q, int64_t ldq, const float* K, int64_t ldk, const float* V,
                                   int64_t ldv, int64_t R, int32_t F, int32_t num_heads, int32_t head_dim,
                                   float scale, float* O, int64_t ldo, float* lse, void* stream);
int b200_autoint_attention_backward(const float* Q, int64_t ldq, const float* K, int64_t ldk, const float* V,
                                    int64_t ldv, const float* O, int64_t ldo, const float* lse, const float* dO,
                                    int64_t lddo, int64_t R, int32_t F, int32_t num_heads, int32_t head_dim,
                                    float scale, float* dQ, float* dK, float* dV, int64_t ldg, void* stream);

/* ---- a14: predict_from_embedding (libreco/prediction/predict.py:36-40) -----------------
 * out[r] = sum_k U[users[r],k] * I[items[r],k]; mode 0: raw, 1: expit (ranking),
 * 2: clip to [lo, hi] (rating) — normalize_prediction (:18-23). */
int b200_gather_dot(const float* U, int64_t ldu, const int64_t* users, const float* I,
                    int64_t ldi, const int64_t* items, int64_t n, int32_t d, int32_t mode,
                    float lo, float hi, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200RECO_H_ */
