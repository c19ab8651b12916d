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
 * both CTAs) + MMA organisation actually used (1, 2 or 3 as in the tune code; 3 runs as 1 when
 * d > 128), out[7] records per candidate list (n_out >= 8); out[8] pre-pass stride and out[9] item
 * tiles the pre-pass visits (sampled fraction f = out[9] / item tiles) when n_out >= 10; out[10 + k]
 * = the speculative rank pre_k of k_row = k, k = 0 .. 288, when n_out >= 299.  Without a device the
 * plan is the one of a 132-SM H100.
 * b200_recommend_embed_tune (process-wide, not thread-safe; 0 keeps a value): organisation code =
 * 100 x cluster size (1|2) + 10 x MMA organisation (1: one N=256 group per item tile; 2: two N=128
 * groups; 3: two N=128 groups pipelined across item tiles, each half-tile epilogue running under the
 * MMAs of the other half; d > 128 falls back to 1) + epilogue variant (3: divergent per-lane group
 * tests, 5: one warp vote per 64-column step + quad-mask record stores; default 215), and the rank
 * coefficient c in [1, 16] of the linear speculative rule pre_k = margin + ceil(c * f * k_row)
 * (about c * k_row items are expected above the threshold; a non-zero c selects that rule, the
 * margin is set by b200_recommend_embed_debug(-margin), default 12). */
int b200_recommend_embed_tune(int32_t organisation_code, float pre_rank_coef);
/* speculative threshold of b200_recommend_embed (process-wide, not thread-safe): the pre-pass visits
 * every pre_stride-th item tile (2 .. 32; 0 = default 8) and pre_k is the smallest r with
 * P[Binomial(k_row + 16, f) >= r] <= delta, the failure budget per row (1e-9 .. 1e-2; 0 = default
 * 1e-5).  Selects this rule (the default) again after a non-zero rank coefficient of
 * b200_recommend_embed_tune. */
int b200_recommend_embed_speculation(int32_t pre_stride, float delta);
/* profiling diagnostics only (results are wrong while level 1 or 2 is set): ablate parts of the main pass
 * (1: nothing is collected, cold epilogue steps only; 2: no epilogue at all, MMAs and stage releases only);
 * 3 (results unchanged): every row is finalized by the one-CTA-per-row kernel instead of the one-warp-per-row
 * kernel, so that tests can compare the two paths on the same inputs */
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
                         void* ev_sweep_stop  /* just before / after the wgmma sweep kernels */,
                         int32_t* n_flagged   /* NULL, or one int32 (pinned host or device): the call's count of
                                                 rows with a non-zero row_status, copied on `stream` after them */);

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

/* ---- ALS training: one half-epoch of libreco/algorithms/_als.pyx als_update (:47-93) ---------
 * Solves every row m of X [n_x, d] in place against the fixed table Y [n_y, d] (both contiguous) given that
 * side's CSR (indptr int64 [n_x+1], indices int32, data float32).  A0 [d, d] is the base matrix: Y^T Y + reg I
 * (implicit, task "ranking") or reg I (explicit, "rating"), float32, built by the caller.
 * Row plan (built once per CSR): rows with at most b200_als_long_row_threshold() nnz are listed in
 * short_rows; the others in long_rows, split into chunks of b200_als_chunk() nnz: chunk c covers nnz
 * [indptr[row] + chunk_k[c] * chunk, ...) of row long_rows[chunk_long[c]], and long_chunk_ptr[n_long+1]
 * delimits each long row's chunks.  n_short + n_long == n_x.  workspace: b200_als_workspace_bytes(),
 * 16-byte aligned.  Supported: 1 <= d <= 128, any nnz per row; anything else returns -2 before a launch.
 * Deterministic (no float atomics).
 *   b200_als_cg      _least_squares_cg (:167-268): cg_steps >= 0 CG iterations warm-started from X[m], with the
 *                    reference's exits (rsold < 1e-10 leaves X[m] untouched; rsnew < 1e-10 breaks).  Rows of
 *                    at most b200_als_stage_rows(d) nnz read their Y slice from shared memory.
 *   b200_als_direct  _least_squares (:96-164): A = A0 + sum w y y^T, b = sum c y, Cholesky solve.  A row whose
 *                    pivot at column j is <= 0 or NaN is not written; *fail_row / *fail_info receive the
 *                    smallest such row and its LAPACK info j+1 (-1 / 0: none).  Synchronises the stream. */
int b200_als_long_row_threshold(void);
int b200_als_chunk(void);
int b200_als_stage_rows(int32_t d);
int b200_als_workspace_bytes(int32_t d, int32_t use_cg, int64_t n_long, int64_t n_chunks, size_t* bytes);
int b200_als_cg(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_x, float* X,
                const float* Y, int64_t n_y, int32_t d, const float* A0, int32_t implicit, int32_t cg_steps,
                const int32_t* short_rows, int64_t n_short, const int32_t* long_rows, const int64_t* long_chunk_ptr,
                int64_t n_long, const int32_t* chunk_long, const int32_t* chunk_k, int64_t n_chunks,
                void* workspace, size_t workspace_bytes, void* stream);
int b200_als_direct(const int64_t* indptr, const int32_t* indices, const float* data, int64_t n_x, float* X,
                    const float* Y, int64_t n_y, int32_t d, const float* A0, int32_t implicit,
                    const int32_t* short_rows, int64_t n_short, const int32_t* long_rows,
                    const int64_t* long_chunk_ptr, int64_t n_long, const int32_t* chunk_long,
                    const int32_t* chunk_k, int64_t n_chunks, void* workspace, size_t workspace_bytes,
                    int64_t* fail_row, int32_t* fail_info, void* stream);

/* ---- BPR training: one epoch of libreco/algorithms/_bpr.pyx bpr_update (:30-110, :116-399) ---------------
 * Tables U [n_users, D], I [n_items, D], D = embed_size + 1 (bias last; U[:, D-1] == 1 is never written), all
 * contiguous float32.  For each of the n samples (users[s], items_pos[s]) in order: a negative, then the
 * reference's update, diff = U[u] . (I[p] - I[n]) over all D columns, g = 1 / (1 + exp(diff)), gradient ascent with
 * reg on every updated element.  optimizer: 0 sgd (_bpr_update_sgd :116-190), 1 momentum (:196-280; state1 =
 * velocity tables), 2 adam (:286-399; state1 / state2 = first / second moment tables, bias correction
 * 1 - rho^epoch from the caller's epoch >= 1).  State tables not used by the optimizer may be NULL.
 * Negatives: items_neg[s] when items_neg is given; otherwise uniform over the items not in the user's CSR row
 * (indptr int64 [n_users+1], indices int32, rows sorted and duplicate-free), one Philox4x32-10 draw keyed by
 * (seed, epoch, s) and rank selection.  A user whose row holds every item is skipped.  neg_out (optional)
 * receives the negatives used (-1: skipped).  Updates are atomic adds of deltas; max_inflight bounds the
 * samples in flight (1: serial, deterministic, the sequential reference semantics; 0: the library default,
 * b200_bpr_default_inflight()).  embed_size outside 1..128, null required pointers, an unknown optimizer or
 * missing state return -2 before a launch. */
int64_t b200_bpr_default_inflight(int32_t embed_size);
int b200_bpr_update(int32_t optimizer, const int32_t* users, const int32_t* items_pos, int64_t n,
                    const int64_t* indptr, const int32_t* indices, int64_t n_users, int64_t n_items, float* U,
                    float* I, int32_t embed_size, float* u_state1, float* i_state1, float* u_state2,
                    float* i_state2, float lr, float reg, float momentum, float rho1, float rho2, int32_t epoch,
                    uint64_t seed, const int32_t* items_neg, int32_t* neg_out, int64_t max_inflight,
                    void* stream);

/* ---- Skip-gram training: gensim Word2Vec(sg=1) as Item2Vec / DeepWalk call it -----------------------------
 * (libreco/bases/gensim_base.py:65-70 training, algorithms/item2vec.py:70-83 hs=0 negative=5,
 * algorithms/deepwalk.py:96-126 hs=1 negative=5 and the Python random walks).  A corpus is a sentence CSR
 * (indptr int64 [S+1], tokens int32 item ids, at most 10 000 tokens per sentence).  Every random draw is one
 * Philox4x32-10 keyed by (seed, pass, position) only, never by the launch shape: pass 0 is DeepWalk's vocabulary
 * walk set, training epoch e (from 1) is pass e.
 *   b200_skipgram_subsample  replaces gensim's per-token downsampling: raw token t of item w is kept when the
 *                            draw's first word is < keep_thr[w] (uint64 per item, 2^32 = always).  The kept tokens
 *                            of sentence s are compacted in place: kept_tokens[indptr[s] + k], k < kept_len[s];
 *                            kept_sent[q] is the sentence of slot q or -1 for an empty slot.  keep_out (optional,
 *                            uint8 [T]) records every decision.
 *   b200_skipgram_epoch      one epoch of skip-gram SGD over the compacted corpus (n_tokens = indptr[S] slots)
 *                            into syn0 / syn1neg [n_items, d] and, with hs = 1, syn1 [V-1, d] along each item's
 *                            Huffman path (hs_ptr int64 [n_items+1] into hs_points int32 / hs_codes int8, root
 *                            first).  Negatives: bisect_left(neg_cum, r) for r uniform in [0, cum_last), cum_last =
 *                            neg_cum[vocab_size-1], mapped to an item by neg_items; neg_guide [guide_buckets+1]
 *                            holds bisect_left(neg_cum, k * ceil(cum_last / guide_buckets)).  alpha of sentence s
 *                            = alpha0 - (alpha0 - min_alpha) min(1, (words_before + indptr[s]) / words_total).
 *                            window_out (optional, int32 [T]) records each centre's reduced window b; neg_out
 *                            (optional, int32 [T, 2 window + 1, negative]) each negative draw by (slot, context
 *                            offset + window, draw).  max_inflight bounds the centres in flight (1: serial,
 *                            deterministic, the sequential semantics; 0: b200_skipgram_default_inflight(d), but at most
 *                            n_tokens / 256, at least 1).
 *   b200_item_walks          replaces deepwalk.py:116-126: walk w = round * n_items + start item, each step
 *                            uniform over the node's out-edges (graph CSR with multiplicity), stopping at
 *                            walk_length tokens or a sink.  Call it twice: with lengths (int64 [n_walks n_items])
 *                            to size the walks, then with their prefix sum in indptr to write tokens.
 * d outside 1..128, window outside 1..4096, negative outside 1..16, bad sizes or null required pointers return -2
 * before a launch. */
int64_t b200_skipgram_default_inflight(int32_t d);
int b200_skipgram_subsample(const int64_t* indptr, const int32_t* tokens, int64_t n_sentences, int64_t n_items,
                            const uint64_t* keep_thr, uint64_t seed, int64_t pass, int32_t* kept_tokens,
                            int32_t* kept_sent, int32_t* kept_len, uint8_t* keep_out, void* stream);
int b200_skipgram_epoch(const int64_t* indptr, int64_t n_sentences, const int32_t* kept_tokens,
                        const int32_t* kept_sent, const int32_t* kept_len, int64_t n_tokens, int64_t n_items,
                        float* syn0, float* syn1neg, float* syn1, int32_t d, int32_t hs, const int64_t* hs_ptr,
                        const int32_t* hs_points, const int8_t* hs_codes, const uint32_t* neg_cum,
                        const int32_t* neg_items, int64_t vocab_size, uint32_t cum_last, const int32_t* neg_guide,
                        int64_t guide_buckets, int32_t window, int32_t negative, double alpha0, double min_alpha,
                        double words_before, double words_total, uint64_t seed, int64_t pass, int32_t* window_out,
                        int32_t* neg_out, int64_t max_inflight, void* stream);
int b200_item_walks(const int64_t* graph_indptr, const int32_t* graph_dst, int64_t n_items, int32_t n_walks,
                    int32_t walk_length, uint64_t seed, int64_t pass, int64_t* lengths, const int64_t* indptr,
                    int32_t* tokens, void* stream);

/* ---- GraphSage / PinSage inference (libreco/bases/sage_base.py:136-173, non-DGL) --------------------------
 * The graph is two CSRs built from the reference's dicts with list order and multiplicity kept: item_consumed
 * (item_ptr int64 [n_items+1], item_users int32) and user_consumed (user_ptr int64 [n_users+1], user_items int32).
 * A sampling call covers one level: nodes int32 [n] (n = n_roots * per_root, node r belongs to roots[r / per_root]
 * at path r % per_root; level 0: the roots themselves, per_root 1); level l+1 is the flattened output of level l with
 * per_root * num_neighbors.  Every draw is Philox4x32-10 keyed by (seed, root, path, level, draw index), never by the
 * batch.  A node id < 0 gives an empty row (-1 ids, weight 0, length 0).
 *   b200_sage_neighbors     replaces bipartite_neighbors (libreco/sampling/random_walks.py:48-76): out int32
 *                           [n, num_neighbors], each slot one-walks item -> consumer -> item with the reference's
 *                           rejection rules (5 redraws while self or taken, 5 while self, then accept).
 *   b200_pinsage_neighbors  replaces bipartite_neighbors_with_weights (random_walks.py:79-147) with items_pos =
 *                           None: num_walks walks of at most walk_len one-walks, step s > 0 taken when the draw's
 *                           word is >= cont_threshold (ceil(termination_prob 2^32)); the target removed, the top
 *                           num_neighbors visits by count (ties: first visit), weight count / kept total.  out_ids
 *                           int32 / out_weights float [n, num_neighbors], padded with -1 / 0; out_lens int32 [n].
 *   b200_sage_aggregate     the per-layer input of the w_linears (graphsage_module.py:136-149,
 *                           pinsage_module.py:79-97): out[r] = [S[self_idx ? self_idx[r] : r] (zeros for an index < 0),
 *                           sum_j w_j N[nb_idx ? nb_idx[j] : j]] over row r's neighbour rows j = start .. start + len:
 *                           start = nb_offsets[r] (or r * nb_stride), len = nb_lens[r] when given, else
 *                           nb_offsets[r+1] - start (or nb_stride).  w_j = nb_weights[j], or 1 / len without weights
 *                           (embedding_bag "mean"; an empty bag gives zeros).  out [n_rows, ldo >= 2 d].
 * num_neighbors outside 1..32, num_walks * walk_len outside 1..256, d outside 1..128, bad sizes or null required
 * pointers return -2 before a launch. */
int b200_sage_neighbors(const int64_t* item_ptr, const int32_t* item_users, const int64_t* user_ptr,
                        const int32_t* user_items, const int32_t* roots, const int32_t* nodes, int64_t n,
                        int64_t per_root, int32_t level, int32_t num_neighbors, uint64_t seed, int32_t* out,
                        void* stream);
int b200_pinsage_neighbors(const int64_t* item_ptr, const int32_t* item_users, const int64_t* user_ptr,
                           const int32_t* user_items, const int32_t* roots, const int32_t* nodes, int64_t n,
                           int64_t per_root, int32_t level, int32_t num_neighbors, int32_t num_walks,
                           int32_t walk_len, uint64_t cont_threshold, uint64_t seed, int32_t* out_ids,
                           float* out_weights, int32_t* out_lens, void* stream);
int b200_sage_aggregate(const float* S, int64_t lds, const int32_t* self_idx, int64_t n_rows, const float* N,
                        int64_t ldn, const int32_t* nb_idx, const int64_t* nb_offsets, const int32_t* nb_lens,
                        int32_t nb_stride, const float* nb_weights, int32_t d, float* out, int64_t ldo,
                        void* stream);

/* GraphSage training (the non-DGL GraphSageModel, libreco/algorithms/torch_modules/graphsage_module.py:82-140, and
 * GraphCollator, libreco/batch/collators.py:338-386):
 *   b200_sage_aggregate_backward  backward of b200_sage_aggregate in mean mode (no weights), the bags read as there:
 *                           dout [n_rows, ldo >= 2 d] is d loss / d [self | mean] of each row; dout[r, :d] is ADDED
 *                           into dS[self_idx ? self_idx[r] : r] (skipped for an index < 0) and dout[r, d:] / len into
 *                           dN[nb_idx ? nb_idx[j] : j] for each neighbour j of row r (ids < 0 and empty bags add
 *                           nothing).  Both buffers accumulate (+=): zero them first.  A hidden level gets gradient as
 *                           the self input of one layer and as the neighbours of the level above it, so the caller
 *                           adds both calls into one buffer.  No float atomics: the self rows must be distinct over r,
 *                           and so must the neighbour rows (the sampler's layout: num_neighbors consecutive rows per
 *                           node, one parent each).  The result is then bit-identical from run to run.
 *   b200_sage_walk_pairs    pairs_from_random_walk (libreco/sampling/random_walks.py:21-41) for n_starts start items
 *                           drawn uniformly on the device (starts int32 [n_starts]): per start, the (v, v) pair when no
 *                           consumer of v has another item (has_no_neighbor), then num_walks walks of walk_length
 *                           one-walks; one-walk cur -> next gives (cur, next) when next != cur, or with focus_start
 *                           (v, next) when next != v.  Order: start, walk, step.  Draws: Philox4x32-10 keyed by
 *                           (seed, step, start index, walk * walk_length + step in walk).  Two calls: the count pass
 *                           (items == NULL) writes starts, counts int64 [n_starts (num_walks + 1)] and their exclusive
 *                           prefix sum offsets int64 [n_starts (num_walks + 1) + 1] (the last entry: the number of
 *                           pairs); the fill pass (same arguments, items / items_pos int32 [total]) writes the pairs.
 *                           Every item must have a consumer.  num_walks / walk_length outside 1..1024 return -2.
 *   b200_sage_i2i_negatives negatives_from_random with items (libreco/sampling/negatives.py:17-31): out int32 [n num_neg],
 *                           negatives of pair j at out[j num_neg ..]; uniform over n_items, a draw equal to items[j] or
 *                           items_pos[j] is drawn again up to `tolerance` times; keyed by (seed, step, slot, attempt).
 * d outside 1..128, bad sizes or null required pointers return -2 before a launch. */
int b200_sage_aggregate_backward(const float* dout, int64_t ldo, const int32_t* self_idx, int64_t n_rows, float* dS,
                                 int64_t lds, const int32_t* nb_idx, const int64_t* nb_offsets, const int32_t* nb_lens,
                                 int32_t nb_stride, int32_t d, float* dN, int64_t ldn, void* stream);
int b200_sage_walk_pairs(const int64_t* item_ptr, const int32_t* item_users, const int64_t* user_ptr,
                         const int32_t* user_items, int64_t n_items, int64_t n_starts, int32_t num_walks,
                         int32_t walk_length, int32_t focus_start, uint64_t seed, uint64_t step, int32_t* starts,
                         int64_t* counts, int64_t* offsets, int32_t* items, int32_t* items_pos, void* stream);
int b200_sage_i2i_negatives(const int32_t* items, const int32_t* items_pos, int64_t n, int32_t num_neg,
                            int64_t n_items, int32_t tolerance, uint64_t seed, uint64_t step, int32_t* out,
                            void* stream);

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
 * scoring (outputs are indexed by the local r).  R = 0 launches nothing (users / items may then be NULL).
 * Any output may be NULL:
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
 * Wt is the TRANSPOSED kernel [dout, din]; fp32 SIMT (exact fma chain in k).  act is an activation code:
 * 0 none, 1 relu, 2 swish x / (1 + expf(-x)) (layers/activation.py:10-11); any other value returns -2. */
int b200_linear_f32(const float* X, int64_t ldx, int64_t R, const float* Wt, int64_t ldw,
                    const float* bias, int32_t din, int32_t dout, int32_t act, float* Y,
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
                       const float* Wsplit, const float* bias, int32_t din, int32_t dout, int32_t act,
                       float* Y, int64_t ldy, void* stream);

/* Split-K form for products with few output tiles and a long reduction (the weight gradients dWt = dY^T X of
 * the training steps: 1792 x 128 outputs over 8192 rows = 14 tiles): `splits` CTAs along the reduction per
 * output tile write partial products into workspace (splits * R * dout floats), a second kernel adds them in a
 * fixed order (+ bias, activation).  splits == 1 is b200_linear_tf32x3 without a pre-split weight copy. */
int b200_linear_tf32x3_splitk(const float* X, int64_t ldx, int64_t R, const float* Wt, int64_t ldw, const float* bias,
                              int32_t din, int32_t dout, int32_t act, int32_t splits, float* workspace,
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
 * Max-margin ties follow torch's clamp_min: a pair exactly on the hinge (margin == pos - neg) has loss 0
 * and gradient -1/n_neg w.r.t. pos (TF's relu would give 0 there).
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
/* SIM's dual sequences (libreco/batch/sequence.py:94-147, get_dual_seqs; batch/collators.py:114-116) with the same
 * position rule p and the same draw stream: short = the s = min(p, S) items before p, long = the up to L items before
 * those (none when p <= S), each padded with pad_index, lengths max(count, 1).  A user with no items gets p = 0 (two
 * all-pad rows of length 1), where the reference raises. */
int b200_interacted_dual_seqs(const int64_t* indptr, const int32_t* idx, int64_t n_users, const int64_t* users,
                              const int64_t* items, int64_t n, int32_t long_max_len, int32_t short_max_len,
                              int32_t pad_index, const int64_t* rand_pos, uint64_t seed, uint64_t step,
                              int32_t* long_seqs, int32_t* long_lens, int32_t* short_seqs, int32_t* short_lens,
                              void* stream);

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

/* ---- Transformer inference (libreco/algorithms/transformer.py:203-339, layers/transformer.py) --------
 * G [n_items+1, Kp] is the item feature table (combine_seq_features), pos [T, Kpos] the positional table,
 * D = Kp + Kpos.  Slot s encodes the sequence seqs[users[s], :T] with len = lens[s] (clamped to [0, T]):
 *   X = [G[seq_t] || pos_t];  per layer:  a = MHA(rms_att(X)) + X;  X = a + gelu_erf(rms_ffn(a) W1) W2;
 *   S[s] = rms_last(X)  [T, D]  (S: [n_slots, T, D] contiguous).
 * rms(x) = x / sqrt(mean(x^2) + 1e-8) * scale.  MHA: num_heads heads of D / num_heads columns, no biases, scores
 * <q, k> / sqrt(hd); key k is visible to query q when k < len, or k <= q with `causal` (the reference ORs the two
 * masks); a hidden score becomes fl32(score - 1e9).  weights: per layer rms_att [D], Wq, Wk, Wv, Wo [D, D] (Wv the
 * EFFECTIVE value map), rms_ffn [D], W1 [D, 4D], W2 [4D, D], row-major; rms_last [D].  Every dot product is one
 * fmaf chain over an ascending index; the softmax is max, expf, an ascending sum, then a division.
 * Supported: 1 <= T <= 64, 1 <= D <= 128, 1 <= n_layers <= 4, num_heads dividing D; anything else returns -2
 * before launching.
 * b200_transformer_pair_scores: scores[b * lds + n] for every slot b < B and item n < N:
 *   p = softmax_t(<Qi[n], S[b, t]>) over t < lens[b] (over all T with every score - 1e9 when lens[b] = 0),
 *   h1 = swish(Pu[b] + Pi[n] + sum_t p_t Vp[b*T + t]),  h2 = h1 W2 + b2,
 *   H3 > 0: out = <swish(h2) W3 + b3, w_out> + b_out;  H3 = 0: out = <h2, w_out> + b_out.
 * Qi [N, ldq] = [rms_item(G[n]) || 1..1], Vp [B*T, H1] = S W1_seq, Pu [B, H1] (first-layer bias included),
 * Pi [N, ldpi], W2 [H1, H2], W3 [H2, H3] (row-major, BN folded).  Supported: H1 <= 256, H2 <= 64, H3 <= 32,
 * B <= 65535 and b200_transformer_pair_smem_bytes(T, D, H1) within the device's shared-memory opt-in.
 * b200_transformer_target_attention: out[r, :D] = sum_t p_t S[slot, t] for row r, slot = slot_of_row[r] and
 * item = items[r] (explicit rows) or, both NULL, row g = row_offset + r of the grid: slot g / grid_items, item
 * g % grid_items. */
int b200_transformer_encode(const int64_t* users, int64_t n_slots, const int32_t* lens, const int32_t* seqs,
                            int64_t ld_seq, const float* G, int64_t ldg, int32_t Kp, const float* pos, int32_t Kpos,
                            int32_t T, int32_t num_heads, int32_t n_layers, int32_t causal, const float* weights,
                            const float* rms_last, float* S, void* stream);
int64_t b200_transformer_pair_smem_bytes(int32_t T, int32_t D, int32_t H1);
int b200_transformer_pair_scores(const float* Qi, int64_t ldq, int64_t N, const float* S, const float* Vp,
                                 const float* Pu, const int32_t* lens, int64_t B, const float* Pi, int64_t ldpi,
                                 int32_t T, int32_t D, int32_t H1, int32_t H2, int32_t H3, const float* W2,
                                 const float* b2, const float* W3, const float* b3, const float* w_out, float b_out,
                                 float* scores, int64_t lds, void* stream);
int b200_transformer_target_attention(const float* Qi, int64_t ldq, const float* S, int32_t T, int32_t D,
                                      const int32_t* lens, const int32_t* slot_of_row, const int64_t* items, int64_t n,
                                      int64_t grid_items, int64_t row_offset, float* out, int64_t ldo, void* stream);

/* ---- SIM inference (libreco/algorithms/sim.py:193-304, soft search; the second stage only) --------------------
 * Gp [N+1, ldg] is the projected item table combine_seq_features(concat) Wp, K columns.  A slot s has the long
 * sequence long_seqs[s, :L] with length long_lens[s] and the short one short_seqs[s, :S] with short_lens[s] (both
 * clamped to [0, L] / [0, S]); Kl, Vl [n_slots, L, K] are Gp[long] Wk and Gp[long] Wv (Wv the EFFECTIVE value map).
 * For a pair (slot s, item n), q = Gp[n]:
 *   GSU (sim.py:264-286): score_t = q . Gp[long_t] for t < long_len, -1e9 otherwise; the topk largest are selected,
 *       equal scores resolving to the lower position.  Every score is acc = fmaf(q[d], Gp[long_t][d], acc) over d
 *       ascending from 0 in both functions, so both select the same positions.
 *   ESU (sim.py:288-299): per head h of K / H columns, logits (Qp[n]_h . Kl[t]_h) / sqrt(K / H) over the selected t,
 *       fl32(logit - 1e9) where t >= long_len; o_h = sum p_t Vl[t]_h; long_out = o Wo.
 *   short (sim.py:301-304): logits q . Gp[short_s], fl32(logit - 1e9) where s >= short_len; short_out =
 *       (sum_s e_s Gp[short_s]) / sum_s e_s with e_s = exp(logit_s - max).
 * Supported: 1 <= K <= 64 with H dividing K, 1 <= L <= 256, 1 <= S <= 64, 1 <= topk <= min(32, L); anything else
 * returns -2 before launching.
 * b200_sim_attention (rows mode): out[r, :K] = long_out, out[r, K:2K] = short_out for row r, slot = slot_of_row[r]
 * and item = items[r] (explicit rows) or, both NULL, row g = row_offset + r of the grid: slot g / grid_items, item
 * g % grid_items.  Qp [N+1, ldq] = Gp Wq, Wo [K, K].  gsu_pos (NULL: not written) [n, topk] receives the selected
 * positions in ascending order.
 * b200_sim_pair_scores (grid mode): scores[b * lds + n] for every slot b < B and item n < N:
 *   h1 = relu(Pu[b] + PiT[:, n] + [o || short_out] W_att),  h2 = h1 W2 + b2,
 *   H3 > 0: out = <relu(h2) W3 + b3, w_out> + b_out;  H3 = 0: out = <h2, w_out> + b_out.
 * GpT, QpT [K, ldt] hold Gp and Qp transposed (column n = item n); W_att [2K, H1] = [Wo W1_long ; W1_short],
 * Pu [B, H1] (first-layer bias included), PiT [H1, ldpi], W2 [H1, H2], W3 [H2, H3] (row-major, BN folded).
 * Supported: H1 <= 256, H2 <= 128, H3 <= 64, B <= 65535 and b200_sim_pair_smem_bytes(...) within the device's
 * shared-memory opt-in. */
int b200_sim_attention(const float* Gp, int64_t ldg, const float* Qp, int64_t ldq, int32_t K, int32_t H,
                       const int32_t* long_seqs, int64_t ld_long, const int32_t* long_lens, const float* Kl,
                       const float* Vl, int32_t L, const int32_t* short_seqs, int64_t ld_short,
                       const int32_t* short_lens, int32_t S, int32_t topk, const float* Wo,
                       const int32_t* slot_of_row, const int64_t* items, int64_t n, int64_t grid_items,
                       int64_t row_offset, float* out, int64_t ldo, int32_t* gsu_pos, void* stream);
int64_t b200_sim_pair_smem_bytes(int32_t K, int32_t L, int32_t S, int32_t topk, int32_t H1, int32_t H2, int32_t H3);
int b200_sim_pair_scores(const float* GpT, const float* QpT, int64_t ldt, int64_t N, const float* Gp, int64_t ldg,
                         const int32_t* long_seqs, int64_t ld_long, const int32_t* long_lens,
                         const int32_t* short_seqs, int64_t ld_short, const int32_t* short_lens, const float* Kl,
                         const float* Vl, const float* Pu, int64_t B, const float* PiT, int64_t ldpi, int32_t K,
                         int32_t H, int32_t L, int32_t S, int32_t topk, int32_t H1, int32_t H2, int32_t H3,
                         const float* W_att, const float* W2, const float* b2, const float* W3, const float* b3,
                         const float* w_out, float b_out, float* scores, int64_t lds, void* stream);

/* ---- SIM training (libreco/algorithms/sim.py:193-304, training mode) -------------------------------------------
 * Row r carries its own long sequence long_seqs[r, :L] (length long_lens[r]) and target item items[r]; Gp as above.
 * b200_sim_gsu_forward: one warp per row.  sel_pos [R, topk] receives the GSU positions in ascending order, selected
 *   by the very code of b200_sim_attention (same scores, same tie rule: the same positions bit for bit on the same
 *   Gp and sequence), pooled [R, ldp] (K columns) the first stage's sum_{t < long_len} Gp[long_t] over t ascending
 *   (long_len clamped to [0, L]; pad ids inside the length are summed).
 * b200_sim_esu_forward: per head h of hd = K / H columns, one query Q[r] over its topk selected keys
 *   Ksel / Vsel [R * topk, ldkv] (row r * topk + i = the i-th selected position): logits (Q_h . Ksel_h) / sqrt(hd) as
 *   one fmaf chain, p = softmax over the visible keys, O[r]_h = sum_i p_i Vsel_h (i ascending).  Key i is visible when
 *   sel_pos[r, i] < max(long_lens[r], 1); a hidden key gets probability exactly 0.  P [R, H, topk] is saved.
 * b200_sim_esu_backward: WRITES dQ [R, lddq], dKsel and dVsel [R * topk, lddkv] from dO and the saved P; hidden keys'
 *   rows are exact zeros.  Both: one warp per (row, head), no atomics, bit-identical repeats.
 * b200_sim_long_backward: ADDS (float atomics) dpooled[r] into dGp[long_seqs[r, t]] for t < long_len and
 *   dXsel[r * topk + i] into dGp[long_seqs[r, sel_pos[r, i]]].
 * Supported: 1 <= K <= 64 (H dividing K), 1 <= L <= 256, 1 <= topk <= min(32, L); anything else returns -2 before
 * launching. */
int b200_sim_gsu_forward(const float* Gp, int64_t ldg, int32_t K, const int64_t* items, const int32_t* long_seqs,
                         int64_t ld_long, const int32_t* long_lens, int32_t L, int32_t topk, int64_t R,
                         int32_t* sel_pos, float* pooled, int64_t ldp, void* stream);
int b200_sim_esu_forward(const float* Q, int64_t ldq, const float* Ksel, const float* Vsel, int64_t ldkv,
                         const int32_t* sel_pos, const int32_t* long_lens, int64_t R, int32_t K, int32_t H,
                         int32_t topk, float* O, int64_t ldo, float* P, void* stream);
int b200_sim_esu_backward(const float* Q, int64_t ldq, const float* Ksel, const float* Vsel, int64_t ldkv,
                          const int32_t* sel_pos, const int32_t* long_lens, int64_t R, int32_t K, int32_t H,
                          int32_t topk, const float* P, const float* dO, int64_t lddo, float* dQ, int64_t lddq,
                          float* dKsel, float* dVsel, int64_t lddkv, void* stream);
int b200_sim_long_backward(const int32_t* long_seqs, int64_t ld_long, const int32_t* long_lens, int32_t L,
                           const int32_t* sel_pos, int32_t topk, int64_t R, int32_t K, const float* dpooled,
                           int64_t ldp, const float* dXsel, int64_t ldx, float* dGp, int64_t ldg, void* stream);

/* ---- Transformer training (libreco/algorithms/transformer.py:203-339 in training mode) ------------------------
 * The dense products over the R*T sequence rows (Q / K / V / O projections, FFN, MLP and their gradients) run on
 * b200_linear_*; these are the rest.  Every `lens` here is clamped to [1, T] on the device, as the training
 * collator gives it (position 0 of a history is len 1 holding the pad id): key 0 is always visible.
 * b200_transformer_attention_forward / _backward: the attention core of b200_autoint_attention_* (same layouts,
 * Q, K, V, O [R*T, ld], lse [R, H, T], dQ / dK / dV WRITTEN, one warp per (row, head), no atomics, bit-identical
 * repeats) with a mask: key g is visible to query f of row r when g < lens[r], or g <= f with `causal`; a hidden
 * key gets probability exactly 0.  Supported: 1 <= T <= 64, num_heads, head_dim >= 1, num_heads * head_dim <= 128,
 * every stride >= that product, a finite scale; anything else returns -2 before launching.  The backward needs
 * (6 T odd(hd) + 32 odd(T)) * 4 bytes of shared memory per (row, head): 206 464 B at T = 64, hd = 128.
 * b200_rms_norm_forward: Y = X * rstd * scale per row of width D, rstd[r] = rsqrt(mean(X[r]^2) + 1e-8) saved.
 * b200_rms_norm_backward: dX = rstd (dY o scale - X rstd^2 <dY o scale, X> / D).  The scale's gradient
 * sum_r rstd[r] dY[r, c] X[r, c] is b200_col_reduce(dY, wrow = rstd, Y = X).
 * b200_activation_forward / _backward: y = act(x), dx = dy * act'(x) elementwise over n floats from the
 * pre-activation x; act 1 relu, 2 swish x / (1 + exp(-x)), 3 gelu 0.5 x (1 + erf(x / sqrt 2)).
 * b200_transformer_target_attention_backward: the backward of b200_transformer_target_attention with one slot per
 * row (query Q[r], sequence S[r] = S + r T D, [T, D] contiguous): p = softmax_t(<q, S_t>) over t < len,
 * out = sum_t p_t S_t recomputed, ds_t = p_t (<dout, S_t> - <dout, out>); WRITES dq[r] = sum_t ds_t S_t and
 * dS[r, t] = p_t dout + ds_t q for t < len, 0 for t >= len.  One warp per row, no atomics.
 * Supported: 1 <= T <= 64, 1 <= D <= 128. */
int b200_transformer_attention_forward(const float* Q, int64_t ldq, const float* K, int64_t ldk, const float* V,
                                       int64_t ldv, const int32_t* lens, int64_t R, int32_t T, int32_t num_heads,
                                       int32_t head_dim, int32_t causal, float scale, float* O, int64_t ldo, float* lse,
                                       void* stream);
int b200_transformer_attention_backward(const float* Q, int64_t ldq, const float* K, int64_t ldk, const float* V,
                                        int64_t ldv, const float* O, int64_t ldo, const float* lse, const float* dO,
                                        int64_t lddo, const int32_t* lens, int64_t R, int32_t T, int32_t num_heads,
                                        int32_t head_dim, int32_t causal, float scale, float* dQ, float* dK, float* dV,
                                        int64_t ldg, void* stream);
int b200_rms_norm_forward(const float* X, int64_t ldx, int64_t R, int32_t D, const float* scale, float* Y, int64_t ldy,
                          float* rstd, void* stream);
int b200_rms_norm_backward(const float* dY, int64_t lddy, const float* X, int64_t ldx, const float* rstd, int64_t R,
                           int32_t D, const float* scale, float* dX, int64_t lddx, void* stream);
int b200_activation_forward(const float* x, int64_t n, int32_t act, float* y, void* stream);
int b200_activation_backward(const float* dy, const float* x, int64_t n, int32_t act, float* dx, void* stream);
int b200_transformer_target_attention_backward(const float* Q, int64_t ldq, const float* S, int32_t T, int32_t D,
                                               const int32_t* lens, const float* dout, int64_t lddo, int64_t R,
                                               float* dq, int64_t lddq, float* dS, void* stream);

/* ---- RNN4Rec inference (libreco/algorithms/rnn4rec.py:151-237, layers/recurrent.py:4-63) ----------------------
 * Slot s encodes the sequence seqs[users[s], :T] (row-major, ld_seq) with len = lens[users[s]] clamped to [0, T]
 * over the input table X [*, ldx] (seq_embeds, in_dim columns) through n_layers stacked recurrent layers and
 * writes out[s, :H_last] (ldo): the last layer's state after step len - 1.  Steps t >= len leave every state
 * unchanged and len = 0 gives the zero state (dynamic_rnn(sequence_length=len); the Keras graph with a mask when
 * masked steps repeat the previous output).  Layer l (input width in_l = l ? hidden[l-1] : in_dim, hidden size H,
 * G gates) has cell_kinds[l]:
 *   0 GRU reset-after (Keras), blocks z | r | h:  h~ = act(ax_h + r * ah_h),  h' = z h + (1 - z) h~
 *   1 GRU reset-before (TF1 GRUCell), blocks z | r | c:  c = act(ax_c + (r o h) . U_c + bh_c),  h' = z h + (1 - z) c
 *   2 LSTM, blocks i | f | c | o:  c' = f c + i act(ax_c + ah_c),  h' = o act(c')
 * with ax_g = x . W_g + bx_g and ah_g = h . U_g + bh_g, each dot product one fmaf chain over the index ascending,
 * and z, r, i, f, o = sigmoid(ax_g + ah_g) = 1 / (1 + expf(-v)).  acts[l]: 0 act = tanhf; 1 act = identity and the
 * layer's output is tanh(LayerNorm(h)) (eps 1e-3, mean and variance over H), which is the next layer's input and,
 * for the last layer, the result.  weights packs the layers back to back, each W [in_l, G*H], U [H, G*H],
 * bx [G*H], bh [G*H], gamma [H], beta [H] row-major (b200_rnn_layer_floats floats; gamma / beta are read only when
 * acts[l] = 1).  cell_kinds, hidden and acts are HOST arrays of n_layers entries.  A slot's result depends only on
 * its own sequence: the same bits whatever the other slots, n or the call.
 * Supported: 1 <= T <= 128, 1 <= in_dim, hidden[l] <= 256, 1 <= n_layers <= 4; anything else returns -2 before
 * launching; n = 0 launches nothing. */
int64_t b200_rnn_layer_floats(int32_t cell_kind, int32_t in_dim, int32_t hidden);
int b200_rnn_encode(const int64_t* users, int64_t n, const int32_t* lens, const int32_t* seqs, int64_t ld_seq,
                    int32_t T, const float* X, int64_t ldx, int32_t in_dim, int32_t n_layers, const int32_t* cell_kinds,
                    const int32_t* hidden, const int32_t* acts, const float* weights, float* out, int64_t ldo,
                    void* stream);

/* ---- RNN4Rec training (rnn4rec.py:151-237 in training mode, no dropout) ------------------------------------------
 * b200_rnn_train_forward: b200_rnn_encode (the same out, bit for bit) that also saves what the backward needs.
 * saved is a HOST array of 6 * n_layers device pointers; layer l's six tensors have n * T rows, row s * T + t:
 *   [0] h_{t-1} [H]   [1] the layer output y_t [H] (h_t, or tanh(LayerNorm(h_t)))   [2] the post-activation gates
 *   [G*H] (z | r | h~, z | r | c, i | f | c~ | o)   [3] LSTM c_t, Keras GRU U_c h_{t-1} + bh_c, TF1 GRU r o h_{t-1}
 *   [H]   [4] x^ = (h_t - mean) rstd [H] and [5] rstd [1] (acts[l] = 1 only; NULL otherwise).
 * Rows t >= len are 0.  Same envelope and errors as b200_rnn_encode.
 * b200_rnn_backward: one layer's backward through time.  The layer (cell_kind, input width in_dim, hidden, act,
 * layer_weights = its packed weights) reads its six saved tensors (saved: HOST array of 6 device pointers) and ONE of
 * dout [n, lddo] (top layer: the gradient of the encoder output, taken at step len - 1) or dy [n * T, hidden] (the
 * gradient of the layer's outputs y_t).  It WRITES, rows s * T + t, dgx [n * T, G*H] = d loss / d (x W + bx) per
 * gate and, for the Keras GRU only, dgh [n * T, G*H] = d loss / d (h U + bh) (the candidate block scaled by r); for
 * the other cells the h part equals dgx (TF1 GRU: the candidate block acts on r o h_{t-1}).  With act = 1 it also
 * writes dln = dy (1 - y^2) and dlnx = dln x^ [n * T, hidden] (beta / gamma column sums); a len-0 row of the top
 * layer writes its dln (through tanh(beta)) at t = 0.  Rows t >= len are otherwise 0.  No atomics.  Supported as
 * b200_rnn_encode: 1 <= T <= 128, 1 <= in_dim, hidden <= 256; anything else returns -2 before launching; n = 0
 * launches nothing. */
int b200_rnn_train_forward(const int64_t* users, int64_t n, const int32_t* lens, const int32_t* seqs, int64_t ld_seq,
                           int32_t T, const float* X, int64_t ldx, int32_t in_dim, int32_t n_layers,
                           const int32_t* cell_kinds, const int32_t* hidden, const int32_t* acts, const float* weights,
                           float* out, int64_t ldo, float* const* saved, void* stream);
int b200_rnn_backward(const int64_t* users, int64_t n, const int32_t* lens, int32_t T, int32_t cell_kind,
                      int32_t in_dim, int32_t hidden, int32_t act, const float* layer_weights, const float* dout,
                      int64_t lddo, const float* dy, const float* const* saved, float* dgx, float* dgh, float* dln,
                      float* dlnx, void* stream);

/* ---- Caser / WaveNet inference (libreco/algorithms/caser.py:177-221, wave_net.py:181-222) ----------------------
 * Slot s reads the sequence seqs[users[s], :T] (row-major, ld_seq; pad positions are ordinary rows: neither model
 * masks by length) and x = X[seq] [T, K] (X = seq_embeds [*, ldx]).  Every pre-activation below is ONE fmaf chain
 * that starts at the bias and runs over the terms in the order written; max and ReLU are order-free.  A slot's
 * result depends only on its own sequence: the same bits whatever the other slots, n or the call.
 * b200_caser_encode writes out[s, :T*nh + K*nv] (ldo), the concat the Dense head reads:
 *   column (h-1)*nh + f, h = 1..T:  max_{p <= T-h} relu(b_h[f] + sum_{j<h} sum_{k<K} x[p+j, k] W_h[j, k, f]),
 *                                    j ascending, then k ascending (Conv1D(nh, h, valid, relu) + MaxPool1D);
 *   column T*nh + k*nv + f:          relu(bv[f] + sum_{t<T} x[t, k] Wv[t, f]), t ascending (Conv1D(nv, 1) over x^T).
 * weights packs W_1 .. W_T ([h, K, nh] each, Keras layout) back to back, then b_h [T, nh], Wv [T, nv], bv [nv]
 * (b200_caser_weight_floats floats).
 * b200_wavenet_encode runs n_conv causal layers Conv1D(F, 2, causal, dilation d_l = dilations[l], relu) (C_in = K
 * for the first layer, F after):  y[t, f] = relu(b[f] + sum_c x[t-d, c] W[0, c, f] + sum_c x[t, c] W[1, c, f]),
 * the first sum (c ascending, absent while t < d) before the second (c ascending); then the 1x1 layer
 * z[t, f] = relu(b1[f] + sum_c y[t, c] W1[c, f]) (c ascending), and writes out[s, f] = max_t z[t, f] (ldo).
 * weights packs per causal layer W [2, C_in, F], b [F], then W1 [F, F], b1 [F] (b200_wavenet_weight_floats
 * floats).  dilations is a HOST array of n_conv entries.
 * Supported: 1 <= T <= 64, 1 <= K <= 128, 1 <= nh, nv <= 32, 1 <= F <= 128, 1 <= n_conv <= 16, dilations >= 1;
 * anything else returns -2 before launching (the weight-float helpers too); n = 0 launches nothing. */
int64_t b200_caser_weight_floats(int32_t T, int32_t K, int32_t nh, int32_t nv);
int64_t b200_wavenet_weight_floats(int32_t K, int32_t F, int32_t n_conv);
int b200_caser_encode(const int64_t* users, int64_t n, const int32_t* seqs, int64_t ld_seq, int32_t T, const float* X,
                      int64_t ldx, int32_t K, int32_t nh, int32_t nv, const float* weights, float* out, int64_t ldo,
                      void* stream);
int b200_wavenet_encode(const int64_t* users, int64_t n, const int32_t* seqs, int64_t ld_seq, int32_t T,
                        const float* X, int64_t ldx, int32_t K, int32_t n_conv, int32_t F, const int32_t* dilations,
                        const float* weights, float* out, int64_t ldo, void* stream);

/* ---- Caser / WaveNet training (caser.py:135-221, wave_net.py:139-222 in training mode) ---------------------------
 * b200_caser_train_forward / b200_wavenet_train_forward: b200_caser_encode / b200_wavenet_encode (the same out, bit
 * for bit) that also save what the backward needs.  argmax is a max-pool's argmax: the LOWEST position reaching the
 * maximum, or -1 when the maximum is <= 0 (the ReLU then passes no gradient).  Caser: argmax [n, T*nh] (column
 * (h-1)*nh + f, a window start p in [0, T-h]).  WaveNet: layer_out [n_conv, n * T, F] (causal layer l's output y_l at
 * row s * T + t of block l) and argmax [n, F] over t of the 1x1 layer.  Same envelope and errors as the encoders.
 * b200_caser_backward: given dF [n, T*nh + K*nv] (lddf) = d loss / d out, the features feat (ldfe) and argmax of the
 * training forward, the gathered input rows X [n * T, ldx] (row s * T + t = seq_embeds[seq[s, t]]) and the packed
 * weights, WRITES dX [n * T, lddx] and dW (b200_caser_weight_floats floats, the packed layout of weights).  A
 * horizontal column routes g = dF to its argmax window (nothing for -1); a vertical column passes g = dF where
 * feat > 0.  dX[s, t, k] = sum over (h ascending, f ascending) with p* <= t < p* + h of g W_h[t - p*, k, f], then
 * sum_f (ascending) gv[k, f] Wv[t, f].  dW: each chunk of rows is summed in row order into workspace
 * (b200_caser_backward_workspace_floats(n, ...) floats), then the chunks in a fixed order (b200_col_reduce).  No
 * atomics: a repeated call gives the same bits.
 * b200_wavenet_pool_backward: dZ [n * T, F] = dF[s, f] at t = argmax[s, f], 0 elsewhere (the 1x1 layer's max).
 * b200_wavenet_layer_inputs: out [n * T, 2C] = [x[s*T + t - d] (0 for t < d) | x[s*T + t]], so that one dense
 * product with a causal layer's kernel [2, C, F] seen as [2C, F] gives its pre-activation, and its transpose the
 * kernel gradient.
 * b200_wavenet_layer_dx: given P = dpre [2, C, F]^T [n * T, 2C], dx[s*T + t, c] = P[s*T + t, C + c] +
 * P[s*T + t + d, c] (the second term while t + d < T, for every dilation up to INT32_MAX).
 * Supported: the encoders' envelope (C <= 128, dilation >= 1 for the layer helpers); anything else returns -2
 * before launching; n = 0 launches nothing. */
int b200_caser_train_forward(const int64_t* users, int64_t n, const int32_t* seqs, int64_t ld_seq, int32_t T,
                             const float* X, int64_t ldx, int32_t K, int32_t nh, int32_t nv, const float* weights,
                             float* out, int64_t ldo, int32_t* argmax, void* stream);
int b200_wavenet_train_forward(const int64_t* users, int64_t n, const int32_t* seqs, int64_t ld_seq, int32_t T,
                               const float* X, int64_t ldx, int32_t K, int32_t n_conv, int32_t F,
                               const int32_t* dilations, const float* weights, float* out, int64_t ldo,
                               float* layer_out, int32_t* argmax, void* stream);
int64_t b200_caser_backward_workspace_floats(int64_t n, int32_t T, int32_t K, int32_t nh, int32_t nv);
int b200_caser_backward(int64_t n, int32_t T, int32_t K, int32_t nh, int32_t nv, const float* dF, int64_t lddf,
                        const float* feat, int64_t ldfe, const int32_t* argmax, const float* X, int64_t ldx,
                        const float* weights, float* dX, int64_t lddx, float* dW, float* workspace,
                        int64_t workspace_floats, void* stream);
int b200_wavenet_pool_backward(int64_t n, int32_t T, int32_t F, const float* dF, int64_t lddf, const int32_t* argmax,
                               float* dZ, void* stream);
int b200_wavenet_layer_inputs(const float* x, int64_t ldx, int64_t n, int32_t T, int32_t C, int32_t dilation,
                              float* out, void* stream);
int b200_wavenet_layer_dx(const float* P, int64_t n, int32_t T, int32_t C, int32_t dilation, float* dx, int64_t lddx,
                          void* stream);

/* ---- a14: predict_from_embedding (libreco/prediction/predict.py:36-40) -----------------
 * out[r] = sum_k U[users[r],k] * I[items[r],k]; mode 0: raw, 1: expit (ranking),
 * 2: clip to [lo, hi] (rating) — normalize_prediction (:18-23). */
int b200_gather_dot(const float* U, int64_t ldu, const int64_t* users, const float* I,
                    int64_t ldi, const int64_t* items, int64_t n, int32_t d, int32_t mode,
                    float lo, float hi, float* out, void* stream);

/* ---- Swing (libreco/algorithms/swing.py; recfarm rust/src/graph.rs, swing.rs, inference.rs) -------------------
 * The graph: R, the user x item CSR of train_data.sparse_interaction (user_ptr int64 [n_users+1], user_items int32,
 * user_labels float), and R^T (item_ptr int64 [n_items+1], item_users int32); rows sorted and duplicate-free.
 *   b200_swing_scores   replaces compute_swing_scores (graph.rs:147-234): w_u = 1 / sqrt(|I_u|); for each item i and
 *                       users u < v of row i of R^T, C = I_u ∩ I_v, the term (w_u * w_v) * (alpha + |C| - 1)^-1 (fp32,
 *                       the reference's rounding) is added to score_i[j] for every j in C, j != i.  Out: nbr_ids int32 /
 *                       nbr_scores float [n_items, top_k], item i's top_k nonzero scores by (score desc, id asc),
 *                       padded with -1 / 0, and nbr_count int64 [n_items], its number of nonzero scores (what
 *                       swing.rs:150-151 sums).  Sums run in atomic order: repeated calls may differ in the last
 *                       bits.  Synchronises `stream` (the task plan is built on the host from item_ptr).  top_k
 *                       outside 1..4096, a catalogue whose bitmap does not fit in shared memory (n_items above
 *                       about 1.8 M at top_k 20, 1.6 M at top_k 4096), a negative or non-finite alpha return -2 before a launch.
 *   b200_swing_plan     which accumulator the scores kernel uses for n_items (1: shared memory, 0: one global row
 *                       per resident CTA) and how many CTAs it keeps resident.
 *   Recommend and predict are b200_nbr_recommend (item-based), b200_nbr_random_keys and b200_nbr_predict (task 1,
 *                       ranking: swing.rs:153-185) on the Swing neighbour table over R. */
int b200_swing_scores_workspace_bytes(int64_t n_users, int64_t n_items, int32_t top_k, size_t* bytes);
int b200_swing_scores(const int64_t* user_ptr, const int32_t* user_items, int64_t n_users, const int64_t* item_ptr,
                      const int32_t* item_users, int64_t n_items, float alpha, int32_t top_k, int32_t* nbr_ids,
                      float* nbr_scores, int64_t* nbr_count, void* workspace, size_t workspace_bytes, void* stream);
int b200_swing_plan(int64_t n_items, int32_t top_k, int32_t* smem_acc, int32_t* ctas);

/* ---- UserCF / ItemCF (libreco/bases/cf_base_rs.py; recfarm rust/src/similarities.rs, item_cf.rs, user_cf.rs,
 * inference.rs) ---------------------------------------------------------------------------------------------------
 * The "sim side" S (sim_ptr int64 [n_x+1], sim_idx int32, sim_val float) is the CSR whose rows are compared:
 * item_interactions (R^T) for ItemCF, user_interactions (R) for UserCF; the "middle" M (mid_*) is its transpose.  Rows
 * sorted and duplicate-free.
 *   b200_cf_cosine      replaces compute_similarities (similarities.rs): sq[x] = sum of r^2 over row x of S (fp32, row
 *                       order); for each x1 and x2 != x1 sharing count >= min_common middle rows p, cosine =
 *                       prod / (sqrt(sq1) * sqrt(sq2)) with prod = sum of r[x1,p] * r[x2,p], or 0 if prod, sq1 or sq2
 *                       is 0 (fp32, the reference's expression; only the order of the prod sum differs).  Zero and
 *                       negative cosines are kept.  Out: nbr_ids int32 / nbr_scores float [n_x, k_sim], row x1's
 *                       first k_sim kept entries by (cosine desc, id asc), padded with -1 / 0, and nbr_count int64
 *                       [n_x], its kept count (what num_sim_elements sums).  Synchronises `stream` (the task plan is
 *                       built on the host).  k_sim outside 1..4096 or min_common < 1 return -2 before a launch.
 *   b200_cf_cosine_workspace_bytes  its workspace: (4 + 8) n_x bytes of row state, 4 n_x bytes per resident CTA
 *                       (touched lists), 8 n_x more per resident CTA when the accumulator rows do not fit in shared
 *                       memory (n_x above about 28.7 k at k_sim 20), and 12 n_x per split slot (64 slots).
 *   b200_cf_plan        which accumulator b200_cf_cosine uses for n_x (1: shared memory, 0: one global row per
 *                       resident CTA) and how many CTAs it keeps resident.
 *   Recommend and predict are b200_nbr_recommend (ItemCF item-based: item_cf.rs:156-209; UserCF
 *                       user-based: user_cf.rs:151-205), b200_nbr_random_keys and b200_nbr_predict (the engine's
 *                       task; ItemCF: rows = users over R, queries = items; UserCF: rows = items over R^T, queries =
 *                       users) on the neighbour table, with top_k = k_sim. */
int b200_cf_cosine_workspace_bytes(int64_t n_x, int32_t k_sim, size_t* bytes);
int b200_cf_plan(int64_t n_x, int32_t k_sim, int32_t* smem_acc, int32_t* ctas);
int b200_cf_cosine(const int64_t* sim_ptr, const int32_t* sim_idx, const float* sim_val, int64_t n_x,
                   const int64_t* mid_ptr, const int32_t* mid_idx, const float* mid_val, int64_t n_y,
                   int64_t min_common, int32_t k_sim, int32_t* nbr_ids, float* nbr_scores, int64_t* nbr_count,
                   void* workspace, size_t workspace_bytes, void* stream);

/* ---- Neighbourhood serving (recfarm rust/src/swing.rs, item_cf.rs, user_cf.rs, inference.rs) ----------------------
 * A neighbour table is nbr_ids int32 / nbr_scores float [n, top_k] and nbr_count int64 [n] (b200_swing_scores,
 * b200_cf_cosine): row q's first min(top_k, nbr_count[q]) entries are its neighbours.
 *   b200_nbr_recommend  row r (user u = users[r]) of scores [B, ld] gets, unless filter_consumed and the item is in
 *                       the consumed CSR's row u (always, not b200_mask_consumed's rule):
 *                       user_based 0 (Swing, ItemCF: the table is over items): for every (i, label) of row u of R and
 *                       each of i's neighbours (j, s), s * label added at j;
 *                       user_based 1 (UserCF: the table is over users): for each of u's neighbours (v, sim) and each
 *                       (i, label) of row v of R, sim * label added at i.
 *                       Items that got no term hold REMOVED, so b200_topk_rows ranks them last; counts[r] is the
 *                       number that got one (the candidates).  A user outside [0, n_users) gets an all-REMOVED row
 *                       and count 0.
 *   b200_nbr_random_keys  random_rec (inference.rs:78-86): a row with more than n_rec candidates gets a uniform
 *                       key in [1, 2) at each candidate, Philox4x32-10 keyed by (seed, user, item); b200_topk_rows
 *                       then draws n_rec distinct candidates.
 *   b200_nbr_predict    predict with compute_pred (inference.rs:48-71): query q's neighbours intersected with row r of
 *                       the sorted CSR (ptr, idx, labels); task 0 (rating) gives sum(label * sim / sum(sims)) per
 *                       term (a zero sum of sims gives NaN or inf, as in the reference), task 1 (ranking)
 *                       sum(sims) / n and reads no labels (labels may be null).  default_pred for an id outside range or an empty
 *                       intersection. */
int b200_nbr_recommend(const int64_t* user_ptr, const int32_t* user_items, const float* user_labels, int64_t n_users,
                       const int32_t* nbr_ids, const float* nbr_scores, const int64_t* nbr_count, int64_t n_items,
                       int32_t top_k, int32_t user_based, const int64_t* consumed_ptr, const int32_t* consumed_idx,
                       int32_t filter_consumed, const int64_t* users, int64_t B, float* scores, int64_t ld,
                       int64_t* counts, void* stream);
int b200_nbr_random_keys(float* scores, int64_t ld, int64_t B, int64_t n_items, const int64_t* users,
                         const int64_t* counts, int32_t n_rec, uint64_t seed, void* stream);
int b200_nbr_predict(const int64_t* ptr, const int32_t* idx, const float* labels, int64_t n_rows,
                     const int32_t* nbr_ids, const float* nbr_scores, const int64_t* nbr_count, int64_t n_queries,
                     int32_t top_k, const int64_t* rows, const int64_t* queries, int64_t n, int32_t task,
                     float default_pred, float* out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200RECO_H_ */
