"""GPU parity of the BENCHMARKED branch of the fused scorer: shapes whose plan enables the
speculative pre-pass (``sweep_kernel<PRE>`` + ``guess_kernel`` + the status-3 check in
``finalize_kernel``) — C2's catalogue size (1 M items, d = 64, top-100, Zipf consumed lists with
500-item users), a wider embedding with a ragged last tile / short last split, embeddings far from
unit scale, and the kernel-organisation variants (cluster multicast on / off, MMA groups, epilogue).

Contract (reference: libreco/recommendation/recommend.py:57-78 + ranking.py:10-56):
* rows the fused path accepts (status 0) equal the exact materialised path BIT FOR BIT (ids and
  fp32 scores: same exact-score definition, same tie rule);
* every row, after the exact-path repair of flagged rows, equals the exact path;
* against the numpy oracle (OpenBLAS sgemm) ids may differ only inside near-ties
  (<= 1e-6 relative score gap) and the returned scores agree to 1e-5 relative.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _tables(seed, n_users, N, d, u_scale=1.0, i_scale=1.0):
    rng = np.random.default_rng(seed)
    U = rng.standard_normal((n_users + 1, d)).astype(np.float32)
    I = rng.standard_normal((N + 1, d)).astype(np.float32)
    U /= np.linalg.norm(U, axis=1, keepdims=True)
    I /= np.linalg.norm(I, axis=1, keepdims=True)
    return (U * np.float32(u_scale)), (I * np.float32(i_scale))


def _zipf_consumed(seed, n_users, N, mean_c=50, cap=500, heavy_every=97):
    """bench.py's consumed model (SURVEY 8d C2): c_u ~ min(Poisson(mean), cap) distinct items drawn
    Zipf(1.0)-like (log-uniform ranks over a fixed permutation); every `heavy_every`-th user gets the
    full `cap` items.  Returns the CSR arrays."""
    from librecommender_b200.consumed import ConsumedCSR

    rng = np.random.default_rng(seed)
    counts = np.minimum(rng.poisson(mean_c, size=n_users), cap).astype(np.int64)
    counts[::heavy_every] = cap
    perm = rng.permutation(N)
    owner = np.repeat(np.arange(n_users, dtype=np.int64), counts)
    rank = np.minimum((np.exp(rng.random(len(owner)) * np.log(N)) - 1).astype(np.int64), N - 1)
    key = np.unique(owner * N + perm[rank])                       # sorted, duplicates inside a user removed
    owner, item = key // N, (key % N).astype(np.int32)
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    np.cumsum(np.bincount(owner, minlength=n_users), out=indptr[1:])
    return ConsumedCSR(indptr, item)


def _check(sc, U, I, csr, users, K, n_oracle, min_ok_frac):
    import torch
    from oracle import ranking as orc

    N = sc.n_items
    uid = torch.as_tensor(users).cuda()
    ids_f, sc_f, status = sc.recommend_fused(uid, K, True, True)
    ids_e, sc_e = sc.recommend_exact(uid, K, True, True)
    torch.cuda.synchronize()
    status = status.cpu().numpy()
    ok = status == 0
    codes = {int(c): int((status == c).sum()) for c in np.unique(status)}
    assert ok.mean() >= min_ok_frac, codes
    ids_f, sc_f, ids_e, sc_e = (t.cpu().numpy() for t in (ids_f, sc_f, ids_e, sc_e))
    np.testing.assert_array_equal(ids_f[ok], ids_e[ok])
    np.testing.assert_array_equal(sc_f[ok], sc_e[ok])
    assert (ids_f[~ok] == -1).all()
    # the public device call repairs the flagged rows on the exact path
    got_ids, got_sc = sc.recommend_device(uid, K, True, True)
    np.testing.assert_array_equal(got_ids.cpu().numpy(), ids_e)
    np.testing.assert_array_equal(got_sc.cpu().numpy(), sc_e)
    # numpy oracle on a sample of the rows (heavy users first)
    known = np.minimum(users, csr.n_users - 1)
    deg = np.where(users < csr.n_users, csr.indptr[known + 1] - csr.indptr[known], 0)   # OOV row: no history
    pick = np.unique(np.concatenate([np.argsort(-deg)[: n_oracle // 4],
                                     np.random.default_rng(0).choice(len(users), n_oracle, replace=False)]))
    u_s = users[pick]
    consumed = {int(u): csr.row(int(u)).tolist() for u in u_s if u < csr.n_users and len(csr.row(int(u)))}
    ref_ids, ref_sc = orc.recommend_from_embedding("rating", u_s.tolist(), K, U, I, N, consumed, True,
                                                   return_scores=True)
    full = orc.embed_scores(U, I, u_s, N)
    assert orc.near_tie_mask(ref_ids, ids_e[pick], full, 1e-6).all()
    assert (ids_e[pick] == ref_ids).mean() > 0.995
    scale = np.abs(full).max(axis=1, keepdims=True)
    assert (np.abs(sc_e[pick] - ref_sc) <= 1e-5 * scale).all()
    for r, u in zip(pick, u_s):
        assert not set(ids_e[r].tolist()) & set(consumed.get(int(u), []))
    return codes


@pytest.mark.parametrize("B", [1024, 8192])
def test_c2_shape_speculative_path(B):
    """1 M items, d = 64, top-100 — the shape and the branch bench.py measures."""
    from librecommender_b200.engine import EmbedScorer

    n_users, N, d, K = 100_000, 1_000_000, 64, 100
    U, I = _tables(7, n_users, N, d)
    csr = _zipf_consumed(3, n_users, N)
    sc = EmbedScorer(U, I, N, csr, n_users=n_users)
    plan = sc.fused_plan(B, K)
    assert plan["use_pre"] == 1, plan                    # the speculative branch is the one under test
    users = np.random.default_rng(4).choice(n_users, size=B, replace=False).astype(np.int64)
    users[:3] = [0, 97, n_users]                          # two 500-item users and the OOV row
    codes = _check(sc, U, I, csr, users, K, n_oracle=64 if B > 2048 else 128, min_ok_frac=0.97)
    print("status codes", codes, "plan", plan)


def test_wide_embedding_ragged_catalogue_and_scale():
    """d = 128 (two K blocks), N not a multiple of the 256-item tile, rows far from unit scale
    (the fp16 operands are rescaled per row / per table by powers of two)."""
    from librecommender_b200.engine import EmbedScorer

    n_users, N, d, K = 20_000, 800_003, 128, 50
    U, I = _tables(11, n_users, N, d, u_scale=37.5, i_scale=1.0e-3)
    U[5] *= 1.0e4                                         # per-row scales differ by orders of magnitude
    U[6] *= 1.0e-4
    csr = _zipf_consumed(5, n_users, N, mean_c=20, cap=150)
    sc = EmbedScorer(U, I, N, csr, n_users=n_users)
    B = 2048
    plan = sc.fused_plan(B, K)
    assert plan["use_pre"] == 1, plan
    users = np.random.default_rng(9).choice(n_users, size=B, replace=False).astype(np.int64)
    users[:3] = [5, 6, n_users]
    _check(sc, U, I, csr, users, K, n_oracle=96, min_ok_frac=0.97)


@pytest.mark.parametrize("code", [113, 215, 223, 125, 115, 225, 213, 123])
def test_kernel_organisation_variants(code):
    """The tuning variants of the sweep give the same answers as the default (code 215: cluster of 2 with
    TMA multicast, one N=256 MMA group per tile, predicated record stores): no cluster (1xx), two
    N=128 MMA groups per tile (x2x), divergent per-group record stores (xx3)."""
    from librecommender_b200 import _lib
    from librecommender_b200.engine import EmbedScorer

    n_users, N, d, K = 30_000, 600_000, 64, 100
    U, I = _tables(13, n_users, N, d)
    csr = _zipf_consumed(6, n_users, N)
    sc = EmbedScorer(U, I, N, csr, n_users=n_users)
    users = np.random.default_rng(2).choice(n_users, size=2048, replace=False).astype(np.int64)
    try:
        _lib.check(_lib.lib.b200_recommend_embed_tune(code, 0.0))
        plan = sc.fused_plan(len(users), K)
        assert plan["use_pre"] == 1 and plan["cluster_x10_plus_mma_groups"] == code // 10, plan
        _check(sc, U, I, csr, users, K, n_oracle=64, min_ok_frac=0.97)
    finally:
        _lib.check(_lib.lib.b200_recommend_embed_tune(215, 0.0))
