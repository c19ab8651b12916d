"""GPU tests of the fused scorer's speculative threshold (b200_recommend_embed_speculation: pre-pass
stride and failure budget delta of the rank pre_k; b200_recommend_embed_tune's linear rule):

* the benchmarked shape (1 M items, d = 64, top-100, 32 768 users per launch, Zipf consumed lists with
  500-item users) under the default rule: failed speculation (status 3) within the budget, every row
  equal to the exact path after the repair;
* stride and delta at the ends of their ranges;
* an adversarial catalogue whose best items all sit in the sampled tiles: most rows fail the
  speculation check (status 3, or 2 when the guess leaves fewer than k_row items) and every one is
  repaired exactly;
* the linear rule of the former default (stride 16, pre_k = 12 + ceil(2 f k_row)) is still accepted.
Every test sets the rule it needs and restores the default afterwards.
"""
import numpy as np
import pytest

from test_gpu_fused_c2 import _tables, _zipf_consumed

pytestmark = pytest.mark.gpu


def _run(sc, uid, K, filt, stride=0, delta=0.0, legacy=False):
    """(ids, scores, status) of the fused call and (ids, scores) of the repaired device path."""
    import torch
    from librecommender_b200 import _lib

    try:
        _lib.check(_lib.lib.b200_recommend_embed_speculation(stride, delta))
        if legacy:
            _lib.check(_lib.lib.b200_recommend_embed_tune(0, 2.0))
            _lib.check(_lib.lib.b200_recommend_embed_debug(-12))
        plan = sc.fused_plan(len(uid), K)
        ids_f, sc_f, status = sc.recommend_fused(uid, K, filt, True)
        ids_d, sc_d = sc.recommend_device(uid, K, filt, True)
        torch.cuda.synchronize()
    finally:
        _lib.check(_lib.lib.b200_recommend_embed_speculation(0, 0.0))
    return plan, tuple(t.cpu().numpy() for t in (ids_f, sc_f, status, ids_d, sc_d))


def _exact(sc, uid, K, filt):
    import torch

    ids_e, sc_e = sc.recommend_exact(uid, K, filt, True)
    torch.cuda.synchronize()
    return ids_e.cpu().numpy(), sc_e.cpu().numpy()


def _assert_exact(got, exact):
    ids_f, sc_f, status, ids_d, sc_d = got
    ids_e, sc_e = exact
    ok = status == 0
    np.testing.assert_array_equal(ids_f[ok], ids_e[ok])
    np.testing.assert_array_equal(sc_f[ok], sc_e[ok])
    assert (ids_f[~ok] == -1).all()
    np.testing.assert_array_equal(ids_d, ids_e)
    np.testing.assert_array_equal(sc_d, sc_e)


def _codes(status):
    return {int(c): int((status == c).sum()) for c in np.unique(status)}


@pytest.fixture(scope="module")
def bench_shape():
    import torch
    from librecommender_b200.engine import EmbedScorer

    n_users, N, d, K, B = 100_000, 1_000_000, 64, 100, 32768
    U, I = _tables(61, n_users, N, d)
    csr = _zipf_consumed(62, n_users, N)
    sc = EmbedScorer(U, I, N, csr, n_users=n_users)
    users = np.random.default_rng(63).choice(n_users, size=B, replace=False).astype(np.int64)
    users[:2] = [0, 97]                                    # two 500-item users
    uid = torch.as_tensor(users).cuda()
    return sc, uid, K, _exact(sc, uid, K, True)


def test_bench_shape_default_rule(bench_shape):
    sc, uid, K, exact = bench_shape
    plan, got = _run(sc, uid, K, True)
    assert plan["use_pre"] == 1, plan
    status = got[2]
    # delta = 1e-5 per row: about 0.3 expected failures in 32 768 rows; 8 leaves room for the tie allowance.
    # Every 97th user of this fixture consumed 500 items (k_row capped at 288): some of those rows overflow a
    # candidate list (status 1) whatever the rule, as in test_gpu_fused_pipelined's bench shape.
    assert (status == 3).sum() <= 8, _codes(status)
    assert (status == 0).mean() >= 0.97, _codes(status)
    _assert_exact(got, exact)


@pytest.mark.parametrize("stride, delta", [(2, 1e-9), (2, 1e-2), (32, 1e-9), (32, 1e-2), (4, 1e-5)])
def test_stride_and_budget_extremes(bench_shape, stride, delta):
    sc, uid, K, exact = bench_shape
    n = 8192
    plan, got = _run(sc, uid[:n], K, True, stride, delta)
    n_pre = -(-plan["tiles_per_split"] // stride)
    assert plan["n_pre_tiles"] == n_pre
    assert plan["use_pre"] == int(2 * plan["n_splits"] * n_pre >= 256)
    status = got[2]
    budget = delta * n if plan["use_pre"] else 0.0
    assert (status == 3).sum() <= budget + 4 * np.sqrt(budget) + 8, _codes(status)
    assert (status == 0).mean() >= 0.97, _codes(status)
    _assert_exact(got, tuple(e[:n] for e in exact))


def test_legacy_linear_rule_still_accepted(bench_shape):
    sc, uid, K, exact = bench_shape
    n = 8192
    plan, got = _run(sc, uid[:n], K, True, 16, 0.0, legacy=True)
    assert plan["use_pre"] == 1
    assert (got[2] == 0).mean() >= 0.97, _codes(got[2])
    _assert_exact(got, tuple(e[:n] for e in exact))


def test_adversarial_catalogue_top_items_in_sampled_tiles():
    """Every sampled tile holds items 1.5x longer than the rest, so each row's best items sit in the
    sampled tiles, the pre_k-th sampled block maximum lies above c_k - 2 eps and finalize rejects the guess."""
    import torch
    from librecommender_b200.engine import EmbedScorer

    n_users, N, d, K, B, stride = 20_000, 1_000_000, 64, 100, 8192, 8
    U, I = _tables(71, n_users, N, d)
    import ctypes

    from librecommender_b200 import _lib

    out = (ctypes.c_int32 * 10)()
    try:
        _lib.check(_lib.lib.b200_recommend_embed_speculation(stride, 0.0))
        _lib.check(_lib.lib.b200_recommend_embed_plan(B, N, d, K, out, 10))
    finally:
        _lib.check(_lib.lib.b200_recommend_embed_speculation(0, 0.0))
    n_splits, tps = int(out[1]), int(out[2])
    assert out[0] == 1 and out[8] == stride
    tiles = np.arange(-(-N // 256))
    sampled = tiles[(tiles - (tiles // tps) * tps) % stride == 0]
    rows = (sampled[:, None] * 256 + np.arange(256)[None, :]).ravel()
    rows = rows[rows < N]
    I[rows] *= np.float32(1.5)
    sc = EmbedScorer(U, I, N, None, n_users=n_users)
    uid = torch.as_tensor(np.random.default_rng(72).choice(n_users, size=B, replace=False).astype(np.int64)).cuda()
    plan, got = _run(sc, uid, K, False, stride, 0.0)
    assert plan["use_pre"] == 1 and plan["n_splits"] == n_splits
    status = got[2]
    # the guess lies above c_k - 2 eps: status 3, or status 2 when it is above c_k and fewer than k_row
    # items were collected
    assert np.isin(status, (2, 3)).mean() >= 0.5, _codes(status)
    _assert_exact(got, _exact(sc, uid, K, False))
