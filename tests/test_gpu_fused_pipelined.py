"""GPU tests of the fused scorer's pipelined MMA organisation (tune codes x3x: two N=128 MMA groups per
item tile, the MMAs of one half-tile running under the epilogue of the other, across item tiles).

* the one-hot-slot catalogue of test_gpu_fused_slots: every record slot, both lists, both CTAs of a
  cluster and the partial last tile, bit for bit against the exact path with status 0 on every row;
* the benchmarked shape (1 M items, d = 64, top-100, 32 768 users per launch, Zipf consumed lists with
  500-item users): one item split per row, so the threshold history does not depend on timing and ids,
  scores and row_status must equal the unpipelined default organisation's (215) bit for bit;
* forced compactions during the pipeline (low speculative threshold): exact after the repair;
* unit edges (several item splits with a one-tile last split, N = 257, N = 1, B not a multiple of the
  user tile) and embedding widths 65, 128 and 192 (d > 128 runs one N=256 group: the plan says so).
"""
import ctypes

import numpy as np
import pytest

from test_gpu_fused_c2 import _tables, _zipf_consumed
from test_gpu_fused_slots import D as SLOT_D, K as SLOT_K, N as SLOT_N, N_USERS as SLOT_USERS, _catalogue

pytestmark = pytest.mark.gpu

CODES = [235, 233, 135, 133]
DEFAULT_COEF, DEFAULT_MARGIN = 2.0, 12   # b200_recommend_embed_tune / _debug defaults


def _plan(B, N, d, K):
    from librecommender_b200 import _lib

    out = (ctypes.c_int32 * 8)()
    _lib.check(_lib.lib.b200_recommend_embed_plan(B, N, d, K, out, 8))
    return [int(v) for v in out]


def _fused(sc, uid, K, filt, code, coef=0.0, margin=None):
    """(ids, scores, status) of the fused path and of the repaired device path under organisation `code`."""
    import torch
    from librecommender_b200 import _lib

    try:
        _lib.check(_lib.lib.b200_recommend_embed_tune(code, coef))
        if margin is not None:
            _lib.check(_lib.lib.b200_recommend_embed_debug(-margin))
        ids_f, sc_f, status = sc.recommend_fused(uid, K, filt, True)
        ids_d, sc_d = sc.recommend_device(uid, K, filt, True)
        torch.cuda.synchronize()
    finally:
        _lib.check(_lib.lib.b200_recommend_embed_tune(215, DEFAULT_COEF))
        _lib.check(_lib.lib.b200_recommend_embed_debug(-DEFAULT_MARGIN))
    return tuple(t.cpu().numpy() for t in (ids_f, sc_f, status, ids_d, sc_d))


def _exact(sc, uid, K, filt):
    import torch

    ids_e, sc_e = sc.recommend_exact(uid, K, filt, True)
    torch.cuda.synchronize()
    return ids_e.cpu().numpy(), sc_e.cpu().numpy()


def _assert_exact(got, exact, min_ok_frac):
    ids_f, sc_f, status, ids_d, sc_d = got
    ids_e, sc_e = exact
    ok = status == 0
    assert ok.mean() >= min_ok_frac, {int(c): int((status == c).sum()) for c in np.unique(status)}
    np.testing.assert_array_equal(ids_f[ok], ids_e[ok])
    np.testing.assert_array_equal(sc_f[ok], sc_e[ok])
    assert (ids_f[~ok] == -1).all()
    np.testing.assert_array_equal(ids_d, ids_e)
    np.testing.assert_array_equal(sc_d, sc_e)


# ---------------------------------------------------------------- one hot group per record slot
@pytest.fixture(scope="module")
def slots():
    from librecommender_b200.engine import EmbedScorer

    use_pre, n_splits, tiles_per_split = _plan(SLOT_USERS, SLOT_N, SLOT_D, SLOT_K)[:3]
    assert use_pre == 1
    U, I, planted, sel = _catalogue(n_splits, tiles_per_split)
    return EmbedScorer(U, I, SLOT_N, None, n_users=SLOT_USERS), planted[sel][:, ::-1]


@pytest.mark.parametrize("code", CODES)
def test_one_hot_group_per_slot(slots, code):
    import torch

    sc, expected = slots
    uid = torch.arange(SLOT_USERS, dtype=torch.int64, device="cuda")
    ids_f, sc_f, status, _, _ = _fused(sc, uid, SLOT_K, False, code)
    ids_e, sc_e = _exact(sc, uid, SLOT_K, False)
    assert (status == 0).all(), {int(c): int((status == c).sum()) for c in np.unique(status)}
    np.testing.assert_array_equal(ids_e, expected)
    np.testing.assert_array_equal(ids_f, ids_e)
    np.testing.assert_array_equal(sc_f, sc_e)


# ---------------------------------------------------------------- the benchmarked shape
@pytest.fixture(scope="module")
def bench_shape():
    import torch
    from librecommender_b200.engine import EmbedScorer

    n_users, N, d, K, B = 100_000, 1_000_000, 64, 100, 32768
    U, I = _tables(21, n_users, N, d)
    csr = _zipf_consumed(8, n_users, N)
    sc = EmbedScorer(U, I, N, csr, n_users=n_users)
    users = np.random.default_rng(22).choice(n_users, size=B, replace=False).astype(np.int64)
    users[:2] = [0, 97]                                    # two 500-item users
    uid = torch.as_tensor(users).cuda()
    return sc, uid, K, _fused(sc, uid, K, True, 215), _exact(sc, uid, K, True)


@pytest.mark.parametrize("code", CODES)
def test_bench_shape_equals_unpipelined(bench_shape, code):
    sc, uid, K, base, exact = bench_shape
    plan = sc.fused_plan(len(uid), K)
    assert plan["use_pre"] == 1 and plan["n_splits"] == 1, plan
    got = _fused(sc, uid, K, True, code)
    for a, b in zip(got[:3], base[:3]):                    # ids, scores, row_status of the fused call
        np.testing.assert_array_equal(a, b)
    _assert_exact(got, exact, min_ok_frac=0.97)


@pytest.mark.parametrize("code", CODES)
def test_forced_compactions(bench_shape, code):
    """A low speculative threshold (rank coefficient 16, margin 64) fills the lists, so rows compact
    while the pipeline runs; the result stays exact after the repair."""
    sc, uid, K, _, exact = bench_shape
    n = 8192
    got = _fused(sc, uid[:n], K, True, code, coef=16.0, margin=64)
    _assert_exact(got, tuple(e[:n] for e in exact), min_ok_frac=0.9)


# ---------------------------------------------------------------- unit edges and widths
def _one_tile_last_split(B, d, K):
    """A catalogue size whose plan has several item splits and a last split of a single tile."""
    for tiles in range(40, 400):
        N = tiles * 256 - 100
        use_pre, n_splits, tps = _plan(B, N, d, K)[:3]
        if n_splits > 1 and tiles - (n_splits - 1) * tps == 1:
            return N
    raise AssertionError("no catalogue size with a one-tile last split")


@pytest.mark.parametrize("code", CODES)
@pytest.mark.parametrize("case", ["one_tile_last_split", "N257", "N1"])
def test_unit_edges(code, case):
    import torch
    from librecommender_b200.engine import EmbedScorer

    d, B = 64, 300                                          # B: not a multiple of the 128-row user tile (or 256)
    K = {"one_tile_last_split": 20, "N257": 10, "N1": 1}[case]
    N = {"one_tile_last_split": None, "N257": 257, "N1": 1}[case] or _one_tile_last_split(B, d, K)
    n_users = 2000
    U, I = _tables(31, n_users, N, d)
    csr = _zipf_consumed(9, n_users, N, mean_c=min(10, N // 4), cap=max(0, min(40, N - K)), heavy_every=53) \
        if N > 4 * K else None
    sc = EmbedScorer(U, I, N, csr, n_users=n_users)
    uid = torch.as_tensor(np.random.default_rng(3).choice(n_users, size=B, replace=False).astype(np.int64)).cuda()
    filt = csr is not None
    _assert_exact(_fused(sc, uid, K, filt, code), _exact(sc, uid, K, filt), min_ok_frac=0.97)


@pytest.mark.parametrize("code", CODES)
@pytest.mark.parametrize("d", [65, 128, 192])
def test_embedding_widths(code, d):
    import torch
    from librecommender_b200.engine import EmbedScorer

    n_users, N, K, B = 5000, 300_007, 50, 1024
    U, I = _tables(41 + d, n_users, N, d)
    csr = _zipf_consumed(10, n_users, N, mean_c=20, cap=150)
    sc = EmbedScorer(U, I, N, csr, n_users=n_users)
    uid = torch.as_tensor(np.random.default_rng(5).choice(n_users, size=B, replace=False).astype(np.int64)).cuda()
    from librecommender_b200 import _lib

    try:
        _lib.check(_lib.lib.b200_recommend_embed_tune(code, 0.0))
        groups = sc.fused_plan(B, K)["cluster_x10_plus_mma_groups"]
    finally:
        _lib.check(_lib.lib.b200_recommend_embed_tune(215, 0.0))
    cl = code // 100
    assert groups == 10 * cl + (1 if d > 128 else 3)       # d_pad > 128: one N=256 group per tile
    _assert_exact(_fused(sc, uid, K, True, code), _exact(sc, uid, K, True), min_ok_frac=0.97)
