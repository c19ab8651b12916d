"""The materialised ranking path, each C-ABI entry point called directly and compared with an exact restatement of
its definition (tests/_rank_kernels_ref.py):

* ``b200_score_rows_f32`` and ``b200_gather_dot`` modes 0 / 2 bit for bit against the exact-score definition (one
  float32 ``fmaf`` chain in k order, emulated with correct rounding), mode 1 (sigmoid) within 4 ulp; the fused
  tensor-core path's scores against the same emulation, so the fused == exact tests are anchored to the definition.
* ``b200_topk_rows`` ids exactly and scores bit for bit against the selection order restated on values (REMOVED
  below everything, -0.0 == +0.0, NaN above +inf, ties by id) at K 1 ... 4096 and N from K to 2^20 + 7 (chunks of
  8192), past 65 535 rows (the row-group loop), with ld > N, a null ``out_scores``, ties cut across chunks, constant
  rows and every special value; its workspace size is enough and one byte less is rejected.
* ``b200_mask_consumed`` and ``rank_recommendations`` against the reference's removal: duplicates counted in
  ``n_rec + len(consumed) <= n_items``, ids outside [0, N), OOV users, empty lists, and ``-inf`` / NaN scores on kept
  items that the answer reaches; ``merge_topk_shards`` with real ``-inf`` candidates beside empty slots.
* ``b200_fm_pair_scores`` / ``b200_deepfm_pair_scores`` against float64 past the grid caps (grid-stride loops, the
  DeepFM cp.async double buffer across block iterations), H1 with partial and odd / even counts of 32-column chunks,
  H3 = 0, the zeroed FM block, ``lds > N`` with a guard column, and the size checks.  Bound per element:
  C_PAIR * u * mag, with mag from tests/_rank_kernels_ref.py (calibrated in tests/test_rank_kernels_cpu.py).
"""
from __future__ import annotations

import ctypes

import numpy as np
import pytest

import _rank_kernels_ref as rk

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
C_PAIR = 8.0         # FM / DeepFM pair scores (tests/test_rank_kernels_cpu.py)
SIGMOID_ULP = 4      # 1 / (1 + expf(-x)): expf is within 2 ulp, the add and the division round once each


def _lib():
    from librecommender_b200 import _lib as L

    return L


def _dev(a, dtype=None):
    import torch

    t = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return t if dtype is None else t.to(dtype)


def _sync():
    import torch

    torch.cuda.synchronize()


def _f32_from_bits(b):
    return np.asarray(b, dtype=np.uint32).view(F32)


# =====================================================================================================================
# exact scorer
# =====================================================================================================================
def _score_rows(Uall, uid, Iall, N, d, lds):
    import torch

    L = _lib()
    B = len(uid) if uid is not None else Uall.shape[0]
    Ud, Id = _dev(Uall), _dev(Iall)
    uid_d = _dev(np.asarray(uid, dtype=np.int64)) if uid is not None else None
    out = torch.full((max(B, 1), lds), float("nan"), dtype=torch.float32, device="cuda")
    L.check(L.lib.b200_score_rows_f32(L.ptr(Ud), Ud.stride(0), L.ptr(uid_d), B, L.ptr(Id), Id.stride(0), N, d,
                                      L.ptr(out), lds, L.current_stream()))
    _sync()
    return out.cpu().numpy()[:B]


@pytest.mark.parametrize("d", [1, 7, 8, 9, 63, 64, 65, 129, 256])
def test_score_rows_f32_bit_exact(d):
    rng = np.random.default_rng(d)
    for B, N, with_ids in ((1, 1, False), (127, 129, True), (128, 128, False), (129, 127, True)):
        ldu, ldi = d + 3, d + 5
        n_users = B + 7
        Uall = np.full((n_users, ldu), np.nan, dtype=F32)      # the padding must never be read
        Iall = np.full((N, ldi), np.nan, dtype=F32)
        Uall[:, :d] = rng.standard_normal((n_users, d))
        Iall[:, :d] = rng.standard_normal((N, d))
        uid = rng.integers(0, n_users, B) if with_ids else None
        if with_ids and B > 3:
            uid[1] = uid[2] = uid[0]                            # repeated users
        urows = Uall[uid, :d] if with_ids else Uall[:B, :d]
        lds = N + 9
        got = _score_rows(Uall if with_ids else Uall[:B], uid, Iall, N, d, lds)
        want = rk.dot_chain(urows, Iall[:, :d])
        np.testing.assert_array_equal(rk.bits(got[:, :N]), rk.bits(want), err_msg=f"B={B} N={N} d={d}")
        assert np.isnan(got[:, N:]).all(), "wrote past N"


def test_score_rows_f32_special_rows():
    """Zero rows, products that round to -0.0 (fmaf(tiny, -tiny, +0) is -0.0) and rows that overflow to +-inf."""
    d, N = 9, 6
    Uu = np.zeros((5, d), dtype=F32)
    Uu[1] = 1e-30                                      # products of 1e-60 underflow to -0.0 / +0.0
    Uu[2] = 3e38                                       # partial sums overflow
    Uu[3] = -3e38
    Uu[4, :] = np.float32(1e-20) * np.arange(1, d + 1, dtype=F32)
    It = np.zeros((N, d), dtype=F32)
    It[1] = -1e-30
    It[2] = 1e-30
    It[3] = 3e38
    It[4] = -2.0
    It[5, ::2] = 5e37
    It[5, 1::2] = -5e37
    got = _score_rows(Uu, None, It, N, d, N)
    want = rk.dot_chain(Uu, It)
    np.testing.assert_array_equal(rk.bits(got), rk.bits(want))
    assert rk.bits(want)[1, 1] == 0x80000000, "the case must produce -0.0"
    assert np.isposinf(want[2, 3]) and np.isneginf(want[3, 3]) and np.isneginf(want[2, 4])


def _gather_dot(Uall, users, Iall, items, d, mode, lo=0.0, hi=0.0):
    import torch

    L = _lib()
    Ud, Id = _dev(Uall), _dev(Iall)
    u, i = _dev(np.asarray(users, np.int64)), _dev(np.asarray(items, np.int64))
    out = torch.empty(len(users), dtype=torch.float32, device="cuda")
    L.check(L.lib.b200_gather_dot(L.ptr(Ud), Ud.stride(0), L.ptr(u), L.ptr(Id), Id.stride(0), L.ptr(i), len(users), d,
                                  mode, lo, hi, L.ptr(out), L.current_stream()))
    _sync()
    return out.cpu().numpy()


@pytest.mark.parametrize("d", [1, 16, 65])
def test_gather_dot_modes(d):
    rng = np.random.default_rng(300 + d)
    n = 1000                                           # four blocks of 256, the last partial
    Uall = np.full((50, d + 3), np.nan, dtype=F32)
    Iall = np.full((70, d + 1), np.nan, dtype=F32)
    Uall[:, :d] = rng.standard_normal((50, d)) * 0.7
    Iall[:, :d] = rng.standard_normal((70, d)) * 0.7
    users, items = rng.integers(0, 50, n), rng.integers(0, 70, n)
    raw = rk.pair_chain(Uall[users, :d], Iall[items, :d])
    np.testing.assert_array_equal(rk.bits(_gather_dot(Uall, users, Iall, items, d, 0)), rk.bits(raw))
    lo, hi = float(F32(-0.75)), float(F32(1.5))
    clip = np.minimum(np.maximum(raw, F32(lo)), F32(hi))
    np.testing.assert_array_equal(rk.bits(_gather_dot(Uall, users, Iall, items, d, 2, lo, hi)), rk.bits(clip))
    sig = _gather_dot(Uall, users, Iall, items, d, 1)
    ref = 1.0 / (1.0 + np.exp(-raw.astype(F64)))
    ulp = np.spacing(ref.astype(F32)).astype(F64)
    err = np.abs(sig.astype(F64) - ref) / ulp
    assert err.max() <= SIGMOID_ULP, f"sigmoid off by {err.max():.2f} ulp"


def test_fused_scores_match_fma_definition():
    """The tensor-core path's returned scores are the exact-score definition bit for bit, its ids that order."""
    import torch

    from librecommender_b200.engine import EmbedScorer

    rng = np.random.default_rng(11)
    n_users, N, d, K, B = 300, 20_000, 64, 50, 64
    Uu = rng.standard_normal((n_users, d)).astype(F32)
    It = rng.standard_normal((N + 1, d)).astype(F32)
    sc = EmbedScorer(Uu, It, N)
    users = rng.choice(n_users, size=B, replace=False)
    ids, scores, status = sc.recommend_fused(torch.as_tensor(users, device="cuda"), K, False, True)
    _sync()
    ok = status.cpu().numpy() == 0
    assert ok.mean() > 0.9, "the fused path repaired most rows"
    ids, scores = ids.cpu().numpy(), scores.cpu().numpy()
    want = rk.dot_chain(Uu[users], It[:N])
    order = rk.rank_order(want, K)
    np.testing.assert_array_equal(ids[ok], order[ok])
    np.testing.assert_array_equal(rk.bits(scores[ok]), rk.canonical_bits(np.take_along_axis(want, order, 1))[ok])


# =====================================================================================================================
# top-K
# =====================================================================================================================
def _ws_bytes(B, N, K):
    L = _lib()
    n = ctypes.c_size_t(0)
    L.check(L.lib.b200_topk_rows_workspace_bytes(B, N, K, ctypes.byref(n)))
    return n.value


def _topk(x, K, ld=None, with_scores=True, ws_delta=0):
    """b200_topk_rows on x [B, N] stored with leading dimension ld (padding = NaN, which would win if read), a
    workspace of exactly the reported size filled with 0xff, and guard cells after both outputs."""
    import torch

    L = _lib()
    B, N = x.shape
    ld = ld or N
    buf = np.full((B, ld), np.nan, dtype=F32)
    buf[:, :N] = x
    xd = _dev(buf)
    nbytes = _ws_bytes(B, N, K) + ws_delta
    ws = torch.full((nbytes,), 255, dtype=torch.uint8, device="cuda")
    guard = 16
    oid = torch.full((B * K + guard,), -7, dtype=torch.int64, device="cuda")
    osc = torch.full((B * K + guard,), 7.0, dtype=torch.float32, device="cuda") if with_scores else None
    rc = L.lib.b200_topk_rows(L.ptr(xd), ld, B, N, K, L.ptr(oid), L.ptr(osc), L.ptr(ws), nbytes, L.current_stream())
    _sync()
    if rc != 0:
        return rc, None, None
    oid = oid.cpu().numpy()
    assert (oid[B * K:] == -7).all(), "wrote past the ids"
    if osc is not None:
        osc = osc.cpu().numpy()
        assert (osc[B * K:] == 7.0).all(), "wrote past the scores"
        osc = osc[:B * K].reshape(B, K)
    return 0, oid[:B * K].reshape(B, K), osc


def _check_topk(x, K, **kw):
    rc, ids, sc = _topk(x, K, **kw)
    assert rc == 0, _lib().lib.b200_last_error()
    want = rk.rank_order(x, K)
    bad = np.nonzero((ids != want).any(axis=1))[0]
    assert len(bad) == 0, f"rows {bad[:8]} differ, first: got {ids[bad[0]][:12]} want {want[bad[0]][:12]}"
    if sc is not None:
        np.testing.assert_array_equal(rk.bits(sc), rk.canonical_bits(np.take_along_axis(x, want, 1)))


def _rows(N, rng):
    """Three rows: continuous values, small integers (the K-th value tied across every chunk), and a mix."""
    a = rng.standard_normal(N).astype(F32)
    b = rng.integers(0, 48, N).astype(F32)
    c = np.where(rng.random(N) < 0.5, a, b).astype(F32)
    return np.stack([a, b, c])


@pytest.mark.parametrize("K", [1, 2, 31, 32, 33, 1023, 1024, 1025, 4095, 4096])
def test_topk_shapes(K):
    rng = np.random.default_rng(K)
    for N in (K, 8191, 8192, 8193, 3 * 8192 + 1, 2 ** 20 + 7):
        if N < K:
            continue
        x = _rows(N, rng)
        _check_topk(x, K, ld=N + (5 if N % 2 else 0), with_scores=(N % 2 == 1))


def test_topk_row_groups():
    """More than 65 535 rows: the launcher runs groups of 65 535 rows on one workspace."""
    rng = np.random.default_rng(5)
    B, N, K = 65535 + 300, 40, 5
    x = rng.integers(0, 12, (B, N)).astype(F32)
    x[65535:] += 100.0 * rng.random((300, 1)).astype(F32)   # the second group's rows differ from the first's
    _check_topk(x, K)


def test_topk_tie_cut_across_chunks():
    """The K-th key is shared by items in several chunks and only the lowest-id part of the tie is taken."""
    N = 5 * 8192 + 3
    x = np.zeros((2, N), dtype=F32)
    x[:, ::4096] = 2.0                                     # 11 items above the tie
    tie = np.arange(7, N, 977)                             # spread over every chunk
    x[:, tie] = 1.0
    x[1, 8192 * 3 + 5] = 1.0                               # a tie inside one chunk's warp
    for K in (12, 11 + len(tie) // 2, 11 + len(tie)):
        _check_topk(x, K)


def test_topk_constant_rows():
    N = 3 * 8192 + 1
    x = np.stack([np.full(N, 3.25, F32), np.full(N, -np.inf, F32), np.full(N, np.inf, F32),
                  np.full(N, np.nan, F32), np.zeros(N, F32)])
    x[4, 1::2] = -0.0
    for K in (1, 33, 4096):
        _check_topk(x, K)


def test_topk_special_values():
    """Subnormals, +-0, +-inf, NaN of both signs (quiet, signalling, with payloads) and REMOVED entries."""
    rng = np.random.default_rng(17)
    N = 2 * 8192 + 77
    specials = _f32_from_bits([0x7FC00000, 0xFFC00000, 0x7F800001, 0xFF800001, 0x7FFFFFFF, 0xFFBFFFFF,
                               0x00000001, 0x80000001, 0x007FFFFF, 0x807FFFFF, 0x00000000, 0x80000000,
                               0x7F800000, 0xFF800000, 0xFFFFFFFF])
    x = np.empty((4, N), dtype=F32)
    for r in range(3):
        x[r] = rng.choice(specials, N)
        sub = rng.random(N) < 0.3
        x[r, sub] = (rng.standard_normal(int(sub.sum())) * 1e-39).astype(F32)      # subnormals
    x[3, :] = specials[rng.integers(10, 12, N)]            # only +0.0 and -0.0: ids decide
    for K in (1, 40, 1000, 4096):
        _check_topk(x, K, ld=N + 3)


def test_topk_removed_below_neg_inf():
    N = 9000
    x = np.full((2, N), -np.inf, dtype=F32)
    x[:, ::3] = _f32_from_bits([0xFFFFFFFF])[0]
    x[0, 5] = np.nan
    x[1, 7] = 0.0
    for K in (1, 4096):
        _check_topk(x[:, :3000], 2001)                  # reaches one removed entry past every -inf
        rc, ids, _ = _topk(x, K)
        assert rc == 0 and not (ids % 3 == 0).any(), "a removed entry came back while -inf were left"


def test_topk_workspace_and_rejections():
    import torch

    L = _lib()
    x = np.random.default_rng(1).standard_normal((3, 20_000)).astype(F32)
    _check_topk(x, 100)
    rc, _, _ = _topk(x, 100, ws_delta=-1)
    assert rc == -2 and b"workspace too small" in L.lib.b200_last_error()
    xd = _dev(np.zeros((3, 5000), F32))
    oid = torch.empty(3 * 4097, dtype=torch.int64, device="cuda")
    ws = torch.empty(_ws_bytes(3, 5000, 4096) * 2, dtype=torch.uint8, device="cuda")
    for N, K in ((5000, 0), (5000, 4097), (100, 101)):
        rc = L.lib.b200_topk_rows(L.ptr(xd), 5000, 3, N, K, L.ptr(oid), None, L.ptr(ws), ws.numel(), None)
        assert rc == -2, (N, K)


# =====================================================================================================================
# consumed mask and rank_recommendations
# =====================================================================================================================
def _csr(lists, n_users):
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    for u in range(n_users):
        indptr[u + 1] = indptr[u] + len(lists.get(u, []))
    idx = np.concatenate([np.asarray(lists.get(u, []), np.int32) for u in range(n_users)] + [np.zeros(0, np.int32)])
    return indptr, idx


def test_mask_consumed_direct():
    """Rows are removed iff the list is non-empty and K + len(list) <= N (duplicates and ids outside [0, N)
    counted, as the reference's len() counts them); only ids in [0, N) are written, with the REMOVED pattern."""
    import torch

    L = _lib()
    N, K, ld = 50, 10, 56
    lists = {0: [3, 3, 7, 49],                       # duplicates
             1: [1, -4, 50, 55, 2],                  # ids outside [0, N): counted, never written (55 < ld)
             2: list(range(40)),                     # K + 40 == N: filtered
             3: list(range(40)) + [0],               # K + 41 == N + 1: not filtered
             4: []}                                  # empty list
    n_users = 5
    indptr, idx = _csr(lists, n_users)
    users = np.array([0, 1, 2, 3, 4, 7, 0], dtype=np.int64)   # 7 >= n_users: OOV; user 0 twice
    x = np.random.default_rng(2).standard_normal((len(users), ld)).astype(F32)
    xd, ud, pd, idd = _dev(x), _dev(users), _dev(indptr), _dev(idx)
    L.check(L.lib.b200_mask_consumed(L.ptr(xd), ld, L.ptr(ud), len(users), N, K, L.ptr(pd), L.ptr(idd), n_users,
                                     L.current_stream()))
    _sync()
    got = rk.bits(xd.cpu().numpy())
    want = rk.bits(x).copy()
    for r, u in enumerate(users):
        c = lists.get(int(u), []) if u < n_users else []
        if len(c) and K + len(c) <= N:
            v = np.asarray(c)
            want[r, v[(v >= 0) & (v < N)]] = rk.REMOVED_BITS
    np.testing.assert_array_equal(got, want)


def test_rank_recommendations_removes_consumed_at_neg_inf_and_nan():
    """Kept items scored -inf or NaN, n_rec reaching past them: a consumed item is never returned."""
    from librecommender_b200 import rank_recommendations
    from oracle.ranking import rank_recommendations as orc_rank

    rng = np.random.default_rng(4)
    N, n_users = 12, 6
    preds = rng.standard_normal((n_users, N)).astype(F32)
    preds[:, 8:] = -np.inf
    preds[1, 2] = np.nan
    with np.errstate(invalid="ignore"):
        preds[2, 3] = np.float32(np.inf) - np.float32(np.inf)   # the negative NaN x86 arithmetic makes
    preds[3, :] = -np.inf
    preds[4, [0, 5]] = [0.0, -0.0]
    consumed = {0: [8, 9, 9], 1: [2, 10], 2: [3, 11, 11, -1, 99], 3: [0, 1, 2], 4: [5, 0]}
    users = [0, 1, 2, 3, 4, 5]
    for n_rec in (1, 5, 7, 9):
        ids, sc = rank_recommendations("rating", users, preds, n_rec, N, consumed, True, False, True)
        rid, rsc = orc_rank("rating", users, preds, n_rec, N, consumed, True, True)
        np.testing.assert_array_equal(ids, rid, err_msg=f"n_rec={n_rec}")
        np.testing.assert_array_equal(rk.bits(sc), rk.canonical_bits(rsc))
        for r, u in enumerate(users):
            c = consumed.get(u, [])
            if c and n_rec + len(c) <= N:
                assert not set(ids[r].tolist()) & set(c), (n_rec, u)
    # the caller's array is left as it was
    assert np.isnan(preds[1, 2]) and preds[4, 5] == 0


def test_rank_recommendations_nan_first_and_signed_zero():
    from librecommender_b200 import rank_recommendations
    from oracle.ranking import rank_recommendations as orc_rank

    N = 20
    preds = np.linspace(-1.0, 1.0, N, dtype=F32)[None].repeat(3, 0)
    preds[0, 4] = np.nan
    preds[1, [3, 9]] = _f32_from_bits([0xFFC00000, 0x7FC00000])   # both signs: ties by id
    preds[2, :] = 0.0
    preds[2, ::3] = -0.0
    for n_rec in (1, 2, 20):
        got = rank_recommendations("rating", [0, 1, 2], preds, n_rec, N, {}, True, False, False)
        np.testing.assert_array_equal(got, orc_rank("rating", [0, 1, 2], preds, n_rec, N, {}, True))
    assert got[0, 0] == 4 and list(got[1, :2]) == [3, 9] and list(got[2, :3]) == [0, 1, 2]


def test_rank_recommendations_random_rec_keeps_neg_inf_sampleable():
    """random_rec: consumed items are never drawn; a -inf prediction keeps the 1e-8 floor and can be drawn."""
    from librecommender_b200 import rank_recommendations

    N = 6
    preds = np.array([[5.0, -np.inf, -np.inf, -np.inf, -np.inf, 3.0]], dtype=F32)
    consumed = {0: [0]}
    for _ in range(5):        # 5 of the 5 kept items: every -inf item is drawn, the consumed one never
        ids = rank_recommendations("rating", [0], preds, 5, N, consumed, True, True, False)
        assert sorted(ids[0].tolist()) == [1, 2, 3, 4, 5] and ids[0, 0] == 5


def test_merge_topk_shards_neg_inf_candidates():
    import torch

    from librecommender_b200.parallel import merge_topk_shards

    ninf = -np.inf
    ids = np.array([[[4, 9, 13, 20]], [[30, 31, -1, -1]]], dtype=np.int64)      # [G=2, B=1, K=4]
    sc = np.array([[[1.0, ninf, ninf, ninf]], [[0.5, ninf, 0.0, 0.0]]], dtype=F32)
    oid, osc = merge_topk_shards(torch.as_tensor(ids, device="cuda"), torch.as_tensor(sc, device="cuda"), 6)
    _sync()
    np.testing.assert_array_equal(oid.cpu().numpy(), [[4, 30, 9, 13, 20, 31]])
    np.testing.assert_array_equal(osc.cpu().numpy(), [[1.0, 0.5, ninf, ninf, ninf, ninf]])
    oid, osc = merge_topk_shards(torch.as_tensor(ids, device="cuda"), torch.as_tensor(sc, device="cuda"), 8)
    np.testing.assert_array_equal(oid.cpu().numpy(), [[4, 30, 9, 13, 20, 31, -1, -1]])
    assert np.isneginf(osc.cpu().numpy()[0, 6:]).all()


# =====================================================================================================================
# FM / DeepFM pair scores
# =====================================================================================================================
def _sample_items(N, per_iter, rng, n_mid=3000):
    """Every item of the first and the last block iteration, and a random sample in between."""
    first = np.arange(min(N, per_iter))
    last0 = (N - 1) // per_iter * per_iter
    last = np.arange(last0, N)
    mid = rng.integers(per_iter, max(last0, per_iter + 1), n_mid) if last0 > per_iter else np.zeros(0, np.int64)
    return np.unique(np.concatenate([first, last, mid]))


def _check_pair(got, ref, mag, what):
    err = np.abs(got.astype(F64) - ref)
    bound = C_PAIR * rk.U * mag
    worst = np.unravel_index(np.argmax(err / bound), err.shape)
    assert (err <= bound).all(), f"{what}: err {err[worst]:.3g} > bound {bound[worst]:.3g} at {worst}"


def _out_buffer(B, lds):
    import torch

    return torch.full((B, lds), float("nan"), dtype=torch.float32, device="cuda")


def _fm_call(c, B, N, out, lds):
    L = _lib()
    d = {k: (_dev(v) if isinstance(v, np.ndarray) else None) for k, v in c.items()}
    return L.lib.b200_fm_pair_scores(L.ptr(d["Su"]), L.ptr(d["Qu"]), L.ptr(d["lu"]), B, L.ptr(d["Si"]),
                                     L.ptr(d["Qi"]), L.ptr(d["li"]), N, c["Su"].shape[1], c["lin_bias"],
                                     L.ptr(d["bn_scale"]), L.ptr(d["bn_shift"]), L.ptr(d["pw_kernel"]),
                                     c["pw_bias"], L.ptr(out), lds, L.current_stream())


@pytest.mark.parametrize("B,K,bn", [(1, 1, True), (3, 17, False), (3, 64, True), (1, 64, False)])
def test_fm_pair_scores(B, K, bn):
    N = 600_001                                           # 1024 blocks x 256 items per pass: three passes
    c = rk.make_fm_case(B, K, N, bn, seed=10 * K + B)
    lds = N + 3
    out = _out_buffer(B, lds)
    assert _fm_call(c, B, N, out, lds) == 0
    _sync()
    got = out.cpu().numpy()
    assert np.isnan(got[:, N:]).all(), "wrote past N"
    items = _sample_items(N, 1024 * 256, np.random.default_rng(K))
    for i0 in range(0, len(items), 32768):                # float64 in slices of items
        part = items[i0:i0 + 32768]
        ref, mag = rk.fm_pair_ref(c, np.arange(B), part)
        _check_pair(got[:, part], ref, mag, f"fm B={B} K={K} bn={bn}")
        if i0 == 0:
            elu = ref[0, :64] - (np.float64(c["lu"][0]) + c["lin_bias"] + c["li"][:64])
            assert (elu > 0).any() and (elu < 0).any() and np.abs(elu).min() < 1e-3, "acc next to 0, both signs"


def _deepfm_call(c, B, N, out, lds, **over):
    L = _lib()
    d = {k: (_dev(v) if isinstance(v, np.ndarray) else None) for k, v in c.items()}
    K = over.get("K", c["Su"].shape[1])
    return L.lib.b200_deepfm_pair_scores(
        L.ptr(d["Su"]), L.ptr(d["Qu"]), L.ptr(d["lu"]), L.ptr(d["Pu"]), B, L.ptr(d["Si"]),
        L.ptr(d["Qi"]), L.ptr(d["li"]), L.ptr(d["Pi"]), N, K, over.get("H1", c["H1"]), over.get("H2", c["H2"]),
        over.get("H3", c["H3"]), c["lin_bias"], L.ptr(d["W2"]), L.ptr(d["b2"]), L.ptr(d["W3"]), L.ptr(d["b3"]),
        L.ptr(d["w_out"]), c["b_out"], L.ptr(out), lds, L.current_stream())


DEEPFM_CASES = [  # (B, K, H1, H2, H3, fm_zero)
    (1, 8, 1, 1, 0, False), (3, 16, 33, 63, 1, False), (1, 4, 64, 64, 32, False), (3, 1, 96, 64, 0, True),
    (1, 64, 256, 63, 32, False), (3, 8, 96, 1, 32, False),
]


@pytest.mark.parametrize("B,K,H1,H2,H3,fm_zero", DEEPFM_CASES)
def test_deepfm_pair_scores(B, K, H1, H2, H3, fm_zero):
    N = 300_007                                           # 512 blocks x 256 items per pass: three passes
    c = rk.make_deepfm_case(B, K, N, H1, H2, H3, fm_zero, seed=H1 * 7 + H2 + H3)
    lds = N + 1
    out = _out_buffer(B, lds)
    assert _deepfm_call(c, B, N, out, lds) == 0
    _sync()
    got = out.cpu().numpy()
    assert np.isnan(got[:, N:]).all(), "wrote past N"
    items = _sample_items(N, 512 * 256, np.random.default_rng(H1))
    for i0 in range(0, len(items), 32768):                # float64 in slices of items
        part = items[i0:i0 + 32768]
        ref, mag = rk.deepfm_pair_ref(c, np.arange(B), part)
        _check_pair(got[:, part], ref, mag, f"deepfm B={B} K={K} H=({H1},{H2},{H3})")


def test_pair_size_checks():
    L = _lib()
    c = rk.make_deepfm_case(1, 4, 8, 8, 8, 8, False, seed=0)
    out = _out_buffer(1, 8)
    for over in (dict(B=65536), dict(K=65), dict(H1=257), dict(H2=65), dict(H3=33)):
        b = over.pop("B", 1)
        assert _deepfm_call(c, b, 8, out, 8, **over) == -2, (b, over)
    assert L.lib.b200_fm_pair_scores(*([L.ptr(out)] * 3), 65536, *([L.ptr(out)] * 3), 8, 4, 0.0, None, None,
                                     L.ptr(out), 0.0, L.ptr(out), 8, None) == -2
    assert L.lib.b200_fm_pair_scores(*([L.ptr(out)] * 3), 1, *([L.ptr(out)] * 3), 8, 65, 0.0, None, None,
                                     L.ptr(out), 0.0, L.ptr(out), 8, None) == -2
    _sync()
    assert np.isnan(out.cpu().numpy()).all(), "a rejected call wrote"
