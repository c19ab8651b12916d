"""GPU tests of the fused scorer's two finalize paths: ``finalize_warp_kernel`` (one warp per row, the
common case) and ``finalize_kernel`` (one CTA per row, the rows the warp kernel defers).

Each case runs the same inputs twice: in normal operation, and with every row deferred to the block
kernel (``b200_recommend_embed_debug(3)``).  Ids, fp32 scores and row_status must agree bit for bit,
so any difference in the warp kernel's select, consumed filter, exact re-score or sort fails.  Rows
that overflowed a candidate list in the sweep (status 1) are left out of the comparison: when a list
is compacted, the order in which the row's warps raise its threshold can differ between launches, so
the sweep itself may flag a borderline row in one launch and not in the other.

Cases: the benchmarked shape (1 M items, d = 64, top-100, 32 768 users, Zipf consumed lists), embed
widths 7 / 128 / 256 (scalar loads, k-block sweep), K = 1 and 288, consumed lists with duplicated
entries, rows over the warp kernel's buffer (low thresholds of the linear rank rule) and over its
candidate limit (dense ties from duplicated item rows), and rows that end with status 2 / 3 / 4 / 5.
"""
import numpy as np
import pytest

from test_gpu_fused_c2 import _tables, _zipf_consumed

pytestmark = pytest.mark.gpu


def _deferred(sc, B, K):
    """Rows finalize_warp_kernel handed to finalize_kernel in the latest call: the count at the head of
    the deferred-row list, which follows make_plan's workspace layout (csrc/score_topk_tc.cu):
    A, meta, tau, guess, status, cnt, deferred rows."""
    import torch

    plan = sc.fused_plan(B, K)
    al = lambda x: (x + 255) // 256 * 256                      # noqa: E731
    cl = plan["cluster_x10_plus_mma_groups"] // 10
    B_pad = (B + 128 * cl - 1) // (128 * cl) * (128 * cl)
    d_pad = (sc.d + 63) // 64 * 64
    off = al(B_pad * d_pad * 2) + al(B_pad * 32) + 3 * al(B_pad * 4) + al(2 * plan["n_splits"] * B_pad * 4)
    ws = sc._ws
    base = (256 - ws.data_ptr() % 256) % 256
    return int(ws[base + off: base + off + 4].view(torch.int32).item())


def _both(sc, uid, K, filt):
    """((ids, score bits, status), deferred rows) in normal operation and with every row deferred."""
    import torch
    from librecommender_b200 import _lib

    out = []
    try:
        for level in (0, 3):
            _lib.check(_lib.lib.b200_recommend_embed_debug(level))
            ids, scores, status = sc.recommend_fused(uid, K, filt, True)
            torch.cuda.synchronize()
            out.append(((ids.cpu().numpy(), scores.cpu().numpy().view(np.int32), status.cpu().numpy()),
                        _deferred(sc, len(uid), K)))
    finally:
        _lib.check(_lib.lib.b200_recommend_embed_debug(0))
    (warp, n_def), (block, n_all) = out
    assert n_all == len(uid)
    both = (warp[2] != 1) & (block[2] != 1)
    np.testing.assert_array_equal(warp[2][both], block[2][both])
    np.testing.assert_array_equal(warp[0][both], block[0][both])
    np.testing.assert_array_equal(warp[1][both], block[1][both])
    for ids, _, status in (warp, block):
        assert (ids[status != 0] == -1).all()
    return warp[2], n_def


def _codes(status):
    return {int(c): int((status == c).sum()) for c in np.unique(status)}


@pytest.fixture(scope="module")
def c2():
    import torch
    from librecommender_b200.engine import EmbedScorer

    n_users, N, d = 100_000, 1_000_000, 64
    U, I = _tables(81, n_users, N, d)
    csr = _zipf_consumed(82, n_users, N)
    sc = EmbedScorer(U, I, N, csr, n_users=n_users)
    users = np.random.default_rng(83).choice(n_users, size=32768, replace=False).astype(np.int64)
    return sc, torch.as_tensor(users).cuda()


def test_bench_shape(c2):
    sc, uid = c2
    status, n_def = _both(sc, uid, 100, True)
    assert (status == 0).mean() >= 0.97, _codes(status)
    # every 97th user of the fixture consumed 500 items: a capped k_row, deferred; (almost) nothing else is
    assert n_def <= 0.02 * len(uid), n_def


@pytest.mark.parametrize("K", [1, 288])
def test_k_extremes(c2, K):
    sc, uid = c2
    status, n_def = _both(sc, uid[:8192], K, True)
    assert (status == 0).mean() >= 0.9, _codes(status)
    # K = 288: at least 288 candidates, more than the warp kernel sorts: every row is deferred
    assert n_def <= 0.02 * 8192 if K == 1 else n_def == 8192, n_def


@pytest.mark.parametrize("d", [7, 128, 256])
def test_embed_widths(d):
    import torch
    from librecommender_b200.engine import EmbedScorer

    n_users, N = 20_000, 300_000
    U, I = _tables(90 + d, n_users, N, d)
    sc = EmbedScorer(U, I, N, _zipf_consumed(91, n_users, N), n_users=n_users)
    uid = torch.as_tensor(np.random.default_rng(92).choice(n_users, size=4096, replace=False)).cuda()
    status, n_def = _both(sc, uid, 100, True)
    assert (status == 0).mean() >= 0.97, _codes(status)
    assert n_def <= 0.05 * len(uid), n_def


@pytest.mark.parametrize("K", [100, 288])
def test_duplicated_consumed_entries(K):
    """Consumed lists that hold each of the user's 50 best items twice (so the filter removes
    candidates and meets every id twice); every 8th user also consumed 300 more items (a capped k_row:
    deferred).  At K = 288 every k_row is capped and the 50 removed items leave too few survivors:
    status 5."""
    import torch
    from librecommender_b200.consumed import ConsumedCSR
    from librecommender_b200.engine import EmbedScorer

    n_users, N, d, B = 8192, 1_000_000, 64, 8192
    U, I = _tables(101, n_users, N, d)
    sc = EmbedScorer(U, I, N, None, n_users=n_users)
    uid = torch.arange(B, dtype=torch.int64).cuda()
    top = sc.recommend_exact(uid, 50, False, False).cpu().numpy()
    rng = np.random.default_rng(102)
    lists = []
    for u in range(n_users):
        extra = rng.integers(0, N, size=300) if u % 8 == 0 else np.zeros(0, np.int64)
        lists.append(np.concatenate([top[u], top[u][::-1], extra]).astype(np.int32))
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    np.cumsum([len(x) for x in lists], out=indptr[1:])
    sc.set_consumed(ConsumedCSR(indptr, np.concatenate(lists)))
    status, n_def = _both(sc, uid, K, True)
    if K == 100:
        assert (status[1::8] == 0).mean() >= 0.97, _codes(status)
        assert B // 8 <= n_def <= B // 4, n_def
    else:
        assert (status == 5).mean() >= 0.5, _codes(status)


def test_rows_over_the_warp_buffer():
    """The linear rank rule with coefficient 5 and margin 1 starts the main pass about 5 k_row items below
    c_k: rows collect more elements than the warp kernel keeps and go to the block kernel."""
    import torch
    from librecommender_b200 import _lib
    from librecommender_b200.engine import EmbedScorer

    n_users, N, d, B = 20_000, 1_000_000, 64, 8192
    U, I = _tables(111, n_users, N, d)
    sc = EmbedScorer(U, I, N, _zipf_consumed(112, n_users, N), n_users=n_users)
    uid = torch.as_tensor(np.random.default_rng(113).choice(n_users, size=B, replace=False)).cuda()
    try:
        _lib.check(_lib.lib.b200_recommend_embed_speculation(16, 0.0))
        _lib.check(_lib.lib.b200_recommend_embed_tune(0, 5.0))
        _lib.check(_lib.lib.b200_recommend_embed_debug(-1))
        status, n_def = _both(sc, uid, 100, True)
    finally:
        _lib.check(_lib.lib.b200_recommend_embed_debug(-12))
        _lib.check(_lib.lib.b200_recommend_embed_speculation(0, 0.0))
    assert n_def >= B // 4, (n_def, _codes(status))
    assert (status == 0).mean() >= 0.5, _codes(status)


def test_dense_ties_over_the_candidate_limit():
    """A catalogue of 250 item rows, each repeated 400 times: a row's best coarse score is shared by at
    least 400 items, more candidates than the warp kernel sorts (block kernel: exact ties ordered by
    id, or status 4 above its own limit)."""
    import torch
    from librecommender_b200.engine import EmbedScorer

    n_users, N, d, B = 4096, 100_000, 64, 4096
    U, I = _tables(121, n_users, N, d)
    I[:N] = np.tile(I[:250], (400, 1))
    sc = EmbedScorer(U, I, N, _zipf_consumed(122, n_users, N), n_users=n_users)
    uid = torch.arange(B, dtype=torch.int64).cuda()
    status, n_def = _both(sc, uid, 100, True)
    assert n_def >= B // 2, (n_def, _codes(status))
    assert (status == 0).mean() >= 0.5, _codes(status)


def test_failed_speculation_statuses():
    """test_gpu_speculation's adversarial catalogue (every sampled tile holds the longest items): most
    rows end with status 3, or 2 when the guess leaves fewer than k_row items."""
    import ctypes

    import torch
    from librecommender_b200 import _lib
    from librecommender_b200.engine import EmbedScorer

    n_users, N, d, K, B, stride = 20_000, 1_000_000, 64, 100, 8192, 8
    U, I = _tables(71, n_users, N, d)
    out = (ctypes.c_int32 * 10)()
    _lib.check(_lib.lib.b200_recommend_embed_plan(B, N, d, K, out, 10))
    tps = int(out[2])
    tiles = np.arange(-(-N // 256))
    sampled = tiles[(tiles - (tiles // tps) * tps) % stride == 0]
    rows = (sampled[:, None] * 256 + np.arange(256)[None, :]).ravel()
    I[rows[rows < N]] *= np.float32(1.5)
    sc = EmbedScorer(U, I, N, None, n_users=n_users)
    uid = torch.as_tensor(np.random.default_rng(72).choice(n_users, size=B, replace=False)).cuda()
    status, n_def = _both(sc, uid, K, False)
    assert np.isin(status, (2, 3)).mean() >= 0.5, _codes(status)
    assert n_def >= np.isin(status, (2, 3)).sum()
