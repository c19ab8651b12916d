"""GPU test of the fused scorer's record stores, slot by slot.

In the m64n256 accumulator fragment a lane holds, for each 64-column epilogue step, 16 (group, row)
slots: 8 groups of 8 items times its two user rows.  A hot step writes a 48-byte record for every slot
whose group reaches the row's threshold.  Here the catalogue is built so that, in 8 chosen item tiles,
every user row has exactly ONE hot group per step, at a slot that moves from tile to tile.  Rows r and
r + 8 (the two rows of a lane) and the 8 quads of a warp sit at different groups of the same step, so
each lane's slot mask differs from the warp's union.  Over the 8 tiles every row visits all 8 group
positions in all 4 steps, hence both candidate lists (column halves) of the tile.  The 256 users fill
two user tiles, the two CTAs of a cluster.  One more hot group per row sits in the last, partial item tile.

Every other item scores 0 or 0.5 except one item per 128-item half of each tile the pre-pass samples,
which scores 1.0 for every row: that fixes the speculative threshold at 1.0, below every planted item
(>= 1.5).  A record stored for the wrong slot, row or list loses a planted item, so the fused result,
status 0 on every row, must equal the exact path bit for bit and the planted items in score order.
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

N_USERS, N, D, TN = 256, 1_000_003, 64, 256
N_SEL = D - 1                      # user r scores e_0 + e_(1 + r % 63)
N_TEST_TILES = 8
K = 4 * N_TEST_TILES + 1           # planted items per row: 4 steps x 8 tiles + the partial tile


def _catalogue(n_splits, tiles_per_split):
    U = np.zeros((N_USERS, D), dtype=np.float32)
    sel = np.arange(N_USERS) % N_SEL
    U[:, 0] = 1.0
    U[np.arange(N_USERS), 1 + sel] = 1.0
    I = np.zeros((N, D), dtype=np.float32)
    total_tiles = (N + TN - 1) // TN
    for sp in range(n_splits):   # the tiles the pre-pass samples: one 1.0 item per 128-column half
        t0 = sp * tiles_per_split
        for t in range(t0, min(t0 + tiles_per_split, total_tiles), 16):
            if (t + 1) * TN <= N:
                I[t * TN, 0] = I[t * TN + TN // 2, 0] = 1.0
    planted = np.zeros((N_SEL, K), dtype=np.int64)   # [selector, rank of the score] -> item id

    def plant(item, s, idx):
        assert not I[item].any()
        I[item, 0] = 0.5
        I[item, 1 + s] = 1.0 + 0.01 * idx      # 1.5 + 0.01 idx for the rows of selector s, 0.5 for the others
        planted[s, idx] = item

    for k in range(N_TEST_TILES):
        t = (k + 1) * tiles_per_split + 1 + k  # not a sampled tile (offset 1 + k in its split)
        assert t < total_tiles - 1
        for step in range(4):
            for s in range(N_SEL):
                a, b = divmod(s, 8)
                jl = (a + b + k) % 8           # selector 8a + b at group jl, column a of the group
                plant(t * TN + 64 * step + 8 * jl + a, s, 4 * k + step)
    last = (total_tiles - 1) * TN
    assert N - last >= N_SEL
    for s in range(N_SEL):
        plant(last + s, s, K - 1)
    return U, I, planted, sel


@pytest.fixture(scope="module")
def setup():
    from librecommender_b200 import _lib
    import ctypes

    out = (ctypes.c_int32 * 8)()
    _lib.check(_lib.lib.b200_recommend_embed_plan(N_USERS, N, D, K, out, 8))
    use_pre, n_splits, tiles_per_split = int(out[0]), int(out[1]), int(out[2])
    assert use_pre == 1 and n_splits >= N_TEST_TILES + 1, list(out)
    U, I, planted, sel = _catalogue(n_splits, tiles_per_split)
    from librecommender_b200.engine import EmbedScorer

    sc = EmbedScorer(U, I, N, None, n_users=N_USERS)
    expected = planted[sel][:, ::-1]       # planted items of the row's selector, best score first
    return sc, expected


@pytest.mark.parametrize("code", [215, 213, 225, 223, 115, 113, 125, 123])
def test_one_hot_group_per_slot(setup, code):
    import torch
    from librecommender_b200 import _lib

    sc, expected = setup
    uid = torch.arange(N_USERS, dtype=torch.int64, device="cuda")
    try:
        _lib.check(_lib.lib.b200_recommend_embed_tune(code, 0.0))
        plan = sc.fused_plan(N_USERS, K)
        assert plan["use_pre"] == 1 and plan["cluster_x10_plus_mma_groups"] == code // 10, plan
        ids_f, sc_f, status = sc.recommend_fused(uid, K, False, True)
    finally:
        _lib.check(_lib.lib.b200_recommend_embed_tune(215, 0.0))
    ids_e, sc_e = sc.recommend_exact(uid, K, False, True)
    torch.cuda.synchronize()
    status = status.cpu().numpy()
    assert (status == 0).all(), {int(c): int((status == c).sum()) for c in np.unique(status)}
    np.testing.assert_array_equal(ids_e.cpu().numpy(), expected)
    np.testing.assert_array_equal(ids_f.cpu().numpy(), ids_e.cpu().numpy())
    np.testing.assert_array_equal(sc_f.cpu().numpy(), sc_e.cpu().numpy())
