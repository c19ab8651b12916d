"""GPU test of the fused scorer's epilogue vote and ballot slot masks on edge-case rows.

Per 64-column step the warp votes whether any of its rows reaches the row threshold tau, and a hot step
takes one ballot per (group, row) slot.  A warp holds the 16 user rows 16 w .. 16 w + 15 of a tile (the
calls below run rows 0 .. B - 1 in order), so the rows are laid out in aligned 16-row blocks: a block of
rows with a non-positive threshold shares its warp with no positive-threshold row.
  * ``mixed``: every fourth block holds rows whose scores are all negative (negative block maxima,
    hence a negative speculative threshold); block 1 holds +0.0 and -0.0 user rows (every score 0);
    the other blocks are ordinary rows with positive thresholds;
  * ``no_prepass``: the same rows over a catalogue too small for the pre-pass (threshold -inf until a
    compaction raises it); the catalogue is small enough for the zero rows to finish too;
  * ``ties``: exact integer scores; about 1 in 512 items score exactly the speculative threshold
    (the largest sampled block maximum level), 20 items score above it;
  * ``tiny``: most scores come from fp16-subnormal item coordinates, so the speculative threshold is
    a tiny positive coarse score, some scores are exactly 0, and 40 items score far above.
    (An fp32-subnormal coarse score cannot occur: the smallest non-zero product of two fp16 values is
    2^-48.)
Every organisation code must give status 0 on the rows listed as safe, and every row with status 0
must equal the exact path bit for bit (ids and scores).
"""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

D, K, B = 64, 20, 512
CODES = [113, 115, 123, 125, 133, 135, 213, 215, 223, 225, 233, 235]
ZERO_BLOCK = slice(16, 32)      # rows 16..23: +0.0, rows 24..31: -0.0


def _mixed_users(rng):
    """Blocks b % 4 == 0: all scores negative against `_half_space_items`; block 1: zero rows;
    others: random directions (positive thresholds)."""
    U = rng.standard_normal((B, D)).astype(np.float32)
    U /= np.linalg.norm(U, axis=1, keepdims=True)
    neg = (np.arange(B) // 16) % 4 == 0
    U[neg] = 0.0
    U[neg, 0] = -1.0
    U[neg, 1:] = 1e-3 * rng.standard_normal((int(neg.sum()), D - 1)).astype(np.float32)
    U[16:24] = 0.0
    U[24:32] = -0.0
    return U


def _half_space_items(rng, N):
    """Unit rows whose first coordinate is >= 0.06: -e0 (+ 1e-3 noise) scores every item below -0.05."""
    I = rng.standard_normal((N, D)).astype(np.float32)
    I[:, 0] = np.abs(I[:, 0]) + 0.5
    I /= np.linalg.norm(I, axis=1, keepdims=True)
    return I


def _case(name):
    """(U, I, safe rows, pre-pass expected)"""
    rng = np.random.default_rng({"mixed": 1, "no_prepass": 2, "ties": 3, "tiny": 4}[name])
    safe = np.ones(B, dtype=bool)
    if name == "mixed":
        safe[ZERO_BLOCK] = False     # every item ties at 0: handed to the exact path
        return _mixed_users(rng), _half_space_items(rng, 600_000), safe, True
    if name == "no_prepass":
        return _mixed_users(rng), _half_space_items(rng, 2_000), safe, False
    N = 600_000
    I = np.zeros((N, D), dtype=np.float32)
    picks = rng.choice(N, size=N // 512 + 60, replace=False)
    U = np.zeros((B, D), dtype=np.float32)
    if name == "ties":
        # score = level of the item: 1 for most items, 2 for 1 in 512 (the threshold), 3 for 40, 4 for 20
        I[:, 0] = 1.0
        I[picks[60:], 0] = 2.0
        I[picks[20:60], 0] = 3.0
        I[picks[:20], 0] = 4.0
        U[:, 0] = 1.0
        return U, I, safe, True
    # tiny: item = e0 + c e1, c in {0} u [2^-30, 2^-20]; the table scale puts e0 at 64, so 64 c is an
    # fp16 subnormal (or 0); 40 items are e1 and score 1.  User = e1.
    I[:, 0] = 1.0
    c = np.exp2(rng.uniform(-30.0, -20.0, size=N)).astype(np.float32)
    c[rng.random(N) < 0.1] = 0.0
    I[:, 1] = c
    I[picks[:40]] = 0.0
    I[picks[:40], 1] = 1.0
    U[:, 1] = 1.0
    return U, I, safe, True


@pytest.fixture(scope="module", params=["mixed", "no_prepass", "ties", "tiny"])
def case(request):
    import torch
    from librecommender_b200.engine import EmbedScorer

    U, I, safe, use_pre = _case(request.param)
    sc = EmbedScorer(U, I, I.shape[0], None, n_users=B)
    assert sc.fused_plan(B, K)["use_pre"] == int(use_pre)
    uid = torch.arange(B, dtype=torch.int64, device="cuda")
    ids_e, sc_e = sc.recommend_exact(uid, K, False, True)
    return sc, uid, ids_e.cpu().numpy(), sc_e.cpu().numpy(), safe


@pytest.mark.parametrize("code", CODES)
def test_fused_equals_exact(case, code):
    import torch
    from librecommender_b200 import _lib

    sc, uid, ids_e, sc_e, safe = case
    try:
        _lib.check(_lib.lib.b200_recommend_embed_tune(code, 0.0))
        ids_f, sc_f, status = sc.recommend_fused(uid, K, False, True)
        torch.cuda.synchronize()
    finally:
        _lib.check(_lib.lib.b200_recommend_embed_tune(215, 0.0))
    status = status.cpu().numpy()
    ok = status == 0
    codes = {int(c): int((status == c).sum()) for c in np.unique(status)}
    assert safe.sum() >= B - 16 and ok[safe].all(), codes
    ids_f, sc_f = ids_f.cpu().numpy(), sc_f.cpu().numpy()
    np.testing.assert_array_equal(ids_f[ok], ids_e[ok])
    np.testing.assert_array_equal(sc_f[ok], sc_e[ok])
    assert (ids_f[~ok] == -1).all()
