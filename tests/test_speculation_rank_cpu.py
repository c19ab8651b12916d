"""CPU tests of the fused scorer's speculative threshold rule (csrc/score_topk_tc.cu, rank_table):

* the rank table the library builds (b200_recommend_embed_plan, n_out >= 299) against scipy.stats.binom:
  pre_k(k_row) = the smallest r with P[Binomial(k_row + 16, f) >= r] <= delta, for every k_row <= 288,
  each pre-pass stride's sampled fraction f and the failure budgets at both ends of their range;
* the linear rule is still selected by a non-zero rank coefficient, and (0, 0) restores the default;
* the numpy model of the selection algorithm (test_k4_algorithm_model_cpu.py) restated with the new rule:
  every accepted row is exact, and the rate of failed speculation on random catalogues is consistent
  with the budget delta.
"""
import ctypes
import math

import numpy as np
import pytest
from scipy.stats import binom

from test_k4_algorithm_model_cpu import ERR_COEF, KROW_MAX, _catalogue, _exact_scores, _f16, _pow2_scale

TIE_ALLOWANCE = 16                     # PRE_TIE_ALLOWANCE of score_topk_tc.cu
BENCH = (32768, 1_000_000, 64, 100)    # B, N, d, K of the benchmarked shape
N_OUT = 10 + KROW_MAX + 1


def _plan(B, N, d, K):
    from librecommender_b200 import _lib

    out = (ctypes.c_int32 * N_OUT)()
    _lib.check(_lib.lib.b200_recommend_embed_plan(B, N, d, K, out, N_OUT))
    return [int(v) for v in out]


@pytest.fixture
def lib():
    from librecommender_b200 import _lib

    yield _lib
    _lib.check(_lib.lib.b200_recommend_embed_speculation(0, 0.0))


def _rank(n, f, delta):
    """smallest r with P[Binomial(n, f) >= r] <= delta"""
    return int(binom.isf(delta, n, f)) + 1 if f < 1 else n + 1


@pytest.mark.parametrize("stride", [2, 4, 8, 16, 32])
@pytest.mark.parametrize("delta", [1e-9, 1e-5, 1e-2])
def test_rank_table_matches_scipy(lib, stride, delta):
    lib.check(lib.lib.b200_recommend_embed_speculation(stride, delta))
    B, N, d, K = BENCH
    out = _plan(B, N, d, K)
    tiles = -(-N // 256)
    assert out[8] == stride
    assert out[4] == -(-out[2] // stride)                     # sampled tiles per split follow the stride
    f = out[9] / tiles
    assert abs(f - 1.0 / stride) < 0.01
    delta32 = float(np.float32(delta))                        # the budget crosses the C ABI as a float
    for k in range(KROW_MAX + 1):
        n, r = k + TIE_ALLOWANCE, out[10 + k]
        assert binom.sf(r - 1, n, f) <= delta32 * (1 + 1e-6), (k, r)
        assert r == 1 or binom.sf(r - 2, n, f) > delta32 * (1 - 1e-6), (k, r)
        if abs(binom.sf(r - 1, n, f) / delta32 - 1) > 1e-6:   # away from the boundary: scipy agrees exactly
            assert r == _rank(n, f, delta32), (k, r)


def test_rank_table_small_catalogue_every_tile_sampled(lib):
    """A plan with one item tile per split samples every tile: f = 1, pre_k = n + 1 (no speculation)."""
    lib.check(lib.lib.b200_recommend_embed_speculation(8, 0.0))
    out = _plan(300, 32 * 256, 64, 10)
    assert out[2] == 1 and out[9] == 32
    assert out[10:] == [k + TIE_ALLOWANCE + 1 for k in range(KROW_MAX + 1)]


def test_defaults_and_linear_rule(lib):
    B, N, d, K = BENCH
    lib.check(lib.lib.b200_recommend_embed_speculation(0, 0.0))
    out = _plan(B, N, d, K)
    assert out[8] == 8
    f = out[9] / -(-N // 256)
    assert out[10 + 150] == _rank(150 + TIE_ALLOWANCE, f, 1e-5)
    # a non-zero rank coefficient selects the linear rule: pre_k = margin + ceil(c * f * k_row) in fp32
    lib.check(lib.lib.b200_recommend_embed_tune(0, 2.0))
    lib.check(lib.lib.b200_recommend_embed_debug(-12))
    lin = _plan(B, N, d, K)
    scale = np.float32(np.float32(2.0) * np.float32(lin[9])) / np.float32(-(-N // 256))
    assert lin[10:] == [12 + math.ceil(float(np.float32(scale * np.float32(k)))) for k in range(KROW_MAX + 1)]
    # ... and the speculation setter selects the failure budget again
    lib.check(lib.lib.b200_recommend_embed_speculation(0, 0.0))
    assert _plan(B, N, d, K) == out


@pytest.mark.parametrize("stride, delta", [(1, 0.0), (33, 0.0), (-8, 0.0), (8, 0.5), (8, 1e-10), (8, -1e-5)])
def test_speculation_setter_rejects_out_of_range(lib, stride, delta):
    before = _plan(*BENCH)
    assert lib.lib.b200_recommend_embed_speculation(stride, delta) != 0
    assert b"b200_recommend_embed_speculation" in lib.lib.b200_last_error()
    assert _plan(*BENCH) == before


# ------------------------------------------------------------------ the algorithm model, new rule
def _model_rows(U, I, consumed, K, stride, delta, block=16):
    """Vectorised restatement of test_k4_algorithm_model_cpu.model_row with the failure-budget rank.
    The kernel samples every stride-th 256-item tile in 128-item blocks; the model uses 16-item blocks so
    that the order statistic is meaningful on a catalogue small enough for a numpy test.
    Returns [(ids or None, status)]: 0 accepted, 2 too few collected, 3 failed speculation."""
    N, d = I.shape
    assert N % 256 == 0
    ni = float(np.linalg.norm(I.astype(np.float64), axis=1).max()) * 1.0001
    si = _pow2_scale(ni)
    Ih = _f16(I * np.float32(si))
    d_pad = -(-d // 64) * 64
    tiles = N // 256
    f = len(range(0, tiles, stride)) / tiles
    res = []
    for u, cons in zip(U, consumed):
        nu = float(np.linalg.norm(u.astype(np.float64))) * 1.0001
        su = _pow2_scale(nu)
        coarse = (Ih @ _f16(u * np.float32(su))).astype(np.float32)
        eps = (ERR_COEF + d_pad * 2.4e-7) * (nu * su) * (ni * si) + np.sqrt(d_pad) * 6.2e-5 * (nu * su + ni * si)
        apply = len(cons) > 0 and K + len(cons) <= N
        k_row = min(K + (len(cons) if apply else 0), KROW_MAX)
        pre_k = _rank(k_row + TIE_ALLOWANCE, f, delta)
        bm = coarse.reshape(tiles, 256 // block, block)[::stride].max(axis=2).ravel()
        tau = np.sort(bm)[::-1][pre_k - 1] if len(bm) >= pre_k else -np.inf
        collected = np.nonzero(coarse >= tau)[0]
        if len(collected) < k_row:
            res.append((None, 2))
            continue
        thr = np.sort(coarse[collected])[::-1][k_row - 1] - 2 * eps
        if tau > thr:
            res.append((None, 3))
            continue
        cand = collected[coarse[collected] >= thr]
        if apply:
            cand = cand[~np.isin(cand, cons)]
        ex = _exact_scores(u, I[cand])
        order = np.lexsort((cand, -ex.astype(np.float64)))
        res.append((cand[order][:K], 0))
    return res


def _reference(u, I, cons, K):
    masked = _exact_scores(u, I).astype(np.float64)
    if len(cons) and K + len(cons) <= len(I):
        masked[cons] = -np.inf
    return np.lexsort((np.arange(len(I)), -masked))[:K]


@pytest.mark.parametrize("mode", ["random", "near_ties"])
def test_model_accepted_rows_are_exact(mode):
    rng = np.random.default_rng(11 + len(mode))
    N, d, K, rows = 8192, 32, 50, 16
    I = _catalogue(rng, N, d, mode)
    U = rng.standard_normal((rows, d)).astype(np.float32)
    U /= np.linalg.norm(U, axis=1, keepdims=True)
    if mode == "near_ties":
        U = (I[0] + 0.3 * U).astype(np.float32)
    consumed = [rng.choice(N, size=int(rng.integers(0, 60)), replace=False) for _ in range(rows)]
    res = _model_rows(U, I, consumed, K, stride=4, delta=1e-3)
    for u, cons, (ids, status) in zip(U, consumed, res):
        if status == 0:
            np.testing.assert_array_equal(ids, _reference(u, I, cons, K))
        else:
            assert status in (2, 3)
    if mode == "random":
        assert sum(s == 0 for _, s in res) >= rows - 2


def test_model_failure_rate_within_budget():
    """On a random catalogue (item order independent of the scores) speculation fails on about a delta
    share of the rows or fewer; a budget well above 1e-5 makes the rate observable."""
    rng = np.random.default_rng(5)
    N, d, K, rows, delta = 20480, 32, 50, 600, 0.02
    I = _catalogue(rng, N, d, "random")
    U = rng.standard_normal((rows, d)).astype(np.float32)
    U /= np.linalg.norm(U, axis=1, keepdims=True)
    consumed = [rng.choice(N, size=int(rng.integers(0, 40)), replace=False) for _ in range(rows)]
    res = _model_rows(U, I, consumed, K, stride=4, delta=delta)
    failed = sum(s != 0 for _, s in res)
    expect = delta * rows
    assert failed <= expect + 3 * math.sqrt(expect) + 1, failed
    # the budget is spent, not wasted: a rule far more cautious than delta would never fail here
    loose = _model_rows(U[:200], I, consumed[:200], K, stride=4, delta=0.3)
    assert sum(s != 0 for _, s in loose) >= 5
