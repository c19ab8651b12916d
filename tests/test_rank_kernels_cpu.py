"""Host checks behind tests/test_gpu_rank_kernels.py.

* ``fma32`` (the emulated float32 fmaf the exact-score tests compare bits with) equals exact rational arithmetic
  rounded to float32: random triples, and triples built so that the float64 sum lands exactly on a float32 midpoint
  with a nonzero error (where a float64 -> float32 cast rounds the wrong way), in the subnormal range and at overflow.
* The pair-score bounds C_PAIR * u * mag: float32 restatements of the kernels' operations on the GPU test's cases
  (fewer items) meet them with a factor 4 to spare and use at least 1/1000 of them.
* The oracle's special-value order (NaN first, -0.0 == +0.0) equals the reference's ``rank_recommendations``.
"""
from __future__ import annotations

import math
from fractions import Fraction

import numpy as np
import pytest

import _rank_kernels_ref as rk
from oracle.ref_loader import load_reference, reference_available

F32, F64 = np.float32, np.float64
FLT_MAX = float(np.finfo(F32).max)


def _round_f32(q: Fraction) -> float:
    """Round a nonzero rational to the nearest float32, ties to even, with subnormals and overflow."""
    sign = -1.0 if q < 0 else 1.0
    q = abs(q)
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1                                             # now 2^e <= q < 2^(e+1)
    e = max(e, -126)                                       # below 2^-126 the quantum stays 2^-149
    quantum = Fraction(2) ** (e - 23)
    n, rem = divmod(q, quantum)
    n = int(n)
    if rem * 2 > quantum or (rem * 2 == quantum and n % 2 == 1):
        n += 1
    v = n * quantum
    if v >= Fraction(2) ** 128:
        return sign * math.inf
    return sign * float(v)


def _exact_fma(a, b, c):
    q = Fraction(float(a)) * Fraction(float(b)) + Fraction(float(c))
    if q == 0:
        return None
    return F32(_round_f32(q))


def _check_triples(a, b, c):
    got = rk.fma32(a, b, c)
    n_checked = 0
    for x, y, z, g in zip(a, b, c, got):
        want = _exact_fma(x, y, z)
        if want is None:
            continue
        assert rk.bits(np.array([g]))[0] == rk.bits(np.array([want]))[0], (x, y, z, g, want)
        n_checked += 1
    return n_checked


def test_fma32_random_triples():
    rng = np.random.default_rng(0)
    n = 4000
    a = (rng.standard_normal(n) * 2.0 ** rng.integers(-60, 60, n)).astype(F32)
    b = (rng.standard_normal(n) * 2.0 ** rng.integers(-60, 60, n)).astype(F32)
    c = (rng.standard_normal(n) * 2.0 ** rng.integers(-120, 120, n)).astype(F32)
    assert _check_triples(a, b, c) == n


def _midpoint_triples(c, rng):
    """For each float32 c: a * b = +-(h (1 - t^2 2^-46)) with h half an ulp of c, so that c + a * b rounds in
    float64 onto the midpoint c +- h while the exact sum lies just inside it."""
    c = np.asarray(c, F32)
    # half an ulp of c (subnormal spacing below 2^-126; measured below |c| so that FLT_MAX has one)
    h = np.spacing(np.nextafter(np.abs(c), F32(0))).astype(F64) / 2
    t = rng.integers(1, 64, len(c))
    u = t * 2.0 ** -23
    eh = np.floor(np.log2(h)).astype(int)
    ka = eh // 2
    kb = eh - ka
    a = (np.ldexp(1.0 + u, ka)).astype(F32)
    b = (np.ldexp(1.0 - u, kb)).astype(F32)
    sgn = np.where(rng.random(len(c)) < 0.5, 1.0, -1.0).astype(F32)
    return a * sgn, b, c


def test_fma32_midpoints_subnormals_overflow():
    rng = np.random.default_rng(1)
    # normal range, odd and even mantissas (ties to even would go either way)
    c_norm = (rng.uniform(1.0, 2.0, 300) * 2.0 ** rng.integers(-100, 100, 300)).astype(F32)
    c_norm[::2] = np.nextafter(c_norm[::2], F32(np.inf))
    # subnormal c: half an ulp is 2^-150
    c_sub = (rng.integers(1, 2 ** 23, 200) * 2.0 ** -149).astype(F32)
    # overflow: FLT_MAX + 2^103 (1 - eps) must stay FLT_MAX, a cast of the float64 sum gives inf
    c_big = np.full(50, FLT_MAX, dtype=F32)
    c_big[::2] = -FLT_MAX
    for c in (c_norm, c_sub, c_big):
        c = np.where(rng.random(len(c)) < 0.5, c, -c).astype(F32)
        a, b, cc = _midpoint_triples(c, rng)
        p = a.astype(F64) * b.astype(F64)
        s = p + cc.astype(F64)
        with np.errstate(over="ignore"):
            naive_wrong = (s.astype(F32) != rk.fma32(a, b, cc)).sum()
        assert _check_triples(a, b, cc) == len(c)
        assert naive_wrong > 0.2 * len(c), "the cases must hit the midpoint rule"
    # plain overflow and underflow to signed zero
    a = np.array([3e38, -3e38, 1e-30, -1e-30, 1e-25], F32)
    b = np.array([10.0, 10.0, 1e-30, 1e-30, 1e-25], F32)
    c = np.array([0.0, 0.0, 0.0, 0.0, -0.0], F32)
    got = rk.fma32(a, b, c)
    assert np.isposinf(got[0]) and np.isneginf(got[1])
    assert rk.bits(got)[2] == 0 and rk.bits(got)[3] == 0x80000000 and rk.bits(got)[4] == 0


# ----- pair-score bound calibration ----------------------------------------------------------------------------------
def _ratio(got, ref, mag):
    return float((np.abs(got.astype(F64) - ref) / (rk.U * mag)).max())


def _calibrate(ratios, C, what):
    worst = max(ratios)
    print(f"{what}: float32 uses {worst / C:.3g} of the bound (C = {C}, {worst:.3g} unscaled)")
    assert 4.0 * worst <= C, f"{what}: float32 error is not 4x inside the bound"
    assert worst >= 1e-3 * C, f"{what}: bound is over 1000x looser than float32 needs"


def test_fm_pair_bound_calibration():
    import test_gpu_rank_kernels as g

    ratios = []
    for B, K, bn in [(1, 1, True), (3, 17, False), (3, 64, True), (1, 64, False)]:
        c = rk.make_fm_case(B, K, 2000, bn, seed=10 * K + B)
        items = np.arange(2000)
        ref, mag = rk.fm_pair_ref(c, np.arange(B), items)
        ratios.append(_ratio(rk.fm_pair_f32(c, np.arange(B), items), ref, mag))
    _calibrate(ratios, g.C_PAIR, "fm pair scores")


def test_deepfm_pair_bound_calibration():
    import test_gpu_rank_kernels as g

    ratios = []
    for B, K, H1, H2, H3, fm_zero in g.DEEPFM_CASES:
        c = rk.make_deepfm_case(B, K, 300, H1, H2, H3, fm_zero, seed=H1 * 7 + H2 + H3)
        items = np.arange(300)
        ref, mag = rk.deepfm_pair_ref(c, np.arange(B), items)
        ratios.append(_ratio(rk.deepfm_pair_f32(c, np.arange(B), items), ref, mag))
    _calibrate(ratios, g.C_PAIR, "deepfm pair scores")


def test_rank_order_restatement():
    """rank_order on hand-checked rows: REMOVED < -inf < ... < -0.0 == +0.0 < ... < +inf < NaN (both signs)."""
    x = np.array([[0.0, -0.0, np.nan, np.inf, -np.inf, 1e-45, -1e-45, 0.0]], F32)
    x[0, 7] = np.array([0xFFFFFFFF], np.uint32).view(F32)[0]
    x[0, 2] = np.array([0xFFC00000], np.uint32).view(F32)[0]
    assert rk.rank_order(x, 8).tolist() == [[2, 3, 5, 0, 1, 6, 4, 7]]


# ----- oracle special-value order against the reference ---------------------------------------------------------------
@pytest.mark.skipif(not reference_available(), reason="reference neither mounted nor staged")
def test_oracle_special_values_match_reference():
    from oracle.ranking import rank_recommendations as orc_rank

    load_reference()
    from libreco.recommendation.ranking import rank_recommendations as ref_rank

    rng = np.random.default_rng(3)
    N = 16
    preds = rng.standard_normal((4, N)).astype(F32)
    preds[0, 5] = np.nan
    with np.errstate(invalid="ignore"):
        preds[1, 7] = np.float32(np.inf) - np.float32(np.inf)        # x86's NaN is negative
    preds[1, 2] = np.inf
    preds[2, [1, 9]] = [-np.inf, np.inf]
    preds[3, 4] = -np.inf
    preds[3, 11] = np.nan
    consumed = {0: [1, 2], 2: [9], 3: [0, 0]}
    users = [0, 1, 2, 3]
    for n_rec in (1, 3, 12):
        want = ref_rank("rating", users, preds, n_rec, N, consumed, True, False, False)
        got = orc_rank("rating", users, preds, n_rec, N, consumed, True)
        np.testing.assert_array_equal(got, want, err_msg=f"n_rec={n_rec}")
