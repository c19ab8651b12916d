"""Host checks behind tests/test_gpu_seq_pair_kernels.py.

* Calibration: float32 restatements of the Transformer, SIM and AutoInt kernels (tests/_seq_pair_kernels_ref.py) on
  the GPU test's cases, with fewer items, use at most 1/4 of each bound C * u * mag and at least 1/1000 of it.
* Discrimination: subtly wrong arithmetic (a softmax over one key fewer, an unclamped length, the last Pi chunk
  dropped, Pu added twice, GSU ties to the higher position, the ESU mask applied by rank) exceeds the bound on every
  GPU case it changes.
* Selection: the dyadic Gp of the SIM cases makes every GSU and short-attention dot exact in float32 (checked
  against rational arithmetic), and masked logits below 32 in magnitude shift to exactly -1e9.
"""
from __future__ import annotations

from fractions import Fraction

import numpy as np
import pytest

import _seq_pair_kernels_ref as sp
import test_gpu_seq_pair_kernels as g
from test_rank_kernels_cpu import _calibrate, _ratio

F32, F64 = np.float32, np.float64
N_CAL = 96                          # items per case for the float32 restatements


def _tfm_cases():
    for B, N, T, D, H1, H2, H3 in g.TFM_CASES:
        yield (B, N, T, D, H1, H2, H3), sp.make_tfm_case(B, N_CAL, T, D, H1, H2, H3, seed=N + D + H1, ldq_pad=3,
                                                         ldpi_pad=5)


def _sim_cases():
    for B, N, K, H, L, S, topk, H1, H2, H3 in g.SIM_CASES:
        yield (B, N, K, H, L, S, topk), sp.make_sim_case(B, N_CAL, K, H, L, S, topk, H1, H2, H3, seed=N + K)


def _ai_cases():
    for B, N, K, H, hds, res, field_map, nu, ni in g.AI_CASES:
        Bc, Nc = min(B, 12), min(N or N_CAL, N_CAL)
        Xu, Xi, w, layers, w_out, b_out = g._ai_setup(Bc, Nc, K, H, hds, field_map, nu, ni, seed=B + (N or 7))
        uu, ii = np.repeat(np.arange(Bc), Nc), np.tile(np.arange(Nc), Bc)
        yield (K, H, hds, res), sp.autoint_block(Xu, Xi, field_map, K, uu, ii), layers, w_out, b_out


# ----- calibration ---------------------------------------------------------------------------------------------------
def test_transformer_pair_bound_calibration():
    ratios = []
    items = np.arange(N_CAL)
    for _, c in _tfm_cases():
        for b in range(len(c["lens"])):
            ref, mag = sp.tfm_pair_ref(c, b, items)
            ratios.append(_ratio(sp.tfm_pair_f32(c, b, items), ref, mag))
    _calibrate(ratios, g.C_TFM, "transformer pair scores")


def test_transformer_rows_bound_calibration():
    ratios = []
    items = np.arange(N_CAL)
    for _, c in _tfm_cases():
        for b in range(len(c["lens"])):
            slots = np.full(N_CAL, b)
            ref, mag = sp.tfm_rows_ref(c["Qi"], c["S"], c["lens"], slots, items)
            ratios.append(_ratio(sp.tfm_rows_f32(c["Qi"], c["S"], c["lens"], b, items), ref, mag))
    _calibrate(ratios, g.C_TFM, "transformer rows")


def test_sim_pair_bound_calibration():
    ratios = []
    items = np.arange(N_CAL)
    for _, c in _sim_cases():
        for b in range(len(c["long_lens"])):
            ref, mag = sp.sim_pair_ref(c, b, items)
            ratios.append(_ratio(sp.sim_pair_f32(c, b, items), ref, mag))
    _calibrate(ratios, g.C_SIM_PAIR, "sim pair scores")


def test_sim_rows_bound_calibration():
    ratios = []
    items = np.arange(N_CAL)
    for _, c in _sim_cases():
        for b in range(len(c["long_lens"])):
            ref, mag, _ = sp.sim_rows_ref(c, np.full(N_CAL, b), items)
            ratios.append(_ratio(sp.sim_rows_f32(c, b, items), ref, mag))
    _calibrate(ratios, g.C_SIM_ROWS, "sim rows")


def test_autoint_bound_calibration():
    ratios = []
    for (_, _, _, res), X, layers, w_out, b_out in _ai_cases():
        ref, mag = sp.autoint_ref(X, layers, w_out, b_out, res)
        ratios.append(_ratio(sp.autoint_f32(X, layers, w_out, b_out, res), ref, mag))
    _calibrate(ratios, g.C_AI, "autoint")


def test_autoint_ref_matches_layerwise_float64():
    """autoint_ref's value is the block through mha_keras + residual, then Dense(1), as a plain float64 loop."""
    for (K, H, hds, res), X, layers, w_out, b_out in _ai_cases():
        x = X.astype(F64)
        for lw in layers:
            y = np.zeros_like(x)
            for r in range(len(x)):
                for h in range(H):
                    Wq, Wk, Wv = (np.asarray(lw[m], F64)[:, h] for m in ("query", "key", "value"))
                    q, k, v = x[r] @ Wq, x[r] @ Wk, x[r] @ Wv
                    s = q @ k.T / np.sqrt(Wq.shape[1])
                    p = np.exp(s - s.max(axis=1, keepdims=True))
                    p /= p.sum(axis=1, keepdims=True)
                    y[r] += (p @ v) @ np.asarray(lw["attention_output"], F64)[h]
            x = x + y if res else y
        want = x.reshape(len(x), -1) @ np.asarray(w_out, F64) + b_out
        got, _ = sp.autoint_ref(X, layers, w_out, b_out, res)
        np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-12)


# ----- discrimination ------------------------------------------------------------------------------------------------
def _exceeds(got, ref, mag, C):
    return bool((np.abs(got.astype(F64) - ref) > C * sp.U * mag).any())


def _check_mutant(cases, users, ref_fn, f32_fn, C, mutant):
    """Every case whose arithmetic the mutant changes rejects it on some element; most cases are changed."""
    items = np.arange(N_CAL)
    changed = 0
    for shape, c in cases:
        diff = rejected = False
        for b in range(users(c)):
            bad, good = f32_fn(c, b, items, mutant=mutant), f32_fn(c, b, items)
            if np.array_equal(bad, good):
                continue                                      # the mutant does not change this user's arithmetic
            diff = True
            ref, mag = ref_fn(c, b, items)
            rejected = rejected or _exceeds(bad, ref, mag, C)
        assert rejected or not diff, f"{mutant} passes the bound on every user of {shape}"
        changed += diff
    assert 2 * changed > len(cases), f"{mutant} changes too few cases"


@pytest.mark.parametrize("mutant", ["nk_minus_1", "len_unclamped", "drop_last_pi_chunk", "pu_twice"])
def test_transformer_bound_rejects_mutants(mutant):
    _check_mutant(list(_tfm_cases()), lambda c: len(c["lens"]), sp.tfm_pair_ref, sp.tfm_pair_f32, g.C_TFM, mutant)


@pytest.mark.parametrize("mutant", ["gsu_tie_high", "esu_mask_rank"])
def test_sim_bound_rejects_mutants(mutant):
    _check_mutant(list(_sim_cases()), lambda c: len(c["long_lens"]), sp.sim_pair_ref, sp.sim_pair_f32, g.C_SIM_PAIR,
                  mutant)


# ----- selection -----------------------------------------------------------------------------------------------------
def _exact_dot(a, b):
    return sum((Fraction(float(x)) * Fraction(float(y)) for x, y in zip(a, b)), Fraction(0))


def test_dyadic_dots_are_exact_in_float32():
    rng = np.random.default_rng(0)
    for K, lim in ((8, 1.0), (33, 1.0), (64, 0.75), (64, 2.0)):
        q = sp.dyadic(rng, (40, K), lim)
        G = sp.dyadic(rng, (50, K), lim)
        assert (np.abs(q) <= lim).all() and (q * 8 == np.round(q * 8)).all()
        chain = np.zeros((40, 50), F32)
        for d in range(K):
            chain = sp.fma32(q[:, d:d + 1], G[None, :, d], chain)
        for i in range(0, 40, 7):
            for j in range(0, 50, 5):
                assert Fraction(float(chain[i, j])) == _exact_dot(q[i], G[j]), (K, i, j)
        np.testing.assert_array_equal(chain.astype(F64), q.astype(F64) @ G.astype(F64).T)


def test_sim_cases_selection_inputs():
    """The SIM cases' Gp is dyadic apart from the NaN row, whose -inf scores lose to every masked position, and
    every case has exact ties at user 3's top-k cut."""
    for shape, c in _sim_cases():
        K = c["K"]
        Gp = c["Gp"][:, :K]
        nan_row = Gp.shape[0] - 1
        assert np.isnan(Gp[nan_row]).all() and not np.isnan(Gp[:nan_row]).any()
        assert (Gp[:nan_row] * 8 == np.round(Gp[:nan_row] * 8)).all() and np.abs(Gp[:nan_row]).max() <= 2
        items = np.arange(N_CAL)
        assert sp.gsu_ties_at_cut(c, 3, items).any(), shape
        for b in range(len(c["long_lens"])):
            sel = sp.gsu_select(sp.gsu_scores(c, b, Gp[items]), c["topk"])
            assert not (c["long_seqs"][b][sel] == nan_row).any(), (shape, b)
        # the ties: equal scores resolve to the lower position
        s = sp.gsu_scores(c, 3, Gp[items])
        lo, hi = sp.gsu_select(s, c["topk"]), sp.gsu_select(s, c["topk"], high_ties=True)
        assert (lo != hi).any(axis=1).any() and (lo.sum(axis=1) <= hi.sum(axis=1)).all()


def test_masked_logits_shift_exactly():
    x = np.linspace(-31.9, 31.9, 2001).astype(F32)
    assert (x - F32(sp.NEG) == F32(-sp.NEG)).all()
    assert F32(40.0) - F32(sp.NEG) != F32(-sp.NEG)
    # a row whose keys are all hidden: weights exactly 1 / nk
    for nk in (1, 3, 10, 64):
        p = sp._f32_softmax(np.full((1, nk), -sp.NEG, F32) + F32(0), False, nk)
        assert (p == F32(1) / F32(nk)).all()
