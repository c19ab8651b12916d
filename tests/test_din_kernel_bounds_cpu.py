"""Calibration of the error bounds of tests/test_gpu_din_kernels.py on the CPU.

Each bound there is C * (a per-row or per-element quantity computed from the inputs).  Here float32 restatements of
the same operations run on the same generated cases: float32 numpy / torch must meet every bound with a factor 4 to
spare (a bound float32 arithmetic cannot meet is wrong), and the worst case of each family must use at least 1/1000 of
it (a bound far looser than float32 needs would not notice a kernel that is subtly wrong).
"""
import numpy as np
import pytest

import test_gpu_din_kernels as dk
from oracle import tf_models as tm

F32, F64 = np.float32, np.float64


def _ratio(got, ref, bound, valid=None):
    """max over rows of max|got - ref| / bound (rows where ``valid`` is False are skipped)."""
    err = np.abs(np.asarray(got, dtype=F64) - ref)
    if err.ndim > 1 and bound.ndim == 1:
        err = err.reshape(len(err), -1).max(axis=1)
    if valid is not None:
        err, bound = err[valid], bound[valid]
    if err.size == 0:
        return 0.0
    return float((err / bound).max())


def _calibrate(ratios, C, what):
    worst = max(ratios)
    print(f"{what}: float32 uses {worst:.3g} of the unscaled bound, C = {C}")
    assert 4.0 * worst <= C, f"{what}: float32 error is not 4x inside the bound ({worst:.3g} * 4 > {C})"
    assert worst >= 1e-3 * C, f"{what}: bound is over 1000x looser than float32 needs ({worst:.3g} vs {C})"


def _att32(att):
    return dict(k1=att["k1"], b1=att["b1"], k2=att["k2"], b2=F32(att["b2"]))


@pytest.mark.parametrize("paper", [True, False], ids=["paper", "dot"])
def test_forward_attention_bounds(paper):
    ratios = []
    for Kp in dk.FWD_KP:
        for T in dk.FWD_T:
            c = dk.make_seq_case(1000 * Kp + T + (0 if paper else 7), Kp, T)
            q, keys, lens = dk.case_rows(c)
            q32, k32 = q.astype(F32), keys.astype(F32)
            if paper:
                ref = tm.din_attention(q, keys, lens, dk.att64(c["att"]), dtype=F64)
                got = tm.din_attention(q32, k32, lens, _att32(c["att"]), dtype=F32)
                base = dk.paper_bound(q, keys, lens, c["att"])
            else:
                ref = tm.tf_attention(q, keys, lens, dtype=F64)
                got = tm.tf_attention(q32, k32, lens, dtype=F32)
                base = dk.dot_bound(q, keys, lens)
            assert got.dtype == F32
            ratios.append(_ratio(got, ref, base, lens > 0))
    _calibrate(ratios, dk.C_ATT if paper else dk.C_DOT, "paper attention" if paper else "dot attention")


def test_dot_attention_large_logit_bound():
    ratios = []
    for Kp, T in [(32, 64), (100, 33), (12, 200)]:
        c = dk.make_seq_case(77 + Kp, Kp, T)
        c["G"] = (c["G"] * np.float32(40.0 / np.sqrt(Kp))).astype(F32)
        q, keys, lens = dk.case_rows(c)
        ref = tm.tf_attention(q, keys, lens, dtype=F64)
        got = tm.tf_attention(q.astype(F32), keys.astype(F32), lens, dtype=F32)
        assert np.isfinite(got).all()
        ratios.append(_ratio(got, ref, dk.dot_bound(q, keys, lens), lens > 0))
    _calibrate(ratios, dk.C_DOT, "dot attention, large logits")


def test_user_weights_bounds():
    ratios = []
    for Kp in (4, 36, 128):
        for L in (1, 17, 64, 65, 256):
            c = dk.make_user_case(10 * Kp + L, Kp, L, 300)
            Wt64, b64, Wmag, bmag = dk.user_weights_ref(c["G"], c["seq"], L, c["att"])
            Wt, b = dk.user_weights_f32(c["G"], c["seq"], L, c["att"])
            ratios.append(float((np.abs(Wt - Wt64) / (dk.U * Wmag)).max()))
            ratios.append(float((np.abs(b - b64) / (dk.U * bmag)).max()))
    _calibrate(ratios, dk.C_UW, "user weights")


def test_hoisted_bounds():
    ratios = []
    for N, Kp, L in dk.HOIST_CASES:
        if L == 0:
            continue
        c, Z32, ref, base = dk.hoisted_case(Kp, L, N)
        got = dk.hoisted_f32(Z32, c["G"][c["seq"][:L]], L, c["att"])
        ratios.append(_ratio(got, ref, base))
    _calibrate(ratios, dk.C_ATT, "hoisted attention")


def test_sigmoid_dot_bounds():
    ratios = []
    for L in dk.SD_LENS:
        for R in (1, 127, 129, 5003):
            c, X, Wt, bias, ref, base = dk.sigmoid_dot_case(L, R)
            got = dk.logits_f32(X, Wt, bias, c["att"]["k2"])
            ratios.append(float((np.abs(got - ref) / base).max()))
    _calibrate(ratios, dk.C_LOGIT, "sigmoid-dot logits (3xTF32 model)")


def test_from_logits_bounds():
    ratios = []
    for Kp, L in dk.FL_CASES:
        c, A32, ref, base = dk.from_logits_case(Kp, L)
        got = dk.from_logits_f32(A32, c["G"][c["seq"][:L]], c["att"]["b2"], Kp)
        ratios.append(_ratio(got, ref, base))
    _calibrate(ratios, dk.C_ATT, "attention from logits")


def test_chain_bounds():
    ratios = []
    for Kp in (32, 64, 128):
        c, ref, base = dk.chain_case(Kp)
        ratios.append(_ratio(dk.chain_f32(c, len(ref)), ref, base))
    _calibrate(ratios, dk.C_CHAIN, "all-items chain (3xTF32 model)")


def test_backward_bounds():
    import torch

    ratios = []
    for Kp, T in dk.BWD_CASES:
        c = dk.make_bwd_case(Kp * 100 + T, Kp, T)
        ref = dk.bwd_autograd(c, torch.float64)
        got = dk.bwd_autograd(c, torch.float32)
        mag = dk.bwd_magnitudes(c)
        for k in ref:
            m = mag[k] > 0
            assert (ref[k][~m] == 0).all() and (got[k][~m] == 0).all()
            ratios.append(float((np.abs(got[k] - ref[k])[m] / (dk.U * mag[k][m])).max()))
    _calibrate(ratios, dk.C_BWD, "backward")


def test_seq_pool_bounds():
    ratios = []
    for d in (1, 33, 100):
        E, seqs, lens, users, R, N, off, ref, base = dk.pool_case(d)
        Ez = E.copy()
        Ez[-1] = 0
        sr = users[(np.arange(R) + off) // N]
        inv = np.where(lens > 0, F32(1) / np.sqrt(np.maximum(lens, 1).astype(F32)), F32(0))
        got = Ez[seqs].sum(axis=1, dtype=F32)[sr] * inv[sr][:, None]
        ok = base > 0
        assert (ref[~ok] == 0).all()
        ratios.append(float((np.abs(got - ref)[ok] / base[ok]).max()))
    _calibrate(ratios, dk.C_POOL, "sequence pooling")
