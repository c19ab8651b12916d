"""Host checks behind tests/test_gpu_seq_encoder_kernels.py.

* Calibration: float32 restatements of the RNN, Caser and WaveNet kernels (tests/_seq_encoder_kernels_ref.py) on the
  GPU test's cases, with fewer slots (and, for the RNN, at most 8 steps; for Caser, the cases whose restatement is
  cheap), use at most 1/4 of each bound C * u * mag and at least 1/1000 of it.
* Discrimination: each subtly wrong variant of the arithmetic is rejected by the checks on every case it changes.
* Restatements: the float64 RNN backward (fed its own gate gradients) equals torch float64 autograd of the
  recurrence, and the Caser backward equals autograd of the convolution and max-pool.
"""
from __future__ import annotations

import functools

import numpy as np
import pytest

import _seq_encoder_kernels_ref as se
import test_gpu_seq_encoder_kernels as g
from test_rank_kernels_cpu import _calibrate, _ratio

F32, F64 = np.float32, np.float64
N_CAL = 6
T_CAL = 8


def _ratios(checks):
    """Worst err / (u * mag) over the checks' inexact elements; the exact ones (mag = 0) must match."""
    worst = 0.0
    for what, got, ref, mag in checks:
        got = np.asarray(got, F64)
        exact = mag == 0
        assert (got[exact] == ref[exact]).all(), f"{what}: an exact element differs"
        if (~exact).any():
            worst = max(worst, _ratio(got[~exact], ref[~exact], mag[~exact]))
    return worst


def _rejects(checks, C):
    try:
        return _ratios(checks) > C
    except AssertionError:
        return True


def _rnn_cases():
    for n, T, in0, kinds, Hs, acts in g.RNN_CASES:
        yield (kinds, Hs, acts), se.make_rnn_case(N_CAL, min(T, T_CAL), in0, kinds, Hs, acts, seed=n + T)


@functools.lru_cache(maxsize=None)
def _rnn_runs():
    """(shape, case, out, saved) of the float32 forward on every case, computed once."""
    return [(shape, c, *se.rnn_forward_f32(c)) for shape, c in _rnn_cases()]


def _rnn_grads(c, l, rng):
    H = c["Hs"][l]
    if l == len(c["Hs"]) - 1:
        return rng.uniform(-1, 1, (c["n"], H)).astype(F32), None
    return None, rng.uniform(-1, 1, (c["n"] * c["T"], H)).astype(F32)


CASER_CAL = [k for k in g.CASER_CASES if k[1] * (k[1] + 1) // 2 * k[2] <= 8192]


def _caser_cases():
    for n, T, K, nh, nv in CASER_CAL:
        yield (n, T, K, nh, nv), se.make_caser_case(min(n, N_CAL), T, K, nh, nv, seed=n + T * K)


def _wavenet_cases():
    for n, T, K, F, dils in g.WAVENET_CASES:
        yield (n, T, K, F, len(dils)), se.make_wavenet_case(min(n, 4), T, K, F, dils, seed=n + T + K)


# ----- calibration ---------------------------------------------------------------------------------------------------
def test_rnn_forward_bound_calibration():
    ratios = []
    for _, c, out, saved in _rnn_runs():
        ratios.append(_ratios(se.rnn_forward_checks(c, saved, out)))
    _calibrate(ratios, g.C_RNN_FWD, "rnn forward")


def test_rnn_backward_bound_calibration():
    ratios = []
    rng = np.random.default_rng(0)
    for _, c, _, saved in _rnn_runs():
        for l in range(len(c["Hs"])):
            dout, dy = _rnn_grads(c, l, rng)
            got = se.rnn_backward_f32(c, l, saved[l], dout, dy)
            ratios.append(_ratios(se.rnn_backward_checks(c, l, saved[l], got, dout, dy)))
    _calibrate(ratios, g.C_RNN_BWD, "rnn backward")


def test_caser_bound_calibration():
    ratios = []
    rng = np.random.default_rng(1)
    for _, c in _caser_cases():
        out, arg = se.caser_forward_f32(c)
        ratios.append(_ratios(se.caser_forward_checks(c, out)))
        assert not se.caser_argmax_violations(c, out, arg, g.C_CASER)
        dF = rng.uniform(-1, 1, out.shape).astype(F32)
        dX, dW = se.caser_backward_f32(c, dF, out, arg)
        ratios.append(_ratios(se.caser_backward_checks(c, dF, out, arg, dX, dW)))
    _calibrate(ratios, g.C_CASER, "caser")


def test_wavenet_bound_calibration():
    ratios = []
    for _, c in _wavenet_cases():
        out, ys, arg = se.wavenet_forward_f32(c)
        checks, (z, mz) = se.wavenet_forward_checks(c, out, ys)
        ratios.append(_ratios(checks))
        assert not se.argmax_violations(z, mz, arg, out, se.wavenet_windows(c), g.C_WAVENET)
    _calibrate(ratios, g.C_WAVENET, "wavenet")


def test_case_tables_reach_the_kernel_edges():
    E = [se.caser_floats(*k[1:5]) for k in g.CASER_DW_CASES]
    chunks = [se.caser_nchunk(k[0], e) for k, e in zip(g.CASER_DW_CASES, E)]
    assert chunks[0] > 1 and -(-g.CASER_DW_CASES[0][0] // 256) == chunks[0], "chunks set by rows"
    assert 1 < chunks[1] < -(-g.CASER_DW_CASES[1][0] // 256), "chunks capped by the partial budget"
    assert E[2] > se.CONV_PART_FLOATS and chunks[2] == 1 and g.CASER_DW_CASES[2][0] > 256
    assert {se.caser_tile(T, K) for _, T, K, _, _ in g.CASER_CASES} >= {2, 3, 32}
    assert {se.wavenet_tile(T, K, F) for _, T, K, F, _ in g.WAVENET_CASES} >= {1, 2, 31, 32}
    assert max(se.elem_passes(n * T * C) for n, T, C in g.HELPER_CASES) >= 3


# ----- discrimination ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mutant", ["gru_r_without_bh", "ln_eps", "no_freeze", "drop_last_w"])
def test_rnn_forward_rejects_mutants(mutant):
    changed = 0
    for shape, c, out, saved in _rnn_runs():
        bout, bsaved = se.rnn_forward_f32(c, mutant=mutant)
        same = np.array_equal(out, bout) and all(
            a is None or np.array_equal(a, b) for sv, bsv in zip(saved, bsaved) for a, b in zip(sv, bsv))
        if same:
            continue
        changed += 1
        assert _rejects(se.rnn_forward_checks(c, bsaved, bout), g.C_RNN_FWD), f"{mutant} passes on {shape}"
    assert changed, f"{mutant} changes no case"


@pytest.mark.parametrize("mutant", ["dgh_no_r", "ln_bwd_no_qx", "lstm_dc_no_f", "tf1_dd_no_r", "len0_row"])
def test_rnn_backward_rejects_mutants(mutant):
    changed = 0
    for shape, c, _, saved in _rnn_runs():
        for l in range(len(c["Hs"])):
            dout, dy = _rnn_grads(c, l, np.random.default_rng(l))
            good = se.rnn_backward_f32(c, l, saved[l], dout, dy)
            bad = se.rnn_backward_f32(c, l, saved[l], dout, dy, mutant=mutant)
            if all(good[k] is None or np.array_equal(good[k], bad[k]) for k in good):
                continue
            changed += 1
            assert _rejects(se.rnn_backward_checks(c, l, saved[l], bad, dout, dy), g.C_RNN_BWD), \
                f"{mutant} passes on {shape} layer {l}"
    assert changed, f"{mutant} changes no case"


def test_caser_rejects_ties_to_the_highest_position():
    changed = 0
    for shape, c in _caser_cases():
        out, arg = se.caser_forward_f32(c)
        bout, barg = se.caser_forward_f32(c, mutant="tie_high")
        if np.array_equal(arg, barg):
            continue
        changed += 1
        assert se.caser_argmax_violations(c, bout, barg, g.C_CASER), shape
    assert changed


def test_wavenet_rejects_ties_to_the_highest_position():
    changed = 0
    for shape, c in _wavenet_cases():
        out, ys, arg = se.wavenet_forward_f32(c)
        bout, bys, barg = se.wavenet_forward_f32(c, mutant="tie_high")
        if np.array_equal(arg, barg):
            continue
        changed += 1
        _, (z, mz) = se.wavenet_forward_checks(c, bout, bys)
        assert se.argmax_violations(z, mz, barg, bout, se.wavenet_windows(c), g.C_WAVENET), shape
    assert changed


@pytest.mark.parametrize("mutant", ["vmask_df", "dw_drop_last_chunk"])
def test_caser_backward_rejects_mutants(mutant):
    cases = list(_caser_cases()) + [((600, 5, 3, 5, 5), se.make_caser_case(600, 5, 3, 5, 5, seed=600))]
    changed = 0
    for shape, c in cases:
        out, arg = se.caser_forward_f32(c)
        dF = np.random.default_rng(3).uniform(-1, 1, out.shape).astype(F32)
        dX, dW = se.caser_backward_f32(c, dF, out, arg)
        bX, bW = se.caser_backward_f32(c, dF, out, arg, mutant=mutant)
        if np.array_equal(dX, bX) and np.array_equal(dW, bW):
            continue
        changed += 1
        assert _rejects(se.caser_backward_checks(c, dF, out, arg, bX, bW), g.C_CASER), f"{mutant} passes on {shape}"
    assert changed


@pytest.mark.parametrize("n,T,C", [(5, 8, 3), (2, 64, 4), (7, 3, 1)])
def test_wavenet_helper_mutants_change_bits(n, T, C):
    rng = np.random.default_rng(T)
    x = rng.uniform(-1, 1, (n * T, C)).astype(F32)
    P = rng.uniform(-1, 1, (n * T, 2 * C)).astype(F32)
    for d in range(1, T):
        assert not np.array_equal(se.wavenet_layer_inputs_ref(x, n, T, C, d),
                                  se.wavenet_layer_inputs_ref(x, n, T, C, d, mutant="cross_slot")), d
        assert not np.array_equal(se.wavenet_layer_dx_ref(P, n, T, C, d),
                                  se.wavenet_layer_dx_ref(P, n, T, C, d, mutant="guard_le")), d


# ----- restatements against torch float64 autograd -------------------------------------------------------------------
def _torch_layer(c, l, x, dout, dy):
    """Layer l of c in torch float64 on inputs x [n, T, in] with the kernel's freezing past len: the saved tensors in
    the kernel layout, and the gradients of sum(dout * out) (top) or sum_t<len(dy_t * y_t) with respect to
    per-step perturbations of the x part (dgx), the h part (dgh) and the layer-norm pre-activation (dln)."""
    import torch

    lw, T, n = c["layers"][l], c["T"], c["n"]
    kind, H, act = lw["kind"], lw["H"], c["acts"][l]
    GH = se.gates(kind) * H
    t64 = lambda a: torch.tensor(np.asarray(a, F64))  # noqa: E731
    W, Uw, bx, bh, gm, bt = (t64(lw[k]) for k in ("W", "U", "bx", "bh", "gamma", "beta"))
    Ls = se.slot_lens(c)
    x = t64(x)
    ex = torch.zeros(T, n, GH, dtype=torch.float64, requires_grad=True)
    eh = torch.zeros(T, n, GH, dtype=torch.float64, requires_grad=True)
    el = torch.zeros(T, n, H, dtype=torch.float64, requires_grad=True)
    sv = [np.zeros((n * T, H)), np.zeros((n * T, H)), np.zeros((n * T, GH)), np.zeros((n * T, H)),
          np.zeros((n * T, H)), np.zeros(n * T)]
    h = torch.zeros(n, H, dtype=torch.float64)
    cs = torch.zeros(n, H, dtype=torch.float64)
    fa = (lambda v: torch.tanh(v)) if act == se.ACT_TANH else (lambda v: v)
    loss = torch.zeros((), dtype=torch.float64)
    for t in range(T):
        on = torch.tensor(t < Ls)[:, None]
        ax = x[:, t] @ W + bx + ex[t]
        if kind == se.LSTM:
            v = ax + h @ Uw + bh + eh[t]
            i, f, gg, o = torch.sigmoid(v[:, :H]), torch.sigmoid(v[:, H:2 * H]), fa(v[:, 2 * H:3 * H]), \
                torch.sigmoid(v[:, 3 * H:])
            cn = f * cs + i * gg
            hn = o * fa(cn)
            G, X = torch.cat([i, f, gg, o], 1), cn
        elif kind == se.GRU_KERAS:
            ah = h @ Uw + bh + eh[t]
            z, r = torch.sigmoid(ax[:, :H] + ah[:, :H]), torch.sigmoid(ax[:, H:2 * H] + ah[:, H:2 * H])
            hh = fa(ax[:, 2 * H:] + r * ah[:, 2 * H:])
            hn = z * h + (1 - z) * hh
            G, X = torch.cat([z, r, hh], 1), ah[:, 2 * H:]
        else:
            ah = h @ Uw[:, :2 * H] + bh[:2 * H] + eh[t][:, :2 * H]
            z, r = torch.sigmoid(ax[:, :H] + ah[:, :H]), torch.sigmoid(ax[:, H:2 * H] + ah[:, H:2 * H])
            rh = r * h
            cc = fa(ax[:, 2 * H:] + rh @ Uw[:, 2 * H:] + bh[2 * H:] + eh[t][:, 2 * H:])
            hn = z * h + (1 - z) * cc
            G, X = torch.cat([z, r, cc], 1), rh
        rows = np.nonzero(t < Ls)[0] * T + t
        act_np = t < Ls
        sv[0][rows] = h.detach().numpy()[act_np]
        h = torch.where(on, hn, h)
        cs = torch.where(on, cn, cs) if kind == se.LSTM else cs
        if act == se.ACT_LN:
            mu = h.mean(1, keepdim=True)
            rs = 1 / torch.sqrt(((h - mu) ** 2).mean(1, keepdim=True) + se.LN_EPS)
            xh = (h - mu) * rs
            y = torch.tanh(xh * gm + bt + el[t])
            sv[4][rows] = xh.detach().numpy()[act_np]
            sv[5][rows] = rs.detach().numpy()[act_np, 0]
        else:
            y = h
        sv[1][rows] = y.detach().numpy()[act_np]
        sv[2][rows] = G.detach().numpy()[act_np]
        sv[3][rows] = X.detach().numpy()[act_np]
        if dy is not None:
            loss = loss + (torch.tensor(dy[np.arange(n) * T + t], dtype=torch.float64) * y)[torch.tensor(act_np)].sum()
        else:
            pick = (t == Ls - 1) | ((Ls == 0) & (t == 0) & (act == se.ACT_LN))
            loss = loss + (torch.tensor(dout, dtype=torch.float64) * y)[torch.tensor(pick)].sum()
    loss.backward()
    grads = dict(dgx=ex.grad.numpy().transpose(1, 0, 2).reshape(n * T, GH),
                 dgh=eh.grad.numpy().transpose(1, 0, 2).reshape(n * T, GH),
                 dln=None if el.grad is None else el.grad.numpy().transpose(1, 0, 2).reshape(n * T, H))
    return sv, grads


@pytest.mark.parametrize("kind", [0, 1, 2])
@pytest.mark.parametrize("act", [0, 1])
@pytest.mark.parametrize("top", [True, False])
def test_rnn_backward_restatement_matches_autograd(kind, act, top):
    c = se.make_rnn_case(7, 6, 3, [kind], [5], [act], seed=kind * 4 + act)
    rng = np.random.default_rng(kind)
    x = rng.uniform(-1, 1, (c["n"], c["T"], 3))
    dout = rng.uniform(-1, 1, (c["n"], 5)) if top else None
    dy = None if top else rng.uniform(-1, 1, (c["n"] * c["T"], 5))
    sv, want = _torch_layer(c, 0, x, dout, dy)
    if not act:
        sv[4], sv[5] = None, None
    got = se.rnn_backward_ref(c, 0, sv, dout, dy)
    np.testing.assert_allclose(got["dgx"][0], want["dgx"], rtol=1e-10, atol=1e-12)
    if kind == se.GRU_KERAS:
        np.testing.assert_allclose(got["dgh"][0], want["dgh"], rtol=1e-10, atol=1e-12)
    if act:
        np.testing.assert_allclose(got["dln"][0], want["dln"], rtol=1e-10, atol=1e-12)


def test_caser_backward_restatement_matches_autograd():
    import torch

    n, T, K, nh, nv = 5, 6, 4, 3, 2
    c = se.make_caser_case(n, T, K, nh, nv, seed=9, n_items=200, patterns=False)
    x = torch.tensor(se.gathered(c).astype(F64), requires_grad=True)
    w = torch.tensor(c["w"].astype(F64), requires_grad=True)
    Wh, bh, Wv, bv, off = [], None, None, None, 0
    for h in range(1, T + 1):
        Wh.append(w[off:off + h * K * nh].reshape(h, K, nh))
        off += h * K * nh
    bh = w[off:off + T * nh].reshape(T, nh)
    Wv = w[off + T * nh:off + T * nh + T * nv].reshape(T, nv)
    bv = w[off + T * nh + T * nv:]
    cols, args = [], []
    for h in range(1, T + 1):
        npos = T - h + 1
        pre = bh[h - 1] + sum(x[:, j:j + npos] @ Wh[h - 1][j] for j in range(h))
        m, a = torch.relu(pre).max(1)
        cols.append(m)
        args.append(torch.where(pre.max(1).values > 0, a, torch.full_like(a, -1)))
    vert = torch.relu(torch.einsum("stk,tf->skf", x, Wv) + bv).reshape(n, -1)
    out = torch.cat(cols + [vert], 1)
    dF = np.random.default_rng(2).uniform(-1, 1, tuple(out.shape)).astype(F32).astype(F64)
    (out * torch.tensor(dF)).sum().backward()
    arg = torch.cat(args, 1).numpy().astype(np.int32)
    (dX, _), (dW, _) = se.caser_backward_ref(c, dF, out.detach().numpy(), arg)
    np.testing.assert_allclose(dX, x.grad.numpy().reshape(n * T, K), rtol=1e-6, atol=1e-7)
    np.testing.assert_allclose(dW, w.grad.numpy(), rtol=1e-6, atol=1e-7)
