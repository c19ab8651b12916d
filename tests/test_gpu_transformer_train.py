"""GPU: Transformer training.

* Each new kernel through the C-ABI against torch float64 (autograd where there is a backward) with per-element
  bounds (below; ``test_transformer_train_cpu.py`` shows a float32 restatement meets each with 4x to spare and uses
  at least 1/1000 of it): the masked attention core (T 1 / 10 / 33 / 64, D up to 128, 1 / 2 / 5 heads, causal on and
  off, lens 1 .. T, strided inputs, logits around +-100), rms_norm (near-zero rows included), the swish / gelu
  activations (0 and large |x|), the target-attention backward; every one of them repeats bit for bit.
* ``training.TransformerTrainer`` against the float64 restatement in ``tests/_transformer_train_oracle.py`` (parity
  unpinned, see its header) over keras / legacy x causal x trainable / sinusoidal positions x BN on / off x ids-only /
  item sparse and dense features: logits, loss and every raw gradient of one batch, parameters after a step, the loss
  over three steps, BN moving statistics, ``step_graph``, ``set_regularisation``, the exported weights in
  ``feat_models.Transformer`` and through a ``_tf_variables.npz`` round trip, and ``ValueError`` before any launch."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _transformer_oracle as to  # noqa: E402
import _transformer_train_oracle as tto  # noqa: E402

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24

# ---------------------------------------------------------------------------------------------------------------
# attention core: cases and bounds (shared with the CPU calibration)
# ---------------------------------------------------------------------------------------------------------------
# (R, T, H, hd, causal)
KERNEL_CASES = [
    (37, 1, 1, 8, False), (37, 1, 2, 64, True), (37, 10, 2, 16, False), (37, 10, 1, 32, True), (37, 33, 5, 3, False),
    (37, 33, 5, 3, True), (9, 64, 1, 128, True), (9, 64, 2, 64, False), (9, 64, 5, 25, True), (2000, 10, 2, 16, True),
]
C_O, C_LSE, C_DV, C_DQK = 8.0, 16.0, 8.0, 8.0


def kernel_case_id(c):
    return "R{}-T{}-H{}-hd{}-causal{}".format(*c)


def make_kernel_case(c, large=False, seed=0):
    """float32 Q, K, V, dO [R, T, D] and lens [R] (1, T and everything between); ``large`` scales Q so the largest
    logit is about 100."""
    R, T, H, hd, _ = c
    rng = np.random.default_rng(seed + 1000 * T + 10 * hd + H)
    D = H * hd
    q, k, v, do = (rng.standard_normal((R, T, D)).astype(np.float32) for _ in range(4))
    if large:
        s = np.abs(np.einsum("rfhd,rghd->rhfg", q.reshape(R, T, H, hd), k.reshape(R, T, H, hd))).max() / np.sqrt(hd)
        q = (q * (100.0 / s)).astype(np.float32)
    lens = rng.integers(1, T + 1, R).astype(np.int32)
    lens[:2] = [1, T]
    return q, k, v, do, lens


def reference(q, k, v, do, lens, H, causal, dtype):
    """torch autograd of the masked core in ``dtype``: numpy (O, lse, dQ, dK, dV)."""
    import torch

    hd = q.shape[2] // H
    t = [torch.tensor(a, dtype=dtype, requires_grad=True) for a in (q, k, v)]
    sc = 1.0 / np.sqrt(hd) if dtype == torch.float64 else float(np.float32(1.0 / np.sqrt(hd)))
    o, lse = tto.attention_core(*t, lens, H, sc, causal)
    (o * torch.as_tensor(do, dtype=dtype)).sum().backward()
    return [a.detach().numpy() for a in (o, lse)] + [a.grad.numpy() for a in t]


def bounds(q, k, v, do, lens, H, causal):
    """Per-element bounds of (O, lse, dQ, dK, dV): C * u32 * (T + hd + A) * G, per (row, head) A = the largest
    scale * sum_j |q_fj k_gj| over visible pairs and G the magnitude each output is built from (float64)."""
    R, T, D = q.shape
    hd = D // H
    sc = 1.0 / np.sqrt(hd)
    sp = lambda a: a.astype(np.float64).reshape(R, T, H, hd).transpose(0, 2, 1, 3)      # noqa: E731
    Q, K, V, dO = sp(q), sp(k), sp(v), sp(do)
    mask = tto.attention_mask(np.asarray(lens), T, causal).numpy()[:, None]              # [R, 1, T, T]
    s = np.where(mask, Q @ K.transpose(0, 1, 3, 2) * sc, -np.inf)
    P = np.exp(s - s.max(-1, keepdims=True))
    P /= P.sum(-1, keepdims=True)
    O = P @ V
    dP = dO @ V.transpose(0, 1, 3, 2)
    Dr = (dO * O).sum(-1, keepdims=True)
    A = np.where(mask, np.abs(Q) @ np.abs(K).transpose(0, 1, 3, 2) * sc, 0.0).max(axis=(2, 3))   # [R, H]
    amp = U32 * (T + hd + A)[:, :, None, None]
    W = P * (np.abs(dP) + np.abs(Dr))
    mx = lambda a: np.abs(a).max(axis=(2, 3), keepdims=True)                            # noqa: E731
    back = lambda a: np.broadcast_to(a, (R, H, T, hd)).transpose(0, 2, 1, 3).reshape(R, T, D)   # noqa: E731
    bO = back(C_O * amp * mx(V))
    bL = C_LSE * amp[:, :, :, 0] * np.ones((R, H, T))
    bdV = back(C_DV * amp * P.sum(2).max(-1)[:, :, None, None] * mx(dO))
    bdQ = back(C_DQK * amp * sc * W.sum(-1).max(-1)[:, :, None, None] * mx(K))
    bdK = back(C_DQK * amp * sc * W.sum(2).max(-1)[:, :, None, None] * mx(Q))
    return bO, bL, bdQ, bdK, bdV


def _run_core(q, k, v, do, lens, H, causal, strided=False):
    """The two kernels on device copies; returns numpy (O, lse, dQ, dK, dV) and the launch count they took."""
    import torch

    from librecommender_b200 import _lib

    R, T, D = q.shape
    hd = D // H
    dev = torch.device("cuda")
    if strided:                         # Q / K / V as column slices of one [R*T, 3D] buffer
        buf = torch.as_tensor(np.concatenate([q, k, v], axis=2).reshape(R * T, 3 * D), device=dev)
        Q, K, V = buf[:, :D], buf[:, D:2 * D], buf[:, 2 * D:]
    else:
        Q, K, V = (torch.as_tensor(a.reshape(R * T, D), device=dev) for a in (q, k, v))
    dO = torch.as_tensor(do.reshape(R * T, D), device=dev)
    L = torch.as_tensor(lens, device=dev)
    O = torch.full((R * T, D), float("nan"), device=dev)
    lse = torch.full((R * H * T,), float("nan"), device=dev)
    dQ, dK, dV = (torch.full((R * T, D), float("nan"), device=dev) for _ in range(3))
    sc = float(np.float32(1.0 / np.sqrt(hd)))
    st = _lib.current_stream()
    n0 = _lib.launch_count()
    _lib.check(_lib.lib.b200_transformer_attention_forward(
        _lib.ptr(Q), Q.stride(0), _lib.ptr(K), K.stride(0), _lib.ptr(V), V.stride(0), _lib.ptr(L), R, T, H, hd,
        int(causal), sc, _lib.ptr(O), O.stride(0), _lib.ptr(lse), st))
    _lib.check(_lib.lib.b200_transformer_attention_backward(
        _lib.ptr(Q), Q.stride(0), _lib.ptr(K), K.stride(0), _lib.ptr(V), V.stride(0), _lib.ptr(O), O.stride(0),
        _lib.ptr(lse), _lib.ptr(dO), dO.stride(0), _lib.ptr(L), R, T, H, hd, int(causal), sc, _lib.ptr(dQ),
        _lib.ptr(dK), _lib.ptr(dV), D, st))
    torch.cuda.synchronize()
    out = [O.cpu().numpy().reshape(R, T, D), lse.cpu().numpy().reshape(R, H, T)]
    out += [a.cpu().numpy().reshape(R, T, D) for a in (dQ, dK, dV)]
    return out, _lib.launch_count() - n0


def _check(names, got, ref, bnds):
    for name, g, r, b in zip(names, got, ref, bnds):
        assert np.isfinite(g).all(), name
        err = np.abs(g.astype(np.float64) - r)
        assert (err <= b).all(), (name, float((err / b).max()))


def _check_core(c, large=False, strided=False):
    import torch

    q, k, v, do, lens = make_kernel_case(c, large)
    H, causal = c[2], c[4]
    got, n = _run_core(q, k, v, do, lens, H, causal, strided)
    assert n == 2
    _check(("O", "lse", "dQ", "dK", "dV"), got, reference(q, k, v, do, lens, H, causal, torch.float64),
           bounds(q, k, v, do, lens, H, causal))
    return got


@pytest.mark.parametrize("c", KERNEL_CASES, ids=kernel_case_id)
def test_attention_core_matches_fp64_autograd(c):
    got = _check_core(c)
    # hidden keys get exactly zero gradient from the rows that cannot see them
    q, k, v, do, lens = make_kernel_case(c)
    R, T, H, hd, causal = c
    if not causal:
        for r in range(R):
            assert not got[3][r, lens[r]:].any() and not got[4][r, lens[r]:].any()


@pytest.mark.parametrize("c", [KERNEL_CASES[3], KERNEL_CASES[5], KERNEL_CASES[8]], ids=kernel_case_id)
def test_attention_core_strided_rows_and_bit_identical_repeats(c):
    a = _check_core(c, strided=True)
    q, k, v, do, lens = make_kernel_case(c)
    b, _ = _run_core(q, k, v, do, lens, c[2], c[4], strided=True)
    contiguous, _ = _run_core(q, k, v, do, lens, c[2], c[4])
    for x, y, z in zip(a, b, contiguous):
        np.testing.assert_array_equal(x, y)
        np.testing.assert_array_equal(x, z)


@pytest.mark.parametrize("c", [(37, 10, 2, 16, True), (9, 64, 1, 128, False)], ids=kernel_case_id)
def test_attention_core_large_logits(c):
    q, k, v, _, _ = make_kernel_case(c, large=True)
    R, T, H, hd, _ = c
    s = np.einsum("rfhd,rghd->rhfg", q.reshape(R, T, H, hd).astype(np.float64),
                  k.reshape(R, T, H, hd).astype(np.float64)) / np.sqrt(hd)
    assert np.abs(s).max() > 80
    _check_core(c, large=True)


def test_attention_core_autoint_envelope_unchanged():
    """The masked core with lens = T and no causal flag is the AutoInt core: same bits on the shared envelope."""
    import torch

    from librecommender_b200 import _lib

    q, k, v, do, _ = make_kernel_case((37, 33, 2, 8, False))
    lens = np.full(37, 33, np.int32)
    got, _ = _run_core(q, k, v, do, lens, 2, False)
    dev = torch.device("cuda")
    Q, K, V, dO = (torch.as_tensor(a.reshape(37 * 33, 16), device=dev) for a in (q, k, v, do))
    O, dQ, dK, dV = (torch.empty((37 * 33, 16), device=dev) for _ in range(4))
    lse = torch.empty(37 * 2 * 33, device=dev)
    sc = float(np.float32(1.0 / np.sqrt(8)))
    st = _lib.current_stream()
    _lib.check(_lib.lib.b200_autoint_attention_forward(_lib.ptr(Q), 16, _lib.ptr(K), 16, _lib.ptr(V), 16, 37, 33, 2, 8,
                                                       sc, _lib.ptr(O), 16, _lib.ptr(lse), st))
    _lib.check(_lib.lib.b200_autoint_attention_backward(_lib.ptr(Q), 16, _lib.ptr(K), 16, _lib.ptr(V), 16, _lib.ptr(O),
                                                        16, _lib.ptr(lse), _lib.ptr(dO), 16, 37, 33, 2, 8, sc,
                                                        _lib.ptr(dQ), _lib.ptr(dK), _lib.ptr(dV), 16, st))
    for a, b in zip(got, (O, lse, dQ, dK, dV)):
        np.testing.assert_array_equal(a.reshape(-1), b.cpu().numpy().reshape(-1))


# ---------------------------------------------------------------------------------------------------------------
# rms_norm, activations, target-attention backward
# ---------------------------------------------------------------------------------------------------------------
C_RMS, C_ACT, C_TA = 8.0, 16.0, 8.0
RMS_CASES = [(300, 1), (300, 32), (300, 80), (1000, 128), (7, 512)]


def make_rms_case(R, D, seed=0):
    """x [R, D] with rows of magnitude 1e-6 .. 1e3 and all-zero rows, scale, dy."""
    rng = np.random.default_rng(seed + D)
    x = rng.standard_normal((R, D)) * (10.0 ** rng.uniform(-6, 3, (R, 1)))
    x[0] = 0.0
    x[1] = 1e-7 * rng.standard_normal(D)
    return (x.astype(np.float32), rng.uniform(0.5, 1.5, D).astype(np.float32),
            rng.standard_normal((R, D)).astype(np.float32))


def rms_reference(x, scale, dy, dtype):
    """torch (y, rstd, dx, dscale) in ``dtype``."""
    import torch

    xt = torch.tensor(x, dtype=dtype, requires_grad=True)
    st = torch.tensor(scale, dtype=dtype, requires_grad=True)
    rs = torch.rsqrt(xt.square().mean(-1, keepdim=True) + 1e-8)
    y = xt * rs * st
    (y * torch.as_tensor(dy, dtype=dtype)).sum().backward()
    return y.detach().numpy(), rs.detach().numpy().reshape(-1), xt.grad.numpy(), st.grad.numpy()


def rms_bounds(x, scale, dy):
    """C * u32 * (D + 8) * the magnitude each output is built from."""
    x, s, dy = (a.astype(np.float64) for a in (x, scale, dy))
    D = x.shape[1]
    rs = 1.0 / np.sqrt(np.mean(x * x, axis=1, keepdims=True) + 1e-8)
    amp = C_RMS * U32 * (D + 8)
    g = np.abs(dy * s)
    by = amp * np.abs(x) * rs * s
    br = amp * rs.reshape(-1)
    bdx = amp * rs * (g + np.abs(x) * rs * rs * (g * np.abs(x)).sum(1, keepdims=True) / D)
    bds = amp * (np.abs(dy) * np.abs(x) * rs).sum(0)
    return [b + 1e-37 for b in (by, br, bdx, bds)]          # the zero row: exact zeros


def _run_rms(x, scale, dy):
    import torch

    from librecommender_b200 import _lib

    R, D = x.shape
    dev = torch.device("cuda")
    X, S, dY = (torch.as_tensor(a, device=dev) for a in (x, scale, dy))
    Y, dX = (torch.full((R, D), float("nan"), device=dev) for _ in range(2))
    rs = torch.full((R,), float("nan"), device=dev)
    ds = torch.zeros(D, device=dev)
    st = _lib.current_stream()
    _lib.check(_lib.lib.b200_rms_norm_forward(_lib.ptr(X), D, R, D, _lib.ptr(S), _lib.ptr(Y), D, _lib.ptr(rs), st))
    _lib.check(_lib.lib.b200_rms_norm_backward(_lib.ptr(dY), D, _lib.ptr(X), D, _lib.ptr(rs), R, D, _lib.ptr(S),
                                               _lib.ptr(dX), D, st))
    _lib.check(_lib.lib.b200_col_reduce(_lib.ptr(dY), D, R, D, _lib.ptr(rs), _lib.ptr(X), D, _lib.ptr(ds), st))
    return [a.cpu().numpy() for a in (Y, rs, dX, ds)]


@pytest.mark.parametrize("R,D", RMS_CASES)
def test_rms_norm_matches_fp64(R, D):
    import torch

    x, s, dy = make_rms_case(R, D)
    got = _run_rms(x, s, dy)
    _check(("y", "rstd", "dx", "dscale"), got, rms_reference(x, s, dy, torch.float64), rms_bounds(x, s, dy))
    again = _run_rms(x, s, dy)
    for a, b in zip(got[:3], again[:3]):
        np.testing.assert_array_equal(a, b)


ACT_CODES = {"swish": 2, "gelu": 3}


def act_inputs():
    base = np.linspace(-12, 12, 4001)
    special = [0.0, -0.0, 1e-30, -1e-30, 1e-7, -1e-7, 50.0, -50.0, 100.0, -100.0, 1e4, -1e4, 3e38, -3e38]
    return np.concatenate([base, special]).astype(np.float32)


def act_reference(x, act, dtype):
    """torch (y, dy/dx) in ``dtype``."""
    import torch

    xt = torch.tensor(x, dtype=dtype, requires_grad=True)
    y = xt * torch.sigmoid(xt) if act == "swish" else 0.5 * xt * (1.0 + torch.erf(xt / np.sqrt(2.0)))
    y.sum().backward()
    return y.detach().numpy(), xt.grad.numpy()


def act_bounds(x, act):
    """(bound of y, bound of dy/dx): C * u32 * the magnitude of the terms each is formed from.  gelu's
    1 + erf(x / sqrt 2) carries an absolute rounding of about u32, hence |x| in its bound; the derivative's second
    term x e(x) (e = the gaussian density for gelu, sigmoid (1 - sigmoid) for swish) cancels against the first."""
    x = x.astype(np.float64)
    with np.errstate(over="ignore"):
        if act == "gelu":
            from scipy.special import erf
            y, e = 0.5 * x * (1.0 + erf(x / np.sqrt(2.0))), np.exp(-0.5 * x * x)
            return C_ACT * U32 * (np.abs(y) + np.abs(x)) + 1e-37, C_ACT * U32 * (1.0 + np.abs(x) * e)
        sg = 1.0 / (1.0 + np.exp(-x))
        y, e = x * sg, sg * (1.0 - sg)
        # 1 - sigmoid(x) in float32 carries an absolute rounding of about u32 for x >> 0: |x| in the derivative's bound
        return C_ACT * U32 * (np.abs(y) + np.abs(x) * e) + 1e-37, C_ACT * U32 * (1.0 + np.abs(x))


def _run_act(x, act):
    import torch

    from librecommender_b200 import _lib

    dev = torch.device("cuda")
    X = torch.as_tensor(x, device=dev)
    ones = torch.ones_like(X)
    Y, dX = torch.empty_like(X), torch.empty_like(X)
    st = _lib.current_stream()
    _lib.check(_lib.lib.b200_activation_forward(_lib.ptr(X), X.numel(), ACT_CODES[act], _lib.ptr(Y), st))
    _lib.check(_lib.lib.b200_activation_backward(_lib.ptr(ones), _lib.ptr(X), X.numel(), ACT_CODES[act], _lib.ptr(dX),
                                                 st))
    return [Y.cpu().numpy(), dX.cpu().numpy()]


@pytest.mark.parametrize("act", sorted(ACT_CODES))
def test_activations_match_fp64(act):
    import torch

    x = act_inputs()
    got = _run_act(x, act)
    ref = [np.nan_to_num(a) for a in act_reference(x, act, torch.float64)]
    _check(("y", "dy/dx"), got, ref, act_bounds(x, act))
    assert (got[0][x == 0] == 0).all() and (got[1][x == 0] == 0.5).all()
    for a, b in zip(got, _run_act(x, act)):
        np.testing.assert_array_equal(a, b)


# (R, T, D)
TA_CASES = [(300, 1, 32), (300, 10, 32), (300, 50, 80), (64, 64, 128), (100, 33, 7)]


def make_ta_case(R, T, D, seed=0, large=False):
    """q [R, D], S [R, T, D], lens [R] (1 .. T), dout [R, D]."""
    rng = np.random.default_rng(seed + 100 * T + D)
    q = rng.standard_normal((R, D)).astype(np.float32)
    S = rng.standard_normal((R, T, D)).astype(np.float32)
    if large:
        q = (q * (100.0 / np.abs(np.einsum("rd,rtd->rt", q, S)).max())).astype(np.float32)
    lens = rng.integers(1, T + 1, R).astype(np.int32)
    lens[:2] = [1, T]
    return q, S, lens, rng.standard_normal((R, D)).astype(np.float32)


def ta_reference(q, S, lens, dout, dtype):
    """torch autograd of the target attention in ``dtype``: (dq, dS)."""
    import torch

    qt = torch.tensor(q, dtype=dtype, requires_grad=True)
    St = torch.tensor(S, dtype=dtype, requires_grad=True)
    T = S.shape[1]
    a = torch.einsum("rd,rtd->rt", qt, St)
    m = torch.arange(T)[None, :] < torch.as_tensor(lens).reshape(-1, 1)
    p = torch.softmax(torch.where(m, a, torch.full_like(a, -np.inf)), dim=1)
    ((p[:, :, None] * St).sum(1) * torch.as_tensor(dout, dtype=dtype)).sum().backward()
    return qt.grad.numpy(), St.grad.numpy()


def ta_bounds(q, S, lens, dout):
    """C * u32 * (T + D + A) * magnitude, A = max_t sum_d |q_d S_td| over the visible keys (float64)."""
    q, S, dout = (a.astype(np.float64) for a in (q, S, dout))
    T = S.shape[1]
    m = np.arange(T)[None, :] < lens[:, None]
    a = np.where(m, np.einsum("rd,rtd->rt", q, S), -np.inf)
    p = np.exp(a - a.max(1, keepdims=True))
    p /= p.sum(1, keepdims=True)
    out = np.einsum("rt,rtd->rd", p, S)
    b = np.einsum("rd,rtd->rt", dout, S)
    c = (dout * out).sum(1, keepdims=True)
    A = np.where(m, np.einsum("rd,rtd->rt", np.abs(q), np.abs(S)), 0).max(1)
    amp = C_TA * U32 * (T + S.shape[2] + A)[:, None]
    W = p * (np.abs(b) + np.abs(c))
    Sm = np.abs(S).max(axis=(1, 2))[:, None]
    bdq = amp * W.sum(1, keepdims=True) * Sm
    bdS = amp[:, :, None] * (p[:, :, None] * np.abs(dout).max(1)[:, None, None] + W[:, :, None] * np.abs(q).max(1)[:, None, None]) + 1e-30
    return bdq, bdS


def _run_ta(q, S, lens, dout):
    import torch

    from librecommender_b200 import _lib

    R, T, D = S.shape
    dev = torch.device("cuda")
    Q, St, L, dO = (torch.as_tensor(a, device=dev) for a in (q, S, lens, dout))
    dq = torch.full((R, D), float("nan"), device=dev)
    dS = torch.full((R, T, D), float("nan"), device=dev)
    n0 = _lib.launch_count()
    _lib.check(_lib.lib.b200_transformer_target_attention_backward(_lib.ptr(Q), D, _lib.ptr(St), T, D, _lib.ptr(L),
                                                                   _lib.ptr(dO), D, R, _lib.ptr(dq), D, _lib.ptr(dS),
                                                                   _lib.current_stream()))
    assert _lib.launch_count() == n0 + 1
    return [dq.cpu().numpy(), dS.cpu().numpy()]


@pytest.mark.parametrize("R,T,D", TA_CASES)
@pytest.mark.parametrize("large", [False, True])
def test_target_attention_backward_matches_fp64_autograd(R, T, D, large):
    import torch

    q, S, lens, dout = make_ta_case(R, T, D, large=large)
    got = _run_ta(q, S, lens, dout)
    _check(("dq", "dS"), got, ta_reference(q, S, lens, dout, torch.float64), ta_bounds(q, S, lens, dout))
    for r in range(R):
        assert not got[1][r, lens[r]:].any()
    for a, b in zip(got, _run_ta(q, S, lens, dout)):
        np.testing.assert_array_equal(a, b)


def test_kernels_reject_shapes_before_launch():
    import test_transformer_train_cpu as cpu

    cpu.test_cabi_rejects_unsupported_shapes_before_launch()


# ---------------------------------------------------------------------------------------------------------------
# the trainer against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------
# (layout, K, num_heads, n_layers, causal, positional, use_bn, version, T)
TRAIN_CASES = [
    ("ids", 16, 1, 1, False, "trainable", True, "keras", 10),        # the reference defaults (D = 32)
    ("feat", 16, 2, 2, True, "sinusoidal", True, "legacy", 10),      # D = 96
    ("feat", 8, 4, 1, False, "trainable", False, "keras", 33),       # D = 48
    ("ids", 8, 2, 2, True, "trainable", False, "legacy", 20),        # D = 16
    ("feat", 16, 3, 1, True, "sinusoidal", False, "keras", 10),
    ("ids", 16, 2, 1, False, "sinusoidal", True, "legacy", 50),
    ("ids", 7, 2, 1, True, "trainable", True, "keras", 10),          # odd K, D = 14
]
# logits rtol = atol = 3e-5 and loss 2e-5 as in test_gpu_din_train.py; gradients <= GRAD_REL * max|ref| +
# GRAD_ABS * (largest gradient of the batch), calibrated in test_transformer_train_cpu.py::test_trainer_bounds
GRAD_REL, GRAD_ABS = 2e-4, 4e-6


def train_case_id(c):
    return "-".join(str(v) for v in c)


def train_batch(c, seed=0, R=512, n_batches=3, n_users=80, n_items=120):
    """(spec, raw weights, [(users, items, seqs [R, T], lens, sparse, dense, labels)] x n_batches).  Rows 0..3 are
    the first position of a history (len 1 holding the pad id), rows 4..7 full; the others len 1 .. T padded with
    the pad id."""
    from oracle import tf_models as tm

    layout, K, H, L, causal, pos, bn, version, T = c
    _, spec, w, _, _ = to.make_case((layout, K, "concat", H, L, causal, pos, bn, version), seed, n_users, n_items, T)
    rng = np.random.default_rng(seed + 7)
    batches = []
    for _ in range(n_batches):
        users, items = rng.integers(0, n_users, R), rng.integers(0, n_items, R)
        lens = rng.integers(1, T + 1, R).astype(np.int32)
        lens[4:8] = T
        seqs = rng.integers(0, n_items, (R, T)).astype(np.int32)
        seqs[np.arange(T)[None, :] >= lens[:, None]] = n_items
        lens[:4] = 1
        seqs[:4] = n_items
        sparse, dense = tm.row_features(spec, users, items)
        batches.append((users, items, seqs, lens, sparse, dense, (rng.random(R) < 0.35).astype(np.float32)))
    return spec, w, batches


def _cu(a):
    import torch

    return torch.as_tensor(np.asarray(a)).cuda()


def _grad_name(k):
    if k.startswith("W") and k[1:].isdigit():
        return "Wt" + k[1:], True
    return k, False


def _got(tr, k, shape, src="grads"):
    name, transposed = _grad_name(k)
    got = getattr(tr, src)[name].cpu().numpy().astype(np.float64)
    return (got.T if transposed else got).reshape(shape)


def _trainer(spec, w, c, **kw):
    from librecommender_b200.training import TransformerTrainer

    return TransformerTrainer(spec, w, use_bn=c[6], **kw)


@pytest.mark.parametrize("c", TRAIN_CASES, ids=train_case_id)
def test_gradients_of_one_batch_match_oracle(c):
    import torch

    spec, w, batches = train_batch(c)
    users, items, seqs, lens, sparse, dense, labels = batches[0]
    tr = _trainer(spec, w, c)
    st = tto.init_state(w, c[6])
    ref_loss, ref_out, ref_g, _ = tto.forward_backward(st, spec, users, items, seqs, lens, sparse, dense, labels)
    logits = tr.forward(_cu(users), _cu(items), _cu(seqs), _cu(lens))
    np.testing.assert_allclose(logits.cpu().numpy(), ref_out, rtol=3e-5, atol=3e-5)
    loss = tr.backward(_cu(labels))
    torch.cuda.synchronize()
    assert abs(float(loss) - ref_loss) < 2e-5
    assert {_grad_name(k)[0] for k in ref_g} == set(tr.grads)
    gmax = max(np.abs(v).max() for v in ref_g.values())
    for k, ref in ref_g.items():
        got = _got(tr, k, ref.shape)
        scale = np.abs(ref).max()
        assert np.abs(got - ref).max() <= GRAD_REL * scale + GRAD_ABS * gmax, (k, float(np.abs(got - ref).max()), scale,
                                                                              gmax)


@pytest.mark.parametrize("c", [TRAIN_CASES[0], TRAIN_CASES[1], TRAIN_CASES[3]], ids=train_case_id)
def test_training_steps_match_oracle_and_export(c, tmp_path):
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import Transformer

    spec, w, batches = train_batch(c, 11)
    lr, eps = 1e-2, 1e-5
    tr = _trainer(spec, w, c, lr=lr, epsilon=eps)
    st = tto.init_state(w, c[6])
    for step, (users, items, seqs, lens, sparse, dense, labels) in enumerate(batches):
        ref_loss = tto.train_step(st, spec, users, items, seqs, lens, sparse, dense, labels, lr, eps)
        loss = tr.step(_cu(users), _cu(items), _cu(seqs), _cu(lens), _cu(labels))
        assert abs(float(loss) - ref_loss) <= 1e-3 * max(1.0, abs(ref_loss)) * (step + 1), (step, float(loss), ref_loss)
        if step == 0:
            for k, ref in st["params"].items():
                got = _got(tr, k, ref.shape, "params")
                assert np.abs(got - ref).max() <= 2e-2 * lr + 1e-6, (k, float(np.abs(got - ref).max()))
    if c[6]:
        for name, (mm, mv) in st["moving"].items():
            gm, gv = (a.cpu().numpy().astype(np.float64) for a in tr.moving[name])
            np.testing.assert_allclose(gm, mm, rtol=1e-3, atol=1e-3 * np.abs(mm).max() + 1e-6)
            np.testing.assert_allclose(gv, mv, rtol=1e-3, atol=1e-3 * np.abs(mv).max() + 1e-6)
    # export: the raw layout of the same scheme, straight into the inference engine
    raw = tr.export_weights()
    assert raw["tfm_scheme"] == w["tfm_scheme"]
    for a, b in zip(raw["tfm_layers"], w["tfm_layers"]):
        assert {k: v.shape for k, v in a.items()} == {k: np.shape(v) for k, v in b.items()}
    assert ("positional_encoding" in raw) == (c[5] == "trainable")
    T = c[8]
    _, _, _, seqs, lens = to.make_case(("ids", c[1], "concat", c[2], c[3], c[4], c[5], c[6], c[7]), 3, spec["n_users"],
                                       spec["n_items"], T)
    lens = np.maximum(lens, 1)
    model = Transformer(spec, wio.transformer_weights(raw), seqs, lens)
    rng = np.random.default_rng(3)
    users, items, sparse, dense = to.case_rows(rng, spec, R=300)
    got = model.logits(users, items).cpu().numpy()
    # the exported weights are the trainer's; the oracle's inference forward on them
    to.close(got, to.transformer_forward(raw, spec, users, items, seqs, lens, sparse, dense))
    # ... and on the float64 oracle's own trained weights (BN moving statistics included)
    to.close(got, to.transformer_forward(tto.raw_weights(st, w), spec, users, items, seqs, lens, sparse, dense),
             tol=3e-3)
    # a save as the reference's <name>_tf_variables.npz and a reload give the same logits bit for bit
    np.savez(tmp_path / "m_tf_variables.npz", **wio.transformer_tf_variables(raw))
    back = wio.load_reference_tf_model(str(tmp_path), "m", "Transformer", len(raw["mlp"]["kernels"]), c[6],
                                       num_heads=c[2], num_tfm_layers=c[3], positional_embedding=c[5],
                                       use_causal_mask=c[4])
    np.testing.assert_array_equal(Transformer(spec, back, seqs, lens).logits(users, items).cpu().numpy(), got)


def test_graph_replay_equals_eager_steps():
    spec, w, batches = train_batch(TRAIN_CASES[1], 21)
    c = TRAIN_CASES[1]
    a = _trainer(spec, w, c, lr=1e-2)
    b = _trainer(spec, w, c, lr=1e-2)
    for users, items, seqs, lens, _, _, labels in batches:
        args = [_cu(x) for x in (users, items, seqs, lens, labels)]
        la = float(a.step(*args))
        lb = float(b.step_graph(*args))
        assert abs(la - lb) <= 1e-5 * max(1.0, abs(la)), (la, lb)
    assert a.t == b.t == 3 and int(b._step_dev.item()) == 3
    assert b.graph_launches_per_step > 30
    for k in a.params:
        d = (a.params[k] - b.params[k]).abs().max().item()
        assert d <= 2e-4, (k, d)          # float atomics in the table scatters: order differs run to run


def test_regularisation_and_lr_decay_match_oracle():
    from librecommender_b200.training import set_regularisation

    c = TRAIN_CASES[0]
    spec, w, batches = train_batch(c, 31, n_batches=2)
    lr, eps, reg = 1e-2, 1e-5, 3e-3
    tr = set_regularisation(_trainer(spec, w, c, lr=lr, epsilon=eps), reg=reg, lr_decay=True, decay_steps=2,
                            decay_rate=0.5)
    plain = _trainer(spec, w, c, lr=lr, epsilon=eps)
    st = tto.init_state(w, c[6])
    for step, (users, items, seqs, lens, sparse, dense, labels) in enumerate(batches + batches):
        ref_loss = tto.train_step(st, spec, users, items, seqs, lens, sparse, dense, labels, lr, eps, reg=reg,
                                  decay_steps=2, decay_rate=0.5)
        args = [_cu(x) for x in (users, items, seqs, lens, labels)]
        loss = tr.step(*args)
        plain.step(*args)
        assert abs(float(loss) - ref_loss) <= 2e-3 * max(1.0, abs(ref_loss)) * (step + 1), (step, float(loss), ref_loss)
    moved = 0.0
    for k in tto.TABLES:
        if k not in st["params"]:
            continue
        ref = st["params"][k]
        got = tr.params[k].cpu().numpy().astype(np.float64).reshape(ref.shape)
        assert np.abs(got - ref).max() <= 0.12 * lr * 3, (k, float(np.abs(got - ref).max()))
        assert np.median(np.abs(got - ref)) <= 0.01 * lr, (k, float(np.median(np.abs(got - ref))))
        moved = max(moved, float((tr.params[k] - plain.params[k]).abs().max()))
    assert moved > 0.5 * lr          # the regulariser + decay changed the trajectory
    # no regulariser on the positions: the same gradient path as the plain trainer up to the tables' influence
    assert "positional_encoding" not in tr.reg_vars


@pytest.mark.parametrize("what", ["elementwise", "multi_sparse", "T", "width", "layers", "heads", "mlp_input",
                                  "batch_T"])
def test_trainer_rejects_before_launch(what):
    from librecommender_b200 import _lib
    from librecommender_b200 import synthetic as syn

    rng = np.random.default_rng(8)
    spec = syn.make_spec(rng, 20, 30, [3], [4], 1, 1)
    K, H, L, T, mode = 8, 2, 1, 10, "concat"
    if what == "multi_sparse":
        spec = syn.make_multi_sparse_spec(rng, 20, 30, [9], [12, 6], [("user", 17, 3), ("item", 23, 2)], 1, 1)
    elif what == "T":
        T = 65
    elif what == "width":
        K = 40                           # K' = 120, D = 160
    elif what == "layers":
        L = 5
    elif what == "elementwise":
        mode = "elementwise"
    w = syn.make_transformer_weights(rng, spec, K, H, L, T, (16, 8), True, "trainable", False, mode, "keras")
    if what == "heads":
        w["num_heads"] = 5               # D = 32 is not a multiple of 5
    elif what == "mlp_input":
        w["mlp"]["kernels"][0] = w["mlp"]["kernels"][0][:-1]
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        tr = _trainer(spec, w, (None,) * 6 + (True,))
        if what == "batch_T":            # a batch whose length differs from the positional table's rows
            seqs = np.zeros((4, T + 1), np.int32)
            tr.step(_cu(np.zeros(4, np.int64)), _cu(np.zeros(4, np.int64)), _cu(seqs), _cu(np.ones(4, np.int32)),
                    _cu(np.zeros(4, np.float32)))
    assert _lib.launch_count() == n0
