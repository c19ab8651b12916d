"""The loss kernels of ``csrc/loss.cu``, called directly through the C-ABI and compared with the float64 restatements
of tests/_loss_kernels_ref.py: ``b200_pairwise_loss`` (BPR, max-margin, pairwise sigmoid CE and focal),
``b200_pointwise_loss`` focal at gamma 0 ... 5, ``b200_softmax_inbatch_loss`` and ``b200_sampled_class_loss``, then
the ``losses.py`` wrappers around them.

Every trainer's loss runs through these kernels, and the reference's torch models train on them through
``dropin.install``.  Here each kernel runs where it branches: one positive, factors 1 / 3 / 17, n_pos past the
262 144-thread grid, pairs exactly on the max-margin hinge, saturated scores; in-batch rows of one and two columns,
partial last warps, B > 8192 (a warp takes a second row), lds > B, temperature 0, corrections clipped at both ends,
rows whose every off-diagonal is an accidental hit; sampled rows with S = 1, S not a multiple of 32, S = 65 536,
several hits in one row, every sampled id a hit, num_tries > S, n_items = S and near 2^31, ld > S.

The error bounds and their constants are stated in tests/_loss_kernels_ref.py and calibrated on the CPU by
tests/test_loss_kernel_bounds_cpu.py.  Where the kernel is exact the test is exact: max-margin gradients, masked and
hit gradients (0.0), temperature 0 (every gradient 0.0), S under ``write_grad = 0`` (bit for bit), the padding
columns and one NaN sentinel element / row after every output (still NaN), repeated calls (same bits).
"""
from __future__ import annotations

import numpy as np
import pytest

import _loss_kernels_ref as R

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
NAN = float("nan")


def _dev(a):
    import torch

    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _nan(*shape):
    import torch

    return torch.full(shape, NAN, dtype=torch.float32, device="cuda")


def _host(t):
    import torch

    torch.cuda.synchronize()
    return t.cpu().numpy()


def _ws(nbytes):
    import torch

    return torch.empty(max(int(nbytes), 8), dtype=torch.uint8, device="cuda")


def _check(got, ref, bound, what):
    """|got - ref| <= bound elementwise (exact where the bound is 0); prints the worst ratio of error to bound."""
    err = np.abs(np.asarray(got, dtype=F64) - ref)
    bound = np.broadcast_to(np.asarray(bound, dtype=F64), err.shape)
    bad = ~(err <= bound)
    pos = bound > 0
    worst = float((err[pos] / bound[pos]).max()) if pos.any() else 0.0
    print(f"RATIO {what.split(',')[0]}: {worst:.3g}")
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err / np.maximum(bound, 1e-300), 0.0) + bad), err.shape)
        raise AssertionError(f"{what}: {int(bad.sum())} elements over the bound, worst at {i}: got "
                             f"{np.asarray(got)[i]!r} ref {ref[i] if np.ndim(ref) else ref!r} bound {bound[i]:.3e}")


# ---------------------------------------------------------------------------------------------------------------------
# pairwise
# ---------------------------------------------------------------------------------------------------------------------
def _pairwise(pos, neg, kind, margin=0.0, mean=True, gamma=2.0):
    """(loss, dpos, dneg) of one b200_pairwise_loss call; every output has one NaN sentinel element after it."""
    from librecommender_b200 import _lib

    p, q = _dev(pos), _dev(neg)
    loss, dp, dn = _nan(2), _nan(len(pos) + 1), _nan(len(neg) + 1)
    ws = _ws(_lib.lib.b200_loss_workspace_bytes())
    _lib.check(_lib.lib.b200_pairwise_loss(_lib.ptr(p), len(pos), _lib.ptr(q), len(neg), kind, float(margin),
                                           R.ALPHA, float(gamma), 1 if mean else 0, _lib.ptr(loss), _lib.ptr(dp),
                                           _lib.ptr(dn), _lib.ptr(ws), ws.numel(), _lib.current_stream()))
    loss, dp, dn = _host(loss), _host(dp), _host(dn)
    assert np.isnan(loss[1]) and np.isnan(dp[-1]) and np.isnan(dn[-1]), "wrote past an output"
    return loss[0], dp[:-1], dn[:-1]


def _pair_params():
    for n_pos, f in R.PAIR_SHAPES:
        for kind in (0, 1, 2, 3):
            for margin in (R.MARGINS if kind == 1 else (0.0,)):
                for mean in ((True, False) if kind >= 2 else (True,)):
                    yield pytest.param(n_pos, f, kind, margin, mean, id=f"{n_pos}x{f}-k{kind}-m{margin}-mean{int(mean)}")


@pytest.mark.parametrize("n_pos,factor,kind,margin,mean", list(_pair_params()))
def test_pairwise_matches_fp64(n_pos, factor, kind, margin, mean):
    pos, neg = R.make_pair_case(n_pos, factor, kind, margin)
    ref = R.pairwise_ref(pos, neg, kind, margin, mean)
    L, dp, dn = _pairwise(pos, neg, kind, margin, mean)
    C = R.C_PAIR
    _check(dp, ref["dpos"], C * ref["b_dpos"], f"pairwise, d pos, kind {kind}")
    _check(dn, ref["dneg"], C * ref["b_dneg"], f"pairwise, d neg, kind {kind}")
    _check(L, ref["loss"], C * ref["b_loss"], f"pairwise, loss, kind {kind}")
    if kind == 1:                     # exact: every gradient is a whole number times the float 1 / n_neg
        inv = F32(1) / F32(len(neg))
        np.testing.assert_array_equal(dn, np.rint(ref["dneg"] * len(neg)).astype(F32) * inv)
        np.testing.assert_array_equal(dp, np.rint(ref["dpos"] * len(neg)).astype(F32) * inv)


def test_pairwise_rejects_bad_arguments_without_a_launch():
    import torch

    from librecommender_b200 import _lib

    lib, P = _lib.lib, _lib.ptr
    p, q = torch.zeros(4, device="cuda"), torch.zeros(12, device="cuda")
    loss, dp, dn = _nan(1), _nan(4), _nan(12)
    ws = _ws(lib.b200_loss_workspace_bytes())
    n0 = _lib.launch_count()
    args = lambda n_neg, kind, nws: (P(p), 4, P(q), n_neg, kind, 0.0, 0.25, 2.0, 1, P(loss), P(dp), P(dn),  # noqa
                                     P(ws), nws, _lib.current_stream())
    assert lib.b200_pairwise_loss(*args(10, 0, ws.numel())) == -2            # n_neg % n_pos != 0
    assert lib.b200_pairwise_loss(*args(10, 1, ws.numel())) == -2
    assert lib.b200_pairwise_loss(*args(12, 4, ws.numel())) == -2            # no kind 4
    for kind in range(4):
        assert lib.b200_pairwise_loss(*args(12, kind, ws.numel() - 1)) == -2  # workspace too small
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0
    assert np.isnan(_host(loss)).all() and np.isnan(_host(dp)).all() and np.isnan(_host(dn)).all()


# ---------------------------------------------------------------------------------------------------------------------
# pointwise focal at several gamma, saturated logits
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("gamma", R.FOCAL_GAMMAS)
def test_pointwise_focal_gamma_matches_fp64(gamma):
    from librecommender_b200 import _lib

    x, y = R.make_focal_case()
    n = len(x)
    xd, yd = _dev(x), _dev(y)
    loss, dl = _nan(2), _nan(n + 1)
    ws = _ws(_lib.lib.b200_loss_workspace_bytes())
    _lib.check(_lib.lib.b200_pointwise_loss(_lib.ptr(xd), _lib.ptr(yd), n, 1, R.ALPHA, float(gamma),
                                            _lib.ptr(loss), _lib.ptr(dl), _lib.ptr(ws), ws.numel(),
                                            _lib.current_stream()))
    v, g, vm, gm = R.pointwise_elems(x, y, 1, R.ALPHA, gamma)
    got, L = _host(dl), _host(loss)
    assert np.isnan(got[n]) and np.isnan(L[1])
    got = got[:n]
    assert np.isfinite(got).all()
    _check(got, g / n, R.C_PAIR * (R.U * gm / n + R.ETA), f"pointwise focal, gradient, gamma {gamma}")
    _check(L[0], v.sum() / n, R.C_PAIR * R.U * (R.grid_rounds(n) + 2) * vm.sum() / n, "pointwise focal, loss")
    if gamma > 0:                     # 1 - p_t == 0 in float: (1 - p_t)^gamma = 0 and its derivative is taken as 0
        sat = (np.abs(x) >= 88) & ((x > 0) == (y > 0))
        assert sat.any() and (got[sat] == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# in-batch softmax
# ---------------------------------------------------------------------------------------------------------------------
def _inbatch(c, write_grad):
    """(loss, S buffer after the call [B + 1, lds]); the padding columns and the sentinel row start as NaN."""
    from librecommender_b200 import _lib

    B, lds = c["B"], c["B"] + c["pad"]
    buf = _nan(B + 1, lds)
    buf[:B, :B] = _dev(c["S"])
    corr = _dev(c["corr"]) if c["corr"] is not None else None
    ids = _dev(c["ids"]) if c["ids"] is not None else None
    loss = _nan(2)
    ws = _ws(_lib.lib.b200_loss_workspace_bytes())
    _lib.check(_lib.lib.b200_softmax_inbatch_loss(_lib.ptr(buf), lds, B, c["temperature"], _lib.ptr(corr),
                                                  _lib.ptr(ids), write_grad, _lib.ptr(loss), _lib.ptr(ws),
                                                  ws.numel(), _lib.current_stream()))
    L = _host(loss)
    assert np.isnan(L[1])
    return L[0], buf


@pytest.mark.parametrize("B,pad,temperature,corr,ids", R.INBATCH_CASES)
def test_inbatch_softmax_matches_fp64(B, pad, temperature, corr, ids):
    c = R.make_inbatch_case(B, pad, temperature, corr, ids)
    L, buf = _inbatch(c, 1)
    G = _host(buf)
    assert np.isnan(G[:, B:]).all() and np.isnan(G[B]).all(), "wrote into the padding or past the last row"
    C = R.C_INBATCH
    loss_sum, loss_bound = 0.0, 0.0
    for r0 in range(0, B, 1024):
        r1 = min(B, r0 + 1024)
        ref = R.inbatch_ref(c, r0, r1)
        _check(G[r0:r1, :B], ref["grad"], C * ref["b_grad"], f"in-batch softmax, gradient, rows {r0}:{r1}")
        assert (G[r0:r1, :B][ref["masked"]] == 0).all()
        loss_sum += ref["loss_rows"].sum()
        loss_bound += ref["b_loss_rows"].sum()
    _check(L, loss_sum / B, C * loss_bound / B, "in-batch softmax, loss")
    if temperature == 0:
        assert (G[:B, :B] == 0).all()
    if ids == "all_equal":
        assert L == 0 and (G[:B, :B] == 0).all()
    L0, buf0 = _inbatch(c, 0)
    S0 = _host(buf0)
    np.testing.assert_array_equal(S0[:B, :B].view(np.uint32), c["S"].view(np.uint32))
    assert np.isnan(S0[:, B:]).all() and np.isnan(S0[B]).all()
    assert np.float32(L0).view(np.uint32) == np.float32(L).view(np.uint32)


def test_inbatch_softmax_rejects_bad_shapes_without_a_launch():
    import torch

    from librecommender_b200 import _lib

    S, loss = _nan(4, 4), _nan(1)
    ws = _ws(_lib.lib.b200_loss_workspace_bytes())
    n0 = _lib.launch_count()
    for B, lds, nws in ((0, 4, ws.numel()), (4, 3, ws.numel()), (4, 4, ws.numel() - 1)):
        assert _lib.lib.b200_softmax_inbatch_loss(_lib.ptr(S), lds, B, 1.0, None, None, 1, _lib.ptr(loss),
                                                  _lib.ptr(ws), nws, _lib.current_stream()) == -2
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0 and np.isnan(_host(S)).all()


# ---------------------------------------------------------------------------------------------------------------------
# sampled softmax / NCE
# ---------------------------------------------------------------------------------------------------------------------
def _sampled(c, loss_kind):
    """(loss, logits buffer [B + 1, ld] after the call, dtrue [B + 1])."""
    import torch

    from librecommender_b200 import _lib

    B, S, ld = c["B"], c["S"], c["S"] + c["pad"]
    buf = _nan(B + 1, ld)
    buf[:B, :S] = _dev(c["L"])
    dtrue, loss = _nan(B + 1), _nan(2)
    tries = torch.tensor([c["tries"]], dtype=torch.int64, device="cuda")
    ws = _ws(_lib.lib.b200_sampled_class_loss_workspace_bytes(B, S))
    keep = [_dev(c["true_dot"]), _dev(c["labels"]), _dev(c["sampled"]), _dev(c["bias"])]
    _lib.check(_lib.lib.b200_sampled_class_loss(loss_kind, _lib.ptr(buf), ld, B, S, *(_lib.ptr(t) for t in keep),
                                                c["kind"], c["n_items"], _lib.ptr(tries), _lib.ptr(loss),
                                                _lib.ptr(dtrue), _lib.ptr(ws), ws.numel(), _lib.current_stream()))
    L = _host(loss)
    assert np.isnan(L[1])
    return L[0], _host(buf), _host(dtrue)


def _sampled_params():
    for args in R.SAMPLED_CASES:
        for lk in (0, 1):
            B, S, pad, kind, n_items, extra, allhit = args
            yield pytest.param(args, lk, id=f"{B}x{S}+{pad}-s{kind}-n{n_items}-t{extra}{'-allhit' if allhit else ''}"
                                            f"-{'softmax' if lk == 0 else 'nce'}")


@pytest.mark.parametrize("args,loss_kind", list(_sampled_params()))
def test_sampled_class_loss_matches_fp64(args, loss_kind):
    c = R.make_sampled_case(*args)
    B, S = c["B"], c["S"]
    L, G, dt = _sampled(c, loss_kind)
    assert np.isnan(G[:, S:]).all() and np.isnan(G[B]).all() and np.isnan(dt[B]), "wrote past an output"
    ref = R.sampled_ref(c, loss_kind)
    C = R.C_SAMPLED
    _check(G[:B, :S], ref["dz"], C * ref["b_dz"], f"sampled, d z_s, kind {loss_kind}")
    _check(dt[:B], ref["dtrue"], C * ref["b_dtrue"], f"sampled, d z0, kind {loss_kind}")
    _check(L, ref["loss_rows"].sum() / B, C * ref["b_loss_rows"].sum() / B, f"sampled, loss, kind {loss_kind}")
    assert (G[:B, :S][ref["hit"]] == 0).all()
    if args[-1]:                       # every sampled id is row 0's label: only the true class is left
        assert ref["hit"][0].all() and (G[0, :S] == 0).all()
        if loss_kind == 0:
            assert dt[0] == 0


def test_sampled_class_loss_rejects_bad_shapes_without_a_launch():
    import torch

    from librecommender_b200 import _lib

    lib, P = _lib.lib, _lib.ptr
    B, S = 4, 8
    big = 65537
    L = _nan(B, big)
    t = torch.zeros(B, device="cuda")
    ids = torch.zeros(big, dtype=torch.int64, device="cuda")
    bias = torch.zeros(big, device="cuda")
    tries = torch.tensor([S], dtype=torch.int64, device="cuda")
    loss, dtrue = _nan(1), _nan(B)
    ws = _ws(lib.b200_sampled_class_loss_workspace_bytes(B, big))
    st = _lib.current_stream()

    def call(S=S, ld=S, n_items=100, labels=ids, null_bias=False):
        return lib.b200_sampled_class_loss(0, P(L), ld, B, S, P(t), P(labels), P(ids), None if null_bias else P(bias),
                                           1, n_items, P(tries), P(loss), P(dtrue), P(ws), ws.numel(), st)

    n0 = _lib.launch_count()
    assert call(S=big, ld=big, n_items=10 ** 6) == -2                 # S > 65 536
    assert call(ld=S - 1) == -2                                       # ld < S
    assert call(n_items=S - 1) == -2                                  # n_items < S
    assert call(labels=None) == -2                                    # a null pointer
    assert call(null_bias=True) == -2
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0
    assert np.isnan(_host(L)).all() and np.isnan(_host(dtrue)).all() and np.isnan(_host(loss)).all()


# ---------------------------------------------------------------------------------------------------------------------
# determinism
# ---------------------------------------------------------------------------------------------------------------------
def _bits(*arrays):
    return [np.ascontiguousarray(np.asarray(a, dtype=F32)).view(np.uint32) for a in arrays]


def test_repeated_calls_give_the_same_bits():
    for kind in (0, 1, 2, 3):
        pos, neg = R.make_pair_case(300_000, 17, kind, 0.5)
        a, b = _bits(*_pairwise(pos, neg, kind, 0.5)), _bits(*_pairwise(pos, neg, kind, 0.5))
        for x, y in zip(a, b):
            np.testing.assert_array_equal(x, y)
    c = R.make_inbatch_case(8193, 5, 0.05, "edges", "few")
    (L1, b1), (L2, b2) = _inbatch(c, 1), _inbatch(c, 1)
    for x, y in zip(_bits(L1, _host(b1)[:8193, :8193]), _bits(L2, _host(b2)[:8193, :8193])):
        np.testing.assert_array_equal(x, y)
    c = R.make_sampled_case(*R.SAMPLED_CASES[7])
    for lk in (0, 1):
        for x, y in zip(_bits(*_sampled(c, lk)), _bits(*_sampled(c, lk))):
            np.testing.assert_array_equal(x, y)


# ---------------------------------------------------------------------------------------------------------------------
# losses.py wrappers
# ---------------------------------------------------------------------------------------------------------------------
def _pair_fns():
    from librecommender_b200 import losses as Lo

    return [("bpr", Lo.bpr_loss), ("max_margin", lambda p, q: Lo.max_margin_loss(p, q, 0.5)),
            ("pbce", Lo.pairwise_bce_loss), ("pbce_sum", lambda p, q: Lo.pairwise_bce_loss(p, q, mean=False)),
            ("pfocal", Lo.pairwise_focal_loss)]


def _value_and_grads(fn, p, q, upstream=1.0):
    import torch

    p = p.detach().requires_grad_(True)
    q = q.detach().requires_grad_(True)
    v = fn(p, q)
    (v * upstream).backward()
    torch.cuda.synchronize()
    return v.detach().cpu().numpy(), p.grad.cpu().numpy(), q.grad.cpu().numpy()


def test_wrappers_take_strided_views_and_scale_by_the_upstream_gradient():
    import torch

    from librecommender_b200 import losses as Lo

    pos, neg = R.make_pair_case(257, 3, 0, 0.5)
    Pm = _dev(np.stack([pos, -pos, pos], 1))                        # [n, 3]: column 2 is a strided view of pos
    Nm = _dev(np.stack([neg, neg], 1))
    for name, fn in _pair_fns():
        pv, nv = Pm[:, 2], Nm[:, 1]
        assert not pv.is_contiguous()
        a = _value_and_grads(fn, pv, nv)
        b = _value_and_grads(fn, pv.contiguous(), nv.contiguous())
        for x, y in zip(_bits(*a), _bits(*b)):
            np.testing.assert_array_equal(x, y, err_msg=name)
        c = _value_and_grads(fn, pv, nv, 3.0)
        np.testing.assert_array_equal(_bits(c[1])[0], _bits(a[1] * F32(3))[0], err_msg=name)
        np.testing.assert_array_equal(_bits(c[2])[0], _bits(a[2] * F32(3))[0], err_msg=name)
    rng = np.random.default_rng(5)
    Um = _dev(rng.standard_normal((300, 2, 16)).astype(F32))
    Im = _dev(rng.standard_normal((300, 16)).astype(F32))
    ids = torch.tensor(rng.integers(0, 100, 300), device="cuda")
    out = []
    for up in (1.0, 3.0):
        u, i = Um[:, 1, :].detach().requires_grad_(True), Im.detach().requires_grad_(True)
        (Lo.softmax_cross_entropy(u, i, 0.1, None, ids) * up).backward()
        out.append((u.grad.cpu().numpy(), i.grad.cpu().numpy()))
    np.testing.assert_array_equal(out[1][0], out[0][0] * F32(3))
    np.testing.assert_array_equal(out[1][1], out[0][1] * F32(3))


@pytest.mark.parametrize("kind", [0, 1])
def test_broadcast_positives_match_repeated_positives(kind):
    """Positives broadcast by the kernel and repeated by the caller give the same per-positive gradient, up to the
    order of the factor-term sum (torch sums the repeated copies)."""
    from librecommender_b200 import losses as Lo

    fn = Lo.bpr_loss if kind == 0 else (lambda p, q: Lo.max_margin_loss(p, q, 1.0))
    for n_pos, f in ((31, 3), (257, 17), (300_000, 3)):
        pos, neg = R.make_pair_case(n_pos, f, kind, 1.0)
        p, q = _dev(pos), _dev(neg)
        vb, gpb, gnb = _value_and_grads(fn, p, q)
        p2 = p.detach().requires_grad_(True)
        q2 = q.detach().requires_grad_(True)
        v = fn(p2.repeat_interleave(f), q2)
        v.backward()
        gpr = p2.grad.cpu().numpy()
        np.testing.assert_array_equal(gnb, q2.grad.cpu().numpy())
        tol = 2 * f * (R.U * np.abs(gnb.astype(F64)).reshape(n_pos, f).sum(1) + R.ETA)
        assert (np.abs(gpb.astype(F64) - gpr) <= tol).all()
        assert abs(float(vb) - float(v)) <= 4 * R.U * (R.grid_rounds(len(neg)) + f + 2) * abs(float(vb)) + 1e-30


def test_softmax_cross_entropy_towers_match_fp64_past_8192_rows():
    """dU and dI of the in-batch softmax at B = 8193 (a warp takes a second row) against float64.  Bound: the in-batch
    bound of G = d loss / d S plus S's own GEMM error (2e-6 sum_k |u_k i_k|, the dense layer's) carried through the
    softmax, then the dense layer's error of G I and G^T U."""
    import torch

    from librecommender_b200 import losses as Lo

    B, d, tau = 8193, 32, 0.05
    rng = np.random.default_rng(8)
    U = rng.standard_normal((B, d)).astype(F32)
    I = rng.standard_normal((B, d)).astype(F32)
    U /= np.linalg.norm(U, axis=1, keepdims=True)
    I /= np.linalg.norm(I, axis=1, keepdims=True)
    corr = (rng.random(B) * 0.01 + 1e-4).astype(F32)
    ids = rng.integers(0, B // 3, B)
    u, i = _dev(U).requires_grad_(True), _dev(I).requires_grad_(True)
    v = Lo.softmax_cross_entropy(u, i, tau, _dev(corr), torch.tensor(ids, device="cuda"))
    v.backward()
    gU, gI = _host(u.grad), _host(i.grad)
    dv = "cuda"
    U64, I64 = torch.tensor(U, dtype=torch.float64, device=dv), torch.tensor(I, dtype=torch.float64, device=dv)
    S = U64 @ I64.T
    SM = U64.abs() @ I64.abs().T
    lg = S / float(F32(tau)) - torch.log(torch.tensor(corr, dtype=torch.float64, device=dv))[None, :]
    it = torch.tensor(ids, device=dv)
    eye = torch.eye(B, dtype=torch.bool, device=dv)
    mask = (it[:, None] == it[None, :]) & ~eye
    lg = torch.where(mask, torch.tensor(-R.FLT_MAX, dtype=torch.float64, device=dv), lg)
    P = torch.softmax(lg, 1)
    G = (P - eye.double()) / float(F32(tau)) / B
    G[mask] = 0.0
    # G's error: the kernel's bound with |S| and the GEMM error 34 u SM of each logit, both over tau
    lse_m = (B // 32 + 6) + lg.max(1).values.abs() + torch.logsumexp(lg, 1).abs() + (P * (2 * lg.abs() + 34 * SM / tau)).sum(1)
    gerr = R.U * (P * (2 * lg.abs() + 34 * SM / tau + lse_m[:, None] + 1) + (P - eye.double()).abs()) / tau / B
    gerr[mask] = 0.0
    gerr = R.C_INBATCH * gerr + 34 * R.U * G.abs()
    ref_U, ref_I = (G @ I64).cpu().numpy(), (G.T @ U64).cpu().numpy()
    bU = (gerr @ I64.abs()).cpu().numpy()
    bI = (gerr.T @ U64.abs()).cpu().numpy()
    _check(gU, ref_U, bU, "softmax_cross_entropy, dU")
    _check(gI, ref_I, bI, "softmax_cross_entropy, dI")


# ---------------------------------------------------------------------------------------------------------------------
# the max-margin hinge
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("margin", R.MARGINS)
def test_max_margin_hinge_ties_match_torch_autograd(margin):
    """Pairs exactly on the hinge (pos - neg == margin) pass the gradient, as torch's margin_ranking_loss does: every
    entry of the gradient is 0 or +-1/n, equal to torch float64 autograd rounded to float."""
    import torch
    import torch.nn.functional as Fn

    from librecommender_b200 import losses as Lo

    rng = np.random.default_rng(int(margin * 10))
    n = 12
    pos = (rng.integers(-64, 64, n) / 8.0).astype(F32)
    d = np.where(np.arange(n) % 3 == 0, margin, rng.integers(-16, 16, n) / 4.0)   # every third pair on the hinge
    d[1] = 0.0                                                                      # identical scores
    neg = (pos - d).astype(F32)
    assert ((pos.astype(F64) - neg) == margin).sum() >= 4
    p64 = torch.tensor(pos.astype(F64), requires_grad=True)
    q64 = torch.tensor(neg.astype(F64), requires_grad=True)
    v64 = Fn.margin_ranking_loss(p64, q64, torch.ones_like(p64), margin=margin)
    v64.backward()
    v, gp, gq = _value_and_grads(lambda a, b: Lo.max_margin_loss(a, b, margin), _dev(pos), _dev(neg))
    assert float(v) == F32(float(v64))
    np.testing.assert_array_equal(gp, p64.grad.numpy().astype(F32))
    np.testing.assert_array_equal(gq, q64.grad.numpy().astype(F32))
    assert set(np.abs(gp).tolist()) <= {0.0, float(F32(1.0 / n))}
