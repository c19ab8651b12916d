"""The sequence encoders' kernels, each C-ABI entry point called directly and compared with its float64 definition
(tests/_seq_encoder_kernels_ref.py):

* ``b200_rnn_encode`` / ``b200_rnn_train_forward``: every cell kind and activation, 1-4 layers of different H, every
  tile width the host picks (RNN_CASES lists each next to the restated ``rnn_layout``), n around the tile, every length
  class, permuted and duplicated users, padded ld_seq / ldx / ldo.  Each saved step is recomputed from the kernel's own
  previous step, and the chain is tied by bitwise identities (SV_Y(t) == SV_HP(t + 1) without LN, out == the top
  SV_Y(len - 1), encode == train_forward).
* ``b200_rnn_backward`` on the same cases, top layer (dout, lddo > H) and lower layers (dy), each step from the kernel's
  own gate gradients of the step after; ``dgh`` untouched for the TF1 GRU and the LSTM; the top layer-norm len-0 row.
* ``b200_caser_encode`` / ``_train_forward`` / ``_backward`` at conv tiles 2, 3 and 32 with partial last tiles, dW in
  every ``caser_nchunk`` regime, and a too-small workspace.
* ``b200_wavenet_encode`` / ``_train_forward`` at tiles 1, 2, 31 and 32, 1-16 layers, dilations 1, T - 1, T, 2^15;
  ``pool_backward``, ``layer_inputs`` and ``layer_dx`` bit-exact over several grid-stride passes.
* The max-pool argmax: the LOWEST position of equal float32 chains (repeated-item windows, constant sequences past
  the receptive field), -1 with output 0 when nothing is positive, and within the bound of the maximum elsewhere.

Outputs are NaN-prefilled with rows past n and columns past each width; those stay NaN.  Every call repeats bit for
bit, a slot's bits do not depend on its tile position, n or a NaN in another slot of its tile, and every rejected
argument returns -2 without a launch.  Bounds: C * u * mag, C calibrated in tests/test_seq_encoder_kernels_cpu.py."""
from __future__ import annotations

import ctypes

import numpy as np
import pytest

import _seq_encoder_kernels_ref as se
from test_gpu_rank_kernels import _dev, _lib, _sync

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
C_RNN_FWD = 4.0
C_RNN_BWD = 8.0
C_CASER = 4.0
C_WAVENET = 4.0
PAD_ROWS = 3

# (n, T, in_dim, kinds, hidden, acts): forward tile / shared bytes from the restated rnn_layout, backward tiles
RNN_CASES = [
    (65, 127, 3, [0], [7], [0]),                                    # tile 64 (9 472 B); n = tile + 1
    (63, 2, 1, [1], [33], [1]),                                     # tile 64 (44 032 B); n = tile - 1
    (24, 128, 256, [2], [128], [0]),                                # tile 24 (87 168 B), bwd 16; n = tile
    (27, 1, 256, [0, 1, 2, 0], [255, 1, 8, 256], [1, 0, 1, 0]),    # tile 8 (58 528 B); bwd 8 / 64 / 64 / 8
    (9, 128, 256, [2, 2, 2, 2], [256] * 4, [1] * 4),               # tile 8 above 96 KB (131 776 B)
    (8, 127, 3, [1, 0], [256, 255], [0, 1]),                        # tile 8 (49 504 B)
    (75, 17, 256, [2, 1, 0], [33, 128, 1], [0, 1, 1]),              # tile 24 (93 696 B); 3 tiles + 3
    (67, 33, 128, [0], [64], [1]),                                  # an intermediate tile
]


def _nan(shape, dtype=None):
    import torch

    return torch.full(shape, float("nan"), dtype=torch.float32 if dtype is None else dtype, device="cuda")


def _bits(x):
    return np.ascontiguousarray(x, dtype=F32).view(np.uint32)


def _check_all(checks, C, worst=None):
    for what, got, ref, mag in checks:
        got = np.asarray(got, F64)
        assert np.isfinite(got).all(), f"{what}: non-finite"
        err = np.abs(got - ref)
        exact = mag == 0
        assert (err[exact] == 0).all(), f"{what}: an exact element differs"
        if (~exact).any():
            r = err[~exact] / (C * se.U * mag[~exact])
            assert r.max() <= 1.0, f"{what}: {r.max():.3g} of the bound"
            if worst is not None:
                worst[0] = max(worst[0], float(r.max()))


def _ptr_table(ptrs):
    return (ctypes.c_void_p * len(ptrs))(*ptrs)


def _i32(v):
    return (ctypes.c_int32 * len(v))(*v)


# =====================================================================================================================
# RNN4Rec
# =====================================================================================================================
def _rnn_dev(c):
    return dict(X=_dev(c["X"]), seqs=_dev(c["seqs"]), lens=_dev(c["lens"]), users=_dev(c["users"]), w=_dev(c["w"]))


def _rnn_encode(c, dv, n=None, off=0, users=None, ldo=None, train=False, **over):
    L = _lib()
    n = c["n"] if n is None else n
    H = c["Hs"][-1]
    ldo = ldo or H + 2
    out = _nan((max(n, 1) + PAD_ROWS, ldo))
    u = dv["users"] if users is None else users
    saved, table = None, None
    if train:
        T = c["T"]
        saved = []
        for l, lw in enumerate(c["layers"]):
            Hl, GH = lw["H"], se.gates(lw["kind"]) * lw["H"]
            sv = [_nan((n * T + PAD_ROWS, Hl)), _nan((n * T + PAD_ROWS, Hl)), _nan((n * T + PAD_ROWS, GH)),
                  _nan((n * T + PAD_ROWS, Hl))]
            sv += [_nan((n * T + PAD_ROWS, Hl)), _nan((n * T + PAD_ROWS,))] if c["acts"][l] else [None, None]
            saved.append(sv)
        table = _ptr_table([t.data_ptr() if t is not None else None for sv in saved for t in sv])
    args = [L.ptr(u[off:]), n, L.ptr(dv["lens"]), L.ptr(dv["seqs"]), over.get("ld_seq", dv["seqs"].stride(0)),
            over.get("T", c["T"]), L.ptr(dv["X"]), over.get("ldx", dv["X"].stride(0)), over.get("in0", c["in0"]),
            over.get("nl", len(c["Hs"])), _i32(over.get("kinds", c["kinds"])), _i32(over.get("Hs", c["Hs"])),
            _i32(over.get("acts", c["acts"])), L.ptr(dv["w"]), L.ptr(out), ldo]
    fn = L.lib.b200_rnn_train_forward if train else L.lib.b200_rnn_encode
    rc = fn(*args, table, L.current_stream()) if train else fn(*args, L.current_stream())
    return rc, out, saved


def _rnn_forward(c, dv, **kw):
    rc, out, saved = _rnn_encode(c, dv, **kw)
    assert rc == 0, _lib().lib.b200_last_error()
    _sync()
    o = out.cpu().numpy()
    n, H = kw.get("n", c["n"]), c["Hs"][-1]
    assert np.isnan(o[n:]).all() and np.isnan(o[:, H:]).all(), "out written past n or H"
    if saved is None:
        return o[:n, :H], None
    nT, sv_np = n * c["T"], []
    for sv in saved:
        arrs = [None if t is None else t.cpu().numpy() for t in sv]
        for a in arrs:
            if a is not None:
                assert np.isnan(a[nT:]).all(), "saved tensor written past n * T"
        sv_np.append([None if a is None else a[:nT] for a in arrs])
    return o[:n, :H], sv_np


def _rnn_case(case, seed):
    n, T, in0, kinds, Hs, acts = case
    return se.make_rnn_case(n, T, in0, kinds, Hs, acts, seed=seed, ld_seq_pad=3, ldx_pad=5)


def test_rnn_cases_reach_every_tile_width():
    tiles = {se.rnn_fwd_tile(c[2], c[3], c[4], c[5]) for c in RNN_CASES}
    widths = {t for t, _ in tiles}
    assert 64 in widths and len(widths - {64, 8}) >= 2, widths
    assert any(t == 8 and b <= se.SMEM_TILE_BYTES for t, b in tiles)
    assert any(t == 8 and b > se.SMEM_TILE_BYTES for t, b in tiles)


@pytest.mark.parametrize("case", RNN_CASES, ids=lambda c: f"n{c[0]}-T{c[1]}-in{c[2]}-k{c[3]}-H{c[4]}-a{c[5]}")
def test_rnn_forward_and_backward(case):
    c = _rnn_case(case, seed=case[0] * 7 + case[1])
    dv = _rnn_dev(c)
    n, T = c["n"], c["T"]
    Lens = se.slot_lens(c)
    out, saved = _rnn_forward(c, dv, train=True)
    enc, _ = _rnn_forward(c, dv)
    np.testing.assert_array_equal(_bits(enc), _bits(out), err_msg="encode != train_forward")
    np.testing.assert_array_equal(_bits(_rnn_forward(c, dv)[0]), _bits(enc), err_msg="repeat")
    worst = [0.0]
    _check_all(se.rnn_forward_checks(c, saved, out), C_RNN_FWD, worst)
    # rows t >= len are exactly 0; the chain identities
    dead = (np.arange(T)[None, :] >= Lens[:, None]).ravel()
    for l, sv in enumerate(saved):
        for a in sv:
            if a is not None:
                assert (a[dead] == 0).all(), f"layer {l}: a row t >= len is not 0"
        s, t = np.nonzero(np.arange(T - 1)[None, :] + 1 < Lens[:, None])
        if c["acts"][l] == se.ACT_TANH:
            np.testing.assert_array_equal(_bits(sv[1][s * T + t]), _bits(sv[0][s * T + t + 1]))
    live = Lens > 0
    top = saved[-1][1]
    np.testing.assert_array_equal(_bits(out[live]), _bits(top[np.nonzero(live)[0] * T + Lens[live] - 1]))
    # one slot alone through an offset users pointer, and every slot in reversed tile positions
    for k in sorted({0, n - 1, n // 2}):
        one, _ = _rnn_forward(c, dv, n=1, off=k)
        np.testing.assert_array_equal(_bits(one[0]), _bits(enc[k]), err_msg=f"slot {k} alone")
    rev, _ = _rnn_forward(c, dv, users=_dev(c["users"][::-1].copy()))
    np.testing.assert_array_equal(_bits(rev[::-1]), _bits(enc), err_msg="tile position")
    # the backward, top layer first
    rng = np.random.default_rng(n)
    for l in range(len(c["Hs"]) - 1, -1, -1):
        top = l == len(c["Hs"]) - 1
        got = _rnn_backward(c, dv, l, saved[l], rng, top=top)
        dout, dyl = got.pop("_dout"), got.pop("_dy")
        again = _rnn_backward(c, dv, l, saved[l], rng, top=top, dout=dout, dy=dyl)
        for k in got:
            if got[k] is not None:
                np.testing.assert_array_equal(_bits(got[k]), _bits(again[k]), err_msg=f"L{l} {k} repeat")
        _check_all(se.rnn_backward_checks(c, l, saved[l], got, dout, dyl), C_RNN_BWD, worst)
        for k in ("dgx", "dgh", "dln", "dlnx"):
            if got[k] is not None:
                z = dead.copy()
                if k == "dln" and dyl is None and c["acts"][l]:
                    z[np.nonzero(Lens == 0)[0] * T] = False             # the len-0 row of the top LN layer
                assert (got[k][z] == 0).all(), f"L{l} {k}: a row t >= len is not 0"
    print(f"rnn {case}: worst {worst[0]:.3g} of the bound")


def _rnn_backward(c, dv, l, sv, rng, top, dout=None, dy=None):
    L = _lib()
    n, T = c["n"], c["T"]
    lw = c["layers"][l]
    H, kind, act = lw["H"], lw["kind"], c["acts"][l]
    GH = se.gates(kind) * H
    if top and dout is None:
        dout = rng.uniform(-1, 1, (n, H + 3)).astype(F32)
        dout[:, H:] = np.nan
    if not top and dy is None:
        dy = rng.uniform(-1, 1, (n * T, H)).astype(F32)
    ddout = _dev(dout) if top else None
    ddy = _dev(dy) if not top else None
    svd = [None if a is None else _dev(a) for a in sv]
    table = _ptr_table([t.data_ptr() if t is not None else None for t in svd])
    outs = {k: _nan((n * T + PAD_ROWS, w)) for k, w in (("dgx", GH), ("dgh", GH), ("dln", H), ("dlnx", H))}
    off = sum(se.rnn_layer_floats(x["kind"], x["ind"], x["H"]) for x in c["layers"][:l])
    rc = L.lib.b200_rnn_backward(
        L.ptr(dv["users"]), n, L.ptr(dv["lens"]), T, kind, lw["ind"], H, act, L.ptr(dv["w"][off:]),
        L.ptr(ddout), (H + 3) if top else 0, L.ptr(ddy), table, L.ptr(outs["dgx"]),
        L.ptr(outs["dgh"]) if kind == se.GRU_KERAS or l % 2 else None, L.ptr(outs["dln"]) if act else None,
        L.ptr(outs["dlnx"]) if act else None, L.current_stream())
    assert rc == 0, L.lib.b200_last_error()
    _sync()
    got = {}
    for k, t in outs.items():
        a = t.cpu().numpy()
        used = k == "dgx" or (k == "dgh" and kind == se.GRU_KERAS) or (k in ("dln", "dlnx") and act)
        if not used:
            assert np.isnan(a).all(), f"{k} written for kind {kind} act {act}"
            got[k] = None
            continue
        assert np.isnan(a[n * T:]).all(), f"{k} written past n * T"
        got[k] = a[:n * T]
    got["_dout"], got["_dy"] = dout, dy
    return got


def test_rnn_nan_in_one_slot_leaves_its_tile_alone():
    c = _rnn_case(RNN_CASES[0], seed=5)
    c["lens"][:] = c["T"]
    dv = _rnn_dev(c)
    base, _ = _rnn_forward(c, dv)
    victim = 3
    seqs = c["seqs"].copy()
    seqs[c["users"][victim], 2] = c["X"].shape[0] - 1                   # the NaN row of X
    dv2 = dict(dv, seqs=_dev(seqs))
    got, _ = _rnn_forward(c, dv2)
    others = np.nonzero(c["users"] != c["users"][victim])[0]
    assert np.isnan(got[victim]).any()
    np.testing.assert_array_equal(_bits(got[others]), _bits(base[others]))


def test_rnn_rejections_launch_nothing():
    L = _lib()
    c = _rnn_case((10, 8, 4, [0, 2], [8, 6], [1, 0]), seed=3)
    dv = _rnn_dev(c)
    bad = [dict(T=0), dict(T=129), dict(in0=0), dict(in0=257), dict(nl=0), dict(nl=5, kinds=[0] * 5, Hs=[8] * 5,
           acts=[0] * 5), dict(kinds=[3, 2]), dict(Hs=[8, 257]), dict(Hs=[0, 6]), dict(acts=[2, 0]),
           dict(ld_seq=7), dict(ldx=3), dict(ldo=5)]
    for train in (False, True):
        for kw in bad:
            before = L.launch_count()
            kw = dict(kw)
            ldo = kw.pop("ldo", None)
            rc, out, _ = _rnn_encode(c, dv, train=train, ldo=ldo, **kw)
            assert rc == -2 and L.launch_count() == before, (train, kw)
        before = L.launch_count()
        rc, out, _ = _rnn_encode(c, dv, n=0, train=train)
        assert rc == 0 and L.launch_count() == before
    assert L.lib.b200_rnn_layer_floats(3, 4, 4) == -2 and L.lib.b200_rnn_layer_floats(0, 0, 4) == -2
    assert L.lib.b200_rnn_layer_floats(2, 5, 7) == se.rnn_layer_floats(2, 5, 7)


# =====================================================================================================================
# Caser
# =====================================================================================================================
CASER_CASES = [  # (n, T, K, nh, nv): tile from the restated conv_launch (one [T*K | 1] buffer per user)
    (35, 64, 128, 32, 32),       # tile 2, partial last tile
    (10, 64, 127, 5, 1),         # tile 3, partial last tile
    (5, 63, 3, 5, 1),            # tile 32, one partial tile
    (70, 5, 128, 1, 5),          # tile 32, two full tiles + 6
    (7, 1, 1, 1, 1),
    (9, 2, 3, 32, 32),
    (40, 5, 3, 5, 5),
]


def _conv_dev(c):
    return dict(X=_dev(c["X"]), seqs=_dev(c["seqs"]), users=_dev(c["users"]), w=_dev(c["w"]))


def _caser_call(c, dv, train, n=None, off=0, ldo=None, **over):
    L = _lib()
    n = c["n"] if n is None else n
    D = c["T"] * c["nh"] + c["K"] * c["nv"]
    ldo = ldo or D + 3
    out = _nan((max(n, 1) + PAD_ROWS, ldo))
    arg = _dev(np.full((max(n, 1) + PAD_ROWS, c["T"] * c["nh"]), -7, np.int32))
    args = [L.ptr(dv["users"][off:]), n, L.ptr(dv["seqs"]), over.get("ld_seq", dv["seqs"].stride(0)),
            over.get("T", c["T"]), L.ptr(dv["X"]), over.get("ldx", dv["X"].stride(0)), over.get("K", c["K"]),
            over.get("nh", c["nh"]), over.get("nv", c["nv"]), L.ptr(dv["w"]), L.ptr(out), ldo]
    if train:
        rc = L.lib.b200_caser_train_forward(*args, L.ptr(arg), L.current_stream())
    else:
        rc = L.lib.b200_caser_encode(*args, L.current_stream())
    return rc, out, arg


def _caser_run(c, dv, train=False, **kw):
    rc, out, arg = _caser_call(c, dv, train, **kw)
    assert rc == 0, _lib().lib.b200_last_error()
    _sync()
    n = kw.get("n", c["n"])
    D = c["T"] * c["nh"] + c["K"] * c["nv"]
    o, a = out.cpu().numpy(), arg.cpu().numpy()
    assert np.isnan(o[n:]).all() and np.isnan(o[:, D:]).all(), "out written past n or its width"
    if train:
        assert (a[n:] == -7).all(), "argmax written past n"
    return o[:n, :D], (a[:n] if train else None)


@pytest.mark.parametrize("n,T,K,nh,nv", CASER_CASES)
def test_caser_forward_argmax_backward(n, T, K, nh, nv):
    c = se.make_caser_case(n, T, K, nh, nv, seed=n + T * K, ld_seq_pad=2, ldx_pad=3)
    dv = _conv_dev(c)
    out, arg = _caser_run(c, dv, train=True)
    enc, _ = _caser_run(c, dv)
    np.testing.assert_array_equal(_bits(enc), _bits(out), err_msg="encode != train_forward")
    np.testing.assert_array_equal(_bits(_caser_run(c, dv)[0]), _bits(enc), err_msg="repeat")
    worst = [0.0]
    _check_all(se.caser_forward_checks(c, out), C_CASER, worst)
    bad = se.caser_argmax_violations(c, out, arg, C_CASER)
    assert not bad, bad[:5]
    if nh > 1:
        assert (arg[:, ::nh] == -1).all() and (out[:, :T * nh:nh] == 0).all()
    for k in sorted({0, n - 1, n // 2}):
        one, a1 = _caser_run(c, dv, train=True, n=1, off=k)
        np.testing.assert_array_equal(_bits(one[0]), _bits(out[k]), err_msg=f"slot {k} alone")
        np.testing.assert_array_equal(a1[0], arg[k])
    # a NaN in one slot's rows leaves the other slots bit-identical
    seqs = c["seqs"].copy()
    seqs[c["users"][0], T - 1] = c["X"].shape[0] - 1
    got, _ = _caser_run(c, dict(dv, seqs=_dev(seqs)))
    np.testing.assert_array_equal(_bits(got[1:]), _bits(enc[1:]))
    # backward
    rng = np.random.default_rng(T)
    dF = rng.uniform(-1, 1, out.shape).astype(F32)
    dX, dW = _caser_backward(c, dF, out, arg)
    dX2, dW2 = _caser_backward(c, dF, out, arg)
    np.testing.assert_array_equal(_bits(dX), _bits(dX2))
    np.testing.assert_array_equal(_bits(dW), _bits(dW2))
    _check_all(se.caser_backward_checks(c, dF, out, arg, dX, dW, dx_slots=np.arange(min(n, 12))), C_CASER, worst)
    print(f"caser {(n, T, K, nh, nv)}: worst {worst[0]:.3g} of the bound")


def _caser_backward(c, dF, feat, arg, ws_floats=None, expect=0):
    L = _lib()
    n, T, K, nh, nv = c["n"], c["T"], c["K"], c["nh"], c["nv"]
    D = T * nh + K * nv
    E = se.caser_floats(T, K, nh, nv)
    need = L.lib.b200_caser_backward_workspace_floats(n, T, K, nh, nv)
    assert need == se.caser_nchunk(n, E) * E
    Xg = se.gathered(c).reshape(n * T, K)
    Xd = _dev(np.pad(Xg, ((0, 0), (0, 2)), constant_values=np.nan))
    dFd = _dev(np.pad(dF, ((0, 0), (0, 1)), constant_values=np.nan))
    fd = _dev(np.pad(feat, ((0, 0), (0, 2)), constant_values=np.nan))
    ad = _dev(arg)
    wd = _dev(c["w"])
    dX = _nan((n * T + PAD_ROWS, K + 1))
    dW = _nan((E + PAD_ROWS,))
    ws = _nan((ws_floats if ws_floats is not None else need,))
    before = L.launch_count()
    rc = L.lib.b200_caser_backward(n, T, K, nh, nv, L.ptr(dFd), D + 1, L.ptr(fd), D + 2, L.ptr(ad), L.ptr(Xd), K + 2,
                                   L.ptr(wd), L.ptr(dX), K + 1, L.ptr(dW), L.ptr(ws), ws.numel(), L.current_stream())
    if expect:
        assert rc == expect and L.launch_count() == before
        _sync()
        assert np.isnan(dX.cpu().numpy()).all() and np.isnan(dW.cpu().numpy()).all()
        return None
    assert rc == 0, L.lib.b200_last_error()
    _sync()
    x, w = dX.cpu().numpy(), dW.cpu().numpy()
    assert np.isnan(x[n * T:]).all() and np.isnan(x[:, K:]).all() and np.isnan(w[E:]).all()
    return x[:n * T, :K], w[:E]


# (n, T, K, nh, nv, heights checked): caser_nchunk regimes
CASER_DW_CASES = [
    (600, 5, 3, 5, 5, None),              # E = 280: 3 chunks by rows (n > 256)
    (1100, 32, 64, 32, 4, (1, 2, 17, 32)),  # E = 1 082 500: by rows 5, capped at 4 Mi / E = 3 chunks of 367 rows
    (300, 64, 128, 32, 32, (1, 2, 64)),   # E = 8 523 808 > 4 Mi: one chunk over all 300 rows
]


@pytest.mark.parametrize("n,T,K,nh,nv,hs", CASER_DW_CASES)
def test_caser_backward_chunk_regimes(n, T, K, nh, nv, hs):
    c = se.make_caser_case(n, T, K, nh, nv, seed=n, n_items=200, patterns=False)
    dv = _conv_dev(c)
    out, arg = _caser_run(c, dv, train=True)
    E = se.caser_floats(T, K, nh, nv)
    print(f"caser dW n={n} E={E}: {se.caser_nchunk(n, E)} chunks")
    rng = np.random.default_rng(n)
    dF = rng.uniform(-1, 1, out.shape).astype(F32)
    dX, dW = _caser_backward(c, dF, out, arg)
    worst = [0.0]
    _check_all(se.caser_backward_checks(c, dF, out, arg, dX, dW, hs=hs, dx_slots=np.arange(8)), C_CASER, worst)
    np.testing.assert_array_equal(_bits(_caser_backward(c, dF, out, arg)[1]), _bits(dW), err_msg="repeat")
    need = se.caser_nchunk(n, E) * E
    _caser_backward(c, dF, out, arg, ws_floats=need - 1, expect=-2)
    print(f"caser dW regime n={n}: worst {worst[0]:.3g} of the bound")


def test_caser_rejections_launch_nothing():
    L = _lib()
    c = se.make_caser_case(6, 4, 3, 2, 2, seed=1)
    dv = _conv_dev(c)
    for train in (False, True):
        for kw in (dict(T=0), dict(T=65), dict(K=0), dict(K=129), dict(nh=33), dict(nv=0), dict(ld_seq=3),
                   dict(ldx=2), dict(ldo=4 * 2 + 3 * 2 - 1)):
            before = L.launch_count()
            rc, out, _ = _caser_call(c, dv, train, **kw)
            assert rc == -2 and L.launch_count() == before, (train, kw)
        before = L.launch_count()
        assert _caser_call(c, dv, train, n=0)[0] == 0 and L.launch_count() == before
    assert L.lib.b200_caser_weight_floats(65, 1, 1, 1) == -2
    assert L.lib.b200_caser_backward_workspace_floats(-1, 4, 3, 2, 2) == -2


# =====================================================================================================================
# WaveNet
# =====================================================================================================================
WAVENET_CASES = [  # (n, T, K, F, dilations): tile from conv_launch with two [T * (max(K, F) | 1) | 1] buffers
    (5, 64, 128, 128, [1, 63, 64, 2 ** 15]),                                   # tile 1
    (5, 64, 64, 64, [1, 2, 4, 8, 16, 32, 1, 2, 4, 8, 16, 32, 1, 2, 4, 8]),    # tile 2, 16 layers
    (40, 5, 16, 33, [1, 4, 5]),                                                # tile 32, 8 in the last
    (7, 1, 1, 1, [1]),
    (7, 2, 16, 5, [1, 1]),
    (33, 3, 128, 128, [2, 1, 3]),                                              # tile 31: two tiles
]


def _wavenet_call(c, dv, train, n=None, off=0, ldo=None, **over):
    L = _lib()
    n = c["n"] if n is None else n
    T, F = over.get("T", c["T"]), c["F"]
    dils = over.get("dils", c["dils"])
    ldo = ldo or F + 2
    out = _nan((max(n, 1) + PAD_ROWS, ldo))
    ys = _nan((len(c["dils"]) * max(n, 1) * c["T"] * F + PAD_ROWS,))
    arg = _dev(np.full((max(n, 1) + PAD_ROWS, F), -7, np.int32))
    args = [L.ptr(dv["users"][off:]), n, L.ptr(dv["seqs"]), over.get("ld_seq", dv["seqs"].stride(0)), T,
            L.ptr(dv["X"]), over.get("ldx", dv["X"].stride(0)), over.get("K", c["K"]), over.get("nl", len(dils)),
            over.get("F", F), _i32(dils), L.ptr(dv["w"]), L.ptr(out), ldo]
    if train:
        rc = L.lib.b200_wavenet_train_forward(*args, L.ptr(ys), L.ptr(arg), L.current_stream())
    else:
        rc = L.lib.b200_wavenet_encode(*args, L.current_stream())
    return rc, out, ys, arg


def _wavenet_run(c, dv, train=False, **kw):
    rc, out, ys, arg = _wavenet_call(c, dv, train, **kw)
    assert rc == 0, _lib().lib.b200_last_error()
    _sync()
    n, T, F, Lc = kw.get("n", c["n"]), c["T"], c["F"], len(c["dils"])
    o = out.cpu().numpy()
    assert np.isnan(o[n:]).all() and np.isnan(o[:, F:]).all()
    if not train:
        return o[:n, :F], None, None
    y = ys.cpu().numpy()
    assert np.isnan(y[Lc * n * T * F:]).all()
    a = arg.cpu().numpy()
    assert (a[n:] == -7).all()
    return o[:n, :F], y[:Lc * n * T * F].reshape(Lc, n, T, F), a[:n]


@pytest.mark.parametrize("n,T,K,F,dils", WAVENET_CASES)
def test_wavenet_forward_argmax(n, T, K, F, dils):
    c = se.make_wavenet_case(n, T, K, F, dils, seed=n + T + K, ld_seq_pad=1, ldx_pad=2)
    dv = _conv_dev(c)
    out, ys, arg = _wavenet_run(c, dv, train=True)
    enc, _, _ = _wavenet_run(c, dv)
    np.testing.assert_array_equal(_bits(enc), _bits(out), err_msg="encode != train_forward")
    np.testing.assert_array_equal(_bits(_wavenet_run(c, dv)[0]), _bits(enc), err_msg="repeat")
    worst = [0.0]
    checks, (z, mz) = se.wavenet_forward_checks(c, out, ys)
    _check_all(checks, C_WAVENET, worst)
    bad = se.argmax_violations(z, mz, arg, out, se.wavenet_windows(c), C_WAVENET)
    assert not bad, bad[:5]
    if F > 1:
        assert (arg[:, 0] == -1).all() and (out[:, 0] == 0).all()
    for k in sorted({0, n - 1}):
        one, y1, a1 = _wavenet_run(c, dv, train=True, n=1, off=k)
        np.testing.assert_array_equal(_bits(one[0]), _bits(out[k]))
        np.testing.assert_array_equal(_bits(y1[:, 0]), _bits(ys[:, k]))
        np.testing.assert_array_equal(a1[0], arg[k])
    seqs = c["seqs"].copy()
    seqs[c["users"][0], 0] = c["X"].shape[0] - 1
    got, _, _ = _wavenet_run(c, dict(dv, seqs=_dev(seqs)))
    np.testing.assert_array_equal(_bits(got[1:]), _bits(enc[1:]))
    print(f"wavenet {(n, T, K, F, len(dils))}: worst {worst[0]:.3g} of the bound")


def test_wavenet_rejections_launch_nothing():
    L = _lib()
    c = se.make_wavenet_case(6, 4, 3, 5, [1, 2], seed=1)
    dv = _conv_dev(c)
    for train in (False, True):
        for kw in (dict(T=0), dict(T=65), dict(K=0), dict(K=129), dict(F=129), dict(nl=0), dict(nl=17, dils=[1] * 17),
                   dict(dils=[1, 0]), dict(ld_seq=3), dict(ldx=2), dict(ldo=4)):
            before = L.launch_count()
            assert _wavenet_call(c, dv, train, **kw)[0] == -2 and L.launch_count() == before, (train, kw)
        before = L.launch_count()
        assert _wavenet_call(c, dv, train, n=0)[0] == 0 and L.launch_count() == before


# (n, T, C): n * T * C past 132 * 32 * 256, so the element kernels' grid-stride loops run several passes
HELPER_CASES = [(400, 64, 128), (1000, 5, 3), (3, 1, 1)]


@pytest.mark.parametrize("n,T,C", HELPER_CASES)
def test_wavenet_position_helpers_bit_exact(n, T, C):
    L = _lib()
    rng = np.random.default_rng(n)
    passes = se.elem_passes(n * T * C)
    print(f"wavenet helpers n={n} T={T} C={C}: {passes} / {se.elem_passes(n * T * 2 * C)} grid-stride passes")
    x = rng.uniform(-1, 1, (n * T, C + 3)).astype(F32)
    x[:, C:] = np.nan
    P = rng.uniform(-1, 1, (n * T, 2 * C)).astype(F32)
    xd, Pd = _dev(x), _dev(P)
    for d in sorted({1, max(1, T - 1), T, 2 ** 15, 2 ** 31 - 1}):
        out = _nan((n * T * 2 * C + PAD_ROWS,))
        assert L.lib.b200_wavenet_layer_inputs(L.ptr(xd), C + 3, n, T, C, d, L.ptr(out), L.current_stream()) == 0
        dx = _nan((n * T + PAD_ROWS, C + 2))
        assert L.lib.b200_wavenet_layer_dx(L.ptr(Pd), n, T, C, d, L.ptr(dx), C + 2, L.current_stream()) == 0
        _sync()
        o = out.cpu().numpy()
        assert np.isnan(o[n * T * 2 * C:]).all()
        np.testing.assert_array_equal(_bits(o[:n * T * 2 * C].reshape(n * T, 2 * C)),
                                      _bits(se.wavenet_layer_inputs_ref(x, n, T, C, d)), err_msg=f"inputs d={d}")
        g = dx.cpu().numpy()
        assert np.isnan(g[n * T:]).all() and np.isnan(g[:, C:]).all()
        np.testing.assert_array_equal(_bits(g[:n * T, :C]), _bits(se.wavenet_layer_dx_ref(P, n, T, C, d)),
                                      err_msg=f"dx d={d}")
    F = min(C, 128)
    dF = rng.uniform(-1, 1, (n, F + 1)).astype(F32)
    arg = rng.integers(-1, T, (n, F)).astype(np.int32)
    dZ = _nan((n * T + PAD_ROWS, F))
    assert L.lib.b200_wavenet_pool_backward(n, T, F, L.ptr(_dev(dF)), F + 1, L.ptr(_dev(arg)), L.ptr(dZ),
                                            L.current_stream()) == 0
    _sync()
    z = dZ.cpu().numpy()
    assert np.isnan(z[n * T:]).all()
    np.testing.assert_array_equal(_bits(z[:n * T]), _bits(se.wavenet_pool_backward_ref(dF, arg, T, F)))
    before = L.launch_count()
    assert L.lib.b200_wavenet_layer_dx(L.ptr(Pd), n, T, C, 0, L.ptr(dx), C + 2, L.current_stream()) == -2
    assert L.lib.b200_wavenet_layer_inputs(L.ptr(xd), C - 1, n, T, C, 1, L.ptr(out), L.current_stream()) == -2
    assert L.lib.b200_wavenet_pool_backward(n, 65, F, L.ptr(_dev(dF)), F + 1, L.ptr(_dev(arg)), L.ptr(dZ),
                                            L.current_stream()) == -2
    assert L.lib.b200_wavenet_layer_dx(L.ptr(Pd), 0, T, C, 1, L.ptr(dx), C + 2, L.current_stream()) == 0
    assert L.launch_count() == before
