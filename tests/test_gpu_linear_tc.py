"""GPU parity of the wgmma 3xTF32 dense layer (b200_linear_tf32x3) against an fp64 restatement
of tf_dense (reference libreco/layers/dense.py:52-80) and against the exact-fma SIMT kernel
(b200_linear_f32).  Tolerance: 2e-6 * sum_k |x_k w_k| — an fp32 sequential sum is itself only
good to ~sqrt(din) * 6e-8 of that quantity, and north_star's 1e-5 relative bar on the scores is
checked end to end by tests/test_gpu_feat_models.py with LINEAR_IMPL forced to this kernel."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _run(fn_name, x, Wt, b, relu, presplit=False):
    import torch

    from librecommender_b200 import _lib

    y = torch.empty((x.shape[0], Wt.shape[0]), dtype=torch.float32, device=x.device)
    bp = _lib.ptr(b) if b is not None else None
    if fn_name == "b200_linear_tf32x3":
        ws = None
        if presplit:
            ld = int(_lib.lib.b200_linear_tf32x3_split_ld(Wt.shape[1]))
            ws = torch.empty(2 * Wt.shape[0] * ld, dtype=torch.float32, device=x.device)
            _lib.check(_lib.lib.b200_linear_tf32x3_split_weights(_lib.ptr(Wt), Wt.stride(0), Wt.shape[1], Wt.shape[0],
                                                                 _lib.ptr(ws), _lib.current_stream()))
        _lib.check(_lib.lib.b200_linear_tf32x3(_lib.ptr(x), x.stride(0), x.shape[0], _lib.ptr(Wt), Wt.stride(0),
                                               _lib.ptr(ws), bp, Wt.shape[1], Wt.shape[0], 1 if relu else 0,
                                               _lib.ptr(y), y.stride(0), _lib.current_stream()))
    else:
        _lib.check(_lib.lib.b200_linear_f32(_lib.ptr(x), x.stride(0), x.shape[0], _lib.ptr(Wt), Wt.stride(0), bp,
                                            Wt.shape[1], Wt.shape[0], 1 if relu else 0, _lib.ptr(y), y.stride(0),
                                            _lib.current_stream()))
    torch.cuda.synchronize()
    return y.cpu().numpy()


@pytest.mark.parametrize("R,din,dout,relu,bias", [
    (5000, 1792, 128, True, True),      # DeepFM first layer, BASELINE C2 feature shape
    (300, 52, 10, False, True),         # tiny: one partial row tile, k tail, n_pad 32
    (1000, 100, 200, True, False),      # k not a multiple of 32, two column blocks
    (129, 32, 32, False, False),        # single k-chunk
    (20000, 160, 64, True, True),       # several tiles per CTA wave
    (777, 1024, 96, True, True),        # 8 accumulator groups
])
@pytest.mark.parametrize("presplit", [False, True])
def test_linear_tf32x3_matches_fp64(R, din, dout, relu, bias, presplit):
    import torch

    rng = np.random.default_rng(R + din)
    x = rng.standard_normal((R, din)).astype(np.float32)
    x[:, ::7] *= 30.0                                    # mixed magnitudes
    Wt = (rng.standard_normal((dout, din)) / np.sqrt(din)).astype(np.float32)
    b = rng.standard_normal(dout).astype(np.float32) if bias else None
    xd, Wd = torch.from_numpy(x).cuda(), torch.from_numpy(Wt).cuda()
    bd = torch.from_numpy(b).cuda() if bias else None

    ref = x.astype(np.float64) @ Wt.astype(np.float64).T
    mag = np.abs(x).astype(np.float64) @ np.abs(Wt).astype(np.float64).T
    if bias:
        ref = ref + b
    if relu:
        ref = np.maximum(ref, 0.0)

    got = _run("b200_linear_tf32x3", xd, Wd, bd, relu, presplit)
    simt = _run("b200_linear_f32", xd, Wd, bd, relu)
    err = np.abs(got - ref) / (mag + 1e-30)
    err_simt = np.abs(simt - ref) / (mag + 1e-30)
    print(f"tf32x3 max err / sum|xw| = {err.max():.3e}   simt fp32 = {err_simt.max():.3e}")
    assert err.max() <= 2e-6, float(err.max())
    # and within 1e-5 of the exact-fma kernel's result relative to the score scale
    scale = np.maximum(np.abs(ref), np.abs(ref).mean())
    assert (np.abs(got - simt) <= 1e-5 * scale + 2e-6 * mag).all()


def test_linear_tf32x3_strided_views():
    """Leading dimensions larger than the logical widths (column slices of wider buffers)."""
    import torch

    rng = np.random.default_rng(5)
    big = torch.from_numpy(rng.standard_normal((4100, 256)).astype(np.float32)).cuda()
    Wbig = torch.from_numpy((rng.standard_normal((64, 512)) * 0.05).astype(np.float32)).cuda()
    x = big[:, 64:64 + 96]          # 16-byte aligned view, ld = 256
    Wt = Wbig[:, 128:128 + 96]
    got = _run("b200_linear_tf32x3", x, Wt, None, False)
    ref = x.double().cpu().numpy() @ Wt.double().cpu().numpy().T
    mag = np.abs(x.cpu().numpy()).astype(np.float64) @ np.abs(Wt.cpu().numpy()).astype(np.float64).T
    assert (np.abs(got - ref) <= 2e-6 * mag).all()


def test_linear_tf32x3_presplit_allows_unaligned_weight_rows():
    """Wt with ldw % 4 != 0 (a column slice) is fine once a split copy exists."""
    import torch

    rng = np.random.default_rng(9)
    x = torch.from_numpy(rng.standard_normal((700, 64)).astype(np.float32)).cuda()
    Wbig = torch.from_numpy((rng.standard_normal((48, 131)) * 0.1).astype(np.float32)).cuda()
    Wt = Wbig[:, 3:3 + 64]
    got = _run("b200_linear_tf32x3", x, Wt, None, True, presplit=True)
    ref = np.maximum(x.double().cpu().numpy() @ Wt.double().cpu().numpy().T, 0)
    mag = np.abs(x.cpu().numpy()).astype(np.float64) @ np.abs(Wt.cpu().numpy()).astype(np.float64).T
    assert (np.abs(got - ref) <= 2e-6 * mag).all()


def test_linear_tf32x3_rejects_misaligned():
    import torch

    from librecommender_b200 import _lib

    x = torch.zeros((256, 35), device="cuda")
    Wt = torch.zeros((16, 35), device="cuda")
    y = torch.empty((256, 16), device="cuda")
    rc = _lib.lib.b200_linear_tf32x3(_lib.ptr(x), x.stride(0), 256, _lib.ptr(Wt), Wt.stride(0), None, None, 35, 16, 0,
                                     _lib.ptr(y), y.stride(0), _lib.current_stream())
    assert rc != 0


@pytest.mark.parametrize("impl", ["tf32x3", "f32"])
def test_deepfm_logits_with_forced_linear_impl(impl):
    """End-to-end 1e-5 bar on DeepFM logits with every Dense layer forced through one kernel."""
    from librecommender_b200 import feat_models as fm
    from oracle import tf_models as tm

    rng = np.random.default_rng(11)
    spec = tm.make_spec(rng, 300, 500, [7, 30, 12, 9], [11, 5, 40, 8, 3], 1, 2)
    w = tm.make_deepfm_weights(rng, spec, 16, (128, 64, 32), True)
    old = fm.LINEAR_IMPL
    fm.LINEAR_IMPL = impl
    try:
        model = fm.DeepFM(spec, w)
        users = rng.integers(0, spec["n_users"] + 1, size=3000)
        items = rng.integers(0, spec["n_items"] + 1, size=3000)
        sparse, dense = tm.row_features(spec, users, items)
        ref64 = tm.deepfm_forward(w, users, items, sparse, dense, dtype=np.float64)
        got = model.logits(users, items).cpu().numpy()
    finally:
        fm.LINEAR_IMPL = old
    scale = np.maximum(np.abs(ref64), np.abs(ref64).mean())
    assert (np.abs(got - ref64) <= 1e-5 * scale + 1e-6).all(), float(np.abs(got - ref64).max())


@pytest.mark.parametrize("R,din,dout,splits,relu,bias", [
    (1792, 8192, 128, 10, False, False),    # the DeepFM first-layer weight gradient (X^T dY): 14 tiles x 10 splits
    (128, 8192, 64, 16, False, False),      # one tile, 16 splits
    (300, 1000, 200, 7, True, True),        # k tail (1000 = 31.25 chunks), ragged last split, bias + ReLU in the reduction
    (129, 96, 32, 3, False, True),          # 3 chunks over 3 splits
    (64, 4096, 10, 64, False, False),       # more splits than make sense: clipped to one chunk each
])
def test_linear_tf32x3_splitk_matches_fp64(R, din, dout, splits, relu, bias):
    import torch

    from librecommender_b200 import _lib

    rng = np.random.default_rng(R + din + splits)
    x = rng.standard_normal((R, din)).astype(np.float32)
    Wt = (rng.standard_normal((dout, din)) / np.sqrt(din)).astype(np.float32)
    b = rng.standard_normal(dout).astype(np.float32) if bias else None
    xd, Wd = torch.from_numpy(x).cuda(), torch.from_numpy(Wt).cuda()
    bd = torch.from_numpy(b).cuda() if bias else None
    y = torch.full((R, dout), float("nan"), dtype=torch.float32, device="cuda")
    ws = torch.empty(splits * R * dout, dtype=torch.float32, device="cuda")
    outs = []
    for _ in range(2):
        _lib.check(_lib.lib.b200_linear_tf32x3_splitk(_lib.ptr(xd), xd.stride(0), R, _lib.ptr(Wd), Wd.stride(0),
                                                      _lib.ptr(bd), din, dout, 1 if relu else 0, splits, _lib.ptr(ws),
                                                      ws.numel() * 4, _lib.ptr(y), y.stride(0), _lib.current_stream()))
        torch.cuda.synchronize()
        outs.append(y.cpu().numpy().copy())
    np.testing.assert_array_equal(outs[0], outs[1])                    # fixed reduction order
    ref = x.astype(np.float64) @ Wt.astype(np.float64).T
    mag = np.abs(x).astype(np.float64) @ np.abs(Wt).astype(np.float64).T
    if bias:
        ref = ref + b
    if relu:
        ref = np.maximum(ref, 0.0)
    err = np.abs(outs[0] - ref) / (mag + 1e-30)
    assert err.max() <= 2e-6, float(err.max())


# ===== the dense-layer kernels one by one: widths, tails, sentinels, bit-identity, the dispatcher ====================
#
# Bounds (calibrated on a float32 restatement of each kernel in tests/test_tf32x3_model_cpu.py):
# * b200_linear_tf32x3, pre-activation: 2e-6 * sum_k |x_k w_k| + 6 * 2^-20 * max_k |x_k w_k|, with the bias counted
#   as one more product (1 * b).  Each product's 3xTF32 representation error is below 3 * 2^-20 |x_k w_k|; over many
#   products it averages out under the first term, but one dominant product (din = 1, or one large column) keeps
#   its own error, which the second term allows twice over.  max_k is bounded by max_k |x_k| * max_k |w_k|.
# * swish (act 2): |swish'| <= 1.1, so 1.1 * (the pre-activation bound) + SWISH_REL * u * |swish| for the float32
#   exp, add and divide of x / (1 + exp(-x)), + SWISH_ABS: below x = -88.7 exp(-x) overflows and float32 gives -0.0
#   for a swish of magnitude under 2.7e-37.
# * b200_linear_f32: bit-exact to the fmaf chain (_rank_kernels_ref.dot_chain) plus a float32 bias add; swish within
#   SWISH_REL * u of the float64 swish of that pre-activation.
C_SUM, C_MAX = 2e-6, 6 * 2.0 ** -20
SWISH_SLOPE, SWISH_REL, SWISH_ABS = 1.1, 16, 2.0 ** -118
U32 = 2.0 ** -24
SENT = 0x7FC0BEEF                          # quiet-NaN bit pattern the output buffers are pre-filled with

DOUTS = [1, 16, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129, 200, 256, 257, 383]
DINS = [1, 7, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1023, 1024, 1025]
ROWS = [1, 2, 127, 128, 129, 255]
# 42 cases: every dout (n_pad 32 / 64 / 96 / 128 at both edges, grid.y up to 3 with a one-column last block at 129 and
# 257) and every din (k tails, the 64-k promotion boundary, odd chunk counts) two or three times; the activation /
# bias pair runs through all six combinations every six cases and the row count changes every seven
CASES = [(ROWS[(i // 7) % 6], DINS[i % 14], DOUTS[i % 18], i % 3, (i // 3) % 2 == 0) for i in range(42)]


def make_case(R, din, dout, bias, seed):
    """x [R, din] (every 7th column 30x larger: mixed magnitudes), Wt [dout, din], b [dout] or None (float32)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((R, din)).astype(np.float32)
    x[:, ::7] *= 30.0
    Wt = (rng.standard_normal((dout, din)) / np.sqrt(din)).astype(np.float32)
    b = rng.standard_normal(dout).astype(np.float32) if bias else None
    return x, Wt, b


def swish64(v):
    return v / (1.0 + np.exp(-v))


def ref64(x, Wt, b, act):
    """float64 act(x Wt^T + b) and the tf32x3 bound of every element."""
    z = x.astype(np.float64) @ Wt.astype(np.float64).T
    mag = np.abs(x).astype(np.float64) @ np.abs(Wt).astype(np.float64).T
    mx = np.abs(x).max(axis=1).astype(np.float64)[:, None] * np.abs(Wt).max(axis=1).astype(np.float64)[None, :]
    if b is not None:
        z = z + b
        mag = mag + np.abs(b)
        mx = np.maximum(mx, np.abs(b).astype(np.float64))
    bound = C_SUM * mag + C_MAX * mx
    if act == 1:
        return np.maximum(z, 0.0), bound
    if act == 2:
        y = swish64(z)
        return y, SWISH_SLOPE * bound + SWISH_REL * U32 * np.abs(y) + SWISH_ABS
    return z, bound


def f32_restated(x, Wt, b, act):
    """b200_linear_f32 on the host: the fmaf chain, a float32 bias add (+0.0 without bias), then the activation.
    Returns (pre-activation bits for act 0 / 1, or the float64 swish of the pre-activation for act 2, and a bound
    that is 0 except for swish)."""
    from _rank_kernels_ref import dot_chain

    v = dot_chain(x, Wt) + (b if b is not None else np.float32(0.0))
    if act == 1:
        return np.maximum(v, np.float32(0.0)), np.zeros(v.shape)
    if act == 2:
        y = swish64(v.astype(np.float64))
        return y, SWISH_REL * U32 * np.abs(y) + SWISH_ABS
    return v, np.zeros(v.shape)


def _ld4(n):
    """A leading dimension past n (a gap of at least one column) that keeps 16-byte rows."""
    return (n + 1 + 3) // 4 * 4


class Operands:
    """Device copies of x / Wt inside larger NaN-filled buffers (gap columns, 7 rows past R) and an output buffer
    pre-filled with the SENT bit pattern: [R + 3, ldy]."""

    def __init__(self, x, Wt, b, ldy=None, y_offset=0):
        import torch

        R, din = x.shape
        dout = Wt.shape[0]
        self.R, self.din, self.dout = R, din, dout
        self.xbuf = torch.full((R + 7, _ld4(din)), float("nan"), device="cuda")
        self.xbuf[:R, :din] = torch.from_numpy(x).cuda()
        self.wbuf = torch.full((dout, _ld4(din)), float("nan"), device="cuda")
        self.wbuf[:, :din] = torch.from_numpy(Wt).cuda()
        self.b = torch.from_numpy(b).cuda() if b is not None else None
        self.ldy = ldy if ldy is not None else dout + 1 + (dout + 1) % 2          # even: the float2 stores
        self.yflat = torch.full(((R + 3) * self.ldy + y_offset,), SENT, dtype=torch.int32, device="cuda")
        self.y_offset = y_offset

    def x(self):
        return self.xbuf[:self.R, :self.din]

    def Wt(self):
        return self.wbuf[:, :self.din]

    def yptr(self):
        return ctypes.c_void_p(self.yflat.data_ptr() + 4 * self.y_offset)

    def reset_y(self):
        self.yflat.fill_(SENT)

    def ybits(self):
        """[R + 3, ldy] uint32 (the y_offset floats before the buffer are checked to be untouched)."""
        flat = self.yflat.cpu().numpy().view(np.uint32)
        assert (flat[:self.y_offset] == SENT).all(), "a store before Y"
        return flat[self.y_offset:].reshape(self.R + 3, self.ldy)

    def y(self):
        """The [R, dout] output after checking that it was all written and nothing around it was."""
        bits = self.ybits()
        inner = bits[:self.R, :self.dout]
        assert not (inner == SENT).any(), f"{int((inner == SENT).sum())} outputs not written"
        assert (bits[:self.R, self.dout:] == SENT).all(), "a store into the ldy gap"
        assert (bits[self.R:] == SENT).all(), "a store past row R"
        return inner.view(np.float32)

    def tf32x3(self, act, presplit):
        import torch

        from librecommender_b200 import _lib

        ws = None
        if presplit:
            ld = int(_lib.lib.b200_linear_tf32x3_split_ld(self.din))
            ws = torch.empty(2 * self.dout * ld, dtype=torch.float32, device="cuda")
            _lib.check(_lib.lib.b200_linear_tf32x3_split_weights(_lib.ptr(self.Wt()), self.wbuf.stride(0), self.din,
                                                                 self.dout, _lib.ptr(ws), _lib.current_stream()))
        self.reset_y()
        _lib.check(_lib.lib.b200_linear_tf32x3(_lib.ptr(self.x()), self.xbuf.stride(0), self.R, _lib.ptr(self.Wt()),
                                               self.wbuf.stride(0), _lib.ptr(ws), _lib.ptr(self.b), self.din, self.dout,
                                               act, self.yptr(), self.ldy, _lib.current_stream()))
        torch.cuda.synchronize()
        return self.y().copy()

    def f32(self, act):
        import torch

        from librecommender_b200 import _lib

        self.reset_y()
        _lib.check(_lib.lib.b200_linear_f32(_lib.ptr(self.x()), self.xbuf.stride(0), self.R, _lib.ptr(self.Wt()),
                                            self.wbuf.stride(0), _lib.ptr(self.b), self.din, self.dout, act,
                                            self.yptr(), self.ldy, _lib.current_stream()))
        torch.cuda.synchronize()
        return self.y().copy()


def _assert_within(got, ref, bound, what):
    err = np.abs(got.astype(np.float64) - ref)
    bad = ~(err <= bound)
    assert not bad.any(), (f"{what}: {int(bad.sum())} outside the bound, worst err / bound "
                           f"{float(np.max(err / np.maximum(bound, 1e-300))):.3g}")


def _sample_rows(R, n, seed):
    rng = np.random.default_rng(seed)
    return np.unique(np.concatenate([[0, R - 1], rng.integers(0, R, size=n)]))


@pytest.mark.parametrize("R,din,dout,act,bias", CASES)
def test_tf32x3_widths_tails_sentinels(R, din, dout, act, bias):
    """Every n_pad template at both edges, k / row / column tails read through NaN-filled gaps, every output written and
    nothing else; pre-split, self-split and a repeat give the same bits."""
    x, Wt, b = make_case(R, din, dout, bias, seed=R * 7919 + din * 31 + dout)
    ops = Operands(x, Wt, b)
    got = ops.tf32x3(act, presplit=False)
    np.testing.assert_array_equal(got.view(np.uint32), ops.tf32x3(act, presplit=True).view(np.uint32))
    np.testing.assert_array_equal(got.view(np.uint32), ops.tf32x3(act, presplit=False).view(np.uint32))
    assert np.isfinite(got).all()
    ref, bound = ref64(x, Wt, b, act)
    _assert_within(got, ref, bound, "tf32x3")


@pytest.mark.parametrize("R,din,dout,act,bias", CASES)
def test_f32_exact_fma_chain(R, din, dout, act, bias):
    """b200_linear_f32 equals the fmaf chain bit for bit (swish: within the calibrated bound), same cases, sentinels."""
    x, Wt, b = make_case(R, din, dout, bias, seed=R * 7919 + din * 31 + dout)
    ops = Operands(x, Wt, b)
    got = ops.f32(act)
    rows = _sample_rows(R, 6, R + din + dout)
    want, bound = f32_restated(x[rows], Wt, b, act)
    if act == 2:
        _assert_within(got[rows], want, bound, "f32 swish")
    else:
        np.testing.assert_array_equal(got[rows].view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("dout,act", [(33, 0), (129, 1), (257, 2), (96, 2)])
def test_tf32x3_scalar_store_path(dout, act):
    """Odd ldy, or Y one float past a float2 boundary, takes the scalar stores: same bits as the float2 path."""
    x, Wt, b = make_case(255, 100, dout, True, seed=dout)
    vec = Operands(x, Wt, b).tf32x3(act, presplit=False)
    odd = Operands(x, Wt, b, ldy=dout + 1 + dout % 2).tf32x3(act, presplit=False)
    shifted = Operands(x, Wt, b, y_offset=1).tf32x3(act, presplit=True)
    np.testing.assert_array_equal(vec.view(np.uint32), odd.view(np.uint32))
    np.testing.assert_array_equal(vec.view(np.uint32), shifted.view(np.uint32))


@pytest.mark.parametrize("R,din,dout", [
    (100_003, 160, 1000),    # n_pad 128, 3 stages: 8 column blocks of ~16 CTAs, ~49 tiles each; 5 chunks per tile
    (100_003, 512, 40),      # n_pad 64, 4 stages: ~6 tiles of 16 chunks per CTA
])
def test_tf32x3_many_tiles_per_cta_and_row_bits(R, din, dout):
    """Many tiles per persistent CTA (stage / phase wrap at 3 and 4 stages); a row's bits do not depend on the rows
    around it: computed alone, at row 127 or 128 of a tile, or inside the large call."""
    import torch

    from librecommender_b200 import _lib

    x, Wt, b = make_case(R, din, dout, True, seed=din + dout)
    ops = Operands(x, Wt, b)
    ops.reset_y()
    _lib.check(_lib.lib.b200_linear_tf32x3(_lib.ptr(ops.x()), ops.xbuf.stride(0), R, _lib.ptr(ops.Wt()),
                                           ops.wbuf.stride(0), None, _lib.ptr(ops.b), din, dout, 2, ops.yptr(),
                                           ops.ldy, _lib.current_stream()))
    torch.cuda.synchronize()
    y2 = ops.yflat.view(R + 3, ops.ldy)
    assert bool((y2[:R, dout:] == SENT).all()) and bool((y2[R:] == SENT).all()), "a store outside [R, dout]"
    inner = y2[:R, :dout].view(torch.float32)
    assert bool(torch.isfinite(inner).all()), "an output not written"
    rows = _sample_rows(R, 500, R)
    rows = np.unique(np.concatenate([rows, [127, 128, 129, R // 2, R - 2]]))
    got = inner[torch.from_numpy(rows).cuda()].cpu().numpy()
    ref, bound = ref64(x[rows], Wt, b, 2)
    _assert_within(got, ref, bound, "tf32x3 large R")
    for r in rows[::max(1, len(rows) // 6)][:6].tolist() + [R - 1]:
        alone = Operands(x[r:r + 1], Wt, b).tf32x3(2, presplit=False)
        np.testing.assert_array_equal(alone[0].view(np.uint32), got[np.searchsorted(rows, r)].view(np.uint32))
        block = np.random.default_rng(r).standard_normal((256, din)).astype(np.float32)
        block[127] = block[128] = x[r]
        yb = Operands(block, Wt, b).tf32x3(2, presplit=True)
        np.testing.assert_array_equal(yb[127].view(np.uint32), alone[0].view(np.uint32))
        np.testing.assert_array_equal(yb[128].view(np.uint32), alone[0].view(np.uint32))


@pytest.mark.parametrize("kernel", ["tf32x3", "f32"])
@pytest.mark.parametrize("act", [0, 2])
def test_nan_containment(kernel, act):
    """A NaN in one x row poisons only that output row, a NaN in one Wt row only that output column; every other
    output keeps the clean run's bits."""
    R, din, dout, r0, c0 = 300, 100, 200, 131, 150
    x, Wt, b = make_case(R, din, dout, True, seed=3)
    run = (lambda o: o.tf32x3(act, presplit=False)) if kernel == "tf32x3" else (lambda o: o.f32(act))
    clean = run(Operands(x, Wt, b))
    xn, Wn = x.copy(), Wt.copy()
    xn[r0, 57] = np.nan
    Wn[c0, 3] = np.nan
    dirty = run(Operands(xn, Wn, b))
    poisoned = np.zeros((R, dout), dtype=bool)
    poisoned[r0, :] = poisoned[:, c0] = True
    assert np.isnan(dirty[poisoned]).all()
    np.testing.assert_array_equal(dirty[~poisoned].view(np.uint32), clean[~poisoned].view(np.uint32))


def _splitk_effective(din, splits):
    chunks = -(-din // 32)
    per = -(-chunks // splits)
    return -(-chunks // per)


SPLITK_CASES = [(din, splits) for din in (32, 33, 96, 1000, 8192) for splits in (1, 2, 3, 7, 16, 64)]


@pytest.mark.parametrize("din,splits", SPLITK_CASES)
def test_splitk_splits_acts_sentinels(din, splits):
    """Every split count at one-chunk, short and long reductions; bias and the activation in the reduction; repeats
    give the same bits; the workspace is left alone when the chunks allow only one split."""
    import torch

    from librecommender_b200 import _lib

    i = SPLITK_CASES.index((din, splits))
    act, bias = i % 3, i % 2 == 0
    R, dout = (130, 65) if din == 8192 else (200, 130)
    x, Wt, b = make_case(R, din, dout, bias, seed=din * 100 + splits)
    ops = Operands(x, Wt, b, ldy=dout + 3)
    ws = torch.full((splits * R * dout,), SENT, dtype=torch.int32, device="cuda")
    outs = []
    for _ in range(2):
        ops.reset_y()
        _lib.check(_lib.lib.b200_linear_tf32x3_splitk(_lib.ptr(ops.x()), ops.xbuf.stride(0), R, _lib.ptr(ops.Wt()),
                                                      ops.wbuf.stride(0), _lib.ptr(ops.b), din, dout, act, splits,
                                                      _lib.ptr(ws), ws.numel() * 4, ops.yptr(), ops.ldy,
                                                      _lib.current_stream()))
        torch.cuda.synchronize()
        outs.append(ops.y().copy())
    np.testing.assert_array_equal(outs[0].view(np.uint32), outs[1].view(np.uint32))
    if _splitk_effective(din, splits) == 1:
        assert bool((ws == SENT).all()), "one effective split must write Y directly"
    ref, bound = ref64(x, Wt, b, act)
    _assert_within(outs[0], ref, bound, f"split-K x{splits}")


def test_splitk_rejects_before_launch():
    import torch

    from librecommender_b200 import _lib

    R, din, dout = 64, 256, 32
    x = torch.zeros((R, din), device="cuda")
    Wt = torch.zeros((dout, din), device="cuda")
    y = torch.zeros((R, dout), device="cuda")
    ws = torch.zeros(4 * R * dout, device="cuda")

    def call(splits, nbytes):
        return _lib.lib.b200_linear_tf32x3_splitk(_lib.ptr(x), din, R, _lib.ptr(Wt), din, None, din, dout, 0, splits,
                                                  _lib.ptr(ws), nbytes, _lib.ptr(y), dout, _lib.current_stream())

    n0 = _lib.launch_count()
    assert call(0, ws.numel() * 4) == -2
    assert call(65, ws.numel() * 4) == -2
    assert call(4, 4 * R * dout * 4 - 4) == -2          # one float short
    assert _lib.launch_count() == n0
    assert call(4, 4 * R * dout * 4) == 0                # and exactly enough is accepted
    torch.cuda.synchronize()


def test_f32_slab_rows():
    """More than 65535 row tiles: the rows go out in slabs of 65535 * 64; rows either side of the slab edge, the last
    row and random rows equal the fmaf chain and the same rows computed in their own call."""
    import torch

    from librecommender_b200 import _lib
    from _rank_kernels_ref import dot_chain

    R, din, dout, ldy = 65535 * 64 + 65, 5, 3, 4
    edge = 65535 * 64
    rng = np.random.default_rng(17)
    xd = torch.randn((R, 8), device="cuda", generator=torch.Generator("cuda").manual_seed(5))
    Wt = rng.standard_normal((dout, din)).astype(np.float32)
    b = rng.standard_normal(dout).astype(np.float32)
    Wd, bd = torch.from_numpy(Wt).cuda(), torch.from_numpy(b).cuda()
    y = torch.full((R, ldy), SENT, dtype=torch.int32, device="cuda")
    n0 = _lib.launch_count()
    _lib.check(_lib.lib.b200_linear_f32(_lib.ptr(xd), 8, R, _lib.ptr(Wd), din, _lib.ptr(bd), din, dout, 1,
                                        _lib.ptr(y), ldy, _lib.current_stream()))
    torch.cuda.synchronize()
    assert _lib.launch_count() - n0 == 2                          # two slabs
    assert bool((y[:, dout:] == SENT).all()) and not bool((y[:, :dout] == SENT).any())
    rows = np.unique(np.concatenate([[0, 64, edge - 1, edge, edge + 1, R - 1], rng.integers(0, R, size=10_000)]))
    ri = torch.from_numpy(rows).cuda()
    got = y[ri, :dout].cpu().numpy().view(np.float32)
    xs = xd[ri, :din].cpu().numpy()
    want = np.maximum(dot_chain(xs, Wt) + b, np.float32(0.0))
    np.testing.assert_array_equal(got.view(np.uint32), want.view(np.uint32))
    for r in (edge - 1, edge, edge + 1, R - 1):
        one = torch.full((1, dout), SENT, dtype=torch.int32, device="cuda")
        _lib.check(_lib.lib.b200_linear_f32(_lib.ptr(xd[r:r + 1]), 8, 1, _lib.ptr(Wd), din, _lib.ptr(bd), din, dout, 1,
                                            _lib.ptr(one), dout, _lib.current_stream()))
        torch.cuda.synchronize()
        np.testing.assert_array_equal(one.cpu().numpy()[0].view(np.uint32), got[np.searchsorted(rows, r)].view(np.uint32))


def test_f32_rejects_bad_shapes_before_launch():
    """din / dout <= 0 and leading dimensions that would overlap rows are refused (rc -2) without a launch; R = 0 is
    an empty call."""
    import torch

    from librecommender_b200 import _lib

    R, din, dout = 8, 16, 8
    buf = torch.zeros(4096, device="cuda")       # large enough for any of the calls below had they run
    y = torch.full((4096,), SENT, dtype=torch.int32, device="cuda")

    def call(R=R, ldx=din, ldw=din, din=din, dout=dout, ldy=dout):
        return _lib.lib.b200_linear_f32(_lib.ptr(buf), ldx, R, _lib.ptr(buf), ldw, None, din, dout, 0, _lib.ptr(y), ldy,
                                        _lib.current_stream())

    n0 = _lib.launch_count()
    assert call(din=0) == -2
    assert call(din=-3) == -2
    assert call(dout=0) == -2
    assert call(dout=-1) == -2
    assert call(ldx=din - 1) == -2
    assert call(ldw=din - 1) == -2
    assert call(ldy=dout - 1) == -2
    assert call(R=0) == 0
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0
    assert bool((y == SENT).all())
    assert call() == 0
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0 + 1


# ----- feat_models.linear: which kernel each shape reaches ----------------------------------------------------------
_ENTRY = {"b200_linear_f32": "f32", "b200_linear_tf32x3": "tf32x3", "b200_linear_tf32x3_splitk": "splitk"}


@pytest.fixture
def routes(monkeypatch):
    """Records (route, Wsplit given) of every dense-kernel call made through _lib.lib."""
    from librecommender_b200 import _lib

    seen = []
    for name, tag in _ENTRY.items():
        fn = getattr(_lib.lib, name)

        def spy(*args, _fn=fn, _tag=tag):
            presplit = _tag == "tf32x3" and bool(getattr(args[5], "value", args[5]))
            seen.append(_tag + ("+cached" if presplit else ""))
            return _fn(*args)

        monkeypatch.setattr(_lib.lib, name, spy)
    return seen


def _bound_for(route, x, Wt, b, act):
    ref, bound = ref64(x, Wt, b, act)
    if route == "f32":      # an fmaf chain of din + 1 roundings (bias included): gamma_(din+1) * sum |x w|
        mag = np.abs(x).astype(np.float64) @ np.abs(Wt).astype(np.float64).T + (np.abs(b) if b is not None else 0)
        bound = (x.shape[1] + 2) * U32 * mag
    return ref, bound


@pytest.mark.parametrize("R,din,dout,cache_split,route", [
    (5000, 63, 64, True, "f32"),                      # din < TC_MIN_DIN
    (4096, 64, 64, True, "tf32x3+cached"),            # din == TC_MIN_DIN, R == TC_MIN_ROWS
    (4096, 64, 64, False, "tf32x3"),                  # self-split
    (4095, 64, 64, True, "f32"),                      # one row short, 4095 * 64 * 64 MACs < TC_MIN_MACS
    (2048, 256, 256, True, "tf32x3+cached"),          # R * din * dout == TC_MIN_MACS
    (2047, 256, 256, True, "f32"),                    # just under it
    (100, 1024, 64, False, "splitk"),                 # din == TC_LONG_K, one output tile: split the reduction
    (100, 1024, 64, True, "tf32x3+cached"),           # a cached layer is not split
    (100, 1023, 64, False, "f32"),                    # din < TC_LONG_K, few MACs
])
def test_linear_dispatch_routes(routes, R, din, dout, cache_split, route):
    import torch

    from librecommender_b200 import feat_models as fm

    assert (fm.TC_MIN_DIN, fm.TC_MIN_ROWS, fm.TC_MIN_MACS, fm.TC_LONG_K) == (64, 4096, 1 << 27, 1024)
    x, Wt, b = make_case(R, din, dout, True, seed=R + din)
    got = fm.linear(torch.from_numpy(x).cuda(), torch.from_numpy(Wt).cuda(), torch.from_numpy(b).cuda(), 1,
                    cache_split=cache_split, impl="auto").cpu().numpy()
    assert routes == [route], routes
    ref, bound = _bound_for(route, x, Wt, b, 1)
    _assert_within(got, ref, bound, route)


def test_linear_misaligned_x_falls_back_to_f32(routes):
    import torch

    from librecommender_b200 import feat_models as fm

    R, din, dout = 5000, 128, 64
    x, Wt, b = make_case(R, din, dout, False, seed=1)
    base = torch.empty(R * din + 1, device="cuda")
    xd = base[1:].view(R, din)                          # storage offset 1: rows not 16-byte aligned
    xd.copy_(torch.from_numpy(x))
    got = fm.linear(xd, torch.from_numpy(Wt).cuda(), None, 0, impl="auto").cpu().numpy()
    assert routes == ["f32"], routes
    ref, bound = _bound_for("f32", x, Wt, None, 0)
    _assert_within(got, ref, bound, "misaligned x")


@pytest.mark.parametrize("impl", ["auto", "f32", "tf32x3"])
def test_linear_transposed_views(impl):
    """x = A.t() and a transposed Wt (inner stride != 1) are read as the matrices they are."""
    import torch

    from librecommender_b200 import feat_models as fm

    R, din, dout = 4100, 96, 48
    x, Wt, b = make_case(R, din, dout, True, seed=2)
    A = torch.from_numpy(np.ascontiguousarray(x.T)).cuda()           # [din, R]
    W = torch.from_numpy(np.ascontiguousarray(Wt.T)).cuda()          # [din, dout]
    got = fm.linear(A.t(), W.t(), torch.from_numpy(b).cuda(), 0, impl=impl).cpu().numpy()
    ref, bound = _bound_for("f32", x, Wt, b, 0)
    _assert_within(got, ref, np.maximum(bound, ref64(x, Wt, b, 0)[1]), f"transposed ({impl})")


def test_linear_rejects_wrong_dtype_or_device():
    import torch

    from librecommender_b200 import _lib
    from librecommender_b200 import feat_models as fm

    x = torch.ones((8, 4), device="cuda")
    Wt = torch.ones((3, 4), device="cuda")
    b = torch.ones(3, device="cuda")
    n0 = _lib.launch_count()
    for args in [(x.double(), Wt, b), (x.cpu(), Wt, b), (x, Wt.double(), b), (x, Wt.cpu(), b), (x, Wt, b.double()),
                 (x, Wt, b.cpu()), (x.half(), Wt, None)]:
        with pytest.raises(ValueError):
            fm.linear(*args, 0)
    assert _lib.launch_count() == n0


def test_linear_split_cache_follows_in_place_updates(routes):
    """Wt.add_ bumps the tensor's version: the cached hi / lo split is remade and the output follows."""
    import torch

    from librecommender_b200 import feat_models as fm

    R, din, dout = 4096, 64, 32
    x, Wt, _ = make_case(R, din, dout, False, seed=4)
    xd, Wd = torch.from_numpy(x).cuda(), torch.from_numpy(Wt).cuda()
    y0 = fm.linear(xd, Wd, None, 0).cpu().numpy()
    Wd.add_(0.25)
    y1 = fm.linear(xd, Wd, None, 0).cpu().numpy()
    assert routes.count("tf32x3+cached") == 2, routes
    ref, bound = ref64(x, Wt + np.float32(0.25), None, 0)
    _assert_within(y1, ref, bound, "after Wt.add_")
    assert not np.array_equal(y0, y1)


@pytest.mark.parametrize("R", [4099, 4096])
@pytest.mark.parametrize("din,dout", [(300, 20), (20, 300)])
def test_weight_grad_orientations(R, din, dout):
    """dWt = dY^T X in both orientations of the product, over a batch that is or is not a multiple of 4."""
    import torch

    from librecommender_b200.training import _weight_grad

    rng = np.random.default_rng(R + din)
    dy = rng.standard_normal((R, dout)).astype(np.float32)
    x = rng.standard_normal((R, din)).astype(np.float32)
    got = _weight_grad(torch.from_numpy(dy).cuda(), torch.from_numpy(x).cuda()).cpu().numpy()
    assert got.shape == (dout, din)
    ref = dy.T.astype(np.float64) @ x.astype(np.float64)
    mag = np.abs(dy.T).astype(np.float64) @ np.abs(x).astype(np.float64)
    _assert_within(got, ref, (R + 2) * U32 * mag, "weight gradient")      # the looser of the two kernels' bounds
