"""GPU parity of the wgmma 3xTF32 dense layer (b200_linear_tf32x3) against an fp64 restatement
of tf_dense (reference libreco/layers/dense.py:52-80) and against the exact-fma SIMT kernel
(b200_linear_f32).  Tolerance: 2e-6 * sum_k |x_k w_k| — an fp32 sequential sum is itself only
good to ~sqrt(din) * 6e-8 of that quantity, and north_star's 1e-5 relative bar on the scores is
checked end to end by tests/test_gpu_feat_models.py with LINEAR_IMPL forced to this kernel."""
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
