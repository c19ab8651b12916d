"""Numeric model of the 3xTF32 operand split used by b200_linear_tf32x3 (csrc/mlp_tc.cu): x = hi + lo
with hi = the tf32 truncation of x and lo = x - hi (itself truncated to tf32 by the tensor core),
product ~ hi*hi' + lo*hi' + hi*lo'.  Checks in exact float64 arithmetic that the representation +
dropped-term error is below 3 * 2^-20 * sum|x w| for every input (truncation keeps 10 explicit
mantissa bits: |lo| < 2^-10 |x|, so lo*lo' < 2^-20 |x w| and the two truncated cross terms add 2^-20 each) (the measured kernel error, which also
contains the fp32 accumulation, is <= 1e-6 * sum|x w|: tests/test_gpu_linear_tc.py)."""
import numpy as np
import pytest

import test_gpu_linear_tc as lt


def _tf32_trunc(x):
    b = np.asarray(x, dtype=np.float32).view(np.uint32) & np.uint32(0xFFFFE000)
    return b.view(np.float32)


@pytest.mark.parametrize("din", [32, 1792])
def test_three_product_split_error_bound(din):
    rng = np.random.default_rng(din)
    x = (rng.standard_normal((64, din)) * np.exp(rng.uniform(-6, 6, (64, din)))).astype(np.float32)   # wide dynamic range
    w = (rng.standard_normal((din, 16)) * np.exp(rng.uniform(-6, 6, (din, 16)))).astype(np.float32)
    xh, wh = _tf32_trunc(x), _tf32_trunc(w)
    xl, wl = _tf32_trunc(x - xh), _tf32_trunc(w - wh)        # what the tensor core sees of the lo parts
    assert (np.abs(x - xh) <= np.abs(x) * 2.0 ** -10).all()  # 10 explicit mantissa bits kept
    f = np.float64
    approx = xh.astype(f) @ wh.astype(f) + xl.astype(f) @ wh.astype(f) + xh.astype(f) @ wl.astype(f)
    exact = x.astype(f) @ w.astype(f)
    mag = np.abs(x).astype(f) @ np.abs(w).astype(f)
    err = np.abs(approx - exact) / mag
    assert err.max() <= 3 * 2.0 ** -20, float(err.max())
    # a single tf32 product (no split) is three orders of magnitude worse: why the split exists
    single = np.abs(xh.astype(f) @ wh.astype(f) - exact) / mag
    assert single.max() > 50 * err.max()


# ----- calibration of the bounds of tests/test_gpu_linear_tc.py ------------------------------------------------------
# The kernels restated in float32 on the GPU test's cases, in their operation order: the tf32 truncation of hi and
# lo, each wgmma k8 step as the float32 sum of its 8 exact products added to a float32 accumulator (main: hi*hi;
# correction: lo*hi then hi*lo), the promotion (y + corr) + main every 64 k and at the last chunk of a split, split-K
# partials summed in z order, then the float32 bias add and activation.  Every bound must hold with 4x to spare and be
# at most 1000x looser than the restatement needs.
F32, F64 = np.float32, np.float64


def _mma8(a, b):
    return (a.astype(F64) @ b.astype(F64).T).astype(F32)


def _act32(v, act):
    if act == 1:
        return np.maximum(v, F32(0))
    if act == 2:
        with np.errstate(over="ignore"):
            return v / (F32(1) + np.exp(-v))
    return v


def tf32x3_restated(x, Wt, b, act, splits=1):
    """b200_linear_tf32x3 / _splitk in float32: see above."""
    R, din = x.shape
    chunks = -(-din // 32)
    pad = chunks * 32 - din
    xp, wp = np.pad(x, ((0, 0), (0, pad))), np.pad(Wt, ((0, 0), (0, pad)))
    xh, wh = _tf32_trunc(xp), _tf32_trunc(wp)
    xl, wl = _tf32_trunc(xp - xh), _tf32_trunc(wp - wh)
    per = -(-chunks // splits)
    v = np.zeros((R, Wt.shape[0]), F32)
    for c0 in range(0, chunks, per):                     # split z: chunks [c0, c0 + per), summed in z order
        c1 = min(c0 + per, chunks)
        y = np.zeros_like(v)
        for kc in range(c1 - c0):
            if kc % 2 == 0:
                main, corr = np.zeros_like(v), np.zeros_like(v)
            for k8 in range(4):
                s = slice((c0 + kc) * 32 + 8 * k8, (c0 + kc) * 32 + 8 * k8 + 8)
                main = main + _mma8(xh[:, s], wh[:, s])
                corr = corr + _mma8(xl[:, s], wh[:, s])
                corr = corr + _mma8(xh[:, s], wl[:, s])
            if kc % 2 == 1 or kc == c1 - c0 - 1:
                y = (y + corr) + main
        v = v + y
    if b is not None:
        v = v + b
    return _act32(v, act)


def _ratio(got, ref, bound):
    return float((np.abs(np.asarray(got, F64) - ref) / bound).max())


def _calibrate(ratios, what):
    worst = max(ratios)
    print(f"{what}: the float32 restatement uses {worst:.3g} of the bound")
    assert 4.0 * worst <= 1.0, f"{what}: not 4x inside the bound ({worst:.3g})"
    assert worst >= 1e-3, f"{what}: bound over 1000x looser than float32 needs ({worst:.3g})"


def _rows(case, n=64):
    R, din, dout, act, bias = case
    x, Wt, b = lt.make_case(R, din, dout, bias, seed=R * 7919 + din * 31 + dout)
    return x[:n], Wt, b, act


@pytest.mark.parametrize("family", ["plain", "swish"])
def test_tf32x3_bound_calibration(family):
    ratios = []
    for case in lt.CASES:
        x, Wt, b, act = _rows(case)
        if (act == 2) != (family == "swish"):
            continue
        ref, bound = lt.ref64(x, Wt, b, act)
        ratios.append(_ratio(tf32x3_restated(x, Wt, b, act), ref, bound))
    _calibrate(ratios, f"tf32x3 {family}")


def test_splitk_bound_calibration():
    ratios = []
    for i, (din, splits) in enumerate(lt.SPLITK_CASES):
        act, bias = i % 3, i % 2 == 0
        R, dout = (130, 65) if din == 8192 else (200, 130)
        x, Wt, b = lt.make_case(R, din, dout, bias, seed=din * 100 + splits)
        x = x[:32]
        ref, bound = lt.ref64(x, Wt, b, act)
        ratios.append(_ratio(tf32x3_restated(x, Wt, b, act, splits), ref, bound))
    _calibrate(ratios, "split-K")


def test_f32_swish_bound_calibration():
    from _rank_kernels_ref import dot_chain

    ratios = []
    for case in lt.CASES:
        x, Wt, b, act = _rows(case, 8)
        if act != 2:
            continue
        v = dot_chain(x, Wt) + (b if b is not None else F32(0))
        want, bound = lt.f32_restated(x, Wt, b, 2)
        ratios.append(_ratio(_act32(v, 2), want, bound))
    _calibrate(ratios, "f32 swish")


def test_restatement_follows_the_kernel_order():
    """The restatement is the kernel's arithmetic, not any float32 sum: leaving out the correction products or the
    last-chunk promotion of an odd chunk count breaks the bound it is calibrated against."""
    x, Wt, b = lt.make_case(64, 96, 40, True, seed=1)
    ref, bound = lt.ref64(x, Wt, b, 0)
    assert _ratio(tf32x3_restated(x, Wt, b, 0), ref, bound) <= 0.25
    xh, wh = _tf32_trunc(x), _tf32_trunc(Wt)
    single = (xh.astype(F64) @ wh.astype(F64).T + b).astype(F32)
    assert _ratio(single, ref, bound) > 4.0
