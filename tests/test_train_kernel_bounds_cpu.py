"""Calibration of the error bounds of tests/test_gpu_train_kernels.py on the CPU.

Each bound there is C * u * (a per-element or per-row magnitude computed from the inputs).  Here float32
restatements of the same operations run on the same generated cases, with the kernels' precision choices (float32
arithmetic where the kernel uses float, double sums where it accumulates in double, the same summation shape for
the warp reductions): they must meet every bound with a factor 4 to spare (a bound float32 arithmetic cannot meet is
wrong), and the worst case of each family must use at least 1/1000 of it (a bound far looser than float32 needs would
not notice a kernel that is subtly wrong).
"""
import math

import numpy as np

import test_gpu_train_kernels as tk

F32, F64 = np.float32, np.float64


def _ratio(got, ref, bound):
    """max |got - ref| / bound; where the bound is 0 the restatement must be exact."""
    err = np.abs(np.asarray(got, dtype=F64) - ref)
    bound = np.broadcast_to(np.asarray(bound, dtype=F64), err.shape)
    zero = bound == 0
    assert (err[zero] == 0).all(), "an error where the bound is 0"
    return float((err[~zero] / bound[~zero]).max()) if (~zero).any() else 0.0


def _calibrate(ratios, C, what):
    worst = max(ratios)
    print(f"{what}: float32 uses {worst / C:.3g} of the bound (C = {C}, {worst:.3g} unscaled)")
    assert 4.0 * worst <= C, f"{what}: float32 error is not 4x inside the bound ({worst:.3g} * 4 > {C})"
    assert worst >= 1e-3 * C, f"{what}: bound is over 1000x looser than float32 needs ({worst:.3g} vs {C})"


def _warp_sum(acc):
    """Lane 0's result of the xor-shuffle tree over 32 lanes (acc [..., 32], float32)."""
    for o in (16, 8, 4, 2, 1):
        acc = acc[..., :o] + acc[..., o:2 * o]
    return acc[..., 0]


def _lane_chain(terms):
    """float32 per-lane chains over column k = lane, lane + 32, ... then the shuffle tree: terms [R, n]."""
    R, n = terms.shape
    acc = np.zeros((R, 32), dtype=F32)
    for j0 in range(0, n, 32):
        seg = terms[:, j0:j0 + 32]
        acc[:, :seg.shape[1]] += seg
    return _warp_sum(acc)


# ----- batch norm ----------------------------------------------------------------------------------------------------
def bn_stats_f32(x):
    """The kernel's statistics: double sums, rounded to float."""
    x64 = x.astype(F64)
    mu = x64.mean(axis=0)
    return mu.astype(F32), np.square(x64 - mu).mean(axis=0).astype(F32)


def bn_forward_f32(c):
    mean, var = bn_stats_f32(c["x"])
    inv = F32(1) / np.sqrt(var + F32(tk.EPS_BN))
    y = ((c["x"] - mean) * inv) * c["gamma"] + c["beta"]
    mom = F32(tk.MOMENTUM)
    return dict(y=y, mean=mean, var=var, mm=mom * c["mm"] + (F32(1) - mom) * mean,
                mv=mom * c["mv"] + (F32(1) - mom) * var)


def bn_backward_f32(c):
    x, dy, R = c["x"], c["dy"], c["R"]
    mean, var = bn_stats_f32(x)
    s1 = dy.astype(F64).sum(axis=0)
    s2 = (dy.astype(F64) * x.astype(F64)).sum(axis=0)
    inv = F32(1) / np.sqrt(var + F32(tk.EPS_BN))
    xh = (x - mean) * inv
    T = inv * (s2 - mean.astype(F64) * s1).astype(F32)
    invR = F32(1) / F32(R)
    dx = c["gamma"] * inv * (dy - s1.astype(F32) * invR - xh * T * invR)
    inv64 = 1.0 / np.sqrt(var.astype(F64) + F64(F32(tk.EPS_BN)))
    return dict(dx=dx, g_gamma=c["g0_gamma"] + (inv64 * (s2 - mean.astype(F64) * s1)).astype(F32),
                g_beta=c["g0_beta"] + s1.astype(F32))


def test_bn_bounds():
    ratios = []
    for R, K, pad in tk.BN_CASES:
        c = tk.make_bn_case(R, K, pad)
        ref, got = tk.bn_forward_ref(c), bn_forward_f32(c)
        assert got["y"].dtype == F32
        for k in ("y", "mean", "var", "mm", "mv"):
            ratios.append(_ratio(got[k], ref[k], ref["b_" + k]))
        ref, got = tk.bn_backward_ref(c), bn_backward_f32(c)
        ratios.append(_ratio(got["dx"], ref["dx"], ref["b_dx"]))
        ratios.append(_ratio(got["g_gamma"], ref["g_gamma"], ref["b_gamma"]))
        ratios.append(_ratio(got["g_beta"], ref["g_beta"], ref["b_beta"]))
    _calibrate(ratios, tk.C_BN, "batch norm")


def test_bn_restatement_matches_autograd():
    for R, K, pad in tk.BN_CASES:
        c = tk.make_bn_case(R, K, pad)
        fwd, bwd, auto = tk.bn_forward_ref(c), tk.bn_backward_ref(c), tk.bn_autograd(c)
        assert _ratio(fwd["y"], auto["y"], fwd["b_y"]) <= 1e-3
        assert _ratio(bwd["dx"], auto["dx"], bwd["b_dx"]) <= 1e-3
        assert _ratio(bwd["g_gamma"] - c["g0_gamma"], auto["dgamma"], bwd["b_gamma"]) <= 1e-3


# ----- FM / DeepFM heads, Dense(1) on a concat --------------------------------------------------------------------------
def fm_forward_f32(c):
    y, w = c["y"], c["w"]
    z = np.full(c["R"], c["b"] if c["b"] is not None else F32(0), dtype=F32)
    for k in range(c["K"]):
        z = z + y[:, k] * w[k]
    elu = np.where(z > 0, z, np.expm1(np.minimum(z, F32(0))))
    lb = c["lb"] if c["lb"] is not None else F32(0)
    return z, (c["lin"] + lb) + elu


def fm_backward_f32(c):
    R, K, pw, w, dl, z = c["R"], c["K"], c["pw"], c["w"], c["dlogit"], c["z"]
    dz = dl * np.where(z > 0, F32(1), np.exp(np.minimum(z, F32(0))))
    D = dz.astype(F64).sum()
    out = dict(g_b=c["g0_b"] + F32(D), g_lb=c["g0_lb"] + F32(dl.astype(F64).sum()))
    if c["use_bn"]:
        mean, var = c["mean"], c["var"]
        inv = F32(1) / np.sqrt(var + F32(tk.EPS_BN))
        xh = (pw - mean) * inv
        T = dz.astype(F64) @ xh.astype(F64)
        invR = F32(1) / F32(R)
        g, be = c["gamma"].astype(F64), c["beta"].astype(F64)
        out.update(dpw=inv * w * c["gamma"] * (dz[:, None] - F32(D) * invR - xh * T.astype(F32) * invR),
                   g_w=c["g0_w"] + (g * T + be * D).astype(F32), g_gamma=c["g0_gamma"] + (w.astype(F64) * T).astype(F32),
                   g_beta=c["g0_beta"] + (w.astype(F64) * D).astype(F32))
    else:
        out.update(dpw=dz[:, None] * w, g_w=c["g0_w"] + (dz.astype(F64) @ pw.astype(F64)).astype(F32))
    return out


def deepfm_forward_f32(c):
    K = c["K"]
    w = c["w"]
    lb = c["lb"] if c["lb"] is not None else F32(0)
    acc = (c["b"] if c["b"] is not None else F32(0)) + (c["lin"] + lb) * w[0]
    for k in range(K):
        acc = acc + c["pw"][:, k] * w[1 + k]
    for j in range(c["H"]):
        acc = acc + c["deep"][:, j] * w[1 + K + j]
    return acc


def concat_f32(c):
    w = c["w"]
    acc = np.zeros((c["R"], 32), dtype=F32)
    off = 0
    for b in c["blocks"]:
        m = b.shape[1]
        for j0 in range(0, m, 32):
            seg = b[:, j0:j0 + 32] * w[off + j0:off + min(j0 + 32, m)]
            acc[:, :seg.shape[1]] += seg
        off += m
    return _warp_sum(acc) + c["bias"]


def test_head_bounds():
    ratios = []
    for args in tk.FM_FWD_CASES:
        c = tk.make_fm_fwd_case(*args)
        ref = tk.fm_forward_ref(c)
        z, logit = fm_forward_f32(c)
        ratios += [_ratio(z, ref["z"], ref["b_z"]), _ratio(logit, ref["logit"], ref["b_logit"])]
    for args in tk.FM_BWD_CASES:
        c = tk.make_fm_bwd_case(*args)
        ref, got = tk.fm_backward_ref(c), fm_backward_f32(c)
        for k in got:
            ratios.append(_ratio(got[k], ref[k], ref["b_" + k[2:]] if k.startswith("g_") else ref["b_dpw"]))
    for args in tk.DEEPFM_CASES:
        c = tk.make_deepfm_case(*args)
        ref, bound = tk.deepfm_forward_ref(c)
        ratios.append(_ratio(deepfm_forward_f32(c), ref, bound))
    for args in tk.CONCAT_CASES:
        c = tk.make_concat_case(*args)
        ref, bound = tk.concat_ref(c)
        ratios.append(_ratio(concat_f32(c), ref, bound))
    _calibrate(ratios, tk.C_HEAD, "FM / DeepFM heads, Dense(1) on a concat")


def test_fm_restatement_matches_autograd():
    for args in tk.FM_BWD_CASES:
        tk.check_fm_restatement(tk.make_fm_bwd_case(*args))


def test_fm_forward_cases_reach_both_elu_branches():
    zs = np.concatenate([tk.fm_forward_ref(tk.make_fm_fwd_case(*a))["z"] for a in tk.FM_FWD_CASES])
    assert (zs < -10).any() and (zs > 1).any() and ((np.abs(zs) < 1e-5) & (zs < 0)).any()


# ----- scatters ---------------------------------------------------------------------------------------------------------------
def feat_backward_f32(c):
    """Float32 contributions in the kernel's form, added to the float32 initial values in row order."""
    K = c["K"]
    g = {k: v.copy() for k, v in c["g0"].items()}
    lk = c["lin_kernel"]
    for j, (t, idx, x, lt) in enumerate(tk.feat_fields(c)):
        x = x.astype(F32)
        e = c["w"][t][idx] * x[:, None]
        ge = np.zeros((c["R"], K), dtype=F32)
        if c["dpw"] is not None:
            ge = c["dpw"] * (c["S"] - e)
        if c["dconcat"] is not None:
            ge = ge + c["dconcat"][:, j * K:(j + 1) * K]
        np.add.at(g[t], idx, ge * x[:, None])
        if c["dlogit"] is not None:
            dl = c["dlogit"]
            np.add.at(g[lt], idx, dl * lk[j] * x)
            g["lin_kernel"][j] += (dl * x * c["w"][lt][idx]).sum(dtype=F32)
    return g


def test_scatter_bounds():
    ratios = []
    for args in tk.FEAT_CASES:
        c = tk.make_feat_case(*args)
        ref, mag, cnt = tk.feat_backward_ref(c)
        bound = tk.feat_bound(mag, cnt)
        got = feat_backward_f32(c)
        for k in ref:
            assert got[k].dtype == F32
            ratios.append(_ratio(got[k], ref[k], bound[k]))
    for d in tk.ROW_D:
        c = tk.make_rows_case(d)
        ref, bound, _ = tk.scatter_ref(c)
        g = c["g0"].copy()
        np.add.at(g, c["idx"], c["rows"])
        ratios.append(_ratio(g, ref, bound))
    _calibrate(ratios, tk.C_SCATTER, "scatter-adds")


def test_feat_cases_cover_the_kernel_branches():
    """Partial last warps wherever a warp holds more than one row, every id layout, every input combination."""
    seen = set()
    for K, which, inputs, dl, R in tk.FEAT_CASES:
        lpr = 1
        while lpr < K and lpr < 32:
            lpr *= 2
        rows_per_warp = 32 // lpr
        assert rows_per_warp == 1 or R % rows_per_warp != 0
        seen |= {("layout", which), ("inputs", inputs), ("dlogit", dl), ("lanes", "idle" if K % lpr else "full"),
                 ("loop", K > 32)}
    assert len(seen) == 4 + 3 + 2 + 2 + 2


# ----- L2 normalisation ---------------------------------------------------------------------------------------------------
def l2_f32(c):
    x, dy = c["x"], c["dy"]
    ss = _lane_chain(x * x)
    xd = _lane_chain(x * dy)
    eps = F32(tk.EPS_L2)
    inv = F32(1) / np.sqrt(np.maximum(ss, eps))
    cc = np.where(ss < eps, F32(0), xd * inv * inv * inv)       # in this order: inv^3 alone underflows at |x| ~ 1e18
    return x * inv[:, None], dy * inv[:, None] - x * cc[:, None], ss


def test_l2_bounds():
    ratios = []
    for d in tk.L2_D:
        c = tk.make_l2_case(d)
        ref = tk.l2_ref(c)
        y, dx, ss = l2_f32(c)
        for r in c["tie"]:
            assert ss[r] == F32(tk.EPS_L2)                      # float32 lands on the tie too
        assert ((ss < F32(tk.EPS_L2)) == ref["clamped"]).all()
        ratios += [_ratio(y, ref["y"], ref["b_y"]), _ratio(dx, ref["dx"], ref["b_dx"])]
    _calibrate(ratios, tk.C_L2, "L2 normalisation")


def test_l2_restatement_matches_autograd():
    for d in tk.L2_D:
        c = tk.make_l2_case(d)
        ref = tk.l2_ref(c)
        y, dx = tk.l2_autograd(c)
        assert _ratio(y, ref["y"], ref["b_y"]) <= 1e-3
        assert _ratio(dx, ref["dx"], ref["b_dx"]) <= 1e-3


# ----- Adam ------------------------------------------------------------------------------------------------------------------
def adam_f32(c):
    b1, b2, eps = tk.ADAM_B1, tk.ADAM_B2, tk.ADAM_EPS
    p = c["p0"].copy()
    m, v = np.zeros_like(p), np.zeros_like(p)
    for t in range(1, len(c["g"]) + 1):
        g = c["g"][t - 1]
        m = b1 * m + (F32(1) - b1) * g
        v = b2 * v + (F32(1) - b2) * g * g
        p = p - F32(tk.adam_lr_t(t)) * m / (np.sqrt(v) + eps)
    return dict(p=p, m=m, v=v)


def test_adam_bounds():
    c = tk.make_adam_case()
    ref, got = tk.adam_ref(c), adam_f32(c)
    assert got["p"].dtype == F32
    _calibrate([_ratio(got[k], ref[k], ref["b_" + k]) for k in ("p", "m", "v")], tk.C_ADAM, "Adam, 20 steps")


def test_adam_lr_t_formula():
    """TF's bias-corrected step size, and the staircase: the decay counts completed steps."""
    assert tk.adam_lr_t(1) == float(tk.ADAM_LR) * math.sqrt(1.0 - float(tk.ADAM_B2)) / (1.0 - float(tk.ADAM_B1))
    r = F32(0.5)
    lr = [tk.adam_lr_t(t, decay_rate=r, decay_steps=3) / tk.adam_lr_t(t) for t in range(1, 8)]
    assert lr == [1.0, 1.0, 1.0, 0.5, 0.5, 0.5, 0.25]


# ----- pointwise loss ------------------------------------------------------------------------------------------------------
def loss_f32(c, kind):
    x = c["x"]
    y = c["yr"] if kind == 2 else c["y01"]
    n = c["n"]
    if kind == 2:
        d = x - y
        v, g = d * d, F32(2) * d
    else:
        bce = np.maximum(x, F32(0)) - x * y + np.log1p(np.exp(-np.abs(x)))
        p = np.where(x >= 0, F32(1) / (F32(1) + np.exp(-np.abs(x))), np.exp(-np.abs(x)) / (F32(1) + np.exp(-np.abs(x))))
        if kind == 0:
            v, g = bce, p - y
        else:
            a, gam = tk.FOCAL_ALPHA, tk.FOCAL_GAMMA
            wt = y * a + (F32(1) - y) * (F32(1) - a)
            pt = y * p + (F32(1) - y) * (F32(1) - p)
            om = F32(1) - pt
            mm = np.power(om, gam)
            dpt = (F32(2) * y - F32(1)) * p * (F32(1) - p)
            dm = np.where(om > 0, -gam * np.power(om, gam - F32(1)) * dpt, F32(0))
            v, g = wt * mm * bce, wt * (dm * bce + mm * (p - y))
    assert v.dtype == F32 and g.dtype == F32
    chain = -(-n // tk.LOSS_THREADS)
    vp = np.zeros(chain * tk.LOSS_THREADS, dtype=F32)
    vp[:n] = v
    vp = vp.reshape(chain, tk.LOSS_THREADS)
    acc = np.zeros(tk.LOSS_THREADS, dtype=F32)
    for i in range(chain):                                      # each thread's float sum over its grid-stride rounds
        acc = acc + vp[i]
    return acc.astype(F64).sum() / n, g * (F32(1) / F32(n))


def test_loss_bounds():
    c = tk.make_loss_case()
    chain = -(-c["n"] // tk.LOSS_THREADS)
    ratios = []
    for kind in (0, 1, 2):
        L, g, vm, gm = tk.loss_ref(c, kind)
        L32, g32 = loss_f32(c, kind)
        ratios += [_ratio(g32, g, tk.U * gm / c["n"]), _ratio(L32, L, tk.U * (chain + 2) * vm.sum() / c["n"])]
    _calibrate(ratios, tk.C_LOSS, "pointwise loss")
