"""The shared training kernels, called directly through the C-ABI and compared with float64 restatements of the same
operations: batch norm with batch statistics (``csrc/train.cu``: forward, backward, ReLU mask), the FM and DeepFM
heads, the field-gradient scatter ``b200_feat_backward``, the ReLU backward, TF-Adam on the host and on the device
step counter, ``b200_axpy``, the row helpers of ``csrc/feat.cu`` (gather, scatter-add, Dense(1) on a concat, L2
normalisation forward and backward) and ``b200_pointwise_loss`` past the point where its grid stops growing.

Every trainer runs on these kernels, and the trainer tests see them only through whole-model gradients at one or two
batch shapes.  Here each kernel runs at the shapes where it branches: one and two rows, partial last warps, idle
lanes and k loops of the field scatter (K = 1 ... 64), all four id layouts, leading dimensions above the width,
constant columns, |mean| >> std, exact zeros under the ReLU mask, the elu branches, hot keys, L2 rows below, on and
far above the clamp.

Error bounds are stated per element (or per row) in quantities the test computes, with u = 2^-24:
  BN forward         C_BN u (|gamma| (|xhat| + |mean| inv) + |beta|)        inv = 1 / sqrt(var + eps); the |mean| inv
                     term is the rounding of the float batch mean, which |mean| >> std magnifies;
                     batch mean C_BN u mean|x|, batch variance C_BN u var, moving statistics C_BN u (|moving| + |stat|)
  BN backward        C_BN u |gamma| inv (|dy| + A / R + (|xhat| + |mean| inv) (Tm + |mean| inv A) / R)
                     A = sum_r |dy|, Tm = sum_r |dy xhat| per column; g_gamma C_BN u (|g0| + Tm + |mean| inv A),
                     g_beta C_BN u (|g0| + A)
  FM head            z: C_HEAD u (K + 1) (|b| + sum_k |y w|) (a chain of K fmaf), logit adds |lin| + |lin_bias| +
                     |elu(z)|; the backward is the
                     BN backward with dy = dz w and dz weighted by (1 + |z|) for the elu derivative of a rounded z
  DeepFM head        C_HEAD u (K + H + 2) (|b| + (|lin| + |lin_bias|) |w_0| + sum |pw w| + sum |deep w|); its
                     backward is exact
  scatters           C_SCATTER u (n + 1) (|g0| + sum |contribution|) per element, n = the number of contributions to
                     the element: the float atomics add them in any order
  Dense(1) on concat C_HEAD u (lane chain + 6) (|bias| + sum |a w|)
  L2 normalise       C_L2 u (ceil(d / 32) + 6) |x_k| inv forward; backward C_L2 u (ceil(d / 32) + 6) (|dy_k| inv +
                     |x_k| inv^3 sum_j |x_j dy_j|), inv = rsqrt(max(|x|^2, 1e-12))
  Adam, 20 steps     weights C_ADAM u sum_t (|p_t| + t lr_t (M_t + |m_t|) / (sqrt(v_t) + eps)), slots C_ADAM u t M_t
                     and C_ADAM u t v_t, with M_t the first moment of |g| (the rounding of m and v piles up over t)
  pointwise loss     gradient C_LOSS u gmag / n per element; loss C_LOSS u (per-thread chain + 2) sum vmag / n
The constants are checked against float32 restatements of the same cases on the CPU
(tests/test_train_kernel_bounds_cpu.py): float32 meets every bound with at least a factor 4 to spare, and the worst
case of every family uses at least 1/1000 of its bound.  Where the kernel is exact the test is exact: gathers,
products, the ReLU masks, the step size within 1 ulp, and untouched gradient rows bit for bit.
"""
from __future__ import annotations

import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
F32, F64 = np.float32, np.float64
EPS_BN = float(F32(1e-3))              # tf.layers.batch_normalization epsilon, as the float the kernels add
MOMENTUM = float(F32(0.99))
EPS_L2 = float(F32(1e-12))             # tf.linalg.l2_normalize epsilon

# bound constants (see the module docstring); calibrated by tests/test_train_kernel_bounds_cpu.py
C_BN = 16.0          # batch norm forward and backward
C_HEAD = 16.0        # FM / DeepFM heads, Dense(1) on a concat
C_SCATTER = 4.0      # float-atomic scatters (feat_backward, scatter_add_rows)
C_L2 = 4.0           # L2 normalisation forward / backward
C_ADAM = 4.0         # 20 Adam steps
C_LOSS = 24.0        # pointwise loss


def _f64(a):
    return np.asarray(a, dtype=F64)


# ---------------------------------------------------------------------------------------------------------------------
# case generation and float64 restatements (numpy / CPU torch only: shared with the CPU calibration)
# ---------------------------------------------------------------------------------------------------------------------
# ----- batch norm ----------------------------------------------------------------------------------------------------
BN_CASES = [(1, 8, 0), (2, 5, 3), (7, 33, 1), (129, 64, 4), (1000, 40, 0), (300, 130, 2)]     # (R, K, ld - K)


def make_bn_case(R, K, pad):
    rng = np.random.default_rng(100 * R + K)
    x = rng.standard_normal((R, K)) * rng.uniform(0.1, 3.0, K) + rng.normal(0.0, 1.0, K)
    x[rng.random((R, K)) < 0.2] = 0.0                        # exact zeros: the ReLU mask must stop them
    if K >= 3:
        x[:, 1] = 2.5                                        # constant column: variance 0, rsqrt(eps)
        x[:, 2] = 1000.0 + 0.01 * rng.standard_normal(R)     # |mean| >> std
    return dict(R=R, K=K, pad=pad, x=x.astype(F32), dy=rng.standard_normal((R, K)).astype(F32),
                gamma=rng.uniform(0.5, 1.5, K).astype(F32), beta=rng.normal(0.0, 0.1, K).astype(F32),
                mm=rng.normal(0.0, 0.1, K).astype(F32), mv=rng.uniform(0.5, 1.5, K).astype(F32),
                g0_gamma=rng.normal(0.0, 1.0, K).astype(F32), g0_beta=rng.normal(0.0, 1.0, K).astype(F32))


def bn_stats(x):
    """Batch mean, biased variance and 1 / sqrt(var + eps) per column, float64."""
    x = _f64(x)
    mu = x.mean(axis=0)
    var = np.square(x - mu).mean(axis=0)
    return mu, var, 1.0 / np.sqrt(var + EPS_BN)


def bn_forward_ref(c):
    """y, batch statistics and moving statistics of tf.layers.batch_normalization(training=True), with bounds."""
    x = _f64(c["x"])
    mu, var, inv = bn_stats(x)
    xh = (x - mu) * inv
    g, b = _f64(c["gamma"]), _f64(c["beta"])
    mm = MOMENTUM * _f64(c["mm"]) + (1.0 - MOMENTUM) * mu
    mv = MOMENTUM * _f64(c["mv"]) + (1.0 - MOMENTUM) * var
    return dict(y=g * xh + b, mean=mu, var=var, mm=mm, mv=mv,
                b_y=U * (np.abs(g) * (np.abs(xh) + np.abs(mu) * inv) + np.abs(b)),
                b_mean=U * np.abs(x).mean(axis=0), b_var=U * var,
                b_mm=U * (np.abs(c["mm"]) + np.abs(mu)), b_mv=U * (np.abs(c["mv"]) + var))


def bn_backward_ref(c):
    """dx (before the ReLU mask), g_gamma, g_beta (added to their initial values) of BN with batch statistics."""
    x, dy, R = _f64(c["x"]), _f64(c["dy"]), c["R"]
    mu, var, inv = bn_stats(x)
    xh = (x - mu) * inv
    g = _f64(c["gamma"])
    s1, T = dy.sum(axis=0), (dy * xh).sum(axis=0)
    dx = g * inv * (dy - s1 / R - xh * T / R)
    A, Tm = np.abs(dy).sum(axis=0), (np.abs(dy) * np.abs(xh)).sum(axis=0)
    mi = np.abs(mu) * inv
    return dict(dx=dx, g_gamma=_f64(c["g0_gamma"]) + T, g_beta=_f64(c["g0_beta"]) + s1,
                b_dx=U * np.abs(g) * inv * (np.abs(dy) + A / R + (np.abs(xh) + mi) * (Tm + mi * A) / R),
                b_gamma=U * (np.abs(c["g0_gamma"]) + Tm + mi * A), b_beta=U * (np.abs(c["g0_beta"]) + A))


def bn_autograd(c):
    """torch float64 autograd of BN with batch statistics: y, dx, d gamma, d beta for the loss sum(y * dy)."""
    import torch

    t = {k: torch.tensor(_f64(c[k]), requires_grad=True) for k in ("x", "gamma", "beta")}
    mu = t["x"].mean(dim=0)
    var = ((t["x"] - mu) ** 2).mean(dim=0)
    y = (t["x"] - mu) / torch.sqrt(var + EPS_BN) * t["gamma"] + t["beta"]
    (y * torch.tensor(_f64(c["dy"]))).sum().backward()
    return dict(y=y.detach().numpy(), dx=t["x"].grad.numpy(), dgamma=t["gamma"].grad.numpy(),
                dbeta=t["beta"].grad.numpy())


# ----- FM head ---------------------------------------------------------------------------------------------------------
FM_FWD_CASES = [(1, 1, True, True), (300, 16, True, False), (1000, 33, False, True), (257, 64, False, False)]
FM_BWD_CASES = [(1, 4, True, True), (2, 16, True, False), (777, 16, True, True), (2048, 33, True, True),
                (1000, 16, False, True), (513, 1, False, False)]                     # (R, K, use_bn, g_lin_bias)


def make_fm_fwd_case(R, K, has_b, has_lb):
    """Rows of three magnitudes: y ~ 1e-7 (z next to 0, lin = 0: where expm1f and expf(z) - 1 differ), 1 and 5
    (z of order 10 either way: the strongly negative side of elu)."""
    rng = np.random.default_rng(7 * R + K)
    s = rng.choice([1e-7, 1.0, 5.0], R)
    y = rng.standard_normal((R, K)) * s[:, None]
    lin = rng.standard_normal(R)
    lin[s == 1e-7] = 0.0
    return dict(R=R, K=K, y=y.astype(F32), w=rng.normal(0.0, 2.0 / np.sqrt(K), K).astype(F32),
                b=F32(-0.7) if has_b else None, lin=lin.astype(F32), lb=F32(0.3) if has_lb else None)


def fm_forward_ref(c):
    y, w = _f64(c["y"]), _f64(c["w"])
    b = float(c["b"]) if c["b"] is not None else 0.0
    lb = float(c["lb"]) if c["lb"] is not None else 0.0
    z = y @ w + b
    elu = np.where(z > 0, z, np.expm1(np.minimum(z, 0.0)))
    zmag = (c["K"] + 1) * (np.abs(y) @ np.abs(w) + abs(b))          # a chain of K fmaf
    lin = _f64(c["lin"])
    return dict(z=z, logit=lin + lb + elu, b_z=U * zmag, b_logit=U * (zmag + np.abs(lin) + abs(lb) + np.abs(elu)))


def make_fm_bwd_case(R, K, use_bn, has_glb):
    rng = np.random.default_rng(11 * R + K + (1 if use_bn else 0))
    pw = rng.standard_normal((R, K)) * rng.uniform(0.2, 3.0, K) + rng.normal(0.0, 1.0, K)
    c = dict(R=R, K=K, use_bn=use_bn, has_glb=has_glb, pw=pw.astype(F32),
             gamma=rng.uniform(0.5, 1.5, K).astype(F32), beta=rng.normal(0.0, 0.1, K).astype(F32),
             w=rng.normal(0.0, 2.0 / np.sqrt(K), K).astype(F32), b=F32(-0.5), lin=rng.standard_normal(R).astype(F32),
             lb=F32(0.1), dlogit=rng.standard_normal(R).astype(F32))
    for k, n in (("w", K), ("b", 1), ("gamma", K), ("beta", K), ("lb", 1)):
        c["g0_" + k] = rng.normal(0.0, 1.0, n).astype(F32)
    c["z"] = fm_bwd_z(c).astype(F32)
    if use_bn:
        mu, var, _ = bn_stats(c["pw"])
        c["mean"], c["var"] = mu.astype(F32), var.astype(F32)
    return c


def fm_bwd_z(c):
    """z = <BN(pw), w> + b in float64 (the forward's float z is this, rounded)."""
    y = _f64(c["pw"])
    if c["use_bn"]:
        mu, _, inv = bn_stats(y)
        y = _f64(c["gamma"]) * (y - mu) * inv + _f64(c["beta"])
    return y @ _f64(c["w"]) + float(c["b"])


def fm_backward_ref(c, z=None):
    """d pw and the parameter gradients (added to their initial values) of logit = lin + lin_bias + elu(z),
    z = <BN(pw), w> + b, for the loss sum(dlogit * logit); with their bounds.  The elu derivative is taken at the
    float z the kernel is given (``z`` overrides it)."""
    R, pw, w, dl = c["R"], _f64(c["pw"]), _f64(c["w"]), _f64(c["dlogit"])
    z = _f64(c["z"] if z is None else z)
    dz = dl * np.where(z > 0, 1.0, np.exp(np.minimum(z, 0.0)))
    dzm = np.abs(dz) * (1.0 + np.abs(z))
    D, A = dz.sum(), dzm.sum()
    out = dict(g_b=_f64(c["g0_b"]) + D, g_lb=_f64(c["g0_lb"]) + dl.sum(),
               b_b=U * (np.abs(c["g0_b"]) + A), b_lb=U * (np.abs(c["g0_lb"]) + np.abs(dl).sum()))
    if c["use_bn"]:
        g, be = _f64(c["gamma"]), _f64(c["beta"])
        mu, _, inv = bn_stats(pw)
        xh = (pw - mu) * inv
        T = dz @ xh
        Tm = dzm @ np.abs(xh)
        mi = np.abs(mu) * inv
        Tb = Tm + mi * A
        out.update(dpw=inv * w * g * (dz[:, None] - D / R - xh * T / R),
                   b_dpw=U * np.abs(w * g) * inv * (dzm[:, None] + A / R + (np.abs(xh) + mi) * Tb / R),
                   g_w=_f64(c["g0_w"]) + g * T + be * D, b_w=U * (np.abs(c["g0_w"]) + np.abs(g) * Tb + np.abs(be) * A),
                   g_gamma=_f64(c["g0_gamma"]) + w * T, b_gamma=U * (np.abs(c["g0_gamma"]) + np.abs(w) * Tb),
                   g_beta=_f64(c["g0_beta"]) + w * D, b_beta=U * (np.abs(c["g0_beta"]) + np.abs(w) * A))
    else:
        out.update(dpw=dz[:, None] * w, b_dpw=U * dzm[:, None] * np.abs(w),
                   g_w=_f64(c["g0_w"]) + dz @ pw, b_w=U * (np.abs(c["g0_w"]) + dzm @ np.abs(pw)))
    return out


def fm_head_autograd(c):
    """torch float64 autograd of the same head: gradients of sum(dlogit * logit) (without the initial values)."""
    import torch

    names = ["pw", "w", "b", "lb"] + (["gamma", "beta"] if c["use_bn"] else [])
    t = {k: torch.tensor(_f64(c[k]).reshape(np.shape(c[k])), requires_grad=True) for k in names}
    y = t["pw"]
    if c["use_bn"]:
        mu = y.mean(dim=0)
        var = ((y - mu) ** 2).mean(dim=0)
        y = (y - mu) / torch.sqrt(var + EPS_BN) * t["gamma"] + t["beta"]
    z = y @ t["w"] + t["b"]
    logit = torch.tensor(_f64(c["lin"])) + t["lb"] + torch.nn.functional.elu(z)
    (logit * torch.tensor(_f64(c["dlogit"]))).sum().backward()
    return {k: t[k].grad.numpy() for k in names}


def check_fm_restatement(c):
    """The closed-form backward equals torch float64 autograd (both at the float64 z) far inside the kernel's bound."""
    ref = fm_backward_ref(c, z=fm_bwd_z(c))
    auto = fm_head_autograd(c)
    tiny = 1e-3 * C_HEAD
    _check(ref["dpw"], auto["pw"], tiny * ref["b_dpw"] + 1e-300, "restatement vs autograd: d pw")
    pairs = [("w", "w"), ("b", "b"), ("lb", "lb")] + ([("gamma", "gamma"), ("beta", "beta")] if c["use_bn"] else [])
    for k, a in pairs:
        _check(ref["g_" + k] - c["g0_" + k], auto[a], tiny * ref["b_" + k], f"restatement vs autograd: d {k}")


# ----- DeepFM head ----------------------------------------------------------------------------------------------------
DEEPFM_CASES = [(1000, 1, 1, 2, True), (257, 16, 32, 5, False), (1, 8, 3, 0, True)]     # (R, K, H, ld - H, bias)


def make_deepfm_case(R, K, H, pad, has_b):
    rng = np.random.default_rng(13 * R + K + H)
    return dict(R=R, K=K, H=H, pad=pad, lin=rng.standard_normal(R).astype(F32),
                lb=F32(0.2) if has_b else None, pw=rng.standard_normal((R, K)).astype(F32),
                deep=rng.standard_normal((R, H)).astype(F32), w=rng.standard_normal(1 + K + H).astype(F32),
                b=F32(-0.4) if has_b else None, dlogit=rng.standard_normal(R).astype(F32))


def deepfm_forward_ref(c):
    K = c["K"]
    w = _f64(c["w"])
    b = float(c["b"]) if c["b"] is not None else 0.0
    lb = float(c["lb"]) if c["lb"] is not None else 0.0
    lin = _f64(c["lin"])
    out = b + (lin + lb) * w[0] + _f64(c["pw"]) @ w[1:1 + K] + _f64(c["deep"]) @ w[1 + K:]
    mag = abs(b) + (np.abs(lin) + abs(lb)) * abs(w[0]) + np.abs(c["pw"]) @ np.abs(w[1:1 + K]) + \
        np.abs(c["deep"]) @ np.abs(w[1 + K:])
    return out, U * (K + c["H"] + 2) * mag                            # a chain of K + H + 1 fmaf


# ----- field-gradient scatter (b200_feat_backward) ----------------------------------------------------------------------
# (K, layout, inputs, dlogit, R): K = 1 / 4 / 8 / 12 / 16 have 32 / 8 / 4 / 2 / 2 rows per warp and every R leaves a
# partial last warp; K = 12 / 20 leave lanes idle, K = 48 / 64 loop over k.  Layouts: "full" (id_mask 3), "user"
# (1), "item" (2), "user_noid" (0, the YouTubeRetrieval user tower).
FEAT_CASES = [(1, "full", "both", True, 2047), (12, "full", "dpw", True, 1001), (16, "full", "both", False, 1999),
              (20, "user", "dconcat", False, 999), (48, "item", "both", True, 1000), (64, "full", "dconcat", True, 513),
              (8, "user_noid", "dconcat", False, 1003), (4, "user", "both", True, 1025),
              (12, "item", "dpw", False, 777)]
TABLES = ("user_embeds", "item_embeds", "sparse_embeds", "dense_embeds",
          "user_linear", "item_linear", "sparse_linear", "dense_linear")
LAYOUT_ARGS = {"full": None, "user": ("user", True), "item": ("item", True), "user_noid": ("user", False)}


def feat_layout(fs, which):
    """(b200_feat_layout, global field positions) of a FeatSpec for one of the four layouts."""
    if LAYOUT_ARGS[which] is None:
        return fs.layout, list(range(2 + fs.n_sparse + fs.n_dense))
    return fs.side(*LAYOUT_ARGS[which])


def make_feat_case(K, which, inputs, with_dlogit, R):
    """A real feature layout (oracle.tf_models.make_spec: 5 sparse fields with vocabularies of 3 ... 7, 3 dense fields,
    interleaved user / item columns), hot keys (half the rows share one user, half one item), and a last row whose
    user and item appear nowhere else.  The field positions of the layout come from FeatSpec itself (on the CPU)."""
    import torch

    from librecommender_b200.feat_models import FeatSpec
    from oracle import tf_models as tm

    rng = np.random.default_rng(1000 * K + R)
    n_users, n_items = 60, 80
    spec = tm.make_spec(rng, n_users, n_items, [3, 7], [5, 4, 6], 1, 2)
    w = tm.make_embeddings(rng, spec, K, linear=True)
    users = rng.integers(0, n_users - 1, R)
    items = rng.integers(0, n_items - 1, R)
    users[rng.random(R) < 0.5] = 7
    items[rng.random(R) < 0.5] = 3
    users[-1], items[-1] = n_users - 1, n_items - 1
    fs = FeatSpec(spec, K, device=torch.device("cpu"))
    _, pos = feat_layout(fs, which)
    sparse, dense = tm.row_features(spec, users, items)
    c = dict(K=K, which=which, R=R, spec=spec, w=w, users=users.astype(np.int64), items=items.astype(np.int64),
             pos=pos, sparse=sparse, dense=dense, n_sparse=spec["n_sparse"])
    fields = feat_fields(c)
    Fl = len(pos)
    S = sum(_f64(w[t])[idx] * x[:, None] for t, idx, x, _ in fields)
    c["S"] = S.astype(F32)
    c["dpw"] = rng.standard_normal((R, K)).astype(F32) if inputs in ("dpw", "both") else None
    c["dconcat"] = rng.standard_normal((R, Fl * K)).astype(F32) if inputs in ("dconcat", "both") else None
    c["dlogit"] = rng.standard_normal(R).astype(F32) if with_dlogit else None
    c["lin_kernel"] = rng.standard_normal(Fl).astype(F32)
    c["g0"] = {t: rng.normal(0.0, 0.1, np.shape(w[t])).astype(F32) for t in TABLES}
    c["g0"]["lin_kernel"] = rng.normal(0.0, 0.1, Fl).astype(F32)
    return c


def feat_fields(c):
    """Per field of the layout, in its order: (table, row index per batch row, scale per batch row, linear table)."""
    R, ns = c["R"], c["n_sparse"]
    out = []
    for p in c["pos"]:
        if p == 0:
            out.append(("user_embeds", c["users"], np.ones(R), "user_linear"))
        elif p == 1:
            out.append(("item_embeds", c["items"], np.ones(R), "item_linear"))
        elif p < 2 + ns:
            out.append(("sparse_embeds", c["sparse"][:, p - 2].astype(np.int64), np.ones(R), "sparse_linear"))
        else:
            out.append(("dense_embeds", np.full(R, p - 2 - ns), _f64(c["dense"][:, p - 2 - ns]), "dense_linear"))
    return out


def feat_backward_ref(c):
    """Gradient buffers after the scatter (float64, initial values included), the magnitude sum |g0| + sum |contribution|
    and the number of contributions of every element."""
    K = c["K"]
    w = c["w"]
    g = {k: _f64(v).copy() for k, v in c["g0"].items()}
    mag = {k: np.abs(_f64(v)) for k, v in c["g0"].items()}
    cnt = {k: np.zeros(np.shape(v)[0], dtype=np.int64) for k, v in c["g0"].items()}
    dpw, S, dc, dl = (None if c[k] is None else _f64(c[k]) for k in ("dpw", "S", "dconcat", "dlogit"))
    lk = _f64(c["lin_kernel"])
    for j, (t, idx, x, lt) in enumerate(feat_fields(c)):
        e = _f64(w[t])[idx] * x[:, None]
        ge = np.zeros((c["R"], K))
        gm = np.zeros((c["R"], K))
        if dpw is not None:
            ge += dpw * (S - e)
            gm += np.abs(dpw) * (np.abs(S) + np.abs(e))
        if dc is not None:
            ge += dc[:, j * K:(j + 1) * K]
            gm += np.abs(dc[:, j * K:(j + 1) * K])
        np.add.at(g[t], idx, ge * x[:, None])
        np.add.at(mag[t], idx, gm * np.abs(x)[:, None])
        np.add.at(cnt[t], idx, 1)
        if dl is not None:
            np.add.at(g[lt], idx, dl * lk[j] * x)
            np.add.at(mag[lt], idx, np.abs(dl * lk[j] * x))
            np.add.at(cnt[lt], idx, 1)
            contrib = dl * _f64(w[lt])[idx] * x
            g["lin_kernel"][j] += contrib.sum()
            mag["lin_kernel"][j] += np.abs(contrib).sum()
            cnt["lin_kernel"][j] += c["R"]
    return g, mag, cnt


def feat_bound(mag, cnt):
    """U (n + 1) (|g0| + sum |contribution|) per element."""
    return {k: U * (cnt[k] + 1).reshape((-1,) + (1,) * (mag[k].ndim - 1)) * mag[k] for k in mag}


# ----- gather / scatter-add / Dense(1) on a concat -----------------------------------------------------------------------
ROW_D = [1, 33, 64]


def make_rows_case(d):
    rng = np.random.default_rng(d)
    n_rows, n = 50, 1005
    idx = rng.integers(0, n_rows - 5, n)
    idx[rng.random(n) < 0.3] = 2                                       # a hot row; the last 5 rows stay untouched
    return dict(d=d, table=rng.standard_normal((n_rows, d)).astype(F32), idx=idx.astype(np.int64),
                rows=rng.standard_normal((n, d)).astype(F32), g0=rng.normal(0.0, 0.1, (n_rows, d)).astype(F32))


def scatter_ref(c):
    g = _f64(c["g0"]).copy()
    mag = np.abs(g)
    cnt = np.zeros(len(g), dtype=np.int64)
    np.add.at(g, c["idx"], _f64(c["rows"]))
    np.add.at(mag, c["idx"], np.abs(_f64(c["rows"])))
    np.add.at(cnt, c["idx"], 1)
    return g, U * (cnt + 1)[:, None] * mag, cnt


CONCAT_CASES = [(16, 0, 0), (33, 64, 5), (1, 130, 0), (0, 7, 40)]


def make_concat_case(na, nb, nc, R=999):
    rng = np.random.default_rng(na + 10 * nb + 100 * nc)
    return dict(R=R, n=(na, nb, nc), blocks=[rng.standard_normal((R, m)).astype(F32) for m in (na, nb, nc)],
                w=rng.standard_normal(na + nb + nc).astype(F32), bias=F32(0.25))


def concat_ref(c):
    x = np.concatenate([_f64(b) for b in c["blocks"]], axis=1)
    w = _f64(c["w"])
    depth = sum(-(-m // 32) for m in c["n"]) + 6
    return x @ w + float(c["bias"]), U * depth * (np.abs(x) @ np.abs(w) + abs(float(c["bias"])))


# ----- L2 normalisation ---------------------------------------------------------------------------------------------------
L2_D = [1, 31, 32, 33, 64, 129]
# 4294^2 + 90^2 + 12^2 + 8^2 = 2 * 9223372 and 1e-12f = 9223372 * 2^-63: these four floats times 2^-32 have a squared
# norm of exactly 1e-12f in any summation order, float32 or float64
TIE = (4294.0, 90.0, 12.0, 8.0)


def make_l2_case(d):
    """Rows: ordinary; below the clamp (|x|^2 = 1e-12 / 4 and 0); just above it (4e-12); exactly on it (d >= 4);
    norms around 1e18; dy parallel to x, where the projection term is largest."""
    rng = np.random.default_rng(31 + d)
    R = 40
    x = rng.standard_normal((R, d))
    norms = rng.uniform(0.5, 3.0, R)
    norms[0:4] = 0.5e-6                       # below the clamp
    norms[4:8] = 2e-6                         # above it, with |x|^2 within a factor 4
    norms[8:12] = 1e18
    x = x / np.linalg.norm(x, axis=1, keepdims=True) * norms[:, None]
    x[12] = 0.0
    x = x.astype(F32)
    tie = []
    if d >= 4:
        for r in (13, 14):
            x[r] = 0.0
            cols = rng.choice(d, 4, replace=False)
            x[r, cols] = np.array(TIE, dtype=F32) * F32(2.0 ** -32) * rng.choice([-1, 1], 4).astype(F32)
            tie.append(r)
    dy = rng.standard_normal((R, d))
    dy[15:20] = _f64(x[15:20]) / np.linalg.norm(_f64(x[15:20]), axis=1, keepdims=True)
    for r in tie:
        dy[r] = _f64(x[r]) * 1e6
    return dict(d=d, R=R, x=x, dy=dy.astype(F32), tie=tie)


def l2_ref(c):
    """Forward y, backward dx of y = x rsqrt(max(|x|^2, 1e-12)) (tf.maximum's gradient goes to |x|^2 on a tie), and
    their bounds, float64."""
    x, dy = _f64(c["x"]), _f64(c["dy"])
    ss = np.square(x).sum(axis=1)
    clamped = ss < EPS_L2
    inv = 1.0 / np.sqrt(np.maximum(ss, EPS_L2))
    xd = (x * dy).sum(axis=1)
    cc = np.where(clamped, 0.0, xd * inv ** 3)
    depth = -(-c["d"] // 32) + 6
    return dict(y=x * inv[:, None], dx=dy * inv[:, None] - x * cc[:, None], clamped=clamped, ss=ss,
                b_y=U * depth * np.abs(x) * inv[:, None],
                b_dx=U * depth * (np.abs(dy) * inv[:, None] + np.abs(x) * (inv ** 3 * (np.abs(x * dy)).sum(axis=1))[:, None]))


def l2_autograd(c):
    import torch

    x = torch.tensor(_f64(c["x"]), requires_grad=True)
    ss = (x * x).sum(dim=1, keepdim=True)
    y = x * torch.rsqrt(torch.clamp_min(ss, EPS_L2))           # clamp_min passes the gradient on a tie, like tf.maximum
    (y * torch.tensor(_f64(c["dy"]))).sum().backward()
    return y.detach().numpy(), x.grad.numpy()


# ----- Adam -----------------------------------------------------------------------------------------------------------------
ADAM_N, ADAM_STEPS = 4099, 20
ADAM_LR, ADAM_B1, ADAM_B2, ADAM_EPS = F32(1e-2), F32(0.9), F32(0.999), F32(1e-5)


def make_adam_case():
    """Gradients over eight decades (sqrt(v) from far below eps to far above it), about a third of them zero at every
    step (m and v decay, the weight still moves), some elements that never see a gradient (they must not move)."""
    rng = np.random.default_rng(5)
    n = ADAM_N
    p0 = rng.standard_normal(n).astype(F32)
    scale = 10.0 ** rng.uniform(-7, 1, n)
    sign = rng.choice([-1.0, 1.0], (ADAM_STEPS, n))
    g = sign * scale * rng.uniform(0.5, 1.5, (ADAM_STEPS, n))
    g[rng.random((ADAM_STEPS, n)) < 0.35] = 0.0
    g[:, :50] = 0.0
    return dict(p0=p0, g=g.astype(F32))


def adam_lr_t(t, lr=ADAM_LR, decay_rate=1.0, decay_steps=0):
    """TF-Adam's step size at step t (from 1), with tf.train.exponential_decay(staircase=True) of the completed steps."""
    lr_now = float(lr)
    if decay_steps > 0:
        lr_now *= float(decay_rate) ** ((t - 1) // decay_steps)
    return lr_now * math.sqrt(1.0 - float(ADAM_B2) ** t) / (1.0 - float(ADAM_B1) ** t)


def adam_ref(c):
    """float64 TF-Adam over the case's steps: final p, m, v and their bounds."""
    b1, b2, eps = float(ADAM_B1), float(ADAM_B2), float(ADAM_EPS)
    p = _f64(c["p0"]).copy()
    m, v, M = np.zeros_like(p), np.zeros_like(p), np.zeros_like(p)
    acc = np.zeros_like(p)
    for t in range(1, len(c["g"]) + 1):
        g = _f64(c["g"][t - 1])
        m = b1 * m + (1.0 - b1) * g
        v = b2 * v + (1.0 - b2) * g * g
        M = b1 * M + (1.0 - b1) * np.abs(g)
        lr_t = adam_lr_t(t)
        p = p - lr_t * m / (np.sqrt(v) + eps)
        acc += np.abs(p) + t * lr_t * (M + np.abs(m)) / (np.sqrt(v) + eps)
    T = len(c["g"])
    return dict(p=p, m=m, v=v, b_p=U * acc, b_m=U * T * M, b_v=U * T * v)


# ----- pointwise loss --------------------------------------------------------------------------------------------------------
LOSS_N = (1 << 20) + 1001            # > 1024 blocks x 256 threads: the grid-stride loop runs 5 rounds
LOSS_THREADS = 1024 * 256
FOCAL_ALPHA, FOCAL_GAMMA = F32(0.25), F32(2.0)


def make_loss_case():
    rng = np.random.default_rng(9)
    n = LOSS_N
    x = (rng.standard_normal(n) * 4.0).astype(F32)
    return dict(n=n, x=x, y01=(rng.random(n) < 0.3).astype(F32), yr=rng.standard_normal(n).astype(F32))


def loss_ref(c, kind):
    """(mean loss, d mean loss / d logit, per-element loss magnitude, per-element gradient magnitude), float64."""
    x = _f64(c["x"])
    y = _f64(c["yr"] if kind == 2 else c["y01"])
    n = c["n"]
    if kind == 2:
        d = x - y
        v, g = d * d, 2.0 * d
        vm, gm = v + 2.0 * np.abs(d) * (np.abs(x) + np.abs(y)), 2.0 * (np.abs(x) + np.abs(y))
        return v.sum() / n, g / n, vm, gm
    bce = np.maximum(x, 0.0) - x * y + np.log1p(np.exp(-np.abs(x)))
    p = 1.0 / (1.0 + np.exp(-x))
    bm = np.abs(x) + 1.0
    if kind == 0:
        return bce.sum() / n, (p - y) / n, bce + bm, p + y
    a, gam = float(FOCAL_ALPHA), float(FOCAL_GAMMA)
    wt = y * a + (1.0 - y) * (1.0 - a)
    pt = y * p + (1.0 - y) * (1.0 - p)
    om = 1.0 - pt
    mm = om ** gam
    dpt = (2.0 * y - 1.0) * p * (1.0 - p)
    dm = np.where(om > 0, -gam * om ** (gam - 1.0) * dpt, 0.0)
    g = wt * (dm * bce + mm * (p - y))
    vm = wt * mm * (bce + bm) * (1.0 + np.abs(x))
    gm = wt * (np.abs(dm) * (bce + bm) + mm * (p + y)) * (1.0 + np.abs(x))
    return (wt * mm * bce).sum() / n, g / n, vm, gm


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def _dev(a):
    import torch

    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _padded(a, pad, fill=float("nan")):
    """(buffer, view): a [R, C] float array in a device buffer of width C + pad whose extra columns hold ``fill``."""
    import torch

    a = np.asarray(a, dtype=F32)
    buf = torch.full((a.shape[0], a.shape[1] + pad), fill, dtype=torch.float32, device="cuda")
    v = buf[:, :a.shape[1]]
    v.copy_(torch.as_tensor(a))
    return buf, v


def _nan_buf(R, C, pad):
    import torch

    buf = torch.full((R, C + pad), float("nan"), dtype=torch.float32, device="cuda")
    return buf, buf[:, :C]


def _host(t):
    import torch

    torch.cuda.synchronize()
    return t.cpu().numpy()


def _check(got, ref, bound, what):
    err = np.abs(_f64(got) - ref)
    bad = ~(err <= bound)
    if bad.any():
        i = np.unravel_index(np.argmax(np.where(bad, err / np.maximum(bound, 1e-300), 0.0)), np.shape(err))
        raise AssertionError(f"{what}: {int(bad.sum())} elements over the bound, worst at {i}: err {err[i]:.3e} "
                             f"bound {np.asarray(bound)[i] if np.ndim(bound) else bound:.3e}")


def _ws(nbytes):
    import torch

    return torch.empty(max(int(nbytes), 8), dtype=torch.uint8, device="cuda")


# ----- batch norm ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,K,pad", BN_CASES)
def test_bn_train_forward_matches_fp64(R, K, pad):
    import torch

    from librecommender_b200 import _lib

    c = make_bn_case(R, K, pad)
    ref = bn_forward_ref(c)
    auto = bn_autograd(c)
    _check(ref["y"], auto["y"], 1e-3 * C_BN * ref["b_y"] + 1e-300, "float64 restatement vs autograd")
    xbuf, x = _padded(c["x"], pad)
    gamma, beta = _dev(c["gamma"]), _dev(c["beta"])
    for moving in (True, False):
        ybuf, y = _nan_buf(R, K, pad + 1)
        mean = torch.full((K,), float("nan"), device="cuda")
        var = torch.full((K,), float("nan"), device="cuda")
        mm, mv = (_dev(c["mm"]), _dev(c["mv"])) if moving else (None, None)
        _lib.check(_lib.lib.b200_bn_train_forward(_lib.ptr(x), x.stride(0), R, K, _lib.ptr(gamma), _lib.ptr(beta),
                                                  EPS_BN, MOMENTUM, _lib.ptr(y), y.stride(0), _lib.ptr(mean),
                                                  _lib.ptr(var), _lib.ptr(mm), _lib.ptr(mv), _lib.current_stream()))
        yb = _host(ybuf)
        assert np.isnan(yb[:, K:]).all(), "wrote past K"
        _check(yb[:, :K], ref["y"], C_BN * ref["b_y"], f"y (moving {moving})")
        _check(_host(mean), ref["mean"], C_BN * ref["b_mean"], "batch mean")
        _check(_host(var), ref["var"], C_BN * ref["b_var"], "batch variance")
        if moving:
            _check(_host(mm), ref["mm"], C_BN * ref["b_mm"], "moving mean")
            _check(_host(mv), ref["mv"], C_BN * ref["b_mv"], "moving variance")
        if K >= 3:
            assert (yb[:, 1] == c["beta"][1]).all(), "a constant column normalises to exactly beta"


@pytest.mark.parametrize("R,K,pad", BN_CASES)
def test_bn_train_backward_matches_autograd(R, K, pad):
    from librecommender_b200 import _lib

    c = make_bn_case(R, K, pad)
    ref = bn_backward_ref(c)
    auto = bn_autograd(c)
    _check(ref["dx"], auto["dx"], 1e-3 * C_BN * ref["b_dx"] + 1e-300, "float64 restatement vs autograd: dx")
    _check(ref["g_gamma"] - c["g0_gamma"], auto["dgamma"], 1e-3 * C_BN * ref["b_gamma"], "restatement: d gamma")
    _check(ref["g_beta"] - c["g0_beta"], auto["dbeta"], 1e-3 * C_BN * ref["b_beta"], "restatement: d beta")
    mu, var, _ = bn_stats(c["x"])
    mean, varf = _dev(mu.astype(F32)), _dev(var.astype(F32))
    _, x = _padded(c["x"], pad)
    _, dy = _padded(c["dy"], pad + 2)
    gamma = _dev(c["gamma"])
    ws = _ws(16 * K)
    pos = c["x"] > 0
    for relu in (0, 1):
        dxbuf, dx = _nan_buf(R, K, pad + 1)
        gg, gb = _dev(c["g0_gamma"]), _dev(c["g0_beta"])
        _lib.check(_lib.lib.b200_bn_train_backward(_lib.ptr(dy), dy.stride(0), _lib.ptr(x), x.stride(0), R, K,
                                                   _lib.ptr(mean), _lib.ptr(varf), _lib.ptr(gamma), EPS_BN, relu,
                                                   _lib.ptr(dx), dx.stride(0), _lib.ptr(gg), _lib.ptr(gb), _lib.ptr(ws),
                                                   ws.numel(), _lib.current_stream()))
        got = _host(dxbuf)
        assert np.isnan(got[:, K:]).all(), "wrote past K"
        got = got[:, :K]
        if relu:
            assert (got[~pos] == 0).all() and not np.signbit(got[~pos]).any(), "ReLU mask: inputs <= 0 give +0"
            _check(got[pos], ref["dx"][pos], C_BN * ref["b_dx"][pos], "dx (ReLU mask)")
        else:
            _check(got, ref["dx"], C_BN * ref["b_dx"], "dx")
        _check(_host(gg), ref["g_gamma"], C_BN * ref["b_gamma"], f"g_gamma (relu {relu})")
        _check(_host(gb), ref["g_beta"], C_BN * ref["b_beta"], f"g_beta (relu {relu})")
        if R == 1:
            assert (got[~pos if relu else np.ones_like(pos)] == 0).all(), "one row: dx is exactly 0"


def test_relu_backward_exact():
    from librecommender_b200 import _lib

    rng = np.random.default_rng(2)
    n = 5003
    a = rng.standard_normal(n).astype(F32)
    a[::7] = 0.0
    a[3::7] = -0.0
    a[5::11] = np.float32(1e-45)                               # the smallest subnormal is > 0
    dy = rng.standard_normal(n).astype(F32)
    ad, dyd = _dev(a), _dev(dy)
    dx = _dev(np.full(n, np.nan, dtype=F32))
    _lib.check(_lib.lib.b200_relu_backward(_lib.ptr(dyd), _lib.ptr(ad), n, _lib.ptr(dx), _lib.current_stream()))
    np.testing.assert_array_equal(_host(dx), np.where(a > 0, dy, F32(0)))


# ----- FM head -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,K,has_b,has_lb", FM_FWD_CASES)
def test_fm_head_forward_matches_fp64(R, K, has_b, has_lb):
    import torch

    from librecommender_b200 import _lib

    c = make_fm_fwd_case(R, K, has_b, has_lb)
    ref = fm_forward_ref(c)
    _, y = _padded(c["y"], 3)
    w, lin = _dev(c["w"]), _dev(c["lin"])
    b = _dev(np.array([c["b"]], dtype=F32)) if has_b else None
    lb = _dev(np.array([c["lb"]], dtype=F32)) if has_lb else None
    z = torch.full((R + 1,), float("nan"), device="cuda")
    logit = torch.full((R + 1,), float("nan"), device="cuda")
    _lib.check(_lib.lib.b200_fm_head_forward(_lib.ptr(y), y.stride(0), R, K, _lib.ptr(w), _lib.ptr(b), _lib.ptr(lin),
                                             _lib.ptr(lb), _lib.ptr(z), _lib.ptr(logit), _lib.current_stream()))
    zg, lg = _host(z), _host(logit)
    assert np.isnan(zg[R]) and np.isnan(lg[R])
    _check(zg[:R], ref["z"], C_HEAD * ref["b_z"], "z")
    _check(lg[:R], ref["logit"], C_HEAD * ref["b_logit"], "logit")


@pytest.mark.parametrize("R,K,use_bn,has_glb", FM_BWD_CASES)
def test_fm_head_backward_matches_autograd(R, K, use_bn, has_glb):
    from librecommender_b200 import _lib

    c = make_fm_bwd_case(R, K, use_bn, has_glb)
    ref = fm_backward_ref(c)
    check_fm_restatement(c)
    _, pw = _padded(c["pw"], 2)
    dl, z, w = _dev(c["dlogit"]), _dev(c["z"]), _dev(c["w"])
    bn = {k: _dev(c[k]) for k in ("mean", "var", "gamma", "beta")} if use_bn else {}
    g = {k: _dev(c["g0_" + k]) for k in ("w", "b", "gamma", "beta", "lb")}
    dbuf, dpw = _nan_buf(R, K, 3)
    ws = _ws(_lib.lib.b200_fm_head_backward_workspace_bytes(R, K))
    _lib.check(_lib.lib.b200_fm_head_backward(
        _lib.ptr(dl), _lib.ptr(z), _lib.ptr(pw), pw.stride(0), R, K, _lib.ptr(bn.get("mean")), _lib.ptr(bn.get("var")),
        _lib.ptr(bn.get("gamma")), _lib.ptr(bn.get("beta")), EPS_BN, _lib.ptr(w), _lib.ptr(dpw), dpw.stride(0),
        _lib.ptr(g["w"]), _lib.ptr(g["b"]), _lib.ptr(g["gamma"] if use_bn else None),
        _lib.ptr(g["beta"] if use_bn else None), _lib.ptr(g["lb"] if has_glb else None), _lib.ptr(ws), ws.numel(),
        _lib.current_stream()))
    got = _host(dbuf)
    assert np.isnan(got[:, K:]).all(), "wrote past K"
    _check(got[:, :K], ref["dpw"], C_HEAD * ref["b_dpw"], "d pw")
    _check(_host(g["w"]), ref["g_w"], C_HEAD * ref["b_w"], "g pw_kernel")
    _check(_host(g["b"]), ref["g_b"], C_HEAD * ref["b_b"], "g pw_bias")
    if has_glb:
        _check(_host(g["lb"]), ref["g_lb"], C_HEAD * ref["b_lb"], "g lin_bias")
    else:
        np.testing.assert_array_equal(_host(g["lb"]), c["g0_lb"])
    if use_bn:
        _check(_host(g["gamma"]), ref["g_gamma"], C_HEAD * ref["b_gamma"], "g gamma")
        _check(_host(g["beta"]), ref["g_beta"], C_HEAD * ref["b_beta"], "g beta")


# ----- DeepFM head ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R,K,H,pad,has_b", DEEPFM_CASES)
def test_deepfm_head_forward_and_backward(R, K, H, pad, has_b):
    import torch

    from librecommender_b200 import _lib

    c = make_deepfm_case(R, K, H, pad, has_b)
    ref, bound = deepfm_forward_ref(c)
    st = _lib.current_stream()
    lin, w, dl = _dev(c["lin"]), _dev(c["w"]), _dev(c["dlogit"])
    _, pw = _padded(c["pw"], 1)
    _, deep = _padded(c["deep"], pad)
    lb = _dev(np.array([c["lb"]], dtype=F32)) if has_b else None
    b = _dev(np.array([c["b"]], dtype=F32)) if has_b else None
    logit = torch.full((R + 1,), float("nan"), device="cuda")
    _lib.check(_lib.lib.b200_deepfm_head_forward(_lib.ptr(lin), _lib.ptr(lb), _lib.ptr(pw), pw.stride(0), K,
                                                 _lib.ptr(deep), deep.stride(0), H, _lib.ptr(w), _lib.ptr(b), R,
                                                 _lib.ptr(logit), st))
    got = _host(logit)
    assert np.isnan(got[R])
    _check(got[:R], ref, C_HEAD * bound, "DeepFM logit")
    dlin = torch.full((R + 1,), float("nan"), device="cuda")
    dpbuf, dpw = _nan_buf(R, K, 2)
    ddbuf, ddeep = _nan_buf(R, H, pad + 1)
    _lib.check(_lib.lib.b200_deepfm_head_backward(_lib.ptr(dl), _lib.ptr(w), K, H, R, _lib.ptr(dlin), _lib.ptr(dpw),
                                                  dpw.stride(0), _lib.ptr(ddeep), ddeep.stride(0), st))
    d32 = c["dlogit"][:, None]
    gl, gp, gd = _host(dlin), _host(dpbuf), _host(ddbuf)
    # one float product per element: exact
    np.testing.assert_array_equal(gl[:R], (d32 * c["w"][0])[:, 0])
    np.testing.assert_array_equal(gp[:, :K], d32 * c["w"][1:1 + K])
    np.testing.assert_array_equal(gd[:, :H], d32 * c["w"][1 + K:])
    assert np.isnan(gl[R]) and np.isnan(gp[:, K:]).all() and np.isnan(gd[:, H:]).all()


# ----- field-gradient scatter ---------------------------------------------------------------------------------------------
def _feat_device(c):
    """FeatSpec on the device, the layout of the case, tables, inputs and gradient buffers (initial values), and a
    lin_kernel gradient with four -0.0 guard cells after the layout's fields.  The caller keeps the FeatSpec and the
    tables alive: the layout and tables structs hold raw pointers into them."""
    import torch

    from librecommender_b200.feat_models import FeatSpec, tables_struct

    fs = FeatSpec(c["spec"], c["K"])
    layout, pos = feat_layout(fs, c["which"])
    assert pos == c["pos"]
    t = {k: _dev(v) for k, v in c["w"].items() if k in TABLES}
    grads = {k: _dev(v) for k, v in c["g0"].items() if k != "lin_kernel"}
    Fl = len(pos)
    glk = torch.full((Fl + 4,), -0.0, device="cuda")
    glk[:Fl] = torch.as_tensor(c["g0"]["lin_kernel"]).cuda()
    grads["lin_kernel"] = glk
    ins = dict(users=_dev(c["users"]), items=_dev(c["items"]), lin_kernel=_dev(c["lin_kernel"]),
               dlogit=_dev(c["dlogit"]) if c["dlogit"] is not None else None,
               dpw=_padded(c["dpw"], 1)[1] if c["dpw"] is not None else None,
               S=_padded(c["S"], 2)[1] if c["dpw"] is not None else None,
               dconcat=_padded(c["dconcat"], 3)[1] if c["dconcat"] is not None else None)
    return fs, layout, tables_struct(t), t, ins, grads


@pytest.mark.parametrize("K,which,inputs,with_dlogit,R", FEAT_CASES)
def test_feat_backward_matches_fp64(K, which, inputs, with_dlogit, R):
    from librecommender_b200.feat_models import feat_backward

    c = make_feat_case(K, which, inputs, with_dlogit, R)
    ref, mag, cnt = feat_backward_ref(c)
    bound = feat_bound(mag, cnt)
    fs, layout, tstruct, t, ins, grads = _feat_device(c)
    feat_backward(layout, tstruct, ins["users"], ins["items"], R, grads, dpw=ins["dpw"], S=ins["S"],
                  dconcat=ins["dconcat"], dlogit=ins["dlogit"],
                  lin_kernel=ins["lin_kernel"] if with_dlogit else None)
    Fl = len(c["pos"])
    lk = _host(grads["lin_kernel"])
    assert (lk[Fl:] == 0).all() and np.signbit(lk[Fl:]).all(), "lin_kernel gradient written past the layout's fields"
    for k in ref:
        got = _host(grads[k])[:len(ref[k])]
        untouched = cnt[k] == 0
        # rows no batch row touches keep their bits
        np.testing.assert_array_equal(got[untouched].view(np.uint32), c["g0"][k][untouched].view(np.uint32),
                                      err_msg=f"{k}: untouched rows changed")
        _check(got, ref[k], C_SCATTER * bound[k], f"{k} ({which}, K {K})")
    assert max(cnt[k].max() for k in TABLES) > R // 3, "the case has no hot key"


# ----- row helpers of csrc/feat.cu --------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", ROW_D)
def test_gather_and_scatter_add_rows(d):
    from librecommender_b200 import _lib

    c = make_rows_case(d)
    st = _lib.current_stream()
    n = len(c["idx"])
    _, tab = _padded(c["table"], 3)
    idx = _dev(c["idx"])
    obuf, out = _nan_buf(n, d, 1)
    _lib.check(_lib.lib.b200_gather_rows(_lib.ptr(tab), tab.stride(0), d, _lib.ptr(idx), n, _lib.ptr(out),
                                         out.stride(0), st))
    got = _host(obuf)
    np.testing.assert_array_equal(got[:, :d], c["table"][c["idx"]])         # a copy: bit-exact
    assert np.isnan(got[:, d:]).all()
    gbuf, g = _padded(c["g0"], 2, fill=-0.0)
    _, rows = _padded(c["rows"], 1)
    _lib.check(_lib.lib.b200_scatter_add_rows(_lib.ptr(g), g.stride(0), d, _lib.ptr(idx), n, _lib.ptr(rows),
                                              rows.stride(0), st))
    ref, bound, cnt = scatter_ref(c)
    gg = _host(gbuf)
    assert (gg[:, d:] == 0).all() and np.signbit(gg[:, d:]).all(), "scatter wrote past d"
    np.testing.assert_array_equal(gg[cnt == 0, :d].view(np.uint32), c["g0"][cnt == 0].view(np.uint32))
    _check(gg[:, :d], ref, C_SCATTER * bound, "scatter_add_rows")


@pytest.mark.parametrize("na,nb,nc", CONCAT_CASES)
def test_concat_dense_matches_fp64(na, nb, nc):
    import torch

    from librecommender_b200 import _lib

    c = make_concat_case(na, nb, nc)
    ref, bound = concat_ref(c)
    R = c["R"]
    views = [(_padded(b, 2 + i)[1] if b.shape[1] else None) for i, b in enumerate(c["blocks"])]
    w = _dev(c["w"])
    out = torch.full((R + 1,), float("nan"), device="cuda")

    def ld(v):
        return v.stride(0) if v is not None else 0

    _lib.check(_lib.lib.b200_concat_dense(_lib.ptr(views[0]), ld(views[0]), na, _lib.ptr(views[1]), ld(views[1]), nb,
                                          _lib.ptr(views[2]), ld(views[2]), nc, _lib.ptr(w), float(c["bias"]), R,
                                          _lib.ptr(out), _lib.current_stream()))
    got = _host(out)
    assert np.isnan(got[R])
    _check(got[:R], ref, C_HEAD * bound, "concat Dense(1)")


@pytest.mark.parametrize("d", L2_D)
def test_l2_normalize_forward_backward(d):
    from librecommender_b200 import _lib

    c = make_l2_case(d)
    ref = l2_ref(c)
    y_auto, dx_auto = l2_autograd(c)
    _check(ref["y"], y_auto, 1e-3 * C_L2 * ref["b_y"] + 1e-300, "restatement vs autograd: y")
    _check(ref["dx"], dx_auto, 1e-3 * C_L2 * ref["b_dx"] + 1e-300, "restatement vs autograd: dx")
    for r in c["tie"]:
        assert ref["ss"][r] == EPS_L2 and not ref["clamped"][r]
    assert ref["clamped"][:4].all() and not ref["clamped"][4:8].any()
    R, st = c["R"], _lib.current_stream()
    xbuf, x = _padded(c["x"], 3)
    _, dy = _padded(c["dy"], 1)
    dbuf, dx = _nan_buf(R, d, 2)
    _lib.check(_lib.lib.b200_l2_normalize_backward(_lib.ptr(x), x.stride(0), _lib.ptr(dy), dy.stride(0), R, d,
                                                   _lib.ptr(dx), dx.stride(0), st))
    got = _host(dbuf)
    assert np.isnan(got[:, d:]).all()
    _check(got[:, :d], ref["dx"], C_L2 * ref["b_dx"], f"L2 backward d {d}")
    _lib.check(_lib.lib.b200_l2_normalize_rows(_lib.ptr(x), x.stride(0), R, d, st))     # in place
    got = _host(xbuf)
    assert np.isnan(got[:, d:]).all()
    _check(got[:, :d], ref["y"], C_L2 * ref["b_y"], f"L2 forward d {d}")
    assert (got[12, :d] == 0).all()


# ----- Adam ----------------------------------------------------------------------------------------------------------------
def _ulps(a, b):
    """|a - b| in units of the float spacing at the larger magnitude."""
    a, b = np.asarray(a, dtype=F32), np.asarray(b, dtype=F32)
    return np.abs(_f64(a) - _f64(b)) / _f64(np.spacing(np.maximum(np.abs(a), np.abs(b))))


def test_adam_dense_host_and_device_steps_match_fp64():
    import torch

    from librecommender_b200 import _lib

    c = make_adam_case()
    ref = adam_ref(c)
    st = _lib.current_stream()
    n = ADAM_N
    state = {}
    for path in ("host", "device"):
        p = _dev(c["p0"])
        m, v = torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
        step = torch.zeros(1, dtype=torch.int64, device="cuda")
        lr_t = torch.full((1,), float("nan"), device="cuda")
        for t in range(1, ADAM_STEPS + 1):
            g = _dev(c["g"][t - 1])
            if path == "host":
                _lib.check(_lib.lib.b200_adam_dense(_lib.ptr(p), _lib.ptr(m), _lib.ptr(v), _lib.ptr(g), n,
                                                    float(ADAM_LR), float(ADAM_B1), float(ADAM_B2), float(ADAM_EPS),
                                                    t, st))
            else:
                _lib.check(_lib.lib.b200_adam_begin_step(_lib.ptr(step), float(ADAM_LR), float(ADAM_B1),
                                                         float(ADAM_B2), 1.0, 0, _lib.ptr(lr_t), st))
                _lib.check(_lib.lib.b200_adam_dense_dev(_lib.ptr(p), _lib.ptr(m), _lib.ptr(v), _lib.ptr(g), n,
                                                        _lib.ptr(lr_t), float(ADAM_B1), float(ADAM_B2),
                                                        float(ADAM_EPS), st))
                assert int(_host(step)[0]) == t
                assert _ulps(_host(lr_t)[0], adam_lr_t(t)) <= 1.0, (t, float(_host(lr_t)[0]), adam_lr_t(t))
            gh = _host(g)
            assert (gh == 0).all() and not np.signbit(gh).any(), "the gradient is zeroed after the step"
        state[path] = {k: _host(a) for k, a in (("p", p), ("m", m), ("v", v))}
        got = state[path]
        _check(got["p"], ref["p"], C_ADAM * ref["b_p"], f"Adam weights ({path})")
        _check(got["m"], ref["m"], C_ADAM * ref["b_m"], f"Adam m ({path})")
        _check(got["v"], ref["v"], C_ADAM * ref["b_v"], f"Adam v ({path})")
        np.testing.assert_array_equal(got["p"][:50], c["p0"][:50])             # never a gradient: never a move
    # the two paths differ only in where lr_t is computed (double on the host / on the device)
    np.testing.assert_array_equal(state["host"]["m"], state["device"]["m"])
    np.testing.assert_array_equal(state["host"]["v"], state["device"]["v"])
    assert _ulps(state["host"]["p"], state["device"]["p"]).max() <= 1.0


def test_adam_step_counter_and_staircase_decay():
    import torch

    from librecommender_b200 import _lib

    st = _lib.current_stream()
    step = torch.full((1,), 5, dtype=torch.int64, device="cuda")          # resumes from a completed step 5
    lr_t = torch.full((1,), float("nan"), device="cuda")
    rate, every = F32(0.5), 3
    for t in range(6, 16):                                                   # crosses the boundaries at t = 7, 10, 13
        _lib.check(_lib.lib.b200_adam_begin_step(_lib.ptr(step), float(ADAM_LR), float(ADAM_B1), float(ADAM_B2),
                                                 float(rate), every, _lib.ptr(lr_t), st))
        assert int(_host(step)[0]) == t
        want = adam_lr_t(t, decay_rate=rate, decay_steps=every)
        assert _ulps(_host(lr_t)[0], want) <= 1.0, (t, float(_host(lr_t)[0]), want)


def test_axpy_is_one_fma():
    from librecommender_b200 import _lib

    rng = np.random.default_rng(8)
    n = 70001
    x = rng.standard_normal(n).astype(F32)
    y = (rng.standard_normal(n) * 10.0 ** rng.uniform(-6, 2, n)).astype(F32)
    alpha = F32(2.0 * 1e-3)
    yd, xd = _dev(y), _dev(x)
    _lib.check(_lib.lib.b200_axpy(_lib.ptr(yd), _lib.ptr(xd), float(alpha), n, _lib.current_stream()))
    exact = float(alpha) * _f64(x) + _f64(y)                  # the product is exact in float64; one rounding to float
    got = _host(yd)
    assert (np.abs(_f64(got) - exact) <= U * np.abs(exact)).all()


# ----- pointwise loss past the grid cap --------------------------------------------------------------------------------------
def test_pointwise_loss_grid_stride_past_max_blocks():
    import torch

    from librecommender_b200 import _lib

    c = make_loss_case()
    n = c["n"]
    assert n > LOSS_THREADS
    x = _dev(c["x"])
    ws = _ws(_lib.lib.b200_loss_workspace_bytes())
    chain = -(-n // LOSS_THREADS)
    for kind in (0, 1, 2):
        y = _dev(c["yr"] if kind == 2 else c["y01"])
        loss = torch.full((1,), float("nan"), device="cuda")
        dl = torch.full((n + 1,), float("nan"), device="cuda")
        _lib.check(_lib.lib.b200_pointwise_loss(_lib.ptr(x), _lib.ptr(y), n, kind, float(FOCAL_ALPHA),
                                                float(FOCAL_GAMMA), _lib.ptr(loss), _lib.ptr(dl), _lib.ptr(ws),
                                                ws.numel(), _lib.current_stream()))
        L, g, vm, gm = loss_ref(c, kind)
        got = _host(dl)
        assert np.isnan(got[n]), "wrote past n"
        _check(got[:n], g, C_LOSS * U * gm / n, f"d loss / d logit, kind {kind}")
        _check(_host(loss)[0], L, C_LOSS * U * (chain + 2) * vm.sum() / n, f"loss, kind {kind}")


# ----- host-side fixes: empty batches, missing gradient buffers -------------------------------------------------------------
def test_empty_batch_backward_is_a_no_op():
    import torch

    from librecommender_b200 import _lib

    lib, st, P = _lib.lib, _lib.current_stream(), _lib.ptr
    K = 8
    rng = np.random.default_rng(4)
    bufs = {k: _dev(rng.standard_normal(n).astype(F32)) for k, n in
            (("a", 4 * K), ("b", 4 * K), ("mean", K), ("var", K), ("gamma", K), ("beta", K), ("w", K), ("gw", K),
             ("gb", 1), ("gg", K), ("gbe", K), ("glb", 1), ("out", 4 * K))}
    before = {k: _host(v).copy() for k, v in bufs.items()}
    ws = _ws(1 << 12)
    n0 = _lib.launch_count()
    B = bufs
    assert lib.b200_fm_head_backward(P(B["a"]), P(B["a"]), P(B["b"]), K, 0, K, P(B["mean"]), P(B["var"]),
                                     P(B["gamma"]), P(B["beta"]), EPS_BN, P(B["w"]), P(B["out"]), K, P(B["gw"]),
                                     P(B["gb"]), P(B["gg"]), P(B["gbe"]), P(B["glb"]), P(ws), ws.numel(), st) == 0
    assert lib.b200_bn_train_backward(P(B["a"]), K, P(B["b"]), K, 0, K, P(B["mean"]), P(B["var"]), P(B["gamma"]),
                                      EPS_BN, 1, P(B["out"]), K, P(B["gg"]), P(B["gbe"]), P(ws), ws.numel(), st) == 0
    # batch statistics of no rows are undefined: the forward keeps rejecting R = 0
    assert lib.b200_bn_train_forward(P(B["a"]), K, 0, K, P(B["gamma"]), P(B["beta"]), EPS_BN, MOMENTUM, P(B["out"]),
                                     K, P(B["mean"]), P(B["var"]), None, None, st) == -2
    torch.cuda.synchronize()
    assert _lib.launch_count() == n0, "an empty batch launched a kernel"
    for k, v in bufs.items():
        np.testing.assert_array_equal(_host(v), before[k], err_msg=k)


@pytest.mark.parametrize("missing,with_dlogit", [("user_embeds", False), ("item_embeds", False),
                                                 ("sparse_embeds", False), ("dense_embeds", False),
                                                 ("user_linear", True), ("item_linear", True),
                                                 ("sparse_linear", True), ("dense_linear", True)])
def test_feat_backward_rejects_a_missing_gradient_buffer(missing, with_dlogit):
    from librecommender_b200 import _lib
    from librecommender_b200.feat_models import feat_backward

    c = make_feat_case(4, "full", "both", with_dlogit, 64)
    fs, layout, tstruct, t, ins, grads = _feat_device(c)
    grads = {k: v for k, v in grads.items() if k != missing}
    before = {k: _host(v).copy() for k, v in grads.items()}
    n0 = _lib.launch_count()
    with pytest.raises(_lib.B200Error, match=f"g_{missing} is null"):
        feat_backward(layout, tstruct, ins["users"], ins["items"], c["R"], grads, dpw=ins["dpw"], S=ins["S"],
                      dconcat=ins["dconcat"], dlogit=ins["dlogit"],
                      lin_kernel=ins["lin_kernel"] if with_dlogit else None)
    assert _lib.launch_count() == n0
    for k, v in grads.items():
        np.testing.assert_array_equal(_host(v), before[k], err_msg=k)


def test_feat_backward_side_layouts_need_only_their_buffers():
    """A side layout scatters into its own tables only: the other side's buffers may be absent."""
    from librecommender_b200.feat_models import feat_backward

    c = make_feat_case(8, "user_noid", "dconcat", False, 100)
    ref, _, cnt = feat_backward_ref(c)
    fs, layout, tstruct, t, ins, grads = _feat_device(c)
    need = {k for k in ref if cnt[k].any()}
    assert "user_embeds" not in need and "item_embeds" not in need
    grads = {k: v for k, v in grads.items() if k in need}
    feat_backward(layout, tstruct, ins["users"], ins["items"], c["R"], grads, dconcat=ins["dconcat"])
    for k in need:
        assert np.isfinite(_host(grads[k])).all()
