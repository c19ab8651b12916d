"""Float64 restatements of the loss kernels of ``csrc/loss.cu``, with the per-element magnitudes their error bounds use
(TEST INFRASTRUCTURE ONLY; shared by tests/test_gpu_loss_kernels.py and tests/test_loss_kernel_bounds_cpu.py).

* ``pairwise_ref``: ``b200_pairwise_loss``.  Kinds 0 (BPR, -log sigmoid(pos - neg)) and 1 (max-margin,
  relu(margin - (pos - neg))) broadcast positive j over its ``factor = n_neg / n_pos`` negatives
  ``neg[j f .. (j + 1) f)``; d loss / d pos[j] is the sum over those negatives.  Max-margin follows torch's
  ``clamp_min``: a pair exactly on the hinge has gradient -1 / n_neg w.r.t. pos.  Kinds 2 / 3 are sigmoid CE / focal
  over ``[pos (label 1) | neg (label 0)]``, mean or sum.
* ``pointwise_elems``: sigmoid CE and focal per element (the pointwise kernel and kinds 2 / 3 above) at any gamma.
  Focal keeps the kernel's guard as its definition: d (1 - p_t)^gamma / dx is 0 where 1 - p_t == 0.  torch's
  ``focal_loss`` differs there on purpose: for 0 < gamma < 1 its autograd multiplies 0^(gamma - 1) = inf into the
  chain at a saturated logit (1 - p_t rounds to 0) and returns NaN or inf; the kernel returns a finite 0.
* ``inbatch_ref``: ``b200_softmax_inbatch_loss``, TwoTower's ``adjust_logits`` (algorithms/two_tower.py:458-479):
  ``divide_no_nan(S, temperature)``, minus ``log(clip(correction, 1e-8, 1))``, off-diagonal columns with the row's own
  item id replaced by ``tf.float32.min``; loss = mean_r (logsumexp(row r) - logit[r, r]), gradient w.r.t. S.  Masked
  entries have gradient exactly 0; with temperature 0 every gradient is exactly 0.
* ``sampled_ref``: ``b200_sampled_class_loss``, TensorFlow's ``_compute_sampled_logits`` with
  ``remove_accidental_hits`` and ``subtract_log_q``, then ``sampled_softmax_loss`` (kind 0) or ``nce_loss``
  (kind 1).  The expected counts are TensorFlow's float ``ExpectedCountHelper`` (``expected_counts`` of
  tests/_youtube_retrieval_train_oracle.py with ``dtype=np.float32``: that rounding is part of the operation);
  everything after it is float64.  Accidental hits have gradient exactly 0.

Error bounds (u = 2^-24) are stated per element in quantities computed here:
  gradient   C u gmag / n                              (n the kernel's divisor: n_neg, n or 1, B)
  loss       C u (per-thread chain + 2) sum vmag / n  (chain = the float sums one thread or one lane 0 makes)
A gradient that is not exactly 0 by construction also gets C ETA (C ETA (1 + 1 / temperature) in-batch), ETA = 2^-149:
saturated logits give subnormal probabilities, whose rounding is absolute, not relative.
BPR's ``log1pf(__expf(-|d|))`` carries ``__expf``'s documented maximum error, 2 + floor(|1.173 x|) ulp, in its own
magnitude.  The softmax rows carry a term for the per-lane online max / sum and its shuffle merge:
ceil(n_cols / 32) + 5 rounding steps of the row's log-sum-exp.
"""
from __future__ import annotations

import numpy as np
from scipy.special import expit

U = 2.0 ** -24
F32, F64 = np.float32, np.float64
FLT_MAX = float(np.finfo(np.float32).max)
ETA = 2.0 ** -149                                 # smallest float subnormal: the absolute error floor of a gradient
THREADS, MAX_BLOCKS = 256, 1024                   # csrc/loss.cu launch shape
WARPS_PER_BLOCK = THREADS // 32
CORR_MIN = float(F32(1e-8))                       # the clip bound as the float the kernel compares with
ALPHA = 0.25                                      # focal alpha of the reference's pairwise / default focal

# bound constants (see the module docstring); calibrated by tests/test_loss_kernel_bounds_cpu.py
C_PAIR = 24.0         # pairwise kinds 0 - 3 and the pointwise focal sweep
C_INBATCH = 16.0      # in-batch softmax
C_SAMPLED = 8.0       # sampled softmax / NCE


def _f64(a):
    return np.asarray(a, dtype=F64)


def grid_rounds(n):
    """Grid-stride rounds one thread makes over n elements (grid_for: <= 1024 blocks of 256 threads)."""
    blocks = min(max(-(-n // THREADS), 1), MAX_BLOCKS)
    return -(-n // (blocks * THREADS))


def warp_rounds(B):
    """Rows one warp takes in the one-warp-per-row kernels (<= 1024 blocks of 8 warps)."""
    blocks = min(-(-B // WARPS_PER_BLOCK), MAX_BLOCKS)
    return -(-B // (blocks * WARPS_PER_BLOCK))


def expf_fast_ulp(x):
    """Documented maximum error of __expf(x) in ulp (CUDA C++ Programming Guide, intrinsic functions)."""
    return 2.0 + np.floor(np.abs(1.173 * _f64(x)))


# ---------------------------------------------------------------------------------------------------------------------
# pointwise elements: sigmoid CE (kind 0) and focal (kind 1) at any gamma
# ---------------------------------------------------------------------------------------------------------------------
def pointwise_elems(x, y, kind, alpha=ALPHA, gamma=2.0):
    """(value, d value / dx, value magnitude, gradient magnitude) per element, float64."""
    x, y = _f64(x), _f64(y)
    bce = np.maximum(x, 0.0) - x * y + np.log1p(np.exp(-np.abs(x)))
    p = expit(x)
    bm = np.abs(x) + 1.0
    if kind == 0:
        return bce, p - y, bce + bm, p + y
    a, gam = float(F32(alpha)), float(F32(gamma))
    wt = y * a + (1.0 - y) * (1.0 - a)
    pt = y * p + (1.0 - y) * (1.0 - p)
    om = 1.0 - pt
    mm = om ** gam
    dpt = (2.0 * y - 1.0) * p * (1.0 - p)
    with np.errstate(divide="ignore", invalid="ignore"):
        dm = np.where(om > 0, -gam * np.power(np.where(om > 0, om, 1.0), gam - 1.0) * dpt, 0.0)
    g = wt * (dm * bce + mm * (p - y))
    vm = wt * mm * (bce + bm) * (1.0 + np.abs(x))
    gm = wt * (np.abs(dm) * (bce + bm) + mm * (p + y)) * (1.0 + np.abs(x))
    return wt * mm * bce, g, vm, gm


# ---------------------------------------------------------------------------------------------------------------------
# pairwise
# ---------------------------------------------------------------------------------------------------------------------
PAIR_SHAPES = [(1, 1), (1, 17), (31, 3), (257, 1), (257, 17), (300_000, 1), (300_000, 3), (300_000, 17)]
MARGINS = (0.0, 1.0, 0.5)


def make_pair_case(n_pos, factor, kind, margin=0.0, seed=0):
    """pos [n_pos], neg [n_pos * factor], float32.  Scores are multiples of 1/64 below 2^10, so every difference and
    every margin - difference is exact in float: a fifth of the pairs sit exactly on the hinge (pos - neg == margin),
    a fifth are saturated (|pos - neg| up to 100).  BPR and the class losses also get a fifth of unquantised scores."""
    rng = np.random.default_rng(1000 * n_pos + 10 * factor + kind + seed)
    q = lambda a: np.round(a * 64.0) / 64.0                                             # noqa: E731
    pos = q(rng.normal(0.0, 3.0, n_pos))
    n = n_pos * factor
    d = q(rng.normal(0.0, 3.0, n))
    which = rng.integers(0, 5, n)
    d[which == 0] = margin
    d[which == 1] = q(rng.uniform(-100.0, 100.0, int((which == 1).sum())))
    if kind != 1:
        d[which == 2] = rng.normal(0.0, 3.0, int((which == 2).sum()))
    neg = np.repeat(pos, factor) - d
    if kind >= 2:                                      # class losses see raw logits: saturate some of them too
        neg[which == 1] = q(rng.uniform(-90.0, 90.0, int((which == 1).sum())))
    return pos.astype(F32), neg.astype(F32)


def pairwise_ref(pos, neg, kind, margin=0.0, mean=True, gamma=2.0):
    """dict(loss, dpos, dneg, b_loss, b_dpos, b_dneg): float64 values and the unscaled bounds (u * magnitude / n;
    multiply by C_PAIR)."""
    p, q = _f64(pos), _f64(neg)
    n_pos, n_neg = len(p), len(q)
    if kind <= 1:
        f = n_neg // n_pos
        P = np.repeat(p, f)
        d = P - q
        if kind == 0:
            v = np.maximum(-d, 0.0) + np.log1p(np.exp(-np.abs(d)))
            s = expit(-d)
            gp = -s
            vm = v + np.abs(d) + expf_fast_ulp(np.abs(d)) * np.log1p(np.exp(-np.abs(d)))
            gm = s * (3.0 + np.abs(d))
        else:
            t = float(F32(margin)) - d
            t32 = F32(margin) - (pos.astype(F32)[np.arange(n_neg) // f] - neg.astype(F32))
            assert ((t32 >= 0) == (t >= 0)).all(), "a max-margin pair within rounding of the hinge"
            v = np.maximum(t, 0.0)
            gp = np.where(t >= 0, -1.0, 0.0)
            vm = np.abs(t) + np.abs(d)
            gm = np.abs(gp)
        gpos = gp.reshape(n_pos, f)
        eta = ETA if kind == 0 else 0.0                 # max-margin gradients are exact multiples of 1 / n_neg
        chain = f * grid_rounds(n_pos)
        return dict(loss=v.sum() / n_neg, dpos=gpos.sum(1) / n_neg, dneg=-gp / n_neg,
                    b_loss=U * (chain + 2) * vm.sum() / n_neg,
                    b_dpos=U * (gm.reshape(n_pos, f).sum(1) + f * np.abs(gpos).sum(1)) / n_neg + eta,
                    b_dneg=U * gm / n_neg + eta, v=v)
    x = np.concatenate([p, q])
    y = np.concatenate([np.ones(n_pos), np.zeros(n_neg)])
    v, g, vm, gm = pointwise_elems(x, y, 0 if kind == 2 else 1, ALPHA, gamma)
    n = n_pos + n_neg
    sc = 1.0 / n if mean else 1.0
    bg = U * gm * sc + ETA
    return dict(loss=v.sum() * sc, dpos=g[:n_pos] * sc, dneg=g[n_pos:] * sc,
                b_loss=U * (grid_rounds(n) + 2) * vm.sum() * sc, b_dpos=bg[:n_pos], b_dneg=bg[n_pos:], v=v)


# ---------------------------------------------------------------------------------------------------------------------
# pointwise focal at several gamma, saturated logits
# ---------------------------------------------------------------------------------------------------------------------
FOCAL_GAMMAS = (0.0, 0.5, 1.0, 2.0, 5.0)


def make_focal_case(n=4099, seed=3):
    """Logits up to |x| = 90 (where float and double sigmoids saturate to 0 or 1) and labels in {0, 1}."""
    rng = np.random.default_rng(seed)
    x = rng.normal(0.0, 4.0, n)
    x[::7] = rng.uniform(-90.0, 90.0, len(x[::7]))
    x[:8] = [90.0, -90.0, 40.0, -40.0, 17.0, -17.0, 0.0, 88.5]
    y = (rng.random(n) < 0.5).astype(F64)
    y[:8] = [1, 0, 1, 0, 1, 0, 1, 1]
    return x.astype(F32), y.astype(F32)


# ---------------------------------------------------------------------------------------------------------------------
# in-batch softmax
# ---------------------------------------------------------------------------------------------------------------------
# (B, lds - B, temperature, correction, item ids)
INBATCH_CASES = [(1, 0, 1.0, None, None), (1, 5, 0.05, "edges", "all_equal"), (2, 5, 0.05, "edges", "dups"),
                 (2, 0, 0.0, None, "all_equal"), (31, 0, 0.0, "edges", "dups"), (31, 5, 1.0, "edges", None),
                 (33, 5, 0.05, None, "few"), (33, 0, 1.0, "edges", "all_equal"), (257, 5, 1.0, "edges", "dups"),
                 (257, 0, 0.05, "edges", "few"), (257, 5, 0.0, "edges", "few"), (8193, 0, 0.05, "edges", "few"),
                 (8193, 5, 1.0, None, "dups"), (12000, 5, 0.05, "edges", "few")]
CORR_EDGES = (0.0, 1e-9, 1.0, 2.0)


def make_inbatch_case(B, pad, temperature, corr, ids, seed=0):
    rng = np.random.default_rng(B * 31 + pad + seed)
    S = rng.normal(0.0, 0.3, (B, B)).astype(F32)
    S[rng.random((B, B)) < 0.01] *= 10.0                                # a few large logits
    c = None
    if corr == "edges":
        c = rng.uniform(1e-4, 0.5, B)
        for k, e in enumerate(CORR_EDGES):
            c[k::len(CORR_EDGES) * 3] = e
        c = c.astype(F32)
    i = None
    if ids == "dups":
        i = rng.integers(0, max(B // 2, 1), B)
    elif ids == "few":
        i = np.arange(B, dtype=np.int64) * 7
        k = rng.choice(B, size=min(B, 6), replace=False)
        i[k] = i[k[0]]                                                  # a handful of rows share one item
    elif ids == "all_equal":
        i = np.full(B, 5, dtype=np.int64)                               # each row keeps only its diagonal
    return dict(B=B, pad=pad, temperature=float(F32(temperature)), S=S, corr=c,
                ids=None if i is None else i.astype(np.int64))


def inbatch_ref(c, r0=0, r1=None):
    """Rows r0:r1 of the in-batch softmax: dict(loss_rows, grad, b_loss_rows, b_grad, masked) with unscaled bounds
    (multiply by C_INBATCH).  loss = sum(loss_rows) / B, its bound sum(b_loss_rows) / B."""
    B = c["B"]
    r1 = B if r1 is None else r1
    S = _f64(c["S"][r0:r1])
    tau = c["temperature"]
    inv = 1.0 / tau if tau != 0.0 else 0.0
    lg = S * inv
    mag = np.abs(lg) * 2.0                                      # S * float(1 / tau): two roundings
    if c["corr"] is not None:
        lq = np.log(np.clip(_f64(c["corr"]), CORR_MIN, 1.0))
        lg = lg - lq[None, :]
        mag = mag + 2.0 * np.abs(lq)[None, :] + np.abs(lg)
    rows = np.arange(r0, r1)
    eye = np.zeros_like(lg, dtype=bool)
    eye[np.arange(r1 - r0), rows] = True
    masked = np.zeros_like(eye)
    if c["ids"] is not None:
        masked = (c["ids"][rows][:, None] == c["ids"][None, :]) & ~eye
        lg[masked] = -FLT_MAX
        mag[masked] = 0.0
    m = lg.max(1, keepdims=True)
    e = np.exp(lg - m)
    se = e.sum(1, keepdims=True)
    lse = m + np.log(se)
    p = e / se
    diag = lg[eye]
    loss_rows = lse[:, 0] - diag
    lse_mag = -(-B // 32) + 5 + np.abs(m[:, 0]) + np.abs(lse[:, 0]) + (p * mag).sum(1)
    chain = warp_rounds(B)
    grad = (p - eye) * inv / B
    grad[masked] = 0.0
    gm = (p * (mag + lse_mag[:, None] + 1.0) + np.abs(p - eye)) * abs(inv)
    b_grad = np.where(masked, 0.0, U * gm / B + (ETA * (1.0 + abs(inv)) if inv != 0.0 else 0.0))
    return dict(loss_rows=loss_rows, grad=grad, masked=masked,
                b_loss_rows=U * (chain + 2) * (lse_mag + mag[eye] + np.abs(loss_rows)), b_grad=b_grad)


# ---------------------------------------------------------------------------------------------------------------------
# sampled softmax / NCE
# ---------------------------------------------------------------------------------------------------------------------
# (B, S, ld - S, sampler kind, n_items, num_tries - S, every sampled id equal to row 0's label)
SAMPLED_CASES = [(1, 1, 0, 0, 1, 0, False), (1, 1, 3, 1, 10 ** 6, 5, False), (37, 31, 0, 1, 31, 0, False),
                 (37, 31, 3, 0, 2 ** 31 - 1, 40, False), (37, 31, 0, 1, 2 ** 31 - 1, 0, True),
                 (256, 33, 3, 0, 10 ** 6, 0, False), (256, 33, 0, 1, 10 ** 6, 100, False),
                 (9000, 1000, 3, 1, 10 ** 6, 3000, False), (9000, 1000, 0, 0, 10 ** 6, 0, False),
                 (64, 65536, 0, 1, 2 ** 31 - 1, 200_000, False), (64, 65536, 3, 0, 65536, 0, False)]
ID_CAP = 1 << 20                     # ids stay below this, so the bias table stays small at n_items near 2^31


def _distinct_ids(rng, kind, n_items, S):
    hi = min(n_items, ID_CAP)
    if hi == S:
        return rng.permutation(S).astype(np.int64)
    out = np.empty(0, dtype=np.int64)
    while len(out) < S:
        if kind == 0:
            draw = rng.integers(0, hi, 4 * S)
        else:
            draw = (np.exp(rng.random(4 * S) * np.log1p(float(n_items))).astype(np.int64) - 1)
            draw = draw[draw < hi]
        out = np.concatenate([out, draw])
        _, first = np.unique(out, return_index=True)
        out = out[np.sort(first)]
    return out[:S]


def make_sampled_case(B, S, pad, kind, n_items, extra, allhit, seed=0):
    """Sampled ids (one id repeated a few times when S > 3, so one row has several accidental hits), labels hit by
    zero, one or several sampled ids, logits with a few large entries."""
    rng = np.random.default_rng(B * 7 + S + pad + kind + seed)
    sampled = _distinct_ids(rng, kind, n_items, S)
    if S > 3:
        sampled[rng.choice(np.arange(1, S), size=min(3, S - 1), replace=False)] = sampled[0]
    if allhit:
        sampled[:] = sampled[0]
    labels = _distinct_ids(rng, kind, n_items, min(B, min(n_items, ID_CAP)))
    labels = np.resize(labels, B)
    labels[0] = sampled[0]                                          # several hits (every id a hit with ``allhit``)
    if B > 1:
        labels[1] = sampled[-1]                                     # one hit
    L = rng.normal(0.0, 2.0, (B, S))
    L[rng.random((B, S)) < 0.01] *= 15.0
    nb = int(max(sampled.max(), labels.max())) + 1
    return dict(B=B, S=S, pad=pad, kind=kind, n_items=n_items, tries=S + extra, sampled=sampled, labels=labels,
                L=L.astype(F32), true_dot=rng.normal(0.0, 2.0, B).astype(F32),
                bias=rng.normal(0.0, 0.1, nb).astype(F32))


def adjustments(c):
    """(bias - log E) of the sampled ids and the labels, float64 from TensorFlow's float expected counts."""
    from _youtube_retrieval_train_oracle import expected_counts

    b = _f64(c["bias"])
    out = []
    for ids in (c["sampled"], c["labels"]):
        E = expected_counts(c["kind"], ids, c["n_items"], c["S"], c["tries"], np.float32)
        le = np.log(_f64(E))
        out.append((b[ids] - le, np.abs(b[ids]) + np.abs(le) + 4.0))
    return out


def sampled_ref(c, loss_kind):
    """dict(loss_rows, dtrue, dz, b_loss_rows, b_dtrue, b_dz, hit) with unscaled bounds (multiply by C_SAMPLED)."""
    B, S = c["B"], c["S"]
    (adj_s, am_s), (adj_l, am_l) = adjustments(c)
    L, t = _f64(c["L"]), _f64(c["true_dot"])
    z = L + adj_s[None, :]
    z0 = t + adj_l
    zm = np.abs(L) + am_s[None, :] + np.abs(z)
    zm0 = np.abs(t) + am_l + np.abs(z0)
    hit = c["labels"][:, None] == c["sampled"][None, :]
    lanes = -(-S // 32) + 5
    chain = warp_rounds(B)
    if loss_kind == 0:
        zz = np.where(hit, -np.inf, z)
        m = np.maximum(zz.max(1), z0)
        e, e0 = np.exp(zz - m[:, None]), np.exp(z0 - m)
        se = e.sum(1) + e0
        lse = m + np.log(se)
        p, p0 = e / se[:, None], e0 / se
        loss_rows = lse - z0
        lse_mag = 3.0 * lanes + np.abs(m) + np.abs(lse) + (p * zm).sum(1) + p0 * zm0
        dz, dtrue = p / B, (p0 - 1.0) / B
        gm = p * (zm + lse_mag[:, None] + 1.0)
        gm0 = p0 * (zm0 + lse_mag + 1.0) + np.abs(p0 - 1.0)
        vm = lse_mag + zm0 + np.abs(loss_rows)
    else:
        sp = np.maximum(z, 0.0) + np.log1p(np.exp(-np.abs(z)))          # sigmoid CE(z, 0)
        sp0 = np.maximum(-z0, 0.0) + np.log1p(np.exp(-np.abs(z0)))       # sigmoid CE(z0, 1)
        sg, sg0 = expit(z), expit(z0)
        sp = np.where(hit, 0.0, sp)
        loss_rows = sp.sum(1) + sp0
        dz, dtrue = np.where(hit, 0.0, sg) / B, (sg0 - 1.0) / B
        gm = np.where(hit, 0.0, sg * (2.0 + (1.0 - sg) * zm))
        gm0 = sg0 * (1.0 + (1.0 - sg0) * zm0) + np.abs(sg0 - 1.0)
        bm = np.where(hit, 0.0, sp * (lanes + 1.0) + sg * zm + np.abs(z) + 1.0)
        vm = bm.sum(1) + sp0 + (1.0 - sg0) * zm0 + np.abs(z0) + 1.0 + np.abs(loss_rows)
    dz = np.where(hit, 0.0, dz)
    gm = np.where(hit, 0.0, gm)
    return dict(loss_rows=loss_rows, dtrue=dtrue, dz=dz, hit=hit, b_loss_rows=U * (chain + 2) * vm,
                b_dtrue=U * gm0 / B + ETA, b_dz=np.where(hit, 0.0, U * gm / B + ETA))
