"""Calibration of the error bounds of the loss kernels (tests/_loss_kernels_ref.py) on the CPU, and the float64
restatements checked against torch float64 autograd.

Each bound is C * u * (a magnitude computed from the inputs).  Float32 restatements of each kernel's chain (the same
formulas, the same per-thread grid-stride sums and per-lane column order, the same shuffle trees and online max /
sum merges, double block sums) run on the cases the GPU tests use: they must meet every bound with a factor 4 to
spare, and the worst case of each family must use at least 1/1000 of its bound.  The restatements use numpy's expf,
not __expf: BPR's bound carries __expf's documented error separately.
"""
import numpy as np
import pytest
from scipy.special import expit

import _loss_kernels_ref as R

F32, F64 = np.float32, np.float64
INBATCH_CALIB = [c for c in R.INBATCH_CASES if c[0] <= 257] + [(2049, 3, 0.05, "edges", "dups")]
PAIR_CALIB = [s for s in R.PAIR_SHAPES if s[0] * s[1] <= 1_000_000] + [(300_000, 3)]


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


def _sigmoid32(x):
    e = np.exp(-np.abs(x))
    return np.where(x >= 0, F32(1) / (F32(1) + e), e / (F32(1) + e))


def _thread_sums(v, rounds):
    """Each thread's float sum over its grid-stride rounds (v in element order), then the double block sums."""
    T = -(-len(v) // rounds)
    vp = np.zeros(rounds * T, dtype=F32)
    vp[:len(v)] = v
    acc = np.zeros(T, dtype=F32)
    for r in range(rounds):
        acc = acc + vp[r * T:(r + 1) * T]
    return acc.astype(F64).sum()


def _warp_tree(acc, op=np.add):
    for o in (16, 8, 4, 2, 1):
        acc = op(acc[..., :o], acc[..., o:2 * o])
    return acc[..., 0]


def _lanes(a, fill):
    """[R, n] -> [R, ceil(n / 32), 32]: column c on lane c % 32, step c // 32."""
    Rn, n = a.shape
    k = -(-n // 32)
    out = np.full((Rn, k * 32), fill, dtype=a.dtype)
    out[:, :n] = a
    return out.reshape(Rn, k, 32)


def _row_loss_sum(loss_rows, B):
    """Lane 0's float sum over the rows of its warp, then double sums."""
    ch = R.warp_rounds(B)
    return _thread_sums(loss_rows.astype(F32), ch)


# ----- elements --------------------------------------------------------------------------------------------------------
def elems_f32(x, y, kind, gamma):
    x, y = x.astype(F32), y.astype(F32)
    bce = np.maximum(x, F32(0)) - x * y + np.log1p(np.exp(-np.abs(x)))
    p = _sigmoid32(x)
    if kind == 0:
        return bce, p - y
    a, gam = F32(R.ALPHA), F32(gamma)
    wt = y * a + (F32(1) - y) * (F32(1) - a)
    pt = y * p + (F32(1) - y) * (F32(1) - p)
    om = F32(1) - pt
    mm = np.power(om, gam)
    dpt = (F32(2) * y - F32(1)) * p * (F32(1) - p)
    with np.errstate(divide="ignore", invalid="ignore"):
        dm = np.where(om > 0, -gam * np.power(om, gam - F32(1)) * dpt, F32(0))
    return wt * mm * bce, wt * (dm * bce + mm * (p - y))


# ----- pairwise ---------------------------------------------------------------------------------------------------------
def pairwise_f32(pos, neg, kind, margin=0.0, mean=True):
    n_pos, n_neg = len(pos), len(neg)
    if kind <= 1:
        f = n_neg // n_pos
        d = np.repeat(pos, f) - neg
        if kind == 0:
            v = np.maximum(-d, F32(0)) + np.log1p(np.exp(-np.abs(d)))
            gp = -_sigmoid32(-d)
        else:
            t = F32(margin) - d
            v = np.maximum(t, F32(0))
            gp = np.where(t >= 0, F32(-1), F32(0))
        inv = F32(1) / F32(n_neg)
        gs = np.zeros(n_pos, dtype=F32)
        for k in range(f):
            gs = gs + gp.reshape(n_pos, f)[:, k]
        # thread j sums its f values per round: element order j * f + k, rounds over j
        rounds = R.grid_rounds(n_pos)
        T = -(-n_pos // rounds)
        acc = np.zeros(T, dtype=F32)
        vv = v.reshape(n_pos, f)
        for r in range(rounds):
            seg = vv[r * T:(r + 1) * T]
            for k in range(f):
                acc[:len(seg)] = acc[:len(seg)] + seg[:, k]
        return F32(acc.astype(F64).sum() / n_neg), gs * inv, -gp * inv
    n = n_pos + n_neg
    x = np.concatenate([pos, neg])
    y = np.concatenate([np.ones(n_pos, F32), np.zeros(n_neg, F32)])
    v, g = elems_f32(x, y, 0 if kind == 2 else 1, 2.0)
    sc = 1.0 / n if mean else 1.0
    g = g * F32(sc)
    return F32(_thread_sums(v, R.grid_rounds(n)) * sc), g[:n_pos], g[n_pos:]


def _pair_cases():
    for n_pos, f in PAIR_CALIB:
        for kind in (0, 1, 2, 3):
            for margin in (R.MARGINS if kind == 1 else (0.0,)):
                for mean in ((True, False) if kind >= 2 else (True,)):
                    yield n_pos, f, kind, margin, mean


def test_pairwise_bounds():
    ratios = []
    for n_pos, f, kind, margin, mean in _pair_cases():
        pos, neg = R.make_pair_case(n_pos, f, kind, margin)
        if kind >= 2:
            neg = neg[:max(len(neg) // 2, 1)]                       # the class losses take any n_neg
        ref = R.pairwise_ref(pos, neg, kind, margin, mean)
        L, gp, gn = pairwise_f32(pos, neg, kind, margin, mean)
        ratios += [_ratio(L, ref["loss"], ref["b_loss"]), _ratio(gp, ref["dpos"], ref["b_dpos"]),
                   _ratio(gn, ref["dneg"], ref["b_dneg"])]
    _calibrate(ratios, R.C_PAIR, "pairwise")


def test_max_margin_restatement_is_exact_on_quantised_scores():
    """Every max-margin case is exact in float: the restatement agrees bit for bit, ties included."""
    for n_pos, f in PAIR_CALIB[2:]:
        for margin in R.MARGINS:
            pos, neg = R.make_pair_case(n_pos, f, 1, margin)
            ref = R.pairwise_ref(pos, neg, 1, margin)
            _, gp, gn = pairwise_f32(pos, neg, 1, margin)
            inv = F32(1) / F32(len(neg))
            np.testing.assert_array_equal(gn, np.rint(ref["dneg"] * len(neg)).astype(F32) * inv)
            np.testing.assert_array_equal(gp, np.rint(ref["dpos"] * len(neg)).astype(F32) * inv)
            assert (ref["v"] == 0).any() and (ref["dneg"] != 0).any()


def test_focal_gamma_sweep_bounds():
    x, y = R.make_focal_case()
    n = len(x)
    ratios = []
    for gamma in R.FOCAL_GAMMAS:
        v, g, vm, gm = R.pointwise_elems(x, y, 1, R.ALPHA, gamma)
        v32, g32 = elems_f32(x, y, 1, gamma)
        g32 = g32 * (F32(1) / F32(n))
        L32 = _thread_sums(v32, R.grid_rounds(n)) / n
        ratios += [_ratio(g32, g / n, R.U * gm / n + R.ETA),
                   _ratio(L32, v.sum() / n, R.U * (R.grid_rounds(n) + 2) * vm.sum() / n)]
        assert np.isfinite(g32).all()
    _calibrate(ratios, R.C_PAIR, "pointwise focal, gamma sweep")


# ----- in-batch softmax ----------------------------------------------------------------------------------------------------
def inbatch_f32(c):
    B, S = c["B"], c["S"]
    tau = F32(c["temperature"])
    inv = F32(1) / tau if tau != 0 else F32(0)
    lg = S * inv if inv != 0 else np.zeros_like(S)
    if c["corr"] is not None:
        lg = lg - np.log(np.minimum(np.maximum(c["corr"], F32(1e-8)), F32(1)))[None, :]
    eye = np.eye(B, dtype=bool)
    masked = np.zeros_like(eye)
    if c["ids"] is not None:
        masked = (c["ids"][:, None] == c["ids"][None, :]) & ~eye
        lg = np.where(masked, F32(-R.FLT_MAX), lg)
    mx = _warp_tree(_lanes(lg, F32(-R.FLT_MAX)).max(1), np.maximum)
    with np.errstate(over="ignore"):
        e = np.exp(lg - mx[:, None])
    se = _warp_tree(_lane_chain(e))
    lse = mx + np.log(se)
    loss_rows = lse - lg[eye]
    with np.errstate(over="ignore"):
        g = (np.exp(lg - lse[:, None]) - eye.astype(F32)) * inv * (F32(1) / F32(B))
    g = np.where(masked, F32(0), g)
    return F32(_row_loss_sum(loss_rows, B) / B), g


def _lane_chain(a):
    """Per-lane float chains over the column steps: [R, n] -> [R, 32]."""
    t = _lanes(a, F32(0))
    acc = np.zeros((a.shape[0], 32), dtype=F32)
    for k in range(t.shape[1]):
        acc = acc + t[:, k]
    return acc


def test_inbatch_bounds():
    ratios = []
    for args in INBATCH_CALIB:
        c = R.make_inbatch_case(*args)
        ref = R.inbatch_ref(c)
        L, g = inbatch_f32(c)
        B = c["B"]
        ratios += [_ratio(L, ref["loss_rows"].sum() / B, ref["b_loss_rows"].sum() / B),
                   _ratio(g, ref["grad"], ref["b_grad"])]
    _calibrate(ratios, R.C_INBATCH, "in-batch softmax")


def test_inbatch_cases_reach_every_branch():
    seen = set()
    for B, pad, tau, corr, ids in R.INBATCH_CASES:
        seen |= {("tau", tau), ("corr", corr), ("ids", ids), ("pad", pad > 0), ("rows", R.warp_rounds(B) > 1),
                 ("partial warp", B % 32 != 0)}
    assert len(seen) == 3 + 2 + 4 + 2 + 2 + 2
    c = R.make_inbatch_case(257, 0, 1.0, "edges", None)
    assert {0.0, F32(1e-9), 1.0, 2.0} <= set(c["corr"].tolist())


# ----- sampled softmax / NCE -------------------------------------------------------------------------------------------------
SAMPLED_CALIB = R.SAMPLED_CASES


def sampled_f32(c, loss_kind):
    from _youtube_retrieval_train_oracle import expected_counts

    B, S = c["B"], c["S"]
    adj = []
    for ids in (c["sampled"], c["labels"]):
        E = expected_counts(c["kind"], ids, c["n_items"], S, c["tries"], np.float32)
        adj.append(c["bias"][ids] - np.log(E.astype(F32)))
    adj_s, adj_l = adj
    z0 = c["true_dot"] + adj_l
    hit = c["labels"][:, None] == c["sampled"][None, :]
    z = c["L"] + adj_s[None, :]
    invB = F32(1) / F32(B)
    if loss_kind == 0:
        zl, hl = _lanes(z, F32(0)), _lanes(hit, True)
        m = np.repeat(z0[:, None], 32, 1).astype(F32)
        s = np.zeros((B, 32), dtype=F32)
        with np.errstate(over="ignore", invalid="ignore"):      # the branch np.where discards may overflow
            for k in range(zl.shape[1]):
                zk, skip = zl[:, k], hl[:, k]
                up = (zk > m) & ~skip
                s = np.where(skip, s, np.where(up, s * np.exp(m - zk) + F32(1), s + np.exp(zk - m)))
                m = np.where(up, zk, m)
            for o in (16, 8, 4, 2, 1):
                m1, s1, m2, s2 = m[:, :o], s[:, :o], m[:, o:2 * o], s[:, o:2 * o]
                mm = np.maximum(m1, m2)
                s, m = s1 * np.exp(m1 - mm) + s2 * np.exp(m2 - mm), mm
        m, s = m[:, 0], s[:, 0]
        lse = m + np.log(s + np.exp(z0 - m))
        loss_rows = lse - z0
        d0 = (np.exp(z0 - lse) - F32(1)) * invB
        dz = np.where(hit, F32(0), np.exp(z - lse[:, None]) * invB)
    else:
        bce = np.maximum(z, F32(0)) + np.log1p(np.exp(-np.abs(z)))
        bce = np.where(hit, F32(0), bce)
        ls = _warp_tree(_lane_chain(bce))
        loss_rows = ls + (np.maximum(z0, F32(0)) - z0 + np.log1p(np.exp(-np.abs(z0))))
        d0 = (_sigmoid32(z0) - F32(1)) * invB
        dz = np.where(hit, F32(0), _sigmoid32(z) * invB)
    return F32(_row_loss_sum(loss_rows, B) / B), d0, dz


def test_sampled_bounds():
    ratios = []
    for args in SAMPLED_CALIB:
        c = R.make_sampled_case(*args)
        for lk in (0, 1):
            ref = R.sampled_ref(c, lk)
            L, d0, dz = sampled_f32(c, lk)
            B = c["B"]
            ratios += [_ratio(L, ref["loss_rows"].sum() / B, ref["b_loss_rows"].sum() / B),
                       _ratio(d0, ref["dtrue"], ref["b_dtrue"]), _ratio(dz, ref["dz"], ref["b_dz"])]
    _calibrate(ratios, R.C_SAMPLED, "sampled softmax / NCE")


def test_sampled_cases_reach_every_branch():
    seen = set()
    for args in R.SAMPLED_CASES:
        c = R.make_sampled_case(*args)
        hits = (c["labels"][:, None] == c["sampled"][None, :]).sum(1)
        seen |= {("hits", int(min(h, 2))) for h in hits}
        seen |= {("pad", c["pad"] > 0), ("tries", c["tries"] > c["S"]), ("sampler", c["kind"]),
                 ("n_items", "S" if c["n_items"] == c["S"] else "big" if c["n_items"] > 2 ** 30 else "mid"),
                 ("S % 32", c["S"] % 32 != 0), ("rows", R.warp_rounds(c["B"]) > 1), ("allhit", bool(hits[0] == c["S"]))}
    assert len(seen) == 3 + 2 + 2 + 2 + 3 + 2 + 2 + 2, sorted(seen)


# ----- float64 restatements against torch float64 autograd --------------------------------------------------------------------
def _torch_focal(x, y, gamma, alpha=R.ALPHA):
    import torch

    p = torch.sigmoid(x)
    pt = y * p + (1 - y) * (1 - p)
    w = y * alpha + (1 - y) * (1 - alpha)
    bce = torch.nn.functional.binary_cross_entropy_with_logits(x, y, reduction="none")
    return w * torch.pow(1.0 - pt, gamma) * bce


@pytest.mark.parametrize("kind", [0, 1, 2, 3])
def test_pairwise_restatement_matches_autograd(kind):
    import torch
    import torch.nn.functional as Fn

    for margin in (R.MARGINS if kind == 1 else (0.0,)):
        for n_pos, f in ((31, 3), (257, 1), (1, 17)):
            pos, neg = R.make_pair_case(n_pos, f, kind, margin)
            p = torch.tensor(pos.astype(F64), requires_grad=True)
            q = torch.tensor(neg.astype(F64), requires_grad=True)
            for mean in ((True, False) if kind >= 2 else (True,)):
                p.grad = q.grad = None
                if kind == 0:
                    v = -Fn.logsigmoid(p.repeat_interleave(f) - q).mean()
                elif kind == 1:
                    pr = p.repeat_interleave(f)
                    v = Fn.margin_ranking_loss(pr, q, torch.ones_like(pr), margin=float(margin))
                else:
                    x = torch.cat([p, q])
                    y = torch.cat([torch.ones_like(p), torch.zeros_like(q)])
                    e = (Fn.binary_cross_entropy_with_logits(x, y, reduction="none") if kind == 2
                         else _torch_focal(x, y, 2.0))
                    v = e.mean() if mean else e.sum()
                v.backward()
                ref = R.pairwise_ref(pos, neg, kind, margin, mean)
                assert _ratio(v.item(), ref["loss"], ref["b_loss"]) <= 1e-3
                assert _ratio(p.grad.numpy(), ref["dpos"], ref["b_dpos"] + 1e-300) <= 1e-3
                assert _ratio(q.grad.numpy(), ref["dneg"], ref["b_dneg"] + 1e-300) <= 1e-3
                if kind == 1:                                       # ties included: exact
                    np.testing.assert_array_equal(q.grad.numpy(), ref["dneg"])


def test_focal_restatement_matches_autograd_but_at_saturation():
    """Equal to torch wherever torch is finite; where 1 - p_t == 0 and 0 < gamma < 1 torch's gradient is NaN or inf
    and the restatement (like the kernel) gives 0."""
    import torch

    x, y = R.make_focal_case()
    for gamma in R.FOCAL_GAMMAS:
        xt = torch.tensor(x.astype(F64), requires_grad=True)
        v = _torch_focal(xt, torch.tensor(y.astype(F64)), gamma)
        v.sum().backward()
        ev, g, vm, gm = R.pointwise_elems(x, y, 1, R.ALPHA, gamma)
        tg = xt.grad.numpy()
        fin = np.isfinite(tg)
        assert _ratio(v.detach().numpy(), ev, R.U * vm) <= 1e-3
        assert _ratio(tg[fin], g[fin], R.U * gm[fin] + 1e-300) <= 1e-3
        sat = (1.0 - (y * expit(x.astype(F64)) + (1 - y) * (1 - expit(x.astype(F64))))) == 0
        assert sat.any()
        if 0 < gamma < 1:
            assert not np.isfinite(tg[sat]).any()
        assert np.isfinite(g).all()
        if gamma > 0:
            assert (g[sat] == 0).all()


def test_inbatch_restatement_matches_autograd():
    import torch

    for args in [a for a in R.INBATCH_CASES if a[0] <= 257]:
        c = R.make_inbatch_case(*args)
        B = c["B"]
        S = torch.tensor(c["S"].astype(F64), requires_grad=True)
        tau = c["temperature"]
        lg = S / tau if tau != 0 else S * 0.0                       # divide_no_nan
        if c["corr"] is not None:
            lg = lg - torch.log(torch.clamp(torch.tensor(c["corr"].astype(F64)), R.CORR_MIN, 1.0))[None, :]
        if c["ids"] is not None:
            ids = torch.tensor(c["ids"])
            mask = (ids[:, None] == ids[None, :]) & ~torch.eye(B, dtype=torch.bool)
            lg = torch.where(mask, torch.tensor(-R.FLT_MAX, dtype=torch.float64), lg)
        v = torch.nn.functional.cross_entropy(lg, torch.arange(B))
        v.backward()
        ref = R.inbatch_ref(c)
        assert _ratio(v.item(), ref["loss_rows"].sum() / B, ref["b_loss_rows"].sum() / B) <= 1e-3
        assert _ratio(S.grad.numpy(), ref["grad"], ref["b_grad"]) <= 1e-3
        if tau == 0:
            assert (ref["grad"] == 0).all()
        if args[4] == "all_equal":
            assert (ref["loss_rows"] == 0).all() and (ref["grad"] == 0).all()


def test_sampled_restatement_matches_autograd():
    import torch

    for args in R.SAMPLED_CASES[:7]:
        c = R.make_sampled_case(*args)
        B = c["B"]
        (adj_s, _), (adj_l, _) = R.adjustments(c)
        for lk in (0, 1):
            L = torch.tensor(c["L"].astype(F64), requires_grad=True)
            t = torch.tensor(c["true_dot"].astype(F64), requires_grad=True)
            # _compute_sampled_logits: label in column 0, accidental hits at -FLT_MAX
            z = torch.cat([(t + torch.tensor(adj_l))[:, None], L + torch.tensor(adj_s)[None, :]], 1)
            hit = torch.tensor(c["labels"][:, None] == c["sampled"][None, :])
            z = torch.cat([z[:, :1], z[:, 1:] + torch.where(hit, -R.FLT_MAX, 0.0)], 1)
            if lk == 0:
                v = torch.nn.functional.cross_entropy(z, torch.zeros(B, dtype=torch.int64))
            else:
                y = torch.zeros_like(z)
                y[:, 0] = 1.0
                v = torch.nn.functional.binary_cross_entropy_with_logits(z, y, reduction="none").sum(1).mean()
            v.backward()
            ref = R.sampled_ref(c, lk)
            assert _ratio(v.item(), ref["loss_rows"].sum() / B, ref["b_loss_rows"].sum() / B) <= 1e-3
            assert _ratio(t.grad.numpy(), ref["dtrue"], ref["b_dtrue"]) <= 1e-3
            assert _ratio(L.grad.numpy(), ref["dz"], ref["b_dz"]) <= 1e-3
