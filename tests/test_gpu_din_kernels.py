"""The DIN attention kernels of ``csrc/seq.cu`` and the fused sigmoid-dot epilogue of ``csrc/mlp_tc.cu``, called
directly through the C-ABI and compared with float64 restatements of the same operations, at the shapes where these
kernels branch: partial warps (K' < 32), every column chunk count TKC = 1..4, K' % 4 != 0 and misaligned tables
(which take the first-version kernels), positions 32..63 (the second round of the lane-owns-position kernels),
sequences longer than 64 (first version only), lengths outside [0, T] (clamped), repeated keys and items that are
their own keys.

Error bounds are stated per row in quantities the test computes, with u = 2^-24 (fp32 unit roundoff):
  attention output  C u kmax (L + 2 amag + 1)
    kmax  = max |k_t[c]| over the row's L valid keys,
    amag  = max_t of the logit's sensitivity to rounding: rsqrt(K') (sum_j |k2_j| (h_j + h_j (1 - h_j) zmag_j) + |b2|)
            for the paper attention (zmag_j = sum_i |x_i| |W1_ij| + |b1_j|, the magnitude of the pre-activation),
            2 sum_c |q_c k_t[c]| for the dot-product attention;
  a logit error d moves the output by at most 2 d kmax, the weighted key sum and the softmax add L u kmax.
The constants C are checked against float32 restatements of the same cases on the CPU
(tests/test_din_kernel_bounds_cpu.py): float32 numpy meets every bound with at least a factor 4 to spare.
"""
from __future__ import annotations

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

U = 2.0 ** -24
F32, F64 = np.float32, np.float64

# bound constants (see the module docstring); calibrated by tests/test_din_kernel_bounds_cpu.py
C_ATT = 8.0          # paper attention output
C_DOT = 8.0          # dot-product attention output
C_UW = 16.0          # din_user_weights: Wt and bias
C_LOGIT = 16.0       # sigmoid-dot logits A (3xTF32 GEMM + sigmoid + Dense(1))
C_CHAIN = 12.0       # user weights -> 3xTF32 GEMM -> attention, against the paper attention
C_BWD = 8.0          # backward: dG and the weight gradients
C_POOL = 4.0         # sequence pooling

FWD_KP = [1, 12, 30, 32, 36, 64, 72, 100, 128]
FWD_T = [1, 31, 32, 33, 64, 65, 200, 256]


# ---------------------------------------------------------------------------------------------------------------------
# case generation (numpy only: shared with the CPU calibration)
# ---------------------------------------------------------------------------------------------------------------------
def make_att(rng, Kp):
    """Attention MLP weights scaled so that pre-activations are O(1) and logits O(1) at every K'."""
    return dict(k1=(rng.standard_normal((4 * Kp, 16)) / np.sqrt(2 * Kp)).astype(F32),
                b1=(0.5 * rng.standard_normal(16)).astype(F32),
                k2=(rng.standard_normal(16) * max(1.0, np.sqrt(Kp) / 2)).astype(F32),
                b2=F32(0.3))


def att64(att):
    return {k: (np.asarray(v, dtype=F64) if k != "b2" else F64(v)) for k, v in att.items()}


def make_seq_case(seed, Kp, T, n_items=40, n_users=10, N=None, off=5):
    """Item table G [n_items + 1, K'] (last row = pad row, random so that a read past len shows), per-user sequences
    [n_users, T] padded with the pad id, lens covering 0, 1, T, > T, < 0 and random values; a grid of (user, item)
    pairs for the all-items mode and the same pairs plus items-in-their-own-sequence as explicit rows."""
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n_items + 1, Kp)).astype(F32)
    lens = np.array([0, 1, T, T + 7, -3] + list(rng.integers(1, T + 1, 3)) + [min(T, 33), max(T - 1, 1)],
                    dtype=np.int32)[:n_users]
    seqs = np.full((n_users, T), n_items, dtype=np.int32)
    for u in range(n_users):
        L = int(np.clip(lens[u], 0, T))
        seqs[u, :L] = rng.integers(0, n_items, L)
    L7 = int(np.clip(lens[7], 0, T))
    seqs[7, :L7] = rng.choice(rng.integers(0, n_items, 3), L7)          # few keys, many repeats
    if N is None:
        N = 23 if T <= 64 else 5
    R_grid = n_users * N - off - 3
    assert R_grid % N != 0
    grid_users = rng.permutation(n_users).astype(np.int64)
    idx = np.arange(R_grid) + off
    g_user, g_item = grid_users[idx // N], idx % N
    own = [u for u in range(n_users) if np.clip(lens[u], 0, T) > 0]
    e_user = np.concatenate([g_user, own]).astype(np.int64)
    e_item = np.concatenate([g_item, [seqs[u, 0] for u in own]]).astype(np.int64)
    return dict(G=G, seqs=seqs, lens=lens, T=T, Kp=Kp, att=make_att(rng, Kp), N=N, off=off, R_grid=R_grid,
                grid_users=grid_users, e_user=e_user, e_item=e_item, n_items=n_items)


def case_rows(c):
    """(q, keys, clamped lens) of the explicit rows, float64."""
    G = c["G"].astype(F64)
    return G[c["e_item"]], G[c["seqs"][c["e_user"]]], np.clip(c["lens"][c["e_user"]], 0, c["T"])


def _valid(lens, T):
    return np.arange(T)[None, :] < np.asarray(lens).reshape(-1, 1)


def _sig(z):
    return 1.0 / (1.0 + np.exp(-z))


def out_bound(amag_rt, keys, lens):
    """u kmax (L + 2 amag + 1) per row; amag_rt [R, T] is masked to the valid positions here."""
    m = _valid(lens, keys.shape[1])
    amag = np.where(m, amag_rt, 0.0).max(axis=1)
    kmax = np.where(m[:, :, None], np.abs(keys), 0.0).max(axis=(1, 2))
    return U * kmax * (np.asarray(lens, dtype=F64) + 2.0 * amag + 1.0)


def paper_features(q, keys, att):
    """float64 pre-activations z, their magnitudes zmag and the hidden units h of the paper attention."""
    a = att64(att)
    T = keys.shape[1]
    qq = np.repeat(q[:, None, :], T, axis=1)
    feat = np.concatenate([qq, keys, qq - keys, qq * keys], axis=2)
    z = feat @ a["k1"] + a["b1"]
    zmag = np.abs(feat) @ np.abs(a["k1"]) + np.abs(a["b1"])
    return feat, z, zmag, _sig(z)


def logit_mag(h, zmag, att, Kp):
    """rsqrt(K') (sum_j |k2_j| (h_j + h_j (1 - h_j) zmag_j) + |b2|) over the last axis of h."""
    k2 = np.abs(np.asarray(att["k2"], dtype=F64))
    return ((h + h * (1.0 - h) * zmag) @ k2 + abs(float(att["b2"]))) / np.sqrt(Kp)


def paper_bound(q, keys, lens, att):
    _, _, zmag, h = paper_features(q, keys, att)
    return out_bound(logit_mag(h, zmag, att, keys.shape[2]), keys, lens)


def dot_bound(q, keys, lens):
    return out_bound(2.0 * np.einsum("rc,rtc->rt", np.abs(q), np.abs(keys)), keys, lens)


def softmax_sum(logits, keys, lens):
    """float64 masked softmax over the valid positions and the weighted key sum (zero rows for L = 0)."""
    m = _valid(lens, keys.shape[1])
    a = np.where(m, logits, -np.inf)
    amax = np.where(m.any(axis=1), a.max(axis=1), 0.0)
    p = np.where(m, np.exp(a - amax[:, None]), 0.0)
    p = p / np.maximum(p.sum(axis=1, keepdims=True), 1e-300)
    return np.einsum("rt,rtc->rc", p, keys), p


# ----- all-items (hoisted) family: one user, N items --------------------------------------------------------------------
def make_user_case(seed, Kp, L, n_items):
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n_items + 1, Kp)).astype(F32)
    seq = rng.integers(0, n_items, max(L, 1)).astype(np.int32)
    if L >= 4:
        seq[1] = seq[0]                                                  # a repeated key
    return dict(G=G, seq=seq, L=L, Kp=Kp, att=make_att(rng, Kp), n_items=n_items)


def user_weights_ref(G, seq, L, att):
    """Wt [16 L, K'] with row (t, j) = A_t[:, j] = (W1q + W1d)[:, j] + k_t * W1p[:, j] and
    bias[16 t + j] = b1[j] + sum_c k_t[c] (W1k - W1d)[c][j], float64, with their rounding magnitudes."""
    a = att64(att)
    Kp = G.shape[1]
    Wq, Wk, Wd, Wp = (a["k1"][i * Kp:(i + 1) * Kp] for i in range(4))
    keys = G[seq[:L]].astype(F64)
    Wt = ((Wq + Wd).T[None] + keys[:, None, :] * Wp.T[None]).reshape(16 * L, Kp)
    bias = (a["b1"][None] + keys @ (Wk - Wd)).reshape(-1)
    Wt_mag = ((np.abs(Wq) + np.abs(Wd)).T[None] + np.abs(keys)[:, None, :] * np.abs(Wp).T[None]).reshape(16 * L, Kp)
    bias_mag = (np.abs(a["b1"])[None] + np.abs(keys) @ (np.abs(Wk) + np.abs(Wd))).reshape(-1)
    return Wt, bias, Wt_mag, bias_mag


def user_weights_f32(G, seq, L, att):
    k1 = att["k1"]
    Kp = G.shape[1]
    Wq, Wk, Wd, Wp = (k1[i * Kp:(i + 1) * Kp] for i in range(4))
    keys = G[seq[:L]]
    Wt = ((Wq + Wd).T[None] + keys[:, None, :] * Wp.T[None]).reshape(16 * L, Kp)
    bias = (att["b1"][None] + keys @ (Wk - Wd)).reshape(-1)
    return Wt.astype(F32), bias.astype(F32)


def hoisted_ref(Z, keys, L, att):
    """Attention output per item from the pre-activations Z [N, 16 L] (float64) and its bound."""
    a = att64(att)
    N, Kp = Z.shape[0], keys.shape[1]
    lens = np.full(N, L)
    if L == 0:
        return np.zeros((N, Kp)), np.zeros(N)
    h = _sig(Z.reshape(N, L, 16))
    logits = (h @ a["k2"] + a["b2"]) / np.sqrt(Kp)
    kb = np.broadcast_to(keys[None], (N, L, Kp))
    out, _ = softmax_sum(logits, kb, lens)
    return out, out_bound(logit_mag(h, np.abs(Z.reshape(N, L, 16)), att, Kp), kb, lens)


def hoisted_f32(Z32, keys32, L, att):
    N, Kp = Z32.shape[0], keys32.shape[1]
    if L == 0:
        return np.zeros((N, Kp), F32)
    h = F32(1) / (F32(1) + np.exp(-Z32.reshape(N, L, 16)))
    a = (h @ att["k2"] + att["b2"]) * F32(1.0 / np.sqrt(Kp))
    a = a - a.max(axis=1, keepdims=True)
    p = np.exp(a)
    p = p / p.sum(axis=1, keepdims=True)
    return (p @ keys32).astype(F32)


def logits_ref(X, Wt, bias, k2):
    """A[n, t] = sum_j k2[j] sigmoid(X[n] . Wt[16 t + j] + bias[16 t + j]) in float64, and its bound
    u sum_j |k2_j| (1 + h_j (1 - h_j) zmag_j)."""
    X, Wt, bias, k2 = (np.asarray(v, dtype=F64) for v in (X, Wt, bias, k2))
    L = Wt.shape[0] // 16
    z = (X @ Wt.T + bias).reshape(-1, L, 16)
    zmag = (np.abs(X) @ np.abs(Wt).T + np.abs(bias)).reshape(-1, L, 16)
    h = _sig(z)
    return h @ k2, U * ((1.0 + h * (1.0 - h) * zmag) @ np.abs(k2))


def _tf32(x):
    return (np.ascontiguousarray(x, dtype=F32).view(np.uint32) & np.uint32(0xFFFFE000)).view(F32)


def linear_3xtf32_f32(X, Wt, bias):
    """CPU model of b200_linear_tf32x3: x = hi + lo with hi, lo truncated to tf32, hi*hi + (lo*hi + hi*lo), fp32 sums."""
    xh, wh = _tf32(X), _tf32(Wt)
    xl, wl = _tf32(X - xh), _tf32(Wt - wh)
    main = xh @ wh.T
    corr = xl @ wh.T + xh @ wl.T
    return ((corr + main) + bias).astype(F32)


def logits_f32(X, Wt, bias, k2):
    L = Wt.shape[0] // 16
    z = linear_3xtf32_f32(X, Wt, bias).reshape(-1, L, 16)
    return ((F32(1) / (F32(1) + np.exp(-z))) @ k2).astype(F32)


def from_logits_ref(A, keys, L, b2, Kp):
    N = A.shape[0]
    lens = np.full(N, L)
    logits = (np.asarray(A, dtype=F64) + float(b2)) / np.sqrt(Kp)
    kb = np.broadcast_to(keys[None], (N, L, Kp))
    out, _ = softmax_sum(logits, kb, lens)
    return out, out_bound((np.abs(A) + abs(float(b2))) / np.sqrt(Kp), kb, lens)


def from_logits_f32(A32, keys32, b2, Kp):
    a = (A32 + F32(b2)) * F32(1.0 / np.sqrt(Kp))
    a = a - a.max(axis=1, keepdims=True)
    p = np.exp(a)
    p = p / p.sum(axis=1, keepdims=True)
    return (p @ keys32).astype(F32)


# ----- backward ----------------------------------------------------------------------------------------------------------
def make_bwd_case(seed, Kp, T, R=5000, n_items=50, n_users=40, n_pairs=160):
    """R rows drawn from n_pairs distinct (user, item) pairs over a small table: the same keys and items recur in
    hundreds of rows, so the atomics pile onto few rows.  The loss of the rows is sum_r <dout_r, out(pair_r)>, so the
    reference needs only the pairs with their summed dout."""
    rng = np.random.default_rng(seed)
    G = rng.standard_normal((n_items + 1, Kp)).astype(F32)
    lens = rng.integers(1, T + 1, n_users).astype(np.int32)
    lens[:4] = [0, 1, T, T + 9]
    lens[4] = min(T, 33)
    seqs = np.full((n_users, T), n_items, dtype=np.int32)
    hot = rng.integers(0, n_items, 4)
    for u in range(n_users):
        L = int(np.clip(lens[u], 0, T))
        pool = hot if u % 3 == 0 else np.arange(n_items)                  # every third user: 4 hot keys, repeated
        seqs[u, :L] = rng.choice(pool, L)
    p_user = rng.integers(0, n_users, n_pairs)
    p_item = rng.integers(0, n_items, n_pairs)
    for i in range(0, n_pairs, 5):                                         # items that are also their own keys
        L = int(np.clip(lens[p_user[i]], 0, T))
        if L:
            p_item[i] = seqs[p_user[i], rng.integers(0, L)]
    row_pair = rng.integers(0, n_pairs, R)
    dout = rng.standard_normal((R, Kp)).astype(F32)
    return dict(G=G, seqs=seqs, lens=lens, T=T, Kp=Kp, att=make_att(rng, Kp), p_user=p_user.astype(np.int64),
                p_item=p_item.astype(np.int64), row_pair=row_pair, dout=dout, n_items=n_items)


def bwd_pair_inputs(c):
    """Per pair: key ids [P, T], clamped lens, summed dout and summed |dout| (zero for L = 0: no gradient)."""
    P = len(c["p_user"])
    lens = np.clip(c["lens"][c["p_user"]], 0, c["T"])
    dsum = np.zeros((P, c["Kp"]))
    dabs = np.zeros((P, c["Kp"]))
    np.add.at(dsum, c["row_pair"], c["dout"].astype(F64))
    np.add.at(dabs, c["row_pair"], np.abs(c["dout"]).astype(F64))
    dsum[lens == 0] = 0.0
    dabs[lens == 0] = 0.0
    return c["seqs"][c["p_user"]].astype(np.int64), lens, dsum, dabs


def bwd_autograd(c, dtype):
    """Gradients of sum_p <dsum_p, out_p> (the attention of oracle/din_train.py) w.r.t. G and the attention weights,
    by torch autograd in ``dtype``."""
    import torch

    keyids, lens, dsum, _ = bwd_pair_inputs(c)
    t = {k: torch.tensor(np.asarray(v, dtype=F64), dtype=dtype, requires_grad=True)
         for k, v in [("G", c["G"])] + [(k, c["att"][k]) for k in ("k1", "b1", "k2")]}
    b2 = torch.tensor([float(c["att"]["b2"])], dtype=dtype, requires_grad=True)
    Kp = c["Kp"]
    q = t["G"][torch.as_tensor(c["p_item"])]
    keys = t["G"][torch.as_tensor(keyids)]
    T = keys.shape[1]
    qq = q[:, None, :].expand(-1, T, -1)
    feat = torch.cat([qq, keys, qq - keys, qq * keys], dim=2)
    h = torch.sigmoid(feat @ t["k1"] + t["b1"])
    a = (h @ t["k2"] + b2[0]) * (1.0 / np.sqrt(Kp))
    mask = torch.arange(T)[None, :] < torch.as_tensor(lens).reshape(-1, 1)
    a = torch.where(mask, a, torch.full_like(a, -(2.0 ** 32) + 1))
    p = torch.softmax(a, dim=1)
    out = (p[:, :, None] * keys).sum(1)
    (out * torch.tensor(dsum, dtype=dtype)).sum().backward()
    return dict(dG=t["G"].grad.double().numpy(), k1=t["k1"].grad.double().numpy(), b1=t["b1"].grad.double().numpy(),
                k2=t["k2"].grad.double().numpy(), b2=b2.grad.double().numpy())


def bwd_magnitudes(c):
    """Rounding magnitudes of every gradient element: each (pair, position) contributes its terms in absolute value,
    weighted by the pair's amplification e = 1 + L + 2 amag (the forward's), the softmax backward term
    rsqrt(K') p_t (|<dout, k_t>| + max_t' |<dout, k_t'>|) standing for d loss / d logit; the contributions of
    different (pair, position)s to one element combine as the root of their summed squares."""
    keyids, lens, _, dabs = bwd_pair_inputs(c)
    G = c["G"].astype(F64)
    a = att64(c["att"])
    Kp, T = c["Kp"], c["T"]
    q, keys = G[c["p_item"]], G[keyids]
    feat, z, zmag, h = paper_features(q, keys, c["att"])
    m = _valid(lens, T)
    logits = (h @ a["k2"] + a["b2"]) / np.sqrt(Kp)
    _, p = softmax_sum(logits, keys, lens)
    amag = np.where(m, logit_mag(h, zmag, c["att"], Kp), 0.0).max(axis=1)
    e = (1.0 + lens + 2.0 * amag) * (lens > 0)
    mdp = np.einsum("ptc,pc->pt", np.abs(keys), dabs) * m
    mda = p * (mdp + mdp.max(axis=1, keepdims=True)) / np.sqrt(Kp)
    hd = h * (1.0 - h)
    mdz = mda[:, :, None] * np.abs(a["k2"]) * hd * (1.0 + zmag)
    w = e[:, None]
    # root of the summed squares: the rounding errors of many contributions add like independent variables
    mag = dict(b2=np.array([((w * mda) ** 2).sum()]),
               k2=np.einsum("pt,ptj->j", (w * mda) ** 2, (h + hd * zmag) ** 2),
               b1=np.einsum("p,ptj->j", e ** 2, mdz ** 2),
               k1=np.einsum("pti,ptj->ij", (np.abs(feat) * e[:, None, None]) ** 2, mdz ** 2))
    F = mdz @ np.abs(a["k1"]).T
    Fq, Fk, Fd, Fp = (F[:, :, i * Kp:(i + 1) * Kp] for i in range(4))
    aq = np.abs(q)[:, None, :]
    kc = (p[:, :, None] * dabs[:, None, :] + Fk + Fd + aq * Fp) * e[:, None, None] * m[:, :, None]
    qc = ((Fq + Fd + np.abs(keys) * Fp) * m[:, :, None]).sum(axis=1) * e[:, None]
    dG = np.zeros_like(G)
    np.add.at(dG, keyids.reshape(-1), kc.reshape(-1, Kp) ** 2)
    np.add.at(dG, c["p_item"], qc ** 2)
    mag = {k: np.sqrt(v) for k, v in mag.items()}
    mag["dG"] = np.sqrt(dG)
    return mag


# ---------------------------------------------------------------------------------------------------------------------
# GPU helpers
# ---------------------------------------------------------------------------------------------------------------------
def _dev(a):
    import torch

    return torch.as_tensor(np.ascontiguousarray(a)).cuda()


def _g_layout(G, layout):
    """G on the device: contiguous; a 16-byte aligned column slice (ld = K' + 4); ld = K' + 1; or offset by one float.
    The columns outside the slice are NaN, so a read outside [0, K') shows in the output."""
    import torch

    n, Kp = G.shape
    if layout == "contig":
        return _dev(G)
    extra, c0 = {"ld4": (4, 0), "ld1": (1, 0), "off1": (4, 1)}[layout]
    buf = torch.full((n, Kp + extra), float("nan"), dtype=torch.float32, device="cuda")
    v = buf[:, c0:c0 + Kp]
    v.copy_(torch.as_tensor(G))
    return v


LAYOUTS = ["contig", "ld4", "ld1", "off1"]


def _din_attention(Gd, c, attd, grid, out_pad=3):
    import torch

    from librecommender_b200 import _lib

    Kp, T = c["Kp"], c["T"]
    if grid:
        R, users, items, N, off = c["R_grid"], c["users_g"], None, c["N"], c["off"]
    else:
        R, users, items, N, off = len(c["e_user"]), c["users_e"], c["items_e"], 0, 0
    out = torch.full((R, Kp + out_pad), float("nan"), dtype=torch.float32, device="cuda")
    k1, b1, k2 = (attd[k] if attd else None for k in ("k1", "b1", "k2"))
    _lib.check(_lib.lib.b200_din_attention(
        _lib.ptr(Gd), Gd.stride(0), Kp, _lib.ptr(items), _lib.ptr(c["seqs_d"]), c["seqs_d"].stride(0),
        _lib.ptr(c["lens_d"]), T, _lib.ptr(users), R, N, off, _lib.ptr(k1), _lib.ptr(b1), _lib.ptr(k2),
        float(c["att"]["b2"]), _lib.ptr(out), out.stride(0), _lib.current_stream()))
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert np.isnan(o[:, Kp:]).all(), "wrote past K'"
    return o[:, :Kp]


def _to_device(c):
    c["seqs_d"], c["lens_d"] = _dev(c["seqs"]), _dev(c["lens"])
    c["users_g"], c["users_e"], c["items_e"] = _dev(c["grid_users"]), _dev(c["e_user"]), _dev(c["e_item"])
    return c


def _check_rows(got, ref, bound, lens, what):
    zero = np.asarray(lens) == 0
    assert (got[zero] == 0).all(), f"{what}: rows with an empty sequence must be exactly zero"
    err = np.abs(got - ref).max(axis=1)
    bad = np.nonzero(~zero & ~(err <= bound))[0]
    assert bad.size == 0, (f"{what}: {bad.size} rows over the bound, first row {bad[0]}: err {err[bad[0]]:.3e} "
                           f"bound {bound[bad[0]]:.3e} L {lens[bad[0]]}")


def _set_tune(v):
    from librecommender_b200 import _lib

    _lib.check(_lib.lib.b200_din_attention_tune(v))


def _forward_matrix(Kp, T, paper):
    from oracle import tf_models as tm

    c = _to_device(make_seq_case(1000 * Kp + T + (0 if paper else 7), Kp, T))
    q, keys, lens = case_rows(c)
    if paper:
        ref = tm.din_attention(q, keys, lens, att64(c["att"]), dtype=F64)
        bound = C_ATT * paper_bound(q, keys, lens, c["att"])
        attd = {k: _dev(c["att"][k]) for k in ("k1", "b1", "k2")}
    else:
        ref = tm.tf_attention(q, keys, lens, dtype=F64)
        bound = C_DOT * dot_bound(q, keys, lens)
        attd = None
    Rg = c["R_grid"]
    try:
        for tune in ((1, 0) if paper else (1,)):
            _set_tune(tune)
            for layout in LAYOUTS:
                Gd = _g_layout(c["G"], layout)
                got = _din_attention(Gd, c, attd, grid=False)
                _check_rows(got, ref, bound, lens, f"tune {tune} layout {layout}")
                got_grid = _din_attention(Gd, c, attd, grid=True)
                # same kernel, same per-row arithmetic: all-items mode must equal the explicit pairs bit for bit
                np.testing.assert_array_equal(got_grid, got[:Rg], err_msg=f"grid != pairs, tune {tune} {layout}")
                if layout == "contig":
                    np.testing.assert_array_equal(_din_attention(Gd, c, attd, grid=False), got)   # deterministic
    finally:
        _set_tune(1)


@pytest.mark.parametrize("T", FWD_T)
@pytest.mark.parametrize("Kp", FWD_KP)
def test_din_attention_paper_matches_fp64(Kp, T):
    _forward_matrix(Kp, T, paper=True)


@pytest.mark.parametrize("T", FWD_T)
@pytest.mark.parametrize("Kp", FWD_KP)
def test_dot_attention_matches_fp64(Kp, T):
    _forward_matrix(Kp, T, paper=False)


@pytest.mark.parametrize("Kp,T", [(32, 64), (100, 33), (12, 200)])
def test_dot_attention_large_logits(Kp, T):
    """<q, k_t> of order 10^3: without the max subtraction exp overflows."""
    from oracle import tf_models as tm

    c = make_seq_case(77 + Kp, Kp, T)
    c["G"] = (c["G"] * np.float32(40.0 / np.sqrt(Kp))).astype(F32)
    c = _to_device(c)
    q, keys, lens = case_rows(c)
    dots = np.einsum("rc,rtc->rt", q, keys)
    assert np.abs(dots).max() > 500
    ref = tm.tf_attention(q, keys, lens, dtype=F64)
    for grid in (False, True):
        got = _din_attention(_dev(c["G"]), c, None, grid=grid)
        assert np.isfinite(got).all()
        n = len(got)
        _check_rows(got, ref[:n], C_DOT * dot_bound(q, keys, lens)[:n], lens[:n], "large logits")


# ----- all-items family -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L", [1, 17, 64, 65, 256])
@pytest.mark.parametrize("Kp", [4, 36, 128])
def test_din_user_weights_matches_fp64(Kp, L):
    import torch

    from librecommender_b200 import _lib

    c = make_user_case(10 * Kp + L, Kp, L, 300)
    Wt64, b64, Wmag, bmag = user_weights_ref(c["G"], c["seq"], L, c["att"])
    Gd, sd = _dev(c["G"]), _dev(c["seq"])
    k1, b1 = _dev(c["att"]["k1"]), _dev(c["att"]["b1"])
    Wt = torch.full((16 * L, Kp + 5), float("nan"), dtype=torch.float32, device="cuda")     # ldw > K'
    bias = torch.full((16 * L + 2,), float("nan"), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.b200_din_user_weights(_lib.ptr(Gd), Gd.stride(0), Kp, _lib.ptr(sd), L, _lib.ptr(k1), _lib.ptr(b1),
                                              _lib.ptr(Wt), Wt.stride(0), _lib.ptr(bias), _lib.current_stream()))
    torch.cuda.synchronize()
    W, b = Wt.cpu().numpy(), bias.cpu().numpy()
    assert np.isnan(W[:, Kp:]).all() and np.isnan(b[16 * L:]).all()
    assert (np.abs(W[:, :Kp] - Wt64) <= C_UW * U * Wmag).all(), float((np.abs(W[:, :Kp] - Wt64) / Wmag).max())
    assert (np.abs(b[:16 * L] - b64) <= C_UW * U * bmag).all(), float((np.abs(b[:16 * L] - b64) / bmag).max())


def _hoisted(Z, N, Gd, c, L, z_off=0):
    import torch

    from librecommender_b200 import _lib

    Kp = c["Kp"]
    out = torch.full((N, Kp + 1), float("nan"), dtype=torch.float32, device="cuda")
    if Z is None:
        Zd, ldz = None, 0
    else:
        buf = torch.full((N, Z.shape[1] + 4), float("nan"), dtype=torch.float32, device="cuda")
        Zd = buf[:, z_off:z_off + Z.shape[1]]
        Zd.copy_(torch.as_tensor(Z))
        ldz = buf.stride(0)
    _lib.check(_lib.lib.b200_din_attention_hoisted(_lib.ptr(Zd), ldz, N, _lib.ptr(Gd), Gd.stride(0), Kp, _lib.ptr(c["seq_d"]),
                                                   L, _lib.ptr(c["k2_d"]), float(c["att"]["b2"]), _lib.ptr(out),
                                                   out.stride(0), _lib.current_stream()))
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert np.isnan(o[:, Kp:]).all()
    return o[:, :Kp]


def hoisted_case(Kp, L, N):
    c = make_user_case(7 * Kp + L + N, Kp, L, max(N, 300))
    if L == 0:
        return c, None, np.zeros((N, Kp)), np.zeros(N)
    Wt64, b64, _, _ = user_weights_ref(c["G"], c["seq"], L, c["att"])
    Z32 = (c["G"][:N].astype(F64) @ Wt64.T + b64).astype(F32)
    keys = c["G"][c["seq"][:L]].astype(F64)
    ref, bound = hoisted_ref(Z32.astype(F64), keys, L, c["att"])
    return c, Z32, ref, bound


HOIST_CASES = [(N, Kp, L) for N in (300, 5003) for Kp in (4, 32, 36, 64, 100, 128)
               for L in (0, 1, 31, 32, 33, 64, 65, 256) if not (N == 5003 and L > 64)]     # L > 64: first version only


@pytest.mark.parametrize("N,Kp,L", HOIST_CASES)
def test_din_attention_hoisted_matches_fp64(N, Kp, L):
    c, Z32, ref, bound = hoisted_case(Kp, L, N)
    Gd = _dev(c["G"])
    c["seq_d"], c["k2_d"] = _dev(c["seq"]), _dev(c["att"]["k2"])
    got = _hoisted(Z32, N, Gd, c, L)
    _check_rows(got, ref, C_ATT * bound, np.full(N, L), f"hoisted N {N}")
    if N >= 1024 and L in (33, 64):
        got1 = _hoisted(Z32, N, Gd, c, L, z_off=1)                       # Z not 16-byte aligned: first version
        _check_rows(got1, ref, C_ATT * bound, np.full(N, L), "hoisted, misaligned Z")


def _sigmoid_dot(X, Wt, bias, k2, lda, presplit, pad_rows=2):
    import torch

    from librecommender_b200 import _lib

    R, Kp = X.shape
    dout = Wt.shape[0]
    Xd, Wd, bd, kd = _dev(X), _dev(Wt), _dev(bias), _dev(k2)
    ws = None
    if presplit:
        ld = int(_lib.lib.b200_linear_tf32x3_split_ld(Kp))
        ws = torch.empty(2 * dout * ld, dtype=torch.float32, device="cuda")
        _lib.check(_lib.lib.b200_linear_tf32x3_split_weights(_lib.ptr(Wd), Wd.stride(0), Kp, dout, _lib.ptr(ws),
                                                             _lib.current_stream()))
    A = torch.full((R + pad_rows, lda), float("nan"), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.b200_linear_tf32x3_sigmoid_dot(_lib.ptr(Xd), Xd.stride(0), R, _lib.ptr(Wd), Wd.stride(0),
                                                       _lib.ptr(ws), _lib.ptr(bd), Kp, dout, _lib.ptr(kd), _lib.ptr(A),
                                                       A.stride(0), _lib.current_stream()))
    torch.cuda.synchronize()
    return A.cpu().numpy()


def sigmoid_dot_case(L, R):
    Kp = (36, 64, 128)[L % 3]
    c = make_user_case(31 * L + R, Kp, L, 300)
    rng = np.random.default_rng(L * 7 + R)
    X = rng.standard_normal((R, Kp)).astype(F32)
    Wt, bias = user_weights_f32(c["G"], c["seq"], L, c["att"])
    ref, bound = logits_ref(X, Wt, bias, c["att"]["k2"])
    return c, X, Wt, bias, ref, bound


SD_LENS = [1, 2, 3, 4, 5, 6, 7, 8, 9, 16, 33, 64]


@pytest.mark.parametrize("R", [1, 127, 129, 5003])
@pytest.mark.parametrize("L", SD_LENS)
def test_linear_sigmoid_dot_matches_fp64(L, R):
    """dout = 16 L: n_pad 32 / 64 / 96 / 128 and 1..8 column blocks of 128; R tails of the 128-row tiles."""
    c, X, Wt, bias, ref, bound = sigmoid_dot_case(L, R)
    for presplit in (False, True):
        for lda in (L, L + 3):
            A = _sigmoid_dot(X, Wt, bias, c["att"]["k2"], lda, presplit)
            assert np.isnan(A[R:]).all(), "wrote rows past R"
            assert np.isnan(A[:R, L:]).all(), "wrote columns past len"
            err = np.abs(A[:R, :L] - ref)
            assert (err <= C_LOGIT * bound).all(), (presplit, lda, float((err / bound).max()))


FL_CASES = [(Kp, L) for Kp in (4, 36, 100, 128) for L in (1, 32, 33, 64)]


def from_logits_case(Kp, L, N=1001):
    c = make_user_case(3 * Kp + L, Kp, L, 300)
    rng = np.random.default_rng(Kp + 100 * L)
    X = c["G"][:N] if N <= c["n_items"] else rng.standard_normal((N, Kp)).astype(F32)
    Wt, bias = user_weights_f32(c["G"], c["seq"], L, c["att"])
    A32 = logits_ref(X, Wt, bias, c["att"]["k2"])[0].astype(F32)
    keys = c["G"][c["seq"][:L]].astype(F64)
    ref, bound = from_logits_ref(A32, keys, L, c["att"]["b2"], Kp)
    return c, A32, ref, bound


@pytest.mark.parametrize("Kp,L", FL_CASES)
def test_din_attention_from_logits_matches_fp64(Kp, L):
    import torch

    from librecommender_b200 import _lib

    N = 1001                                                            # not a multiple of the 8 warps per CTA
    c, A32, ref, bound = from_logits_case(Kp, L, N)
    Ad, Gd, sd = _dev(A32), _dev(c["G"]), _dev(c["seq"])
    out = torch.full((N, Kp + 2), float("nan"), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.b200_din_attention_from_logits(_lib.ptr(Ad), Ad.stride(0), N, _lib.ptr(Gd), Gd.stride(0), Kp,
                                                       _lib.ptr(sd), L, float(c["att"]["b2"]), _lib.ptr(out),
                                                       out.stride(0), _lib.current_stream()))
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert np.isnan(o[:, Kp:]).all()
    _check_rows(o[:, :Kp], ref, C_ATT * bound, np.full(N, L), "from_logits")


def chain_case(Kp, L=40, N=5003):
    """One user with L keys over an N-item table; reference = the paper attention with q = every item, float64."""
    from oracle import tf_models as tm

    c = make_user_case(5 * Kp, Kp, L, N)
    G64 = c["G"].astype(F64)
    keys = G64[c["seq"][:L]]
    ref = np.empty((N, Kp))
    bound = np.empty(N)
    lens = np.full(N, L)
    for s in range(0, N, 256):
        q = G64[s:min(s + 256, N)]
        kb = np.broadcast_to(keys[None], (len(q), L, Kp))
        ref[s:s + 256] = tm.din_attention(q, kb, lens[:len(q)], att64(c["att"]), dtype=F64)
        bound[s:s + 256] = paper_bound(q, kb, lens[:len(q)], c["att"])
    return c, ref, bound


def chain_f32(c, N):
    """float32 CPU model of the chain: user weights, 3xTF32 GEMM, sigmoid / Dense(1) / softmax / key sum."""
    L, Kp = c["L"], c["Kp"]
    Wt, bias = user_weights_f32(c["G"], c["seq"], L, c["att"])
    Z = linear_3xtf32_f32(c["G"][:N], Wt, bias)
    return hoisted_f32(Z, c["G"][c["seq"][:L]], L, c["att"])


@pytest.mark.parametrize("Kp", [32, 64, 128])
def test_din_all_items_chain_matches_paper_attention(Kp):
    import torch

    from librecommender_b200 import _lib

    N, L = 5003, 40
    c, ref, bound = chain_case(Kp, L, N)
    st = _lib.current_stream()
    Gd, sd = _dev(c["G"]), _dev(c["seq"])
    k1, b1, k2 = (_dev(c["att"][k]) for k in ("k1", "b1", "k2"))
    b2 = float(c["att"]["b2"])
    Gn = Gd[:N]
    Wt = torch.empty((16 * L, Kp), dtype=torch.float32, device="cuda")
    bias = torch.empty(16 * L, dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.b200_din_user_weights(_lib.ptr(Gd), Gd.stride(0), Kp, _lib.ptr(sd), L, _lib.ptr(k1), _lib.ptr(b1),
                                              _lib.ptr(Wt), Wt.stride(0), _lib.ptr(bias), st))
    # fused: logits in the GEMM epilogue, then the softmax / key sum
    A = torch.empty((N, L), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.b200_linear_tf32x3_sigmoid_dot(_lib.ptr(Gn), Gn.stride(0), N, _lib.ptr(Wt), Wt.stride(0), None,
                                                       _lib.ptr(bias), Kp, 16 * L, _lib.ptr(k2), _lib.ptr(A), A.stride(0),
                                                       st))
    fused = torch.empty((N, Kp), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.b200_din_attention_from_logits(_lib.ptr(A), A.stride(0), N, _lib.ptr(Gd), Gd.stride(0), Kp,
                                                       _lib.ptr(sd), L, b2, _lib.ptr(fused), fused.stride(0), st))
    # unfused: pre-activations Z, then the hoisted kernel
    Z = torch.empty((N, 16 * L), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.b200_linear_tf32x3(_lib.ptr(Gn), Gn.stride(0), N, _lib.ptr(Wt), Wt.stride(0), None, _lib.ptr(bias),
                                           Kp, 16 * L, 0, _lib.ptr(Z), Z.stride(0), st))
    unfused = torch.empty((N, Kp), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.b200_din_attention_hoisted(_lib.ptr(Z), Z.stride(0), N, _lib.ptr(Gd), Gd.stride(0), Kp,
                                                   _lib.ptr(sd), L, _lib.ptr(k2), b2, _lib.ptr(unfused),
                                                   unfused.stride(0), st))
    torch.cuda.synchronize()
    for name, got in (("fused", fused), ("unfused", unfused)):
        _check_rows(got.cpu().numpy(), ref, C_CHAIN * bound, np.full(N, L), name)


# ----- backward ----------------------------------------------------------------------------------------------------------
BWD_CASES = [(Kp, T) for Kp in (4, 30, 64, 96, 128) for T in (1, 32, 33, 64)]


@pytest.mark.parametrize("Kp,T", BWD_CASES)
def test_din_attention_backward_matches_autograd(Kp, T):
    import torch

    from librecommender_b200 import _lib

    c = make_bwd_case(Kp * 100 + T, Kp, T)
    ref = bwd_autograd(c, torch.float64)
    mag = bwd_magnitudes(c)
    R = len(c["row_pair"])
    users = _dev(c["p_user"][c["row_pair"]])
    items = _dev(c["p_item"][c["row_pair"]])
    Gd, sd, ld, dd = _dev(c["G"]), _dev(c["seqs"]), _dev(c["lens"]), _dev(c["dout"])
    k1, b1, k2 = (_dev(c["att"][k]) for k in ("k1", "b1", "k2"))
    pre = {"dG": 0.5, "k1": -0.25, "b1": 0.125, "k2": 1.5, "b2": -2.0}         # the kernel ADDS into its outputs
    outs = {k: torch.full(ref[k].shape, v, dtype=torch.float32, device="cuda") for k, v in pre.items()}
    _lib.check(_lib.lib.b200_din_attention_backward(
        _lib.ptr(Gd), Gd.stride(0), Kp, _lib.ptr(items), _lib.ptr(sd), sd.stride(0), _lib.ptr(ld), T, _lib.ptr(users), R,
        _lib.ptr(k1), _lib.ptr(b1), _lib.ptr(k2), float(c["att"]["b2"]), _lib.ptr(dd), dd.stride(0), _lib.ptr(outs["dG"]),
        outs["dG"].stride(0), _lib.ptr(outs["k1"]), _lib.ptr(outs["b1"]), _lib.ptr(outs["k2"]), _lib.ptr(outs["b2"]),
        _lib.current_stream()))
    torch.cuda.synchronize()
    for k, v in pre.items():
        got = outs[k].cpu().numpy()
        want = v + ref[k]
        bound = C_BWD * U * mag[k] + 2 * U * (abs(v) + np.abs(want))
        err = np.abs(got - want)
        assert (err <= bound).all(), (k, float((err / bound).max()), float(err.max()))


# ----- host-side rejections --------------------------------------------------------------------------------------------
def test_host_rejects_bad_shapes():
    import torch

    from librecommender_b200 import _lib

    lib, st = _lib.lib, _lib.current_stream()
    G = torch.zeros((8, 132), device="cuda")
    seqs = torch.zeros((2, 300), dtype=torch.int32, device="cuda")
    lens = torch.ones(2, dtype=torch.int32, device="cuda")
    ids = torch.zeros(2, dtype=torch.int64, device="cuda")
    w = torch.zeros(4 * 132 * 16 + 16, device="cuda")
    out = torch.zeros((2, 132), device="cuda")
    big = torch.zeros((16 * 300, 132), device="cuda")
    P = _lib.ptr

    def fwd(Kp, T, k1=w):
        return lib.b200_din_attention(P(G), G.stride(0), Kp, P(ids), P(seqs), seqs.stride(0), P(lens), T, P(ids), 2, 0, 0,
                                      P(k1), P(w), P(w), 0.0, P(out), out.stride(0), st)

    def bwd(Kp, T):
        return lib.b200_din_attention_backward(P(G), G.stride(0), Kp, P(ids), P(seqs), seqs.stride(0), P(lens), T, P(ids),
                                               2, P(w), P(w), P(w), 0.0, P(out), out.stride(0), P(big), big.stride(0),
                                               P(w), P(w), P(w), P(w), st)

    for Kp in (0, 129):
        assert fwd(Kp, 4) != 0 and fwd(Kp, 4, k1=None) != 0 and bwd(Kp, 4) != 0
    for T in (0, 257):
        assert fwd(16, T) != 0 and fwd(16, T, k1=None) != 0
    assert bwd(16, 0) != 0 and bwd(16, 65) != 0
    assert lib.b200_din_attention_from_logits(P(out), 70, 2, P(G), G.stride(0), 16, P(seqs), 65, 0.0, P(out),
                                              out.stride(0), st) != 0
    assert lib.b200_din_attention_hoisted(P(big), 16 * 257, 2, P(G), G.stride(0), 16, P(seqs), 257, P(w), 0.0, P(out),
                                          out.stride(0), st) != 0
    assert lib.b200_din_user_weights(P(G), G.stride(0), 16, P(seqs), 257, P(w), P(w), P(big), big.stride(0), P(w),
                                     st) != 0
    X = torch.zeros((256, 32), device="cuda")
    assert lib.b200_linear_tf32x3_sigmoid_dot(P(X), 32, 256, P(big), big.stride(0), None, None, 32, 24, P(w), P(out),
                                              out.stride(0), st) != 0
    torch.cuda.synchronize()
    assert (out == 0).all() and (big == 0).all()                        # nothing was launched


# ----- sequence pooling, all-items grid -------------------------------------------------------------------------------
def pool_case(d, n_items=60, n_users=9, T=11, N=17, off=6):
    rng = np.random.default_rng(d)
    E = rng.standard_normal((n_items + 1, d)).astype(F32)
    lens = rng.integers(0, T + 1, n_users).astype(np.int32)
    lens[:2] = [0, T]
    seqs = np.full((n_users, T), n_items, dtype=np.int32)
    for u in range(n_users):
        seqs[u, :lens[u]] = rng.integers(0, n_items, lens[u])
    users = rng.permutation(n_users).astype(np.int64)
    R = n_users * N - off - 4
    sr = users[(np.arange(R) + off) // N]
    Ez = E.astype(F64)
    Ez[n_items] = 0.0
    inv = np.where(lens > 0, 1.0 / np.sqrt(np.maximum(lens, 1)), 0.0)
    ref = Ez[seqs].sum(axis=1) * inv[:, None]
    mag = np.abs(Ez)[seqs].sum(axis=1) * inv[:, None]
    return E, seqs, lens, users, R, N, off, ref[sr], mag[sr] * (T + 2) * U


@pytest.mark.parametrize("d", [1, 33, 100])
def test_seq_pool_grid_mode(d):
    import torch

    from librecommender_b200 import _lib

    E, seqs, lens, users, R, N, off, ref, bound = pool_case(d)
    Ed, sd, ld, ud = _dev(E), _dev(seqs), _dev(lens), _dev(users)
    out = torch.full((R, d + 2), float("nan"), dtype=torch.float32, device="cuda")
    _lib.check(_lib.lib.b200_seq_pool(_lib.ptr(Ed), Ed.stride(0), d, E.shape[0] - 1, _lib.ptr(sd), sd.stride(0),
                                      _lib.ptr(ld), seqs.shape[1], _lib.ptr(ud), R, N, off, _lib.ptr(out), out.stride(0),
                                      _lib.current_stream()))
    torch.cuda.synchronize()
    o = out.cpu().numpy()
    assert np.isnan(o[:, d:]).all()
    assert (np.abs(o[:, :d] - ref) <= C_POOL * bound).all()
