"""Host restatements for tests/test_gpu_seq_pair_kernels.py and tests/test_seq_pair_kernels_cpu.py (numpy only).

Each all-items scorer of the sequence models is restated from its C ABI, on arrays in the kernel's own layouts:

* ``b200_transformer_pair_scores`` / ``b200_transformer_target_attention`` (``csrc/transformer.cu``): per (b, n) with
  len = clamp(lens[b], 0, T) and nk = len if len > 0 else T, the logits Qi[n] . S[b, t] over the nk keys (each shifted
  as fl32(logit - 1e9) when len = 0), their softmax p, then either s_u = sum_t p_t S[b, t] (rows) or
  h1 = swish(Pu[b] + Pi[n] + sum_t p_t Vp[b, t]), h2 = h1 W2 and the head (pair).
* ``b200_sim_pair_scores`` / ``b200_sim_attention`` (``csrc/sim.cu``): the GSU selection by (score desc, position asc)
  of q . Gp[long_t] (NaN -> -inf, -1e9 past llen), the ESU heads over the selection, the short attention, then either
  [o Wo || s] (rows) or relu(Pu + PiT[:, n] + [o || s] W_att), h2 = h1 W2 and the head (pair).
* ``b200_autoint_grid`` / ``b200_autoint_rows`` (``csrc/autoint.cu``): L layers of field self-attention on the block
  assembled through ``field_map``, then Dense(1) on the flat block.

The head of both pair kernels: H3 > 0: out = b_out + sum_j (act(h2 + b2) W3 + b3)_j w_out_j; H3 = 0:
out = b_out + sum_j (h2 + b2)_j w_out_j (no activation on the last hidden layer).

Every ``*_ref`` returns the float64 result and a magnitude ``mag`` such that the kernel's float32 result is within
C * U * mag per element.  ``mag`` is a first-order propagation of absolute values: a k-term dot costs k |x||y|, the
softmax Jacobian maps logit errors d_t to p_t (d_t + sum_u p_u d_u), swish' <= 1.1 and relu' <= 1, |W| carries the
magnitudes through the layers, and every rounded step adds its own |value| times the length of its chain.  Masked
logits contribute no error: the test data keeps them below 32 in magnitude, where fl32(x - 1e9) is exactly -1e9.

The ``*_f32`` functions restate the kernels' float32 operations in their order (``fma32`` chains) for the bound
calibration only; their ``mutant`` argument gives the subtly wrong variants the CPU test shows the bounds reject.
"""
from __future__ import annotations

import numpy as np

from _autoint_oracle import mha_keras
from _rank_kernels_ref import U, fma32  # noqa: F401  (U: the unit roundoff every bound is written in)

F32, F64 = np.float32, np.float64
NEG = 1.0e9
MASKED_LOGIT_LIMIT = 32.0        # |x| < 32: fl32(x - 1e9) == -1e9 (the float32 spacing at 1e9 is 64)
TP_KCH = 32                      # the Transformer pair kernel's Qi / Pi chunk width


def _softmax(l):
    e = np.exp(l - l.max(axis=-1, keepdims=True))
    return e / e.sum(axis=-1, keepdims=True)


def _softmax_mag(p, l, d):
    """Error magnitude of the float32 softmax: logit errors d (in units of U), the rounded l - max, exp and division,
    and a sequential sum over the last axis."""
    nk = l.shape[-1]
    shift = np.abs(l - l.max(axis=-1, keepdims=True))
    e = d + shift + 2.0
    return p * (e + (p * e).sum(axis=-1, keepdims=True) + nk + 2.0)


def _head(h2, b2, W3, b3, w_out, b_out, m2, act, dact):
    """The pair kernels' head on h2 [n, H2] (without b2) and its magnitude m2."""
    H2 = h2.shape[1]
    if W3 is not None and W3.shape[1] > 0:
        z = h2 + b2
        v = act(z)
        mv = dact * (m2 + np.abs(h2) + np.abs(b2)) + 4.0 * np.abs(v)
        h3 = v @ W3
        mh3 = mv @ np.abs(W3) + H2 * (np.abs(v) @ np.abs(W3))
        y = h3 + b3
        out = b_out + y @ w_out
        m = (mh3 + np.abs(h3) + np.abs(b3)) @ np.abs(w_out) + (W3.shape[1] + 2) * (np.abs(y) @ np.abs(w_out) + abs(b_out))
    else:
        y = h2 + b2
        out = b_out + y @ w_out
        m = (m2 + np.abs(h2) + np.abs(b2)) @ np.abs(w_out) + (H2 + 2) * (np.abs(y) @ np.abs(w_out) + abs(b_out))
    return out, m


def _swish(x):
    return x / (1.0 + np.exp(-x))


def _relu(x):
    return np.maximum(x, 0.0)


# ===================================================================================================================
# Transformer
# ===================================================================================================================
def tfm_nk(len_raw, T):
    ln = min(max(int(len_raw), 0), T)
    return ln, (ln if ln > 0 else T)


def tfm_attention_ref(q, Sb, len_raw):
    """q [n, D], Sb [T, D] of one slot: (p [n, nk], mag_p [n, nk], logits, nk) in float64."""
    T, D = Sb.shape
    ln, nk = tfm_nk(len_raw, T)
    s = Sb[:nk].astype(F64)
    q = q.astype(F64)
    l = q @ s.T
    if ln == 0:
        assert np.abs(l).max() < MASKED_LOGIT_LIMIT, "masked logits must stay below 32 in magnitude"
        l = (l - NEG).astype(F32).astype(F64)              # == -1e9 exactly: uniform weights
        d = np.zeros_like(l)
    else:
        d = D * (np.abs(q) @ np.abs(s).T)
    p = _softmax(l)
    return p, _softmax_mag(p, l, d), l, nk


def tfm_pair_ref(c, b, items):
    """float64 b200_transformer_pair_scores for user b and the items ``items``: (out [n], mag [n])."""
    T, D, H1 = c["T"], c["D"], c["H1"]
    p, mp, _, nk = tfm_attention_ref(c["Qi"][items, :D], c["S"][b], c["lens"][b])
    V = c["Vp"][b, :nk].astype(F64)
    Pu, Pi = c["Pu"][b].astype(F64), c["Pi"][items, :H1].astype(F64)
    m = p @ V
    z = Pu + Pi + m
    mz = 2.0 * (np.abs(Pu) + np.abs(Pi) + np.abs(m)) + mp @ np.abs(V) + nk * (p @ np.abs(V))
    h1 = _swish(z)
    mh1 = 1.1 * mz + 4.0 * np.abs(h1)
    W2 = c["W2"].astype(F64)
    h2 = h1 @ W2
    m2 = mh1 @ np.abs(W2) + H1 * (np.abs(h1) @ np.abs(W2))
    W3 = c["W3"].astype(F64) if c["H3"] else None
    b3 = c["b3"].astype(F64) if c["H3"] else None
    return _head(h2, c["b2"].astype(F64), W3, b3, c["w_out"].astype(F64), float(c["b_out"]), m2, _swish, 1.1)


def tfm_rows_ref(Qi, S, lens, slots, items):
    """float64 b200_transformer_target_attention rows: s_u [n, D] and its magnitude."""
    D = S.shape[2]
    out = np.zeros((len(slots), D))
    mag = np.zeros((len(slots), D))
    for sl in np.unique(slots):
        r = np.nonzero(slots == sl)[0]
        p, mp, _, nk = tfm_attention_ref(Qi[items[r], :D], S[sl], lens[sl])
        Sv = S[sl, :nk].astype(F64)
        out[r] = p @ Sv
        mag[r] = mp @ np.abs(Sv) + (nk + 2) * (p @ np.abs(Sv))
    return out, mag


def _f32_softmax(l, all_masked, n_keys):
    """The pair kernel's softmax on float32 logits [n, nk]: max, expf, an ascending sum, a division."""
    l = l[:, :n_keys].copy()
    if all_masked:
        l = l - F32(NEG)
    mx = l.max(axis=1, keepdims=True)
    e = np.exp(l - mx).astype(F32)
    s = np.zeros(len(l), F32)
    for t in range(n_keys):
        s = s + e[:, t]
    return (e / s[:, None]).astype(F32)


def tfm_pair_f32(c, b, items, mutant=None):
    """The pair kernel's float32 operations in its order.  Mutants: ``nk_minus_1`` (softmax over nk - 1 keys),
    ``len_unclamped`` (len used as given: negative lengths neither clamp to 0 nor mask), ``drop_last_pi_chunk`` (the
    last 32-column Pi chunk of the tile never added), ``pu_twice`` (Pu added twice)."""
    T, D, H1, H2, H3 = c["T"], c["D"], c["H1"], c["H2"], c["H3"]
    f = lambda k: np.asarray(c[k], F32)  # noqa: E731
    q, Sb, V = f("Qi")[items, :D], f("S")[b], f("Vp")[b]
    ln, nk = tfm_nk(c["lens"][b], T)
    all_masked = ln == 0
    if mutant == "len_unclamped":
        ln_raw = int(c["lens"][b])
        nk = min(ln_raw, T) if ln_raw > 0 else T
        all_masked = ln_raw == 0
    l = np.zeros((len(items), nk), F32)
    for d in range(D):
        l = fma32(q[:, d:d + 1], Sb[None, :nk, d], l)
    n_soft = nk - 1 if mutant == "nk_minus_1" and nk > 1 else nk
    p = np.zeros((len(items), nk), F32)
    p[:, :n_soft] = _f32_softmax(l, all_masked, n_soft)
    m = np.zeros((len(items), H1), F32)
    for t in range(nk):
        m = fma32(p[:, t:t + 1], V[None, t, :H1], m)
    Pu = f("Pu")[b, :H1]
    Pi = f("Pi")[items, :H1].copy()
    if mutant == "drop_last_pi_chunk":
        Pi[:, (H1 - 1) // TP_KCH * TP_KCH:] = 0
    if mutant == "pu_twice":
        Pu = Pu + Pu
    z = (Pu + Pi) + m
    h1 = (z / (F32(1) + np.exp(-z))).astype(F32)
    W2 = f("W2")
    h2 = np.zeros((len(items), H2), F32)
    for k in range(H1):
        h2 = fma32(h1[:, k:k + 1], W2[None, k], h2)
    out = np.full(len(items), F32(c["b_out"]), F32)
    b2, wo = f("b2"), f("w_out")
    if H3 > 0:
        zz = h2 + b2
        v = (zz / (F32(1) + np.exp(-zz))).astype(F32)
        W3, b3 = f("W3"), f("b3")
        for j in range(H3):
            h3 = np.zeros(len(items), F32)
            for k in range(H2):
                h3 = fma32(v[:, k], W3[k, j], h3)
            out = fma32(h3 + b3[j], wo[j], out)
    else:
        for j in range(H2):
            out = fma32(h2[:, j] + b2[j], wo[j], out)
    return out


def tfm_rows_f32(Qi, S, lens, b, items):
    """The rows kernel's float32 s_u for slot b: logits, softmax, then acc = fmaf(p_t, S[t, d], acc) over t."""
    T, D = S.shape[1:]
    ln, nk = tfm_nk(lens[b], T)
    q, Sb = np.asarray(Qi, F32)[items, :D], np.asarray(S, F32)[b]
    l = np.zeros((len(items), nk), F32)
    for d in range(D):
        l = fma32(q[:, d:d + 1], Sb[None, :nk, d], l)
    p = _f32_softmax(l, ln == 0, nk)
    acc = np.zeros((len(items), D), F32)
    for t in range(nk):
        acc = fma32(p[:, t:t + 1], Sb[None, t], acc)
    return acc


def make_tfm_case(B, N, T, D, H1, H2, H3, seed, lens=None, ldq_pad=0, ldpi_pad=0):
    """Random pair-kernel inputs.  The logits Qi . S have a spread of about 2 (masked ones stay well below 32); Qi
    and Pi carry NaN padding columns past D / H1.  ``lens`` defaults to cycling -3, 0, 1, T, T + 5."""
    rng = np.random.default_rng(seed)
    Qi = np.full((N, D + ldq_pad), np.nan, F32)
    Qi[:, :D] = rng.standard_normal((N, D))
    Pi = np.full((N, H1 + ldpi_pad), np.nan, F32)
    Pi[:, :H1] = rng.normal(0.0, 0.7, (N, H1))
    if lens is None:
        base = [-3, 0, 1, T, T + 5]
        lens = np.array([base[i % 5] if i < 5 else int(rng.integers(-1, T + 2)) for i in range(B)], np.int32)
    c = dict(T=T, D=D, H1=H1, H2=H2, H3=H3, Qi=Qi, Pi=Pi, lens=np.asarray(lens, np.int32),
             S=(rng.standard_normal((B, T, D)) * (2.0 / np.sqrt(D))).astype(F32),
             Vp=rng.normal(0.0, 0.6, (B, T, H1)).astype(F32),
             Pu=rng.normal(0.0, 0.7, (B, H1)).astype(F32),
             W2=rng.normal(0.0, 1.0 / np.sqrt(H1), (H1, H2)).astype(F32),
             b2=rng.normal(0.0, 0.1, H2).astype(F32),
             W3=rng.normal(0.0, 1.0 / np.sqrt(H2), (H2, max(H3, 1)))[:, :H3].copy().astype(F32) if H3 else None,
             b3=rng.normal(0.0, 0.1, H3).astype(F32) if H3 else None,
             w_out=rng.normal(0.0, 0.3, H3 if H3 else H2).astype(F32),
             b_out=float(F32(-0.25)))
    return c


# ===================================================================================================================
# SIM
# ===================================================================================================================
def dyadic(rng, shape, limit=1.0):
    """Multiples of 1/8 with |v| <= limit (<= 2): every dot of up to 64 such products is exact in float32."""
    n = int(round(8 * limit))
    return (rng.integers(-n, n + 1, size=shape) / 8.0).astype(F32)


def sim_lens(c, b):
    return min(max(int(c["long_lens"][b]), 0), c["L"]), min(max(int(c["short_lens"][b]), 0), c["S"])


def gsu_scores(c, b, q):
    """Exact GSU scores [n, L] in float64 (the dots are exact in float32): NaN -> -inf, -1e9 past llen."""
    L, K = c["L"], c["K"]
    llen, _ = sim_lens(c, b)
    g = c["Gp"][c["long_seqs"][b, :L], :K].astype(F64)
    with np.errstate(invalid="ignore"):
        s = q.astype(F64) @ g.T
    s[np.isnan(s)] = -np.inf
    s[:, llen:] = -NEG
    return s


def gsu_select(scores, k, high_ties=False):
    """The top k positions by (score desc, position asc), ascending.  ``high_ties``: ties to the higher position."""
    n, L = scores.shape
    pos = np.broadcast_to(np.arange(L), (n, L))
    key2 = -pos if high_ties else pos
    order = np.lexsort((key2, -scores), axis=-1)[:, :k]
    return np.sort(order, axis=1)


def _sim_core(c, b, items, sel=None):
    """Float64 o [n, K], s [n, K], their magnitudes, and the selection [n, topk] for user b."""
    K, H, S, k = c["K"], c["H"], c["S"], c["topk"]
    hd = K // H
    llen, slen = sim_lens(c, b)
    q = c["Gp"][items, :K].astype(F64)
    if sel is None:
        sel = gsu_select(gsu_scores(c, b, c["Gp"][items, :K]), k)
    n = len(items)
    qp = c["Qp"][items, :K].astype(F64)
    Kl, Vl = c["Kl"][b].astype(F64), c["Vl"][b].astype(F64)
    ks, vs = Kl[sel], Vl[sel]                                    # [n, k, K]
    masked = sel >= llen
    o = np.zeros((n, K))
    mo = np.zeros((n, K))
    sc = 1.0 / np.sqrt(hd)
    for h in range(H):
        cs = slice(h * hd, (h + 1) * hd)
        l = np.einsum("nd,nkd->nk", qp[:, cs], ks[:, :, cs]) * sc
        d = sc * (hd + 2) * np.einsum("nd,nkd->nk", np.abs(qp[:, cs]), np.abs(ks[:, :, cs]))
        if masked.any():
            assert np.abs(l[masked]).max() < MASKED_LOGIT_LIMIT, "masked ESU logits must stay below 32"
            l = np.where(masked, (l - NEG).astype(F32).astype(F64), l)
            d = np.where(masked, 0.0, d)
        p = _softmax(l)
        mp = _softmax_mag(p, l, d)
        o[:, cs] = np.einsum("nk,nkd->nd", p, vs[:, :, cs])
        mo[:, cs] = np.einsum("nk,nkd->nd", mp, np.abs(vs[:, :, cs])) + (k + 2) * np.einsum(
            "nk,nkd->nd", p, np.abs(vs[:, :, cs]))
    g = c["Gp"][c["short_seqs"][b, :S], :K].astype(F64)           # [S, K]
    ls = q @ g.T                                                 # exact
    if slen < S:
        assert np.abs(ls[:, slen:]).max() < MASKED_LOGIT_LIMIT, "masked short logits must stay below 32"
        ls[:, slen:] = (ls[:, slen:] - NEG).astype(F32).astype(F64)
    w = _softmax(ls)
    s = w @ g
    shift = np.abs(ls - ls.max(axis=1, keepdims=True))
    wg = w @ np.abs(g)
    ms = (w * (shift + 2 * S + 6)) @ np.abs(g) + wg * (w * (shift + 2)).sum(axis=1, keepdims=True)
    return o, mo, s, ms, sel


def sim_pair_ref(c, b, items):
    """float64 b200_sim_pair_scores for user b and the items ``items``: (out [n], mag [n])."""
    K, H1 = c["K"], c["H1"]
    o, mo, s, ms, _ = _sim_core(c, b, items)
    x = np.concatenate([o, s], axis=1)
    mx = np.concatenate([mo, ms], axis=1)
    Wa = c["W_att"].astype(F64)
    Pu, Pi = c["Pu"][b].astype(F64), c["PiT"][:H1, items].T.astype(F64)
    a = x @ Wa
    z = Pu + Pi + a
    mz = 2.0 * (np.abs(Pu) + np.abs(Pi)) + mx @ np.abs(Wa) + (2 * K + 2) * (np.abs(x) @ np.abs(Wa))
    h1 = _relu(z)
    W2 = c["W2"].astype(F64)
    h2 = h1 @ W2
    m2 = mz @ np.abs(W2) + H1 * (np.abs(h1) @ np.abs(W2))
    W3 = c["W3"].astype(F64) if c["H3"] else None
    b3 = c["b3"].astype(F64) if c["H3"] else None
    return _head(h2, c["b2"].astype(F64), W3, b3, c["w_out"].astype(F64), float(c["b_out"]), m2, _relu, 1.0)


def sim_rows_ref(c, slots, items):
    """float64 b200_sim_attention rows: ([o Wo || s] [n, 2K], mag, selection [n, topk] ascending)."""
    K = c["K"]
    n = len(slots)
    out, mag = np.zeros((n, 2 * K)), np.zeros((n, 2 * K))
    sel = np.zeros((n, c["topk"]), np.int64)
    Wo = c["Wo"].astype(F64)
    for sl in np.unique(slots):
        r = np.nonzero(slots == sl)[0]
        o, mo, s, ms, se = _sim_core(c, sl, items[r])
        out[r, :K] = o @ Wo
        mag[r, :K] = mo @ np.abs(Wo) + K * (np.abs(o) @ np.abs(Wo))
        out[r, K:], mag[r, K:], sel[r] = s, ms, se
    return out, mag, sel


def _sim_f32_core(c, b, items, mutant=None):
    """Float32 o [n, K] and s [n, K] of the kernels (the ESU over the selection in ascending position order)."""
    K, H, S, k = c["K"], c["H"], c["S"], c["topk"]
    hd = K // H
    f = lambda x: np.asarray(c[x], F32)  # noqa: E731
    llen, slen = sim_lens(c, b)
    n = len(items)
    q = f("Gp")[items, :K]
    sel = gsu_select(gsu_scores(c, b, q), k, high_ties=mutant == "gsu_tie_high")
    g = f("Gp")[c["short_seqs"][b, :S], :K]
    ls = np.zeros((n, S), F32)
    for d in range(K):
        ls = fma32(q[:, d:d + 1], g[None, :, d], ls)
    ls[:, slen:] = ls[:, slen:] - F32(NEG)
    e = np.exp(ls - ls.max(axis=1, keepdims=True)).astype(F32)
    acc = np.zeros((n, K), F32)
    ssum = np.zeros(n, F32)
    for s in range(S):
        ssum = ssum + e[:, s]
        acc = fma32(e[:, s:s + 1], g[None, s], acc)
    sv = (acc / ssum[:, None]).astype(F32)
    qp, Kl, Vl = f("Qp")[items, :K], f("Kl")[b], f("Vl")[b]
    scale = F32(1) / np.sqrt(F32(hd))
    masked = (np.arange(k)[None, :] >= llen) if mutant == "esu_mask_rank" else (sel >= llen)
    masked = np.broadcast_to(masked, sel.shape)
    o = np.zeros((n, K), F32)
    for h in range(H):
        l = np.zeros((n, k), F32)
        for d in range(h * hd, (h + 1) * hd):
            l = fma32(qp[:, d:d + 1], Kl[sel, d], l)
        l = (l * scale).astype(F32)
        l = np.where(masked, l - F32(NEG), l).astype(F32)
        p = _f32_softmax(l, False, k)
        for d in range(h * hd, (h + 1) * hd):
            a = np.zeros(n, F32)
            for i in range(k):
                a = fma32(p[:, i], Vl[sel[:, i], d], a)
            o[:, d] = a
    return o, sv


def sim_rows_f32(c, b, items, mutant=None):
    """The rows kernel's float32 [o Wo || s] for user b."""
    o, sv = _sim_f32_core(c, b, items, mutant)
    Wo = np.asarray(c["Wo"], F32)
    lo = np.zeros_like(o)
    for d in range(c["K"]):
        lo = fma32(o[:, d:d + 1], Wo[None, d], lo)
    return np.concatenate([lo, sv], axis=1)


def sim_pair_f32(c, b, items, mutant=None):
    """The pair kernel's float32 operations in its order.  Mutants: ``gsu_tie_high`` (GSU ties to the higher
    position), ``esu_mask_rank`` (the ESU mask applied to the i-th selected key when i >= llen instead of when its
    position is >= llen)."""
    K, H1, H2, H3 = c["K"], c["H1"], c["H2"], c["H3"]
    f = lambda x: np.asarray(c[x], F32)  # noqa: E731
    n = len(items)
    o, sv = _sim_f32_core(c, b, items, mutant)
    x = np.concatenate([o, sv], axis=1)
    Wa = f("W_att")
    m = np.zeros((n, H1), F32)
    for cc in range(2 * K):
        m = fma32(x[:, cc:cc + 1], Wa[None, cc], m)
    h1 = np.maximum((f("Pu")[b] + f("PiT")[:H1, items].T) + m, F32(0))
    W2 = f("W2")
    h2 = np.zeros((n, H2), F32)
    for kk in range(H1):
        h2 = fma32(h1[:, kk:kk + 1], W2[None, kk], h2)
    out = np.full(n, F32(c["b_out"]), F32)
    b2, wo = f("b2"), f("w_out")
    if H3 > 0:
        v = np.maximum(h2 + b2, F32(0))
        W3, b3 = f("W3"), f("b3")
        for j in range(H3):
            h3 = np.zeros(n, F32)
            for kk in range(H2):
                h3 = fma32(v[:, kk], W3[kk, j], h3)
            out = fma32(h3 + b3[j], wo[j], out)
    else:
        for j in range(H2):
            out = fma32(h2[:, j] + b2[j], wo[j], out)
    return out


def make_sim_case(B, N, K, H, L, S, topk, H1, H2, H3, seed, pad=3):
    """Random pair / rows kernel inputs on a table of N + 12 items (queries are items 0 .. N-1).

    Gp is dyadic (every GSU and short dot exact); Qp, Kl, Vl and the MLP are ordinary floats.  The last table row is
    NaN: it sits in the long sequences of users 1 and 3 and is never a query or a short item.  Long lengths cycle
    0, 1, topk - 3, L; short lengths 0, S.  Users 2 and 3 draw their long items from a pool of 3, so the GSU has exact
    ties at the cut.  Tables carry ``pad`` NaN columns (``ldt`` = N + pad for the transposed ones)."""
    rng = np.random.default_rng(seed)
    NT = N + 12
    nan_item = NT - 1
    Gp = np.full((NT, K + pad), np.nan, F32)
    Gp[:, :K] = dyadic(rng, (NT, K), 1.0 if K <= 32 else 0.75)
    Gp[nan_item, :K] = np.nan
    Qp = np.full((NT, K + pad), np.nan, F32)
    Qp[:, :K] = rng.normal(0.0, 1.0, (NT, K)) / np.sqrt(K) * 2.0
    GpT = np.full((K, N + pad), np.nan, F32)
    GpT[:, :N] = Gp[:N, :K].T
    QpT = np.full((K, N + pad), np.nan, F32)
    QpT[:, :N] = Qp[:N, :K].T
    long_seqs = np.full((B, L + pad), -1, np.int32)
    long_seqs[:, :L] = rng.integers(0, NT - 1, (B, L))
    short_seqs = np.full((B, S + pad), -1, np.int32)
    short_seqs[:, :S] = rng.integers(0, NT - 1, (B, S))
    ll_cycle = [0, 1, max(topk - 3, 1), L]
    long_lens = np.array([ll_cycle[i % 4] if i < 8 else int(rng.integers(1, L + 1)) for i in range(B)], np.int32)
    short_lens = np.array([(0 if i % 2 == 0 else S) if i < 8 else int(rng.integers(0, S + 1)) for i in range(B)],
                          np.int32)
    for u in (2, 3):
        if u < B:
            pool = rng.integers(0, NT - 1, 3)
            long_seqs[u, :L] = pool[rng.integers(0, 3, L)]
    for u, t in ((1, 0), (3, L // 2)):
        if u < B:
            long_seqs[u, t] = nan_item
    if B > 1:
        long_lens[1] = max(topk - 3, 2)                              # the NaN item inside fewer valid keys than topk
    d = 2 * K
    c = dict(K=K, H=H, L=L, S=S, topk=topk, H1=H1, H2=H2, H3=H3, N=N, Gp=Gp, Qp=Qp, GpT=GpT, QpT=QpT,
             long_seqs=long_seqs, long_lens=long_lens, short_seqs=short_seqs, short_lens=short_lens,
             Kl=rng.normal(0.0, 1.0, (B, L, K)).astype(F32),
             Vl=rng.normal(0.0, 1.0, (B, L, K)).astype(F32),
             Wo=rng.normal(0.0, 1.0 / np.sqrt(K), (K, K)).astype(F32),
             Pu=rng.normal(0.0, 0.5, (B, H1)).astype(F32),
             W_att=rng.normal(0.0, 1.0 / np.sqrt(d), (d, H1)).astype(F32),
             W2=rng.normal(0.0, 1.0 / np.sqrt(H1), (H1, H2)).astype(F32),
             b2=rng.normal(0.0, 0.1, H2).astype(F32),
             W3=rng.normal(0.0, 1.0 / np.sqrt(H2), (H2, max(H3, 1)))[:, :H3].copy().astype(F32) if H3 else None,
             b3=rng.normal(0.0, 0.1, H3).astype(F32) if H3 else None,
             w_out=rng.normal(0.0, 0.3, H3 if H3 else H2).astype(F32),
             b_out=float(F32(0.125)))
    PiT = np.full((H1, N + pad), np.nan, F32)
    PiT[:, :N] = rng.normal(0.0, 0.5, (H1, N))
    c["PiT"] = PiT
    return c


def gsu_ties_at_cut(c, b, items):
    """Items (of ``items``) whose float64 GSU scores tie across the top-k cut for user b."""
    s = gsu_scores(c, b, c["Gp"][items, :c["K"]])
    sel = gsu_select(s, c["topk"])
    kth = np.take_along_axis(s, sel, 1).min(axis=1)
    chosen = np.zeros_like(s, bool)
    np.put_along_axis(chosen, sel, True, 1)
    return ((s == kth[:, None]) & ~chosen).any(axis=1)


# ===================================================================================================================
# AutoInt
# ===================================================================================================================
def autoint_weights(rng, K, H, hds, w_scale=1.0):
    """Packed per-layer [Wq, Wk, Wv (K, D), Wo (D, K)] with D = H * hd, and the same as mha_keras layer dicts."""
    flat, layers = [], []
    for hd in hds:
        D = H * hd
        Wq, Wk, Wv = (rng.normal(0.0, w_scale / np.sqrt(K), (K, D)).astype(F32) for _ in range(3))
        Wo = rng.normal(0.0, 1.0 / np.sqrt(D), (D, K)).astype(F32)
        flat += [Wq.ravel(), Wk.ravel(), Wv.ravel(), Wo.ravel()]
        layers.append(dict(query=Wq.reshape(K, H, hd), key=Wk.reshape(K, H, hd), value=Wv.reshape(K, H, hd),
                           attention_output=Wo.reshape(H, hd, K)))
    return np.concatenate(flat).astype(F32), layers


def autoint_block(Xu, Xi, field_map, K, users, items):
    """The [n, F, K] block the grid kernel assembles for the pairs (users[i], items[i])."""
    F = len(field_map)
    X = np.empty((len(users), F, K), F32)
    for f, m in enumerate(field_map):
        X[:, f] = Xu[users, m * K:(m + 1) * K] if m >= 0 else Xi[items, (-1 - m) * K:(-m) * K]
    return X


def autoint_ref(X, layers, w_out, b_out, residual):
    """float64 autoint_pair on blocks X [n, F, K] (mha_keras per layer): (logit [n], mag [n])."""
    x = X.astype(F64)
    n, F, K = x.shape
    mx = np.zeros_like(x)
    for lw in layers:
        lw64 = {k: np.asarray(v, F64) for k, v in lw.items()}
        H, hd = lw64["query"].shape[1:]
        y = mha_keras(x, lw64, F64)
        # magnitudes: projections, logits, softmax, mix, output map
        ax = np.abs(x)
        q, k, v = (np.einsum("rfk,khd->rfhd", x, lw64[m]) for m in ("query", "key", "value"))
        mq, mk, mv = (np.einsum("rfk,khd->rfhd", mx, np.abs(lw64[m])) + K * np.einsum("rfk,khd->rfhd", ax,
                      np.abs(lw64[m])) for m in ("query", "key", "value"))
        sc = 1.0 / np.sqrt(hd)
        l = np.einsum("rfhd,rghd->rhfg", q, k) * sc
        dl = sc * ((hd + 2) * np.einsum("rfhd,rghd->rhfg", np.abs(q), np.abs(k))
                   + np.einsum("rfhd,rghd->rhfg", mq, np.abs(k)) + np.einsum("rfhd,rghd->rhfg", np.abs(q), mk))
        p = _softmax(l)
        mp = _softmax_mag(p, l, dl)
        o = np.einsum("rhfg,rghd->rfhd", p, v)
        mo = (np.einsum("rhfg,rghd->rfhd", mp, np.abs(v)) + np.einsum("rhfg,rghd->rfhd", p, mv)
              + F * np.einsum("rhfg,rghd->rfhd", p, np.abs(v)))
        Wo = np.abs(lw64["attention_output"])
        my = np.einsum("rfhd,hdk->rfk", mo, Wo) + H * hd * np.einsum("rfhd,hdk->rfk", np.abs(o), Wo)
        x_new = x + y if residual else y
        mx = (mx + my + np.abs(x_new)) if residual else my
        x = x_new
    flat, mflat = x.reshape(n, -1), mx.reshape(n, -1)
    w = np.asarray(w_out, F64)
    out = flat @ w + b_out
    mag = mflat @ np.abs(w) + (F * K + 2) * (np.abs(flat) @ np.abs(w) + abs(b_out))
    return out, mag


def autoint_f32(X, layers, w_out, b_out, residual):
    """The kernel's float32 operations in its order (one fmaf chain per output, ascending index)."""
    x = np.asarray(X, F32).copy()
    n, F, K = x.shape
    for lw in layers:
        H, hd = lw["query"].shape[1:]
        D = H * hd
        W = [np.asarray(lw[m], F32).reshape(K, D) for m in ("query", "key", "value")]
        Q, Kt, V = (np.zeros((n, F, D), F32) for _ in range(3))
        for dst, Wm in zip((Q, Kt, V), W):
            for kk in range(K):
                dst[:] = fma32(x[:, :, kk:kk + 1], Wm[None, None, kk], dst)
        scale = F32(1) / np.sqrt(F32(hd))
        O = np.zeros((n, F, D), F32)
        for h in range(H):
            cs = slice(h * hd, (h + 1) * hd)
            l = np.zeros((n, F, F), F32)
            for j in range(cs.start, cs.stop):
                l = fma32(Q[:, :, None, j], Kt[:, None, :, j], l)
            l = (l * scale).astype(F32)
            e = np.exp(l - l.max(axis=2, keepdims=True)).astype(F32)
            s = np.zeros((n, F), F32)
            for g in range(F):
                s = s + e[:, :, g]
            p = (e / s[:, :, None]).astype(F32)
            for g in range(F):
                O[:, :, cs] = fma32(p[:, :, g:g + 1], V[:, None, g, cs], O[:, :, cs])
        Wo = np.asarray(lw["attention_output"], F32).reshape(D, K)
        y = np.zeros((n, F, K), F32)
        for d in range(D):
            y = fma32(O[:, :, d:d + 1], Wo[None, None, d], y)
        x = (x + y).astype(F32) if residual else y
    flat = x.reshape(n, -1)
    w = np.asarray(w_out, F32)
    acc = np.zeros(n, F32)
    for i in range(F * K):
        acc = fma32(flat[:, i], w[i], acc)
    return (acc + F32(b_out)).astype(F32)
