"""Host restatements for tests/test_gpu_seq_encoder_kernels.py and tests/test_seq_encoder_kernels_cpu.py (numpy only).

The sequence encoders' C ABI (include/b200reco.h) restated on arrays in the kernels' own packed layouts:

* RNN4Rec (``csrc/rnn.cu``): layers packed ``W [in, G*H] | U [H, G*H] | bx | bh | gamma | beta``; the training
  forward's six saved tensors per layer (SV_HP, SV_Y, SV_G, SV_X, SV_XH, SV_RS), rows s * T + t; one layer's backward
  through time (dgx, dgh, dln, dlnx).
* Caser (``csrc/conv.cu``): ``W_1 .. W_T ([h, K, nh]) | b_h [T, nh] | Wv [T, nv] | bv [nv]``; the encoder, its
  max-pool argmax and the backward (dX, dW).
* WaveNet: per causal layer ``W [2, C, F] | b [F]``, then ``W1 [F, F] | b1 [F]``; the encoder, the saved layer outputs
  and argmax, and the three position helpers.

Every ``*_checks`` function returns ``(what, got, ref, mag)`` tuples: the kernel's float32 ``got`` is within
``C * U * mag`` of the float64 ``ref`` element by element.  ``mag`` is a first-order propagation of absolute values:
a k-term fmaf chain costs k times the sum of its |terms|, each rounded operation adds its own |value|, and the libm
calls add their documented errors (expf and tanhf 2 ulp, rsqrtf 2 ulp).  Every inexact element's magnitude also
carries a floor of 2^-100 for float32 underflow (a gradient through a long chain of gates can fall below 2^-126).

The references are STEP-LOCAL so that the bounds do not grow with T or with depth: step t of a recurrent layer is
recomputed from the kernel's own float32 state of step t - 1 (SV_HP, LSTM c = SV_X(t - 1)) and the kernel's own
input (the gathered row, or the layer below's SV_Y); a WaveNet layer from the kernel's own output of the layer below;
the backward of step t from the kernel's own gate gradients of step t + 1, carrying only the contractive factor
(z for a GRU, f for the LSTM cell) on the reference's float64 dh / dc with its magnitude.

The ``*_f32`` functions restate the kernels in float32 in their operation order (``fma32`` chains) for the bound
calibration only; their ``mutant`` argument gives the subtly wrong variants the CPU test shows the checks reject.
"""
from __future__ import annotations

import numpy as np

from _rank_kernels_ref import U, fma32  # noqa: F401  (U: the unit roundoff every bound is written in)

F32, F64 = np.float32, np.float64
GRU_KERAS, GRU_TF1, LSTM = 0, 1, 2
ACT_TANH, ACT_LN = 0, 1
LN_EPS = 1e-3
EXP_ULP = TANH_ULP = RSQRT_ULP = 2.0
RNN_MAX_TILE, RNN_UPT = 64, 8
CONV_PB, CONV_MAX_TILE = 4, 32
CONV_CHUNK_ROWS, CONV_PART_FLOATS = 256, 1 << 22
SMEM_TILE_BYTES = 96 * 1024
# every inexact element's magnitude also covers float32 underflow: a product or sum below 2^-126 rounds to a multiple
# of 2^-149, so each operation may lose that much absolutely however small its operands
UNDERFLOW_MAG = 2.0 ** -100
ELEM_BLOCK_CAP, ELEM_THREADS = 132 * 32, 256


def odd(n):
    return n | 1


def gates(kind):
    return 4 if kind == LSTM else 3


# ===================================================================================================================
# RNN4Rec: layouts
# ===================================================================================================================
def rnn_layer_floats(kind, ind, H):
    GH = gates(kind) * H
    return ind * GH + H * GH + 2 * GH + 2 * H


def rnn_layout_floats(in0, kinds, Hs, acts, tile):
    """csrc/rnn.cu rnn_layout: the forward's shared-memory floats for a tile."""
    off = tile * odd(in0)
    for k, H, a in zip(kinds, Hs, acts):
        off += tile * odd(H) * (1 + (k == LSTM) + (a == ACT_LN))
    off += 3 * tile * odd(max(Hs)) + 2 * tile
    off += off & 1
    return off + 4 * tile


def rnn_bwd_layout_floats(kind, H, tile):
    return 4 * tile * odd(H) + tile * odd(gates(kind) * H) + 3 * tile


def _shrink(floats):
    tile = RNN_MAX_TILE
    while tile > RNN_UPT and floats(tile) * 4 > SMEM_TILE_BYTES:
        tile -= RNN_UPT
    return tile, floats(tile) * 4


def rnn_fwd_tile(in0, kinds, Hs, acts):
    """(tile, shared bytes) the host of b200_rnn_encode / b200_rnn_train_forward picks."""
    return _shrink(lambda t: rnn_layout_floats(in0, kinds, Hs, acts, t))


def rnn_bwd_tile(kind, H):
    return _shrink(lambda t: rnn_bwd_layout_floats(kind, H, t))


def rnn_unpack(w, in0, kinds, Hs):
    layers, off = [], 0
    for l, (k, H) in enumerate(zip(kinds, Hs)):
        ind, GH = (in0 if l == 0 else Hs[l - 1]), gates(k) * H
        parts = {}
        for name, m, shape in (("W", ind * GH, (ind, GH)), ("U", H * GH, (H, GH)), ("bx", GH, (GH,)),
                               ("bh", GH, (GH,)), ("gamma", H, (H,)), ("beta", H, (H,))):
            parts[name] = w[off:off + m].reshape(shape)
            off += m
        parts.update(kind=k, H=H, ind=ind)
        layers.append(parts)
    assert off == len(w)
    return layers


def make_rnn_case(n, T, in0, kinds, Hs, acts, seed, lens=None, users=None, ld_seq_pad=0, ldx_pad=0, n_items=40):
    """Seeded data for one encoder: X [n_items + 1, in0 + ldx_pad] (the last row and the pad columns NaN, so a read of
    a pad position or column shows), seqs [rows, T + ld_seq_pad] (pad columns point at the NaN row), raw lens of every
    class, slots ``users`` (permuted and duplicated rows by default) and the packed weights."""
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (n_items + 1, in0 + ldx_pad)).astype(F32)
    X[n_items] = np.nan
    X[:, in0:] = np.nan
    rows = max(n, 4)
    seqs = np.full((rows, T + ld_seq_pad), n_items, np.int32)
    seqs[:, :T] = rng.integers(0, n_items, (rows, T))
    if lens is None:
        classes = [T, 0, 1, T // 2 + 1, -3, T + 5, T - 1 if T > 1 else 1]
        lens = np.array([classes[i % len(classes)] if i < 2 * len(classes) else rng.integers(-2, T + 3)
                         for i in range(rows)], np.int32)
    if users is None:
        users = rng.permutation(np.arange(n) % rows).astype(np.int64)
        if n > 3:
            users[n // 2] = users[1]                                  # a duplicated row
    w = []
    for l, (k, H) in enumerate(zip(kinds, Hs)):
        ind, GH = (in0 if l == 0 else Hs[l - 1]), gates(k) * H
        w += [rng.uniform(-1.5, 1.5, ind * GH) / np.sqrt(ind), rng.uniform(-1.5, 1.5, H * GH) / np.sqrt(H),
              rng.uniform(-0.5, 0.5, GH), rng.uniform(-0.5, 0.5, GH), rng.uniform(0.5, 1.5, H),
              rng.uniform(-0.5, 0.5, H)]
    w = np.concatenate(w).astype(F32)
    return dict(n=n, T=T, in0=in0, kinds=list(kinds), Hs=list(Hs), acts=list(acts), X=X, seqs=seqs, lens=lens,
                users=users, w=w, layers=rnn_unpack(w, in0, kinds, Hs))


def slot_lens(c):
    return np.clip(c["lens"][c["users"]], 0, c["T"]).astype(np.int64)


def _floored(checks):
    return [(w, got, ref, np.where(mag > 0, mag + UNDERFLOW_MAG, 0.0)) for w, got, ref, mag in checks]


def _sig(v):
    return 1.0 / (1.0 + np.exp(-v))


def _sig_mag(s, mv):
    return s * (1.0 - s) * (mv + EXP_ULP) + 2.0 * s


def _act(a, v):
    return np.tanh(v) if a == ACT_TANH else v


def _act_mag(a, y, mv):
    return (1.0 - y * y) * mv + TANH_ULP * np.abs(y) if a == ACT_TANH else mv


# ===================================================================================================================
# RNN4Rec forward: one step in float64 from the kernel's own float32 inputs
# ===================================================================================================================
def rnn_step_ref(lw, act, x, hp, cp=None, rh=None):
    """Step of one layer for rows x [R, in], h_{t-1} [R, H] (float32, the kernel's), LSTM c_{t-1}, TF1 GRU the
    kernel's r o h_{t-1}: dict of float64 values g, xs (the SV_X block), h and their magnitudes."""
    kind, H = lw["kind"], lw["H"]
    W, Uw, bx, bh = (np.asarray(lw[k], F64) for k in ("W", "U", "bx", "bh"))
    x, hp = x.astype(F64), hp.astype(F64)
    ind = W.shape[0]
    axb = x @ W + bx
    max_ = ind * (np.abs(x) @ np.abs(W) + np.abs(bx)) + np.abs(axb)
    if kind == GRU_TF1:
        Uzr = Uw[:, :2 * H]
        ahb = hp @ Uzr + bh[:2 * H]
        mah = H * (np.abs(hp) @ np.abs(Uzr) + np.abs(bh[:2 * H])) + np.abs(ahb)
    else:
        ahb = hp @ Uw + bh
        mah = H * (np.abs(hp) @ np.abs(Uw) + np.abs(bh)) + np.abs(ahb)
    out = {}
    if kind == LSTM:
        v = axb + ahb
        mv = max_ + mah + np.abs(v)
        sl = [slice(i * H, (i + 1) * H) for i in range(4)]
        ig, fg, og = _sig(v[:, sl[0]]), _sig(v[:, sl[1]]), _sig(v[:, sl[3]])
        mi, mf, mo = _sig_mag(ig, mv[:, sl[0]]), _sig_mag(fg, mv[:, sl[1]]), _sig_mag(og, mv[:, sl[3]])
        gg = _act(act, v[:, sl[2]])
        mg = _act_mag(act, gg, mv[:, sl[2]])
        c0 = np.zeros_like(hp) if cp is None else cp.astype(F64)
        cn = fg * c0 + ig * gg
        mc = np.abs(c0) * mf + np.abs(gg) * mi + np.abs(ig) * mg + np.abs(fg * c0) + np.abs(ig * gg) + np.abs(cn)
        ta = _act(act, cn)
        mta = _act_mag(act, ta, mc)
        h = og * ta
        mh = np.abs(ta) * mo + np.abs(og) * mta + np.abs(h)
        out.update(g=np.hstack([ig, fg, gg, og]), mg=np.hstack([mi, mf, mg, mo]), xs=cn, mxs=mc)
    else:
        z = _sig(axb[:, :H] + ahb[:, :H])
        mz = _sig_mag(z, max_[:, :H] + mah[:, :H] + np.abs(axb[:, :H] + ahb[:, :H]))
        r = _sig(axb[:, H:2 * H] + ahb[:, H:2 * H])
        mr = _sig_mag(r, max_[:, H:2 * H] + mah[:, H:2 * H] + np.abs(axb[:, H:2 * H] + ahb[:, H:2 * H]))
        if kind == GRU_KERAS:
            a_c, ma_c = ahb[:, 2 * H:], mah[:, 2 * H:]
            v = axb[:, 2 * H:] + r * a_c
            mv = max_[:, 2 * H:] + np.abs(r) * ma_c + np.abs(a_c) * mr + np.abs(r * a_c) + np.abs(v)
            xs, mxs = ahb[:, 2 * H:], mah[:, 2 * H:]
        else:
            xs = r * hp
            mxs = np.abs(hp) * mr + np.abs(xs)
            rhk = xs if rh is None else rh.astype(F64)                # the kernel's own r o h feeds its chain
            Uc = Uw[:, 2 * H:]
            ac = rhk @ Uc + bh[2 * H:]
            v = axb[:, 2 * H:] + ac
            mv = max_[:, 2 * H:] + H * (np.abs(rhk) @ np.abs(Uc) + np.abs(bh[2 * H:])) + np.abs(ac) + np.abs(v)
        hh = _act(act, v)
        mhh = _act_mag(act, hh, mv)
        h = z * hp + (1.0 - z) * hh
        mh = (np.abs(hp - hh) * mz + np.abs(1.0 - z) * mhh + np.abs(1.0 - z) * np.abs(hh) + np.abs(z * hp)
              + np.abs((1.0 - z) * hh) + np.abs(h))
        out.update(g=np.hstack([z, r, hh]), mg=np.hstack([mz, mr, mhh]), xs=xs, mxs=mxs)
    out.update(h=h, mh=mh)
    return out


def ln_ref(h, mh, gamma, beta, eps=LN_EPS):
    """tanh(LayerNorm(h)) per row from h [R, H] (float64) with magnitude mh: (y, my, xh, mxh, rs, mrs)."""
    H = h.shape[1]
    gamma, beta = np.asarray(gamma, F64), np.asarray(beta, F64)
    mean = h.sum(1, keepdims=True) / H
    mmean = (H * np.abs(h).sum(1, keepdims=True) + mh.sum(1, keepdims=True)) / H + np.abs(mean)
    d = h - mean
    md = mh + mmean + np.abs(d)
    q = (d * d).sum(1, keepdims=True)
    mq = (2.0 * np.abs(d) * md).sum(1, keepdims=True) + H * q
    v = q / H + eps
    mv = mq / H + 2.0 * v
    rs = 1.0 / np.sqrt(v)
    mrs = 0.5 * rs / v * mv + RSQRT_ULP * rs
    xh = d * rs
    mxh = rs * md + np.abs(d) * mrs + np.abs(xh)
    a = xh * gamma + beta
    ma = np.abs(gamma) * mxh + 2.0 * np.abs(xh * gamma) + np.abs(a)
    y = np.tanh(a)
    my = (1.0 - y * y) * ma + TANH_ULP * np.abs(y)
    return y, my, xh, mxh, rs[:, 0], mrs[:, 0]


def _active_rows(c):
    T, L = c["T"], slot_lens(c)
    s, t = np.nonzero(np.arange(T)[None, :] < L[:, None])
    return s, t, s * T + t, L


def rnn_forward_checks(c, saved, out):
    """The training forward's saved tensors (per layer a list of six [n * T, .] arrays, None where absent) and out
    [n, H_last], each step recomputed from the kernel's own inputs: (what, got, ref, mag) tuples."""
    T, n = c["T"], c["n"]
    s, t, r, L = _active_rows(c)
    x = c["X"][c["seqs"][c["users"][s], t], :c["in0"]]
    checks = []
    for l, lw in enumerate(c["layers"]):
        H, act, kind, sv = lw["H"], c["acts"][l], lw["kind"], saved[l]
        hp = sv[0][r]
        cp = np.where((t > 0)[:, None], sv[3][np.maximum(r - 1, 0)], 0).astype(F32) if kind == LSTM else None
        st = rnn_step_ref(lw, act, x, hp, cp, rh=sv[3][r] if kind == GRU_TF1 else None)
        checks += [(f"L{l} gates", sv[2][r], st["g"], st["mg"]), (f"L{l} SV_X", sv[3][r], st["xs"], st["mxs"])]
        nxt = t + 1 < L[s]
        checks.append((f"L{l} h_t (SV_HP of t + 1)", sv[0][r[nxt] + 1], st["h"][nxt], st["mh"][nxt]))
        if act == ACT_LN:
            hk = np.where(nxt[:, None], sv[0][np.minimum(r + 1, n * T - 1)].astype(F64), st["h"])
            mhk = np.where(nxt[:, None], 0.0, st["mh"])
            y, my, xh, mxh, rs, mrs = ln_ref(hk, mhk, lw["gamma"], lw["beta"])
            checks += [(f"L{l} SV_Y", sv[1][r], y, my), (f"L{l} SV_XH", sv[4][r], xh, mxh),
                       (f"L{l} SV_RS", sv[5][r], rs, mrs)]
            top, mtop = y, my
        else:
            checks.append((f"L{l} SV_Y", sv[1][r], st["h"], st["mh"]))
            top, mtop = st["h"], st["mh"]
        x = sv[1][r]
    # out: the top layer's output at step len - 1 (from its own state at len - 2); len 0 gives 0 or tanh(beta)
    last = t == L[s] - 1
    H = c["Hs"][-1]
    ref, mag = np.zeros((n, H)), np.zeros((n, H))
    ref[s[last]], mag[s[last]] = top[last], mtop[last]
    if c["acts"][-1] == ACT_LN:
        beta = np.asarray(c["layers"][-1]["beta"], F64)
        ref[L == 0] = np.tanh(beta)
        mag[L == 0] = TANH_ULP * np.abs(np.tanh(beta))
    checks.append(("out", out, ref, mag))
    return _floored(checks)


def rnn_forward_f32(c, mutant=None):
    """The training forward in float32 in the kernel's order: (out [n, H_last], saved).  Mutants: gru_r_without_bh,
    ln_eps, no_freeze (the state keeps stepping past len)."""
    T, n = c["T"], c["n"]
    L = slot_lens(c)
    eps = F32(1e-5 if mutant == "ln_eps" else LN_EPS)
    saved = []
    for l, lw in enumerate(c["layers"]):
        H, GH = lw["H"], gates(lw["kind"]) * lw["H"]
        z = lambda w: np.zeros((n * T, w), F32)  # noqa: E731
        saved.append([z(H), z(H), z(GH), z(H)] + ([z(H), np.zeros(n * T, F32)] if c["acts"][l] else [None, None]))
    h = [np.zeros((n, lw["H"]), F32) for lw in c["layers"]]
    cs = [np.zeros((n, lw["H"]), F32) for lw in c["layers"]]
    ys = [np.zeros((n, lw["H"]), F32) for lw in c["layers"]]
    xin0 = np.zeros((n, c["in0"]), F32)
    steps = T if mutant == "no_freeze" else int(L.max(initial=0))
    for t in range(steps):
        act_rows = (t < L) if mutant != "no_freeze" else np.ones(n, bool)
        xin0 = np.where(act_rows[:, None], c["X"][c["seqs"][c["users"], t], :c["in0"]], xin0).astype(F32)
        x = xin0
        for l, lw in enumerate(c["layers"]):
            act = c["acts"][l]
            hn, gsv, xs, cn = _rnn_cell_f32(lw, act, x, h[l], cs[l], mutant)
            rows = np.nonzero(act_rows)[0]
            sr = rows * T + t
            rec = t < L[rows]
            if len(rows):
                saved[l][0][sr[rec]] = h[l][rows[rec]]
                saved[l][2][sr[rec]] = gsv[rows[rec]]
                saved[l][3][sr[rec]] = xs[rows[rec]]
            h[l] = np.where(act_rows[:, None], hn, h[l])
            if lw["kind"] == LSTM:
                cs[l] = np.where(act_rows[:, None], cn, cs[l])
            if act == ACT_LN:
                ys[l], xh, rs = _ln_f32(h[l], lw["gamma"], lw["beta"], eps)
                if len(rows):
                    saved[l][4][sr[rec]] = xh[rows[rec]]
                    saved[l][5][sr[rec]] = rs[rows[rec]]
                x = ys[l]
            else:
                x = h[l]
            if len(rows):
                saved[l][1][sr[rec]] = x[rows[rec]]
    lw = c["layers"][-1]
    if c["acts"][-1] == ACT_LN:
        out = _ln_f32(h[-1], lw["gamma"], lw["beta"], eps)[0]
    else:
        out = h[-1]
    return out.astype(F32), saved


def _chain32(x, W, b=None):
    """acc = sum_k x[:, k] W[k] (fmaf, k ascending, from 0), then + b when given."""
    acc = np.zeros((x.shape[0], W.shape[1]), F32)
    for k in range(x.shape[1]):
        acc = fma32(x[:, k:k + 1], W[k][None, :], acc)
    return acc if b is None else (acc + np.asarray(b, F32)).astype(F32)


def _sig32(v):
    return (F32(1) / (F32(1) + np.exp(-v.astype(F32)))).astype(F32)


def _act32(a, v):
    return np.tanh(v).astype(F32) if a == ACT_TANH else v


def _rnn_cell_f32(lw, act, x, h, c, mutant):
    kind, H = lw["kind"], lw["H"]
    W, Uw, bx, bh = (np.asarray(lw[k], F32) for k in ("W", "U", "bx", "bh"))
    axb = _chain32(x[:, :-1], W[:-1], bx) if mutant == "drop_last_w" else _chain32(x, W, bx)
    if kind == LSTM:
        ahb = _chain32(h, Uw, bh)
        v = (axb + ahb).astype(F32)
        ig, fg, og = _sig32(v[:, :H]), _sig32(v[:, H:2 * H]), _sig32(v[:, 3 * H:])
        gg = _act32(act, v[:, 2 * H:3 * H])
        cn = fma32(fg, c, (ig * gg).astype(F32))
        hn = (og * _act32(act, cn)).astype(F32)
        return hn, np.hstack([ig, fg, gg, og]), cn, cn
    if kind == GRU_KERAS:
        ahb = _chain32(h, Uw, bh)
        z = _sig32(axb[:, :H] + ahb[:, :H])
        r = _sig32(axb[:, H:2 * H] + ahb[:, H:2 * H])
        if mutant == "gru_r_without_bh":
            a_c = _chain32(h, Uw[:, 2 * H:])
            v = (axb[:, 2 * H:] + fma32(r, a_c, bh[2 * H:][None, :])).astype(F32)
        else:
            v = fma32(r, ahb[:, 2 * H:], axb[:, 2 * H:])
        hh = _act32(act, v)
        hn = fma32(z, h, ((F32(1) - z) * hh).astype(F32))
        return hn, np.hstack([z, r, hh]), ahb[:, 2 * H:], None
    ahb = _chain32(h, Uw[:, :2 * H], bh[:2 * H])
    z = _sig32(axb[:, :H] + ahb[:, :H])
    r = _sig32(axb[:, H:2 * H] + ahb[:, H:2 * H])
    rh = (r * h).astype(F32)
    ac = _chain32(rh, Uw[:, 2 * H:], bh[2 * H:])
    cc = _act32(act, (axb[:, 2 * H:] + ac).astype(F32))
    hn = fma32(z, h, ((F32(1) - z) * cc).astype(F32))
    return hn, np.hstack([z, r, cc]), rh, None


def _ln_f32(h, gamma, beta, eps):
    H = h.shape[1]
    s = np.zeros(h.shape[0], F32)
    for j in range(H):
        s = (s + h[:, j]).astype(F32)
    mean = (s / F32(H)).astype(F32)
    q = np.zeros(h.shape[0], F32)
    for j in range(H):
        d = (h[:, j] - mean).astype(F32)
        q = fma32(d, d, q)
    rs = (F32(1) / np.sqrt((q / F32(H) + eps).astype(F32))).astype(F32)
    xh = ((h - mean[:, None]) * rs[:, None]).astype(F32)
    y = np.tanh(fma32(xh, np.asarray(gamma, F32)[None, :], np.asarray(beta, F32)[None, :])).astype(F32)
    return y, xh, rs


# ===================================================================================================================
# RNN4Rec backward through time
# ===================================================================================================================
def rnn_backward_ref(c, l, sv, dout=None, dy=None, kern=None):
    """Float64 backward of layer l from its saved tensors ``sv`` and dout [n, H] (top) or dy [n * T, H].  ``kern``
    = dict(dgx, dgh) of the kernel: step t's carry is rebuilt from the kernel's own gate gradients of step t + 1 (None:
    from the reference's own, which is the exact float64 recursion).  Returns dict name -> (ref, mag) over all
    n * T rows (rows t >= len are 0 with magnitude 0)."""
    lw, T, n = c["layers"][l], c["T"], c["n"]
    kind, H, act = lw["kind"], lw["H"], c["acts"][l]
    GH = gates(kind) * H
    Uw, gamma = np.asarray(lw["U"], F64), np.asarray(lw["gamma"], F64)
    L = slot_lens(c)
    dgx, mdgx = np.zeros((n * T, GH)), np.zeros((n * T, GH))
    dgh, mdgh = np.zeros((n * T, GH)), np.zeros((n * T, GH))
    dln, mdln = np.zeros((n * T, H)), np.zeros((n * T, H))
    dlnx, mdlnx = np.zeros((n * T, H)), np.zeros((n * T, H))
    ln = act == ACT_LN
    if ln and dout is not None:
        y0 = np.tanh(np.asarray(lw["beta"], F64))
        z0 = L == 0
        row0 = np.nonzero(z0)[0] * T
        dln[row0] = dout[z0, :H] * (1.0 - y0 * y0)
        mdln[row0] = np.abs(dout[z0, :H]) * (2.0 * TANH_ULP * y0 * y0 + 3.0) + np.abs(dln[row0])
    dh_c, mdh_c = np.zeros((n, H)), np.zeros((n, H))      # the carry into step t: dh from step t + 1
    dc_c, mdc_c = np.zeros((n, H)), np.zeros((n, H))
    G, Sx, Shp = sv[2].astype(F64), sv[3].astype(F64), sv[0].astype(F64)
    src = kern
    for t in range(T - 1, -1, -1):
        a = t < L
        s = np.nonzero(a)[0]
        if not len(s):
            continue
        r = s * T + t
        # the carry from step t + 1 (rows with t + 1 < len)
        nx = t + 1 < L[s]
        carry, mcarry = np.zeros((len(s), H)), np.zeros((len(s), H))
        if nx.any():
            r1 = r[nx] + 1
            gx1 = (src["dgx"] if src is not None else dgx)[r1].astype(F64)
            if kind == LSTM:
                carry[nx] = gx1 @ Uw.T
                mcarry[nx] = GH * (np.abs(gx1) @ np.abs(Uw.T)) + np.abs(carry[nx])
            else:
                z1 = G[r1, :H]
                gh1 = (src["dgh"] if src is not None else dgh)[r1].astype(F64) if kind == GRU_KERAS else gx1
                if kind == GRU_KERAS:
                    acc = gh1 @ Uw.T
                    macc = GH * (np.abs(gh1) @ np.abs(Uw.T))
                    extra, mextra = 0.0, 0.0
                else:
                    r_1 = G[r1, H:2 * H]
                    dcU = gx1[:, 2 * H:] @ Uw[:, 2 * H:].T
                    mdcU = H * (np.abs(gx1[:, 2 * H:]) @ np.abs(Uw[:, 2 * H:].T))
                    extra = dcU * r_1
                    mextra = np.abs(r_1) * mdcU + 2.0 * np.abs(extra)
                    acc = gx1[:, :2 * H] @ Uw[:, :2 * H].T
                    macc = 2 * H * (np.abs(gx1[:, :2 * H]) @ np.abs(Uw[:, :2 * H].T))
                dd = dh_c[s[nx]] * z1 + extra
                carry[nx] = dd + acc
                mcarry[nx] = (np.abs(z1) * mdh_c[s[nx]] + np.abs(dh_c[s[nx]] * z1) + mextra + macc
                              + 2.0 * np.abs(dd) + np.abs(carry[nx]))
        # the direct term dY_t
        if dy is not None:
            add = dy[r, :H].astype(F64)
        else:
            add = np.where((t == L[s] - 1)[:, None], dout[s, :H].astype(F64), 0.0)
        if ln:
            yk, xh, rs = sv[1][r].astype(F64), sv[4][r].astype(F64), sv[5][r].astype(F64)
            dl = add * (1.0 - yk * yk)
            mdl = np.abs(add) * (np.abs(1.0 - yk * yk) + 2.0 * yk * yk) + 2.0 * np.abs(dl)
            dln[r], mdln[r] = dl, mdl
            dlnx[r], mdlnx[r] = dl * xh, np.abs(xh) * mdl + np.abs(dl * xh)
            q = dl * gamma
            mq = np.abs(gamma) * mdl + np.abs(q)
            mq1 = q.mean(1, keepdims=True)
            mqx = (q * xh).mean(1, keepdims=True)
            m1 = (mq.sum(1, keepdims=True) + H * np.abs(q).sum(1, keepdims=True)) / H + np.abs(mq1)
            m2 = (H * np.abs(q * xh).sum(1, keepdims=True) + (np.abs(xh) * mq).sum(1, keepdims=True)) / H \
                + np.abs((q * xh).mean(1, keepdims=True))
            inner = q - mq1 - xh * mqx
            minner = mq + m1 + np.abs(xh) * m2 + 3.0 * (np.abs(q) + np.abs(mq1) + np.abs(xh * mqx))
            direct = rs[:, None] * inner
            mdirect = np.abs(rs[:, None]) * minner + np.abs(direct)
        else:
            direct, mdirect = add, 0.0
        dh = carry + direct
        mdh = mcarry + mdirect + np.abs(dh)
        g = G[r]
        if kind == LSTM:
            ig, fg, gg, og = (g[:, i * H:(i + 1) * H] for i in range(4))
            c1 = Sx[r]
            c0 = np.where((t > 0), Sx[np.maximum(r - 1, 0)], 0.0)
            tc = _act(act, c1)
            dtc = 1.0 - tc * tc if act == ACT_TANH else 1.0
            mtc = 2.0 * TANH_ULP * tc * tc + 3.0 if act == ACT_TANH else 0.0
            dcv = dc_c[s] + dh * og * dtc
            mdcv = mdc_c[s] + np.abs(og * dtc) * mdh + np.abs(dh * og) * mtc + 4.0 * np.abs(dh * og * dtc) + np.abs(dcv)
            di = dcv * gg * ig * (1.0 - ig)
            df = dcv * c0 * fg * (1.0 - fg)
            dgg = dcv * ig * (1.0 - gg * gg if act == ACT_TANH else 1.0)
            dov = dh * tc * og * (1.0 - og)
            mdi = np.abs(gg * ig * (1.0 - ig)) * mdcv + 5.0 * np.abs(di)
            mdf = np.abs(c0 * fg * (1.0 - fg)) * mdcv + 5.0 * np.abs(df)
            mdg = np.abs(ig * (1.0 - gg * gg if act == ACT_TANH else 1.0)) * mdcv + 5.0 * np.abs(dgg)
            mdo = np.abs(tc * og * (1.0 - og)) * mdh + 5.0 * np.abs(dov)
            dgx[r], mdgx[r] = np.hstack([di, df, dgg, dov]), np.hstack([mdi, mdf, mdg, mdo])
            dc_c[s] = dcv * fg
            mdc_c[s] = np.abs(fg) * mdcv + np.abs(dcv * fg)
        else:
            z, rg, hh = g[:, :H], g[:, H:2 * H], g[:, 2 * H:]
            hp = Shp[r]
            dact = 1.0 - hh * hh if act == ACT_TANH else 1.0
            dn = dh * (1.0 - z) * dact
            mdn = np.abs((1.0 - z) * dact) * mdh + 5.0 * np.abs(dn)
            dz = dh * (hp - hh) * z * (1.0 - z)
            mdz = np.abs((hp - hh) * z * (1.0 - z)) * mdh + 6.0 * np.abs(dz)
            if kind == GRU_KERAS:
                dr = dn * Sx[r] * rg * (1.0 - rg)
                mdr = np.abs(Sx[r] * rg * (1.0 - rg)) * mdn + 4.0 * np.abs(dr)
                dgx[r], mdgx[r] = np.hstack([dz, dr, dn]), np.hstack([mdz, mdr, mdn])
                dgh[r] = np.hstack([dz, dr, dn * rg])
                mdgh[r] = np.hstack([mdz, mdr, np.abs(rg) * mdn + np.abs(dn * rg)])
            else:
                gx_dn = (src["dgx"][r, 2 * H:].astype(F64) if src is not None else dn)
                acc = gx_dn @ Uw[:, 2 * H:].T
                macc = H * (np.abs(gx_dn) @ np.abs(Uw[:, 2 * H:].T)) + np.abs(acc)
                dr = acc * hp * rg * (1.0 - rg)
                mdr = np.abs(hp * rg * (1.0 - rg)) * macc + 4.0 * np.abs(dr)
                dgx[r], mdgx[r] = np.hstack([dz, dr, dn]), np.hstack([mdz, mdr, mdn])
            dh_c[s], mdh_c[s] = dh, mdh
    res = dict(dgx=(dgx, mdgx), dln=(dln, mdln), dlnx=(dlnx, mdlnx))
    if kind == GRU_KERAS:
        res["dgh"] = (dgh, mdgh)
    return res


def rnn_backward_f32(c, l, sv, dout=None, dy=None, mutant=None):
    """b200_rnn_backward in float32 in the kernel's order (dh kept per slot, steps in reverse)."""
    lw, T, n = c["layers"][l], c["T"], c["n"]
    kind, H, act = lw["kind"], lw["H"], c["acts"][l]
    GH = gates(kind) * H
    Uw, gamma = np.asarray(lw["U"], F32), np.asarray(lw["gamma"], F32)
    L = slot_lens(c)
    ln = act == ACT_LN
    dgx = np.zeros((n * T, GH), F32)
    dgh = np.zeros((n * T, GH), F32)
    dln = np.zeros((n * T, H), F32)
    dlnx = np.zeros((n * T, H), F32)
    if ln and dout is not None:
        y0 = np.tanh(np.asarray(lw["beta"], F32)).astype(F32)
        for s in np.nonzero(L == 0)[0]:
            row = s * T + (1 if mutant == "len0_row" and T > 1 else 0)
            dln[row] = (dout[s, :H] * (F32(1) - y0 * y0)).astype(F32)
    dh = np.zeros((n, H), F32)
    dc = np.zeros((n, H), F32)
    one = F32(1)
    for t in range(int(L.max(initial=0)) - 1, -1, -1):
        s = np.nonzero(t < L)[0]
        r = s * T + t
        add = dy[r, :H] if dy is not None else np.where((t == L[s] - 1)[:, None], dout[s, :H], F32(0)).astype(F32)
        if ln:
            yk, xh, rs = sv[1][r], sv[4][r], sv[5][r]
            dl = (add * (one - yk * yk)).astype(F32)
            dln[r], dlnx[r] = dl, (dl * xh).astype(F32)
            q = (dl * gamma).astype(F32)
            a = np.zeros(len(s), F32)
            b = np.zeros(len(s), F32)
            for j in range(H):
                a = (a + q[:, j]).astype(F32)
                b = fma32(q[:, j], xh[:, j], b)
            a, b = (a / F32(H)).astype(F32), (b / F32(H)).astype(F32)
            if mutant == "ln_bwd_no_qx":
                b = np.zeros_like(b)
            dh[s] = (dh[s] + rs[:, None] * ((q - a[:, None]).astype(F32) - (xh * b[:, None]).astype(F32))).astype(F32)
        else:
            dh[s] = (dh[s] + add).astype(F32)
        g = sv[2][r]
        dhv = dh[s]
        if kind == LSTM:
            ig, fg, gg, og = (g[:, i * H:(i + 1) * H] for i in range(4))
            c1 = sv[3][r]
            c0 = sv[3][r - 1] if t else np.zeros_like(c1)
            tc = _act32(act, c1)
            dt = (one - tc * tc).astype(F32) if act == ACT_TANH else one
            dcv = (dc[s] + (dhv * og * dt).astype(F32)).astype(F32)
            di = (dcv * gg * ig * (one - ig)).astype(F32)
            df = (dcv * c0 * fg * (one - fg)).astype(F32)
            dg = (dcv * ig * ((one - gg * gg) if act == ACT_TANH else one)).astype(F32)
            do = (dhv * tc * og * (one - og)).astype(F32)
            dc[s] = dcv if mutant == "lstm_dc_no_f" else (dcv * fg).astype(F32)
            sg = np.hstack([di, df, dg, do])
            dgx[r] = sg
            dd = np.zeros_like(dhv)
        elif kind == GRU_KERAS:
            z, rg, hh = g[:, :H], g[:, H:2 * H], g[:, 2 * H:]
            hp = sv[0][r]
            dn = (dhv * (one - z) * ((one - hh * hh) if act == ACT_TANH else one)).astype(F32)
            dz = (dhv * (hp - hh) * z * (one - z)).astype(F32)
            dr = (dn * sv[3][r] * rg * (one - rg)).astype(F32)
            dgx[r] = np.hstack([dz, dr, dn])
            sg = np.hstack([dz, dr, dn if mutant == "dgh_no_r" else (dn * rg).astype(F32)])
            dgh[r] = sg
            dd = (dhv * z).astype(F32)
        else:
            z, rg, cc = g[:, :H], g[:, H:2 * H], g[:, 2 * H:]
            hp = sv[0][r]
            dn = (dhv * (one - z) * ((one - cc * cc) if act == ACT_TANH else one)).astype(F32)
            dz = (dhv * (hp - cc) * z * (one - z)).astype(F32)
            acc = _chain32(dn, Uw[:, 2 * H:].T.copy())
            dr = (acc * hp * rg * (one - rg)).astype(F32)
            dgx[r] = np.hstack([dz, dr, dn])
            sg = np.hstack([dz, dr])
            dd = (dhv * z).astype(F32) if mutant == "tf1_dd_no_r" else fma32(acc, rg, (dhv * z).astype(F32))
        nc = sg.shape[1]
        dh[s] = (dd + _chain32(sg, Uw[:, :nc].T.copy())).astype(F32)
    return dict(dgx=dgx, dgh=dgh if kind == GRU_KERAS else None, dln=dln if ln else None, dlnx=dlnx if ln else None)


def rnn_backward_checks(c, l, sv, got, dout=None, dy=None):
    """(what, got, ref, mag) for the kernel's (or a restatement's) backward outputs ``got`` of layer l."""
    ref = rnn_backward_ref(c, l, sv, dout, dy, kern=dict(dgx=got["dgx"], dgh=got.get("dgh")))
    return _floored([(f"L{l} {k}", got[k], v, m) for k, (v, m) in ref.items() if got.get(k) is not None])


# ===================================================================================================================
# Caser
# ===================================================================================================================
def caser_floats(T, K, nh, nv):
    return K * nh * T * (T + 1) // 2 + T * nh + T * nv + nv


def caser_unpack(w, T, K, nh, nv):
    Wh, off = [], 0
    for h in range(1, T + 1):
        Wh.append(w[off:off + h * K * nh].reshape(h, K, nh))
        off += h * K * nh
    bh = w[off:off + T * nh].reshape(T, nh)
    off += T * nh
    Wv = w[off:off + T * nv].reshape(T, nv)
    off += T * nv
    return Wh, bh, Wv, w[off:off + nv]


def caser_nchunk(n, E):
    return max(1, min(-(-n // CONV_CHUNK_ROWS), CONV_PART_FLOATS // E, 65535))


def conv_tile(us, buffers):
    return max(1, min(CONV_MAX_TILE, SMEM_TILE_BYTES // (buffers * us * 4)))


def caser_tile(T, K):
    return conv_tile((T * K) | 1, 1)


def wavenet_tile(T, K, F):
    return conv_tile((T * (max(K, F) | 1)) | 1, 2)


def elem_passes(total):
    blocks = max(1, min(-(-total // ELEM_THREADS), ELEM_BLOCK_CAP))
    return -(-total // (blocks * ELEM_THREADS))


def make_seq_slots(rng, n, T, n_items, patterns=True):
    """Sequences [n, T] over n_items items: random rows, and (patterns) constant rows, period-2 / period-3 rows and
    rows constant after position 3 (equal windows: exact ties across a CONV_PB block boundary)."""
    seqs = rng.integers(0, n_items, (n, T)).astype(np.int32)
    if patterns:
        for i in range(n):
            kind = i % 6
            a, b, cc = rng.integers(0, n_items, 3)
            if kind == 1:
                seqs[i] = a
            elif kind == 2:
                seqs[i] = np.where(np.arange(T) % 2, a, b)
            elif kind == 3:
                seqs[i] = np.array([a, b, cc])[np.arange(T) % 3]
            elif kind == 4:
                seqs[i, 3:] = a
    return seqs


def make_conv_x(rng, n_items, K, ldx_pad):
    X = rng.uniform(-1, 1, (n_items + 1, K + ldx_pad)).astype(F32)
    X[n_items] = np.nan
    X[:, K:] = np.nan
    return X


def make_caser_case(n, T, K, nh, nv, seed, ld_seq_pad=0, ldx_pad=0, n_items=24, patterns=True):
    rng = np.random.default_rng(seed)
    X = make_conv_x(rng, n_items, K, ldx_pad)
    seqs = np.full((n, T + ld_seq_pad), n_items, np.int32)
    seqs[:, :T] = make_seq_slots(rng, n, T, n_items, patterns)
    users = rng.permutation(n).astype(np.int64)
    parts = [rng.uniform(-1, 1, h * K * nh) / np.sqrt(h * K) for h in range(1, T + 1)]
    bh = rng.uniform(-0.3, 0.3, (T, nh))
    if nh > 1:
        bh[:, 0] = -1e3                      # filter 0 of every height: max <= 0, argmax -1, output 0
    parts += [bh.ravel(), rng.uniform(-1, 1, T * nv) / np.sqrt(T), rng.uniform(-0.3, 0.3, nv)]
    w = np.concatenate(parts).astype(F32)
    return dict(n=n, T=T, K=K, nh=nh, nv=nv, X=X, seqs=seqs, users=users, w=w, parts=caser_unpack(w, T, K, nh, nv))


def gathered(c):
    """x [n, T, K] of every slot (float32)."""
    return c["X"][c["seqs"][c["users"]][:, :c["T"]]][:, :, :c["K"]]


def caser_pre_ref(c, x=None):
    """Float64 horizontal pre-activations per height: list of (pre [n, npos, nh], mag), and the vertical (v, mag)."""
    x = gathered(c) if x is None else x
    T, K = c["T"], c["K"]
    Wh, bh, Wv, bv = c["parts"]
    x64, ax = x.astype(F64), np.abs(x.astype(F64))
    hor = []
    for h in range(1, T + 1):
        npos = T - h + 1
        W = np.asarray(Wh[h - 1], F64)
        b = np.asarray(bh[h - 1], F64)
        pre = np.broadcast_to(b, (x.shape[0], npos, len(b))).copy()
        m = np.broadcast_to(np.abs(b), pre.shape).copy()
        for j in range(h):
            pre += x64[:, j:j + npos] @ W[j]
            m += ax[:, j:j + npos] @ np.abs(W[j])
        hor.append((pre, h * K * m + np.abs(pre)))
    Wv64, bv64 = np.asarray(Wv, F64), np.asarray(bv, F64)
    v = np.einsum("stk,tf->skf", x64, Wv64) + bv64
    mv = T * (np.einsum("stk,tf->skf", ax, np.abs(Wv64)) + np.abs(bv64)) + np.abs(v)
    return hor, (v, mv)


def caser_forward_checks(c, out, arg=None):
    """(what, got, ref, mag) for out [n, T*nh + K*nv]; with arg [n, T*nh] also the argmax rules (assertions)."""
    T, K, nh, nv, n = c["T"], c["K"], c["nh"], c["nv"], c["n"]
    hor, (v, mv) = caser_pre_ref(c)
    ref_h = np.concatenate([np.maximum(p, 0).max(1) for p, _ in hor], axis=1)
    mag_h = np.concatenate([m.max(1) for _, m in hor], axis=1)
    checks = [("caser horizontal", out[:, :T * nh], ref_h, mag_h),
              ("caser vertical", out[:, T * nh:T * nh + K * nv], np.maximum(v, 0).reshape(n, -1),
               mv.reshape(n, -1))]
    return _floored(checks)


def argmax_violations(pre, mag, arg, out, windows, C):
    """The max-pool argmax rules on one column family: pre / mag [n, npos, F] float64, arg [n, F] from the kernel,
    out [n, F] the kernel's max, windows [n, npos] hashable ids (equal id = equal float32 chain): returns a list of
    messages.  -1 iff out == 0 and every position is <= 0 within the bound; otherwise out > 0, arg reaches the
    maximum within the bound, and no lower position has the same window (the LOWEST equal position wins)."""
    bad = []
    tol = C * U * mag
    hi = pre + tol
    n, npos, F = pre.shape
    for s in range(n):
        for f in range(F):
            a = int(arg[s, f])
            if a == -1:
                if out[s, f] != 0 or (pre[s, :, f] - tol[s, :, f] > 0).any():
                    bad.append(f"slot {s} col {f}: -1 with a positive position or output {out[s, f]}")
                continue
            if not 0 <= a < npos or not out[s, f] > 0:
                bad.append(f"slot {s} col {f}: arg {a} of {npos}, out {out[s, f]}")
                continue
            if hi[s, a, f] < (pre[s, :, f] - tol[s, :, f]).max():
                bad.append(f"slot {s} col {f}: arg {a} does not reach the maximum")
            if (windows[s, :a] == windows[s, a]).any():
                bad.append(f"slot {s} col {f}: arg {a} has an equal window at a lower position")
    return bad


def caser_windows(c, h):
    """Per slot and window start, an id equal for windows of equal item rows."""
    sq = c["seqs"][c["users"]][:, :c["T"]].astype(np.int64)
    npos = c["T"] - h + 1
    ids = np.zeros((c["n"], npos), np.int64)
    for j in range(h):
        ids = ids * 1_000_003 + sq[:, j:j + npos] + 1
    return ids


def caser_argmax_violations(c, out, arg, C):
    T, nh = c["T"], c["nh"]
    hor, _ = caser_pre_ref(c)
    bad = []
    for h in range(1, T + 1):
        pre, m = hor[h - 1]
        cols = slice((h - 1) * nh, h * nh)
        bad += [f"h={h} {b}" for b in argmax_violations(pre, m, arg[:, cols], out[:, cols], caser_windows(c, h), C)]
    return bad


def caser_forward_f32(c, mutant=None):
    """b200_caser_train_forward in float32 (out, argmax).  Mutant tie_high: ties go to the highest position."""
    T, K, nh, nv, n = c["T"], c["K"], c["nh"], c["nv"], c["n"]
    x = gathered(c)
    Wh, bh, Wv, bv = c["parts"]
    out = np.zeros((n, T * nh + K * nv), F32)
    arg = np.full((n, T * nh), -1, np.int32)
    for h in range(1, T + 1):
        npos = T - h + 1
        acc = np.broadcast_to(np.asarray(bh[h - 1], F32), (n, npos, nh)).copy()
        for j in range(h):
            for k in range(K):
                acc = fma32(x[:, j:j + npos, k][:, :, None], Wh[h - 1][j, k][None, None, :], acc)
        m = np.maximum(acc.max(1), 0)
        out[:, (h - 1) * nh:h * nh] = m
        pos = acc if mutant != "tie_high" else acc[:, ::-1]
        a = np.argmax(pos, axis=1)
        a = a if mutant != "tie_high" else npos - 1 - a
        arg[:, (h - 1) * nh:h * nh] = np.where(m > 0, a, -1)
    acc = np.broadcast_to(np.asarray(bv, F32), (n, K, nv)).copy()
    for t in range(T):
        acc = fma32(x[:, t, :, None], np.asarray(Wv, F32)[t][None, None, :], acc)
    out[:, T * nh:] = np.maximum(acc, 0).reshape(n, -1)
    return out, arg


def caser_backward_ref(c, dF, feat, arg, hs=None, dx_slots=None):
    """Float64 dX [n * T, K] and dW (packed) of b200_caser_backward from the kernel's own argmax and feat, with
    magnitudes.  ``hs``: the heights whose W_h block is checked (None: all; others get ref NaN, mag 0); dX of the
    slots ``dx_slots`` only (None: all), rows in that order."""
    T, K, nh, nv, n = c["T"], c["K"], c["nh"], c["nv"], c["n"]
    x = gathered(c).astype(F64)
    Wh, bh, Wv, bv = c["parts"]
    nhor = T * nh
    dF, feat = dF[:, :nhor + K * nv].astype(F64), feat[:, :nhor + K * nv]
    g = np.where(arg >= 0, dF[:, :nhor], 0.0)
    gv = np.where(feat[:, nhor:] > 0, dF[:, nhor:], 0.0).reshape(n, K, nv)
    E = caser_floats(T, K, nh, nv)
    nchunk = caser_nchunk(n, E)
    chunk = -(-n // nchunk)
    ds = np.arange(n) if dx_slots is None else np.asarray(dx_slots)
    m_ = len(ds)
    dX = np.zeros(m_ * T * K)
    sX = np.zeros(m_ * T * K)
    cnt = np.zeros(m_ * T * K)
    base = (np.arange(m_) * T * K)[:, None, None]
    for h in range(1, T + 1):
        A = arg[ds, (h - 1) * nh:h * nh].astype(np.int64)
        G = g[ds, (h - 1) * nh:h * nh]
        Wf = np.asarray(Wh[h - 1], F64).transpose(2, 0, 1).reshape(nh, h * K)    # [f, (j, k)]
        on = A >= 0
        idx = (base + np.maximum(A, 0)[:, :, None] * K + np.arange(h * K)[None, None, :])[on]
        val = (G[:, :, None] * Wf[None])[on]
        dX += np.bincount(idx.ravel(), val.ravel(), m_ * T * K)
        sX += np.bincount(idx.ravel(), np.abs(val).ravel(), m_ * T * K)
        cnt += np.bincount(idx.ravel(), None, m_ * T * K)
    Wv64 = np.asarray(Wv, F64)
    dX += np.einsum("skf,tf->stk", gv[ds], Wv64).ravel()
    sX += np.einsum("skf,tf->stk", np.abs(gv[ds]), np.abs(Wv64)).ravel()
    mdX = (cnt + nv) * sX + np.abs(dX)
    # dW: chunk chains of `chunk` rows (the vertical ones K terms per row), then nchunk partials
    dW = np.full(E, np.nan)
    mW = np.zeros(E)
    off = 0
    for h in range(1, T + 1):
        sz = h * K * nh
        if hs is None or h in hs:
            A = arg[:, (h - 1) * nh:h * nh].astype(np.int64)
            G = g[:, (h - 1) * nh:h * nh]
            blk, sblk = np.zeros((h, K, nh)), np.zeros((h, K, nh))
            rows = np.arange(n)[:, None]
            for j in range(h):
                xj = x[rows, np.clip(A + j, 0, T - 1)]                        # [n, nh, K]
                blk[j] = np.einsum("sf,sfk->kf", G, xj)
                sblk[j] = np.einsum("sf,sfk->kf", np.abs(G), np.abs(xj))
            dW[off:off + sz] = blk.ravel()
            mW[off:off + sz] = (chunk + nchunk) * sblk.ravel() + np.abs(blk.ravel())
        off += sz
    dW[off:off + nhor] = g.sum(0)
    mW[off:off + nhor] = (chunk + nchunk) * np.abs(g).sum(0) + np.abs(g.sum(0))
    off += nhor
    wv = np.einsum("skf,stk->tf", gv, x)
    dW[off:off + T * nv] = wv.ravel()
    mW[off:off + T * nv] = (chunk * K + nchunk) * np.einsum("skf,stk->tf", np.abs(gv), np.abs(x)).ravel() \
        + np.abs(wv.ravel())
    off += T * nv
    dW[off:] = gv.sum((0, 1))
    mW[off:] = (chunk * K + nchunk) * np.abs(gv).sum((0, 1)) + np.abs(gv.sum((0, 1)))
    return (dX.reshape(m_ * T, K), mdX.reshape(m_ * T, K)), (dW, mW)


def caser_backward_checks(c, dF, feat, arg, dX, dW, hs=None, dx_slots=None):
    """dX [n * T, K] (rows s * T + t) and dW of the kernel against caser_backward_ref."""
    (rx, mx), (rw, mw) = caser_backward_ref(c, dF, feat, arg, hs, dx_slots)
    keep = ~np.isnan(rw)
    if dx_slots is not None:
        dX = dX.reshape(c["n"], c["T"], -1)[np.asarray(dx_slots)].reshape(-1, dX.shape[1])
    return _floored([("caser dX", dX, rx, mx), ("caser dW", dW[keep], rw[keep], mw[keep])])


def caser_backward_f32(c, dF, feat, arg, mutant=None):
    """b200_caser_backward in float32 in the kernels' order.  Mutants: vmask_df (the vertical mask on dF > 0),
    dw_drop_last_chunk."""
    T, K, nh, nv, n = c["T"], c["K"], c["nh"], c["nv"], c["n"]
    x = gathered(c)
    Wh, bh, Wv, bv = c["parts"]
    nhor = T * nh
    g = np.where(arg >= 0, dF[:, :nhor], F32(0)).astype(F32)
    vm = (dF[:, nhor:nhor + K * nv] > 0) if mutant == "vmask_df" else (feat[:, nhor:nhor + K * nv] > 0)
    gv = np.where(vm, dF[:, nhor:nhor + K * nv], F32(0)).astype(F32).reshape(n, K, nv)
    dX = np.zeros((n, T, K), F32)
    for t in range(T):
        acc = np.zeros((n, K), F32)
        for h in range(1, T + 1):
            for f in range(nh):
                a = arg[:, (h - 1) * nh + f]
                j = t - a
                ok = (a >= 0) & (j >= 0) & (j < h)
                w = Wh[h - 1][np.clip(j, 0, h - 1), :, f]                      # [n, K]
                acc = np.where(ok[:, None], fma32(g[:, (h - 1) * nh + f][:, None], w, acc), acc)
        for f in range(nv):
            acc = fma32(gv[:, :, f], F32(Wv[t, f]), acc)
        dX[:, t] = acc
    E = caser_floats(T, K, nh, nv)
    nchunk = caser_nchunk(n, E)
    chunk = -(-n // nchunk)
    parts = np.zeros((nchunk, E), F32)
    for ch in range(nchunk):
        if mutant == "dw_drop_last_chunk" and ch == nchunk - 1 and nchunk > 1:
            continue
        acc = np.zeros(E, F32)
        for b in range(ch * chunk, min(n, (ch + 1) * chunk)):
            acc = _caser_row_accumulate(c, b, arg, feat, g, gv, x, acc)
        parts[ch] = acc
    dW = np.zeros(E, F32)
    for ch in range(nchunk):
        dW = (dW + parts[ch]).astype(F32)
    return dX.reshape(n * T, K), dW


def _caser_row_accumulate(c, b, arg, feat, g, gv, x, acc):
    """One row b of caser_dw_kernel's per-element chains, added to acc (float32, the packed layout)."""
    T, K, nh, nv = c["T"], c["K"], c["nh"], c["nv"]
    nhor = T * nh
    off = 0
    acc = acc.copy()
    for h in range(1, T + 1):
        sz = h * K * nh
        a = arg[b, (h - 1) * nh:h * nh]
        blk = acc[off:off + sz].reshape(h, K, nh)
        for j in range(h):
            xr = x[b, np.clip(a + j, 0, T - 1)]                                    # [nh, K]
            upd = fma32(g[b, (h - 1) * nh:h * nh][None, :], xr.T, blk[j])
            blk[j] = np.where((a >= 0)[None, :], upd, blk[j])
        acc[off:off + sz] = blk.ravel()
        off += sz
    gb = g[b, :]
    acc[off:off + nhor] = np.where(arg[b] >= 0, (acc[off:off + nhor] + gb).astype(F32), acc[off:off + nhor])
    off += nhor
    wv = acc[off:off + T * nv].reshape(T, nv)
    for k in range(K):
        on = feat[b, nhor + k * nv:nhor + (k + 1) * nv] > 0
        upd = fma32(gv[b, k][None, :], x[b, :, k][:, None], wv)
        wv = np.where(on[None, :], upd, wv)
    acc[off:off + T * nv] = wv.ravel()
    off += T * nv
    bvv = acc[off:]
    for k in range(K):
        on = feat[b, nhor + k * nv:nhor + (k + 1) * nv] > 0
        bvv = np.where(on, (bvv + gv[b, k]).astype(F32), bvv)
    acc[off:] = bvv
    return acc


# ===================================================================================================================
# WaveNet
# ===================================================================================================================
def wavenet_floats(K, F, L):
    return (2 * K * F + F) + (L - 1) * (2 * F * F + F) + F * F + F


def wavenet_unpack(w, K, F, L):
    layers, off = [], 0
    for l in range(L):
        C = K if l == 0 else F
        layers.append((w[off:off + 2 * C * F].reshape(2, C, F), w[off + 2 * C * F:off + 2 * C * F + F]))
        off += 2 * C * F + F
    W1 = w[off:off + F * F].reshape(F, F)
    return layers, W1, w[off + F * F:off + F * F + F]


def make_wavenet_case(n, T, K, F, dils, seed, ld_seq_pad=0, ldx_pad=0, n_items=24, patterns=True):
    rng = np.random.default_rng(seed)
    L = len(dils)
    X = make_conv_x(rng, n_items, K, ldx_pad)
    seqs = np.full((n, T + ld_seq_pad), n_items, np.int32)
    seqs[:, :T] = make_seq_slots(rng, n, T, n_items, patterns)
    users = rng.permutation(n).astype(np.int64)
    parts = []
    for l in range(L):
        C = K if l == 0 else F
        parts += [rng.uniform(-1.2, 1.2, 2 * C * F) / np.sqrt(2 * C), rng.uniform(-0.2, 0.3, F)]
    b1 = rng.uniform(-0.3, 0.3, F)
    if F > 1:
        b1[0] = -1e3                           # column 0: max <= 0, argmax -1, output 0
    parts += [rng.uniform(-1.5, 1.5, F * F) / np.sqrt(F), b1]
    w = np.concatenate(parts).astype(F32)
    return dict(n=n, T=T, K=K, F=F, dils=list(dils), X=X, seqs=seqs, users=users, w=w,
                parts=wavenet_unpack(w, K, F, L))


def wavenet_layer_ref(x, W, b, d):
    """Float64 causal layer on the kernel's float32 input x [n, T, C]: (y, mag) before nothing else (relu applied)."""
    x64, ax = x.astype(F64), np.abs(x.astype(F64))
    W, b = np.asarray(W, F64), np.asarray(b, F64)
    T, C = x.shape[1], x.shape[2]
    pre = x64 @ W[1] + b
    m = ax @ np.abs(W[1]) + np.abs(b)
    if d < T:
        pre[:, d:] += x64[:, :T - d] @ W[0]
        m[:, d:] += ax[:, :T - d] @ np.abs(W[0])
    return pre, 2 * C * m + np.abs(pre)


def wavenet_forward_checks(c, out, layer_out=None):
    """(what, got, ref, mag): every causal layer from the kernel's own output of the layer below (layer_out
    [L, n, T, F]; without it, the encoder output only, from the restated float64 chain of the layers), then the 1x1
    layer and the max from the last kernel layer.  Also returns the 1x1 pre-activations for the argmax rules."""
    T, F, n = c["T"], c["F"], c["n"]
    layers, W1, b1 = c["parts"]
    x = gathered(c)
    checks = []
    for l, (W, b) in enumerate(layers):
        pre, m = wavenet_layer_ref(x, W, b, c["dils"][l])
        if layer_out is not None:
            checks.append((f"wavenet layer {l}", layer_out[l], np.maximum(pre, 0), m))
            x = layer_out[l]
        else:
            x = np.maximum(pre, 0).astype(F32)
    y64, ay = x.astype(F64), np.abs(x.astype(F64))
    z = y64 @ np.asarray(W1, F64) + np.asarray(b1, F64)
    mz = F * (ay @ np.abs(np.asarray(W1, F64)) + np.abs(np.asarray(b1, F64))) + np.abs(z)
    checks.append(("wavenet out", out[:, :F], np.maximum(z, 0).max(1), mz.max(1)))
    return _floored(checks), (z, mz)


def wavenet_windows(c):
    """Per slot and position, an id equal exactly where the 1x1 layer's input rows are the same float32 chains:
    position t of layer l is the pair (id of t - d in the layer below or none while t < d, id of t), starting from the
    item ids of the sequence."""
    n, T = c["n"], c["T"]
    ids = c["seqs"][c["users"]][:, :T].astype(np.int64) + 1
    for d in c["dils"]:
        prev = np.zeros_like(ids)
        if d < T:
            prev[:, d:] = ids[:, :T - d]
        pair = prev * (ids.max() + 1) + ids
        _, ids = np.unique(pair, return_inverse=True)
        ids = ids.reshape(n, T) + 1
    return ids


def wavenet_forward_f32(c, mutant=None):
    """b200_wavenet_train_forward in float32: (out, layer_out [L, n, T, F], argmax)."""
    T, K, F, n = c["T"], c["K"], c["F"], c["n"]
    layers, W1, b1 = c["parts"]
    x = gathered(c)
    ys = []
    for l, (W, b) in enumerate(layers):
        d, C = c["dils"][l], x.shape[2]
        acc = np.broadcast_to(np.asarray(b, F32), (n, T, F)).copy()
        for ci in range(C):
            if d < T:
                acc[:, d:] = fma32(x[:, :T - d, ci, None], W[0, ci][None, None, :], acc[:, d:])
        for ci in range(C):
            acc = fma32(x[:, :, ci, None], W[1, ci][None, None, :], acc)
        x = np.maximum(acc, 0).astype(F32)
        ys.append(x)
    acc = np.broadcast_to(np.asarray(b1, F32), (n, T, F)).copy()
    for ci in range(F):
        acc = fma32(x[:, :, ci, None], W1[ci][None, None, :], acc)
    m = np.maximum(acc.max(1), 0)
    a = np.argmax(acc, axis=1) if mutant != "tie_high" else T - 1 - np.argmax(acc[:, ::-1], axis=1)
    return m.astype(F32), np.stack(ys), np.where(m > 0, a, -1).astype(np.int32)


def wavenet_pool_backward_ref(dF, arg, T, F):
    n = arg.shape[0]
    dZ = np.zeros((n, T, F), F32)
    s, f = np.nonzero(arg >= 0)
    dZ[s, arg[s, f], f] = dF[s, f]
    return dZ.reshape(n * T, F)


def wavenet_layer_inputs_ref(x, n, T, C, d, mutant=None):
    """[n * T, 2C] = [x[s*T + t - d] (0 for t < d) | x[s*T + t]] from x [n * T, >= C] (float32, copies)."""
    x = x[:, :C].reshape(n, T, C)
    prev = np.zeros_like(x)
    if mutant == "cross_slot":
        flat = x.reshape(n * T, C)
        rows = np.arange(n * T) - d
        ok = rows >= 0
        prev.reshape(n * T, C)[ok] = flat[rows[ok]]
    elif d < T:
        prev[:, d:] = x[:, :T - d]
    return np.concatenate([prev, x], axis=2).reshape(n * T, 2 * C)


def wavenet_layer_dx_ref(P, n, T, C, d, mutant=None):
    """dx [n * T, C] = P[row, C:] + P[row + d, :C] while t + d < T (one float32 add).  Mutant guard_le: the guard
    t + d <= T, which at t = T - d adds row 0 of the next slot."""
    rows = np.arange(n * T)
    t = rows % T
    dx = P[:, C:].copy()
    ok = t + d < T if mutant != "guard_le" else (t + d <= T) & (rows + d < n * T)
    dx[ok] = (dx[ok] + P[rows[ok] + d, :C]).astype(F32)
    return dx
