"""Host restatements for tests/test_gpu_rank_kernels.py and tests/test_rank_kernels_cpu.py (numpy only).

* ``fma32`` — a correctly rounded float32 ``fmaf`` on arrays: the product of two floats is exact in float64, TwoSum
  gives the exact error of the float64 sum, and that error settles the sums that land exactly on a float32 midpoint
  (where a plain float64 -> float32 cast would round to even).  Float32 subnormals and overflow to +-inf round like
  IEEE 754.  ``dot_chain`` is the exact-score definition of the library built from it: one float32 accumulator,
  ``acc = fmaf(u[k], i[k], acc)`` for k ascending.
* ``rank_order`` — the selection order of ``b200_topk_rows`` restated on values: REMOVED (the float bit pattern
  0xffffffff written over consumed items) below everything, then real values descending with -0.0 == +0.0, every
  NaN above +inf; ties by item id ascending.
* The FM / DeepFM pair formulas of ``csrc/pair.cu`` in float64 with a per-element magnitude for the error bound, and
  in float32 in the kernels' operation order (for the bound calibration).
"""
from __future__ import annotations

import numpy as np

F32, F64 = np.float32, np.float64
U = 2.0 ** -24
REMOVED_BITS = np.uint32(0xFFFFFFFF)
CANON_NAN_BITS = np.uint32(0x7FFFFFFF)
_TWO128 = 2.0 ** 128


# ----- exact fp32 fma ------------------------------------------------------------------------------------------------
def fma32(a, b, c):
    """Correctly rounded float32 a * b + c (finite a, b; c may be +-inf), elementwise with broadcasting."""
    a, b, c = np.broadcast_arrays(np.asarray(a, F32), np.asarray(b, F32), np.asarray(c, F32))
    with np.errstate(over="ignore", invalid="ignore"):
        p = a.astype(F64) * b.astype(F64)                  # exact: 24 + 24 bits, exponent within float64
        c64 = c.astype(F64)
        s = p + c64
        bb = s - p                                         # TwoSum: s + e == p + c exactly
        e = (p - (s - bb)) + (c64 - bb)
        r = s.astype(F32)                                  # round to nearest even
        r64 = r.astype(F64)
        inexact = np.isfinite(s) & (r64 != s)
        if not inexact.any():
            return r
        # the other float32 neighbour of s; +-inf stands for +-2^128 in the midpoint test
        toward = np.where(s > r64, F32(np.inf), F32(-np.inf)).astype(F32)
        other = np.nextafter(r, toward)
        r_fin = np.where(np.isinf(r64), np.copysign(_TWO128, r64), r64)
        o_fin = np.where(np.isinf(other), np.copysign(_TWO128, other.astype(F64)), other.astype(F64))
        mid = inexact & ((r_fin + o_fin) * 0.5 == s) & (e != 0)
        # on a midpoint the exact sum lies on the side of e: take the neighbour on that side
        go_other = mid & (np.sign(e) == np.sign(o_fin - s))
    return np.where(go_other, other, r).astype(F32)


def dot_chain(Urows, Irows):
    """[B, d] x [N, d] -> [B, N]: acc = fmaf(u[k], i[k], acc), k = 0 .. d-1, from acc = +0.0."""
    Urows, Irows = np.asarray(Urows, F32), np.asarray(Irows, F32)
    acc = np.zeros((Urows.shape[0], Irows.shape[0]), dtype=F32)
    for k in range(Urows.shape[1]):
        acc = fma32(Urows[:, k:k + 1], Irows[None, :, k], acc)
    return acc


def pair_chain(Urows, Irows):
    """Row-wise chain: [n, d] x [n, d] -> [n]."""
    Urows, Irows = np.asarray(Urows, F32), np.asarray(Irows, F32)
    acc = np.zeros(Urows.shape[0], dtype=F32)
    for k in range(Urows.shape[1]):
        acc = fma32(Urows[:, k], Irows[:, k], acc)
    return acc


# ----- selection order -----------------------------------------------------------------------------------------------
def bits(x):
    return np.ascontiguousarray(x, dtype=F32).view(np.uint32)


def rank_order(x, K):
    """Positions of the K first entries of every row of x [B, N] under the selection order."""
    x = np.ascontiguousarray(x, dtype=F32)
    B, N = x.shape
    removed = bits(x) == REMOVED_BITS
    nan = np.isnan(x) & ~removed
    tier = np.where(removed, 0, np.where(nan, 2, 1))               # removed < real < NaN
    with np.errstate(invalid="ignore"):
        val = np.where(tier == 1, x.astype(F64), 0.0)              # -0.0 == +0.0 in the comparisons below
    ids = np.broadcast_to(np.arange(N), (B, N))
    if N <= 65536:
        return np.lexsort((ids, -val, -tier), axis=-1)[:, :K]
    out = np.empty((B, K), dtype=np.int64)
    for r in range(B):
        # candidates: everything whose (tier, value) is >= that of the K-th entry
        sv = np.where(tier[r] == 2, np.inf, np.where(tier[r] == 0, -np.inf, val[r]))
        t = np.partition(sv, N - K)[N - K]
        cand = np.nonzero(sv >= t)[0]
        o = np.lexsort((cand, -val[r, cand], -tier[r, cand]))[:K]
        out[r] = cand[o]
    return out


def canonical_bits(x):
    """The bits b200_topk_rows writes for a selected score: -0.0 as +0.0, a NaN as 0x7fffffff, REMOVED as is."""
    b = bits(x).copy()
    nan = np.isnan(np.asarray(x, F32)) & (b != REMOVED_BITS)
    b[nan] = CANON_NAN_BITS
    b[b == np.uint32(0x80000000)] = 0
    return b


# ----- FM / DeepFM pair scores ---------------------------------------------------------------------------------------
def fm_pair_ref(c, rows, items):
    """float64 fm_pair_kernel for the users ``rows`` x the items ``items``, and the bound magnitude per element:
    out = lu + lin_bias + li + elu(sum_k (0.5 ((Su+Si)^2 - (Qu+Qi)) sc_k + sh_k) w_k + pw_bias)."""
    Su, Qu, lu = (np.asarray(c[k], F64)[rows] for k in ("Su", "Qu", "lu"))
    Si, Qi, li = (np.asarray(c[k], F64)[items] for k in ("Si", "Qi", "li"))
    K = Su.shape[1]
    sc = np.asarray(c["bn_scale"], F64) if c["bn_scale"] is not None else np.ones(K)
    sh = np.asarray(c["bn_shift"], F64) if c["bn_shift"] is not None else np.zeros(K)
    w = np.asarray(c["pw_kernel"], F64)
    s = Su[:, None, :] + Si[None]
    q = Qu[:, None, :] + Qi[None]
    acc = ((0.5 * (s * s - q)) * sc + sh) @ w + c["pw_bias"]
    elu = np.where(acc > 0, acc, np.expm1(np.minimum(acc, 0.0)))
    out = lu[:, None] + c["lin_bias"] + li[None] + elu
    sm = np.abs(Su)[:, None, :] + np.abs(Si)[None]
    qm = np.abs(Qu)[:, None, :] + np.abs(Qi)[None]
    macc = ((0.5 * (sm * sm + qm)) * np.abs(sc) + np.abs(sh)) @ np.abs(w) + abs(c["pw_bias"])
    mag = (K + 4) * macc + 4.0 * (np.abs(lu)[:, None] + abs(c["lin_bias"]) + np.abs(li)[None] + np.abs(elu))
    return out, mag


def fm_pair_f32(c, rows, items):
    """The kernel's float32 operations in its order (fmaf exact), expm1 in float32."""
    Su, Qu, lu = (np.asarray(c[k], F32)[rows] for k in ("Su", "Qu", "lu"))
    Si, Qi, li = (np.asarray(c[k], F32)[items] for k in ("Si", "Qi", "li"))
    K = Su.shape[1]
    sc = np.asarray(c["bn_scale"], F32) if c["bn_scale"] is not None else np.ones(K, F32)
    sh = np.asarray(c["bn_shift"], F32) if c["bn_shift"] is not None else np.zeros(K, F32)
    w = np.asarray(c["pw_kernel"], F32)
    acc = np.zeros((len(rows), len(items)), F32)
    for k in range(K):
        s = Su[:, None, k] + Si[None, :, k]
        q = Qu[:, None, k] + Qi[None, :, k]
        pw = F32(0.5) * (s * s - q)
        acc = fma32(fma32(pw, sc[k], sh[k]), w[k], acc)
    acc = acc + F32(c["pw_bias"])
    elu = np.where(acc > 0, acc, np.expm1(np.minimum(acc, F32(0))).astype(F32))
    return (lu + F32(c["lin_bias"]))[:, None] + li[None] + elu


def deepfm_pair_ref(c, rows, items):
    """float64 deepfm_pair_kernel and the bound magnitude per element:
    h1 = relu(Pu + Pi); h2 = h1 W2 + b2; H3 > 0: h3 = relu(h2) W3 + b3, deep = h3 w3_out; else deep = h2 w2_out;
    out = b_out + (lu + lin_bias + li) w_out[0] + sum_k 0.5 ((Su+Si)^2 - (Qu+Qi)) w_out[1+k] + deep.
    ReLU is 1-Lipschitz, so the magnitudes |Pu| + |Pi|, then |W| times those, carry the error through the layers."""
    g = {k: (np.asarray(v, F64) if v is not None and not np.isscalar(v) else v) for k, v in c.items()}
    K, H3 = c["Su"].shape[1], c["H3"]
    wo = g["w_out"]
    Su, Qu, lu, Pu = g["Su"][rows], g["Qu"][rows], g["lu"][rows], g["Pu"][rows]
    Si, Qi, li, Pi = g["Si"][items], g["Qi"][items], g["li"][items], g["Pi"][items]
    out, mag = [], []
    for r in range(len(rows)):
        h1 = np.maximum(Pu[r] + Pi, 0.0)
        m1 = np.abs(Pu[r]) + np.abs(Pi)
        h2 = h1 @ g["W2"] + g["b2"]
        m2 = m1 @ np.abs(g["W2"]) + np.abs(g["b2"])
        if H3 > 0:
            deep = (np.maximum(h2, 0.0) @ g["W3"] + g["b3"]) @ wo[1 + K:1 + K + H3]
            mdeep = (m2 @ np.abs(g["W3"]) + np.abs(g["b3"])) @ np.abs(wo[1 + K:1 + K + H3])
        else:
            deep = h2 @ wo[1 + K:1 + K + c["H2"]]
            mdeep = m2 @ np.abs(wo[1 + K:1 + K + c["H2"]])
        s = Su[r] + Si
        q = Qu[r] + Qi
        lin = lu[r] + c["lin_bias"] + li
        o = c["b_out"] + lin * wo[0] + (0.5 * (s * s - q)) @ wo[1:1 + K] + deep
        sm = np.abs(Su[r]) + np.abs(Si)
        mpw = (0.5 * (sm * sm + np.abs(Qu[r]) + np.abs(Qi))) @ np.abs(wo[1:1 + K])
        m = abs(c["b_out"]) + (abs(lu[r]) + abs(c["lin_bias"]) + np.abs(li)) * abs(wo[0]) + mpw + mdeep
        out.append(o)
        mag.append((c["H1"] + c["H2"] + H3 + K + 8) * m)
    return np.stack(out), np.stack(mag)


def deepfm_pair_f32(c, rows, items):
    """The kernel's float32 operations in its order (h2 and h3 as fmaf chains, the head chain k then j)."""
    f = {k: (np.asarray(v, F32) if v is not None and not np.isscalar(v) else v) for k, v in c.items()}
    K, H1, H2, H3 = c["Su"].shape[1], c["H1"], c["H2"], c["H3"]
    wo = f["w_out"]
    out = []
    for r in rows:
        Pi = f["Pi"][items]
        h2 = np.zeros((len(items), H2), F32)
        for j in range(H1):
            h = np.maximum(f["Pu"][r, j] + Pi[:, j], F32(0))
            h2 = fma32(h[:, None], f["W2"][j][None], h2)
        o = np.full(len(items), F32(c["b_out"]), F32)
        o = o + (f["lu"][r] + F32(c["lin_bias"]) + f["li"][items]) * wo[0]
        for k in range(K):
            s = f["Su"][r, k] + f["Si"][items, k]
            q = f["Qu"][r, k] + f["Qi"][items, k]
            o = fma32(F32(0.5) * (s * s - q), wo[1 + k], o)
        if H3 > 0:
            v = np.maximum(h2 + f["b2"][None], F32(0))
            for j in range(H3):
                h3 = np.full(len(items), f["b3"][j], F32)
                for m in range(H2):
                    h3 = fma32(v[:, m], f["W3"][m, j], h3)
                o = fma32(h3, wo[1 + K + j], o)
        else:
            for m in range(H2):
                o = fma32(h2[:, m] + f["b2"][m], wo[1 + K + m], o)
        out.append(o)
    return np.stack(out)


def make_fm_case(B, K, N, bn, seed):
    rng = np.random.default_rng(seed)
    c = dict(Su=rng.standard_normal((B, K)), Qu=rng.uniform(0.0, 2.0, (B, K)), lu=rng.standard_normal(B),
             Si=rng.standard_normal((N, K)), Qi=rng.uniform(0.0, 2.0, (N, K)), li=rng.standard_normal(N),
             bn_scale=rng.uniform(0.5, 1.5, K) if bn else None, bn_shift=rng.normal(0.0, 0.3, K) if bn else None,
             pw_kernel=rng.normal(0.0, 1.0 / np.sqrt(K), K))
    c = {k: (v.astype(F32) if v is not None else None) for k, v in c.items()}
    sh = c["bn_shift"].astype(F64) if bn else np.zeros(K)
    c["lin_bias"], c["pw_bias"] = float(F32(0.25)), float(F32(-(sh @ c["pw_kernel"].astype(F64))))
    # items 0 .. 63 nearly cancel user 0's pairwise block (s = 0, q ~ +-1e-4): acc next to 0 on both sides
    near = np.arange(min(N, 64))
    c["Si"][near] = -c["Su"][0]
    c["Qi"][near] = -c["Qu"][0] * (1 + 1e-4 * rng.standard_normal((len(near), K)))
    return c


def make_deepfm_case(B, K, N, H1, H2, H3, fm_zero, seed):
    rng = np.random.default_rng(seed)
    c = dict(Su=rng.standard_normal((B, K)), Qu=rng.uniform(0.0, 2.0, (B, K)), lu=rng.standard_normal(B),
             Si=rng.standard_normal((N, K)), Qi=rng.uniform(0.0, 2.0, (N, K)), li=rng.standard_normal(N),
             Pu=rng.standard_normal((B, H1)), Pi=rng.standard_normal((N, H1)),
             W2=rng.normal(0.0, 1.0 / np.sqrt(H1), (H1, H2)), b2=rng.normal(0.0, 0.1, H2),
             W3=rng.normal(0.0, 1.0 / np.sqrt(H2), (H2, max(H3, 1))) if H3 else None,
             b3=rng.normal(0.0, 0.1, H3) if H3 else None,
             w_out=rng.normal(0.0, 0.3, 1 + K + (H3 if H3 else H2)))
    c = {k: (np.ascontiguousarray(v, dtype=F32) if v is not None else None) for k, v in c.items()}
    if H3:
        c["W3"] = np.ascontiguousarray(c["W3"][:, :H3])
    c.update(H1=H1, H2=H2, H3=H3, lin_bias=float(F32(0.125)), b_out=float(F32(-0.3)))
    if fm_zero:   # the sequence models: zero FM / linear blocks and zero output weights over them
        for k in ("Su", "Qu", "lu", "Si", "Qi", "li"):
            c[k] = np.zeros_like(c[k])
        c["w_out"][:1 + K] = 0.0
        c["lin_bias"] = 0.0
    return c
