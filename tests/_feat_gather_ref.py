"""Float64 reference of K1, ``b200_feat_forward`` (include/b200reco.h, "a4/a5/a6: feature models"), its per-element
error bounds, float32 restatements used to calibrate those bounds, and a restatement of the host dispatch that picks
one of the six kernel families (csrc/feat.cu ``b200_feat_forward``, csrc/feat_tma.cu ``launch_feat_forward_tma``).

A case is a plain dict of numpy arrays:
    K, id_mask, sparse_side / sparse_col (one entry per sparse field), dense_side / dense_col / dense_embed_row (one
    per dense field), user_sparse_unique / item_sparse_unique (int32, [n_users+1 | n_items+1, columns]),
    user_dense_unique / item_dense_unique (float32), the eight float32 tables of ``b200_feat_tables`` and the head
    lin_kernel [F], lin_bias, bn_scale / bn_shift / pw_kernel [K], pw_bias.
Field order of a row: user id, item id (as ``id_mask`` keeps them), the sparse fields, the dense fields.  A sparse field
is a row of ``sparse_embeds`` (its linear feature ``sparse_linear`` of the same index); a dense field f with value x is
x * dense_embeds[dense_embed_row[f]] (linear feature x * dense_linear[dense_embed_row[f]]).

Outputs (every row r):  concat[r] = the F embeddings side by side; ssum = sum_f e; sqsum = sum_f e^2;
pw = (ssum^2 - sqsum) / 2; lin = sum_f lin_kernel[f] * linear feature f + lin_bias;
fm_out = lin + elu(sum_k pw_kernel[k] * (bn_scale[k] pw[k] + bn_shift[k]) + pw_bias) (no BN: bn_scale = 1, shift = 0).

Bounds: every output element computed in float32 in any summation order lies within c * u * n * sum|terms| of the
exact value (u = 2^-24, n = the number of rounded operations in the element's chain), propagated through pw and the
head; see ``bounds``.  tests/test_feat_gather_ref_cpu.py shows each holds with 4x to spare for three float32 summation
orders and that a one-field error breaks it."""
import numpy as np

U = 2.0 ** -24
C = 2.0          # the c of every c * u * n * sum|terms| bound (calibrated in tests/test_feat_gather_ref_cpu.py)
F32, F64 = np.float32, np.float64
MAX_FIELDS = 128
ASYNC_MAXS = 16
FT_MAX_RB, FT_NSTAGE = 8, 3
FT_MAX_FJ = (2 + 2 * MAX_FIELDS + 31) // 32


def n_fields(case):
    m = int(case["id_mask"])
    return (m & 1) + ((m >> 1) & 1) + len(case["sparse_side"]) + len(case["dense_side"])


def row_ids(users, items, R, grid_items=0, row_offset=0):
    """(user, item) of the R rows: explicit pairs, or rows row_offset.. of the grid users x range(grid_items)."""
    users = np.asarray(users, dtype=np.int64)
    if grid_items > 0:
        rg = np.arange(R, dtype=np.int64) + int(row_offset)
        return users[rg // grid_items], rg % grid_items
    return users[:R], np.asarray(items, dtype=np.int64)[:R]


def fields(case, u, it, sparse_rows=None, dense_rows=None, xpow=1):
    """Per-row field embeddings E [R, F, K] and linear features Lf [R, F], both float64 and EXACT (a dense field's
    x * e of two float32 values fits a float64), and the mask of the dense fields [F].  ``xpow`` = 2 applies a dense
    value twice (a seeded wrong kernel)."""
    K = int(case["K"])
    m = int(case["id_mask"])
    E, Lf, dense = [], [], []
    if m & 1:
        E.append(case["user_embeds"][u].astype(F64))
        Lf.append(case["user_linear"][u].astype(F64))
        dense.append(False)
    if m & 2:
        E.append(case["item_embeds"][it].astype(F64))
        Lf.append(case["item_linear"][it].astype(F64))
        dense.append(False)
    for f, (side, col) in enumerate(zip(case["sparse_side"], case["sparse_col"])):
        if sparse_rows is not None:
            idx = np.asarray(sparse_rows)[:, f].astype(np.int64)
        else:
            idx = (case["user_sparse_unique"][u, col] if side == 0 else case["item_sparse_unique"][it, col]).astype(np.int64)
        E.append(case["sparse_embeds"][idx].astype(F64))
        Lf.append(case["sparse_linear"][idx].astype(F64))
        dense.append(False)
    for f, (side, col) in enumerate(zip(case["dense_side"], case["dense_col"])):
        if dense_rows is not None:
            x = np.asarray(dense_rows)[:, f].astype(F64)
        else:
            x = (case["user_dense_unique"][u, col] if side == 0 else case["item_dense_unique"][it, col]).astype(F64)
        row = int(case["dense_embed_row"][f])
        E.append(x[:, None] ** xpow * case["dense_embeds"][row].astype(F64)[None, :])
        Lf.append(x * F64(case["dense_linear"][row]))
        dense.append(True)
    R = len(u)
    if not E:
        return np.zeros((R, 0, K)), np.zeros((R, 0)), np.zeros(0, dtype=bool)
    return np.stack(E, axis=1), np.stack(Lf, axis=1), np.asarray(dense)


def _head_terms(case, pw, bn):
    sc = case["bn_scale"].astype(F64) if bn else np.ones(pw.shape[1])
    sh = case["bn_shift"].astype(F64) if bn else np.zeros(pw.shape[1])
    return sc, sh, case["pw_kernel"].astype(F64)


def elu(z):
    return np.where(z > 0, z, np.expm1(np.minimum(z, 0)))


def ref(case, users, items=None, R=None, grid_items=0, row_offset=0, sparse_rows=None, dense_rows=None, bn=True):
    """Float64 outputs of b200_feat_forward for R rows and their error bounds (``bounds``).  ``concat`` is float32:
    each element is one float32 value of a table or one float32 product x * e, so the kernel must match it bit for
    bit."""
    R = len(users) if R is None else R
    u, it = row_ids(users, items, R, grid_items, row_offset)
    E, Lf, dense = fields(case, u, it, sparse_rows, dense_rows)
    F = E.shape[1]
    s, q = E.sum(axis=1), np.square(E).sum(axis=1)
    pw = 0.5 * (s * s - q)
    lk = case["lin_kernel"].astype(F64)[:F]
    lin = Lf @ lk + F64(case["lin_bias"])
    sc, sh, pk = _head_terms(case, pw, bn)
    z = (pw * sc + sh) @ pk + F64(case["pw_bias"])
    out = dict(concat=E.astype(F32).reshape(R, F * E.shape[2]), ssum=s, sqsum=q, pw=pw, lin=lin, z=z, fm_out=lin + elu(z))
    out["bound"] = bounds(case, E, Lf, s, q, pw, lin, z, bn)
    return out


def bounds(case, E, Lf, s, q, pw, lin, z, bn):
    """Per-element bounds |float32 result - exact| <= B for any summation order.
    ssum:  n = F + 1 (F - 1 additions, the rounding of a dense product x * e) over sum_f |e|.
    sqsum: n = F + 3 (F fused multiply-adds, the product's rounding doubled by the square) over sum_f e^2.
    pw:    (|s| + B_s) B_s + B_q / 2 (the errors of s and q through (s^2 - q) / 2) + u (s^2 + q + ...) (its own two
           roundings).
    lin:   n = F + 3 over sum_f |lin_kernel[f] * feature_f| + |lin_bias| (dense feature product, head product, sum).
    fm_out: B_lin + sum_k |pw_kernel[k] bn_scale[k]| B_pw[k] + u (K + 3) (sum_k |pw_kernel[k] (bn_scale[k] pw[k] +
           bn_shift[k])| + |pw_bias|) + 2u |elu| (expm1f) + u |lin + elu| (the final add); elu is 1-Lipschitz."""
    F, K = E.shape[1], E.shape[2]
    A1, A2 = np.abs(E).sum(axis=1), np.square(E).sum(axis=1)
    Bs = C * U * (F + 1) * A1
    Bq = C * U * (F + 3) * A2
    sb = np.abs(s) + Bs
    Bpw = sb * Bs + 0.5 * Bq + C * U * (sb * sb + A2 + Bq)
    lk = case["lin_kernel"].astype(F64)[:F]
    Blin = C * U * (F + 3) * (np.abs(Lf * lk).sum(axis=1) + abs(F64(case["lin_bias"])))
    sc, sh, pk = _head_terms(case, pw, bn)
    zk = np.abs(pk) * (np.abs(pw * sc) + np.abs(sh) + np.abs(sc) * Bpw)
    Bz = (np.abs(pk * sc) * Bpw).sum(axis=1) + C * U * (K + 3) * (zk.sum(axis=1) + abs(F64(case["pw_bias"])))
    e = elu(z)
    Bfm = Blin + Bz + C * U * (2 * np.abs(e) + np.abs(lin) + np.abs(e) + Blin + Bz)
    return dict(ssum=Bs, sqsum=Bq, pw=Bpw, lin=Blin, fm_out=Bfm)


def worst(got, want, bound):
    """max over elements of |got - want| / bound (> 1: the bound is broken); NaN counts as broken."""
    got = np.asarray(got, dtype=F64)
    err = np.abs(got - want)
    err = np.where(np.isnan(err), np.inf, err)
    return float((err / np.maximum(bound, np.finfo(F64).tiny)).max()) if err.size else 0.0


# ---- float32 restatements (calibration) -------------------------------------------------------------------------------
def _fma32(a, b, c):
    return (a.astype(F64) * b.astype(F64) + c.astype(F64)).astype(F32)


def _order(F, order, groups=8):
    """Field visiting order and, for "group", the field-group of each position: "field" 0..F-1, "reversed"
    F-1..0, "group" fields round-robin over ``groups`` groups summed in field order, then an xor-shuffle tree over
    the groups (the field-group and staged kernels with 32 / K4 groups)."""
    if order == "field":
        return np.arange(F), None
    if order == "reversed":
        return np.arange(F)[::-1], None
    return np.arange(F), np.arange(F) % groups


def _sum32(vals, order, groups=8, sq=False):
    """float32 sum (sq: fma(v, v, acc)) over axis 1 of vals [R, F, ...] in the given order."""
    F = vals.shape[1]
    idx, grp = _order(F, order, groups)
    G = 1 if grp is None else groups
    acc = np.zeros((G, vals.shape[0]) + vals.shape[2:], dtype=F32)
    for p, f in enumerate(idx):
        g = 0 if grp is None else grp[p]
        v = vals[:, f]
        acc[g] = _fma32(v, v, acc[g]) if sq else (acc[g] + v).astype(F32)
    off = 1
    while off < G:                      # xor-shuffle tree: every group ends with the same total
        acc = (acc + acc[np.arange(G) ^ off]).astype(F32)
        off <<= 1
    return acc[0]


def restate32(case, users, items=None, R=None, grid_items=0, row_offset=0, sparse_rows=None, dense_rows=None,
              bn=True, order="field", mutate=None):
    """b200_feat_forward in float32 in one summation order.  ``mutate`` names a seeded wrong kernel (value changes
    only): "drop_field" (the last field left out of the sums), "no_bn_shift", "relu" (elu -> relu),
    "ignore_row_offset", "dense_twice" (a dense field's value applied twice)."""
    R = len(users) if R is None else R
    off = 0 if mutate == "ignore_row_offset" else row_offset
    u, it = row_ids(users, items, R, grid_items, off)
    E64, L64, dense = fields(case, u, it, sparse_rows, dense_rows, xpow=2 if mutate == "dense_twice" else 1)
    E = E64.astype(F32)                 # one rounding of x * e
    Lf = L64.astype(F32)                # one rounding of x * dense_linear
    F = E.shape[1]
    if mutate == "drop_field":
        E, Lf = E[:, : F - 1], Lf[:, : F - 1]
    s = _sum32(E, order)
    q = _sum32(E, order, sq=True)
    pw = (F32(0.5) * (s * s - q).astype(F32)).astype(F32)
    lk = case["lin_kernel"].astype(F32)[: Lf.shape[1]]
    lin = (_sum32((Lf * lk).astype(F32), order) + F32(case["lin_bias"])).astype(F32)
    sc = case["bn_scale"].astype(F32) if bn else np.ones(pw.shape[1], F32)
    sh = case["bn_shift"].astype(F32) if bn and mutate != "no_bn_shift" else np.zeros(pw.shape[1], F32)
    zk = _fma32(pw, np.broadcast_to(sc, pw.shape), np.broadcast_to(sh, pw.shape))
    acc = np.zeros(R, F32)
    for k in range(pw.shape[1]):
        acc = _fma32(zk[:, k], np.full(R, case["pw_kernel"][k], F32), acc)
    z = (acc + F32(case["pw_bias"])).astype(F32)
    act = np.maximum(z, F32(0)) if mutate == "relu" else np.where(z > 0, z, np.expm1(np.minimum(z, F32(0))))
    fm = (lin + act.astype(F32)).astype(F32)
    return dict(concat=E.reshape(R, E.shape[1] * E.shape[2]), ssum=s, sqsum=q, pw=pw, lin=lin, fm_out=fm)


# ---- dispatch ------------------------------------------------------------------------------------------------------
def _tma_eligible(K, R, F):
    if K % 4 or K > 32 or R < 2048 or F < 1 or F > 32 * FT_MAX_FJ or (K // 4) not in (1, 2, 4, 8):
        return False
    row_bytes, aux_bytes = F * K * 4, (F * 8 + 15) & ~15
    RB = FT_MAX_RB
    while RB > 1 and FT_NSTAGE * RB * (row_bytes + aux_bytes) > 100 * 1024:
        RB >>= 1
    return 128 + FT_NSTAGE * RB * (row_bytes + aux_bytes) + 2 * FT_NSTAGE * 8 + 64 <= 220 * 1024


def _async_fits(K4, F, NS):
    FPW = 32 // K4
    per_warp = 2 * NS * 512 + 2 * 2 * NS * FPW * 4
    meta = F * 8 + NS * FPW * 4
    best = 0
    for wpb in range(8, 1, -1):
        nb = min((228 * 1024) // (wpb * per_warp + meta + 1024), 16 // wpb)
        best = max(best, nb * wpb)
    return best >= 8


def expected_kernel(K, R, F, aligned=True, explicit_rows=False, tune=0):
    """(family, template argument) of the kernel b200_feat_forward launches: family one of "generic",
    "lanefield", "fieldgroup", "pipe", "async", "tma" (template argument K / 4; None for generic), or ("none", None)
    when R == 0.  ``aligned``: every table and the concat 16-byte aligned and ld_concat % 4 == 0; ``tune``: the
    b200_feat_forward_tune code (bit 0 TMA, bit 1 lane-per-field, bit 2 no staged kernel, bit 3 cp.async)."""
    if R == 0:
        return "none", None
    K4 = K // 4
    fast = K % 4 == 0 and K <= 32 and aligned
    if fast and tune & 1 and _tma_eligible(K, R, F):
        return "tma", K4
    group_ok = fast and not tune & 2 and K4 in (1, 2, 4, 8)
    staged_ok = group_ok and not tune & 4 and R >= 4096 and not explicit_rows
    NS = -(-F // (32 // K4)) if group_ok else 0
    if staged_ok and not tune & 8 and NS <= 16:
        return "pipe", K4
    if staged_ok and tune & 8 and NS <= ASYNC_MAXS and _async_fits(K4, F, NS):
        return "async", K4
    if group_ok:
        return "fieldgroup", K4
    if fast:
        return "lanefield", K4
    return "generic", None


KERNEL_NAMES = {"generic": "feat_forward_kernel", "lanefield": "feat_forward_lanefield_kernel",
                "fieldgroup": "feat_forward_fieldgroup_kernel", "pipe": "feat_forward_pipe_kernel",
                "async": "feat_forward_async_kernel", "tma": "feat_forward_tma_kernel"}


def kernel_of(name):
    """(family, template argument) of a profiler kernel name, demangled ("...feat_forward_pipe_kernel<4>(...") or
    mangled ("...24feat_forward_pipe_kernelILi4EE..."); None for a kernel that is not K1's."""
    import re

    for fam, base in KERNEL_NAMES.items():
        if fam == "generic":
            if re.search(base + r"(?:\(|E)", name):
                return fam, None
            continue
        m = re.search(base + r"(?:<(\d+)>|ILi(\d+)E)", name)
        if m:
            return fam, int(m.group(1) or m.group(2))
    return None


# ---- cases -----------------------------------------------------------------------------------------------------------
def make_case(rng, K, n_us=0, n_is=0, n_ud=0, n_id=0, id_mask=3, n_users=300, n_items=400, vocab=500,
              dense_scale=1.0, dense_row_perm=False, pw_bias_center=True, elu_negative=True):
    """A random layout: n_us / n_is sparse fields from the user / item unique tables (interleaved columns, some
    index-0 entries), n_ud / n_id dense fields (values with zeros and negatives, times ``dense_scale``), tables with
    an OOV row (n_users / n_items), a BN head with shifts far from 0."""
    f32 = lambda *s: rng.standard_normal(s).astype(F32)
    ns, nd = n_us + n_is, n_ud + n_id
    sparse_side = np.array([0] * n_us + [1] * n_is, dtype=np.int32)
    rng.shuffle(sparse_side)
    sparse_col = np.zeros(ns, np.int32)
    for side, n in ((0, n_us), (1, n_is)):
        sparse_col[sparse_side == side] = np.arange(n)
    dense_side = np.array([0] * n_ud + [1] * n_id, dtype=np.int32)
    rng.shuffle(dense_side)
    dense_col = np.zeros(nd, np.int32)
    for side, n in ((0, n_ud), (1, n_id)):
        dense_col[dense_side == side] = np.arange(n)
    dense_embed_row = rng.permutation(nd).astype(np.int32) if dense_row_perm else np.arange(nd, dtype=np.int32)

    def uniq_sparse(n_rows, ncol):
        t = rng.integers(0, vocab, (n_rows, max(ncol, 1))).astype(np.int32)
        t[rng.random(t.shape) < 0.05] = 0
        return t

    def uniq_dense(n_rows, ncol):
        t = (rng.standard_normal((n_rows, max(ncol, 1))) * dense_scale).astype(F32)
        t[rng.random(t.shape) < 0.05] = 0
        return t

    F = (id_mask & 1) + ((id_mask >> 1) & 1) + ns + nd
    case = dict(K=K, id_mask=id_mask, sparse_side=sparse_side, sparse_col=sparse_col, dense_side=dense_side,
                dense_col=dense_col, dense_embed_row=dense_embed_row,
                user_sparse_unique=uniq_sparse(n_users + 1, n_us), item_sparse_unique=uniq_sparse(n_items + 1, n_is),
                user_dense_unique=uniq_dense(n_users + 1, n_ud), item_dense_unique=uniq_dense(n_items + 1, n_id),
                user_embeds=f32(n_users + 1, K) * F32(0.3), item_embeds=f32(n_items + 1, K) * F32(0.3),
                sparse_embeds=f32(vocab, K) * F32(0.3), dense_embeds=f32(max(nd, 1), K) * F32(0.3),
                user_linear=f32(n_users + 1), item_linear=f32(n_items + 1), sparse_linear=f32(vocab),
                dense_linear=f32(max(nd, 1)) + F32(0.1),
                lin_kernel=f32(max(F, 1)) * F32(0.5), lin_bias=F32(0.25),
                bn_scale=(np.abs(f32(K)) + F32(0.5)), bn_shift=f32(K) * F32(0.5),
                pw_kernel=f32(K) * F32(1.0 / np.sqrt(K)), pw_bias=F32(0.0))
    if pw_bias_center:
        # centre the head's pre-activation so that both sides of elu (z > 0 and the expm1 side) are exercised
        uu = rng.integers(0, n_users + 1, 256)
        ii = rng.integers(0, n_items + 1, 256)
        z = ref(case, uu, ii)["z"]
        case["pw_bias"] = F32(-np.median(z) if elu_negative else 0.0)
    return case


def case_from_spec(spec, w, K, fold_dtype=F32):
    """The case of an FM model built by librecommender_b200.synthetic (make_spec / make_fm_weights): the layout the
    model's FeatSpec builds (sparse / dense field f from the side that owns column f) and its BN folded to
    scale / shift (in ``fold_dtype``; float64 keeps the fold exact for cross-checks)."""
    from oracle import tf_models as tm

    case = dict(K=K, id_mask=3)
    for kind in ("sparse", "dense"):
        side, col = tm.field_index(spec, None, None, kind)
        case[f"{kind}_side"], case[f"{kind}_col"] = side, col
        for s in ("user", "item"):
            t = spec.get(f"{s}_{kind}_unique")
            n = spec["n_users" if s == "user" else "n_items"] + 1
            case[f"{s}_{kind}_unique"] = t if t is not None else np.zeros((n, 1), np.int32 if kind == "sparse" else F32)
    case["dense_embed_row"] = np.arange(spec["n_dense"], dtype=np.int32)
    for name in ("user_embeds", "item_embeds", "sparse_embeds", "user_linear", "item_linear", "sparse_linear"):
        case[name] = np.asarray(w[name], dtype=F32)
    for name in ("dense_embeds", "dense_linear"):
        case[name] = np.asarray(w[name], dtype=F32) if spec["n_dense"] else np.zeros((1, K) if name == "dense_embeds" else 1, F32)
    case.update(lin_kernel=np.asarray(w["lin_kernel"], F32).reshape(-1), lin_bias=F32(w["lin_bias"]),
                pw_kernel=np.asarray(w["pw_kernel"], F32).reshape(-1), pw_bias=F32(w["pw_bias"]))
    bn = w.get("fm_bn")
    if bn is not None:
        g, b, m, v = (np.asarray(bn[k], dtype=fold_dtype) for k in ("gamma", "beta", "mean", "var"))
        scale = g / np.sqrt(v + fold_dtype(tm.BN_EPS))
        case.update(bn_scale=scale, bn_shift=b - m * scale)
    else:
        case.update(bn_scale=np.ones(K, F32), bn_shift=np.zeros(K, F32))
    return case
