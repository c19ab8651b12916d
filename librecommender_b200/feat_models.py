"""Inference engines for the reference's feature ("TfBase") models on the GPU: FM, DeepFM
(``libreco/algorithms/fm.py``, ``deepfm.py``) — forward (``predict``) and all-items scoring
(``recommend_user`` = ``recommend_tf_feat``, ``libreco/recommendation/recommend.py:81-105``).

* The per-row feed the reference materialises on the host (``process_tf_feat`` /
  ``get_original_feats``) is never built: ``b200_feat_forward`` reads the per-user / per-item
  unique feature tables in the kernel, and for all-items scoring rows are the implicit grid
  (user, item 0..N-1).
* BatchNorm layers are folded into scale/shift (inference = moving statistics, TF defaults
  epsilon 1e-3) and, inside ``dense_nn``, into the following Dense layer.
* Weights arrive as a dict with the keys of ``WEIGHT_KEYS`` (numpy arrays) — see
  ``from_tf_variables`` for the mapping from a reference ``*_tf_variables.npz``.
"""
from __future__ import annotations

import ctypes
from ctypes import Structure, c_int32, c_int64, c_void_p

import numpy as np

from . import _lib
from .consumed import ConsumedCSR, as_csr
from .engine import masked_topk

MAX_FIELDS = 128
BN_EPS = 1e-3

WEIGHT_KEYS = (
    "user_embeds", "item_embeds", "sparse_embeds", "dense_embeds",
    "user_linear", "item_linear", "sparse_linear", "dense_linear",
    "lin_kernel", "lin_bias", "pw_kernel", "pw_bias", "fm_bn", "mlp", "out_kernel", "out_bias",
)


class FeatLayoutStruct(Structure):
    _fields_ = [
        ("embed_size", c_int32), ("n_sparse", c_int32), ("n_dense", c_int32),
        ("id_mask", c_int32), ("dense_embed_row", c_int32 * MAX_FIELDS),
        ("sparse_side", c_int32 * MAX_FIELDS), ("sparse_col", c_int32 * MAX_FIELDS),
        ("dense_side", c_int32 * MAX_FIELDS), ("dense_col", c_int32 * MAX_FIELDS),
        ("user_sparse_unique", c_void_p), ("ld_us", c_int64),
        ("item_sparse_unique", c_void_p), ("ld_is", c_int64),
        ("user_dense_unique", c_void_p), ("ld_ud", c_int64),
        ("item_dense_unique", c_void_p), ("ld_id", c_int64),
        ("sparse_rows", c_void_p), ("ld_sparse_rows", c_int64),
        ("dense_rows", c_void_p), ("ld_dense_rows", c_int64),
    ]


class FeatTablesStruct(Structure):
    _fields_ = [(n, c_void_p) for n in ("user_embeds", "item_embeds", "sparse_embeds", "dense_embeds",
                                        "user_linear", "item_linear", "sparse_linear", "dense_linear")]


def _dev(x, device, dtype):
    import torch

    if x is None:
        return None
    if isinstance(x, torch.Tensor):
        return x.to(device=device, dtype=dtype).contiguous()
    return torch.as_tensor(np.ascontiguousarray(x)).to(device=device, dtype=dtype).contiguous()


def tables_struct(tensors):
    """FeatTablesStruct over the device tables in the dict ``tensors`` (missing or None: NULL)."""
    T = FeatTablesStruct()
    for name, _ in FeatTablesStruct._fields_:
        t = tensors.get(name)
        setattr(T, name, t.data_ptr() if t is not None else None)
    return T


def _ld(t):
    return t.stride(0) if t is not None else 0


def feat_forward(layout, tables, users, items, R, *, grid_items=0, row_offset=0, concat=None, pw=None, lin=None,
                 fm_out=None, lin_kernel=None, lin_bias=0.0, head=None, ssum=None, sqsum=None):
    """K1, ``b200_feat_forward``: gathers the field embeddings of R (user, item) rows — explicit ``users`` /
    ``items``, or rows ``row_offset`` .. of the implicit grid of every user with items 0..``grid_items``-1 — into whichever outputs are given: the concat [R, F*K], the FM pairwise block ``pw``
    [R, K], the linear term ``lin`` (``lin_kernel``, ``lin_bias``), FM's whole output ``fm_out`` (``head``: BN
    scale / shift, pw kernel / bias) and the field sums ``ssum`` / ``sqsum`` [R, K]."""
    head = head or {}
    _lib.check(_lib.lib.b200_feat_forward(
        ctypes.byref(layout), ctypes.byref(tables), _lib.ptr(users), _lib.ptr(items), R, grid_items, row_offset,
        _lib.ptr(concat), _ld(concat), _lib.ptr(pw), _ld(pw), _lib.ptr(lin), _lib.ptr(fm_out), _lib.ptr(lin_kernel),
        float(lin_bias), _lib.ptr(head.get("bn_scale")), _lib.ptr(head.get("bn_shift")),
        _lib.ptr(head.get("pw_kernel")), float(head.get("pw_bias", 0.0)), _lib.ptr(ssum), _lib.ptr(sqsum), _ld(ssum),
        _lib.current_stream()))


def feat_backward(layout, tables, users, items, R, grads, *, dpw=None, S=None, dconcat=None, dlogit=None,
                  lin_kernel=None):
    """Backward of :func:`feat_forward` (``b200_feat_backward``): the field gradients of the FM block (``dpw``,
    ``S``), of the concat (``dconcat``) and of the linear term (``dlogit``, ``lin_kernel``) scatter-ADDED into the
    buffers of ``grads`` named like the tables (and ``lin_kernel``); absent names are skipped."""
    _lib.check(_lib.lib.b200_feat_backward(
        ctypes.byref(layout), ctypes.byref(tables), _lib.ptr(users), _lib.ptr(items), R, _lib.ptr(dpw), _ld(dpw),
        _lib.ptr(S), _ld(S), _lib.ptr(dconcat), _ld(dconcat), _lib.ptr(dlogit), _lib.ptr(lin_kernel),
        *[_lib.ptr(grads.get(name)) for name, _ in FeatTablesStruct._fields_], _lib.ptr(grads.get("lin_kernel")),
        _lib.current_stream()))


# Dense-layer kernel selection: "auto" sends layers that are compute-bound on the SIMT kernel
# (din >= TC_MIN_DIN, enough rows to fill the SMs) to the wgmma 3xTF32 kernel; both are this
# library's own CUDA kernels and both meet the 1e-5 bar.  "f32" / "tf32x3" force one (tests).
LINEAR_IMPL = "auto"
TC_MIN_DIN = 64
TC_MIN_ROWS = 4096
TC_MIN_MACS = 1 << 27
DIN_FUSED_ATTENTION = False   # DIN all-items: sigmoid / Dense(1) fused into the attention GEMM's epilogue.  Measured
# (profiles/r02_launches_din_*.csv): no gain — the fused GEMM 524 us + softmax kernel 242 us per user vs 359 + 395 us
# for the [N, 16 len] round trip; the per-tile cost of the K = 64 product dominates either way.  Kept as a tested variant.
TC_LONG_K = 1024        # long reductions (weight gradients over the batch) starve the SIMT kernel's few CTAs


_SPLIT_CACHE = {}


def split_weights(Wt):
    """hi / lo tf32 copies of a layer's weights for b200_linear_tf32x3, made once per weight tensor
    (keyed by storage pointer + shape + version counter, so in-place updates re-split)."""
    import torch

    dout, din = Wt.shape
    ldw = Wt.stride(0) if dout > 1 else din      # one row: torch's row stride is arbitrary
    key = (Wt.data_ptr(), tuple(Wt.shape), ldw, Wt._version)
    hit = _SPLIT_CACHE.get(key)
    if hit is None:
        ld = int(_lib.lib.b200_linear_tf32x3_split_ld(din))
        buf = torch.empty(2 * dout * ld, dtype=torch.float32, device=Wt.device)
        _lib.check(_lib.lib.b200_linear_tf32x3_split_weights(_lib.ptr(Wt), ldw, din, dout, _lib.ptr(buf),
                                                             _lib.current_stream()))
        if len(_SPLIT_CACHE) > 256:
            _SPLIT_CACHE.clear()
        hit = _SPLIT_CACHE[key] = (buf, Wt)      # keep Wt alive so the pointer key stays unique
    return hit[0]


ACT_NONE, ACT_RELU, ACT_SWISH = 0, 1, 2     # activation codes of b200_linear_* (include/b200reco.h)
ACT_GELU = 3                                # b200_activation_* only: the erf gelu


def _row_major(t, name):
    """``t`` as the dense kernels read a matrix operand — float32 CUDA rows with unit inner stride, a copy when the
    view is transposed or its rows overlap (a broadcast) — and its leading dimension.  Torch gives a single row an
    arbitrary row stride (``y.t()`` of an [n, 1] column has stride 1), so one row reads as ``ld`` = its width."""
    import torch

    if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or not t.is_cuda or t.dim() != 2:
        raise ValueError(f"linear: {name} must be a 2-D float32 CUDA tensor, got "
                         f"{getattr(t, 'dtype', type(t).__name__)} {tuple(getattr(t, 'shape', ()))} on "
                         f"{getattr(t, 'device', 'host')}")
    if (t.shape[1] > 1 and t.stride(1) != 1) or (t.shape[0] > 1 and t.stride(0) < t.shape[1]):
        t = t.contiguous()
    return t, (t.stride(0) if t.shape[0] > 1 else t.shape[1])


def linear(x, Wt, b, act, cache_split=True, impl=None):
    """tf_dense (libreco/layers/dense.py:52-80) with BN folded: act(x Wt^T + b), fp32 device tensors.  ``act`` is an
    activation code (a bool reads as relu on / off): 0 none, 1 relu, 2 swish.  ``impl`` overrides ``LINEAR_IMPL``
    for this call ("f32": one fmaf chain per output, so a row's bits do not depend on how many rows come with it).
    Any strided view works (a transposed ``x`` or ``Wt`` is copied); another dtype or a host tensor raises
    ``ValueError``."""
    import torch

    impl = LINEAR_IMPL if impl is None else impl
    x, ldx = _row_major(x, "x")
    Wt_in = Wt
    Wt, ldw = _row_major(Wt, "Wt")
    cache_split = cache_split and Wt is Wt_in      # a fresh copy would only fill the split cache
    if b is not None:
        if not isinstance(b, torch.Tensor) or b.dtype != torch.float32 or not b.is_cuda:
            raise ValueError(f"linear: b must be a float32 CUDA tensor, got {getattr(b, 'dtype', type(b).__name__)} "
                             f"on {getattr(b, 'device', 'host')}")
        b = b.contiguous()
    R, din, dout = x.shape[0], Wt.shape[1], Wt.shape[0]
    y = torch.empty((R, dout), dtype=torch.float32, device=x.device)
    bp = _lib.ptr(b) if b is not None else None
    aligned = ldx % 4 == 0 and x.data_ptr() % 16 == 0
    # few output rows but a long reduction (the weight gradients dWt = dY^T X of the training steps: 128 x 1792
    # outputs over 8192 rows) would run on a handful of SIMT CTAs: send those to the tensor-core kernel too
    use_tc = impl == "tf32x3" or (impl == "auto" and din >= TC_MIN_DIN and
                                  (R >= TC_MIN_ROWS or din >= TC_LONG_K or R * din * dout >= TC_MIN_MACS))
    w_ok = cache_split or (ldw % 4 == 0 and Wt.data_ptr() % 16 == 0)
    if use_tc and aligned and w_ok and not cache_split and din >= TC_LONG_K:
        # few output tiles, long reduction: split the reduction over enough CTAs to fill the SMs
        tiles = -(-R // 128) * -(-dout // 128)
        sms = torch.cuda.get_device_properties(x.device).multi_processor_count
        splits = max(1, min(16, sms // tiles, din // 256))
        if splits > 1:
            part = torch.empty(splits * R * dout, dtype=torch.float32, device=x.device)
            _lib.check(_lib.lib.b200_linear_tf32x3_splitk(_lib.ptr(x), ldx, R, _lib.ptr(Wt), ldw, bp, din,
                                                          dout, int(act), splits, _lib.ptr(part),
                                                          part.numel() * 4, _lib.ptr(y), y.stride(0),
                                                          _lib.current_stream()))
            return y
    if use_tc and aligned and w_ok:
        ws = split_weights(Wt) if cache_split else None
        _lib.check(_lib.lib.b200_linear_tf32x3(_lib.ptr(x), ldx, R, _lib.ptr(Wt), ldw, _lib.ptr(ws), bp,
                                               din, dout, int(act), _lib.ptr(y), y.stride(0),
                                               _lib.current_stream()))
    else:
        _lib.check(_lib.lib.b200_linear_f32(_lib.ptr(x), ldx, R, _lib.ptr(Wt), ldw, bp, din, dout,
                                            int(act), _lib.ptr(y), y.stride(0), _lib.current_stream()))
    return y


def _side_cols(user_cols, item_cols):
    n = len(user_cols) + len(item_cols)
    side, col = [0] * n, [0] * n
    for f in range(n):
        if f in user_cols:
            side[f], col[f] = 0, list(user_cols).index(f)
        else:
            side[f], col[f] = 1, list(item_cols).index(f)
    return side, col


def fold_bn(bn):
    """BN(x) = x * scale + shift at inference."""
    if bn is None:
        return None, None
    scale = (bn["gamma"] / np.sqrt(bn["var"] + np.float32(BN_EPS))).astype(np.float32)
    shift = (bn["beta"] - bn["mean"] * scale).astype(np.float32)
    return scale, shift


def fold_mlp(mlp, act=ACT_RELU):
    """dense_nn (libreco/layers/dense.py:12-49) -> [(Wt [dout, din], bias, act)], BN folded into
    the Dense that FOLLOWS it: Dense(BN(a)) = a (diag(s) W) + (t W + b).  ``act``: the activation code of the
    hidden layers (relu, or swish for the Transformer); the last layer has none."""
    layers = []
    scale, shift = fold_bn(mlp.get("bn_in"))
    n = len(mlp["kernels"])
    for i in range(n):
        W = np.asarray(mlp["kernels"][i], dtype=np.float32)
        b = np.asarray(mlp["biases"][i], dtype=np.float32)
        if scale is not None:
            b = (shift @ W + b).astype(np.float32)
            W = (scale[:, None] * W).astype(np.float32)
        layers.append((np.ascontiguousarray(W.T), b, i != n - 1 if act == ACT_RELU else (act if i != n - 1 else 0)))
        scale, shift = (None, None)
        if i != n - 1 and mlp.get("bns"):
            scale, shift = fold_bn(mlp["bns"][i])
    return layers


_COMBINERS = {"sum": 0, "mean": 1, "sqrtn": 2}


def _spec_get(spec):
    """Uniform read access to a layout description: a plain dict (tests, fixtures) or the reference's
    ``DataInfo`` object (libreco/data/data_info.py:107-290), whose column indices live in
    ``data_info.user_sparse_col.index`` etc. (`Feature(name, index)` tuples, :209-247)."""
    if isinstance(spec, dict):
        return spec.get

    def g(k, d=None):
        if k.endswith("_col_index") and not hasattr(spec, k):
            feat = getattr(spec, k[: -len("_index")], None)
            return list(feat.index) if feat is not None and getattr(feat, "index", None) is not None else d
        v = getattr(spec, k, d)
        return d if v is None else v

    return g


def combine_multi_sparse(spec, weights, combiner="sqrtn", device=None):
    """multi_sparse_combine_embedding (libreco/tfops/features.py:47-118) hoisted out of the row path.

    A multi-sparse field (e.g. genre1..genre3 sharing one vocabulary and one OOV slot) is a function
    of the user or of the item only, so its pooled embedding / pooled linear weight is computed ONCE
    per unique-table row (``b200_multi_sparse_combine``) and appended to the shared sparse tables;
    the field then is an ordinary single-index field for every downstream kernel.  Returns
    ``(spec_dict, weights_dict)`` in the reduced field layout the reference's graph uses after
    combining (``true_sparse_field_size``, feature/multi_sparse.py:146-157): plain sparse fields
    first, then one field per multi-sparse group.  With ``combiner="normal"`` or no multi-sparse info
    the inputs are returned unchanged."""
    import torch

    g = _spec_get(spec)
    info = g("multi_sparse_combine_info")
    if info is None or combiner not in _COMBINERS:
        return spec, weights
    ig = info.get if isinstance(info, dict) else (lambda k, d=None: getattr(info, k, d))
    offs, lens, oovs = list(ig("field_offset")), list(ig("field_len")), [int(x) for x in ig("feat_oov")]
    device = device if device is not None else _lib.require_cuda()
    ucol, icol = list(g("user_sparse_col_index") or []), list(g("item_sparse_col_index") or [])
    sparse_end = offs[0]
    E = _dev(weights["sparse_embeds"], device, torch.float32)
    K = E.shape[1]
    lin = _dev(weights.get("sparse_linear"), device, torch.float32)
    uniq = {"user": _dev(g("user_sparse_unique"), device, torch.int32) if ucol else None,
            "item": _dev(g("item_sparse_unique"), device, torch.int32) if icol else None}
    cols = {"user": ucol, "item": icol}
    new_cols = {"user": [c for c in ucol if c < sparse_end], "item": [c for c in icol if c < sparse_end]}
    new_uniq = {w: [uniq[w][:, [cols[w].index(c) for c in new_cols[w]]]] if new_cols[w] else [] for w in ("user", "item")}
    add_e, add_l, base = [], [], E.shape[0]
    for gi, (off, ln, oov) in enumerate(zip(offs, lens, oovs)):
        which = "user" if off in ucol else "item"
        members = list(range(off, off + ln))
        if any(c not in cols[which] for c in members):
            raise ValueError(f"multi-sparse field at offset {off} straddles the user / item sides")
        idx = uniq[which][:, [cols[which].index(c) for c in members]].contiguous()
        n = idx.shape[0]
        ce = torch.empty((n, K), dtype=torch.float32, device=device)
        _lib.check(_lib.lib.b200_multi_sparse_combine(_lib.ptr(E), E.stride(0), K, _lib.ptr(idx), idx.stride(0), ln, n,
                                                      oov, _COMBINERS[combiner], _lib.ptr(ce), ce.stride(0),
                                                      _lib.current_stream()))
        add_e.append(ce)
        if lin is not None:
            cl = torch.empty(n, dtype=torch.float32, device=device)
            _lib.check(_lib.lib.b200_multi_sparse_combine(_lib.ptr(lin), 1, 1, _lib.ptr(idx), idx.stride(0), ln, n, oov,
                                                          _COMBINERS[combiner], _lib.ptr(cl), 1, _lib.current_stream()))
            add_l.append(cl)
        new_uniq[which].append((base + torch.arange(n, device=device, dtype=torch.int32)).view(-1, 1))
        new_cols[which].append(sparse_end + gi)
        base += n
    out_spec = {k: g(k) for k in ("n_users", "n_items", "user_dense_col_index", "item_dense_col_index",
                                  "user_dense_unique", "item_dense_unique")}
    out_spec.update(user_sparse_col_index=new_cols["user"], item_sparse_col_index=new_cols["item"],
                    user_sparse_unique=torch.cat(new_uniq["user"], dim=1).contiguous() if new_uniq["user"] else None,
                    item_sparse_unique=torch.cat(new_uniq["item"], dim=1).contiguous() if new_uniq["item"] else None,
                    n_sparse=sparse_end + len(offs), n_dense=g("n_dense"), multi_sparse_combine_info=None)
    out_w = dict(weights)
    out_w["sparse_embeds"] = torch.cat([E] + add_e, dim=0)
    if lin is not None:
        out_w["sparse_linear"] = torch.cat([lin] + add_l, dim=0)
    return out_spec, out_w


class FeatSpec:
    """Device-resident feature layout (from the reference's DataInfo or an equivalent dict)."""

    def __init__(self, spec, embed_size, device=None):
        import torch

        self.device = device if device is not None else _lib.require_cuda()
        g = _spec_get(spec)
        self.n_users, self.n_items = int(g("n_users")), int(g("n_items"))
        ucol, icol = list(g("user_sparse_col_index") or []), list(g("item_sparse_col_index") or [])
        udc, idc = list(g("user_dense_col_index") or []), list(g("item_dense_col_index") or [])
        self.n_sparse, self.n_dense = len(ucol) + len(icol), len(udc) + len(idc)
        if self.n_sparse > MAX_FIELDS or self.n_dense > MAX_FIELDS:
            raise ValueError("too many feature fields")
        self.us = _dev(g("user_sparse_unique"), self.device, torch.int32) if ucol else None
        self.is_ = _dev(g("item_sparse_unique"), self.device, torch.int32) if icol else None
        self.ud = _dev(g("user_dense_unique"), self.device, torch.float32) if udc else None
        self.id_ = _dev(g("item_dense_unique"), self.device, torch.float32) if idc else None
        L = FeatLayoutStruct()
        L.embed_size, L.n_sparse, L.n_dense = int(embed_size), self.n_sparse, self.n_dense
        L.id_mask = 3
        for f in range(self.n_dense):
            L.dense_embed_row[f] = f
        side, col = _side_cols(ucol, icol)
        for f in range(self.n_sparse):
            L.sparse_side[f], L.sparse_col[f] = side[f], col[f]
        side, col = _side_cols(udc, idc)
        for f in range(self.n_dense):
            L.dense_side[f], L.dense_col[f] = side[f], col[f]
        for name, t in (("user_sparse_unique", self.us), ("item_sparse_unique", self.is_),
                        ("user_dense_unique", self.ud), ("item_dense_unique", self.id_)):
            setattr(L, name, t.data_ptr() if t is not None else None)
        L.ld_us = self.us.stride(0) if self.us is not None else 0
        L.ld_is = self.is_.stride(0) if self.is_ is not None else 0
        L.ld_ud = self.ud.stride(0) if self.ud is not None else 0
        L.ld_id = self.id_.stride(0) if self.id_ is not None else 0
        L.sparse_rows, L.dense_rows = None, None
        self.layout = L
        self.item_sparse_cols, self.item_dense_cols = icol, idc
        self.user_sparse_cols, self.user_dense_cols = ucol, udc
        self._sides = {}

    def side(self, which, with_id=True):
        """(layout restricted to the fields of one side, ``which`` = "user" or "item", and their positions in the
        global field order [user, item, sparse.., dense..]), built once.  ``with_id=False`` leaves out the side's
        id field."""
        key = (which, with_id)
        if key not in self._sides:
            s = 0 if which == "user" else 1
            scols = self.user_sparse_cols if s == 0 else self.item_sparse_cols
            dcols = self.user_dense_cols if s == 0 else self.item_dense_cols
            L = FeatLayoutStruct.from_buffer_copy(self.layout)
            L.id_mask = (1 << s) if with_id else 0
            L.n_sparse, L.n_dense = len(scols), len(dcols)
            for f in range(len(scols)):
                L.sparse_side[f], L.sparse_col[f] = s, f
            for f in range(len(dcols)):
                L.dense_side[f], L.dense_col[f] = s, f
                L.dense_embed_row[f] = dcols[f]
            pos = ([s] if with_id else []) + [2 + c for c in scols] + [2 + self.n_sparse + c for c in dcols]
            self._sides[key] = (L, pos)
        return self._sides[key]

    def with_rows(self, sparse_rows, dense_rows):
        """Layout copy that reads explicit per-row features (predict with given feature rows)."""
        L = FeatLayoutStruct.from_buffer_copy(self.layout)
        if sparse_rows is not None:
            L.sparse_rows, L.ld_sparse_rows = sparse_rows.data_ptr(), sparse_rows.stride(0)
        if dense_rows is not None:
            L.dense_rows, L.ld_dense_rows = dense_rows.data_ptr(), dense_rows.stride(0)
        return L


class _FeatModelBase:
    """Shared machinery: device tables, row forward, all-items scoring + masked top-K."""

    needs_linear = True

    def __init__(self, spec, weights, user_consumed=None, task="ranking", device=None):
        import torch

        self._torch = torch
        K = int(weights["user_embeds"].shape[1])
        if not isinstance(spec, FeatSpec):   # multi-sparse fields pooled once (default combiner as the reference's)
            spec, weights = combine_multi_sparse(spec, weights, weights.get("multi_sparse_combiner", "sqrtn"), device)
        self.spec = spec if isinstance(spec, FeatSpec) else FeatSpec(spec, K, device)
        self.device = self.spec.device
        self.K = K
        self.task = task
        self.n_users, self.n_items = self.spec.n_users, self.spec.n_items
        self.F = 2 + self.spec.n_sparse + self.spec.n_dense
        f32 = torch.float32
        self.t = {k: _dev(weights.get(k), self.device, f32) for k, _ in FeatTablesStruct._fields_}
        self.tables = tables_struct(self.t)
        if self.needs_linear:
            self.lin_kernel = _dev(np.asarray(weights["lin_kernel"]).reshape(-1), self.device, f32)
            self.lin_bias = float(np.asarray(weights["lin_bias"]).reshape(-1)[0])
        csr = user_consumed if user_consumed is not None else ConsumedCSR(
            np.zeros(1, dtype=np.int64), np.zeros(0, dtype=np.int32))
        self.csr = as_csr(csr, self.n_users)
        self.indptr_d, self.idx_d = self.csr.device(self.device)

    # -- row forward: chunks of materialised rows -------------------------------------------------
    def _row_width(self):
        """Floats per row of the input a chunk of ``_forward`` materialises: the F field embeddings."""
        return self.F * self.K

    def _chunk_logits(self, layout, users_d, items_d, n, grid_items, row_offset, x, out):
        """Logits ``out`` [n] of one chunk of rows; ``x`` [n, _row_width()] is free for the chunk's input."""
        raise NotImplementedError

    def _forward(self, layout, users_d, items_d, R, grid_items):
        torch = self._torch
        out = torch.empty(R, dtype=torch.float32, device=self.device)
        step = self.max_grid_rows()
        for r0 in range(0, R, step):                  # bound the materialised [rows, width] input
            r1 = min(R, r0 + step)
            n = r1 - r0
            x = torch.empty((n, self._row_width()), dtype=torch.float32, device=self.device)
            if grid_items > 0:
                self._chunk_logits(layout, users_d, None, n, grid_items, r0, x, out[r0:r1])
            else:
                self._chunk_logits(layout, users_d[r0:r1], items_d[r0:r1], n, 0, 0, x, out[r0:r1])
        return out

    # -- hoisted all-items scoring: one-sided partial sums (SURVEY.md §7.2-4) -----------------------
    def _side_concat(self, which, ids_d, want_concat=True, extra=0, **outs):
        """[n, F_side*K + extra] field embeddings of ONE side for the given ids, in the order of
        :meth:`FeatSpec.side` (``extra`` columns left for the caller); ``outs``: further outputs of the same
        gather."""
        L, pos = self.spec.side(which)
        n = int(ids_d.numel())
        x = None
        if want_concat:
            x = self._torch.empty((n, len(pos) * self.K + extra), dtype=self._torch.float32, device=self.device)
        self._feat_forward(L, ids_d, ids_d, n, 0, concat=x, **outs)
        return x

    def _side_partials(self, which, ids_d, want_concat):
        """S = sum_f e, Q = sum_f e^2, linear partial (no bias) and optionally the concatenated
        embeddings of ONE side for the given ids."""
        torch = self._torch
        n = int(ids_d.numel())
        S = torch.empty((n, self.K), dtype=torch.float32, device=self.device)
        Q = torch.empty((n, self.K), dtype=torch.float32, device=self.device)
        lin = torch.empty(n, dtype=torch.float32, device=self.device)
        lk = self.__dict__.setdefault("_side_lin", {})
        if which not in lk:
            pos = self.spec.side(which)[1]
            lk[which] = self.lin_kernel[torch.as_tensor(pos, device=self.device)].contiguous()
        concat = self._side_concat(which, ids_d, want_concat, lin=lin, ssum=S, sqsum=Q, lin_kernel=lk[which],
                                   lin_bias=0.0)
        return S, Q, lin, concat

    # -- hoisted all-items scoring of the MLP models (DeepFM, YouTubeRanking, DIN) -------------------
    def _hoistable(self):
        """The pair kernel takes the MLP's small layers: 2 or 3 Dense layers of at most 256, 64, 32 units."""
        dims = [w.shape[0] for w, _, _ in self.mlp]
        n = len(dims)
        return self.K <= 64 and n in (2, 3) and dims[0] <= 256 and dims[1] <= 64 and (n == 2 or dims[2] <= 32)

    def _first_layer_partial(self, which, x, with_bias, extra_groups=()):
        """x [n, F_side*K (+ K per extra group)] times the first MLP layer's columns of ONE side's fields (BN
        folded), then those of ``extra_groups`` (K-blocks after the F fields); the layer bias when ``with_bias``."""
        cache = self.__dict__.setdefault("_w1_side", {})
        if which not in cache:
            torch = self._torch
            groups = list(self.spec.side(which)[1]) + list(extra_groups)
            cols = torch.cat([torch.arange(g * self.K, (g + 1) * self.K, device=self.device) for g in groups])
            cache[which] = self.mlp[0][0][:, cols].contiguous()          # Wt [H1, F_side*K]
        return linear(x, cache[which], self.mlp[0][1] if with_bias else None, False)

    def _pair_scores(self, Pu, Pi, scores, fm=None):
        """``b200_deepfm_pair_scores``: scores [b, N] of every (user b, item n) pair from the first-layer partials
        Pu [b, H1] and Pi [N, H1] through the MLP's small layers and the output kernel.  ``fm`` = (Su, Qu, lu, Si,
        Qi, li): DeepFM's FM block and linear term; without it (the sequence models) those inputs are zero blocks
        and their output weights zero."""
        torch = self._torch
        K = self.K
        b, N = int(Pu.shape[0]), int(Pi.shape[0])
        if "_tail" not in self.__dict__:
            three = len(self.mlp) == 3
            self._tail = (self.mlp[1][0].t().contiguous(), self.mlp[2][0].t().contiguous() if three else None)
        W2, W3 = self._tail
        three = W3 is not None
        if fm is not None:
            w_out, lin_bias = self.out_kernel, self.lin_bias
        else:
            if "_w_out" not in self.__dict__:
                self._w_out = torch.cat([torch.zeros(1 + K, dtype=torch.float32, device=self.device),
                                         self.out_kernel]).contiguous()
                self._zeros_i = torch.zeros((self.n_items, K + 1), dtype=torch.float32, device=self.device)
            if self.__dict__.get("_zeros_u") is None or self._zeros_u.shape[0] < b:
                self._zeros_u = torch.zeros((b, K + 1), dtype=torch.float32, device=self.device)
            zu, zi = self._zeros_u, self._zeros_i
            fm, w_out, lin_bias = (zu, zu, zu, zi, zi, zi), self._w_out, 0.0
        Su, Qu, lu, Si, Qi, li = fm
        _lib.check(_lib.lib.b200_deepfm_pair_scores(
            _lib.ptr(Su), _lib.ptr(Qu), _lib.ptr(lu), _lib.ptr(Pu), b, _lib.ptr(Si), _lib.ptr(Qi), _lib.ptr(li),
            _lib.ptr(Pi), N, K, Pu.shape[1], W2.shape[1], W3.shape[1] if three else 0, lin_bias, _lib.ptr(W2),
            _lib.ptr(self.mlp[1][1]), _lib.ptr(W3), _lib.ptr(self.mlp[2][1]) if three else None, _lib.ptr(w_out),
            self.out_bias, _lib.ptr(scores), scores.stride(0), _lib.current_stream()))

    # -- public ------------------------------------------------------------------------------------
    def logits(self, users, items, sparse_rows=None, dense_rows=None):
        torch = self._torch
        u = torch.as_tensor(np.asarray(users, dtype=np.int64)).to(self.device)
        i = torch.as_tensor(np.asarray(items, dtype=np.int64)).to(self.device)
        layout = self.spec.layout
        if sparse_rows is not None or dense_rows is not None:
            sr = _dev(sparse_rows, self.device, torch.int32)
            dr = _dev(dense_rows, self.device, torch.float32)
            layout = self.spec.with_rows(sr, dr)
            self._keep = (sr, dr)
        return self._forward(layout, u, i, u.numel(), 0)

    def predict(self, users, items):
        """predict_tf_feat + normalize_prediction (prediction/predict.py:18-33,43-92), known ids."""
        z = self.logits(users, items)
        if self.task == "ranking":
            z = self._torch.sigmoid(z)
        return z.cpu().numpy()

    def score_all_items(self, user_ids_d):
        """[b, n_items] logits of every (user, item) pair — rows are the implicit grid."""
        b = int(user_ids_d.numel())
        out = self._forward(self.spec.layout, user_ids_d, None, b * self.n_items, self.n_items)
        return out.view(b, self.n_items)

    def recommend(self, user_ids, n_rec, filter_consumed=True, return_scores=False, rows_per_chunk=None):
        """recommend_tf_feat (recommend.py:81-105): all-items scoring, consumed filter, top-K."""
        torch = self._torch
        if n_rec > self.n_items:
            raise ValueError(f"`n_rec` {n_rec} exceeds num of items {self.n_items}")
        uid = torch.as_tensor(np.asarray(user_ids, dtype=np.int64)).to(self.device)
        B = uid.numel()
        if rows_per_chunk is None:   # users per chunk: bound the [users, n_items] score matrix to ~1 GiB
            rows_per_chunk = max(1, min(B, (1 << 28) // max(self.n_items, 1)))
        out_ids = torch.empty((B, n_rec), dtype=torch.int64, device=self.device)
        out_sc = torch.empty((B, n_rec), dtype=torch.float32, device=self.device)
        for r0 in range(0, B, rows_per_chunk):
            u = uid[r0:r0 + rows_per_chunk]
            b = u.numel()
            scores = self.score_all_items(u).contiguous()
            masked_topk(self, scores, u, n_rec, filter_consumed, out_ids[r0:r0 + b], out_sc[r0:r0 + b])
        return self._recs_to_host(out_ids, out_sc, return_scores)

    def _recs_to_host(self, out_ids, out_sc, return_scores):
        """Top-K ids (and scores, sigmoid for ranking) of ``recommend`` / ``recommend_dynamic`` on the host."""
        ids = out_ids.cpu().numpy()
        if return_scores:
            sc = out_sc.cpu().numpy()
            return ids, (1.0 / (1.0 + np.exp(-sc)) if self.task == "ranking" else sc)
        return ids

    def max_grid_rows(self):
        return 1 << 22

    def default_recs(self, n_rec=2000):
        """Top-``min(n_rec, n_items)`` for the OOV user without the consumed filter — what
        ``TfBase.fit`` stores as ``default_recs`` for cold-start users (``bases/tf_base.py:145-153``)."""
        return self.recommend([self.n_users], min(int(n_rec), self.n_items), filter_consumed=False).flatten()

    def recommend_dynamic(self, user_id, n_rec, data_info, user_feats=None, seq=None, filter_consumed=True,
                          inner_id=False, return_scores=False):
        """``recommend_tf_feat`` for ONE user with features / behaviour sequence supplied for this call
        (``recommendation/recommend.py:39-54,81-105``, ``recommendation/preprocess.py:104-159``): the
        user's feature columns are overridden in a per-row feature matrix of the N (user, item) rows
        (``dynamic_feats.dynamic_feature_rows``; the device tables are not touched), a sequence model
        reads the supplied sequence instead of the cached one."""
        torch = self._torch
        from .dynamic_feats import dynamic_feature_rows

        if getattr(self, "has_multi_sparse", False) and user_feats:
            raise NotImplementedError("feature overrides on layouts with multi-sparse fields")
        if n_rec > self.n_items:
            raise ValueError(f"`n_rec` {n_rec} exceeds num of items {self.n_items}")
        u = int(user_id)
        uid = torch.tensor([u], dtype=torch.int64, device=self.device)
        N = self.n_items
        layout = self.spec.layout
        keep = None
        if user_feats:
            sp, de = dynamic_feature_rows(data_info, u, user_feats)
            sr = _dev(sp, self.device, torch.int32)
            dr = _dev(de, self.device, torch.float32)
            layout = self.spec.with_rows(sr, dr)
            keep = (sr, dr)
        restore = None
        if seq is not None and len(seq) > 0:
            restore = self._swap_user_seq(u, seq, data_info, inner_id)
        try:
            if user_feats:          # explicit per-row features: the flat (user, item) grid
                scores = self._forward(layout, uid, None, N, N).view(1, N).contiguous()
            else:
                scores = self.score_all_items(uid).contiguous()
        finally:
            if restore is not None:
                restore()
        del keep
        out_ids = torch.empty((1, n_rec), dtype=torch.int64, device=self.device)
        out_sc = torch.empty((1, n_rec), dtype=torch.float32, device=self.device)
        masked_topk(self, scores, uid, n_rec, filter_consumed, out_ids, out_sc)
        return self._recs_to_host(out_ids, out_sc, return_scores)

    def _swap_user_seq(self, u, seq, data_info, inner_id):
        """Put the sequence built from ``seq`` in user ``u``'s row of the device sequence table for one
        ``recommend_dynamic`` call; returns the callable that restores the row (None: the model reads no sequence)."""
        from .dynamic_feats import build_rec_seq

        if not hasattr(self, "seqs"):
            return None
        torch = self._torch
        row, ln = build_rec_seq(seq, self.n_items, self.T, getattr(data_info, "item2id", None), inner_id)
        old = (self.seqs[u].clone(), self.lens[u].clone())
        self.seqs[u] = torch.from_numpy(row[0]).to(self.device)
        self.lens[u] = int(ln[0])

        def restore():
            self.seqs[u], self.lens[u] = old
        return restore

    def assign_oov(self, sparse_oov=None):
        """``assign_tf_variables_oov`` (``bases/tf_base.py:310-353``) on the device tables, in place."""
        torch = self._torch
        with torch.no_grad():
            for name, n in (("user_embeds", self.n_users), ("user_linear", self.n_users),
                            ("item_embeds", self.n_items), ("item_linear", self.n_items)):
                v = self.t.get(name)
                if v is not None and v.shape[0] > n:
                    v[n] = v[:n].mean(dim=0)
            if sparse_oov is not None:
                for name in ("sparse_embeds", "sparse_linear"):
                    v = self.t.get(name)
                    if v is None:
                        continue
                    start = 0
                    for oov in [int(o) for o in sparse_oov]:
                        if start >= oov:
                            continue
                        v[oov] = v[start:oov].mean(dim=0)
                        start = oov + 1
        for k in ("_item_part", "_item_side"):               # cached item-side partials depend on the tables
            self.__dict__.pop(k, None)
        if hasattr(self, "_rebuild_item_features"):
            self._rebuild_item_features()

    # -- helpers -----------------------------------------------------------------------------------
    def _feat_forward(self, layout, users_d, items_d, R, grid_items, concat=None, pw=None, lin=None,
                      fm_out=None, head=None, row_offset=0, ssum=None, sqsum=None, lin_kernel=None, lin_bias=None):
        if self.needs_linear:         # the model's linear term unless the caller passes its own
            lin_kernel = self.lin_kernel if lin_kernel is None else lin_kernel
            lin_bias = self.lin_bias if lin_bias is None else lin_bias
        feat_forward(layout, self.tables, users_d, items_d, R, grid_items=grid_items, row_offset=row_offset,
                     concat=concat, pw=pw, lin=lin, fm_out=fm_out, lin_kernel=lin_kernel,
                     lin_bias=0.0 if lin_bias is None else lin_bias, head=head, ssum=ssum, sqsum=sqsum)

    def _mlp(self, x, layers):
        torch = self._torch
        for Wt, b, act in layers:
            x = linear(x, Wt, b, act)
        return x

    def _upload_mlp(self, mlp, act=ACT_RELU):
        torch = self._torch
        return [(_dev(Wt, self.device, torch.float32), _dev(b, self.device, torch.float32), a)
                for Wt, b, a in fold_mlp(mlp, act)]


class FM(_FeatModelBase):
    """libreco/algorithms/fm.py:140-172 (inference)."""

    def __init__(self, spec, weights, user_consumed=None, task="ranking", device=None):
        super().__init__(spec, weights, user_consumed, task, device)
        torch = self._torch
        scale, shift = fold_bn(weights.get("fm_bn"))
        self.head = dict(bn_scale=_dev(scale, self.device, torch.float32),
                         bn_shift=_dev(shift, self.device, torch.float32),
                         pw_kernel=_dev(np.asarray(weights["pw_kernel"]).reshape(-1), self.device, torch.float32),
                         pw_bias=float(np.asarray(weights["pw_bias"]).reshape(-1)[0]))

    def _forward(self, layout, users_d, items_d, R, grid_items):
        out = self._torch.empty(R, dtype=self._torch.float32, device=self.device)
        self._feat_forward(layout, users_d, items_d, R, grid_items, fm_out=out, head=self.head)
        return out

    def score_all_items(self, user_ids_d):
        """Hoisted: item-side sums once per model, user-side sums once per call, K adds per pair."""
        torch = self._torch
        if self.K > 64:
            return super().score_all_items(user_ids_d)
        if "_item_side" not in self.__dict__:
            ids = torch.arange(self.n_items, device=self.device)
            self._item_side = self._side_partials("item", ids, False)[:3]
        Si, Qi, li = self._item_side
        Su, Qu, lu, _ = self._side_partials("user", user_ids_d, False)
        b = int(user_ids_d.numel())
        scores = torch.empty((b, self.n_items), dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_fm_pair_scores(
            _lib.ptr(Su), _lib.ptr(Qu), _lib.ptr(lu), b, _lib.ptr(Si), _lib.ptr(Qi), _lib.ptr(li), self.n_items,
            self.K, self.lin_bias, _lib.ptr(self.head["bn_scale"]), _lib.ptr(self.head["bn_shift"]),
            _lib.ptr(self.head["pw_kernel"]), self.head["pw_bias"], _lib.ptr(scores), scores.stride(0),
            _lib.current_stream()))
        return scores

    def max_grid_rows(self):
        return 1 << 28


class DeepFM(_FeatModelBase):
    """libreco/algorithms/deepfm.py:143-175 (inference)."""

    def __init__(self, spec, weights, user_consumed=None, task="ranking", device=None):
        super().__init__(spec, weights, user_consumed, task, device)
        torch = self._torch
        self.mlp = self._upload_mlp(weights["mlp"])
        self.hidden_last = self.mlp[-1][0].shape[0]
        self.out_kernel = _dev(np.asarray(weights["out_kernel"]).reshape(-1), self.device, torch.float32)
        self.out_bias = float(np.asarray(weights["out_bias"]).reshape(-1)[0])

    def _chunk_logits(self, layout, users_d, items_d, n, grid_items, row_offset, x, out):
        pw = self._torch.empty((n, self.K), dtype=self._torch.float32, device=self.device)
        lin = self._torch.empty(n, dtype=self._torch.float32, device=self.device)
        self._feat_forward(layout, users_d, items_d, n, grid_items, concat=x, pw=pw, lin=lin, row_offset=row_offset)
        deep = self._mlp(x, self.mlp)
        lin2 = lin.view(n, 1)
        _lib.check(_lib.lib.b200_concat_dense(
            _lib.ptr(lin2), 1, 1, _lib.ptr(pw), pw.stride(0), self.K, _lib.ptr(deep), deep.stride(0),
            self.hidden_last, _lib.ptr(self.out_kernel), self.out_bias, n, _lib.ptr(out), _lib.current_stream()))

    def score_all_items(self, user_ids_d):
        """Hoisted: first-layer partial products per side, only the small layers per (user, item)."""
        torch = self._torch
        if not self._hoistable():
            return super().score_all_items(user_ids_d)
        if "_item_side" not in self.__dict__:
            ids = torch.arange(self.n_items, device=self.device)
            Si, Qi, li, ci = self._side_partials("item", ids, True)
            self._item_side = (Si, Qi, li, self._first_layer_partial("item", ci, False))
        Si, Qi, li, Pi = self._item_side
        Su, Qu, lu, cu = self._side_partials("user", user_ids_d, True)
        Pu = self._first_layer_partial("user", cu, True)
        scores = torch.empty((int(user_ids_d.numel()), self.n_items), dtype=torch.float32, device=self.device)
        self._pair_scores(Pu, Pi, scores, fm=(Su, Qu, lu, Si, Qi, li))
        return scores

    def max_grid_rows(self):
        # deep input bytes per row = F*K*4; keep a chunk under ~1 GiB
        return max(1, (1 << 30) // (self._row_width() * 4))


AUTOINT_MAX_K = 64          # the shapes b200_autoint_rows / _grid accept (include/b200reco.h)
AUTOINT_MAX_D = 64
AUTOINT_MAX_LAYERS = 4
AUTOINT_MAX_F = 130


class AutoInt(_FeatModelBase):
    """libreco/algorithms/autoint.py:146-168 (inference): the field embeddings [user, item, sparse.., dense..]
    stacked into X [F, K], ``L`` layers of multi-head self-attention across the fields (layers/attention.py:67-138,
    optional residual), then Dense(1) on the flattened block.  No linear tables, and no BN or dropout in the
    inference graph even though the reference accepts ``use_bn``.

    Weights (besides the embedding tables): ``autoint_layers`` = [{wq, wk, wv [K, D], wo [D, K]}] per layer with
    head-major columns and ``wv`` the effective value map, ``num_heads``, ``use_residual``, ``out_kernel [F*K]``,
    ``out_bias`` — :func:`weights_io.autoint_weights` makes them from either TensorFlow graph's variables.

    Every (user, item) pair is a chain of small attentions that nothing outside the pair can be hoisted from, so
    ``_forward`` runs ``b200_autoint_rows`` on the K1 concat and all-items scoring runs ``b200_autoint_grid`` on a
    per-model item-side block and a per-call user-side block; both give bit-identical logits."""

    needs_linear = False

    def __init__(self, spec, weights, user_consumed=None, task="ranking", device=None):
        super().__init__(spec, weights, user_consumed, task, device)
        torch = self._torch
        K, F = self.K, self.F
        H = int(weights["num_heads"])
        layers = list(weights["autoint_layers"])
        if K > AUTOINT_MAX_K:
            raise ValueError(f"AutoInt: embed size {K} > {AUTOINT_MAX_K} is not supported")
        if F > AUTOINT_MAX_F:
            raise ValueError(f"AutoInt: {F} fields > {AUTOINT_MAX_F} (2 ids + 128 features) is not supported")
        if not 1 <= len(layers) <= AUTOINT_MAX_LAYERS:
            raise ValueError(f"AutoInt: {len(layers)} attention layers, supported 1..{AUTOINT_MAX_LAYERS}")
        if H < 1:
            raise ValueError(f"AutoInt: num_heads {H} < 1")
        hds, packed = [], []
        for i, lw in enumerate(layers):
            wq, wk, wv, wo = (np.asarray(lw[k], dtype=np.float32) for k in ("wq", "wk", "wv", "wo"))
            D = wq.shape[1]
            if D % H or D > AUTOINT_MAX_D:
                raise ValueError(f"AutoInt layer {i}: width {D} must be num_heads ({H}) x head size and <= "
                                 f"{AUTOINT_MAX_D}")
            if wq.shape != (K, D) or wk.shape != (K, D) or wv.shape != (K, D) or wo.shape != (D, K):
                raise ValueError(f"AutoInt layer {i}: shapes wq {wq.shape} wk {wk.shape} wv {wv.shape} wo {wo.shape}, "
                                 f"expected [{K}, {D}] x 3 and [{D}, {K}]")
            hds.append(D // H)
            packed += [wq.reshape(-1), wk.reshape(-1), wv.reshape(-1), wo.reshape(-1)]
        out_kernel = np.asarray(weights["out_kernel"], dtype=np.float32).reshape(-1)
        if out_kernel.size != F * K:
            raise ValueError(f"AutoInt: out_kernel has {out_kernel.size} entries, expected F*K = {F}*{K}")
        self.num_heads, self.head_dims = H, hds
        self.use_residual = bool(weights.get("use_residual", True))
        self._hd_host = np.asarray(hds, dtype=np.int32)
        self.w_layers = _dev(np.concatenate(packed), self.device, torch.float32)
        self.out_kernel = _dev(out_kernel, self.device, torch.float32)
        self.out_bias = float(np.asarray(weights["out_bias"]).reshape(-1)[0])

    def _head(self):
        return (self.F, self.K, self.num_heads, len(self.head_dims), _lib.ptr(self._hd_host), _lib.ptr(self.w_layers),
                _lib.ptr(self.out_kernel), self.out_bias, int(self.use_residual))

    def _chunk_logits(self, layout, users_d, items_d, n, grid_items, row_offset, x, out):
        self._feat_forward(layout, users_d, items_d, n, grid_items, concat=x, row_offset=row_offset)
        _lib.check(_lib.lib.b200_autoint_rows(_lib.ptr(x), x.stride(0), n, *self._head(), _lib.ptr(out),
                                              _lib.current_stream()))

    def _field_map(self):
        """int32 [F]: global field f comes from user-side slot m (m >= 0) or item-side slot -1 - m."""
        if "_fmap" not in self.__dict__:
            m = np.zeros(self.F, dtype=np.int32)
            for j, f in enumerate(self.spec.side("user")[1]):
                m[f] = j
            for j, f in enumerate(self.spec.side("item")[1]):
                m[f] = -1 - j
            self._fmap = _dev(m, self.device, self._torch.int32)
        return self._fmap

    def score_all_items(self, user_ids_d):
        """All L layers per (user, item) pair in one kernel: the item-side block once per model (rebuilt after
        ``assign_oov``), the user-side block once per call; the [b*N, F*K] concat is never built."""
        torch = self._torch
        if "_item_side" not in self.__dict__:
            self._item_side = self._side_concat("item", torch.arange(self.n_items, device=self.device))
        Xi = self._item_side
        Xu = self._side_concat("user", user_ids_d)
        b, N = int(user_ids_d.numel()), self.n_items
        scores = torch.empty((b, N), dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_autoint_grid(_lib.ptr(Xu), Xu.stride(0), b, _lib.ptr(Xi), Xi.stride(0), N,
                                              _lib.ptr(self._field_map()), *self._head(), _lib.ptr(scores),
                                              scores.stride(0), _lib.current_stream()))
        return scores

    def max_grid_rows(self):
        return max(1, (1 << 30) // (self._row_width() * 4))


def wide_deep_weights(user_wide, item_wide, sparse_wide, dense_wide, wide_kernel, wide_bias, user_deep, item_deep,
                      sparse_deep, dense_deep, mlp, deep_kernel, deep_bias):
    """WideDeep (``libreco/algorithms/wide_deep.py:150-262``, SURVEY 8f-4) on the DeepFM engine: the wide term
    ``Dense1(concat of the 1-d wide embeddings)`` IS DeepFM's linear term, the deep tower IS DeepFM's, and
    ``output = wide_term + Dense1(deep)`` is DeepFM's head ``<[lin, pw, deep], w> + b`` with weight 1 on ``lin``, 0 on
    the pairwise block and the ``deep_term`` kernel / bias on the rest.  Returns the weight dict :class:`DeepFM` takes
    (variables named as in the reference: ``user_wide_var`` ... ``dense_deep_var``, ``wide_term`` / ``deep_term``)."""
    K = int(np.asarray(user_deep).shape[1])
    w = dict(user_embeds=user_deep, item_embeds=item_deep, user_linear=np.asarray(user_wide).reshape(-1),
             item_linear=np.asarray(item_wide).reshape(-1), lin_kernel=np.asarray(wide_kernel).reshape(-1),
             lin_bias=np.float32(np.asarray(wide_bias).reshape(-1)[0]), mlp=mlp,
             out_kernel=np.concatenate([np.ones(1, np.float32), np.zeros(K, np.float32),
                                        np.asarray(deep_kernel, dtype=np.float32).reshape(-1)]),
             out_bias=np.float32(np.asarray(deep_bias).reshape(-1)[0]))
    if sparse_deep is not None:
        w["sparse_embeds"], w["sparse_linear"] = sparse_deep, np.asarray(sparse_wide).reshape(-1)
    if dense_deep is not None:
        w["dense_embeds"], w["dense_linear"] = dense_deep, np.asarray(dense_wide).reshape(-1)
    return w


def from_tf_variables(npz, names=None):
    """Map a reference ``<name>_tf_variables.npz`` (utils/save_load.py:70-80) to WEIGHT_KEYS.
    Embedding names are fixed by the reference code (SURVEY.md Appendix C); the un-named
    ``tf_dense`` heads get TF-version-dependent auto names, so `names` may override the defaults."""
    names = names or {}
    g = lambda k, d: npz[names.get(k, d)] if names.get(k, d) in npz else None
    w = {}
    for k in ("user_embeds", "item_embeds", "sparse_embeds", "dense_embeds"):
        v = g(k, f"embedding/{k}_var:0")
        if v is not None:
            w[k] = v
    for k in ("user_linear", "item_linear", "sparse_linear", "dense_linear"):
        v = g(k, f"embedding/{k}_var:0")
        if v is not None:
            w[k] = np.asarray(v).reshape(-1)
    return w


# ==============================================================================================
# sequence models (DIN, YouTubeRanking) and TwoTower
# ==============================================================================================
def recent_sequences(user_consumed, n_users, n_items, max_seq_len):
    """get_recent_seqs (libreco/batch/sequence.py:75-91): last `max_seq_len` consumed items per
    user, padded with n_items; an extra all-pad OOV row with length 1."""
    seqs = np.full((n_users + 1, max_seq_len), n_items, dtype=np.int32)
    lens = np.ones(n_users + 1, dtype=np.int32)
    for u in range(n_users):
        items = user_consumed[u] if u in user_consumed else []
        n = min(len(items), max_seq_len)
        if n:
            seqs[u, :n] = items[-n:] if len(items) >= max_seq_len else items
        lens[u] = n if len(items) < max_seq_len else max_seq_len
    return seqs, lens


def recent_sequences_csr(consumed, n_items, max_seq_len):
    """Vectorised get_recent_seqs (libreco/batch/sequence.py:75-91) over a ConsumedCSR (arrival
    order): no per-user Python loop (SURVEY.md 8f-3) — 10 M users in seconds instead of minutes."""
    indptr, idx = consumed.indptr, consumed.idx
    n_users = len(indptr) - 1
    clen = np.diff(indptr)
    lens = np.minimum(clen, max_seq_len).astype(np.int32)
    seqs = np.full((n_users + 1, max_seq_len), n_items, dtype=np.int32)
    t = np.arange(max_seq_len, dtype=np.int64)[None, :]
    src = (indptr[1:] - lens)[:, None] + t
    valid = t < lens[:, None]
    seqs[:n_users][valid] = idx[src[valid]]
    return seqs, np.append(lens, np.int32(1)).astype(np.int32)


def permute_mlp_input(mlp, perm):
    """Re-order the input features of a dense_nn (first kernel rows + input BN) by `perm`."""
    out = dict(mlp)
    out["kernels"] = [np.asarray(mlp["kernels"][0])[perm]] + list(mlp["kernels"][1:])
    if mlp.get("bn_in") is not None:
        out["bn_in"] = {k: np.asarray(v)[perm] for k, v in mlp["bn_in"].items()}
    return out


class _SeqModelBase(_FeatModelBase):
    needs_linear = False

    def __init__(self, spec, weights, recent_seqs, recent_seq_lens, user_consumed=None, task="ranking",
                 device=None):
        super().__init__(spec, weights, user_consumed, task, device)
        torch = self._torch
        self.seqs = _dev(recent_seqs, self.device, torch.int32)
        self.lens = _dev(recent_seq_lens, self.device, torch.int32)
        self.T = int(self.seqs.shape[1])
        self.out_kernel = _dev(np.asarray(weights["out_kernel"]).reshape(-1), self.device, torch.float32)
        self.out_bias = float(np.asarray(weights["out_bias"]).reshape(-1)[0])
        self.extra = 0          # width of the sequence block appended to the concatenated row

    def _seq_block(self, users_d, items_d, n, grid_items, row_offset, out_view):
        raise NotImplementedError

    def _row_width(self):
        return self.F * self.K + self.extra

    def _chunk_logits(self, layout, users_d, items_d, n, grid_items, row_offset, x, out):
        self._feat_forward(layout, users_d, items_d, n, grid_items, concat=x, row_offset=row_offset)
        self._seq_block(users_d, items_d, n, grid_items, row_offset, x[:, self.F * self.K:])
        h = self._mlp(x, self.mlp)
        _lib.check(_lib.lib.b200_concat_dense(
            _lib.ptr(h), h.stride(0), h.shape[1], None, 0, 0, None, 0, 0, _lib.ptr(self.out_kernel),
            self.out_bias, n, _lib.ptr(out), _lib.current_stream()))

    def max_grid_rows(self):
        return max(1, (1 << 30) // (self._row_width() * 4))


class YouTubeRanking(_SeqModelBase):
    """libreco/algorithms/youtube_ranking.py:167-218 (inference)."""

    def __init__(self, spec, weights, recent_seqs, recent_seq_lens, user_consumed=None, task="ranking",
                 device=None):
        super().__init__(spec, weights, recent_seqs, recent_seq_lens, user_consumed, task, device)
        K, F = self.K, self.F
        self.extra = K
        # reference order [user, item, pooled, sparse.., dense..] -> ours [user, item, sparse.., dense.., pooled]
        perm = np.concatenate([np.arange(0, 2 * K), np.arange(3 * K, (F + 1) * K), np.arange(2 * K, 3 * K)])
        self.mlp = self._upload_mlp(permute_mlp_input(weights["mlp"], perm))

    # ---- hoisted all-items scoring (SURVEY.md §7.2-4): everything user-only or item-only once ----
    def score_all_items(self, user_ids_d):
        """youtube_ranking.py:199-218 over the implicit (user, item) grid: the first Dense layer splits
        into a user part (id, user features, pooled history) and an item part, computed once per user /
        once per item; a pair then costs H1 adds + the small layers (the DeepFM pair kernel with an
        empty FM part)."""
        torch = self._torch
        if not self._hoistable():
            return super().score_all_items(user_ids_d)
        if "_item_part" not in self.__dict__:
            xi = self._side_concat("item", torch.arange(self.n_items, device=self.device))
            self._item_part = self._first_layer_partial("item", xi, False)
        xu = self._side_concat("user", user_ids_d, extra=self.K)
        self._seq_block(user_ids_d, user_ids_d, xu.shape[0], 0, 0, xu[:, xu.shape[1] - self.K:])
        Pu = self._first_layer_partial("user", xu, True, [self.F])     # the pooled block sits after the F fields
        scores = torch.empty((int(user_ids_d.numel()), self.n_items), dtype=torch.float32, device=self.device)
        self._pair_scores(Pu, self._item_part, scores)
        return scores

    def _seq_block(self, users_d, items_d, n, grid_items, row_offset, out_view):
        E = self.t["item_embeds"]
        _lib.check(_lib.lib.b200_seq_pool(
            _lib.ptr(E), E.stride(0), self.K, self.n_items, _lib.ptr(self.seqs), self.seqs.stride(0),
            _lib.ptr(self.lens), self.T, _lib.ptr(users_d), n, grid_items, row_offset,
            _lib.ptr(out_view), out_view.stride(0), _lib.current_stream()))


class DIN(_SeqModelBase):
    """libreco/algorithms/din.py:165-250 (inference; ``use_tf_attention`` either way: with
    ``weights["use_tf_attention"]`` the attention is the weight-free dot-product form of
    ``layers/attention.py:5-25`` and all-items scoring runs on the flat (user, item) grid)."""

    def __init__(self, spec, weights, recent_seqs, recent_seq_lens, user_consumed=None, task="ranking",
                 device=None):
        super().__init__(spec, weights, recent_seqs, recent_seq_lens, user_consumed, task, device)
        torch = self._torch
        self._rebuild_item_features()
        self.Kp = int(self.G.shape[1])
        self.extra = self.Kp
        # use_tf_attention=True (din.py:247-248, layers/attention.py:5-25): dot-product attention, no weights
        self.use_tf_attention = bool(weights.get("use_tf_attention", False)) or weights.get("attention") is None
        if self.use_tf_attention:
            self.att = dict(k1=None, b1=None, k2=None, b2=0.0)
        else:
            att = weights["attention"]
            self.att = dict(k1=_dev(att["k1"], self.device, torch.float32), b1=_dev(att["b1"], self.device, torch.float32),
                            k2=_dev(np.asarray(att["k2"]).reshape(-1), self.device, torch.float32),
                            b2=float(np.asarray(att["b2"]).reshape(-1)[0]))
        self.mlp = self._upload_mlp(weights["mlp"])

    def _rebuild_item_features(self):
        """item feature table G (combine_seq_features, concat mode; tfops/features.py:165-218): built once
        per set of tables (again after ``assign_oov``)."""
        torch = self._torch
        parts = [self.t["item_embeds"]]
        if self.spec.is_ is not None:
            parts.append(self.t["sparse_embeds"][self.spec.is_.long()].reshape(self.n_items + 1, -1))
        if self.spec.id_ is not None:
            cols = torch.as_tensor(self.spec.item_dense_cols, device=self.device)
            parts.append((self.spec.id_[:, :, None] * self.t["dense_embeds"][cols][None]).reshape(self.n_items + 1, -1))
        self.G = torch.cat(parts, dim=1).contiguous()

    # ---- hoisted all-items scoring (SURVEY.md 8d "a7 DIN all-items") ---------------------------------
    def _hoistable(self):
        return super()._hoistable() and self.Kp % 4 == 0 and not self.use_tf_attention

    def score_all_items(self, user_ids_d):
        """din.py:165-250 over (this user) x (every item).  Per user: the attention's Dense(16) becomes
        one GEMM [N, K'] x [K', 16 len] on the library GEMM kernel (wgmma 3xTF32 for large N), a warp
        per item finishes sigmoid / Dense(1) / softmax / weighted key sum, the first MLP layer splits
        into user / item / attention parts and the pair kernel runs the small layers."""
        torch = self._torch
        if not self._hoistable():
            return super().score_all_items(user_ids_d)
        N, Kp, FK = self.n_items, self.Kp, self.F * self.K
        if "_item_part" not in self.__dict__:
            xi = self._side_concat("item", torch.arange(N, device=self.device))
            self._item_part = self._first_layer_partial("item", xi, False)
            self._w_att = self.mlp[0][0][:, FK:FK + Kp].contiguous()           # [H1, K']
        b = int(user_ids_d.numel())
        xu = self._side_concat("user", user_ids_d)
        Pu_all = self._first_layer_partial("user", xu, True)                     # [b, H1] incl. bias
        scores = torch.empty((b, N), dtype=torch.float32, device=self.device)
        lens_h = self.lens[user_ids_d].clamp(0, self.T).cpu().numpy()            # one small D2H per call
        Gn = self.G[:N]
        att = torch.empty((N, Kp), dtype=torch.float32, device=self.device)
        lib, st = _lib.lib, _lib.current_stream()
        for r in range(b):
            ln = int(lens_h[r])
            seq = self.seqs[user_ids_d[r]]                                       # int32 [T] view (device)
            Z = None
            fused = False
            if ln > 0:
                Wt = torch.empty((16 * ln, Kp), dtype=torch.float32, device=self.device)
                bias = torch.empty(16 * ln, dtype=torch.float32, device=self.device)
                _lib.check(lib.b200_din_user_weights(_lib.ptr(self.G), self.G.stride(0), Kp, _lib.ptr(seq), ln,
                                                     _lib.ptr(self.att["k1"]), _lib.ptr(self.att["b1"]), _lib.ptr(Wt),
                                                     Wt.stride(0), _lib.ptr(bias), st))
                fused = (DIN_FUSED_ATTENTION and ln <= 64 and ln * Kp * 4 <= 48 * 1024 and Kp % 4 == 0
                         and Gn.stride(0) % 4 == 0 and N >= TC_MIN_ROWS)
                if fused:
                    # sigmoid + Dense(1) in the GEMM's epilogue: [N, ln] logits instead of [N, 16 ln] pre-activations
                    A = torch.empty((N, ln), dtype=torch.float32, device=self.device)
                    _lib.check(lib.b200_linear_tf32x3_sigmoid_dot(
                        _lib.ptr(Gn), Gn.stride(0), N, _lib.ptr(Wt), Wt.stride(0), None, _lib.ptr(bias), Kp, 16 * ln,
                        _lib.ptr(self.att["k2"]), _lib.ptr(A), A.stride(0), st))
                    _lib.check(lib.b200_din_attention_from_logits(
                        _lib.ptr(A), A.stride(0), N, _lib.ptr(self.G), self.G.stride(0), Kp, _lib.ptr(seq), ln,
                        self.att["b2"], _lib.ptr(att), att.stride(0), st))
                else:
                    Z = linear(Gn, Wt, bias, False, cache_split=False)           # [N, 16 ln]
            if not fused:
                _lib.check(lib.b200_din_attention_hoisted(
                    _lib.ptr(Z), Z.stride(0) if Z is not None else 0, N, _lib.ptr(self.G), self.G.stride(0), Kp,
                    _lib.ptr(seq), ln, _lib.ptr(self.att["k2"]), self.att["b2"], _lib.ptr(att), att.stride(0), st))
            Pi = self._item_part + linear(att, self._w_att, None, False)         # [N, H1]
            self._pair_scores(Pu_all[r:r + 1], Pi, scores[r:r + 1])
        return scores

    def _seq_block(self, users_d, items_d, n, grid_items, row_offset, out_view):
        _lib.check(_lib.lib.b200_din_attention(
            _lib.ptr(self.G), self.G.stride(0), self.Kp, _lib.ptr(items_d), _lib.ptr(self.seqs),
            self.seqs.stride(0), _lib.ptr(self.lens), self.T, _lib.ptr(users_d), n, grid_items, row_offset,
            _lib.ptr(self.att["k1"]), _lib.ptr(self.att["b1"]), _lib.ptr(self.att["k2"]), self.att["b2"],
            _lib.ptr(out_view), out_view.stride(0), _lib.current_stream()))


TRANSFORMER_MAX_T = 64          # the shapes b200_transformer_* accept (include/b200reco.h)
TRANSFORMER_MAX_D = 128
TRANSFORMER_MAX_LAYERS = 4


def sinusoidal_positions(T, d):
    """The non-trainable positional table of ``positional_encoding`` (libreco/layers/transformer.py:113-144), [T, d]:
    column c holds t / 10000^(2 floor(c/2) / d), through sin for even c and cos for odd c (odd d included)."""
    ang = np.arange(T, dtype=np.float64)[:, None] / np.power(10000.0, (np.arange(d) // 2 * 2) / d)[None, :]
    pe = np.where(np.arange(d)[None, :] % 2 == 0, np.sin(ang), np.cos(ang))
    return pe.astype(np.float32)


def _rms(x, scale):
    """rms_norm (layers/normalization.py:21-29) on device tensors: x / sqrt(mean(x^2) + 1e-8) * scale."""
    return x * (x.square().mean(dim=-1, keepdim=True) + 1e-8).rsqrt() * scale


class Transformer(_SeqModelBase):
    """libreco/algorithms/transformer.py:203-339 (inference): the BST-style sequence model.  The user's recent items
    (rows of the item feature table G, ``combine_seq_features`` in ``concat`` or ``elementwise`` mode) and a positional
    table [T, K] form X [T, D = K' + K]; ``L`` layers of pre-norm multi-head self-attention + gelu FFN and a final RMS
    norm give S_u [T, D]; the target item's query [rms_item(G[n]) || 1..1] attends over S_u (Keras dot-product
    attention, no scale); ``dense_nn`` with swish on [user, item, sparse.., dense.., s_u], then Dense(1).

    Weights (besides the embedding tables): ``tfm_layers`` = [{rms_att, wq, wk, wv, wo, rms_ffn, w1, w2}] per layer
    (``wv`` the effective value map), ``rms_last``, ``rms_item``, ``positional_encoding`` (absent: sinusoidal),
    ``num_heads``, ``use_causal_mask``, ``feat_agg_mode``, ``ln_sparse`` / ``ln_dense`` ({scale, bias}; elementwise
    mode), ``mlp``, ``out_kernel``, ``out_bias`` — :func:`weights_io.transformer_weights` makes them from either
    TensorFlow graph's variables.

    The encoder runs ONCE per user of a call (``b200_transformer_encode``).  All-items scoring splits the first MLP
    layer into a per-model item part Pi, a per-call user part Pu and V'_u = S_u W1_seq, and ``b200_transformer_pair_scores``
    finishes every pair; rows mode (``predict``, feature rows, ``recommend_dynamic`` with features, an MLP outside the
    pair kernel's envelope) encodes each distinct user of a chunk once and writes s_u into the concat
    (``b200_transformer_target_attention``) for the swish MLP on the library's dense layers."""

    def __init__(self, spec, weights, recent_seqs, recent_seq_lens, user_consumed=None, task="ranking",
                 device=None):
        raw_is = None
        if not isinstance(spec, FeatSpec):
            g = _spec_get(spec)
            raw_is = g("item_sparse_unique") if g("item_sparse_col_index") else None
        super().__init__(spec, weights, recent_seqs, recent_seq_lens, user_consumed, task, device)
        torch = self._torch
        f32 = torch.float32
        K, T, F = self.K, self.T, self.F
        self.feat_agg_mode = weights.get("feat_agg_mode", "concat")
        if self.feat_agg_mode not in ("concat", "elementwise"):
            raise ValueError("Transformer: `feat_agg_mode` must be `concat` or `elementwise`")
        # combine_seq_features reads the item sparse columns as they are (multi-sparse sub-columns one by one)
        self._item_sparse = _dev(raw_is, self.device, torch.int32) if raw_is is not None else self.spec.is_
        self.ln = {k: {n: _dev(np.asarray(v[n]).reshape(-1), self.device, f32) for n in ("scale", "bias")}
                   for k, v in (("sparse", weights.get("ln_sparse")), ("dense", weights.get("ln_dense"))) if v is not None}
        self.rms_item = _dev(np.asarray(weights["rms_item"]).reshape(-1), self.device, f32)
        self._rebuild_item_features()
        self.Kp = int(self.G.shape[1])
        D = self.D = self.Kp + K
        H = self.num_heads = int(weights["num_heads"])
        layers = list(weights["tfm_layers"])
        if T > TRANSFORMER_MAX_T:
            raise ValueError(f"Transformer: sequence length {T} > {TRANSFORMER_MAX_T} is not supported")
        if D > TRANSFORMER_MAX_D:
            raise ValueError(f"Transformer: model width {D} (item features {self.Kp} + positions {K}) > "
                             f"{TRANSFORMER_MAX_D} is not supported")
        if not 1 <= len(layers) <= TRANSFORMER_MAX_LAYERS:
            raise ValueError(f"Transformer: {len(layers)} layers, supported 1..{TRANSFORMER_MAX_LAYERS}")
        if H < 1 or D % H:
            raise ValueError(f"Transformer: width {D} must be divisible by num_heads {H}")
        if self.rms_item.numel() != self.Kp:
            raise ValueError(f"Transformer: rms_item has {self.rms_item.numel()} entries, expected {self.Kp}")
        shapes = dict(rms_att=(D,), wq=(D, D), wk=(D, D), wv=(D, D), wo=(D, D), rms_ffn=(D,), w1=(D, 4 * D),
                      w2=(4 * D, D))
        packed = []
        for i, lw in enumerate(layers):
            for k, shp in shapes.items():
                a = np.asarray(lw[k], dtype=np.float32)
                if a.shape != shp:
                    raise ValueError(f"Transformer layer {i}: {k} has shape {a.shape}, expected {shp}")
                packed.append(a.reshape(-1))
        self.n_layers = len(layers)
        self.w_layers = _dev(np.concatenate(packed), self.device, f32)
        self.rms_last = _dev(np.asarray(weights["rms_last"], dtype=np.float32).reshape(-1), self.device, f32)
        if self.rms_last.numel() != D:
            raise ValueError(f"Transformer: rms_last has {self.rms_last.numel()} entries, expected {D}")
        pos = weights.get("positional_encoding")
        pos = sinusoidal_positions(T, K) if pos is None else np.asarray(pos, dtype=np.float32)
        if pos.shape != (T, K):
            raise ValueError(f"Transformer: positional table has shape {pos.shape}, expected ({T}, {K})")
        self.pos = _dev(pos, self.device, f32)
        self.causal = bool(weights.get("use_causal_mask", False))
        self.extra = D
        self.mlp = self._upload_mlp(weights["mlp"], ACT_SWISH)
        if self.mlp[0][0].shape[1] != F * K + D:
            raise ValueError(f"Transformer: the first MLP layer takes {self.mlp[0][0].shape[1]} inputs, expected "
                             f"F*K + D = {F}*{K} + {D}")

    def _rebuild_item_features(self):
        """G [n_items+1, K'] (combine_seq_features, tfops/features.py:151-236) and the target queries
        Qi = [rms_item(G) || 1..1] [n_items+1, D]: once per set of tables (again after ``assign_oov``)."""
        torch = self._torch
        E = self.t["item_embeds"]
        n = self.n_items + 1
        sp = self.t["sparse_embeds"][self._item_sparse.long()] if self._item_sparse is not None else None
        de = None
        if self.spec.id_ is not None:
            cols = torch.as_tensor(self.spec.item_dense_cols, device=self.device)
            de = self.spec.id_[:, :, None] * self.t["dense_embeds"][cols][None]
        if self.feat_agg_mode == "concat":
            self.G = torch.cat([E] + [x.reshape(n, -1) for x in (sp, de) if x is not None], dim=1).contiguous()
        else:
            agg = torch.ones_like(E)
            for name, x in (("sparse", sp), ("dense", de)):
                if x is None:
                    continue
                mean = x.mean(dim=-1, keepdim=True)
                var = (x - mean).square().mean(dim=-1, keepdim=True)   # layer_normalization, eps 1e-8
                ln = self.ln[name]
                agg = agg + ((x - mean) * (var + 1e-8).rsqrt() * ln["scale"] + ln["bias"]).sum(dim=1)
            self.G = (E * agg).contiguous()
        self.Qi = torch.cat([_rms(self.G, self.rms_item), torch.ones((n, self.K), dtype=torch.float32,
                                                                       device=self.device)], dim=1).contiguous()

    def _encode(self, users_d):
        """S [n, T, D] of the given users' sequences (one encoder pass each) and their lengths (int32 [n])."""
        torch = self._torch
        users = users_d.to(torch.int64).contiguous()
        lens = self.lens[users].contiguous()
        n = int(users.numel())
        S = torch.empty((n, self.T, self.D), dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_transformer_encode(
            _lib.ptr(users), n, _lib.ptr(lens), _lib.ptr(self.seqs), self.seqs.stride(0), _lib.ptr(self.G),
            self.G.stride(0), self.Kp, _lib.ptr(self.pos), self.K, self.T, self.num_heads, self.n_layers,
            int(self.causal), _lib.ptr(self.w_layers), _lib.ptr(self.rms_last), _lib.ptr(S), _lib.current_stream()))
        return S, lens

    def _hoistable(self):
        if not super()._hoistable():
            return False
        need = _lib.lib.b200_transformer_pair_smem_bytes(self.T, self.D, self.mlp[0][0].shape[0])
        return 0 < need <= self._torch.cuda.get_device_properties(self.device).shared_memory_per_block_optin

    def score_all_items(self, user_ids_d):
        """transformer.py:203-339 over (these users) x (every item): the encoder once per user, V'_u = S_u W1_seq on
        the library GEMM, then every pair in ``b200_transformer_pair_scores``; the item part Pi of the first layer
        once per model.  The [b*N, F*K + D] concat is never built."""
        torch = self._torch
        if not self._hoistable():
            return super().score_all_items(user_ids_d)
        N, FK, D, T = self.n_items, self.F * self.K, self.D, self.T
        if "_item_part" not in self.__dict__:
            xi = self._side_concat("item", torch.arange(N, device=self.device))
            self._item_part = self._first_layer_partial("item", xi, False)
            self._w_seq = self.mlp[0][0][:, FK:FK + D].contiguous()             # [H1, D]
            three = len(self.mlp) == 3
            self._tail = (self.mlp[1][0].t().contiguous(), self.mlp[2][0].t().contiguous() if three else None)
        Pi = self._item_part
        W2, W3 = self._tail
        H1 = Pi.shape[1]
        b = int(user_ids_d.numel())
        scores = torch.empty((b, N), dtype=torch.float32, device=self.device)
        for r0 in range(0, b, 65535):
            u = user_ids_d[r0:r0 + 65535]
            nb = int(u.numel())
            Pu = self._first_layer_partial("user", self._side_concat("user", u), True)     # [nb, H1] incl. bias
            S, lens = self._encode(u)
            Vp = linear(S.view(nb * T, D), self._w_seq, None, ACT_NONE)                     # [nb*T, H1]
            out = scores[r0:r0 + nb]
            _lib.check(_lib.lib.b200_transformer_pair_scores(
                _lib.ptr(self.Qi), self.Qi.stride(0), N, _lib.ptr(S), _lib.ptr(Vp), _lib.ptr(Pu), _lib.ptr(lens), nb,
                _lib.ptr(Pi), Pi.stride(0), T, D, H1, W2.shape[1], W3.shape[1] if W3 is not None else 0, _lib.ptr(W2),
                _lib.ptr(self.mlp[1][1]), _lib.ptr(W3), _lib.ptr(self.mlp[2][1]) if W3 is not None else None,
                _lib.ptr(self.out_kernel), self.out_bias, _lib.ptr(out), out.stride(0), _lib.current_stream()))
        return scores

    def _seq_block(self, users_d, items_d, n, grid_items, row_offset, out_view):
        """s_u of each row, every distinct user (grid slot) of the chunk encoded once."""
        torch = self._torch
        if grid_items > 0:
            u0 = row_offset // grid_items
            u1 = (row_offset + n - 1) // grid_items
            S, lens = self._encode(users_d[u0:u1 + 1])
            slot, items, off = None, None, row_offset - u0 * grid_items
        else:
            uniq, inv = torch.unique(users_d, return_inverse=True)
            S, lens = self._encode(uniq)
            slot, items, off = inv.to(torch.int32).contiguous(), items_d.to(torch.int64).contiguous(), 0
        _lib.check(_lib.lib.b200_transformer_target_attention(
            _lib.ptr(self.Qi), self.Qi.stride(0), _lib.ptr(S), self.T, self.D, _lib.ptr(lens), _lib.ptr(slot),
            _lib.ptr(items), n, grid_items, off, _lib.ptr(out_view), out_view.stride(0), _lib.current_stream()))


SIM_MAX_L = 256                 # the shapes b200_sim_* accept (include/b200reco.h)
SIM_MAX_S = 64
SIM_MAX_TOPK = 32
SIM_MAX_K = 64


def recent_dual_sequences(user_consumed, n_users, n_items, long_max_len, short_max_len):
    """get_recent_dual_seqs (libreco/batch/sequence.py:150-188): per user the last ``short_max_len`` consumed items
    (short) and up to ``long_max_len`` items before them (long), padded with n_items.  A user with at most
    ``short_max_len`` items has long length 1 over an all-pad row; the extra OOV row n_users is all pad with both
    lengths 1.  Returns (long_seqs, long_lens, short_seqs, short_lens)."""
    long_seqs = np.full((n_users + 1, long_max_len), n_items, dtype=np.int32)
    short_seqs = np.full((n_users + 1, short_max_len), n_items, dtype=np.int32)
    long_lens = np.ones(n_users + 1, dtype=np.int32)
    short_lens = np.ones(n_users + 1, dtype=np.int32)
    total = long_max_len + short_max_len
    for u in range(n_users):
        items = list(user_consumed[u]) if u in user_consumed else []
        n = len(items)
        if n <= short_max_len:
            short_seqs[u, :n] = items
            short_lens[u] = n
            continue
        if n < total:
            long_seqs[u, :n - short_max_len] = items[:n - short_max_len]
            long_lens[u] = n - short_max_len
        else:
            long_seqs[u] = items[n - total:n - short_max_len]
            long_lens[u] = long_max_len
        short_seqs[u] = items[n - short_max_len:]
        short_lens[u] = short_max_len
    return long_seqs, long_lens, short_seqs, short_lens


def recent_dual_sequences_csr(consumed, n_items, long_max_len, short_max_len):
    """Vectorised :func:`recent_dual_sequences` over a ConsumedCSR (arrival order), no per-user Python loop."""
    indptr, idx = np.asarray(consumed.indptr, dtype=np.int64), consumed.idx
    n_users = len(indptr) - 1
    c = np.diff(indptr)
    slen = np.minimum(c, short_max_len)
    lreal = np.clip(c - short_max_len, 0, long_max_len)          # items before the short window, capped
    t_l = np.arange(long_max_len, dtype=np.int64)[None, :]
    t_s = np.arange(short_max_len, dtype=np.int64)[None, :]
    long_seqs = np.full((n_users + 1, long_max_len), n_items, dtype=np.int32)
    short_seqs = np.full((n_users + 1, short_max_len), n_items, dtype=np.int32)
    src = (indptr[:-1] + c - short_max_len - lreal)[:, None] + t_l
    valid = t_l < lreal[:, None]
    long_seqs[:n_users][valid] = idx[src[valid]]
    src = (indptr[1:] - slen)[:, None] + t_s
    valid = t_s < slen[:, None]
    short_seqs[:n_users][valid] = idx[src[valid]]
    long_lens = np.append(np.where(c <= short_max_len, 1, lreal), 1).astype(np.int32)
    short_lens = np.append(slen, 1).astype(np.int32)
    return long_seqs, long_lens, short_seqs, short_lens


class SIM(_SeqModelBase):
    """libreco/algorithms/sim.py:193-304 (inference = the second stage, ``sim.py:206-207``): the item table
    Gp = combine_seq_features(concat) Wp [n_items+1, K]; for a pair (u, n) with q = Gp[n] the GSU selects the
    ``search_topk`` positions of the user's long sequence with the largest q . Gp[long_t] (masked positions score -1e9,
    equal scores resolve to the lower position), the ESU runs ``multi_head_attention`` of q over the selected rows, the
    short sequence gets Keras dot-product attention, and ``dense_nn`` (relu) runs on [long_out, short_out, user, item,
    sparse.., dense..], then Dense(1).

    Weights (besides the embedding tables): ``seq_proj`` [K', K], ``sim_attention`` {wq, wk, wv, wo [K, K]} (``wv``
    the effective value map), ``num_heads``, ``mlp``, ``out_kernel``, ``out_bias`` — :func:`weights_io.sim_weights`
    makes them from either TensorFlow graph's variables.  ``long_seqs`` / ``short_seqs`` and their lengths are the
    reference's ``cached_long_seqs`` ... (:func:`recent_dual_sequences`).

    All-items scoring (``b200_sim_pair_scores``) builds Gp, the item queries Qp = Gp Wq and the item part of the first
    layer once per model and each user's Gp[long] Wk / Wv once per call, then scores every pair without building the
    [B*N, F*K + 2K] concat.  Rows mode (``predict``, feature rows, ``recommend_dynamic`` with features, an MLP outside
    the pair kernel's envelope) writes [long_out, short_out] into the concat (``b200_sim_attention``) for the relu MLP
    on the library's dense layers."""

    def __init__(self, spec, weights, long_seqs, long_lens, short_seqs, short_lens, user_consumed=None,
                 task="ranking", search_topk=10, device=None):
        raw_is = None
        if not isinstance(spec, FeatSpec):
            g = _spec_get(spec)
            raw_is = g("item_sparse_unique") if g("item_sparse_col_index") else None
        super().__init__(spec, weights, short_seqs, short_lens, user_consumed, task, device)
        torch = self._torch
        f32 = torch.float32
        K, F = self.K, self.F
        self.long_seqs = _dev(long_seqs, self.device, torch.int32)
        self.long_lens = _dev(long_lens, self.device, torch.int32)
        self.L, self.S = int(self.long_seqs.shape[1]), self.T
        self.topk = int(search_topk)
        H = self.num_heads = int(weights["num_heads"])
        if K > SIM_MAX_K:
            raise ValueError(f"SIM: embed size {K} > {SIM_MAX_K} is not supported")
        if H < 1 or K % H:
            raise ValueError(f"SIM: embed size {K} must be divisible by num_heads {H}")
        if not 1 <= self.L <= SIM_MAX_L:
            raise ValueError(f"SIM: long sequence length {self.L} outside [1, {SIM_MAX_L}]")
        if not 1 <= self.S <= SIM_MAX_S:
            raise ValueError(f"SIM: short sequence length {self.S} outside [1, {SIM_MAX_S}]")
        if not 1 <= self.topk <= min(SIM_MAX_TOPK, self.L):
            raise ValueError(f"SIM: search_topk {self.topk} outside [1, min({SIM_MAX_TOPK}, long length {self.L})]")
        # combine_seq_features reads the item sparse columns as they are (multi-sparse sub-columns one by one)
        self._item_sparse = _dev(raw_is, self.device, torch.int32) if raw_is is not None else self.spec.is_
        att = weights["sim_attention"]
        for k in ("wq", "wk", "wv", "wo"):
            if np.shape(att[k]) != (K, K):
                raise ValueError(f"SIM: attention {k} has shape {np.shape(att[k])}, expected ({K}, {K})")
        self._wo64 = np.asarray(att["wo"], dtype=np.float64)
        tr = lambda a: _dev(np.ascontiguousarray(np.asarray(a, dtype=np.float32).T), self.device, f32)   # noqa: E731
        self._seq_projT, self._wqT, self._wkT, self._wvT = (tr(weights["seq_proj"]), tr(att["wq"]), tr(att["wk"]),
                                                             tr(att["wv"]))
        self.Wo = _dev(np.asarray(att["wo"], dtype=np.float32), self.device, f32)
        if np.shape(weights["mlp"]["kernels"][0])[0] != (F + 2) * K:
            raise ValueError(f"SIM: the first MLP layer takes {np.shape(weights['mlp']['kernels'][0])[0]} inputs, "
                             f"expected (F + 2)*K = ({F} + 2)*{K}")
        self._rebuild_item_features()
        self.extra = 2 * K
        # reference order [long, short, user, item, sparse.., dense..] -> ours [user, item, sparse.., dense.., long, short]
        perm = np.concatenate([np.arange(2 * K, (F + 2) * K), np.arange(0, 2 * K)])
        self.mlp = self._upload_mlp(permute_mlp_input(weights["mlp"], perm))

    def _rebuild_item_features(self):
        """Gp = combine_seq_features(concat) Wp [n_items+1, K] (sim.py:197-199), the item queries Qp = Gp Wq and their
        transposes for the pair kernel: once per set of tables (again after ``assign_oov``)."""
        torch = self._torch
        n = self.n_items + 1
        parts = [self.t["item_embeds"]]
        if self._item_sparse is not None:
            parts.append(self.t["sparse_embeds"][self._item_sparse.long()].reshape(n, -1))
        if self.spec.id_ is not None:
            cols = torch.as_tensor(self.spec.item_dense_cols, device=self.device)
            parts.append((self.spec.id_[:, :, None] * self.t["dense_embeds"][cols][None]).reshape(n, -1))
        G = torch.cat(parts, dim=1).contiguous()
        if G.shape[1] != self._seq_projT.shape[1]:
            raise ValueError(f"SIM: the item feature table has {G.shape[1]} columns, the sequence projection takes "
                             f"{self._seq_projT.shape[1]}")
        self.Gp = linear(G, self._seq_projT, None, ACT_NONE, impl="f32")
        self.Qp = linear(self.Gp, self._wqT, None, ACT_NONE, impl="f32")
        self.GpT = self.Gp.t().contiguous()
        self.QpT = self.Qp.t().contiguous()

    def _slots(self, users_d):
        """The given users' long / short rows and lengths and their keys / values Gp[long] Wk, Gp[long] Wv."""
        u = users_d.long()
        ls, ll = self.long_seqs[u].contiguous(), self.long_lens[u].contiguous()
        ss, sl = self.seqs[u].contiguous(), self.lens[u].contiguous()
        g = self.Gp[ls.view(-1).long()]
        Kl = linear(g, self._wkT, None, ACT_NONE, impl="f32")
        Vl = linear(g, self._wvT, None, ACT_NONE, impl="f32")
        return ls, ll, ss, sl, Kl, Vl

    def _pair_dims(self):
        dims = [w.shape[0] for w, _, _ in self.mlp]
        return dims[0], dims[1], dims[2] if len(dims) == 3 else 0

    def _hoistable(self):
        """The pair kernel takes 2 or 3 Dense layers of at most 256, 128, 64 units whose shared memory fits."""
        if len(self.mlp) not in (2, 3):
            return False
        need = _lib.lib.b200_sim_pair_smem_bytes(self.K, self.L, self.S, self.topk, *self._pair_dims())
        return 0 < need <= self._torch.cuda.get_device_properties(self.device).shared_memory_per_block_optin

    def score_all_items(self, user_ids_d):
        """sim.py:249-304 over (these users) x (every item): per call each user's keys / values, then every pair in
        ``b200_sim_pair_scores``.  The item part of the first layer and W_att = [Wo W1_long ; W1_short] (multiplied in
        float64) are made once per model."""
        torch = self._torch
        if not self._hoistable():
            return super().score_all_items(user_ids_d)
        N, FK, K = self.n_items, self.F * self.K, self.K
        if "_item_part" not in self.__dict__:
            xi = self._side_concat("item", torch.arange(N, device=self.device))
            self._item_part = self._first_layer_partial("item", xi, False).t().contiguous()       # [H1, N]
            W1 = self.mlp[0][0].double().cpu().numpy()                                             # [H1, FK + 2K]
            w_att = np.concatenate([self._wo64 @ W1[:, FK:FK + K].T, W1[:, FK + K:FK + 2 * K].T], axis=0)
            self._w_att = _dev(w_att.astype(np.float32), self.device, torch.float32)              # [2K, H1]
            three = len(self.mlp) == 3
            self._sim_tail = (self.mlp[1][0].t().contiguous(), self.mlp[2][0].t().contiguous() if three else None)
        PiT = self._item_part
        W2, W3 = self._sim_tail
        H1, H2, H3 = self._pair_dims()
        b = int(user_ids_d.numel())
        scores = torch.empty((b, N), dtype=torch.float32, device=self.device)
        for r0 in range(0, b, 65535):
            u = user_ids_d[r0:r0 + 65535]
            nb = int(u.numel())
            Pu = self._first_layer_partial("user", self._side_concat("user", u), True)     # [nb, H1] incl. bias
            ls, ll, ss, sl, Kl, Vl = self._slots(u)
            out = scores[r0:r0 + nb]
            _lib.check(_lib.lib.b200_sim_pair_scores(
                _lib.ptr(self.GpT), _lib.ptr(self.QpT), self.GpT.stride(0), N, _lib.ptr(self.Gp), self.Gp.stride(0),
                _lib.ptr(ls), ls.stride(0), _lib.ptr(ll), _lib.ptr(ss), ss.stride(0), _lib.ptr(sl), _lib.ptr(Kl),
                _lib.ptr(Vl), _lib.ptr(Pu), nb, _lib.ptr(PiT), PiT.stride(0), K, self.num_heads, self.L, self.S,
                self.topk, H1, H2, H3, _lib.ptr(self._w_att), _lib.ptr(W2), _lib.ptr(self.mlp[1][1]), _lib.ptr(W3),
                _lib.ptr(self.mlp[2][1]) if W3 is not None else None, _lib.ptr(self.out_kernel), self.out_bias,
                _lib.ptr(out), out.stride(0), _lib.current_stream()))
        return scores

    def _seq_block(self, users_d, items_d, n, grid_items, row_offset, out_view, gsu_pos=None):
        """[long_out, short_out] of each row, every distinct user (grid slot) of the chunk prepared once."""
        torch = self._torch
        if grid_items > 0:
            u0 = row_offset // grid_items
            u1 = (row_offset + n - 1) // grid_items
            su, slot, items, off = users_d[u0:u1 + 1], None, None, row_offset - u0 * grid_items
        else:
            su, inv = torch.unique(users_d, return_inverse=True)
            slot, items, off = inv.to(torch.int32).contiguous(), items_d.to(torch.int64).contiguous(), 0
        ls, ll, ss, sl, Kl, Vl = self._slots(su)
        _lib.check(_lib.lib.b200_sim_attention(
            _lib.ptr(self.Gp), self.Gp.stride(0), _lib.ptr(self.Qp), self.Qp.stride(0), self.K, self.num_heads,
            _lib.ptr(ls), ls.stride(0), _lib.ptr(ll), _lib.ptr(Kl), _lib.ptr(Vl), self.L, _lib.ptr(ss), ss.stride(0),
            _lib.ptr(sl), self.S, self.topk, _lib.ptr(self.Wo), _lib.ptr(slot), _lib.ptr(items), n, grid_items, off,
            _lib.ptr(out_view), out_view.stride(0), _lib.ptr(gsu_pos), _lib.current_stream()))

    def attention_rows(self, users, items):
        """([long_out, short_out] [R, 2K], the GSU's selected positions int32 [R, search_topk] in ascending order) of
        explicit (user, item) rows — the rows-mode kernel on its own."""
        torch = self._torch
        u = torch.as_tensor(np.asarray(users, dtype=np.int64)).to(self.device)
        i = torch.as_tensor(np.asarray(items, dtype=np.int64)).to(self.device)
        n = int(u.numel())
        out = torch.empty((n, 2 * self.K), dtype=torch.float32, device=self.device)
        pos = torch.empty((n, self.topk), dtype=torch.int32, device=self.device)
        if n:
            self._seq_block(u, i, n, 0, 0, out, pos)
        return out, pos

    def _swap_user_seq(self, u, seq, data_info, inner_id):
        """Both rows of user ``u`` from ``seq`` (``build_dual_seq``, recommendation/preprocess.py:49-76)."""
        from .dynamic_feats import build_dual_seq

        ls, ll, ss, sl = build_dual_seq(seq, self.n_items, self.L, self.S, getattr(data_info, "item2id", None),
                                        inner_id)
        tables = (self.long_seqs, self.long_lens, self.seqs, self.lens)
        old = [t[u].clone() for t in tables]
        for t, v in zip(tables, (ls[0], ll[0], ss[0], sl[0])):
            t[u] = self._torch.as_tensor(v).to(self.device)

        def restore():
            for t, v in zip(tables, old):
                t[u] = v
        return restore


class TwoTower:
    """libreco/algorithms/two_tower.py:306-346,400-410 + DynEmbedBase.set_embeddings
    (libreco/bases/dyn_embed_base.py:240-269): both towers over ALL users / items on the GPU; the
    results (plus the mean OOV rows of embed_base.py:257-265) feed the embed scorer directly."""

    def __init__(self, spec, weights, norm_embed=False, device=None):
        import torch

        self._torch = torch
        K = int(weights["user_embeds"].shape[1])
        spec, weights = combine_multi_sparse(spec, weights, weights.get("multi_sparse_combiner", "sqrtn"), device)
        self.base = FeatSpec(spec, K, device)
        self.device = self.base.device
        self.K = K
        self.norm_embed = norm_embed
        self.n_users, self.n_items = self.base.n_users, self.base.n_items
        f32 = torch.float32
        self.t = {k: _dev(weights.get(k), self.device, f32) for k in
                  ("user_embeds", "item_embeds", "sparse_embeds", "dense_embeds")}
        self.tables = tables_struct(self.t)
        self.mlps = {which: [(_dev(Wt, self.device, f32), _dev(b, self.device, f32), relu)
                             for Wt, b, relu in fold_mlp(weights[f"{which}_tower"])] for which in ("user", "item")}

    def tower(self, which, ids):
        torch = self._torch
        ids_d = torch.as_tensor(np.asarray(ids, dtype=np.int64)).to(self.device)
        n = ids_d.numel()
        L, pos = self.base.side(which)
        x = torch.empty((n, len(pos) * self.K), dtype=torch.float32, device=self.device)
        feat_forward(L, self.tables, ids_d, ids_d, n, concat=x)
        for Wt, b, relu in self.mlps[which]:
            x = linear(x, Wt, b, relu)
        if self.norm_embed:
            _lib.check(_lib.lib.b200_l2_normalize_rows(_lib.ptr(x), x.stride(0), n, x.shape[1],
                                                       _lib.current_stream()))
        return x

    def set_embeddings(self, chunk=1 << 20):
        """User / item vectors of every id + the mean OOV row; returns device tensors
        [n_users+1, d], [n_items+1, d]."""
        torch = self._torch
        outs = []
        for which, n in (("user", self.n_users), ("item", self.n_items)):
            E = _chunked_rows(lambda ids: self.tower(which, ids), n, chunk)
            outs.append(torch.cat([E, E.mean(dim=0, keepdim=True)], dim=0))
        return outs[0], outs[1]


class YouTubeRetrieval:
    """libreco/algorithms/youtube_retrieval.py:169-260 (inference; SURVEY 8f-4 adjacent model) + the serving step of
    ``DynEmbedBase.set_embeddings`` / ``dyn_user_embedding`` (``bases/dyn_embed_base.py:166-269``): the user vector is
    ``dense_nn(concat(sqrtn-pooled behaviour sequence over seq_embeds_var, user sparse embeddings, user dense
    value x embedding))`` (optionally L2-normalised) with a pseudo bias 1 appended, the item vector is
    ``[item_embeds_var | item_bias_var]`` — the reference's own trick for folding the softmax bias into the dot
    product — so all-items retrieval IS the embed scorer (K4) on d = H + 1.  The sequence of a user = its last
    ``T`` consumed items (``_set_recent_seqs``; ``feat_models.recent_sequences``), pooled by ``b200_seq_pool``
    (sum / sqrt(count) = ``safe_embedding_lookup_sparse(combiner="sqrtn")``, empty history -> zero vector)."""

    def __init__(self, spec, weights, recent_seqs, recent_seq_lens, norm_embed=False, device=None):
        import torch

        self._torch = torch
        K = int(np.asarray(weights["seq_embeds"]).shape[1])
        self.base = FeatSpec(spec, K, device)
        self.device, self.K, self.norm_embed = self.base.device, K, bool(norm_embed)
        self.n_users, self.n_items = self.base.n_users, self.base.n_items
        f32 = torch.float32
        self.seq_embeds = _dev(weights["seq_embeds"], self.device, f32)              # [n_items, K]
        self.item_embeds = _dev(weights["item_embeds"], self.device, f32)            # [n_items, H]
        self.item_biases = _dev(np.asarray(weights["item_biases"]).reshape(-1), self.device, f32)
        self.t = {k: _dev(weights.get(k), self.device, f32) for k in ("sparse_embeds", "dense_embeds")}
        self.tables = tables_struct(self.t)
        self.seqs = _dev(recent_seqs, self.device, torch.int32)
        self.lens = _dev(recent_seq_lens, self.device, torch.int32)
        self.mlp = [(_dev(Wt, self.device, f32), _dev(b, self.device, f32), relu) for Wt, b, relu in fold_mlp(weights["mlp"])]

    def user_vectors(self, ids):
        """[n, H] user embeddings of the given (inner) user ids, before the pseudo bias.  ``ValueError`` for an id
        outside ``[0, n_users]`` or without a cached sequence row."""
        torch = self._torch
        ids = _check_user_ids("YouTubeRetrieval", ids, self.n_users, self.seqs.shape[0])
        ids_d = torch.as_tensor(ids).to(self.device)
        n, K = int(ids_d.numel()), self.K
        L, pos = self.base.side("user", with_id=False)      # no id-embedding field: the pooled sequence takes its place
        x = torch.empty((n, (1 + len(pos)) * K), dtype=torch.float32, device=self.device)
        pooled = x[:, :K]
        _lib.check(_lib.lib.b200_seq_pool(
            _lib.ptr(self.seq_embeds), self.seq_embeds.stride(0), K, self.n_items, _lib.ptr(self.seqs),
            self.seqs.stride(0), _lib.ptr(self.lens), self.seqs.shape[1], _lib.ptr(ids_d), n, 0, 0, _lib.ptr(pooled),
            x.stride(0), _lib.current_stream()))
        if pos:
            feat_forward(L, self.tables, ids_d, ids_d, n, concat=x[:, K:])
        for Wt, b, relu in self.mlp:
            x = linear(x, Wt, b, relu)
        if self.norm_embed:
            _lib.check(_lib.lib.b200_l2_normalize_rows(_lib.ptr(x), x.stride(0), n, x.shape[1], _lib.current_stream()))
        return x

    def set_embeddings(self, chunk=1 << 20):
        """Device tensors ``U [n_users + 1, H + 1]`` (pseudo bias 1 in the last column, last row = mean OOV row) and
        ``I [n_items + 1, H + 1]`` (``[item_embeds | item_biases]`` + the mean row) for :class:`engine.EmbedScorer`."""
        U = _chunked_rows(self.user_vectors, self.n_users, chunk)
        return dyn_embed_tables(U, self.item_embeds, self.item_biases, self.norm_embed)


def _n_users_items(data_info_or_spec):
    """``(n_users, n_items)`` of a ``DataInfo`` or of a dict holding both."""
    if isinstance(data_info_or_spec, dict):
        return int(data_info_or_spec["n_users"]), int(data_info_or_spec["n_items"])
    return int(data_info_or_spec.n_users), int(data_info_or_spec.n_items)


def _check_user_ids(name, ids, n_users, n_rows=None):
    """``ids`` as a flat host int64 array.  The kernels index the user and sequence tables with them unchecked, so
    an id outside ``[0, n_users]``, or (with ``n_rows``, the cached sequence rows) at or past ``n_rows``, raises
    ``ValueError`` here."""
    ids = np.asarray(ids, dtype=np.int64).reshape(-1)
    if ids.size and (ids.min() < 0 or ids.max() > n_users):
        raise ValueError(f"{name}: user ids must lie in [0, {n_users}]")
    if ids.size and n_rows is not None and ids.max() >= n_rows:
        raise ValueError(f"{name}: user id {ids.max()} has no cached sequence: {n_rows} recent sequence rows")
    return ids


def _chunked_rows(rows_of, n, chunk):
    """``rows_of(ids)`` over the ids ``0 .. n-1`` in chunks of ``chunk`` ids, concatenated on the device."""
    import torch

    return torch.cat([rows_of(np.arange(i, min(n, i + chunk))) for i in range(0, n, chunk)], dim=0)


def dyn_embed_tables(U, item_embeds, item_biases, norm_embed):
    """The serving tables of ``DynEmbedBase.set_embeddings`` (``bases/dyn_embed_base.py:240-269``) and
    ``embed_base.py:257-265`` from the device user vectors ``U [n_users, d]``: ``[U | 1]`` and ``[I | b]`` with
    ``I = item_embeds`` (L2-normalised when ``norm_embed``; the user vectors arrive normalised already), each with
    its column-mean row appended -> ``[n_users + 1, d + 1]``, ``[n_items + 1, d + 1]``."""
    import torch

    I = _dyn_item_rows(item_embeds, item_biases, norm_embed)
    U = torch.cat([U, torch.ones((U.shape[0], 1), dtype=torch.float32, device=U.device)], dim=1)
    return (torch.cat([U, U.mean(dim=0, keepdim=True)], dim=0).contiguous(),
            torch.cat([I, I.mean(dim=0, keepdim=True)], dim=0).contiguous())


def _dyn_item_rows(item_embeds, item_biases, norm_embed):
    """``[I | b]`` [n_items, d + 1] of :func:`dyn_embed_tables`, without the mean row."""
    import torch

    if norm_embed:          # dyn_embed_base.py:264-265: the item side is normalised too (before the bias column)
        I = item_embeds / item_embeds.norm(dim=1, keepdim=True)
    else:
        I = item_embeds
    return torch.cat([I, item_biases[:, None]], dim=1)


class _DynEmbedSeqModel:
    """What the ``DynEmbedBase`` sequence-encoder models share (``bases/dyn_embed_base.py:166-283``,
    ``recommendation/preprocess.py:26-46``): each user's recent sequence (``recent_sequences``: right-padded with
    ``n_items``) goes through the subclass's encoder kernel and a Dense head on :func:`linear` into the user vector
    (L2-normalised as a whole with ``norm_embed``); the item side is ``[item_embeds | item_bias]`` and the user side
    gets the pseudo bias 1, so all-items retrieval is the embed scorer on d = ``item_embeds`` width + 1.

    A subclass supplies ``_check_weights(weights, recent_seqs)``, which raises ``ValueError`` outside the kernel's
    envelope before the device lookup and returns ``{attribute: host array}`` of its own float32 device tables, and
    ``_features(ids_d, rows_d, seqs, lens)``, the [n, d] rows before the normalisation of the users ``ids_d`` over the
    rows ``rows_d`` of ``seqs`` / ``lens`` (None: the recent sequences).  ``_before_set_embeddings`` may prepare the
    tables before ``set_embeddings`` encodes."""

    NAME = ""
    READS_LENS = False      # whether the encoder reads the sequence lengths
    _I = None               # [I | b] of recommend_dynamic, built on its first call

    def __init__(self, data_info_or_spec, weights, recent_seqs, recent_seq_lens, norm_embed, device):
        import torch

        self._torch = torch
        self.n_users, self.n_items = _n_users_items(data_info_or_spec)
        self.norm_embed = bool(norm_embed)
        self.T = int(np.shape(recent_seqs)[1])
        own = self._check_weights(weights, recent_seqs)
        self.device = torch.device(device) if device is not None else _lib.require_cuda()
        f32 = torch.float32
        self.seq_embeds = _dev(weights["seq_embeds"], self.device, f32)          # [n_items + 1, encoder input]
        self.item_embeds = _dev(weights["item_embeds"], self.device, f32)        # [n_items, d]
        self.item_biases = _dev(np.asarray(weights["item_biases"]).reshape(-1), self.device, f32)
        self.dense_Wt = _dev(np.asarray(weights["dense_kernel"]).T, self.device, f32)    # [K, pre-head width]
        self.dense_b = _dev(np.asarray(weights["dense_bias"]).reshape(-1), self.device, f32)
        self.seqs = _dev(recent_seqs, self.device, torch.int32)
        self.lens = _dev(np.asarray(recent_seq_lens).reshape(-1), self.device, torch.int32)
        for k, a in own.items():
            setattr(self, k, _dev(a, self.device, f32))

    def _before_set_embeddings(self):
        pass

    def user_vectors(self, ids, seqs=None, lens=None):
        """[n, d] user vectors of the users ``ids`` (0..n_users; n_users is the unknown user), L2-normalised with
        ``norm_embed``.  The sequence of ``ids[i]`` is its recent sequence or, when given, row i of ``seqs`` [n, T]
        (host or device) with length ``lens[i]``, which only a model that reads lengths reads.  A row's bits depend
        only on its own user and sequence.  ``ValueError`` before any launch for an id outside ``[0, n_users]``, an id
        without a cached sequence row (no ``seqs``), or ``seqs`` / ``lens`` that are not ``[n, T]`` / ``[n]``."""
        torch = self._torch
        ids = _check_user_ids(self.NAME, ids, self.n_users, self.seqs.shape[0] if seqs is None else None)
        n = int(ids.size)
        if self.READS_LENS and (seqs is None) != (lens is None):
            raise ValueError("give both `seqs` and `lens`, or neither")
        ids_d = rows_d = torch.as_tensor(ids).to(self.device)
        if seqs is not None:
            seqs = _dev(seqs, self.device, torch.int32)
            if tuple(seqs.shape) != (n, self.T):
                raise ValueError(f"`seqs` has shape {tuple(seqs.shape)}, expected ({n}, {self.T})")
            if self.READS_LENS:
                lens = _dev(lens.reshape(-1) if isinstance(lens, torch.Tensor) else np.asarray(lens).reshape(-1),
                            self.device, torch.int32)
                if tuple(lens.shape) != (n,):
                    raise ValueError(f"`lens` has shape {tuple(lens.shape)}, expected ({n},)")
            rows_d = torch.arange(n, dtype=torch.int64, device=self.device)
        if n == 0:
            return torch.empty((0, self.item_embeds.shape[1]), dtype=torch.float32, device=self.device)
        x = self._features(ids_d, rows_d, seqs, lens)
        if self.norm_embed:
            _lib.check(_lib.lib.b200_l2_normalize_rows(_lib.ptr(x), x.stride(0), n, x.shape[1],
                                                       _lib.current_stream()))
        return x

    def set_embeddings(self, chunk=1 << 20):
        """Device tensors ``U [n_users + 1, d + 1]`` (pseudo bias 1 in the last column, last row = the mean row) and
        ``I [n_items + 1, d + 1]`` (``[item_embeds | item_biases]`` + the mean row) for :class:`engine.EmbedScorer`."""
        self._before_set_embeddings()
        U = _chunked_rows(self.user_vectors, self.n_users, chunk)
        return dyn_embed_tables(U, self.item_embeds, self.item_biases, self.norm_embed)

    def recommend_dynamic(self, user_id, n_rec, data_info, user_feats=None, seq=None, filter_consumed=True,
                          inner_id=False, return_scores=False):
        """``recommend_user`` for ONE user (inner id; ``n_users`` = the unknown user) with an optional behaviour
        sequence supplied for this call (``dyn_embed_base.py:166-214``, ``recommendation/preprocess.py:26-46``): the
        sequence is cut to its last ``max_seq_len`` items and unknown original ids become the pad id ``n_items``;
        without one the user's cached sequence is used.  ``user_feats`` is accepted and ignored (no user features).
        The vector scores ``I[:n_items]`` with the pseudo bias, then the consumed filter (none for the unknown user)
        and top-K select.  The model's tables are not touched."""
        from .dynamic_feats import build_rec_seq

        if n_rec > self.n_items:
            raise ValueError(f"`n_rec` {n_rec} exceeds num of items {self.n_items}")
        u = int(user_id)
        if seq is not None and len(seq) > 0:
            row, ln = build_rec_seq(seq, self.n_items, self.T, getattr(data_info, "item2id", None), inner_id)
            v = self.user_vectors([u], row, ln)
        else:
            v = self.user_vectors([u])
        return self._dynamic_topk(v, u, n_rec, data_info, filter_consumed, return_scores)

    def _dynamic_topk(self, v, u, n_rec, data_info, filter_consumed, return_scores):
        """The scoring tail of ``recommend_dynamic``: the user vector ``v`` [1, d] with the pseudo bias 1 appended
        scores ``[I | b]`` over ``I[:n_items]``, then the consumed filter of user ``u`` and top-K select."""
        torch = self._torch
        dev = self.device
        if self._I is None:
            self._I = _dyn_item_rows(self.item_embeds, self.item_biases, self.norm_embed).contiguous()
        q = torch.cat([v, torch.ones((1, 1), dtype=torch.float32, device=dev)], dim=1).contiguous()
        N, d = self.n_items, q.shape[1]
        scores = torch.empty((1, N), dtype=torch.float32, device=dev)
        zero = torch.zeros(1, dtype=torch.int64, device=dev)
        _lib.check(_lib.lib.b200_score_rows_f32(_lib.ptr(q), q.stride(0), _lib.ptr(zero), 1, _lib.ptr(self._I),
                                                self._I.stride(0), N, d, _lib.ptr(scores), scores.stride(0),
                                                _lib.current_stream()))
        consumed = getattr(data_info, "user_consumed", None)
        owner = _ConsumedOwner(consumed, self.n_users, self.n_items, dev)
        out_ids = torch.empty((1, n_rec), dtype=torch.int64, device=dev)
        out_sc = torch.empty((1, n_rec), dtype=torch.float32, device=dev)
        uid = torch.tensor([u], dtype=torch.int64, device=dev)
        masked_topk(owner, scores, uid, n_rec, filter_consumed, out_ids, out_sc)
        ids = out_ids.cpu().numpy()
        return (ids, out_sc.cpu().numpy()) if return_scores else ids


RNN_MAX_T, RNN_MAX_DIM, RNN_MAX_LAYERS = 128, 256, 4     # the envelope of b200_rnn_encode


class RNN4Rec(_DynEmbedSeqModel):
    """libreco/algorithms/rnn4rec.py:151-237 (inference) + the serving step of ``DynEmbedBase``
    (:class:`_DynEmbedSeqModel`).  The user vector is ``tf_dense(embed_size)(rnn(seq_embeds[seq]))`` (optionally
    L2-normalised): ``b200_rnn_encode`` runs the stacked GRU / LSTM over each user's recent sequence (len 0 for no
    history) and :func:`linear` the head, so d = embed_size.  ``weights``: the dict of ``weights_io.rnn4rec_weights``
    (or the raw variables it takes).  RNN4Rec has no user table and no user features: users with the same sequence
    get the same vector."""

    NAME = "RNN4Rec"
    READS_LENS = True

    def __init__(self, data_info_or_spec, weights, recent_seqs, recent_seq_lens, norm_embed=False, device=None):
        from .weights_io import rnn4rec_weights

        if "rnn_scheme" in weights:
            weights = rnn4rec_weights(weights)
        super().__init__(data_info_or_spec, weights, recent_seqs, recent_seq_lens, norm_embed, device)

    def _check_weights(self, weights, recent_seqs):
        layers = weights["rnn_layers"]
        self.in_dim = int(np.shape(weights["seq_embeds"])[1])
        self.hidden = [int(np.shape(lw["U"])[0]) for lw in layers]
        self.K = int(np.shape(weights["dense_kernel"])[1])
        if not 1 <= self.T <= RNN_MAX_T:
            raise ValueError(f"RNN4Rec: max_seq_len {self.T} outside [1, {RNN_MAX_T}]")
        if not 1 <= len(layers) <= RNN_MAX_LAYERS:
            raise ValueError(f"RNN4Rec: {len(layers)} recurrent layers, supported 1 to {RNN_MAX_LAYERS}")
        if max([self.in_dim] + self.hidden) > RNN_MAX_DIM:
            raise ValueError(f"RNN4Rec: input width {self.in_dim} / hidden sizes {self.hidden} exceed {RNN_MAX_DIM}")
        packed, d = [], self.in_dim
        for lw, H in zip(layers, self.hidden):
            parts = [np.asarray(lw[k], dtype=np.float32).reshape(-1) for k in ("W", "U", "bx", "bh", "gamma", "beta")]
            flat = np.concatenate(parts)
            if flat.size != int(_lib.lib.b200_rnn_layer_floats(int(lw["kind"]), d, H)):
                raise ValueError(f"RNN4Rec: layer of kind {lw['kind']} with input {d} and hidden {H} has {flat.size} "
                                 "packed floats")
            packed.append(flat)
            d = H
        self.kinds = (ctypes.c_int32 * len(layers))(*[int(lw["kind"]) for lw in layers])
        self.hid = (ctypes.c_int32 * len(layers))(*self.hidden)
        self.acts = (ctypes.c_int32 * len(layers))(*[int(lw["act"]) for lw in layers])
        return {"rnn_w": np.concatenate(packed)}

    def encode(self, ids_d, seqs=None, lens=None):
        """[n, H_last]: ``b200_rnn_encode`` of the rows ``ids_d`` (device int64) of ``seqs`` / ``lens`` (default: the
        model's recent sequences)."""
        torch = self._torch
        seqs = self.seqs if seqs is None else seqs
        lens = self.lens if lens is None else lens
        n = int(ids_d.numel())
        h = torch.empty((n, self.hidden[-1]), dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_rnn_encode(
            _lib.ptr(ids_d), n, _lib.ptr(lens), _lib.ptr(seqs), seqs.stride(0), self.T, _lib.ptr(self.seq_embeds),
            self.seq_embeds.stride(0), self.in_dim, len(self.hidden), self.kinds, self.hid, self.acts,
            _lib.ptr(self.rnn_w), _lib.ptr(h), h.stride(0), _lib.current_stream()))
        return h

    def _features(self, ids_d, rows_d, seqs, lens):
        return linear(self.encode(rows_d, seqs, lens), self.dense_Wt, self.dense_b, ACT_NONE, impl="f32")


CONV_MAX_T, CONV_MAX_K, CONV_MAX_FILTERS, CONV_MAX_F, CONV_MAX_LAYERS = 64, 128, 32, 128, 16   # b200_*_encode envelope


class _ConvSeqModel(_DynEmbedSeqModel):
    """What Caser and WaveNet add to :class:`_DynEmbedSeqModel`: a user table.  The user vector is
    ``[user_embeds[u] | head(encoder(seq_embeds[seq]))]`` (d = 2K), where the encoder is the subclass's kernel (the
    pad positions are ordinary rows, neither model masks by length).  The user table's last row ``n_users`` is the
    unknown user's: ``set_embeddings`` first sets it to the mean of the other rows (``_assign_user_oov``), and a cold
    and a warm user with the same sequence get different vectors."""

    HEAD_ACT = ACT_NONE

    def _check_weights(self, weights, recent_seqs):
        self.K = int(np.shape(weights["seq_embeds"])[1])
        if not 1 <= self.T <= CONV_MAX_T:
            raise ValueError(f"{self.NAME}: max_seq_len {self.T} outside [1, {CONV_MAX_T}]")
        if not 1 <= self.K <= CONV_MAX_K:
            raise ValueError(f"{self.NAME}: embed_size {self.K} outside [1, {CONV_MAX_K}]")
        shapes = {"user_embeds": (self.n_users + 1, self.K), "seq_embeds": (self.n_items + 1, self.K),
                  "item_embeds": (self.n_items, 2 * self.K), "dense_bias": (self.K,)}
        for k, shp in shapes.items():
            if tuple(np.shape(weights[k])) != shp:
                raise ValueError(f"{self.NAME}: `{k}` has shape {np.shape(weights[k])}, expected {shp}")
        if np.shape(recent_seqs)[0] != self.n_users + 1:
            raise ValueError(f"{self.NAME}: {np.shape(recent_seqs)[0]} recent sequences for {self.n_users} users + "
                             "the OOV row")
        self._check_encoder(weights)
        return {"user_embeds": weights["user_embeds"], "conv_w": weights["conv"]}

    def _check_encoder(self, weights):
        raise NotImplementedError

    def _encode_into(self, rows_d, seqs, out):
        raise NotImplementedError

    def encode(self, rows_d, seqs=None):
        """[n, D] pre-head features of the rows ``rows_d`` (device int64) of ``seqs`` (default: the model's recent
        sequences)."""
        seqs = self.seqs if seqs is None else seqs
        out = self._torch.empty((int(rows_d.numel()), self.dense_Wt.shape[1]), dtype=self._torch.float32,
                                device=self.device)
        self._encode_into(rows_d, seqs, out)
        return out

    def _features(self, ids_d, rows_d, seqs, lens):
        n, K = int(ids_d.numel()), self.K
        x = self._torch.empty((n, 2 * K), dtype=self._torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_gather_rows(_lib.ptr(self.user_embeds), self.user_embeds.stride(0), K,
                                             _lib.ptr(ids_d), n, _lib.ptr(x), x.stride(0), _lib.current_stream()))
        x[:, K:] = linear(self.encode(rows_d, seqs), self.dense_Wt, self.dense_b, self.HEAD_ACT, impl="f32")
        return x

    def assign_user_oov(self):
        """``_assign_user_oov`` (dyn_embed_base.py:271-283): the unknown user's row := mean of the known rows."""
        self.user_embeds[self.n_users] = self.user_embeds[:self.n_users].mean(dim=0)

    _before_set_embeddings = assign_user_oov


class Caser(_ConvSeqModel):
    """libreco/algorithms/caser.py:135-221 (inference): ``b200_caser_encode`` runs the T horizontal convolutions
    (kernel sizes 1..T, ReLU, max over the valid positions) and the vertical one over each user's recent sequence;
    the head is ``Dense(K, relu)``.  ``weights``: the dict of ``weights_io.caser_weights`` (or the raw variables it
    takes, ``synthetic.make_caser_weights``).  ``use_bn`` and ``dropout_rate`` are never read by the graph."""

    NAME = "Caser"
    HEAD_ACT = ACT_RELU

    def __init__(self, data_info_or_spec, weights, recent_seqs, recent_seq_lens, norm_embed=False, device=None):
        from .weights_io import caser_weights

        if "conv" not in weights:
            weights = caser_weights(weights)
        super().__init__(data_info_or_spec, weights, recent_seqs, recent_seq_lens, norm_embed, device)

    def _check_encoder(self, weights):
        self.nh, self.nv = int(weights["nh"]), int(weights["nv"])
        if int(weights["T"]) != self.T:
            raise ValueError(f"Caser: {weights['T']} horizontal convolutions, max_seq_len is {self.T}")
        if not (1 <= self.nh <= CONV_MAX_FILTERS and 1 <= self.nv <= CONV_MAX_FILTERS):
            raise ValueError(f"Caser: nh_filters {self.nh} / nv_filters {self.nv} outside [1, {CONV_MAX_FILTERS}]")
        D = self.T * self.nh + self.K * self.nv
        if np.size(weights["conv"]) != int(_lib.lib.b200_caser_weight_floats(self.T, self.K, self.nh, self.nv)):
            raise ValueError(f"Caser: {np.size(weights['conv'])} packed convolution floats do not match T {self.T}, "
                             f"K {self.K}, nh {self.nh}, nv {self.nv}")
        if tuple(np.shape(weights["dense_kernel"])) != (D, self.K):
            raise ValueError(f"Caser: `dense_kernel` has shape {np.shape(weights['dense_kernel'])}, expected "
                             f"({D}, {self.K})")

    def _encode_into(self, rows_d, seqs, out):
        _lib.check(_lib.lib.b200_caser_encode(
            _lib.ptr(rows_d), int(rows_d.numel()), _lib.ptr(seqs), seqs.stride(0), self.T, _lib.ptr(self.seq_embeds),
            self.seq_embeds.stride(0), self.K, self.nh, self.nv, _lib.ptr(self.conv_w), _lib.ptr(out), out.stride(0),
            _lib.current_stream()))


class WaveNet(_ConvSeqModel):
    """libreco/algorithms/wave_net.py:139-222 (inference): ``b200_wavenet_encode`` runs the causal dilated
    convolutions (kernel size 2, ReLU), the 1x1 convolution (ReLU) and the max over the T positions over each
    user's recent sequence; the head is ``Dense(K)`` without activation.  ``weights``: the dict of
    ``weights_io.wavenet_weights`` (or the raw variables it takes, ``synthetic.make_wavenet_weights``), which
    carries the per-layer dilations: ``2**i`` in layer i of a block, or 1 everywhere for a model built by TF1."""

    NAME = "WaveNet"

    def __init__(self, data_info_or_spec, weights, recent_seqs, recent_seq_lens, norm_embed=False, device=None):
        from .weights_io import wavenet_weights

        if "conv" not in weights:
            weights = wavenet_weights(weights)
        super().__init__(data_info_or_spec, weights, recent_seqs, recent_seq_lens, norm_embed, device)

    def _check_encoder(self, weights):
        self.F, dil = int(weights["F"]), [int(d) for d in weights["dilations"]]
        if not 1 <= self.F <= CONV_MAX_F:
            raise ValueError(f"WaveNet: n_filters {self.F} outside [1, {CONV_MAX_F}]")
        if not 1 <= len(dil) <= CONV_MAX_LAYERS or min(dil) < 1:
            raise ValueError(f"WaveNet: dilations {dil}: 1 to {CONV_MAX_LAYERS} causal layers, each dilation >= 1")
        if np.size(weights["conv"]) != int(_lib.lib.b200_wavenet_weight_floats(self.K, self.F, len(dil))):
            raise ValueError(f"WaveNet: {np.size(weights['conv'])} packed convolution floats do not match K {self.K}, "
                             f"F {self.F}, {len(dil)} causal layers")
        if tuple(np.shape(weights["dense_kernel"])) != (self.F, self.K):
            raise ValueError(f"WaveNet: `dense_kernel` has shape {np.shape(weights['dense_kernel'])}, expected "
                             f"({self.F}, {self.K})")
        self.dilations = dil
        self.dil = (ctypes.c_int32 * len(dil))(*dil)

    def _encode_into(self, rows_d, seqs, out):
        _lib.check(_lib.lib.b200_wavenet_encode(
            _lib.ptr(rows_d), int(rows_d.numel()), _lib.ptr(seqs), seqs.stride(0), self.T, _lib.ptr(self.seq_embeds),
            self.seq_embeds.stride(0), self.K, len(self.dilations), self.F, self.dil, _lib.ptr(self.conv_w),
            _lib.ptr(out), out.stride(0), _lib.current_stream()))


class _ConsumedOwner:
    """What :func:`engine.masked_topk` reads: the catalogue size and the consumed CSR on the device."""

    def __init__(self, user_consumed, n_users, n_items, device):
        csr = user_consumed if user_consumed is not None else ConsumedCSR(np.zeros(1, dtype=np.int64),
                                                                          np.zeros(0, dtype=np.int32))
        self.n_items = n_items
        self.csr = as_csr(csr, n_users)
        self.indptr_d, self.idx_d = self.csr.device(device)
