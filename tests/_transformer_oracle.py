"""Numpy restatement of the reference's Transformer graph (inference forward).  TEST INFRASTRUCTURE ONLY.

**PARITY UNPINNED**, like every graph in ``oracle/tf_models.py``: TensorFlow is not available, so this follows
the graph definitions line by line and is cross-checked in float64, but it is not verified against a
TensorFlow run.

Graph restated (reference @ 7463d9d):
* Transformer          ``libreco/algorithms/transformer.py:203-339``
* item features        ``combine_seq_features`` (``tfops/features.py:151-236``): concat (``tf_models.item_feature_table``)
                       or elementwise ``item * (sum_f LN(sparse_f) + sum_f LN(dense_f) + 1)``, LN eps 1e-8
* positions            ``layers/transformer.py:113-144`` (sinusoidal) or the trainable table
* multi_head_attention ``layers/attention.py:67-138``, both graphs: "keras" adds -1e9 to hidden scores (formed in
                       float32), "legacy" writes -1e9 with ``tf.where`` and applies its value Dense to the projected keys
* the mask             ``t < len`` OR-ed with the causal mask (``transformer.py:320-326``), literally
* tf_attention         Keras dot-product attention without scale, hidden scores - 1e9 formed in float32
* dense_nn             with swish (``layers/dense.py:12-49``, ``layers/activation.py:10-11``)

``w`` holds the raw variables of ``synthetic.make_transformer_weights`` plus the embedding tables and, for
multi-sparse layouts, ``multi_sparse`` as in ``oracle/tf_models.py``.
"""
import numpy as np
from scipy.special import erf

from oracle import tf_models as tm

NEG = 1.0e9


def rms_norm(x, scale):
    return x / np.sqrt(np.mean(np.square(x), axis=-1, keepdims=True) + x.dtype.type(1e-8)) * scale


def layer_norm(x, ln):
    mean = x.mean(axis=-1, keepdims=True)
    var = np.square(x - mean).mean(axis=-1, keepdims=True)
    return (x - mean) / np.sqrt(var + x.dtype.type(1e-8)) * ln["scale"] + ln["bias"]


def gelu(x):
    return 0.5 * x * (1.0 + erf(x / np.sqrt(2.0)))


def swish(x):
    return x / (1.0 + np.exp(-x))


def sinusoidal(T, d):
    """positional_encoding (layers/transformer.py:113-144), restated: for odd d the odd columns take the exponents
    of the even columns before them."""
    dim = np.arange(d) / d
    dim[1::2] = dim[0:d - d % 2:2]
    pe = np.arange(T)[:, None] / np.power(10000.0, dim)[None, :]
    pe[:, 0::2] = np.sin(pe[:, 0::2])
    pe[:, 1::2] = np.cos(pe[:, 1::2])
    return pe


def keras_masked(scores, mask):
    """Keras adds -1e9 to the hidden scores in the graph's float32: fl32(score - 1e9)."""
    hidden = (scores.astype(np.float32) - np.float32(NEG)).astype(scores.dtype)
    return np.where(mask, scores, hidden)


def _softmax(a):
    a = a - a.max(axis=-1, keepdims=True)
    e = np.exp(a)
    return e / e.sum(axis=-1, keepdims=True)


def item_table(w, spec, mode, dtype):
    """G [n_items+1, K'] of combine_seq_features."""
    if mode == "concat":
        return tm.item_feature_table(w, spec, dtype)
    c = tm._cast(w, dtype)
    E = c["item_embeds"]
    agg = np.zeros_like(E)
    if len(spec["item_sparse_col_index"]):
        agg = agg + layer_norm(c["sparse_embeds"][spec["item_sparse_unique"]], c["ln_sparse"]).sum(axis=1)
    if len(spec["item_dense_col_index"]):
        cols = spec["item_dense_col_index"]
        de = spec["item_dense_unique"][:, :, None].astype(dtype) * c["dense_embeds"][cols][None]
        agg = agg + layer_norm(de, c["ln_dense"]).sum(axis=1)
    return E * (agg + 1.0)


def attention_mask(lens, T, causal):
    """[B, Tq, Tk]: key k visible to query q when k < len, OR k <= q with the causal mask."""
    m = np.broadcast_to(np.arange(T)[None, None, :] < np.asarray(lens).reshape(-1, 1, 1), (len(lens), T, T))
    if causal:
        m = np.logical_or(m, np.tril(np.ones((T, T), dtype=bool))[None])
    return m


def mha_keras(x, lw, mask, dtype):
    hd = lw["query"].shape[2]
    q = np.einsum("btd,dhk->bthk", x, lw["query"]) * dtype(1.0 / np.sqrt(hd))
    k = np.einsum("btd,dhk->bthk", x, lw["key"])
    v = np.einsum("btd,dhk->bthk", x, lw["value"])
    s = np.einsum("bshk,bqhk->bhqs", k, q)
    p = _softmax(keras_masked(s, mask[:, None]))
    o = np.einsum("bhqs,bshk->bqhk", p, v)
    return np.einsum("bqhk,hkd->bqd", o, lw["attention_output"])


def mha_legacy(x, lw, H, mask, dtype):
    D = lw["query"].shape[1]
    hd = D // H
    split = lambda a: a.reshape(*a.shape[:-1], H, hd).transpose(0, 2, 1, 3)      # noqa: E731
    queries = x @ lw["query"]
    keys = x @ lw["key"]
    values = keys @ lw["value"]                     # tf_dense(D)(keys): the PROJECTED keys
    att = (split(queries) @ split(keys).transpose(0, 1, 3, 2)) * dtype(1.0 / np.sqrt(dtype(hd)))
    att = np.where(mask[:, None], att, dtype(-NEG))
    out = _softmax(att) @ split(values)
    return out.transpose(0, 2, 1, 3).reshape(x.shape[0], x.shape[1], D) @ lw["output"]


def encode(w, G, seqs, lens, dtype, version=None, causal=None):
    """S [B, T, D] (transformer.py:281-306)."""
    version = version or w["tfm_scheme"]
    causal = w["use_causal_mask"] if causal is None else causal
    seqs = np.asarray(seqs)
    T = seqs.shape[1]
    K = np.shape(w["user_embeds"])[1]
    pos = w.get("positional_encoding")
    pos = sinusoidal(T, K) if pos is None else np.asarray(pos)
    x = np.concatenate([G[seqs], np.broadcast_to(pos.astype(dtype), (len(seqs), T, K))], axis=2)
    mask = attention_mask(lens, T, causal)
    H = int(w["num_heads"])
    for lw in tm._cast(w["tfm_layers"], dtype):
        h = rms_norm(x, lw["rms_att"])
        a = (mha_keras(h, lw, mask, dtype) if version == "keras" else mha_legacy(h, lw, H, mask, dtype)) + x
        x = a + gelu(rms_norm(a, lw["rms_ffn"]) @ lw["ffn1"]) @ lw["ffn2"]
    return rms_norm(x, np.asarray(w["rms_last"], dtype=dtype))


def target_attention(q, S, lens, dtype):
    """tf_attention (layers/attention.py:5-25): <q, S_t>, hidden keys fl32(score - 1e9), softmax, sum_t p_t S_t."""
    a = np.einsum("bd,btd->bt", q, S)
    mask = np.arange(S.shape[1])[None, :] < np.asarray(lens).reshape(-1, 1)
    p = _softmax(keras_masked(a, mask))
    return (p[:, :, None] * S).sum(axis=1)


def dense_nn_swish(x, mlp):
    x = tm._bn(x, mlp.get("bn_in"))
    n = len(mlp["kernels"])
    for i in range(n):
        x = x @ mlp["kernels"][i] + mlp["biases"][i]
        if i != n - 1:
            x = swish(x)
            x = tm._bn(x, mlp["bns"][i] if mlp.get("bns") else None)
    return x


def transformer_forward(w, spec, users, items, seqs, lens, sparse=None, dense=None, dtype=np.float64, version=None,
                        causal=None):
    """transformer.py:203-258 — logits of the rows (users, items); seqs / lens are the per-user tables."""
    users, items = np.asarray(users), np.asarray(items)
    c = tm._cast({k: v for k, v in w.items() if k not in ("tfm_layers",)}, dtype)
    G = item_table(w, spec, w.get("feat_agg_mode", "concat"), dtype)
    uniq, inv = np.unique(users, return_inverse=True)
    S = encode(w, G, np.asarray(seqs)[uniq], np.asarray(lens)[uniq], dtype, version, causal)[inv]
    K = np.shape(w["user_embeds"])[1]
    q = np.concatenate([rms_norm(G[items], c["rms_item"]), np.ones((len(items), K), dtype=dtype)], axis=1)
    s_u = target_attention(q, S, np.asarray(lens)[users], dtype)
    P, _ = tm._stacked_embeds(c, users, items, sparse, dense, dtype)
    x = np.concatenate([P.reshape(len(users), -1), s_u], axis=1)
    h = dense_nn_swish(x, c["mlp"])
    return (h @ c["out_kernel"].reshape(-1, 1) + c["out_bias"].reshape(-1)[0]).reshape(-1)


# ------------------------------------------------------------------------------------------------------
# seeded cases shared by the GPU tests and the CPU check of their tolerance
# ------------------------------------------------------------------------------------------------------
# (layout, K, feat_agg_mode, num_heads, n_layers, causal, positional, use_bn, version)
CASES = [
    ("ids", 16, "concat", 1, 1, False, "trainable", True, "keras"),       # the reference defaults (T = 10, D = 32)
    ("feat", 16, "concat", 2, 2, True, "sinusoidal", True, "legacy"),
    ("feat", 16, "elementwise", 4, 1, False, "trainable", False, "keras"),
    ("feat", 8, "concat", 4, 2, False, "sinusoidal", False, "keras"),
    ("multi", 16, "concat", 2, 1, True, "trainable", True, "keras"),
    ("multi", 8, "elementwise", 1, 2, True, "sinusoidal", True, "legacy"),
    ("ids", 7, "concat", 2, 1, True, "sinusoidal", False, "legacy"),       # odd K: odd sinusoidal branch, D = 14
]
T_DEFAULT = 10


def case_id(c):
    return "-".join(str(v) for v in c)


def make_case(c, seed=0, n_users=60, n_items=90, T=T_DEFAULT, hidden=(64, 32)):
    """(rng, spec, raw weights, seqs, lens): user rows of every length 0..T, the reference's OOV row (all padding,
    len 1)."""
    from librecommender_b200 import synthetic as syn

    layout, K, mode, H, L, causal, pos, bn, version = c
    rng = np.random.default_rng(seed + 11 * K + 3 * H + L)
    if layout == "ids":
        spec = syn.make_spec(rng, n_users, n_items, [], [], 0, 0)
    elif layout == "feat":
        spec = syn.make_spec(rng, n_users, n_items, [7, 30], [11, 5], 1, 2)
    else:
        spec = syn.make_multi_sparse_spec(rng, n_users, n_items, [9], [12, 6], [("user", 17, 3), ("item", 23, 2)], 1, 1)
    w = syn.make_transformer_weights(rng, spec, K, H, L, T, hidden, bn, pos, causal, mode, version)
    if layout == "multi":
        w["multi_sparse"] = dict(spec["multi_sparse_combine_info"], combiner="sqrtn")
    seqs = rng.integers(0, n_items, size=(n_users + 1, T)).astype(np.int32)
    lens = rng.integers(0, T + 1, size=n_users + 1).astype(np.int32)
    lens[:3] = [0, 1, T]
    seqs[n_users], lens[n_users] = n_items, 1
    seqs[np.arange(T)[None, :] >= lens[:, None]] = n_items
    return rng, spec, w, seqs, lens


def case_rows(rng, spec, R=300):
    """(users, items, sparse, dense): OOV users and items included, the len 0 / 1 / T users included."""
    users = rng.integers(0, spec["n_users"] + 1, size=R)
    items = rng.integers(0, spec["n_items"] + 1, size=R)
    users[:3], items[3:6] = spec["n_users"], spec["n_items"]
    users[6:9] = [0, 1, 2]
    sparse, dense = tm.row_features(spec, users, items)
    return users, items, sparse, dense


def close(got, ref, tol=1e-5):
    """|got - ref| <= tol * max(|ref|, mean |ref|) + 1e-6 elementwise: the bound of test_gpu_feat_models._close."""
    scale = np.maximum(np.abs(ref), np.abs(ref).mean())
    err = np.abs(got - ref)
    assert (err <= tol * scale + 1e-6).all(), float(err.max())
