"""Numpy restatement of the reference's AutoInt graph (inference forward).  TEST INFRASTRUCTURE ONLY.

**PARITY UNPINNED**, like every graph in ``oracle/tf_models.py``: TensorFlow is not available, so this follows
the graph definitions line by line and is cross-checked in float64, but it is not verified against a
TensorFlow run.

Graph restated (reference @ 7463d9d):
* AutoInt            ``libreco/algorithms/autoint.py:146-168`` (field block = ``concat_embed``, :152-158)
* multi_head_attention ``libreco/layers/attention.py:67-138``, BOTH graphs it builds:
  - "keras" (TF >= 2.10): ``tf.keras.layers.MultiHeadAttention(num_heads, head_dim, use_bias=False,
    output_shape=K)`` — einsum projections with [K, H, hd] kernels, the query scaled by 1/sqrt(hd) BEFORE the
    product, softmax over the keys, [H, hd, K] output kernel (third-party Keras code, restated from its
    documented computation);
  - "legacy": four bias-free ``tf_dense``; ``values = tf_dense(D)(keys)`` applied to the already projected
    keys (:104-106), the scores multiplied by rsqrt(hd) AFTER the product (:112-113), ``_split_heads`` /
    ``_combine_heads`` reshapes (:124-138).

``w`` holds the raw per-version variables of ``synthetic.make_autoint_weights`` (``autoint_scheme``,
``autoint_mha``, ``num_heads``, ``use_residual``, ``out_kernel``, ``out_bias``) plus the embedding tables and,
for multi-sparse layouts, ``multi_sparse`` as in ``oracle/tf_models.py``.
"""
import numpy as np

from oracle import tf_models as tm


def _softmax(a):
    a = a - a.max(axis=-1, keepdims=True)
    e = np.exp(a)
    return e / e.sum(axis=-1, keepdims=True)


def mha_keras(x, lw, dtype):
    """tf.keras.layers.MultiHeadAttention(query=x, value=x, use_bias=False): x [R, F, K]."""
    hd = lw["query"].shape[2]
    q = np.einsum("rfk,khd->rfhd", x, lw["query"])
    k = np.einsum("rfk,khd->rfhd", x, lw["key"])
    v = np.einsum("rfk,khd->rfhd", x, lw["value"])
    q = q * dtype(1.0 / np.sqrt(hd))
    p = _softmax(np.einsum("rghd,rfhd->rhfg", k, q))
    o = np.einsum("rhfg,rghd->rfhd", p, v)
    return np.einsum("rfhd,hdk->rfk", o, lw["attention_output"])


def _split_heads(x, H, hd):
    return x.reshape(*x.shape[:-1], H, hd).transpose(0, 2, 1, 3)


def mha_legacy(x, lw, H, dtype):
    """attention.py:102-122 for queries = keys = x [R, F, K]."""
    D = lw["query"].shape[1]
    hd = D // H
    queries = x @ lw["query"]
    keys = x @ lw["key"]
    values = keys @ lw["value"]                     # tf_dense(D)(keys): the PROJECTED keys
    q, k, v = _split_heads(queries, H, hd), _split_heads(keys, H, hd), _split_heads(values, H, hd)
    att = (q @ k.transpose(0, 1, 3, 2)) * dtype(1.0 / np.sqrt(dtype(hd)))
    out = _softmax(att) @ v                         # [R, H, F, hd]
    out = out.transpose(0, 2, 1, 3).reshape(x.shape[0], x.shape[1], D)
    return out @ lw["output"]


def field_block(w, users, items, sparse=None, dense=None, dtype=np.float64):
    """``tf.concat(concat_embed, axis=1)`` (autoint.py:152-158): [R, F, K]."""
    w = tm._cast({k: v for k, v in w.items() if k != "autoint_mha"}, dtype)
    P, _ = tm._stacked_embeds(w, np.asarray(users), np.asarray(items), sparse, dense, dtype)
    return P


def autoint_forward(w, users, items, sparse=None, dense=None, dtype=np.float64, version=None):
    """autoint.py:160-168 — logits.  `version` defaults to the scheme the weights were made for."""
    version = version or w["autoint_scheme"]
    x = field_block(w, users, items, sparse, dense, dtype)
    mha = tm._cast(w["autoint_mha"], dtype)
    H = int(w["num_heads"])
    for lw in mha:
        y = mha_keras(x, lw, dtype) if version == "keras" else mha_legacy(x, lw, H, dtype)
        x = x + y if w["use_residual"] else y
    flat = x.reshape(len(x), -1)
    return (flat @ np.asarray(w["out_kernel"], dtype=dtype).reshape(-1, 1)
            + dtype(np.asarray(w["out_bias"]).reshape(-1)[0])).reshape(-1)


# ------------------------------------------------------------------------------------------------------
# seeded cases shared by the GPU tests and the CPU check of their tolerance
# ------------------------------------------------------------------------------------------------------
# (layout, K, att_embed_size, num_heads, use_residual, version)
CASES = [
    ("feat", 16, None, 1, True, "keras"),          # the reference's own test configs (tests/models/test_autoint.py)
    ("feat", 16, 16, 2, False, "legacy"),
    ("feat", 16, (4, 8), 2, False, "keras"),
    ("feat", 16, None, 1, True, "legacy"),
    ("ids", 4, (8, 8, 8), 2, True, "keras"),       # ids only, K = 4
    ("ids", 16, 16, 2, False, "legacy"),
    ("feat", 64, (8, 8, 8), 2, True, "keras"),     # K = 64
    ("feat", 64, 16, 4, True, "legacy"),           # D = 64
    ("multi", 16, (8, 8, 8), 2, True, "keras"),    # multi-sparse fields, sqrtn
    ("multi", 16, (8, 8, 8), 2, True, "legacy"),
    ("feat", 4, (3, 5), 3, False, "keras"),        # D = 9, 15: not a multiple of 4
    ("feat", 8, (1, 1), 5, True, "legacy"),        # hd = 1
]


def case_id(c):
    return "-".join(str(v).replace(" ", "") for v in c)


def make_case(c, seed=0, n_users=120, n_items=150):
    """(spec, raw weights) of one case; ``raw["multi_sparse"]`` is set for the oracle where needed."""
    from librecommender_b200 import synthetic as syn

    layout, K, att, H, res, version = c
    rng = np.random.default_rng(seed + 7 * K + H)
    if layout == "ids":
        spec = syn.make_spec(rng, n_users, n_items, [], [], 0, 0)
    elif layout == "feat":
        spec = syn.make_spec(rng, n_users, n_items, [7, 30], [11, 5, 40], 1, 2)
    else:
        spec = syn.make_multi_sparse_spec(rng, n_users, n_items, [9, 30], [12, 6, 25],
                                          [("user", 17, 3), ("item", 23, 4)], 1, 1)
    w = syn.make_autoint_weights(rng, spec, K, att, H, res, version)
    if layout == "multi":
        w["multi_sparse"] = dict(spec["multi_sparse_combine_info"], combiner="sqrtn")
    return rng, spec, w


def case_rows(rng, spec, R=500):
    """(users, items, sparse, dense) with the OOV user / item rows included."""
    users = rng.integers(0, spec["n_users"] + 1, size=R)
    items = rng.integers(0, spec["n_items"] + 1, size=R)
    users[:3], items[3:6] = spec["n_users"], spec["n_items"]
    sparse, dense = tm.row_features(spec, users, items)
    return users, items, sparse, dense


def close(got, ref, tol=1e-5):
    """|got - ref| <= tol * max(|ref|, mean |ref|) + 1e-6 elementwise: the bound of test_gpu_feat_models._close."""
    scale = np.maximum(np.abs(ref), np.abs(ref).mean())
    err = np.abs(got - ref)
    assert (err <= tol * scale + 1e-6).all(), float(err.max())


# attention logits around +-100: the first layer's query and key maps scaled up
LARGE_LOGIT_CASE = ("feat", 16, (8, 8), 2, True, "keras")


def attention_logits_first_layer(w, users, items, sparse, dense):
    """Scaled scores <q_f, k_g> / sqrt(hd) of the first layer (float64), [R, H, F, F]."""
    x = field_block(w, users, items, sparse, dense, np.float64)
    lw = w["autoint_mha"][0]
    hd = lw["query"].shape[2]
    q = np.einsum("rfk,khd->rfhd", x, lw["query"].astype(np.float64))
    k = np.einsum("rfk,khd->rfhd", x, lw["key"].astype(np.float64))
    return np.einsum("rghd,rfhd->rhfg", k, q) / np.sqrt(hd)


def scale_to_large_logits(w, rows, target=100.0):
    """Scale layer 0's query and key kernels (in place) so the largest attention logit over `rows`
    ((users, items, sparse, dense)) is about `target`."""
    s = np.abs(attention_logits_first_layer(w, *rows)).max()
    f = np.sqrt(target / s)
    lw = w["autoint_mha"][0]
    lw["query"] = (lw["query"] * f).astype(np.float32)
    lw["key"] = (lw["key"] * f).astype(np.float32)
