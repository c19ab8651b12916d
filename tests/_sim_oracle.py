"""Numpy restatement of the reference's SIM inference graph (the second stage).  TEST INFRASTRUCTURE ONLY.

**PARITY UNPINNED**, like every graph in ``oracle/tf_models.py``: TensorFlow is not available, so this follows the graph
definitions line by line and is cross-checked in float64, but it is not verified against a TensorFlow run.

Graph restated (reference @ 7463d9d):
* item table           ``Gp = combine_seq_features(concat) @ Wp`` (``sim.py:197-199``, ``tf_models.item_feature_table``)
* GSU                  ``sim.py:264-286``: q . Gp[long_t], masked positions REPLACED by -1e9, ``tf.math.top_k`` (equal
                       scores resolve to the lower position: a stable sort)
* ESU                  ``multi_head_attention`` (``layers/attention.py:67-138``) of q over the selection, both graphs:
                       "keras" adds -1e9 to hidden logits (formed in float32), "legacy" writes -1e9 with ``tf.where`` and
                       applies its value Dense to the projected keys
* short attention      ``tf_attention`` (Keras dot-product attention, no scale, hidden logits fl32(logit - 1e9))
* head                 ``dense_nn`` (relu) on [long_out, short_out, user, item, sparse.., dense..], then Dense(1)

``w`` holds the raw variables of ``synthetic.make_sim_weights`` plus, for multi-sparse layouts, ``multi_sparse`` as in
``oracle/tf_models.py``.
"""
import numpy as np

from oracle import tf_models as tm
import _transformer_oracle as to

NEG = 1.0e9


def item_table(w, spec, dtype):
    """Gp [n_items+1, K]."""
    return tm.item_feature_table(w, spec, dtype) @ np.asarray(w["seq_proj"], dtype=dtype)


def gsu_scores(Gp, items, long_seqs, long_lens):
    """[R, L]: q . Gp[long_t], -1e9 where t >= long_len (sim.py:264-272)."""
    s = np.einsum("rk,rtk->rt", Gp[items], Gp[long_seqs])
    mask = np.arange(long_seqs.shape[1])[None, :] < np.asarray(long_lens).reshape(-1, 1)
    return np.where(mask, s, -NEG)


def gsu_select(scores, k):
    """tf.math.top_k's set (equal scores: the lower position), returned in ascending position order [R, k]."""
    order = np.argsort(-scores, axis=1, kind="stable")[:, :k]
    return np.sort(order, axis=1)


def gsu_margin(scores, long_lens, k):
    """Per row the float64 gap between the k-th largest VALID score s_k and the nearest other valid score value, above
    or below (inf when at most k positions are valid: the selection is then every valid position plus the lowest
    masked ones), and |s_k|.  Scores equal to s_k are exact ties (copies of one item), which float32 reproduces
    exactly and the lower-position rule resolves, so they do not narrow the margin."""
    R, L = scores.shape
    out, sk = np.full(R, np.inf), np.zeros(R)
    for r in range(R):
        ln = min(max(int(long_lens[r]), 0), L)
        if ln > k:
            b = np.sort(scores[r, :ln])[::-1][k - 1]
            vals = np.unique(scores[r, :ln])
            i = int(np.searchsorted(vals, b))
            gaps = ([b - vals[i - 1]] if i > 0 else []) + ([vals[i + 1] - b] if i + 1 < len(vals) else [])
            out[r], sk[r] = (min(gaps) if gaps else np.inf), abs(b)
    return out, sk


def esu(w, q, sel_rows, sel_valid, dtype, scheme=None):
    """multi_head_attention(q[:, None], sel_rows, H, K/H, mask) [R, K] of either graph."""
    scheme = scheme or w["sim_scheme"]
    H = int(w["num_heads"])
    m = tm._cast(w["sim_mha"], dtype)
    K = q.shape[1]
    hd = K // H
    if scheme == "keras":
        qh = np.einsum("rd,dhk->rhk", q, m["query"]) * dtype(1.0 / np.sqrt(hd))
        kh = np.einsum("rtd,dhk->rthk", sel_rows, m["key"])
        vh = np.einsum("rtd,dhk->rthk", sel_rows, m["value"])
        a = to.keras_masked(np.einsum("rhk,rthk->rht", qh, kh), sel_valid[:, None, :])
        o = np.einsum("rht,rthk->rhk", to._softmax(a), vh)
        return np.einsum("rhk,hkd->rd", o, m["attention_output"])
    split = lambda x: x.reshape(*x.shape[:-1], H, hd)      # noqa: E731
    qh = split(q @ m["query"])
    keys = sel_rows @ m["key"]
    vh = split(keys @ m["value"])
    a = np.einsum("rhk,rthk->rht", qh, split(keys)) * dtype(1.0 / np.sqrt(dtype(hd)))
    a = np.where(sel_valid[:, None, :], a, dtype(-NEG))
    o = np.einsum("rht,rthk->rhk", to._softmax(a), vh)
    return o.reshape(len(q), K) @ m["output"]


def sim_forward(w, spec, users, items, long_seqs, long_lens, short_seqs, short_lens, k, sparse=None, dense=None,
                dtype=np.float64, scheme=None, sel=None):
    """sim.py:249-304 — (logits, the selected positions [R, k] ascending, margins, |s_k|) of the rows (users, items);
    the sequence tables are per user.  ``sel`` forces the GSU selection."""
    users, items = np.asarray(users), np.asarray(items)
    c = tm._cast(w, dtype)
    Gp = item_table(w, spec, dtype)
    ls, ll = np.asarray(long_seqs)[users], np.asarray(long_lens)[users]
    ss, sl = np.asarray(short_seqs)[users], np.asarray(short_lens)[users]
    scores = gsu_scores(Gp, items, ls, ll)
    margin, sk = gsu_margin(scores, ll, k)
    if sel is None:
        sel = gsu_select(scores, k)
    sel = np.asarray(sel)
    q = Gp[items]
    rows = Gp[np.take_along_axis(ls, sel, axis=1)]
    valid = sel < np.clip(ll, 0, None).reshape(-1, 1)
    long_out = esu(w, q, rows, valid, dtype, scheme)
    short_out = to.target_attention(q, Gp[ss], sl, dtype)
    P, _ = tm._stacked_embeds(c, users, items, sparse, dense, dtype)
    x = np.concatenate([long_out, short_out, P.reshape(len(users), -1)], axis=1)
    h = tm.dense_nn(x, c["mlp"])
    z = (h @ c["out_kernel"].reshape(-1, 1) + c["out_bias"].reshape(-1)[0]).reshape(-1)
    return z, sel, margin, sk


# ------------------------------------------------------------------------------------------------------
# seeded cases shared by the GPU tests and the CPU checks
# ------------------------------------------------------------------------------------------------------
# (layout, K, num_heads, use_bn, version)
CASES = [
    ("ids", 16, 2, True, "keras"),          # the reference defaults
    ("feat", 16, 1, False, "legacy"),
    ("feat", 16, 4, True, "keras"),
    ("multi", 16, 2, True, "legacy"),
    ("ids", 8, 4, False, "legacy"),
    ("multi", 32, 2, False, "keras"),
]
L_DEFAULT, S_DEFAULT, TOPK_DEFAULT = 100, 10, 10


def case_id(c):
    return "-".join(str(v) for v in c)


def make_consumed(rng, n_users, n_items, L, S, k):
    """{user: item list} with every history length class: 0 .. S items (long length 1), S+1 .. S+k-1 (fewer valid
    long positions than search_topk), full windows, and histories whose duplicates straddle the top-k boundary."""
    consumed = {}
    for u in range(n_users):
        kind = u % 6
        if kind == 0:
            n = int(rng.integers(0, S + 1))
        elif kind == 1:
            n = S + int(rng.integers(1, k))
        elif kind == 2:
            n = L + S + int(rng.integers(0, 20))
        elif kind == 3:
            n = S + int(rng.integers(k, L))
        else:
            n = int(rng.integers(S + k + 1, L + S + 1))
        items = rng.integers(0, n_items, size=n)
        if kind >= 4 and n > S + 2:
            # a few items repeated across the long window: exact GSU ties for every target item
            pool = rng.integers(0, n_items, size=4)
            items[:n - S] = pool[rng.integers(0, 4, size=n - S)]
        consumed[u] = [int(i) for i in items]
    consumed[0] = []
    consumed[1] = [i % n_items for i in range(L + S)]
    return consumed


def make_case(c, seed=0, n_users=48, n_items=70, L=L_DEFAULT, S=S_DEFAULT, k=TOPK_DEFAULT, hidden=(200, 80)):
    """(rng, spec, raw weights, consumed, (long_seqs, long_lens, short_seqs, short_lens))."""
    from librecommender_b200 import synthetic as syn
    from librecommender_b200.feat_models import recent_dual_sequences

    layout, K, H, bn, version = c
    rng = np.random.default_rng(seed + 7 * K + H)
    if layout == "ids":
        spec = syn.make_spec(rng, n_users, n_items, [], [], 0, 0)
    elif layout == "feat":
        spec = syn.make_spec(rng, n_users, n_items, [7, 30], [11, 5], 1, 2)
    else:
        spec = syn.make_multi_sparse_spec(rng, n_users, n_items, [9], [12, 6], [("user", 17, 3), ("item", 23, 2)], 1, 1)
    w = syn.make_sim_weights(rng, spec, K, H, hidden, bn, version)
    if layout == "multi":
        w["multi_sparse"] = dict(spec["multi_sparse_combine_info"], combiner="sqrtn")
    consumed = make_consumed(rng, n_users, n_items, L, S, k)
    seqs = recent_dual_sequences(consumed, n_users, n_items, L, S)
    return rng, spec, w, consumed, seqs


def case_rows(rng, spec, R=400):
    """(users, items, sparse, dense): OOV users and items included."""
    users = rng.integers(0, spec["n_users"] + 1, size=R)
    items = rng.integers(0, spec["n_items"] + 1, size=R)
    users[:3], items[3:6] = spec["n_users"], spec["n_items"]
    users[6:12] = np.arange(6)
    sparse, dense = tm.row_features(spec, users, items)
    return users, items, sparse, dense
