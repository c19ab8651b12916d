"""Float64 (or float32) numpy restatement of RNN4Rec inference (libreco/algorithms/rnn4rec.py:151-237) from the RAW
variables of either TensorFlow graph of ``layers/recurrent.py:4-63``, written the way TensorFlow computes them and
independently of the engine's canonical W / U layout:

* "legacy" (TF 1): ``MultiRNNCell`` under ``dynamic_rnn(sequence_length=len)``; ``GRUCell`` with the gates and
  candidate kernels over ``[x, h]`` / ``[x, r * h]``, ``LSTMCell`` with blocks i | j | f | o and ``forget_bias`` 1.0
  added at run time.  Steps t >= len copy the state through; the result is the last layer's final state (its h).
* "keras" (TF >= 2): one ``GRU`` (reset_after) / ``LSTM`` layer per hidden size over all T steps with the mask,
  masked steps keeping the state and repeating the previous output, then (``use_layer_norm``) LayerNormalization
  (eps 1e-3) and tanh; the result is ``output[:, -1]``.

The cell formulas are TensorFlow's, restated (no TensorFlow exists here).  Then the Dense head, the optional L2
normalisation and the serving tables of ``DynEmbedBase.set_embeddings``."""
from __future__ import annotations

import numpy as np


def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def _ln(x, gamma, beta, eps=1e-3):
    mean = x.mean(axis=-1, keepdims=True)
    var = ((x - mean) ** 2).mean(axis=-1, keepdims=True)
    return (x - mean) / np.sqrt(var + eps) * gamma + beta


def legacy_rnn(X, lens, layers, rnn_type, dtype=np.float64):
    """dynamic_rnn over MultiRNNCell: X [n, T, in] -> the last layer's final h [n, H_last]."""
    c = lambda a: np.asarray(a, dtype=dtype)      # noqa: E731
    n, T, _ = X.shape
    widths = [np.shape(lw["candidate_kernel"])[1] if rnn_type == "gru" else np.shape(lw["kernel"])[1] // 4
              for lw in layers]
    hs = [np.zeros((n, H), dtype=dtype) for H in widths]
    cs = [np.zeros_like(h) for h in hs]
    one = dtype(1.0)
    for t in range(T):
        live = (t < lens)[:, None]
        x = X[:, t]
        for i, lw in enumerate(layers):
            h = hs[i]
            if rnn_type == "gru":
                H = h.shape[1]
                value = _sig(np.concatenate([x, h], axis=1) @ c(lw["gates_kernel"]) + c(lw["gates_bias"]))
                r, u = value[:, :H], value[:, H:]
                cand = np.tanh(np.concatenate([x, r * h], axis=1) @ c(lw["candidate_kernel"]) + c(lw["candidate_bias"]))
                new_h = u * h + (one - u) * cand
                new_c = cs[i]
            else:
                H = h.shape[1]
                m = np.concatenate([x, h], axis=1) @ c(lw["kernel"]) + c(lw["bias"])
                ig, j, f, o = m[:, :H], m[:, H:2 * H], m[:, 2 * H:3 * H], m[:, 3 * H:]
                new_c = cs[i] * _sig(f + one) + _sig(ig) * np.tanh(j)
                new_h = np.tanh(new_c) * _sig(o)
            hs[i] = np.where(live, new_h, h)
            cs[i] = np.where(live, new_c, cs[i])
            x = hs[i]
    return hs[-1]


def keras_rnn(X, lens, layers, rnn_type, use_layer_norm, dtype=np.float64):
    """The Keras layer stack over all T steps with the sequence mask -> output[:, -1] [n, H_last]."""
    c = lambda a: np.asarray(a, dtype=dtype)      # noqa: E731
    n, T, _ = X.shape
    mask = np.arange(T)[None, :] < lens[:, None]
    act = (lambda v: v) if use_layer_norm else np.tanh
    seq = X
    one = dtype(1.0)
    for lw in layers:
        U = c(lw["recurrent_kernel"])
        H = U.shape[0]
        h = np.zeros((n, H), dtype=dtype)
        cc = np.zeros((n, H), dtype=dtype)
        out_prev = np.zeros((n, H), dtype=dtype)
        outs = np.zeros((n, T, H), dtype=dtype)
        for t in range(T):
            x = seq[:, t]
            if rnn_type == "gru":
                b = c(lw["bias"])
                mx = x @ c(lw["kernel"]) + b[0]
                mi = h @ U + b[1]
                z = _sig(mx[:, :H] + mi[:, :H])
                r = _sig(mx[:, H:2 * H] + mi[:, H:2 * H])
                hh = act(mx[:, 2 * H:] + r * mi[:, 2 * H:])
                new_h, new_c = z * h + (one - z) * hh, cc
            else:
                m = x @ c(lw["kernel"]) + h @ U + c(lw["bias"])
                ig, f, g, o = _sig(m[:, :H]), _sig(m[:, H:2 * H]), m[:, 2 * H:3 * H], _sig(m[:, 3 * H:])
                new_c = f * cc + ig * act(g)
                new_h = o * act(new_c)
            live = mask[:, t][:, None]
            h = np.where(live, new_h, h)
            cc = np.where(live, new_c, cc)
            out_prev = np.where(live, new_h, out_prev)
            outs[:, t] = out_prev
        if use_layer_norm:
            outs = np.tanh(_ln(outs, c(lw["gamma"]), c(lw["beta"])))
        seq = outs
    return seq[:, -1]


def rnn_states(raw, seqs, lens, dtype=np.float64):
    """Encoder output [n, H_last] of the rows ``seqs`` [n, T] / ``lens`` [n] for the raw variables ``raw``."""
    lens = np.clip(np.asarray(lens, dtype=np.int64), 0, seqs.shape[1])
    X = np.asarray(raw["seq_embeds"], dtype=dtype)[np.asarray(seqs, dtype=np.int64)]
    if raw["rnn_scheme"] == "legacy":
        return legacy_rnn(X, lens, raw["rnn_layers"], raw["rnn_type"], dtype)
    return keras_rnn(X, lens, raw["rnn_layers"], raw["rnn_type"], bool(raw.get("use_layer_norm")), dtype)


def user_vectors(raw, seqs, lens, norm_embed=False, dtype=np.float64):
    """``tf_dense(embed_size)`` over the encoder output, L2-normalised with ``norm_embed`` -> [n, K]."""
    h = rnn_states(raw, seqs, lens, dtype)
    v = h @ np.asarray(raw["dense_kernel"], dtype=dtype) + np.asarray(raw["dense_bias"], dtype=dtype).reshape(-1)
    if norm_embed:
        v = v / np.linalg.norm(v, axis=1, keepdims=True)
    return v


def serving_tables(raw, U, norm_embed=False, dtype=np.float64):
    """``[U | 1]`` and ``[I | b]`` with their column-mean rows (dyn_embed_base.py:240-269, embed_base.py:257-265)."""
    I = np.asarray(raw["item_embeds"], dtype=dtype)
    if norm_embed:
        I = I / np.linalg.norm(I, axis=1, keepdims=True)
    U = np.hstack([U, np.ones((U.shape[0], 1), dtype=dtype)])
    I = np.hstack([I, np.asarray(raw["item_biases"], dtype=dtype).reshape(-1, 1)])
    return np.vstack([U, U.mean(axis=0, keepdims=True)]), np.vstack([I, I.mean(axis=0, keepdims=True)])


def recommend(raw, U, users, n_rec, user_consumed, filter_consumed=True, norm_embed=False):
    """Top-K of ``U[users] . I[:n_items]`` through ``oracle.ranking`` -> (ids, full scores)."""
    from oracle import ranking as orc

    Uf, If = serving_tables(raw, U, norm_embed)
    n_items = np.shape(raw["item_embeds"])[0]
    full = Uf[np.asarray(users)] @ If[:n_items].T
    ids = orc.rank_recommendations("ranking", list(map(int, users)), full.astype(np.float32).copy(), n_rec, n_items,
                                   user_consumed, filter_consumed)
    return ids, full
