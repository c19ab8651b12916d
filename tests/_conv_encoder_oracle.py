"""Float64 (or float32) numpy restatement of Caser and WaveNet inference (libreco/algorithms/caser.py:177-221,
wave_net.py:181-222) from the RAW variables (``synthetic.make_caser_weights`` / ``make_wavenet_weights``), written
the way the Keras layers compute them and independently of the engine's packed layout:

* Caser: ``Conv1D(nh, h, valid, relu)`` + ``MaxPool1D`` over the whole valid length for h = 1..T, then
  ``Conv1D(nv, 1, relu)`` over ``x^T`` flattened row-major, the concat, then ``Dense(K, relu)``.
* WaveNet: ``Conv1D(F, 2, causal, dilation, relu)`` per layer (zeros before the sequence), ``Conv1D(F, 1, relu)``,
  the max over T, then ``Dense(K)``.

Neither graph masks by length: the pad positions (row ``n_items`` of ``seq_embeds``) go through like any other.  The
user vector is ``[user_embeds[u] | head]``; the serving tables and the oracle ranking are RNN4Rec's."""
from __future__ import annotations

import numpy as np

from _rnn4rec_oracle import recommend, serving_tables   # noqa: F401  (the same DynEmbedBase serving)


def _relu(x):
    return np.maximum(x, 0)


def caser_features(raw, seqs, dtype=np.float64):
    """Caser's pre-head concat [n, T*nh + K*nv] of the rows ``seqs`` [n, T]."""
    c = lambda a: np.asarray(a, dtype=dtype)      # noqa: E731
    X = c(raw["seq_embeds"])[np.asarray(seqs, dtype=np.int64)]           # [n, T, K]
    n, T, K = X.shape
    outs = []
    for h, layer in enumerate(raw["convs"], start=1):
        W = c(layer["kernel"]).reshape(h * K, -1)                          # [h*K, nh], j-major like the window
        win = np.stack([X[:, p:p + h].reshape(n, h * K) for p in range(T - h + 1)], axis=1)   # [n, T-h+1, h*K]
        outs.append(_relu(win @ W + c(layer["bias"])).max(axis=1))
    Wv = c(raw["vertical"]["kernel"])[0]                                    # [T, nv]
    v = _relu(np.einsum("ntk,tf->nkf", X, Wv) + c(raw["vertical"]["bias"]))   # [n, K, nv]
    outs.append(v.reshape(n, -1))
    return np.concatenate(outs, axis=1)


def wavenet_features(raw, seqs, dilations=None, dtype=np.float64):
    """WaveNet's pre-head features [n, F] (after the 1x1 layer, ReLU and the max over T) of the rows ``seqs``."""
    c = lambda a: np.asarray(a, dtype=dtype)      # noqa: E731
    x = c(raw["seq_embeds"])[np.asarray(seqs, dtype=np.int64)]
    dilations = raw["dilations"] if dilations is None else dilations
    for layer, d in zip(raw["convs"], dilations):
        W = c(layer["kernel"])                                              # [2, C, F]
        prev = np.zeros_like(x)
        if d < x.shape[1]:
            prev[:, d:] = x[:, :-d]
        x = _relu(prev @ W[0] + x @ W[1] + c(layer["bias"]))
    z = _relu(x @ c(raw["out_conv"]["kernel"])[0] + c(raw["out_conv"]["bias"]))
    return z.max(axis=1)


def assign_user_oov(raw):
    """``_assign_user_oov``: a copy of ``raw`` whose user row n_users is the mean of the other rows."""
    out = dict(raw)
    U = np.array(raw["user_embeds"], dtype=np.float64)
    U[-1] = U[:-1].mean(axis=0)
    out["user_embeds"] = U
    return out


def user_vectors(raw, ids, seqs, norm_embed=False, dtype=np.float64):
    """``[user_embeds[ids] | head(encoder(seqs))]`` [n, 2K] (row i of ``seqs`` beside user ``ids[i]``), L2-normalised
    as a whole with ``norm_embed``."""
    c = lambda a: np.asarray(a, dtype=dtype)      # noqa: E731
    if "vertical" in raw:
        h = _relu(caser_features(raw, seqs, dtype) @ c(raw["dense_kernel"]) + c(raw["dense_bias"]))
    else:
        h = wavenet_features(raw, seqs, dtype=dtype) @ c(raw["dense_kernel"]) + c(raw["dense_bias"])
    v = np.concatenate([c(raw["user_embeds"])[np.asarray(ids, dtype=np.int64)], h], axis=1)
    if norm_embed:
        v = v / np.linalg.norm(v, axis=1, keepdims=True)
    return v
