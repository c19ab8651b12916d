"""One RNN4Rec training step (libreco/algorithms/rnn4rec.py:151-237 in training mode, no dropout) restated in torch
float64 with autograd, from the RAW variables of either TensorFlow graph (``layers/recurrent.py:4-63``): the cell
formulas of ``_rnn4rec_oracle`` (TF1 ``GRUCell`` / ``LSTMCell`` with ``forget_bias`` 1.0 under ``dynamic_rnn``;
Keras reset-after GRU / LSTM with the sequence mask, masked steps repeating the previous output, then LayerNorm
(eps 1e-3) and tanh), the Dense head, the optional L2 normalisation, the losses of ``tfops/loss.py:4-25`` and TF-Adam
(``training/tf_trainer.py:103-124``).  ``dtype=torch.float32`` gives the float32 restatement that calibrates the
GPU bounds.  Parity with TensorFlow is unpinned (no TensorFlow exists here), and so is the Keras masked-step hazard
of DESIGN §4."""
from __future__ import annotations

import numpy as np
import torch

TABLES = ("seq_embeds", "item_embeds", "item_biases")


def init_params(raw, dtype=torch.float64):
    """{name: leaf tensor}: the tables, the head and ``rnn{i}_{raw key}`` for every raw layer variable."""
    P = {k: torch.tensor(np.asarray(raw[k], np.float64).reshape(np.shape(raw[k])), dtype=dtype) for k in
         TABLES + ("dense_kernel", "dense_bias")}
    P["item_biases"] = P["item_biases"].reshape(-1)
    P["dense_bias"] = P["dense_bias"].reshape(-1)
    for i, lw in enumerate(raw["rnn_layers"]):
        for k, v in lw.items():
            P[f"rnn{i}_{k}"] = torch.tensor(np.asarray(v, np.float64), dtype=dtype)
    return P


def _ln(x, gamma, beta, eps=1e-3):
    mean = x.mean(dim=-1, keepdim=True)
    var = ((x - mean) ** 2).mean(dim=-1, keepdim=True)
    return (x - mean) / torch.sqrt(var + eps) * gamma + beta


def rnn(P, meta, seqs, lens):
    """Encoder output [n, H_last] of ``seqs`` [n, T] / ``lens`` [n] (clamped to [0, T])."""
    seqs = torch.as_tensor(np.asarray(seqs, np.int64))
    n, T = seqs.shape
    lens = torch.as_tensor(np.clip(np.asarray(lens, np.int64), 0, T))
    X = P["seq_embeds"][seqs]
    L, rt = meta["n_layers"], meta["rnn_type"]
    one = torch.tensor(1.0, dtype=X.dtype)
    if meta["rnn_scheme"] == "legacy":
        hs = [None] * L
        cs = [None] * L
        for t in range(T):
            live = (t < lens)[:, None]
            x = X[:, t]
            for i in range(L):
                if rt == "gru":
                    ck = P[f"rnn{i}_candidate_kernel"]
                    H = ck.shape[1]
                    h = hs[i] if hs[i] is not None else torch.zeros((n, H), dtype=X.dtype)
                    v = torch.sigmoid(torch.cat([x, h], 1) @ P[f"rnn{i}_gates_kernel"] + P[f"rnn{i}_gates_bias"])
                    r, u = v[:, :H], v[:, H:]
                    cand = torch.tanh(torch.cat([x, r * h], 1) @ ck + P[f"rnn{i}_candidate_bias"])
                    nh, nc = u * h + (one - u) * cand, h
                    c = nc
                else:
                    k = P[f"rnn{i}_kernel"]
                    H = k.shape[1] // 4
                    h = hs[i] if hs[i] is not None else torch.zeros((n, H), dtype=X.dtype)
                    c = cs[i] if cs[i] is not None else torch.zeros((n, H), dtype=X.dtype)
                    m = torch.cat([x, h], 1) @ k + P[f"rnn{i}_bias"]
                    ig, j, f, o = m[:, :H], m[:, H:2 * H], m[:, 2 * H:3 * H], m[:, 3 * H:]
                    nc = c * torch.sigmoid(f + one) + torch.sigmoid(ig) * torch.tanh(j)
                    nh = torch.tanh(nc) * torch.sigmoid(o)
                hs[i] = torch.where(live, nh, h)
                cs[i] = torch.where(live, nc, c)
                x = hs[i]
        return hs[-1]
    ln = bool(meta["use_layer_norm"])
    act = (lambda v: v) if ln else torch.tanh
    mask = torch.arange(T)[None, :] < lens[:, None]
    seq = X
    for i in range(L):
        U = P[f"rnn{i}_recurrent_kernel"]
        H = U.shape[0]
        h = torch.zeros((n, H), dtype=X.dtype)
        cc = torch.zeros_like(h)
        out = torch.zeros_like(h)
        outs = []
        for t in range(T):
            x = seq[:, t]
            if rt == "gru":
                b = P[f"rnn{i}_bias"]
                mx = x @ P[f"rnn{i}_kernel"] + b[0]
                mi = h @ U + b[1]
                z = torch.sigmoid(mx[:, :H] + mi[:, :H])
                r = torch.sigmoid(mx[:, H:2 * H] + mi[:, H:2 * H])
                hh = act(mx[:, 2 * H:] + r * mi[:, 2 * H:])
                nh, nc = z * h + (one - z) * hh, cc
            else:
                m = x @ P[f"rnn{i}_kernel"] + h @ U + P[f"rnn{i}_bias"]
                ig, f, g, o = (torch.sigmoid(m[:, :H]), torch.sigmoid(m[:, H:2 * H]), m[:, 2 * H:3 * H],
                               torch.sigmoid(m[:, 3 * H:]))
                nc = f * cc + ig * act(g)
                nh = o * act(nc)
            live = mask[:, t][:, None]
            h = torch.where(live, nh, h)
            cc = torch.where(live, nc, cc)
            out = torch.where(live, nh, out)
            outs.append(out)
        seq = torch.stack(outs, 1)
        if ln:
            seq = torch.tanh(_ln(seq, P[f"rnn{i}_gamma"], P[f"rnn{i}_beta"]))
    return seq[:, -1]


def meta_of(raw):
    return dict(rnn_scheme=raw["rnn_scheme"], rnn_type=raw["rnn_type"], n_layers=len(raw["rnn_layers"]),
                use_layer_norm=bool(raw.get("use_layer_norm", False)) and raw["rnn_scheme"] == "keras")


def _l2n(x):
    return x / torch.linalg.norm(x, dim=1, keepdim=True)


def user_vectors(P, meta, seqs, lens):
    return rnn(P, meta, seqs, lens) @ P["dense_kernel"] + P["dense_bias"]


def loss(P, meta, seqs, lens, items, labels_or_neg, loss_type="cross_entropy", norm_embed=False):
    """The data loss of one batch (a scalar tensor)."""
    u = user_vectors(P, meta, seqs, lens)
    items = torch.as_tensor(np.asarray(items, np.int64))
    if loss_type == "bpr":
        neg = torch.as_tensor(np.asarray(labels_or_neg, np.int64))
        ip, in_ = P["item_embeds"][items], P["item_embeds"][neg]
        if norm_embed:             # rnn4rec.py:189-195: the items are normalised, the user vector is not
            ip, in_ = _l2n(ip), _l2n(in_)
        diff = (P["item_biases"][items] - P["item_biases"][neg]) + (u * (ip - in_)).sum(1)
        return -torch.nn.functional.logsigmoid(diff).mean()
    i = P["item_embeds"][items]
    if norm_embed:
        u, i = _l2n(u), _l2n(i)
    logit = (u * i).sum(1) + P["item_biases"][items]
    y = torch.as_tensor(np.asarray(labels_or_neg, np.float64), dtype=logit.dtype)
    if loss_type == "cross_entropy":
        return torch.nn.functional.binary_cross_entropy_with_logits(logit, y)
    p = torch.sigmoid(logit)          # focal, alpha 0.25, gamma 2 (tfops/loss.py:52-58)
    ce = torch.nn.functional.binary_cross_entropy_with_logits(logit, y, reduction="none")
    pt = y * p + (1 - y) * (1 - p)
    at = y * 0.25 + (1 - y) * 0.75
    return (at * (1 - pt) ** 2 * ce).mean()


def forward_backward(P, meta, seqs, lens, items, labels_or_neg, loss_type="cross_entropy", norm_embed=False):
    """(loss float, {name: gradient ndarray}) of one batch."""
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in P.items()}
    val = loss(leaves, meta, seqs, lens, items, labels_or_neg, loss_type, norm_embed)
    grads = torch.autograd.grad(val, list(leaves.values()), allow_unused=True)
    return float(val.detach()), {k: (g if g is not None else torch.zeros_like(v)).detach().numpy()
                        for (k, v), g in zip(leaves.items(), grads)}


def init_state(raw, dtype=torch.float64):
    P = init_params(raw, dtype)
    return dict(P=P, m={k: torch.zeros_like(v) for k, v in P.items()}, v={k: torch.zeros_like(v) for k, v in P.items()},
                t=0)


def train_step(st, meta, seqs, lens, items, labels_or_neg, lr, eps, loss_type="cross_entropy", norm_embed=False,
               reg=0.0):
    """One TF-Adam step in place; returns the data loss.  ``reg`` adds reg * sum w^2 over the three tables."""
    val, g = forward_backward(st["P"], meta, seqs, lens, items, labels_or_neg, loss_type, norm_embed)
    st["t"] += 1
    t = st["t"]
    lr_t = lr * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
    for k, p in st["P"].items():
        gk = torch.as_tensor(g[k], dtype=p.dtype)
        if reg and k in TABLES:
            gk = gk + 2 * reg * p
        st["m"][k] = 0.9 * st["m"][k] + 0.1 * gk
        st["v"][k] = 0.999 * st["v"][k] + 0.001 * gk * gk
        st["P"][k] = p - lr_t * st["m"][k] / (torch.sqrt(st["v"][k]) + eps)
    return val


def raw_of(P, raw):
    """The raw variable dict of ``raw``'s graph with the values of P."""
    out = {k: v for k, v in raw.items() if k not in TABLES + ("dense_kernel", "dense_bias", "rnn_layers")}
    for k in TABLES + ("dense_kernel", "dense_bias"):
        out[k] = P[k].detach().numpy()
    out["rnn_layers"] = [{k: P[f"rnn{i}_{k}"].detach().numpy() for k in lw} for i, lw in enumerate(raw["rnn_layers"])]
    return out
