"""One Caser / WaveNet training step (libreco/algorithms/caser.py:135-221, wave_net.py:139-222 in training mode)
restated in torch float64 with autograd from the RAW variables (``synthetic.make_caser_weights`` /
``make_wavenet_weights``): the encoders of ``_conv_encoder_oracle``, the Dense head, ``[user row | head]``, the optional
L2 normalisation of the user and item rows, the losses of ``tfops/loss.py:4-25`` (cross entropy, focal) and TF-Adam
(``training/tf_trainer.py:103-124``) with the L2 ``reg`` of the three regularised tables.  ``dtype=torch.float32``
gives the float32 restatement that calibrates the GPU bounds.

Every max-pool routes its gradient explicitly through the FIRST index reaching the maximum (a gather from that
index): ``torch.amax`` splits tied gradients evenly and the tie order of ``torch.max`` is not a documented contract.
ReLU before a max is monotone, so the pooled value is relu(pre[first argmax of pre]).  The parameters are named as
the trainer's variables (``conv{i}_kernel``, ``vertical_*`` / ``out_conv_*``)."""
from __future__ import annotations

import numpy as np
import torch

TABLES = ("user_embeds", "seq_embeds", "item_embeds", "item_biases")
REG_VARS = ("user_embeds", "seq_embeds", "item_embeds")


def last_layer(raw):
    return "vertical" if "vertical" in raw else "out_conv"


def init_params(raw, dtype=torch.float64):
    """{name: tensor}: the tables, the head and every convolution variable in its TF shape."""
    t = lambda a: torch.tensor(np.asarray(a, np.float64), dtype=dtype)      # noqa: E731
    P = {k: t(raw[k]) for k in TABLES + ("dense_kernel", "dense_bias")}
    P["item_biases"] = P["item_biases"].reshape(-1)
    P["dense_bias"] = P["dense_bias"].reshape(-1)
    for i, c in enumerate(raw["convs"]):
        P[f"conv{i}_kernel"], P[f"conv{i}_bias"] = t(c["kernel"]), t(c["bias"])
    last = last_layer(raw)
    P[f"{last}_kernel"], P[f"{last}_bias"] = t(raw[last]["kernel"]), t(raw[last]["bias"])
    return P


def meta_of(raw):
    return dict(model="Caser" if "vertical" in raw else "WaveNet", n_conv=len(raw["convs"]),
                dilations=[int(d) for d in raw.get("dilations", [])])


def first_argmax(v, dim):
    """The lowest index reaching the maximum of v along dim."""
    m = v.max(dim=dim, keepdim=True).values
    shape = [1] * v.dim()
    shape[dim] = v.shape[dim]
    idx = torch.arange(v.shape[dim]).reshape(shape).expand_as(v)
    return torch.where(v == m, idx, torch.full_like(idx, v.shape[dim])).min(dim=dim).values


def _pool(pre, keep, pick):
    """relu(max over positions (dim 1)) with the gradient routed to the first argmax; ``keep`` collects (pre,
    argmax).  ``pick`` [n, columns] overrides a column's position where >= 0, and zeroes the column where -2."""
    a = first_argmax(pre.detach(), 1)
    if keep is not None:
        keep.append((pre, a))
    if pick is not None:
        pick = torch.as_tensor(np.asarray(pick, np.int64))
        a = torch.where(pick >= 0, pick, a)
    out = torch.relu(pre.gather(1, a.unsqueeze(1)).squeeze(1))
    return out if pick is None else torch.where(pick == -2, torch.zeros_like(out), out)


def features(P, meta, seqs, X=None, keep=None, pick=None):
    """Pre-head features [n, D] of the rows ``seqs`` [n, T]; ``X`` [n, T, K] replaces the gathered input rows.
    ``pick`` [n, pooled columns] (see ``_pool``) lets a test follow the device's choice on near-tied columns."""
    seqs = torch.as_tensor(np.asarray(seqs, np.int64))
    if X is None:
        X = P["seq_embeds"][seqs]
    n, T, K = X.shape
    if meta["model"] == "Caser":
        outs = []
        for i in range(meta["n_conv"]):
            h = i + 1
            W = P[f"conv{i}_kernel"].reshape(h * K, -1)
            win = torch.stack([X[:, p:p + h].reshape(n, h * K) for p in range(T - h + 1)], dim=1)   # [n, T-h+1, hK]
            nh = W.shape[1]
            cols = None if pick is None else pick[:, i * nh:(i + 1) * nh]
            outs.append(_pool(win @ W + P[f"conv{i}_bias"], keep, cols))
        v = torch.relu(torch.einsum("ntk,tf->nkf", X, P["vertical_kernel"][0]) + P["vertical_bias"])
        outs.append(v.reshape(n, -1))
        return torch.cat(outs, dim=1)
    x = X
    for i, d in enumerate(meta["dilations"]):
        W = P[f"conv{i}_kernel"]
        prev = torch.zeros_like(x)
        if d < T:
            prev = torch.cat([torch.zeros_like(x[:, :d]), x[:, :-d]], dim=1)
        x = torch.relu(prev @ W[0] + x @ W[1] + P[f"conv{i}_bias"])
    return _pool(x @ P["out_conv_kernel"][0] + P["out_conv_bias"], keep, pick)


def pool_argmax(P, meta, seqs):
    """(argmax [n, columns] with -1 where the max is <= 0, gap [n, columns]) of every max-pooled column (Caser: the
    T*nh horizontal columns, WaveNet: the F columns of the 1x1 layer).  The gap is the maximum minus the largest value
    not bitwise equal to it (inf when every position ties)."""
    keep = []
    with torch.no_grad():
        features(P, meta, seqs, keep=keep)
    args, gaps = [], []
    for pre, a in keep:
        m = pre.max(dim=1).values
        other = torch.where(pre == m[:, None], torch.full_like(pre, -np.inf), pre).max(dim=1).values
        args.append(torch.where(m > 0, a, torch.full_like(a, -1)))
        gaps.append(m - other)
    return torch.cat(args, dim=1).numpy(), torch.cat(gaps, dim=1).numpy()


def _l2n(x):
    return x / torch.linalg.norm(x, dim=1, keepdim=True)


def near_tie_pick(P, meta, seqs, device_arg, gap_limit):
    """The ``pick`` that follows ``device_arg`` (the saved argmax of the device, -1 where its max is <= 0) on every
    column whose float64 maximum lies within ``gap_limit`` of its runner-up or of 0, where float32 may legitimately
    choose otherwise; -1 (the oracle's own choice) elsewhere."""
    keep = []
    with torch.no_grad():
        features(P, meta, seqs, keep=keep)
    m = torch.cat([pre.max(dim=1).values for pre, _ in keep], dim=1).numpy()
    _, gap = pool_argmax(P, meta, seqs)
    near = (gap <= gap_limit) | (np.abs(m) <= gap_limit)
    dev = np.asarray(device_arg, np.int64)
    return np.where(near, np.where(dev >= 0, dev, -2), -1)


def user_vectors(P, meta, users, seqs, X=None, pick=None):
    """``[user_embeds[users] | head(features)]`` [n, 2K] before any normalisation."""
    f = features(P, meta, seqs, X, pick=pick)
    h = f @ P["dense_kernel"] + P["dense_bias"]
    if meta["model"] == "Caser":
        h = torch.relu(h)
    return torch.cat([P["user_embeds"][torch.as_tensor(np.asarray(users, np.int64))], h], dim=1)


def loss(P, meta, users, items, seqs, labels, loss_type="cross_entropy", norm_embed=False, pick=None):
    """The data loss of one batch (a scalar tensor)."""
    u = user_vectors(P, meta, users, seqs, pick=pick)
    i = P["item_embeds"][torch.as_tensor(np.asarray(items, np.int64))]
    if norm_embed:
        u, i = _l2n(u), _l2n(i)
    logit = (u * i).sum(1) + P["item_biases"][torch.as_tensor(np.asarray(items, np.int64))]
    y = torch.as_tensor(np.asarray(labels, np.float64), dtype=logit.dtype)
    if loss_type == "cross_entropy":
        return torch.nn.functional.binary_cross_entropy_with_logits(logit, y)
    p = torch.sigmoid(logit)          # focal, alpha 0.25, gamma 2 (tfops/loss.py:52-62)
    ce = torch.nn.functional.binary_cross_entropy_with_logits(logit, y, reduction="none")
    pt = y * p + (1 - y) * (1 - p)
    at = y * 0.25 + (1 - y) * 0.75
    return (at * (1 - pt) ** 2 * ce).mean()


def forward_backward(P, meta, users, items, seqs, labels, loss_type="cross_entropy", norm_embed=False, pick=None):
    """(loss float, {name: gradient ndarray}) of one batch."""
    leaves = {k: v.detach().clone().requires_grad_(True) for k, v in P.items()}
    val = loss(leaves, meta, users, items, seqs, labels, loss_type, norm_embed, pick)
    grads = torch.autograd.grad(val, list(leaves.values()), allow_unused=True)
    return float(val.detach()), {k: (g if g is not None else torch.zeros_like(v)).detach().numpy()
                                 for (k, v), g in zip(leaves.items(), grads)}


def init_state(raw, dtype=torch.float64):
    P = init_params(raw, dtype)
    return dict(P=P, m={k: torch.zeros_like(v) for k, v in P.items()}, v={k: torch.zeros_like(v) for k, v in P.items()},
                t=0)


def train_step(st, meta, users, items, seqs, labels, lr, eps, loss_type="cross_entropy", norm_embed=False, reg=0.0,
               pick=None):
    """One TF-Adam step in place; returns the data loss.  ``reg`` adds reg * sum w^2 over the three tables."""
    val, g = forward_backward(st["P"], meta, users, items, seqs, labels, loss_type, norm_embed, pick)
    st["t"] += 1
    t = st["t"]
    lr_t = lr * np.sqrt(1 - 0.999 ** t) / (1 - 0.9 ** t)
    for k, p in st["P"].items():
        gk = torch.as_tensor(g[k], dtype=p.dtype)
        if reg and k in REG_VARS:
            gk = gk + 2 * reg * p
        st["m"][k] = 0.9 * st["m"][k] + 0.1 * gk
        st["v"][k] = 0.999 * st["v"][k] + 0.001 * gk * gk
        st["P"][k] = p - lr_t * st["m"][k] / (torch.sqrt(st["v"][k]) + eps)
    return val


def raw_of(P, raw):
    """The raw variable dict of ``raw``'s graph with the values of P."""
    out = {k: v for k, v in raw.items() if k not in TABLES + ("dense_kernel", "dense_bias", "convs", last_layer(raw))}
    for k in TABLES + ("dense_kernel", "dense_bias"):
        out[k] = P[k].detach().numpy()
    out["convs"] = [dict(kernel=P[f"conv{i}_kernel"].detach().numpy(), bias=P[f"conv{i}_bias"].detach().numpy())
                    for i in range(len(raw["convs"]))]
    last = last_layer(raw)
    out[last] = dict(kernel=P[f"{last}_kernel"].detach().numpy(), bias=P[f"{last}_bias"].detach().numpy())
    return out
