"""Torch restatement of ONE Transformer training step of the reference (TEST INFRASTRUCTURE ONLY).

Follows ``libreco/algorithms/transformer.py:203-339`` with ``is_training=True`` and no dropout, on the RAW variables
of either graph ``multi_head_attention`` (``libreco/layers/attention.py:67-138``) builds, as
``tests/_transformer_oracle.py`` restates them for inference:
* the item feature table G of ``combine_seq_features`` in concat mode, rebuilt from the tables;
* X = [G[seq_t] || pos_t] with the trainable positional table or the constant sinusoidal one;
* per layer ``a = x + mha(rms_att(x))``, ``x = a + gelu(rms_ffn(a) W1) W2`` (``layers/transformer.py``, erf gelu,
  ``rms_norm`` of ``layers/normalization.py:21-29``), then ``rms_last``;
* the mask ``t < len`` OR-ed with the causal mask; "keras" adds -1e9 to a hidden score, "legacy" writes -1e9
  (``tf.where``) and applies its value Dense to the PROJECTED keys;
* the target attention (``tf_attention``, ``layers/attention.py:5-25``) of ``[rms_item(G[item]) || 1..1]`` over the
  encoded sequence, hidden keys - 1e9;
* ``dense_nn`` with swish and BN on batch statistics (``layers/dense.py:12-49``), Dense(1), mean sigmoid cross
  entropy (``libreco/tfops/loss.py:14-18``), TF-Adam (``libreco/training/tf_trainer.py:103-124``) with the BN
  moving-statistics update, ``reg`` on the embedding tables only and the staircase learning-rate decay.
``lens`` is clamped to [1, T] as the training collator gives it.  Gradients come from torch autograd.  Float64 by
default; ``dtype=torch.float32`` gives the float32 restatement the CPU tests calibrate the GPU bounds with.

**PARITY UNPINNED**, like every graph in ``oracle/tf_models.py``: TensorFlow is not available, so this follows the
graph definitions line by line and is checked against the inference restatement and central differences, not
against a TensorFlow run.
"""
import os
import sys

import numpy as np
import torch

from oracle.fm_train import B1, B2, BN_EPS, BN_MOMENTUM

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _transformer_oracle as to  # noqa: E402

TABLES = ("user_embeds", "item_embeds", "sparse_embeds", "dense_embeds")
NEG = 1.0e9


def att_names(scheme):
    return ("query", "key", "value", "attention_output") if scheme == "keras" else ("query", "key", "value", "output")


def init_state(w, use_bn):
    p = {k: np.array(w[k], dtype=np.float64) for k in TABLES if w.get(k) is not None}
    mlp = w["mlp"]
    n = len(mlp["kernels"])
    st = dict(use_bn=bool(use_bn), t=0, moving={}, n_layers=n, scheme=w["tfm_scheme"], H=int(w["num_heads"]),
              causal=bool(w.get("use_causal_mask", False)), n_tfm=len(w["tfm_layers"]))
    for i in range(n):
        p[f"W{i}"] = np.array(mlp["kernels"][i], dtype=np.float64)
        p[f"b{i}"] = np.array(mlp["biases"][i], dtype=np.float64)
    if use_bn:
        for j, bn in enumerate([mlp.get("bn_in")] + list(mlp.get("bns") or [])):
            p[f"bn{j}_gamma"] = np.array(bn["gamma"], dtype=np.float64)
            p[f"bn{j}_beta"] = np.array(bn["beta"], dtype=np.float64)
            st["moving"][f"bn{j}"] = [np.array(bn["mean"], dtype=np.float64), np.array(bn["var"], dtype=np.float64)]
    p["out_kernel"] = np.array(w["out_kernel"], dtype=np.float64).reshape(-1)
    p["out_bias"] = np.array(w["out_bias"], dtype=np.float64).reshape(1)
    for l, lw in enumerate(w["tfm_layers"]):
        for k in att_names(st["scheme"]) + ("rms_att", "rms_ffn", "ffn1", "ffn2"):
            p[f"tfm{l}_{k}"] = np.array(lw[k], dtype=np.float64)
    p["rms_last"] = np.array(w["rms_last"], dtype=np.float64).reshape(-1)
    p["rms_item"] = np.array(w["rms_item"], dtype=np.float64).reshape(-1)
    if w.get("positional_encoding") is not None:
        p["positional_encoding"] = np.array(w["positional_encoding"], dtype=np.float64)
    st["params"] = p
    st["m"] = {k: np.zeros_like(v) for k, v in p.items()}
    st["v"] = {k: np.zeros_like(v) for k, v in p.items()}
    return st


def rms(x, scale):
    return x * torch.rsqrt(x.square().mean(-1, keepdim=True) + 1e-8) * scale


def gelu(x):
    return 0.5 * x * (1.0 + torch.erf(x / np.sqrt(2.0)))


def item_table(t, spec):
    parts = [t["item_embeds"]]
    n_rows = t["item_embeds"].shape[0]
    if spec.get("item_sparse_unique") is not None and len(spec["item_sparse_col_index"]):
        idx = torch.as_tensor(np.asarray(spec["item_sparse_unique"], dtype=np.int64))
        parts.append(t["sparse_embeds"][idx].reshape(n_rows, -1))
    if spec.get("item_dense_unique") is not None and len(spec["item_dense_col_index"]):
        vals = torch.as_tensor(np.asarray(spec["item_dense_unique"]), dtype=t["item_embeds"].dtype)
        parts.append((vals[:, :, None] * t["dense_embeds"][list(spec["item_dense_col_index"])][None]).reshape(n_rows, -1))
    return torch.cat(parts, dim=1)


def attention_mask(lens, T, causal):
    """[R, Tq, Tk] bool: key k visible to query q when k < len, OR k <= q with the causal mask."""
    m = torch.arange(T)[None, None, :] < torch.as_tensor(np.asarray(lens)).reshape(-1, 1, 1)
    m = m.expand(len(lens), T, T)
    if causal:
        m = m | torch.tril(torch.ones(T, T, dtype=torch.bool))[None]
    return m


def masked(s, mask, scheme):
    """keras: hidden score + (-1e9) (formed in float32, i.e. rounded: exp gives exactly 0 either way); legacy: -1e9."""
    if scheme == "keras":
        return torch.where(mask, s, s - NEG)
    return torch.where(mask, s, torch.full_like(s, -NEG))


def mha(x, t, l, scheme, H, mask):
    """One ``multi_head_attention`` on x [R, T, D]."""
    R, T, D = x.shape
    hd = D // H
    if scheme == "keras":
        wq, wk, wv, wo = (t[f"tfm{l}_{n}"] for n in att_names(scheme))
        q = torch.einsum("rtd,dhk->rthk", x, wq) * (1.0 / np.sqrt(hd))
        k = torch.einsum("rtd,dhk->rthk", x, wk)
        v = torch.einsum("rtd,dhk->rthk", x, wv)
        s = masked(torch.einsum("rshk,rqhk->rhqs", k, q), mask[:, None], scheme)
        o = torch.einsum("rhqs,rshk->rqhk", torch.softmax(s, dim=-1), v)
        return torch.einsum("rqhk,hkd->rqd", o, wo)
    wq, wk, wv, wo = (t[f"tfm{l}_{n}"] for n in att_names(scheme))
    queries, keys = x @ wq, x @ wk
    values = keys @ wv                                   # tf_dense(D)(keys): the PROJECTED keys
    split = lambda a: a.reshape(R, T, H, hd).permute(0, 2, 1, 3)       # noqa: E731
    s = masked((split(queries) @ split(keys).transpose(-1, -2)) * (1.0 / np.sqrt(hd)), mask[:, None], scheme)
    out = (torch.softmax(s, dim=-1) @ split(values)).permute(0, 2, 1, 3).reshape(R, T, D)
    return out @ wo


def sinusoidal(T, K, dtype):
    """positional_encoding (layers/transformer.py:113-144): a constant, not a variable."""
    return torch.as_tensor(to.sinusoidal(T, K), dtype=dtype)


def logits(st, t, spec, users, items, seqs, lens, sparse, dense, bn_frozen=False, stats=None):
    """Training-mode logits (batch statistics in the BN, recorded into ``stats``); ``bn_frozen``: the moving
    statistics instead (the inference graph)."""
    dt = t["item_embeds"].dtype
    seqs = np.asarray(seqs)
    R, T = seqs.shape
    lens = np.clip(np.asarray(lens), 1, T)
    G = item_table(t, spec)
    K = t["user_embeds"].shape[1]
    pos = t["positional_encoding"] if "positional_encoding" in t else sinusoidal(T, K, dt)
    x = torch.cat([G[torch.as_tensor(seqs.astype(np.int64))], pos[None].expand(R, T, K)], dim=2)
    mask = attention_mask(lens, T, st["causal"])
    for l in range(st["n_tfm"]):
        a = x + mha(rms(x, t[f"tfm{l}_rms_att"]), t, l, st["scheme"], st["H"], mask)
        x = a + gelu(rms(a, t[f"tfm{l}_rms_ffn"]) @ t[f"tfm{l}_ffn1"]) @ t[f"tfm{l}_ffn2"]
    S = rms(x, t["rms_last"])
    qi = rms(G[torch.as_tensor(np.asarray(items))], t["rms_item"])
    q = torch.cat([qi, torch.ones((R, K), dtype=dt)], dim=1)
    sc = torch.einsum("rd,rtd->rt", q, S)
    tmask = torch.arange(T)[None, :] < torch.as_tensor(lens).reshape(-1, 1)
    p_att = torch.softmax(torch.where(tmask, sc, sc - NEG), dim=1)
    s_u = (p_att[:, :, None] * S).sum(1)
    xs = [t["user_embeds"][torch.as_tensor(np.asarray(users))], t["item_embeds"][torch.as_tensor(np.asarray(items))]]
    if sparse is not None:
        xs.append(t["sparse_embeds"][torch.as_tensor(np.asarray(sparse, dtype=np.int64))].reshape(R, -1))
    if dense is not None:
        xs.append((torch.as_tensor(np.asarray(dense), dtype=dt)[:, :, None] * t["dense_embeds"][None]).reshape(R, -1))
    xs.append(s_u)
    act = torch.cat(xs, dim=1)

    def bn(z, j):
        if bn_frozen:
            mu, var = (torch.as_tensor(a, dtype=dt) for a in st["moving"][f"bn{j}"])
        else:
            mu, var = z.mean(0), z.var(0, unbiased=False)
            if stats is not None:
                stats[f"bn{j}"] = (mu.detach().numpy().astype(np.float64), var.detach().numpy().astype(np.float64))
        return (z - mu) / torch.sqrt(var + BN_EPS) * t[f"bn{j}_gamma"] + t[f"bn{j}_beta"]

    if st["use_bn"]:
        act = bn(act, 0)
    n = st["n_layers"]
    for i in range(n):
        act = act @ t[f"W{i}"] + t[f"b{i}"]
        if i != n - 1:
            act = act * torch.sigmoid(act)
            if st["use_bn"]:
                act = bn(act, i + 1)
    return act @ t["out_kernel"] + t["out_bias"][0]


def forward_backward(st, spec, users, items, seqs, lens, sparse, dense, labels, dtype=torch.float64):
    """Returns (loss, logits, {variable: gradient}, batch BN statistics) of one batch."""
    t = {k: torch.tensor(v, dtype=dtype, requires_grad=True) for k, v in st["params"].items()}
    stats = {}
    out = logits(st, t, spec, users, items, seqs, lens, sparse, dense, stats=stats)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(out, torch.as_tensor(np.asarray(labels), dtype=dtype))
    loss.backward()
    g = {k: (v.grad.numpy().astype(np.float64) if v.grad is not None else np.zeros(v.shape)) for k, v in t.items()}
    return float(loss.detach()), out.detach().numpy().astype(np.float64), g, stats


def train_step(st, spec, users, items, seqs, lens, sparse, dense, labels, lr, eps=1e-5, reg=0.0, decay_steps=0,
               decay_rate=0.96):
    """One TF-Adam step with the BN moving-statistics update; returns the data loss (the regulariser excluded)."""
    p = st["params"]
    loss, _, g, stats = forward_backward(st, spec, users, items, seqs, lens, sparse, dense, labels)
    if reg:
        for k in TABLES:
            if k in p:
                g[k] = g[k] + 2.0 * reg * p[k]
    if decay_steps:
        lr = lr * decay_rate ** (st["t"] // decay_steps)          # global_step = completed steps
    st["t"] += 1
    t = st["t"]
    lr_t = lr * np.sqrt(1 - B2 ** t) / (1 - B1 ** t)
    for k in p:
        st["m"][k] = B1 * st["m"][k] + (1 - B1) * g[k]
        st["v"][k] = B2 * st["v"][k] + (1 - B2) * np.square(g[k])
        p[k] -= lr_t * st["m"][k] / (np.sqrt(st["v"][k]) + eps)
    for name, (mu, var) in stats.items():
        mm, mv = st["moving"][name]
        st["moving"][name] = [BN_MOMENTUM * mm + (1 - BN_MOMENTUM) * mu, BN_MOMENTUM * mv + (1 - BN_MOMENTUM) * var]
    return loss


def raw_weights(st, w):
    """The raw weight dict of ``w`` with the oracle's current variables and BN moving statistics."""
    p = st["params"]
    out = dict(w)
    for k in TABLES:
        if k in p:
            out[k] = p[k].astype(np.float32)
    out["tfm_layers"] = [{k: p[f"tfm{l}_{k}"].astype(np.float32) for k in lw} for l, lw in enumerate(w["tfm_layers"])]
    for k in ("rms_last", "rms_item", "positional_encoding"):
        if k in p:
            out[k] = p[k].astype(np.float32)
    n = st["n_layers"]
    mlp = dict(kernels=[p[f"W{i}"].astype(np.float32) for i in range(n)],
               biases=[p[f"b{i}"].astype(np.float32) for i in range(n)])
    if st["use_bn"]:
        def bn(j):
            mm, mv = st["moving"][f"bn{j}"]
            return dict(gamma=p[f"bn{j}_gamma"].astype(np.float32), beta=p[f"bn{j}_beta"].astype(np.float32),
                        mean=mm.astype(np.float32), var=mv.astype(np.float32))
        mlp["bn_in"] = bn(0)
        mlp["bns"] = [bn(i + 1) for i in range(n - 1)]
    out["mlp"] = mlp
    out["out_kernel"] = p["out_kernel"].astype(np.float32).reshape(-1, 1)
    out["out_bias"] = p["out_bias"].astype(np.float32).reshape(1)
    return out


def attention_core(q, k, v, lens, H, scale, causal):
    """The masked per-(row, head) core the attention kernels compute, on Q, K, V [R, T, D]: (O [R, T, D],
    lse [R, H, T]); hidden keys get probability exactly 0."""
    R, T, D = q.shape
    hd = D // H
    split = lambda a: a.reshape(R, T, H, hd).permute(0, 2, 1, 3)       # noqa: E731
    s = (split(q) @ split(k).transpose(-1, -2)) * scale                 # [R, H, T, T]
    mask = attention_mask(np.clip(np.asarray(lens), 1, T), T, causal)[:, None]
    s = torch.where(mask, s, torch.full_like(s, -np.inf))
    o = (torch.softmax(s, dim=-1) @ split(v)).permute(0, 2, 1, 3).reshape(R, T, D)
    return o, torch.logsumexp(s, dim=-1)
