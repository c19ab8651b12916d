"""Torch restatement of ONE AutoInt training step of the reference (TEST INFRASTRUCTURE ONLY).

Follows ``libreco/algorithms/autoint.py:146-168`` with ``is_training=True`` (the graph has no BN and no dropout)
on the RAW variables of either graph ``multi_head_attention`` (``libreco/layers/attention.py:67-125``) builds, as
``tests/_autoint_oracle.py`` restates them for inference:
* "keras" (TF >= 2.10): ``query`` / ``key`` / ``value`` [K, H, hd], ``attention_output`` [H, hd, K], no biases,
  the query scaled by 1/sqrt(hd) before the product;
* "legacy": bias-free ``query`` / ``key`` [K, D], ``value`` [D, D] applied to the PROJECTED keys and ``output``
  [D, K]; the scores scaled after the product.
then Flatten and ``tf_dense(1)`` with a bias, mean sigmoid cross entropy (``libreco/tfops/loss.py:14-18``) and
TF-Adam (``libreco/training/tf_trainer.py:112-123``) with ``reg`` on the embedding tables only and the staircase
learning-rate decay, as in ``oracle/deepfm_train.py``.  Gradients come from torch autograd.  Float64 by default;
``dtype=torch.float32`` gives the float32 restatement the CPU tests calibrate the GPU bounds with.

**PARITY UNPINNED**, like every graph in ``oracle/tf_models.py``: TensorFlow is not available, so this follows the
graph definitions line by line and is checked against the inference restatement and central differences, not
against a TensorFlow run.  Multi-sparse layouts only with the combiner "normal" (every member its own field).
"""
import numpy as np
import torch

from oracle.fm_train import B1, B2

TABLES = ("user_embeds", "item_embeds", "sparse_embeds", "dense_embeds")


def init_state(w):
    p = {k: np.array(w[k], dtype=np.float64) for k in TABLES if w.get(k) is not None}
    for l, lw in enumerate(w["autoint_mha"]):
        for n, a in lw.items():
            p[f"mha{l}_{n}"] = np.array(a, dtype=np.float64)
    p["out_kernel"] = np.array(w["out_kernel"], dtype=np.float64).reshape(-1)
    p["out_bias"] = np.array(w["out_bias"], dtype=np.float64).reshape(1)
    return dict(t=0, scheme=w["autoint_scheme"], H=int(w["num_heads"]), residual=bool(w["use_residual"]),
                n_layers=len(w["autoint_mha"]), params=p, m={k: np.zeros_like(v) for k, v in p.items()},
                v={k: np.zeros_like(v) for k, v in p.items()})


def field_block(t, users, items, sparse, dense):
    """``concat_embed`` (autoint.py:152-158) on the variables ``t``: [R, F, K], the field order of
    ``oracle.tf_models._stacked_embeds`` (user, item, sparse.., dense value x embedding..)."""
    dt = t["user_embeds"].dtype
    parts = [t["user_embeds"][torch.as_tensor(np.asarray(users))][:, None],
             t["item_embeds"][torch.as_tensor(np.asarray(items))][:, None]]
    if sparse is not None:
        parts.append(t["sparse_embeds"][torch.as_tensor(np.asarray(sparse, dtype=np.int64))])
    if dense is not None:
        parts.append(torch.as_tensor(np.asarray(dense), dtype=dt)[:, :, None] * t["dense_embeds"][None])
    return torch.cat(parts, dim=1)


def mha(x, t, l, scheme, H):
    """One ``multi_head_attention(x, x)`` on x [R, F, K]."""
    if scheme == "keras":
        wq, wk, wv, wo = (t[f"mha{l}_{n}"] for n in ("query", "key", "value", "attention_output"))
        hd = wq.shape[2]
        q = torch.einsum("rfk,khd->rfhd", x, wq) * (1.0 / np.sqrt(hd))
        k = torch.einsum("rfk,khd->rfhd", x, wk)
        v = torch.einsum("rfk,khd->rfhd", x, wv)
        p = torch.softmax(torch.einsum("rghd,rfhd->rhfg", k, q), dim=-1)
        o = torch.einsum("rhfg,rghd->rfhd", p, v)
        return torch.einsum("rfhd,hdk->rfk", o, wo)
    wq, wk, wv, wo = (t[f"mha{l}_{n}"] for n in ("query", "key", "value", "output"))
    R, F = x.shape[:2]
    D = wq.shape[1]
    hd = D // H
    queries, keys = x @ wq, x @ wk
    values = keys @ wv                                  # tf_dense(D)(keys): the PROJECTED keys (attention.py:104-106)
    split = lambda a: a.reshape(R, F, H, hd).permute(0, 2, 1, 3)       # noqa: E731
    att = (split(queries) @ split(keys).transpose(-1, -2)) * (1.0 / np.sqrt(hd))
    out = (torch.softmax(att, dim=-1) @ split(values)).permute(0, 2, 1, 3).reshape(R, F, D)
    return out @ wo


def logits(st, t, users, items, sparse, dense):
    x = field_block(t, users, items, sparse, dense)
    for l in range(st["n_layers"]):
        y = mha(x, t, l, st["scheme"], st["H"])
        x = x + y if st["residual"] else y
    return x.reshape(len(x), -1) @ t["out_kernel"] + t["out_bias"][0]


def forward_backward(st, users, items, sparse, dense, labels, dtype=torch.float64):
    """Returns (loss, logits, {variable: gradient}) of one batch, the gradients in the variables' own shapes."""
    t = {k: torch.tensor(v, dtype=dtype, requires_grad=True) for k, v in st["params"].items()}
    out = logits(st, t, users, items, sparse, dense)
    loss = torch.nn.functional.binary_cross_entropy_with_logits(out, torch.as_tensor(np.asarray(labels), dtype=dtype))
    loss.backward()
    g = {k: (v.grad.numpy() if v.grad is not None else np.zeros(v.shape)) for k, v in t.items()}
    return float(loss.detach()), out.detach().numpy(), g


def train_step(st, users, items, sparse, dense, labels, lr, eps=1e-5, reg=0.0, decay_steps=0, decay_rate=0.96):
    """One TF-Adam step; returns the data loss (the reported loss excludes the regulariser)."""
    p = st["params"]
    loss, _, g = forward_backward(st, users, items, sparse, dense, labels)
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
    return loss


def attention_core(q, k, v, H, scale):
    """The per-(row, head) core the attention kernels compute, on Q, K, V [R, F, D]: (O [R, F, D], lse [R, H, F])."""
    R, F, D = q.shape
    hd = D // H
    split = lambda a: a.reshape(R, F, H, hd).permute(0, 2, 1, 3)       # noqa: E731
    s = (split(q) @ split(k).transpose(-1, -2)) * scale                 # [R, H, F, F]
    o = (torch.softmax(s, dim=-1) @ split(v)).permute(0, 2, 1, 3).reshape(R, F, D)
    return o, torch.logsumexp(s, dim=-1)
