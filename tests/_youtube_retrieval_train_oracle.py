"""Host restatements for YouTubeRetrieval training (TEST INFRASTRUCTURE ONLY).

1. ``unique_candidates`` restates the device candidate sampler (``b200_unique_candidates``,
   ``librecommender_b200/csrc/sampler.cu``): draw j = Philox4x32-10(seed, step, j) (``oracle.sampling``), uniform
   (the bounded 64-bit draw) or log-uniform (``(int64)exp(u log1p(n)) - 1``, then ``% n``), and TensorFlow's unique
   rejection: keep first occurrences until S distinct ids, ``num_tries`` = draws taken.
2. ``expected_counts`` restates TensorFlow's ``ExpectedCountHelper`` (``range_sampler.cc``), in float32 (what the
   kernel computes) or float64.
3. ``forward_backward`` / ``train_step``: one training step of ``libreco/algorithms/youtube_retrieval.py:169-260``
   (``dense_nn`` in training mode) with ``YoutubeRetrievalTrainer._build_train_ops``
   (``libreco/training/tf_trainer.py:162-245``) in torch float64 with autograd: TensorFlow's
   ``_compute_sampled_logits`` (true logit ``<u, w_label> + b_label - log E``, sampled logits ``U W_s^T + b_s -
   log E``, ``-FLT_MAX`` added where a sampled id equals the row's label), ``sampled_softmax_loss`` (softmax CE with
   the label in column 0) or ``nce_loss`` (sum of sigmoid CE over the 1 + S columns), mean over the batch, ``reg``
   on the five tables, the staircase learning-rate decay and TF-Adam.  The sampled ids and ``num_tries`` are inputs.

**PARITY UNPINNED**, like ``oracle/two_tower_train.py``: TensorFlow is not available, so its sampler, expected
counts and sampled logits are restated from its documented behaviour, not checked against a TensorFlow run.  The
TensorFlow random stream itself cannot be reproduced; parity is defined given the sampled ids and ``num_tries``.
"""
import numpy as np
import torch

from oracle.fm_train import B1, B2, BN_EPS, BN_MOMENTUM
from oracle.sampling import philox4x32_10

TABLES = ("seq_embeds", "item_embeds", "item_biases", "sparse_embeds", "dense_embeds")
FLT_MAX = float(np.finfo(np.float32).max)
TAG = 0xCA7D                     # Philox counter word 2 of the candidate draws


def draws(kind, n_items, seed, step, j):
    """(ids, ambiguous) of the draws with indices ``j``; ``ambiguous`` flags log-uniform draws whose exp lies within
    4 ulp of an integer (device and host exp may truncate differently there)."""
    j = np.asarray(j, dtype=np.uint64)
    k0 = seed & 0xFFFFFFFF
    k1 = ((seed >> 32) ^ (step >> 32)) & 0xFFFFFFFF
    r0, r1, r2, r3 = philox4x32_10(j.astype(np.uint32), np.zeros_like(j, dtype=np.uint32), TAG, step & 0xFFFFFFFF,
                                   k0, k1)
    r0, r1, r2, r3 = (x.astype(np.uint64) for x in (r0, r1, r2, r3))
    n = np.uint64(n_items)
    if kind == 0:               # high 64 bits of (r0:r1) * n, exact in two 64-bit halves (n < 2^31)
        ids = (r0 * n + ((r1 * n) >> np.uint64(32))) >> np.uint64(32)
        return ids.astype(np.int64), np.zeros(len(j), dtype=bool)
    u = (((r2 << np.uint64(32)) | r3) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    e = np.exp(u * np.log1p(float(n_items)))
    ids = (e.astype(np.int64) - 1) % n_items
    amb = np.abs(e - np.round(e)) <= 4 * np.spacing(e)
    return ids, amb


def unique_candidates(kind, n_items, S, seed, step):
    """(ids [S] in draw order, num_tries, ambiguous draws among the first num_tries) of the sequential process."""
    n = max(2 * S, 1024)
    while True:
        ids, amb = draws(kind, n_items, seed, step, np.arange(n))
        uniq, first = np.unique(ids, return_index=True)
        if len(uniq) >= S:
            first = np.sort(first)[:S]
            tries = int(first[-1]) + 1
            return ids[first], tries, int(amb[:tries].sum())
        n *= 4


def probabilities(kind, ids, n_items, dtype=np.float64):
    ids = np.asarray(ids, dtype=np.float64)
    if kind == 0:
        p = np.full(ids.shape, 1.0 / n_items)
    else:
        p = np.log((ids + 2.0) / (ids + 1.0)) / np.log1p(float(n_items))
    return p.astype(dtype)


def expected_counts(kind, ids, n_items, S, num_tries, dtype=np.float64):
    """ExpectedCountHelper: p S when num_tries == S, else -expm1(num_tries log1p(-p)), in ``dtype``."""
    p = probabilities(kind, ids, n_items, dtype)
    if num_tries == S:
        return p * dtype(S)
    return -np.expm1(dtype(num_tries) * np.log1p(-p))


# ---- one training step ------------------------------------------------------------------------------------
def init_state(w, use_bn):
    p = {k: np.array(w[k], dtype=np.float64) for k in TABLES if w.get(k) is not None}
    p["item_biases"] = p["item_biases"].reshape(-1)
    mlp = w["mlp"]
    n = len(mlp["kernels"])
    st = dict(use_bn=bool(use_bn), t=0, moving={}, n_layers=n)
    for i in range(n):
        p[f"W{i}"] = np.array(mlp["kernels"][i], dtype=np.float64)
        p[f"b{i}"] = np.array(mlp["biases"][i], dtype=np.float64)
    if use_bn:
        for j, bn in enumerate([mlp.get("bn_in")] + list(mlp.get("bns") or [])):
            p[f"bn{j}_gamma"] = np.array(bn["gamma"], dtype=np.float64)
            p[f"bn{j}_beta"] = np.array(bn["beta"], dtype=np.float64)
            st["moving"][f"bn{j}"] = [np.array(bn["mean"], dtype=np.float64), np.array(bn["var"], dtype=np.float64)]
    st["params"] = p
    st["m"] = {k: np.zeros_like(v) for k, v in p.items()}
    st["v"] = {k: np.zeros_like(v) for k, v in p.items()}
    return st


def _l2(x):
    return x * torch.rsqrt(torch.clamp((x * x).sum(1, keepdim=True), min=1e-12))


def user_vectors(st, t, spec, users, seqs, lens, stats):
    """dense_nn(concat(sqrtn-pooled history, user sparse embeddings, user dense value x embedding)), BN with batch
    statistics (recorded in ``stats``)."""
    E = t["seq_embeds"]
    n_items, dt = E.shape[0], E.dtype
    B = len(users)
    Ez = torch.cat([E, torch.zeros((1, E.shape[1]), dtype=dt)], dim=0)            # pad id n_items reads as zero
    pooled = Ez[torch.as_tensor(np.asarray(seqs, dtype=np.int64))].sum(1)
    ln = torch.sqrt(torch.as_tensor(np.asarray(lens), dtype=dt)).reshape(-1, 1)
    pooled = torch.where(ln > 0, pooled / torch.clamp(ln, min=1e-30), torch.zeros_like(pooled))
    parts = [pooled]
    users = np.asarray(users)
    if len(spec["user_sparse_col_index"]):
        idx = torch.as_tensor(spec["user_sparse_unique"][users].astype(np.int64))
        parts.append(t["sparse_embeds"][idx].reshape(B, -1))
    if len(spec["user_dense_col_index"]):
        cols = list(spec["user_dense_col_index"])
        x = torch.as_tensor(spec["user_dense_unique"][users], dtype=dt)
        parts.append((x[:, :, None] * t["dense_embeds"][cols][None]).reshape(B, -1))
    a = torch.cat(parts, dim=1)

    def bn(a, j):
        mu, var = a.mean(0), a.var(0, unbiased=False)
        stats[f"bn{j}"] = (mu.detach().numpy(), var.detach().numpy())
        return (a - mu) / torch.sqrt(var + BN_EPS) * t[f"bn{j}_gamma"] + t[f"bn{j}_beta"]

    if st["use_bn"]:
        a = bn(a, 0)
    n = st["n_layers"]
    for i in range(n):
        a = a @ t[f"W{i}"] + t[f"b{i}"]
        if i != n - 1:
            a = torch.relu(a)
            if st["use_bn"]:
                a = bn(a, i + 1)
    return a


def sampled_logits(U, W, b, labels, sampled, log_e_true, log_e_sampled):
    """_compute_sampled_logits: [B, 1 + S] logits, label in column 0, accidental hits at -FLT_MAX."""
    lab = torch.as_tensor(np.asarray(labels, dtype=np.int64))
    smp = torch.as_tensor(np.asarray(sampled, dtype=np.int64))
    true = (U * W[lab]).sum(1) + b[lab] - log_e_true
    s = U @ W[smp].T + b[smp][None] - log_e_sampled[None]
    hit = lab[:, None] == smp[None, :]
    s = s + torch.where(hit, torch.tensor(-FLT_MAX, dtype=s.dtype), torch.tensor(0.0, dtype=s.dtype))
    return torch.cat([true[:, None], s], dim=1)


def forward_backward(st, spec, users, items, seqs, lens, sampled, num_tries, loss_type="sampled_softmax",
                     sampler_kind=0, norm=False, dtype=torch.float64):
    """(loss, grads in the variables' shapes, batch BN statistics, user vectors after any normalisation)."""
    t = {k: torch.tensor(v, dtype=dtype, requires_grad=True) for k, v in st["params"].items()}
    stats = {}
    n_items = st["params"]["seq_embeds"].shape[0]
    U = user_vectors(st, t, spec, users, seqs, lens, stats)
    W = t["item_embeds"]
    if norm:
        U, W = _l2(U), _l2(W)          # normalising the whole table: only the gathered rows matter
    S = len(sampled)
    npdt = np.float64 if dtype == torch.float64 else np.float32
    le_t = torch.as_tensor(np.log(expected_counts(sampler_kind, items, n_items, S, num_tries, npdt)))
    le_s = torch.as_tensor(np.log(expected_counts(sampler_kind, sampled, n_items, S, num_tries, npdt)))
    z = sampled_logits(U, W, t["item_biases"], items, sampled, le_t, le_s)
    B = len(users)
    if loss_type == "sampled_softmax":
        loss = torch.nn.functional.cross_entropy(z, torch.zeros(B, dtype=torch.int64))
    else:
        y = torch.zeros_like(z)
        y[:, 0] = 1.0
        loss = torch.nn.functional.binary_cross_entropy_with_logits(z, y, reduction="none").sum(1).mean()
    loss.backward()
    g = {k: (v.grad.numpy() if v.grad is not None else np.zeros(v.shape)) for k, v in t.items()}
    return float(loss.detach()), g, stats, U.detach().numpy()


def train_step(st, spec, users, items, seqs, lens, sampled, num_tries, lr, eps=1e-5, reg=0.0, decay_steps=0,
               decay_rate=0.96, **kw):
    """One TF-Adam step; returns the data loss (the reported loss excludes the regulariser)."""
    loss, g, stats, _ = forward_backward(st, spec, users, items, seqs, lens, sampled, num_tries, **kw)
    p = st["params"]
    if reg:
        for k in TABLES:
            if k in p:
                g[k] = g[k] + 2.0 * reg * p[k]
    if decay_steps:
        lr = lr * decay_rate ** (st["t"] // decay_steps)
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
