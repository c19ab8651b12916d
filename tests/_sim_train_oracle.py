"""Torch restatement of ONE SIM training step of the reference (TEST INFRASTRUCTURE ONLY).

Follows ``libreco/algorithms/sim.py:193-304`` with ``is_training=True`` and no dropout, on the RAW variables of
``synthetic.make_sim_weights`` / ``weights_io.load_reference_tf_model(..., "SIM", ...)``:
* ``Gp = combine_seq_features(concat) @ seq_proj``, ``q = Gp[item]``;
* first stage: ``pooled = sum_{t < long_len} Gp[long_t]`` (pad rows inside the length included), ``dense_nn`` on
  ``[q, pooled]`` (``first_stage_mlp``), Dense(1) = z1;
* second stage: the GSU selection (``_sim_oracle.gsu_select`` on the float64 scores, or a forced one), the ESU
  ``multi_head_attention`` of q over the selected rows in either graph (restated here in torch, checked against
  ``_sim_oracle.esu``), the short ``tf_attention``, ``dense_nn`` on ``[long_out, short_out, user, item, sparse..,
  dense..]`` (``second_stage_mlp``), Dense(1) = z2;
* BN on batch statistics (``layers/dense.py:12-49``), mean sigmoid cross entropy or focal loss
  (``tfops/loss.py:14-18, 52-58``) on ``alpha z1 + beta z2``, TF-Adam with the BN moving-statistics update, ``reg`` on
  the embedding tables.
Lengths are clamped to [1, L] / [1, S] as the training collator gives them.  Gradients come from torch autograd.
Float64 by default; ``dtype=torch.float32`` gives the float32 restatement the CPU tests calibrate the GPU bounds with.

**PARITY UNPINNED**, like every graph in ``oracle/tf_models.py``: TensorFlow is not available.
"""
import os
import sys

import numpy as np
import torch

from oracle.fm_train import B1, B2, BN_EPS, BN_MOMENTUM

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _sim_oracle as so  # noqa: E402
import _transformer_train_oracle as tto  # noqa: E402

TABLES = ("user_embeds", "item_embeds", "sparse_embeds", "dense_embeds")
NEG = 1.0e9


def _stack_params(p, moving, prefix, mlp, use_bn):
    n = len(mlp["kernels"])
    for i in range(n):
        p[f"{prefix}W{i}"] = np.array(mlp["kernels"][i], dtype=np.float64)
        p[f"{prefix}b{i}"] = np.array(mlp["biases"][i], dtype=np.float64)
    if use_bn:
        for j, bn in enumerate([mlp.get("bn_in")] + list(mlp.get("bns") or [])):
            p[f"{prefix}bn{j}_gamma"] = np.array(bn["gamma"], dtype=np.float64)
            p[f"{prefix}bn{j}_beta"] = np.array(bn["beta"], dtype=np.float64)
            moving[f"{prefix}bn{j}"] = [np.array(bn["mean"], dtype=np.float64), np.array(bn["var"], dtype=np.float64)]
    return n


def init_state(w, use_bn, topk, alpha=1.0, beta=1.0, loss_type="cross_entropy"):
    p = {k: np.array(w[k], dtype=np.float64) for k in TABLES if w.get(k) is not None}
    st = dict(use_bn=bool(use_bn), t=0, moving={}, scheme=w["sim_scheme"], H=int(w["num_heads"]), topk=int(topk),
              alpha=float(alpha), beta=float(beta), loss_type=loss_type)
    st["n_layers"] = _stack_params(p, st["moving"], "", w["mlp"], use_bn)
    st["n_fs"] = _stack_params(p, st["moving"], "fs_", w["first_stage_mlp"], use_bn)
    for k in ("out_kernel", "first_stage_out_kernel"):
        p[k] = np.array(w[k], dtype=np.float64).reshape(-1)
    for k in ("out_bias", "first_stage_out_bias"):
        p[k] = np.array(w[k], dtype=np.float64).reshape(1)
    p["seq_proj"] = np.array(w["seq_proj"], dtype=np.float64)
    for k in tto.att_names(st["scheme"]):
        p[f"sim_{k}"] = np.array(w["sim_mha"][k], dtype=np.float64)
    st["params"] = p
    st["m"] = {k: np.zeros_like(v) for k, v in p.items()}
    st["v"] = {k: np.zeros_like(v) for k, v in p.items()}
    return st


def esu(t, q, rows, valid, scheme, H):
    """multi_head_attention of q [R, K] over rows [R, k, K] (layers/attention.py:67-138), key i visible where
    ``valid``: keras adds -1e9 to a hidden score, legacy writes -1e9 and applies its value Dense to the projected
    keys."""
    R, K = q.shape
    hd = K // H
    names = [f"sim_{n}" for n in tto.att_names(scheme)]
    vm = torch.as_tensor(np.asarray(valid))[:, None, :]
    if scheme == "keras":
        wq, wk, wv, wo = (t[n] for n in names)
        qh = torch.einsum("rd,dhk->rhk", q, wq) * (1.0 / np.sqrt(hd))
        kh = torch.einsum("rtd,dhk->rthk", rows, wk)
        vh = torch.einsum("rtd,dhk->rthk", rows, wv)
        a = torch.einsum("rhk,rthk->rht", qh, kh)
        o = torch.einsum("rht,rthk->rhk", torch.softmax(torch.where(vm, a, a - NEG), dim=-1), vh)
        return torch.einsum("rhk,hkd->rd", o, wo)
    wq, wk, wv, wo = (t[n] for n in names)
    keys = rows @ wk
    qh = (q @ wq).reshape(R, H, hd)
    vh = (keys @ wv).reshape(R, -1, H, hd)
    a = torch.einsum("rhk,rthk->rht", qh, keys.reshape(R, -1, H, hd)) * (1.0 / np.sqrt(hd))
    o = torch.einsum("rht,rthk->rhk", torch.softmax(torch.where(vm, a, torch.full_like(a, -NEG)), dim=-1), vh)
    return o.reshape(R, K) @ wo


def _stack(st, t, prefix, n, act, bn_frozen, stats):
    dt = act.dtype

    def bn(z, j):
        name = f"{prefix}bn{j}"
        if bn_frozen:
            mu, var = (torch.as_tensor(a, dtype=dt) for a in st["moving"][name])
        else:
            mu, var = z.mean(0), z.var(0, unbiased=False)
            if stats is not None:
                stats[name] = (mu.detach().numpy().astype(np.float64), var.detach().numpy().astype(np.float64))
        return (z - mu) / torch.sqrt(var + BN_EPS) * t[f"{name}_gamma"] + t[f"{name}_beta"]

    if st["use_bn"]:
        act = bn(act, 0)
    for i in range(n):
        act = act @ t[f"{prefix}W{i}"] + t[f"{prefix}b{i}"]
        if i != n - 1:
            act = torch.relu(act)
            if st["use_bn"]:
                act = bn(act, i + 1)
    return act


def logits(st, t, spec, users, items, long_seqs, long_lens, short_seqs, short_lens, sparse, dense, sel=None,
           bn_frozen=False, stats=None):
    """Training-mode (alpha z1 + beta z2, z1, z2, the selection [R, k], margins, |s_k|) of explicit rows (batch
    statistics in the BN, recorded into ``stats``); ``bn_frozen``: the moving statistics (the inference graph).
    ``sel`` forces the GSU selection."""
    ls, ss = np.asarray(long_seqs, dtype=np.int64), np.asarray(short_seqs, dtype=np.int64)
    R, L = ls.shape
    S = ss.shape[1]
    ll, sl = np.clip(np.asarray(long_lens), 1, L), np.clip(np.asarray(short_lens), 1, S)
    items = np.asarray(items, dtype=np.int64)
    Gp = tto.item_table(t, spec) @ t["seq_proj"]
    q = Gp[torch.as_tensor(items)]
    rows = Gp[torch.as_tensor(ls)]                                      # [R, L, K]
    scores = so.gsu_scores(Gp.detach().double().numpy(), items, ls, ll)
    margin, sk = so.gsu_margin(scores, ll, st["topk"])
    if sel is None:
        sel = so.gsu_select(scores, st["topk"])
    sel = np.asarray(sel, dtype=np.int64)
    inside = torch.as_tensor(np.arange(L)[None, :] < ll[:, None])
    pooled = (rows * inside[:, :, None].to(rows.dtype)).sum(1)
    z1 = _stack(st, t, "fs_", st["n_fs"], torch.cat([q, pooled], dim=1), bn_frozen, stats) @ \
        t["first_stage_out_kernel"] + t["first_stage_out_bias"][0]
    selrows = torch.gather(rows, 1, torch.as_tensor(sel)[:, :, None].expand(-1, -1, rows.shape[2]))
    long_out = esu(t, q, selrows, sel < ll[:, None], st["scheme"], st["H"])
    Sg = Gp[torch.as_tensor(ss)]
    a = torch.einsum("rd,rtd->rt", q, Sg)
    smask = torch.as_tensor(np.arange(S)[None, :] < sl[:, None])
    short_out = (torch.softmax(torch.where(smask, a, a - NEG), dim=1)[:, :, None] * Sg).sum(1)
    xs = [long_out, short_out, t["user_embeds"][torch.as_tensor(np.asarray(users, dtype=np.int64))], t["item_embeds"][
        torch.as_tensor(items)]]
    if sparse is not None:
        xs.append(t["sparse_embeds"][torch.as_tensor(np.asarray(sparse, dtype=np.int64))].reshape(R, -1))
    if dense is not None:
        xs.append((torch.as_tensor(np.asarray(dense), dtype=q.dtype)[:, :, None] * t["dense_embeds"][None]).reshape(R, -1))
    z2 = _stack(st, t, "", st["n_layers"], torch.cat(xs, dim=1), bn_frozen, stats) @ t["out_kernel"] + \
        t["out_bias"][0]
    return st["alpha"] * z1 + st["beta"] * z2, z1, z2, sel, margin, sk


def loss_of(z, labels, loss_type):
    y = torch.as_tensor(np.asarray(labels), dtype=z.dtype)
    bce = torch.nn.functional.binary_cross_entropy_with_logits(z, y, reduction="none")
    if loss_type == "focal":
        p = torch.sigmoid(z)
        p_t = y * p + (1 - y) * (1 - p)
        bce = (y * 0.25 + (1 - y) * 0.75) * (1 - p_t) ** 2 * bce
    return bce.mean()


def forward_backward(st, spec, users, items, ls, ll, ss, sl, sparse, dense, labels, sel=None, dtype=torch.float64):
    """Returns (loss, logits, {variable: gradient}, batch BN statistics, selection, margins, |s_k|) of one batch."""
    t = {k: torch.tensor(v, dtype=dtype, requires_grad=True) for k, v in st["params"].items()}
    stats = {}
    z, _, _, sel, margin, sk = logits(st, t, spec, users, items, ls, ll, ss, sl, sparse, dense, sel=sel, stats=stats)
    loss = loss_of(z, labels, st["loss_type"])
    loss.backward()
    g = {k: (v.grad.numpy().astype(np.float64) if v.grad is not None else np.zeros(v.shape)) for k, v in t.items()}
    return float(loss.detach()), z.detach().numpy().astype(np.float64), g, stats, sel, margin, sk


def train_step(st, spec, users, items, ls, ll, ss, sl, sparse, dense, labels, lr, eps=1e-5, reg=0.0, decay_steps=0,
               decay_rate=0.96, sel=None):
    """One TF-Adam step with the BN moving-statistics update; returns (the data loss, the selection used)."""
    p = st["params"]
    loss, _, g, stats, sel, _, _ = forward_backward(st, spec, users, items, ls, ll, ss, sl, sparse, dense, labels, sel)
    if reg:
        for k in TABLES:
            if k in p:
                g[k] = g[k] + 2.0 * reg * p[k]
    if decay_steps:
        lr = lr * decay_rate ** (st["t"] // decay_steps)
    st["t"] += 1
    lr_t = lr * np.sqrt(1 - B2 ** st["t"]) / (1 - B1 ** st["t"])
    for k in p:
        st["m"][k] = B1 * st["m"][k] + (1 - B1) * g[k]
        st["v"][k] = B2 * st["v"][k] + (1 - B2) * np.square(g[k])
        p[k] -= lr_t * st["m"][k] / (np.sqrt(st["v"][k]) + eps)
    for name, (mu, var) in stats.items():
        mm, mv = st["moving"][name]
        st["moving"][name] = [BN_MOMENTUM * mm + (1 - BN_MOMENTUM) * mu, BN_MOMENTUM * mv + (1 - BN_MOMENTUM) * var]
    return loss, sel


def raw_weights(st, w):
    """The raw weight dict of ``w`` with the oracle's current variables and BN moving statistics."""
    p = st["params"]
    out = dict(w)
    for k in TABLES:
        if k in p:
            out[k] = p[k].astype(np.float32)

    def stack(prefix, n):
        mlp = dict(kernels=[p[f"{prefix}W{i}"].astype(np.float32) for i in range(n)],
                   biases=[p[f"{prefix}b{i}"].astype(np.float32) for i in range(n)])
        if st["use_bn"]:
            def bn(j):
                mm, mv = st["moving"][f"{prefix}bn{j}"]
                return dict(gamma=p[f"{prefix}bn{j}_gamma"].astype(np.float32),
                            beta=p[f"{prefix}bn{j}_beta"].astype(np.float32), mean=mm.astype(np.float32),
                            var=mv.astype(np.float32))
            mlp["bn_in"] = bn(0)
            mlp["bns"] = [bn(i + 1) for i in range(n - 1)]
        return mlp

    out["mlp"], out["first_stage_mlp"] = stack("", st["n_layers"]), stack("fs_", st["n_fs"])
    for k in ("out_kernel", "first_stage_out_kernel"):
        out[k] = p[k].astype(np.float32).reshape(-1, 1)
    for k in ("out_bias", "first_stage_out_bias"):
        out[k] = p[k].astype(np.float32).reshape(1)
    out["seq_proj"] = p["seq_proj"].astype(np.float32)
    out["sim_mha"] = {k: p[f"sim_{k}"].astype(np.float32) for k in tto.att_names(st["scheme"])}
    return out


# ------------------------------------------------------------------------------------------------------
# seeded training cases shared by the GPU tests and the CPU checks
# ------------------------------------------------------------------------------------------------------
def make_train_case(layout, K, H, use_bn, version, seed=0, n_users=40, n_items=60, L=24, S=6, k=6, R=96,
                    hidden=(24, 12)):
    """(spec, raw weights, consumed, rows): rows = (users, items, long_seqs, long_lens, short_seqs, short_lens,
    sparse, dense, labels) with per-row dual windows from a numpy restatement of ``get_dual_seqs`` (every length
    class, exact GSU ties from repeated items)."""
    from librecommender_b200 import synthetic as syn

    rng = np.random.default_rng(seed + 11 * K + H)
    if layout == "ids":
        spec = syn.make_spec(rng, n_users, n_items, [], [], 0, 0)
        w = syn.make_sim_weights(rng, spec, K, H, hidden, use_bn, version)
    elif layout == "feat":
        spec = syn.make_spec(rng, n_users, n_items, [7, 30], [11, 5], 1, 2)
        w = syn.make_sim_weights(rng, spec, K, H, hidden, use_bn, version)
    else:
        spec = syn.make_multi_sparse_spec(rng, n_users, n_items, [9], [12, 6], [("user", 17, 3), ("item", 23, 2)], 1, 1)
        w = syn.make_sim_weights(rng, spec, K, H, hidden, use_bn, version, combiner="normal")
        w["multi_sparse_combiner"] = "normal"
    consumed = so.make_consumed(rng, n_users, n_items, L, S, k)
    consumed[0] = [3]
    users = rng.integers(0, n_users, size=R)
    pos = np.array([int(rng.integers(0, max(len(consumed[u]), 1))) for u in users])
    items = np.array([consumed[u][p] if consumed[u] and rng.random() < 0.7 else int(rng.integers(0, n_items))
                      for u, p in zip(users, pos)])
    ls, ll, ss, sl = dual_windows(consumed, users, pos, n_items, L, S)
    from oracle import tf_models as tm
    sparse, dense = tm.row_features(spec, users, items)
    labels = (rng.random(R) < 0.5).astype(np.float32)
    return spec, w, consumed, (users, items, ls, ll, ss, sl, sparse, dense, labels)


def dual_windows(consumed, users, positions, pad, L, S):
    """get_dual_seqs (libreco/batch/sequence.py:94-147) at given positions."""
    n = len(users)
    ls, ss = np.full((n, L), pad, dtype=np.int32), np.full((n, S), pad, dtype=np.int32)
    ll, sl = np.ones(n, dtype=np.int32), np.ones(n, dtype=np.int32)
    for j, (u, p) in enumerate(zip(users, positions)):
        c = consumed[int(u)]
        p = int(p)
        s_cnt = min(p, S)
        l_cnt = 0 if p <= S else min(p - S, L)
        ss[j, :s_cnt] = c[p - s_cnt:p]
        ls[j, :l_cnt] = c[p - s_cnt - l_cnt:p - s_cnt]
        ll[j], sl[j] = max(l_cnt, 1), max(s_cnt, 1)
    return ls, ll, ss, sl
