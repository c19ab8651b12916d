"""Float64 restatement of one GraphSage training step (``librecommender_b200.sage.GraphSageTrainer``; DESIGN.md §4,
"GraphSage training") for checking the device trainer on the batch it sampled.

* :func:`item_repr` is ``GraphSageModel.forward`` (``graphsage_module.py:103-140``, dropout 0) in torch float64
  autograd over given per-level neighbour ids and offsets; :func:`user_repr` is ``user_repr`` / ``get_raw_features``.
* :func:`pair_scores` and :func:`loss` restate ``compute_pair_scores`` and ``GraphTrainer._loss_scores``
  (``torchops/loss.py``, ``training/torch_trainer.py:254-282``).
* :func:`step` runs the forward, the loss, ``backward`` and one ``torch.optim.Adam(lr, eps, weight_decay=reg)`` step.
* :func:`reference_model` builds the reference's own ``GraphSageModel`` on a data-info stand-in, for pinning the
  restatement when the reference is importable.
"""
import types

import numpy as np
import torch
import torch.nn.functional as F


def params(sd):
    """Leaf float64 tensors of a state dict (numpy or torch values)."""
    return {k: torch.tensor(np.asarray(v, dtype=np.float64), requires_grad=True) for k, v in sd.items()}


def raw(P, ids, feats, prefix):
    """get_raw_features (graphsage_module.py:54-78): [sparse.., dense.., id] then the projection."""
    sparse_unique, dense_unique, dense_cols = feats
    ids = torch.as_tensor(np.asarray(ids, dtype=np.int64))
    parts = []
    if sparse_unique is not None:
        idx = torch.as_tensor(np.asarray(sparse_unique, dtype=np.int64)[ids.numpy()])
        parts.append(P["sparse_embeds.weight"][idx].flatten(start_dim=1))
    if dense_unique is not None:
        vals = torch.as_tensor(np.asarray(dense_unique, dtype=np.float64)[ids.numpy()])
        emb = P["dense_embeds"][list(dense_cols)]
        parts.append((emb[None, :, :] * vals[:, :, None]).flatten(start_dim=1))
    parts.append(P[f"{prefix}_embeds.weight"][ids])
    x = torch.cat(parts, dim=1)
    return x @ P[f"{prefix}_proj.weight"].T + P[f"{prefix}_proj.bias"]


def item_repr(P, items, neighbors, offsets, num_layers, feats):
    """GraphSageModel.forward in float64: ``neighbors[k]`` the ids of level k + 1, ``offsets[k]`` their bag starts."""
    hidden = [raw(P, items, feats, "item")] + [raw(P, n, feats, "item") for n in neighbors]
    for layer in range(num_layers):
        nxt = []
        for k in range(num_layers - layer):
            nb = hidden[k + 1]
            mean = F.embedding_bag(torch.arange(nb.shape[0]), nb, offsets=torch.as_tensor(np.asarray(offsets[k])),
                                   mode="mean")
            h = torch.cat([hidden[k], mean], dim=1) @ P[f"w_linears.{layer}.weight"].T + P[f"w_linears.{layer}.bias"]
            nxt.append(h if layer == num_layers - 1 else F.relu(h))
        hidden = nxt
    return hidden[0]


def user_repr(P, users, feats):
    return raw(P, users, feats, "user")


def pair_scores(q, p, n, repeat_positives):
    """compute_pair_scores (torchops/loss.py:67-90)."""
    if len(q) == len(p) == len(n):
        return (q * p).sum(1), (q * n).sum(1)
    f = len(n) // len(p)
    pos = torch.einsum("ij,ij->i", q, p)
    if repeat_positives:
        pos = pos.repeat_interleave(f)
    neg = torch.einsum("i...k,ijk->ij", q, n.view(len(p), f, -1)).ravel()
    return pos, neg


def _focal(logits, labels, alpha=0.25, gamma=2.0):
    w = labels * alpha + (1 - labels) * (1 - alpha)
    prob = torch.sigmoid(logits)
    p_t = labels * prob + (1 - labels) * (1 - prob)
    return w * torch.pow(1.0 - p_t, gamma) * F.binary_cross_entropy_with_logits(logits, labels, reduction="none")


def loss(loss_type, pos, neg, paradigm, margin=1.0):
    """GraphTrainer._loss_scores: BCE / focal with mean = (paradigm == "u2i"), BPR, max-margin."""
    if loss_type in ("cross_entropy", "focal"):
        if loss_type == "cross_entropy":
            lp = F.binary_cross_entropy_with_logits(pos, torch.ones_like(pos), reduction="none")
            ln = F.binary_cross_entropy_with_logits(neg, torch.zeros_like(neg), reduction="none")
        else:
            lp, ln = _focal(pos, torch.ones_like(pos)), _focal(neg, torch.zeros_like(neg))
        v = torch.cat([lp, ln])
        return v.mean() if paradigm == "u2i" else v.sum()
    if loss_type == "bpr":
        return -F.logsigmoid(pos - neg).mean()
    return F.margin_ranking_loss(pos, neg, torch.ones_like(pos), margin=margin)


def step(sd, batch, cfg, item_feats, user_feats=None):
    """One training step in float64 on a recorded batch.

    ``batch``: ``users`` (u2i), ``items`` (i2i query items), ``items_pos``, ``items_neg`` and ``levels``: the node
    ids per level of the encoder's roots (query items, then positives, then negatives; u2i positives, negatives),
    ``num_neighbors`` per node.  ``cfg``: paradigm, loss_type, num_layers, num_neighbors, margin, lr, epsilon, reg.
    Returns (loss, {key: gradient}, {key: parameter after the Adam step}) as float64 numpy."""
    P = params(sd)
    L, nn = cfg["num_layers"], cfg["num_neighbors"]
    levels = [np.asarray(a, dtype=np.int64) for a in batch["levels"]]
    offsets = [np.arange(a.size, dtype=np.int64) * nn for a in levels[:-1]]
    R = item_repr(P, levels[0], levels[1:], offsets, L, item_feats)
    n = len(batch["items_pos"])
    if cfg["paradigm"] == "u2i":
        q = user_repr(P, batch["users"], user_feats)
        p, ng = R[:n], R[n:]
    else:
        q, p, ng = R[:n], R[n:2 * n], R[2 * n:]
    pos, neg = pair_scores(q, p, ng, cfg["loss_type"] in ("bpr", "max_margin"))
    value = loss(cfg["loss_type"], pos, neg, cfg["paradigm"], cfg.get("margin", 1.0))
    opt = torch.optim.Adam(list(P.values()), lr=cfg["lr"], eps=cfg["epsilon"], weight_decay=cfg.get("reg") or 0.0)
    opt.zero_grad()
    value.backward()
    # a table no side of the paradigm reads has no gradient; torch's Adam leaves it alone
    grads = {k: (v.grad.detach().numpy().copy() if v.grad is not None else np.zeros(tuple(v.shape)))
             for k, v in P.items()}
    opt.step()
    return float(value.detach()), grads, {k: v.detach().numpy().copy() for k, v in P.items()}


def reference_model(di, paradigm, embed_size, num_layers):
    """The reference's GraphSageModel (dropout 0) over a stand-in for its DataInfo built from the dict ``di``."""
    from libreco.algorithms.torch_modules.graphsage_module import GraphSageModel

    def col(names, index):
        return types.SimpleNamespace(name=list(names), index=list(index))

    cols = {}
    for side in ("user", "item"):
        for kind in ("sparse", "dense"):
            idx = list(di.get(f"{side}_{kind}_col_index") or [])
            cols[f"{side}_{kind}"] = col([f"{side}_{kind}_{i}" for i in idx], idx)
    info = types.SimpleNamespace(
        n_users=di["n_users"], n_items=di["n_items"],
        user_col=cols["user_sparse"].name + cols["user_dense"].name,
        item_col=cols["item_sparse"].name + cols["item_dense"].name,
        user_dense_col=cols["user_dense"], item_dense_col=cols["item_dense"],
        sparse_col=col(cols["user_sparse"].name + cols["item_sparse"].name, []),
        dense_col=col(cols["user_dense"].name + cols["item_dense"].name, []),
        user_sparse_unique=di.get("user_sparse_unique"), item_sparse_unique=di.get("item_sparse_unique"))
    return GraphSageModel(paradigm, info, embed_size, 256, num_layers, 0.0)


# ---- i2i walk pairs (csrc/sage_train.cu b200_sage_walk_pairs) -------------------------------------------------------
TAG_START, TAG_WALK, TAG_NEG = 0x5A6E0001, 0x5A6E0002, 0x5A6E0003


def keyed_words(a, b, tag, seed, step):
    """The kernels' Philox words for counter (a, b, step lo, tag), key (seed lo, seed hi ^ step hi)."""
    from oracle.sampling import philox4x32_10

    return philox4x32_10(a, b, step & 0xFFFFFFFF, tag, seed & 0xFFFFFFFF, ((seed >> 32) ^ (step >> 32)) & 0xFFFFFFFF)


def start_nodes(n_starts, n_items, seed, step):
    from _sage_oracle import bounded

    r = keyed_words(np.arange(n_starts, dtype=np.uint32), 0xFFFFFFFF, TAG_START, seed, step)
    return bounded(r[0], r[1], n_items)


def walk_rule(starts, has_no_neighbor, one_walk, num_walks, walk_length, focus_start):
    """pairs_from_random_walk's rule over a draw provider ``one_walk(start index, walk, step, cur) -> next``:
    (items, items_pos, counts per (start, slot)) with slot 0 the no-neighbour pair and slot 1 + w walk w."""
    items, items_pos, counts = [], [], []
    for i, node in enumerate(starts):
        node = int(node)
        lonely = has_no_neighbor(node)
        if lonely:
            items.append(node)
            items_pos.append(node)
        counts.append(int(lonely))
        for w in range(num_walks):
            cur, c = node, 0
            for t in range(walk_length):
                nxt = int(one_walk(i, w, t, cur))
                if focus_start and nxt != node:
                    items.append(node)
                    items_pos.append(nxt)
                    c += 1
                elif not focus_start and nxt != cur:
                    items.append(cur)
                    items_pos.append(nxt)
                    c += 1
                cur = nxt
            counts.append(c)
    return np.asarray(items, dtype=np.int64), np.asarray(items_pos, dtype=np.int64), np.asarray(counts, np.int64)


def keyed_walk_pairs(graph, n_items, n_starts, num_walks, walk_length, focus_start, seed, step):
    """The kernel's expected output: (starts, items, items_pos, counts) on the keyed draws."""
    starts = start_nodes(n_starts, n_items, seed, step)

    def one_walk(i, w, t, cur):
        r = keyed_words(i, w * walk_length + t, TAG_WALK, seed, step)
        return graph.one_walk(np.asarray([cur]), [np.asarray([x]) for x in r])[0]

    return (starts,) + walk_rule(starts, graph.has_no_neighbor, one_walk, num_walks, walk_length, focus_start)
