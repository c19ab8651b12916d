"""Golden data for GraphSage / PinSage inference, from the live reference (non-DGL path, CPU, no DGL needed).

    python tests/golden/gen_sage.py

Data: C1 pure (``sample_movielens_rating.dat``, ``DatasetPure``) and C1 feat (``sample_movielens_merged.csv``,
``DatasetFeat``: user sex / occupation sparse and age dense, item genre1..3 sparse), both ``split_by_ratio_chrono(
test_size=0.2)``.  For each data set, model (GraphSage, PinSage) and paradigm (i2i, u2i) the reference model is fit
for one epoch on the CPU (embed 8, batch 2048, seed 42, the reference's other defaults), then stored under
``{case}_``:

* ``sd__<key>``: the torch state dict.  Only the C1 pure i2i cases, which the recall comparison serves, keep the
  whole ``item_embeds`` / ``user_embeds`` tables; the others keep the rows the recorded message and the kept users
  read (``sd_rows__<key>``: their ids, ``sd__<key>``: those rows), the rest of the table reads as zeros;
* ``msg_*``: ``NeighborWalker(ITEMS)`` recorded under ``random.seed(7)`` (per-level neighbours, offsets, PinSage
  weights), and ``msg_out``: ``torch_model`` on that message;
* ``users`` / ``user_rows`` (u2i): ``get_user_repr`` of the first users;
* ``ref_metrics``: recall@10 / ndcg@10 of the reference's own ``set_embeddings`` tables on the held-out pairs, and
  for C1 pure i2i ``ref_metrics_walk_seeds``: the same after ``set_embeddings`` under ``random.seed(1000 + s)``,
  s < 5 (the spread the walks alone give on the same weights).

Per data set (``{data}_``): n_users / n_items, the consumed lists as CSRs in list order (``uc_*``, ``ic_*``), the
feature layout and unique tables, and for C1 pure the held-out pairs.  ``cw_*``: ``compute_weights`` (via
``bipartite_neighbors_with_weights`` on a crafted graph) cases with tied counts.  Data only: no reference source.
"""
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle.ref_loader import REFERENCE_ROOT, load_reference, sample_data_path  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "sage.npz")
EMBED, BATCH, SEED, MSG_SEED = 8, 2048, 42, 7
N_MSG_ITEMS, N_USERS_KEPT, WALK_SEEDS = 48, 32, 5
CASES = [(data, model, paradigm) for data in ("pure", "feat") for model in ("graphsage", "pinsage")
         for paradigm in ("i2i", "u2i")]


def _csr(consumed, n):
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum([len(consumed[k]) for k in range(n)], out=indptr[1:])
    return indptr, np.concatenate([np.asarray(consumed[k], dtype=np.int32) for k in range(n)])


def load(data):
    import pandas as pd

    from libreco.data import DatasetFeat, DatasetPure, split_by_ratio_chrono

    if data == "pure":
        df = pd.read_csv(sample_data_path(), sep="::", names=["user", "item", "label", "time"], engine="python")
        train, test = split_by_ratio_chrono(df, test_size=0.2)
        train_data, di = DatasetPure.build_trainset(train)
        eval_data = DatasetPure.build_evalset(test)
    else:
        df = pd.read_csv(os.path.join(REFERENCE_ROOT, "examples/sample_data/sample_movielens_merged.csv"))
        train, test = split_by_ratio_chrono(df, test_size=0.2)
        train_data, di = DatasetFeat.build_trainset(train, ["sex", "age", "occupation"], ["genre1", "genre2", "genre3"],
                                                    ["sex", "occupation", "genre1", "genre2", "genre3"], ["age"])
        eval_data = DatasetFeat.build_evalset(test)
    return train_data, di, eval_data


def data_arrays(di, eval_data):
    out = dict(shape=np.array([di.n_users, di.n_items]))
    out["uc_indptr"], out["uc_items"] = _csr(di.user_consumed, di.n_users)
    out["ic_indptr"], out["ic_users"] = _csr(di.item_consumed, di.n_items)
    assert max(di.n_users, di.n_items) < 1 << 15
    out["uc_items"], out["ic_users"] = out["uc_items"].astype(np.int16), out["ic_users"].astype(np.int16)
    for side in ("user", "item"):
        for kind in ("sparse", "dense"):
            col = getattr(di, f"{side}_{kind}_col")
            out[f"{side}_{kind}_col_index"] = np.asarray(col.index if col.index else [], dtype=np.int64)
            uniq = getattr(di, f"{side}_{kind}_unique")
            if uniq is not None:
                uniq = np.asarray(uniq)
                out[f"{side}_{kind}_unique"] = uniq.astype(np.int32) if kind == "sparse" else uniq
    keep = (eval_data.user_indices < di.n_users) & (eval_data.item_indices < di.n_items)
    out["eval_users"] = eval_data.user_indices[keep].astype(np.int16)
    out["eval_items"] = eval_data.item_indices[keep].astype(np.int16)
    return out


def fit(kind, paradigm, train_data, di):
    import torch

    from libreco.algorithms import GraphSage, PinSage

    torch.manual_seed(SEED)
    random.seed(SEED)
    np.random.seed(SEED)
    cls = GraphSage if kind == "graphsage" else PinSage
    model = cls("ranking", di, paradigm=paradigm, embed_size=EMBED, n_epochs=1, batch_size=BATCH, seed=SEED,
                device="cpu")
    model.fit(train_data, neg_sampling=True, verbose=0, shuffle=True)
    return model


def record(model, kind, paradigm, d_arrays):
    import torch

    from _bpr_oracle import ranking_metrics

    out = {}
    items = np.random.default_rng(MSG_SEED).choice(model.n_items, N_MSG_ITEMS, replace=False).astype(np.int64)
    random.seed(MSG_SEED)
    msg = model.neighbor_walker(items.tolist())
    full = d_arrays["full_tables"]
    rows = {"item_embeds.weight": np.unique(np.concatenate([items] + [n.numpy() for n in msg.neighbors])),
            "user_embeds.weight": np.arange(N_USERS_KEPT)}
    for k, v in model.torch_model.state_dict().items():
        v = v.detach().cpu().numpy()
        if k in rows and not full:
            out[f"sd_rows__{k}"] = rows[k].astype(np.int32)
            v = v[rows[k]]
        out[f"sd__{k}"] = v
    out["msg_items"] = items
    for k in range(model.num_layers):
        out[f"msg_nbs_{k}"] = msg.neighbors[k].numpy().astype(np.int32)
        out[f"msg_offsets_{k}"] = msg.offsets[k].numpy().astype(np.int64)
        if kind == "pinsage":
            out[f"msg_weights_{k}"] = msg.weights[k].numpy().astype(np.float32)
    model.torch_model.eval()
    with torch.inference_mode():
        out["msg_out"] = model.get_item_repr(msg).numpy()
        if paradigm == "u2i":
            users = np.arange(N_USERS_KEPT)
            out["users"] = users
            out["user_rows"] = model.get_user_repr(model.neighbor_walker.get_user_feats(users)).numpy()
    n_u, n_i = model.n_users, model.n_items
    out["ref_metrics"] = np.array(ranking_metrics(model.user_embeds_np[:n_u], model.item_embeds_np[:n_i],
                                                  d_arrays["uc_indptr"], d_arrays["uc_items"],
                                                  d_arrays["eval_users"], d_arrays["eval_items"]))
    if full:     # the reference's own tables under other walk seeds: the spread its sampling alone gives
        runs = []
        for s in range(WALK_SEEDS):
            random.seed(1000 + s)
            model.set_embeddings()
            runs.append(ranking_metrics(model.user_embeds_np[:n_u], model.item_embeds_np[:n_i],
                                        d_arrays["uc_indptr"], d_arrays["uc_items"], d_arrays["eval_users"],
                                        d_arrays["eval_items"]))
        out["ref_metrics_walk_seeds"] = np.array(runs)
    return out


def weight_cases():
    """bipartite_neighbors_with_weights on a small graph whose walks tie counts often."""
    from libreco.sampling.random_walks import bipartite_neighbors_with_weights

    # users 0..5, items 0..7: every item reachable from item 0 in few steps, several with equal degree
    user_consumed = {0: [0, 1, 2], 1: [0, 3, 4], 2: [1, 3, 5], 3: [2, 4, 5, 6], 4: [6, 7], 5: [7, 0, 0]}
    item_consumed = {}
    for u, its in user_consumed.items():
        for i in its:
            item_consumed.setdefault(i, []).append(u)
    out = {"cw_uc_indptr": None}
    out["cw_uc_indptr"], out["cw_uc_items"] = _csr(user_consumed, 6)
    out["cw_ic_indptr"], out["cw_ic_users"] = _csr(item_consumed, 8)
    nodes = list(range(8)) * 6
    ids, wts, lens = [], [], []
    for s, (nn, walks, wl) in enumerate([(2, 3, 2), (3, 4, 1), (4, 6, 3), (1, 5, 2), (3, 2, 4), (5, 10, 2)]):
        random.seed(100 + s)
        nb, w, off, _ = bipartite_neighbors_with_weights(nodes, user_consumed, item_consumed, nn, walks, wl)
        ids.append(np.asarray(nb, dtype=np.int32))
        wts.append(np.asarray(w, dtype=np.float64))
        lens.append(np.diff(np.append(off, len(nb))).astype(np.int32))
        out[f"cw_params_{s}"] = np.array([nn, walks, wl, 100 + s])
    for s in range(len(ids)):
        out[f"cw_ids_{s}"], out[f"cw_weights_{s}"], out[f"cw_lens_{s}"] = ids[s], wts[s], lens[s]
    out["cw_nodes"] = np.asarray(nodes, dtype=np.int32)
    return out


def main():
    load_reference()
    out = weight_cases()
    for data in ("pure", "feat"):
        train_data, di, eval_data = load(data)
        arrays = data_arrays(di, eval_data)
        out.update({f"{data}_{k}": v for k, v in arrays.items() if data == "pure" or not k.startswith("eval_")})
        for kind in ("graphsage", "pinsage"):
            for paradigm in ("i2i", "u2i"):
                model = fit(kind, paradigm, train_data, di)
                rec = record(model, kind, paradigm, dict(arrays, full_tables=data == "pure" and paradigm == "i2i"))
                print(data, kind, paradigm, "reference recall/ndcg@10", rec["ref_metrics"], file=sys.stderr)
                out.update({f"{data}_{kind}_{paradigm}_{k}": v for k, v in rec.items()})
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), file=sys.stderr)


if __name__ == "__main__":
    main()
