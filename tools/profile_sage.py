"""Time GraphSage / PinSage inference on the GPU (``librecommender_b200.sage``): the neighbour walks, the hoisted
projection, the layer-wise encoder and the user pooling, each on its own, and a whole ``set_embeddings``.

    python tools/profile_sage.py [--large-items 1000000] [--large-users 10000000] [--out /tmp/sage.json]

Graphs: C1 (``tests/golden/sage.npz``, the fitted pure i2i weights) and a seeded synthetic one: ``--large-users``
users with ``1 + Poisson(4)`` items each drawn Zipf(1.1) over ``--large-items`` items, and user ``i`` also consuming
item ``i`` so that every item has a consumer; random weights at embed 16.  Both models at the reference's defaults
(2 layers, 3 neighbours; PinSage 10 walks of at most 2 steps, termination 0.5), i2i.

Reported per phase: seconds (CUDA events, after a warm-up), nodes sampled per second and one-walks per second
(GraphSage computes all 12 attempts of a slot; PinSage counts the steps taken, about num_walks * 1.5 per node at
termination 0.5), and for the encoder the bytes it moves from shapes over its time against 3.35 TB/s.  The card's
name and power limit are read in the same run.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _profile_common import HBM_PEAK, card, event_seconds, write_report  # noqa: E402


def synthetic(n_items, n_users, d, seed=0):
    g = np.random.default_rng(seed)
    lens = 1 + g.poisson(4, n_users)
    lens[:n_items] += 1
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    np.cumsum(lens, out=indptr[1:])
    items = ((g.zipf(1.1, int(indptr[-1])) - 1) % n_items).astype(np.int32)
    items[indptr[1:n_items + 1] - 1] = np.arange(n_items, dtype=np.int32)
    owner = np.repeat(np.arange(n_users, dtype=np.int32), lens)
    order = np.argsort(items, kind="stable")
    ic_ptr = np.zeros(n_items + 1, dtype=np.int64)
    np.cumsum(np.bincount(items, minlength=n_items), out=ic_ptr[1:])
    di = dict(n_users=n_users, n_items=n_items, user_consumed=(indptr, items), item_consumed=(ic_ptr, owner[order]))
    w = lambda *s: (g.standard_normal(s) / np.sqrt(s[-1])).astype(np.float32)  # noqa: E731
    sd = {"item_embeds.weight": w(n_items, d), "item_proj.weight": w(d, d), "item_proj.bias": w(d)}
    for layer in range(2):
        sd.update({f"w_linears.{layer}.weight": w(d, 2 * d), f"w_linears.{layer}.bias": w(d),
                   f"q_linears.{layer}.weight": w(d, d), f"q_linears.{layer}.bias": w(d)})
    sd.update({"G1.weight": w(d, d), "G1.bias": w(d), "G2.weight": w(d, d)})
    return di, sd


def c1():
    from test_sage_cpu import data_info, golden, state_dict

    z = golden()
    di = data_info(z, "pure")
    return di, {k: state_dict(z, f"pure_{k}_i2i") for k in ("graphsage", "pinsage")}


def encoder_bytes(eng, n):
    """Bytes the encoder moves for n roots: every aggregation reads its self and neighbour rows and writes [n_k, 2d];
    every dense layer reads that and writes [n_k, d] (PinSage also the q layer and the normalisation in place)."""
    d, nn, L = eng.d, eng.num_neighbors, eng.num_layers
    pin = eng.KIND == "PinSage"
    total = 0
    for layer in range(L):
        for k in range(L - layer):
            n_k = n * nn ** k
            total += n_k * (1 + nn) * d * 4 + n_k * 2 * d * 4          # aggregation
            total += n_k * 2 * d * 4 + n_k * d * 4                     # w_linears
            if pin:
                total += 2 * n_k * d * 4 + (n_k * nn * 2 * d * 4 if layer else 0)   # normalise, q
    return total


def profile(name, kind, di, sd, reps):
    import torch

    from librecommender_b200 import sage

    cls = sage.GraphSage if kind == "graphsage" else sage.PinSage
    eng = cls(di, {k: v for k, v in sd.items() if kind == "pinsage" or not k.startswith(("q_", "G"))})
    n = eng.n_items
    roots = torch.arange(n, dtype=torch.int32, device=eng.device)
    nodes = n * sum(eng.num_neighbors ** level for level in range(eng.num_layers))
    walk_s = event_seconds(lambda: eng._sample(roots), reps)
    hoist_s = event_seconds(lambda: (setattr(eng, "P", None), eng._hoist()), reps)
    levels = eng._sample(roots)
    ids = [roots] + [lv[0].reshape(-1) for lv in levels]
    bags = [(None, lv[2], None if lv[1] is None else lv[1].reshape(-1)) for lv in levels]
    enc_s = event_seconds(lambda: eng._encode(ids, bags), reps)
    I = eng._encode(ids, bags)
    pool_s = event_seconds(lambda: eng.user_embeddings(I), reps)
    set_s = event_seconds(lambda: (setattr(eng, "P", None), eng.set_embeddings()), max(1, reps // 2))
    steps = eng.num_neighbors * 12 if kind == "graphsage" else eng.num_walks * (1 + (eng.walk_len - 1) * 0.5)
    eb = encoder_bytes(eng, n)
    res = dict(graph=name, model=kind, n_items=n, n_users=eng.n_users, d=eng.d, walks_sec=walk_s,
               nodes_per_s=nodes / walk_s, one_walks_per_s=nodes * steps / walk_s, hoist_sec=hoist_s,
               encoder_sec=enc_s, encoder_bytes=eb, encoder_bytes_per_s=eb / enc_s,
               encoder_hbm_share=eb / enc_s / HBM_PEAK, user_pool_sec=pool_s, set_embeddings_sec=set_s)
    print(res, file=sys.stderr)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--large-items", type=int, default=1_000_000)
    ap.add_argument("--large-users", type=int, default=10_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    out = dict(card=card(), runs=[])
    di, sds = c1()
    for kind in ("graphsage", "pinsage"):
        out["runs"].append(profile("C1", kind, di, sds[kind], a.reps))
    di, sd = synthetic(a.large_items, a.large_users, 16)
    for kind in ("graphsage", "pinsage"):
        out["runs"].append(profile(f"synthetic {a.large_items} items x {a.large_users} users", kind, di, sd,
                                   max(1, a.reps // 2)))
    write_report(out, a.out)


if __name__ == "__main__":
    main()
