"""Time GraphSage training on the GPU (``librecommender_b200.sage.GraphSageTrainer``): one step split into its phases
(i2i walk pairs, negatives and neighbour sampling, encoder forward, backward, Adam) and a whole step.

    python tools/profile_sage_train.py [--large-items 1000000] [--large-users 10000000] [--batch 256] [--out f.json]

Graphs: C1 (``tests/golden/sage.npz``, pure) and the seeded synthetic graph of ``tools/profile_sage.py``
(``--large-items`` items, ``--large-users`` users).  The reference's defaults: embed 16, 2 layers, 3 neighbours,
10 walks of 5 one-walks, one negative, cross entropy, batch 256; both paradigms (u2i on random training pairs).

Phases (CUDA events over ``--reps`` calls after a warm-up; the walk-pair phase includes its one device-to-host copy):
``walk_pairs_sec`` (i2i), ``sample_sec`` (negatives + neighbours of the query, positive and negative items),
``forward_sec`` (gather, projection, layers), ``backward_sec`` (every layer back to the tables), ``adam_sec``,
``step_sec`` (a whole ``step``; the pieces also include the pair scores and the loss).  The card's name and power limit
are read in the same run.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _profile_common import card, event_seconds, write_report  # noqa: E402
from profile_sage import synthetic  # noqa: E402


def profile(name, di, paradigm, batch, reps):
    import torch

    from librecommender_b200.sage import GraphSageTrainer

    tr = GraphSageTrainer(di, paradigm=paradigm, seed=0)
    rng = np.random.default_rng(0)
    users = torch.as_tensor(rng.integers(0, tr.n_users, batch)).cuda()
    items = torch.as_tensor(rng.integers(0, tr.n_items, batch).astype(np.int32)).cuda()
    res = dict(graph=name, paradigm=paradigm, n_items=tr.n_items, n_users=tr.n_users, batch=batch, d=tr.d)
    if paradigm == "i2i":
        res["walk_pairs_sec"] = event_seconds(lambda: tr.walk_pairs(batch), reps)
        _, q, pos = tr.walk_pairs(batch)
        res["pairs"] = int(q.numel())

        def sample():
            neg = tr.negatives(pos, items=q)
            return tr.levels(torch.cat([q, pos, neg]))
    else:
        pos = items

        def sample():
            neg = tr.negatives(pos, users=users)
            return tr.levels(torch.cat([pos, neg]))
    res["sample_sec"] = event_seconds(sample, reps)
    ids = sample()
    res["encoder_rows"] = int(sum(a.numel() for a in ids))
    res["forward_sec"] = event_seconds(lambda: tr.encode(ids), reps)
    R, c = tr.encode(ids)
    dR = torch.randn_like(R)
    res["backward_sec"] = event_seconds(lambda: tr.encode_backward(c, dR), reps)
    res["adam_sec"] = event_seconds(tr.adam_update, reps)
    if paradigm == "i2i":
        res["step_sec"] = event_seconds(lambda: tr.step(batch_size=batch), reps)
    else:
        res["step_sec"] = event_seconds(lambda: tr.step(users, items), reps)
    print(res, file=sys.stderr)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--large-items", type=int, default=1_000_000)
    ap.add_argument("--large-users", type=int, default=10_000_000)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    from test_sage_cpu import data_info, golden

    out = dict(card=card(), runs=[])
    di = data_info(golden(), "pure")
    for paradigm in ("i2i", "u2i"):
        out["runs"].append(profile("C1", di, paradigm, a.batch, a.reps))
    di, _ = synthetic(a.large_items, a.large_users, 16)
    for paradigm in ("i2i", "u2i"):
        out["runs"].append(profile(f"synthetic {a.large_items} items x {a.large_users} users", di, paradigm, a.batch,
                                   a.reps))
    write_report(out, a.out)


if __name__ == "__main__":
    main()
