"""Time Transformer inference (feat_models.Transformer): ``recommend`` top-100 with the consumed filter at two shapes,
and all-items grid mode against rows mode over the flat (user, item) grid for the same users.

    python tools/profile_transformer.py [--out results/profile_transformer.json]

Shapes: C1-like (6 040 users x 3 200 items, T = 10, K = 16, ids only; D = 32) and serving (1 M items, K = 16, three
item sparse fields so D = 80, T = 50, hidden (128, 64, 32)).  Algorithmic FLOP per pair counts 2 FLOP per FMA:
target-attention logits 2*len*D + the mix 2*len*H1 + the pair's MLP layers 2*sum H_i*H_{i+1} + the head 2*H_last
(the hoisted item / user parts and the encoder are per item / per user and left out).  The share is of the H100 SXM
data-sheet FP32 rate (67 TFLOP/s); the card name and power limit are read in the same run."""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from _profile_common import FP32_PEAK, card  # noqa: E402


def build(n_users, n_items, K, T, item_sparse, hidden, seed=0):
    from librecommender_b200 import synthetic as syn
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.consumed import ConsumedCSR
    from librecommender_b200.feat_models import Transformer

    rng = np.random.default_rng(seed)
    spec = syn.make_spec(rng, n_users, n_items, [], item_sparse, 0, 0)
    raw = syn.make_transformer_weights(rng, spec, K, 1, 1, T, hidden, True)
    lens = rng.integers(1, T + 1, size=n_users + 1).astype(np.int32)
    lens[n_users] = 1
    seqs = rng.integers(0, n_items, size=(n_users + 1, T)).astype(np.int32)
    seqs[np.arange(T)[None, :] >= lens[:, None]] = n_items
    indptr = np.concatenate([[0], np.cumsum(lens[:n_users])]).astype(np.int64)
    idx = np.concatenate([seqs[u, :lens[u]] for u in range(n_users)]).astype(np.int32)
    return Transformer(spec, wio.transformer_weights(raw), seqs, lens, ConsumedCSR(indptr, idx)), lens


def flop_per_pair(model, mean_len):
    dims = [Wt.shape[0] for Wt, _, _ in model.mlp]
    return 2 * mean_len * model.D + 2 * mean_len * dims[0] + sum(2 * a * b for a, b in zip(dims, dims[1:])) + 2 * dims[-1]


def timed(fn, reps):
    import torch

    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps, out


def recommend_rate(model, lens, users, reps):
    sec, _ = timed(lambda: model.recommend(users, 100, True), reps)
    pairs = len(users) * model.n_items
    f = flop_per_pair(model, float(lens[users].mean()))
    return dict(users=len(users), sec=sec, users_per_s=len(users) / sec, pairs_per_s=pairs / sec, flop_per_pair=f,
                share_fp32_peak=pairs * f / sec / FP32_PEAK)


def grid_vs_rows(model, users, reps):
    import torch

    u = torch.as_tensor(users, device=model.device)
    N = model.n_items
    uu = np.repeat(users, N)
    ii = np.tile(np.arange(N), len(users))
    g_sec, g = timed(lambda: model.score_all_items(u), reps)
    r_sec, r = timed(lambda: model.logits(uu, ii).view(len(users), N), reps)
    g, r = g.cpu().numpy(), r.cpu().numpy()
    scale = np.maximum(np.abs(r), np.abs(r).mean())
    return dict(users=len(users), items=N, grid_sec=g_sec, rows_sec=r_sec, grid_speedup=r_sec / g_sec,
                max_rel_diff=float((np.abs(g - r) / scale).max()), agree_1e5=bool((np.abs(g - r) <= 1e-5 * scale + 1e-6).all()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card()}
    m, lens = build(6040, 3200, 16, 10, [], (128, 64, 32))
    res["c1_recommend"] = recommend_rate(m, lens, np.arange(6040), 3)
    res["c1_grid_vs_rows"] = grid_vs_rows(m, np.arange(64), 5)
    del m
    m, lens = build(1000, 1_000_000, 16, 50, [20, 50, 300], (128, 64, 32))
    assert m.D == 80
    res["serving_recommend"] = recommend_rate(m, lens, np.arange(8), 2)
    res["serving_grid_vs_rows"] = grid_vs_rows(m, np.arange(2), 3)
    line = json.dumps(res, indent=1)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line)


if __name__ == "__main__":
    main()
