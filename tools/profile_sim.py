"""Time SIM inference (feat_models.SIM): ``recommend`` top-100 with the consumed filter at two shapes, and all-items
grid mode against rows mode over the flat (user, item) grid for the same users.

    python tools/profile_sim.py [--out results/profile_sim.json]

Shapes: C1-like (6 040 users x 3 200 items, ids only) and serving (1 M items, 1 000 users); both at the reference
defaults K = 16, L = 100, S = 10, search_topk = 10, 2 heads, hidden (200, 80), with history lengths drawn so that
long windows are full for most users.  Algorithmic FLOP per pair counts 2 FLOP per FMA: the GSU 2*long_len*K, the ESU
logits and mix 2*2*k*K, the short attention 2*2*S*K, the re-associated first layer 2*2K*H1, the pair's later MLP
layers 2*sum H_i*H_{i+1} and the head 2*H_last (the hoisted item / user parts and the per-user keys / values are per
item / per user and left out).  The share is of the H100 SXM data-sheet FP32 rate (67 TFLOP/s); the card name and
power limit are read in the same run."""
import argparse
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from _profile_common import FP32_PEAK, card, write_report  # noqa: E402


def build(n_users, n_items, K=16, L=100, S=10, k=10, H=2, hidden=(200, 80), seed=0):
    from librecommender_b200 import synthetic as syn
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.consumed import ConsumedCSR
    from librecommender_b200.feat_models import SIM, recent_dual_sequences_csr

    rng = np.random.default_rng(seed)
    spec = syn.make_spec(rng, n_users, n_items, [], [], 0, 0)
    raw = syn.make_sim_weights(rng, spec, K, H, hidden, True)
    n_hist = rng.integers(1, L + S + 40, size=n_users)
    indptr = np.concatenate([[0], np.cumsum(n_hist)]).astype(np.int64)
    csr = ConsumedCSR(indptr, rng.integers(0, n_items, size=int(indptr[-1])).astype(np.int32))
    seqs = recent_dual_sequences_csr(csr, n_items, L, S)
    return SIM(spec, wio.sim_weights(raw), *seqs, user_consumed=csr, search_topk=k), seqs[1]


def flop_per_pair(model, mean_long_len):
    dims = [Wt.shape[0] for Wt, _, _ in model.mlp]
    K = model.K
    return (2 * mean_long_len * K + 4 * model.topk * K + 4 * model.S * K + 4 * K * dims[0]
            + sum(2 * a * b for a, b in zip(dims, dims[1:])) + 2 * dims[-1])


def timed(fn, reps):
    import torch

    fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps, out


def recommend_rate(model, long_lens, users, reps):
    sec, _ = timed(lambda: model.recommend(users, 100, True), reps)
    pairs = len(users) * model.n_items
    f = flop_per_pair(model, float(long_lens[users].mean()))
    return dict(users=len(users), sec=sec, users_per_s=len(users) / sec, pairs_per_s=pairs / sec, flop_per_pair=f,
                share_fp32_peak=pairs * f / sec / FP32_PEAK)


def grid_vs_rows(model, long_lens, users, reps):
    import torch

    u = torch.as_tensor(users, device=model.device)
    N = model.n_items
    uu = np.repeat(users, N)
    ii = np.tile(np.arange(N), len(users))
    assert model._hoistable()
    g_sec, g = timed(lambda: model.score_all_items(u), reps)
    r_sec, r = timed(lambda: model.logits(uu, ii).view(len(users), N), reps)
    g, r = g.cpu().numpy(), r.cpu().numpy()
    scale = np.maximum(np.abs(r), np.abs(r).mean())
    err = np.abs(g - r)
    pairs = len(users) * N
    f = flop_per_pair(model, float(long_lens[users].mean()))
    return dict(users=len(users), items=N, grid_sec=g_sec, rows_sec=r_sec, grid_speedup=r_sec / g_sec,
                grid_pairs_per_s=pairs / g_sec, rows_pairs_per_s=pairs / r_sec,
                grid_share_fp32_peak=pairs * f / g_sec / FP32_PEAK, rows_share_fp32_peak=pairs * f / r_sec / FP32_PEAK,
                max_rel_diff=float((err / scale).max()), share_within_1e5=float((err <= 1e-5 * scale + 1e-6).mean()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card()}
    m, ll = build(6040, 3200)
    res["c1_recommend"] = recommend_rate(m, ll, np.arange(6040), 3)
    res["c1_grid_vs_rows"] = grid_vs_rows(m, ll, np.arange(64), 3)
    del m
    m, ll = build(1000, 1_000_000)
    res["serving_recommend"] = recommend_rate(m, ll, np.arange(8), 2)
    res["serving_grid_vs_rows"] = grid_vs_rows(m, ll, np.arange(2), 2)
    write_report(res, args.out)


if __name__ == "__main__":
    main()
