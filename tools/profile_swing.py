"""Time Swing on the GPU (``librecommender_b200.swing``): ``compute_swing`` (``b200_swing_scores``), recommend for a set
of users (``b200_nbr_recommend`` + ``b200_topk_rows``) and predict (``b200_nbr_predict``).

    python tools/profile_swing.py [--reps 5] [--out /tmp/swing.json]

Workloads:
* C1: the reference's ``sample_movielens_rating.dat`` (duplicates dropped, keep last), when the reference is staged;
* synthetic: 1 M users x 200 k items, user degree ``clip(Poisson(30), 1, 300)``, items drawn with Zipf popularity
  ``p_i ~ (i + 1)^-s`` (duplicates dropped), ``s`` set by bisection so that the expected ``sum_i C(d_i, 2)`` is 10^10.

Reported: the median and spread of ``--reps`` timed calls (host clock around work that ends in a device synchronise,
after one warm-up call), user pairs per second (``sum_i C(d_i, 2)``), probed entries per second (``sum`` over pairs
of ``|I_v|``, the row the warps scan), the workspace bytes, recommend users per second at top_k 20 / n_rec 10 and
predictions per second.  The card's name, power limit and max SM clock are read in the same run.
"""
import argparse
import os
import sys
import time

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _profile_common import card, write_report  # noqa: E402


def c1():
    import pandas as pd

    from oracle.ref_loader import reference_available, sample_data_path

    if not reference_available():
        return None
    df = pd.read_csv(sample_data_path(), sep="::", names=["user", "item", "label", "time"], engine="python")
    u, _ = pd.factorize(df["user"])
    i, _ = pd.factorize(df["item"])
    df = pd.DataFrame({"u": u, "i": i, "label": df["label"].astype(np.float32)})
    df = df.drop_duplicates(subset=["u", "i"], keep="last")
    R = sp.csr_matrix((df["label"].to_numpy(), (df["u"].to_numpy(), df["i"].to_numpy())), dtype=np.float32)
    R.sort_indices()
    return R


def synthetic(n_users=1_000_000, n_items=200_000, mean_deg=30, max_deg=300, pairs=1e10, seed=0):
    g = np.random.default_rng(seed)
    deg = np.clip(g.poisson(mean_deg, n_users), 1, max_deg)
    n = int(deg.sum())
    rank = np.arange(1, n_items + 1, dtype=np.float64)

    def expected_pairs(s):
        p = rank ** -s
        p /= p.sum()
        d = n_users * -np.expm1(n / n_users * np.log1p(-np.minimum(p, 1 - 1e-12)))   # E[distinct users per item]
        return float((d * (d - 1) / 2).sum()), p

    lo, hi = 0.0, 2.0
    for _ in range(40):
        mid = (lo + hi) / 2
        lo, hi = (mid, hi) if expected_pairs(mid)[0] < pairs else (lo, mid)
    s = (lo + hi) / 2
    p = expected_pairs(s)[1]
    items = np.searchsorted(np.cumsum(p), g.random(n) * np.cumsum(p)[-1]).clip(0, n_items - 1)
    users = np.repeat(np.arange(n_users, dtype=np.int64), deg)
    key = np.unique(users * n_items + items)
    R = sp.csr_matrix((np.ones(len(key), np.float32), (key // n_items, key % n_items)), shape=(n_users, n_items))
    return R, s


def counts(R):
    """(user pairs, probed entries): sum_i C(d_i, 2) and, over the pairs u < v of every item, sum |I_v|."""
    RT = R.T.tocsr()
    d = np.diff(RT.indptr).astype(np.float64)
    pos = np.arange(RT.nnz) - np.repeat(RT.indptr[:-1], np.diff(RT.indptr))
    udeg = np.diff(R.indptr).astype(np.float64)
    return float((d * (d - 1) / 2).sum()), float((pos * udeg[RT.indices]).sum())


def timed(fn, reps):
    import torch

    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return float(np.median(ts)), float(min(ts)), float(max(ts))


def profile(name, R, reps, n_rec_users):
    import torch

    from librecommender_b200.swing import Swing, plan

    from librecommender_b200.consumed import ConsumedCSR

    n_users, n_items = R.shape
    eng = Swing(20, 1.0, 0, n_users, n_items, R, R.T.tocsr(), ConsumedCSR(R.indptr, R.indices), 0.0)
    pairs, probes = counts(R)
    med, lo, hi = timed(eng.compute_swing, reps)
    smem_acc, ctas = plan(n_items, 20)
    g = np.random.default_rng(1)
    users = torch.as_tensor(g.choice(n_users, size=min(n_rec_users, n_users), replace=False)).cuda()
    rmed, rlo, rhi = timed(lambda: eng.recommend_device(users, 10, True, False), reps)
    pu = torch.as_tensor(g.integers(0, n_users, 1 << 20)).cuda()
    pi = torch.as_tensor(g.integers(0, n_items, 1 << 20)).cuda()
    pmed, plo, phi = timed(lambda: eng.predict_device(pu, pi), reps)
    return dict(workload=name, n_users=n_users, n_items=n_items, nnz=int(R.nnz), user_pairs=pairs,
                probed_entries=probes, swing_elements=eng.num_swing_elements(),
                shared_memory_accumulator=smem_acc, resident_ctas=ctas, workspace_bytes=eng.workspace_bytes,
                compute_swing_sec=dict(median=med, min=lo, max=hi), user_pairs_per_s=pairs / med,
                probed_entries_per_s=probes / med,
                recommend_users=int(users.numel()), recommend_sec=dict(median=rmed, min=rlo, max=rhi),
                recommend_users_per_s=users.numel() / rmed,
                predict_rows=int(pu.numel()), predict_sec=dict(median=pmed, min=plo, max=phi),
                predict_rows_per_s=pu.numel() / pmed)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("profile_swing.py needs a CUDA device")
    res = dict(card=card(), runs=[])
    R = c1()
    if R is not None:
        res["runs"].append(profile("C1", R, a.reps, R.shape[0]))
    R, s = synthetic()
    run = profile("synthetic 1M x 200k", R, a.reps, 131072)
    run["zipf_exponent"] = s
    res["runs"].append(run)
    write_report(res, a.out)


if __name__ == "__main__":
    main()
