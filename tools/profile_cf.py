"""Time UserCF and ItemCF on the GPU (``librecommender_b200.cf``): ``compute_similarities`` (``b200_cf_cosine``),
recommend for a set of users (``b200_nbr_recommend``, item-based for ItemCF and user-based for UserCF, then
``b200_topk_rows``) and predict (``b200_nbr_predict``).

    python tools/profile_cf.py [--reps 5] [--out /tmp/cf.json]

Workloads (``tools/profile_swing.py``'s graphs):
* C1: the reference's ``sample_movielens_rating.dat`` (duplicates dropped, keep last), both engines, when the
  reference is staged;
* synthetic: 1 M users x 200 k items with Zipf item popularity, 10^10 expected user pairs; ItemCF and UserCF.  The
  largest user count whose UserCF workspace fits in the card's free memory is reported from the workspace query (it
  is computed, not run).

Reported: the median and spread of ``--reps`` timed calls (host clock around work that ends in a device synchronise,
after one warm-up call), co-occurrence pairs per second (``sum`` over middle rows p of ``d_p (d_p - 1)``: every
ordered (x1, x2) pair that shares p, the CAS adds the kernel makes), the workspace bytes, recommend users per second
at k_sim 20 / n_rec 10 and predictions per second.  The card's name, power limit and max SM clock are read in the same
run.  There is no CPU baseline: recfarm is a Rust extension that is not built here.
"""
import argparse
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from _profile_common import card, write_report  # noqa: E402
from profile_swing import c1, synthetic, timed  # noqa: E402


def cooccurrence_pairs(R, user_based):
    """Ordered (x1, x2 != x1) pairs over the middle rows: items' users for UserCF, users' items for ItemCF."""
    mid = R.T.tocsr() if user_based else R
    d = np.diff(mid.indptr).astype(np.float64)
    return float((d * (d - 1)).sum())


def profile(name, R, user_based, reps, n_rec_users):
    import torch

    from librecommender_b200.cf import ItemCF, UserCF, plan
    from librecommender_b200.consumed import ConsumedCSR

    n_users, n_items = R.shape
    n_x = n_users if user_based else n_items
    cls = UserCF if user_based else ItemCF
    eng = cls("ranking", 20, n_users, n_items, 1, R, R.T.tocsr(), ConsumedCSR(R.indptr, R.indices), 0.0)
    pairs = cooccurrence_pairs(R, user_based)
    med, lo, hi = timed(eng.compute_similarities, reps)
    smem_acc, ctas = plan(n_x, 20)
    g = np.random.default_rng(1)
    users = torch.as_tensor(g.choice(n_users, size=min(n_rec_users, n_users), replace=False)).cuda()
    rmed, rlo, rhi = timed(lambda: eng.recommend_device(users, 10, True, False), reps)
    pu = torch.as_tensor(g.integers(0, n_users, 1 << 20)).cuda()
    pi = torch.as_tensor(g.integers(0, n_items, 1 << 20)).cuda()
    pmed, plo, phi = timed(lambda: eng.predict_device(pu, pi), reps)
    return dict(workload=name, engine=cls.__name__, n_users=n_users, n_items=n_items, nnz=int(R.nnz),
                cooccurrence_pairs=pairs, sim_elements=eng.num_sim_elements(), shared_memory_accumulator=smem_acc,
                resident_ctas=ctas, workspace_bytes=eng.workspace_bytes,
                compute_similarities_sec=dict(median=med, min=lo, max=hi), cooccurrence_pairs_per_s=pairs / med,
                recommend_users=int(users.numel()), recommend_sec=dict(median=rmed, min=rlo, max=rhi),
                recommend_users_per_s=users.numel() / rmed,
                predict_rows=int(pu.numel()), predict_sec=dict(median=pmed, min=plo, max=phi),
                predict_rows_per_s=pu.numel() / pmed)


def largest_user_cf(free_bytes, k_sim=20):
    """Largest n_users whose UserCF workspace plus outputs fit in ``free_bytes`` (bisection on the workspace query)."""
    from librecommender_b200.cf import workspace_bytes

    def need(n):
        return workspace_bytes(n, k_sim) + n * (k_sim * 8 + 8)

    lo, hi = 1, 1 << 30
    while lo < hi:
        mid = (lo + hi + 1) // 2
        lo, hi = (mid, hi) if need(mid) <= free_bytes else (lo, mid - 1)
    return dict(free_bytes=int(free_bytes), n_users=lo, bytes=need(lo), bytes_per_user=need(lo) / lo)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("profile_cf.py needs a CUDA device")
    res = dict(card=card(), runs=[])
    R = c1()
    if R is not None:
        for user_based in (False, True):
            res["runs"].append(profile("C1", R, user_based, a.reps, R.shape[0]))
    R, s = synthetic()
    for user_based in (False, True):
        run = profile("synthetic 1M x 200k", R, user_based, a.reps, 131072)
        run["zipf_exponent"] = s
        res["runs"].append(run)
        torch.cuda.empty_cache()
    res["user_cf_largest_fit"] = largest_user_cf(torch.cuda.mem_get_info()[0])
    write_report(res, a.out)


if __name__ == "__main__":
    main()
