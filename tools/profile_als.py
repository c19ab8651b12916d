"""Profile ALS training half-epochs (``csrc/als.cu``) on a C5-like interaction graph generated on the device.

    python tools/profile_als.py [--scales 1.0,0.1] [--reps 3] [--out results/als.json]

Graph (seeded): 10 M users x 1 M items at scale 1.0 (one tenth of both at 0.1); user degrees min(Poisson(50), 2000)
(at least 1); items drawn from Zipf(1.0) over the catalogue, so popular items have millions of users and take the
chunked long-row path on the items side.  Ranking data are alpha * 1 + 1 = 11 (alpha = 10); rating data are
uniform in 1..5.  Swept: d in {16, 64} over ranking/CG (the reference default, cg_steps = 3), ranking/direct and
rating/CG, reg = 1.0.  Per half-epoch, CUDA events time the users side, the items side and each side's A0 (the
Gram of the fixed table on the split-K dense product).

Each timed call restores its table first (the copy is timed separately and subtracted), so every call does the
work of a first half-epoch from the same start.

Minimal bytes of a side (the algorithm's compulsory traffic, once): nnz (8 + 4 d) (index, value, the gathered
row) plus n_x 8 d (read and write X); the Gram reads n_y 4 d.  FP32 FLOP (a multiply-add counts 2): CG
(1 + cg_steps) (4 d nnz + 2 d^2 n_x); direct 2 d^2 nnz + 2 d nnz + n_x (d^3 / 3 + 2 d^2); Gram 2 n_y d^2.  The
share of peak is the larger of bytes / HBM peak and FLOP / FP32 peak over the measured time, and the report says
which of the two bounds it.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from _profile_common import FP32_PEAK, HBM_PEAK, card, event_seconds, write_report  # noqa: E402

CG_STEPS = 3


def make_graph(n_users, n_items, seed=0):
    """Users CSR (indptr int64, indices int32) on the device, items by Zipf(1.0) inverse CDF."""
    import torch

    g = torch.Generator(device="cuda").manual_seed(seed)
    deg = torch.poisson(torch.full((n_users,), 50.0, device="cuda"), generator=g).clamp_(1, 2000).to(torch.int64)
    indptr = torch.zeros(n_users + 1, dtype=torch.int64, device="cuda")
    indptr[1:] = torch.cumsum(deg, 0)
    nnz = int(indptr[-1])
    cdf = torch.cumsum(1.0 / torch.arange(1, n_items + 1, device="cuda", dtype=torch.float64), 0)
    cdf /= cdf[-1].clone()
    indices = torch.empty(nnz, dtype=torch.int32, device="cuda")
    step = 1 << 26
    for s in range(0, nnz, step):
        e = min(nnz, s + step)
        u = torch.rand(e - s, generator=g, device="cuda", dtype=torch.float64)
        indices[s:e] = torch.searchsorted(cdf, u).clamp_(max=n_items - 1).to(torch.int32)
    return indptr, indices


def side_cost(n_x, n_y, nnz, d, use_cg):
    bytes_ = nnz * (8 + 4 * d) + n_x * 8 * d
    if use_cg:
        flop = (1 + CG_STEPS) * (4 * d * nnz + 2 * d * d * n_x)
    else:
        flop = 2 * d * d * nnz + 2 * d * nnz + n_x * (d ** 3 / 3 + 2 * d * d)
    return bytes_, flop


def rates(sec, bytes_, flop):
    t_hbm, t_fp = bytes_ / HBM_PEAK, flop / FP32_PEAK
    return dict(sec=sec, min_bytes=bytes_, flop=flop, gb_per_s=bytes_ / sec / 1e9, tflop_per_s=flop / sec / 1e12,
                share_of_peak=max(t_hbm, t_fp) / sec, bound="hbm" if t_hbm >= t_fp else "fp32")


def run_scale(scale, reps):
    import torch

    from librecommender_b200.als import RowPlan, gram, solve

    n_users, n_items = int(10_000_000 * scale), int(1_000_000 * scale)
    indptr, indices = make_graph(n_users, n_items)
    nnz = int(indices.numel())
    # the items side: a stable sort by item keeps each item's users in ascending order
    rows = torch.repeat_interleave(torch.arange(n_users, device="cuda", dtype=torch.int32), indptr[1:] - indptr[:-1])
    order = torch.sort(indices, stable=True).indices
    iptr = torch.zeros(n_items + 1, dtype=torch.int64, device="cuda")
    iptr[1:] = torch.cumsum(torch.bincount(indices, minlength=n_items), 0)
    rows_i = rows[order].contiguous()
    del rows
    g = torch.Generator(device="cuda").manual_seed(1)
    rating = torch.randint(1, 6, (nnz,), generator=g, device="cuda").float()
    data = {"ranking": torch.full((nnz,), 11.0, device="cuda"), "rating": rating}
    plans = {}
    for task in ("ranking", "rating"):
        plans[task] = (RowPlan(indptr, indices, data[task], n_items),
                       RowPlan(iptr, rows_i, data[task][order].contiguous(), n_users))
    del order
    deg_i = (iptr[1:] - iptr[:-1])
    out = dict(scale=scale, n_users=n_users, n_items=n_items, nnz=nnz, max_item_degree=int(deg_i.max()),
               long_items=plans["ranking"][1].n_long, long_item_chunks=plans["ranking"][1].n_chunks,
               long_users=plans["ranking"][0].n_long, configs=[])
    for d in (16, 64):
        U = (torch.randn(n_users, d, generator=g, device="cuda") * 0.03).contiguous()
        I = (torch.randn(n_items, d, generator=g, device="cuda") * 0.03).contiguous()
        for task, use_cg in (("ranking", True), ("ranking", False), ("rating", True)):
            implicit = task == "ranking"
            pu, pi = plans[task]
            A0u, A0i = gram(I, 1.0, implicit), gram(U, 1.0, implicit)
            # every timed call starts from the same table: repeated warm-started calls would converge and take
            # the reference's early exits; the restoring copy is timed alone and subtracted
            U0, I0 = U.clone(), I.clone()
            t_users = event_seconds(lambda: (U.copy_(U0), solve(pu, U, I, A0u, implicit, use_cg, CG_STEPS)), reps)
            t_users -= event_seconds(lambda: U.copy_(U0), reps)
            t_items = event_seconds(lambda: (I.copy_(I0), solve(pi, I, U0, A0i, implicit, use_cg, CG_STEPS)), reps)
            t_items -= event_seconds(lambda: I.copy_(I0), reps)
            U.copy_(U0)
            I.copy_(I0)
            del U0, I0
            t_gram_i = event_seconds(lambda: gram(I, 1.0, True), reps)
            t_gram_u = event_seconds(lambda: gram(U, 1.0, True), reps)
            assert torch.isfinite(U).all() and torch.isfinite(I).all()
            rec = dict(d=d, task=task, use_cg=use_cg,
                       users=rates(t_users, *side_cost(n_users, n_items, nnz, d, use_cg)),
                       items=rates(t_items, *side_cost(n_items, n_users, nnz, d, use_cg)),
                       gram_items_table=rates(t_gram_i, n_items * 4 * d, 2 * n_items * d * d),
                       gram_users_table=rates(t_gram_u, n_users * 4 * d, 2 * n_users * d * d))
            rec["epoch_sec"] = t_users + t_items + (t_gram_i + t_gram_u if implicit else 0.0)
            out["configs"].append(rec)
            print(scale, d, task, use_cg, f"users {t_users * 1e3:.2f} ms items {t_items * 1e3:.2f} ms "
                  f"gram {t_gram_i * 1e3:.2f} / {t_gram_u * 1e3:.2f} ms", file=sys.stderr, flush=True)
        del U, I
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scales", default="1.0,0.1")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("profile_als needs a CUDA device")
    res = dict(card=card(), cg_steps=CG_STEPS, reg=1.0, scales=[])
    for s in a.scales.split(","):
        res["scales"].append(run_scale(float(s), a.reps))
        torch.cuda.empty_cache()
    write_report(res, a.out)


if __name__ == "__main__":
    main()
