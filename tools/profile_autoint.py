"""Time AutoInt all-items recommendation (top-100, consumed filter on) on the GPU with CUDA events.

Two seeded shapes, both with the reference's default AutoInt (att_embed_size (8, 8, 8), 2 heads, residual, K 16):
* c1:      ~6 K users x ~3.2 K items, the fields of examples/feat_ranking_example.py (user: sex, occupation, age;
           item: genre1..3) -> F = 8;
* serving: 1 M items, 4 user + 3 item sparse fields, 1 dense field -> F = 10.
Reports users/s, pairs/s and the algorithmic FLOP per pair
    sum_l [2 F K 3 D_l + 4 F^2 D_l + 2 F D_l K] + 2 F K
as a share of the H100 SXM data-sheet FP32 rate (67 TFLOP/s; the data-sheet figure, not a measured peak).  In the
same run it times rows mode (the [b*N, F*K] concat materialised, then b200_autoint_rows) against grid mode
(b200_autoint_grid) on the same users and checks their scores are bit-equal.  Prints the card name and power limit.

    python tools/profile_autoint.py [--shapes c1,serving] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FP32_DATASHEET = 67e12

SHAPES = {
    # n_users, n_items, user sparse sizes, item sparse sizes, user dense, item dense, users timed per call, rows-vs-grid users
    "c1": (6040, 3200, [2, 21], [18, 18, 18], 1, 0, 6040, 64),
    "serving": (20000, 1_000_000, [2, 30, 100, 1000], [50, 200, 20], 1, 0, 64, 2),
}


def flop_per_pair(F, K, dims):
    return sum(2 * F * K * 3 * D + 4 * F * F * D + 2 * F * D * K for D in dims) + 2 * F * K


def card():
    import torch

    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        power = out[torch.cuda.current_device()] if out else "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def timed(fn, reps):
    import torch

    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    s.record()
    for _ in range(reps):
        out = fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / 1e3 / reps, out


def run_shape(name, reps):
    import torch

    from librecommender_b200 import synthetic as syn
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.consumed import ConsumedCSR
    from librecommender_b200.feat_models import AutoInt

    nu, ni, us, its, ud, idn, b_time, b_cmp = SHAPES[name]
    rng = np.random.default_rng(2024)
    spec = syn.make_spec(rng, nu, ni, us, its, ud, idn)
    K = 16
    w = wio.autoint_weights(syn.make_autoint_weights(rng, spec, K, (8, 8, 8), 2, True, "keras"))
    lens = rng.integers(1, 60, size=nu)
    indptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    idx = rng.integers(0, ni, size=int(indptr[-1])).astype(np.int32)
    model = AutoInt(spec, w, ConsumedCSR(indptr, idx))
    F = model.F
    dims = [model.num_heads * hd for hd in model.head_dims]
    users = rng.choice(nu, size=b_time, replace=False)
    model.recommend(users[: min(8, b_time)], 100, True)          # warm-up: modules, item-side block, workspaces
    model.recommend(users, 100, True)
    t, _ = timed(lambda: model.recommend(users, 100, True), reps)
    pairs = b_time * ni
    fpp = flop_per_pair(F, K, dims)
    res = dict(shape=name, n_users_timed=int(b_time), n_items=ni, F=F, K=K, heads=model.num_heads,
               head_dims=model.head_dims, seconds_per_call=t, users_per_s=b_time / t, pairs_per_s=pairs / t,
               flop_per_pair=fpp, fp32_datasheet_share=pairs / t * fpp / FP32_DATASHEET)
    # rows mode (materialised concat) vs grid mode on the same users
    u = torch.as_tensor(users[:b_cmp], device=model.device)
    grid = lambda: model.score_all_items(u)                                          # noqa: E731
    rows = lambda: model._forward(model.spec.layout, u, None, b_cmp * ni, ni).view(b_cmp, ni)  # noqa: E731
    grid(), rows()
    tg, sg = timed(grid, reps)
    tr, sr = timed(rows, reps)
    res.update(cmp_users=int(b_cmp), grid_seconds=tg, rows_seconds=tr, grid_pairs_per_s=b_cmp * ni / tg,
               rows_pairs_per_s=b_cmp * ni / tr, grid_equals_rows=bool(torch.equal(sg, sr)))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c1,serving")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("profile_autoint.py measures on a CUDA device; none is available")
    name, power = card()
    out = dict(card=name, power_limit_and_max_sm_clock=power, results=[])
    print(f"card: {name}  power.limit, clocks.max.sm: {power}")
    for s in a.shapes.split(","):
        r = run_shape(s, a.reps)
        out["results"].append(r)
        print(f"[{s}] F={r['F']} K={r['K']} H={r['heads']} hd={r['head_dims']}  recommend top-100: "
              f"{r['users_per_s']:.1f} users/s, {r['pairs_per_s'] / 1e6:.1f} M pairs/s, {r['flop_per_pair']} FLOP/pair "
              f"= {100 * r['fp32_datasheet_share']:.1f}% of the 67 TFLOP/s FP32 data-sheet rate")
        print(f"[{s}] {r['cmp_users']} users x {r['n_items']} items: grid {r['grid_seconds'] * 1e3:.2f} ms "
              f"({r['grid_pairs_per_s'] / 1e6:.1f} M pairs/s), rows {r['rows_seconds'] * 1e3:.2f} ms "
              f"({r['rows_pairs_per_s'] / 1e6:.1f} M pairs/s), bit-equal: {r['grid_equals_rows']}")
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)
    if not all(r["grid_equals_rows"] for r in out["results"]):
        raise SystemExit("grid and rows scores differ")


if __name__ == "__main__":
    main()
