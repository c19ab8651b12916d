"""Speculative-threshold settings of the fused scorer at the bench shape (C2: 1 M items, d = 64, top-100,
32 768 users per launch, Zipf consumed lists), one JSON line per setting:

* sweep (PRE + guess + MAIN) and whole-call times from CUDA events, and the sweep at the per-phase levels
  0 (normal), 1 (cold epilogue steps only) and 2 (no epilogue) of b200_recommend_embed_debug;
* per-kernel times (pre-pass, guess, main pass, finalize: the warp kernel and the deferred rows' block
  kernel) from torch.profiler, in a run of their own;
* candidate records per row (sum of the row's list lengths, cand_cnt) and rows per row_status code.

    python tools/profile_speculation.py [--settings legacy,16:1e-5,8:1e-5,4:1e-5] [--steps 10] [--out F]

A setting is ``stride:delta`` (b200_recommend_embed_speculation) or ``legacy`` (stride 16, the linear rank
pre_k = 12 + ceil(2 f k_row)).
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bench  # noqa: E402
from _profile_common import card  # noqa: E402

KERNELS = {"pre": "sweep_kernel<true", "guess": "guess_kernel", "main": "sweep_kernel<false",
           "finalize_warp": "finalize_warp_kernel", "finalize": "finalize_kernel", "prep_users": "prep_users_kernel"}


def select(setting):
    from librecommender_b200 import _lib

    if setting == "legacy":
        _lib.check(_lib.lib.b200_recommend_embed_speculation(16, 0.0))
        _lib.check(_lib.lib.b200_recommend_embed_tune(0, 2.0))
        _lib.check(_lib.lib.b200_recommend_embed_debug(-12))
    else:
        stride, delta = setting.split(":")
        _lib.check(_lib.lib.b200_recommend_embed_speculation(int(stride), float(delta)))


def records_per_row(sc, B, K):
    """Sum over a row's candidate lists of cand_cnt after the latest fused call.  The offsets follow
    make_plan's workspace layout (csrc/score_topk_tc.cu): A, meta, tau, guess, status, cnt."""
    plan = sc.fused_plan(B, K)
    al = lambda x: (x + 255) // 256 * 256                      # noqa: E731
    cl = plan["cluster_x10_plus_mma_groups"] // 10
    B_pad = (B + 128 * cl - 1) // (128 * cl) * (128 * cl)
    d_pad = (sc.d + 63) // 64 * 64
    n_lists = 2 * plan["n_splits"]
    off = al(B_pad * d_pad * 2) + al(B_pad * 32) + 3 * al(B_pad * 4)
    ws = sc._ws
    base = (256 - ws.data_ptr() % 256) % 256
    cnt = ws[base + off: base + off + n_lists * B_pad * 4].view(torch.int32).view(n_lists, B_pad)
    rec = cnt[:, :B].sum(0).cpu().numpy()
    c = cnt.cpu().numpy()
    assert (c >= 0).all() and (c <= plan["records_per_list"]).all() and (c[:, B:] == 0).all(), "layout mismatch"
    return rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--settings", default="legacy,16:1e-5,8:1e-5,4:1e-5")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--users", type=int, default=400_000)
    ap.add_argument("--out", default=None)
    own, rest = ap.parse_known_args()
    sys.argv = [sys.argv[0], "--users", str(own.users)] + rest
    args = bench.parse()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    U, I = bench.make_tables(args, dev)
    indptr, idx = bench.make_consumed_csr(args, dev)
    from librecommender_b200 import _lib
    from librecommender_b200.consumed import ConsumedCSR
    from librecommender_b200.engine import EmbedScorer

    sc = EmbedScorer(U, I, args.items, ConsumedCSR.from_device_tensors(indptr, idx), n_users=args.users, device=dev)
    B, K = args.batch, args.topk
    rng = np.random.default_rng(7)
    batches = [torch.from_numpy(rng.choice(args.users, size=B, replace=False).astype(np.int64)).to(dev)
               for _ in range(own.warmup + own.steps)]
    timed = batches[own.warmup:]
    ids_first = None
    lines = []
    for setting in own.settings.split(","):
        select(setting)
        row = {"setting": setting, "card": card(), "plan": sc.fused_plan(B, K)}
        # ---- levels 0 / 1 / 2: sweep time from the C-ABI's events (1, 2: results are wrong, never kept)
        for level in (0, 1, 2):
            _lib.check(_lib.lib.b200_recommend_embed_debug(level))
            try:
                for bt in batches[:own.warmup]:
                    sc.recommend_fused(bt, K, True, False)
                torch.cuda.synchronize()
                sc.events = []
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                status = []
                for bt in timed:
                    status.append(sc.recommend_fused(bt, K, True, False)[2])
                e1.record()
                torch.cuda.synchronize()
                row[f"sweep_ms_level{level}"] = float(np.median([a.elapsed_time(z) for a, z in sc.events]))
                row[f"call_ms_level{level}"] = e0.elapsed_time(e1) / len(timed)
                sc.events = None
                if level == 0:
                    st = torch.cat(status).cpu().numpy()
                    row["status_rows"] = {int(c): int((st == c).sum()) for c in np.unique(st)}
                    row["rows"] = int(st.size)
                    rec = records_per_row(sc, B, K)
                    row["records_per_row_mean"] = float(rec.mean())
                    row["records_per_row_max"] = int(rec.max())
            finally:
                _lib.check(_lib.lib.b200_recommend_embed_debug(0))
        row["hot_steps_ms"] = row["sweep_ms_level0"] - row["sweep_ms_level1"]
        row["cold_epilogue_ms"] = row["sweep_ms_level1"] - row["sweep_ms_level2"]
        # ---- per-kernel times, profiler on, in a run of its own
        from torch.profiler import ProfilerActivity, profile

        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for bt in timed[:3]:
                sc.recommend_fused(bt, K, True, False)
            torch.cuda.synchronize()
        tot = {k: 0.0 for k in KERNELS}
        for ev in prof.key_averages():
            for k, pat in KERNELS.items():
                if pat in ev.key:
                    tot[k] += getattr(ev, "self_device_time_total", 0.0) / 1e3   # us -> ms
        row.update({f"{k}_ms": v / 3 for k, v in tot.items()})
        # ---- results: the repaired device path equals the exact path and every other setting
        ids = sc.recommend_device(timed[-1], K, True, False)
        ex = sc.recommend_exact(timed[-1][:4096], K, True, False)
        row["ids_equal_exact_4096"] = bool((ids[:4096] == ex).all())
        if ids_first is None:
            ids_first = ids
        row["ids_equal_first_setting"] = bool((ids == ids_first).all())
        print(json.dumps(row), flush=True)
        lines.append(row)
    select("0:0")
    if own.out:
        os.makedirs(os.path.dirname(own.out) or ".", exist_ok=True)
        with open(own.out, "w") as f:
            f.write("\n".join(json.dumps(r) for r in lines) + "\n")


if __name__ == "__main__":
    main()
