"""A/B harness for the K4 tuning knobs on one GPU: same tables, same batches, every variant of
(sweep organisation code, speculative rank coefficient, users per launch) timed with CUDA
events (sweep = PRE + guess + MAIN through the C-ABI's event hooks; step = whole call incl. finalize).
    python tools/sweep_variants.py [--users 400000] > variants.jsonl
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench  # noqa: E402


def main():
    sys.argv = [sys.argv[0]] + ["--users", os.environ.get("PROF_USERS", "400000")] + sys.argv[1:]
    args = bench.parse()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    U, I = bench.make_tables(args, dev)
    indptr, idx = bench.make_consumed_csr(args, dev)
    from librecommender_b200 import _lib
    from librecommender_b200.consumed import ConsumedCSR
    from librecommender_b200.engine import EmbedScorer
    import librecommender_b200.engine as eng

    sc = EmbedScorer(U, I, args.items, ConsumedCSR.from_device_tensors(indptr, idx), n_users=args.users, device=dev)
    # organisation code : rank coefficient : users per launch : ablate level (1: cold epilogue steps only,
    # 2: no epilogue) -- the per-phase breakdown of the default and the two-group organisations
    variants = [(w, 2.0, 32768, a) for w in (215, 225, 235) for a in (0, 1, 2)]
    if os.environ.get("VARIANTS"):
        variants = [tuple(float(x) if "." in x else int(x) for x in v.split(":")) for v in os.environ["VARIANTS"].split(",")]
    rng = np.random.default_rng(5)
    steps, warm = 12, 3
    ref_ids = None
    for var in variants:
        w, c, b = var[:3]
        ablate = int(var[3]) if len(var) > 3 else 0
        hint = int(var[4]) if len(var) > 4 else 20000
        margin = 16
        if ablate < 0:                      # negative 4th field = additive margin of the speculative rank
            margin, ablate = -ablate, 0
        _lib.check(_lib.lib.b200_recommend_embed_debug(-margin))
        _lib.check(_lib.lib.b200_recommend_embed_debug(100 + hint))
        _lib.check(_lib.lib.b200_recommend_embed_debug(ablate))
        _lib.check(_lib.lib.b200_recommend_embed_tune(int(w), float(c)))
        eng.FUSED_ROWS_PER_CALL = int(b)
        batches = [torch.from_numpy(rng.choice(args.users, size=int(b), replace=False).astype(np.int64)).to(dev)
                   for _ in range(steps + warm)]
        run = (lambda bt: sc.recommend_fused(bt, args.topk, True, False)[0]) if ablate else \
            (lambda bt: sc.recommend_device(bt, args.topk, True, False))
        for i in range(warm):
            run(batches[i])
        torch.cuda.synchronize()
        sc.events = []
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fb = 0
        for i in range(warm, warm + steps):
            out = run(batches[i])
            fb += sc.last_fallback_rows if not ablate else 0
        e1.record()
        torch.cuda.synchronize()
        sweep = float(np.mean([a.elapsed_time(z) for a, z in sc.events]))
        sc.events = None
        step = e0.elapsed_time(e1) / steps
        flops = 2.0 * args.dim * args.items * b
        # parity spot check of the last batch against the exact path (256 rows)
        ex = sc.recommend_exact(batches[-1][:256], args.topk, True, False)
        same = bool((out[:256] == ex).all())
        print(json.dumps({"ablate": ablate, "margin": margin, "hint_ns": hint, "W": w, "coef": c, "rows_per_launch": b, "sweep_ms": sweep, "step_ms_sync": step,
                          "tflops": flops / sweep / 1e9, "users_per_s_sync": b / step * 1e3,
                          "fallback_rows": fb, "ids_equal_exact_256": same, "plan": sc.fused_plan(b, args.topk)}),
              flush=True)


if __name__ == "__main__":
    main()
