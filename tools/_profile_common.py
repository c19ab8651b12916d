"""What the profiling tools share: the card a run was measured on, CUDA-event timing, the serving timings of a
dynamic-embedding model, and the JSON report."""
import json
import os
import subprocess
import time

import numpy as np

FP32_PEAK = 67e12       # H100 SXM data sheet, dense FP32
HBM_PEAK = 3.35e12      # H100 SXM data sheet, HBM3 bytes/s


def card():
    """``name, power.limit, clocks.max.sm`` of the GPU, as nvidia-smi prints them."""
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def event_seconds(fn, reps):
    """Seconds per call of ``fn`` over ``reps`` calls between two CUDA events, after one warm-up call."""
    import torch

    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / reps


def serving_times(model, n_users, n_items):
    """``set_embeddings`` of ``model`` timed end to end once, then top-100 retrieval without the consumed filter over
    32768 random users on its tables, timed once after a 1024-user warm-up."""
    import torch

    from librecommender_b200.engine import EmbedScorer

    t0 = time.perf_counter()
    U, I = model.set_embeddings()
    torch.cuda.synchronize()
    set_sec = time.perf_counter() - t0
    sc = EmbedScorer(U, I, n_items, None, n_users=n_users)
    users = np.random.default_rng(2).integers(0, n_users, 32768)
    sc.recommend(users[:1024], 100, False)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sc.recommend(users, 100, False)
    torch.cuda.synchronize()
    rec_sec = time.perf_counter() - t0
    return dict(set_embeddings_sec=set_sec, set_embeddings_users_per_s=n_users / set_sec, recommend_users=len(users),
                recommend_sec=rec_sec, recommend_users_per_s=len(users) / rec_sec)


def write_report(res, out):
    """Print ``res`` as indented JSON and, with ``out``, write it there."""
    line = json.dumps(res, indent=1)
    print(line)
    if out:
        os.makedirs(os.path.dirname(out) or ".", exist_ok=True)
        with open(out, "w") as f:
            f.write(line)
