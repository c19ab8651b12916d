"""Time the AutoInt training step on the GPU with CUDA events.

The C1-like shape of ``tools/profile_autoint.py`` (MovieLens-1M sizes, F = 8 fields, K = 16) with the reference's
default AutoInt (att_embed_size (8, 8, 8), 2 heads, residual, keras graph), batches of 2048 and 8192 rows.
For each batch size it reports ``AutoIntTrainer.step`` and ``step_graph`` time per batch, rows per second, the
algorithmic FLOP per row computed from the shapes
    forward  sum_l [6 F K D_l + 4 F^2 D_l + 2 F D_l K] + 2 F K
    backward sum_l [12 F K D_l + 10 F^2 D_l + 4 F D_l K] + 4 F K
(projections, scores + weighted sum, output projection, Dense(1); the backward recomputes the scores), and the
attention-core kernels alone (``b200_autoint_attention_forward`` / ``_backward`` on one layer's shapes).  Prints the
card name and power limit read in the same run.

    python tools/profile_autoint_train.py [--batches 2048,8192] [--json OUT]
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from profile_autoint import SHAPES, card, timed  # noqa: E402

K, H, ATT = 16, 2, (8, 8, 8)


def flop_per_row(F, K, dims):
    fwd = sum(6 * F * K * D + 4 * F * F * D + 2 * F * D * K for D in dims) + 2 * F * K
    bwd = sum(12 * F * K * D + 10 * F * F * D + 4 * F * D * K for D in dims) + 4 * F * K
    return fwd + bwd


def core_times(R, F, hd, reps):
    """CUDA-event time of the attention forward and backward kernels on one layer's shapes (R rows)."""
    import torch

    from librecommender_b200 import _lib

    D = H * hd
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v, do = (torch.randn((R * F, D), device="cuda", generator=g) for _ in range(4))
    o, dq, dk, dv = (torch.empty((R * F, D), device="cuda") for _ in range(4))
    lse = torch.empty(R * H * F, device="cuda")
    sc, P = float(1.0 / np.sqrt(hd)), _lib.ptr

    def fwd():
        _lib.check(_lib.lib.b200_autoint_attention_forward(P(q), D, P(k), D, P(v), D, R, F, H, hd, sc, P(o), D, P(lse),
                                                           _lib.current_stream()))

    def bwd():
        _lib.check(_lib.lib.b200_autoint_attention_backward(P(q), D, P(k), D, P(v), D, P(o), D, P(lse), P(do), D, R, F,
                                                            H, hd, sc, P(dq), P(dk), P(dv), D, _lib.current_stream()))

    fwd()
    bwd()
    return timed(fwd, reps)[0], timed(bwd, reps)[0]


def run(R, reps):
    import torch

    from librecommender_b200 import synthetic as syn
    from librecommender_b200.training import AutoIntTrainer

    n_users, n_items, us, is_, ud, id_ = SHAPES["c1"][:6]
    rng = np.random.default_rng(0)
    spec = syn.make_spec(rng, n_users, n_items, us, is_, ud, id_)
    w = syn.make_autoint_weights(rng, spec, K, ATT, H, True, "keras")
    eager = AutoIntTrainer(spec, w, lr=1e-3)
    graph = AutoIntTrainer(spec, w, lr=1e-3)
    F = eager.F
    users = torch.as_tensor(rng.integers(0, n_users, R), device="cuda")
    items = torch.as_tensor(rng.integers(0, n_items, R), device="cuda")
    labels = torch.as_tensor((rng.random(R) < 0.3).astype(np.float32), device="cuda")
    for _ in range(3):
        eager.step(users, items, labels)
        graph.step_graph(users, items, labels)
    t_step, _ = timed(lambda: eager.step(users, items, labels), reps)
    t_graph, _ = timed(lambda: graph.step_graph(users, items, labels), reps)
    t_fwd, t_bwd = core_times(R, F, ATT[0], reps)
    fl = flop_per_row(F, K, [H * hd for hd in ATT])
    return dict(batch=R, F=F, K=K, heads=H, att_embed_size=list(ATT), step_ms=t_step * 1e3, step_graph_ms=t_graph * 1e3,
                rows_per_s_step=R / t_step, rows_per_s_step_graph=R / t_graph, flop_per_row=fl,
                tflops_step_graph=fl * R / t_graph / 1e12, launches_per_step=graph.graph_launches_per_step,
                core_forward_ms_per_layer=t_fwd * 1e3, core_backward_ms_per_layer=t_bwd * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="2048,8192")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("profile_autoint_train needs a CUDA device")
    name, power = card()
    out = dict(card=name, power_limit_and_max_sm_clock=power, results=[])
    print(f"card: {name}  power.limit, clocks.max.sm: {power}")
    for R in [int(x) for x in a.batches.split(",")]:
        r = run(R, a.reps)
        out["results"].append(r)
        print(f"batch {R}: step {r['step_ms']:.3f} ms ({r['rows_per_s_step']:.3g} rows/s), step_graph "
              f"{r['step_graph_ms']:.3f} ms ({r['rows_per_s_step_graph']:.3g} rows/s, {r['tflops_step_graph']:.3g} "
              f"TFLOP/s algorithmic), attention core per layer: forward {r['core_forward_ms_per_layer']:.3f} ms, "
              f"backward {r['core_backward_ms_per_layer']:.3f} ms")
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
