"""Time the Transformer training step on the GPU with CUDA events.

The two shapes of ``tools/profile_transformer.py``: C1-like (6 040 users x 3 200 items, T = 10, K = 16, ids only;
D = 32, hidden (128, 64, 32)) and the one with item features (1 M items, three item sparse fields so D = 80, T = 50,
hidden (128, 64, 32)); one layer, one head, keras graph, trainable positions, BN on.  Rows have len 1 .. T.  For
batches of 2048 and 8192 rows it reports ``TransformerTrainer.step`` and ``step_graph`` time per batch, rows per
second, the algorithmic FLOP per row computed from the shapes (2 FLOP per FMA, every position counted whatever its
len)
    encoder, per layer and position:  forward 24 D^2 + 4 T D (Q / K / V / O, FFN 4D, scores, weighted sum),
                                      backward 48 D^2 + 10 T D (the attention core recomputes the scores)
    target attention, per row:        forward 4 T D, backward 8 T D
    MLP on F K + D inputs, per row:   3 (sum_i 2 H_i H_i+1 + 2 H_last)   (forward + both backward products)
and the attention-core (``b200_transformer_attention_forward`` / ``_backward``, one layer) and target-attention
(``b200_transformer_target_attention`` / ``_backward``) kernels alone.  Prints the card name and power limit read
in the same run.

    python tools/profile_transformer_train.py [--batches 2048,8192] [--json OUT]
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

from profile_transformer import card  # noqa: E402

K, HIDDEN = 16, (128, 64, 32)
SHAPES = {"c1": (6040, 3200, 10, []), "item_features": (100_000, 1_000_000, 50, [200, 1000, 50])}


def event_ms(fn, reps):
    """Mean CUDA-event time of ``fn`` in ms (one warm-up call)."""
    import torch

    fn()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / reps


def flop_per_row(T, D, L, F, dims):
    mlp = sum(2 * a * b for a, b in zip(dims, dims[1:])) + 2 * dims[-1]
    return T * L * (72 * D * D + 14 * T * D) + 12 * T * D + 3 * mlp


def kernel_times(tr, R, T, lens, reps):
    """CUDA-event times (ms) of the attention core (one layer's shapes) and the target attention, forward and
    backward, on random inputs of the trainer's widths."""
    import torch

    from librecommender_b200 import _lib

    D, H = tr.D, tr.H
    hd = D // H
    g = torch.Generator(device="cuda").manual_seed(0)
    q, k, v, do = (torch.randn((R * T, D), device="cuda", generator=g) for _ in range(4))
    o, dq, dk, dv = (torch.empty((R * T, D), device="cuda") for _ in range(4))
    lse = torch.empty(R * H * T, device="cuda")
    Qr, dout = (torch.randn((R, D), device="cuda", generator=g) for _ in range(2))
    su, dqr = torch.empty((R, D), device="cuda"), torch.empty((R, D), device="cuda")
    dS = torch.empty((R * T, D), device="cuda")
    rows = torch.arange(R, device="cuda")
    slots = rows.to(torch.int32)
    sc, P, st = float(np.float32(1.0 / np.sqrt(hd))), _lib.ptr, _lib.current_stream()
    lib = _lib.lib
    out = dict(
        core_forward_ms=event_ms(lambda: _lib.check(lib.b200_transformer_attention_forward(
            P(q), D, P(k), D, P(v), D, P(lens), R, T, H, hd, 0, sc, P(o), D, P(lse), st)), reps),
        core_backward_ms=event_ms(lambda: _lib.check(lib.b200_transformer_attention_backward(
            P(q), D, P(k), D, P(v), D, P(o), D, P(lse), P(do), D, P(lens), R, T, H, hd, 0, sc, P(dq), P(dk), P(dv), D,
            st)), reps),
        target_forward_ms=event_ms(lambda: _lib.check(lib.b200_transformer_target_attention(
            P(Qr), D, P(q), T, D, P(lens), P(slots), P(rows), R, 0, 0, P(su), D, st)), reps),
        target_backward_ms=event_ms(lambda: _lib.check(lib.b200_transformer_target_attention_backward(
            P(Qr), D, P(q), T, D, P(lens), P(dout), D, R, P(dqr), D, P(dS), st)), reps))
    return out


def run(shape, R, reps):
    import torch

    from librecommender_b200 import synthetic as syn
    from librecommender_b200.training import TransformerTrainer

    n_users, n_items, T, item_sparse = SHAPES[shape]
    rng = np.random.default_rng(0)
    spec = syn.make_spec(rng, n_users, n_items, [], item_sparse, 0, 0)
    w = syn.make_transformer_weights(rng, spec, K, 1, 1, T, HIDDEN, True)
    eager = TransformerTrainer(spec, w, lr=1e-3)
    graph = TransformerTrainer(spec, w, lr=1e-3)
    lens = rng.integers(1, T + 1, R).astype(np.int32)
    seqs = rng.integers(0, n_items, (R, T)).astype(np.int32)
    seqs[np.arange(T)[None, :] >= lens[:, None]] = n_items
    cu = lambda a: torch.as_tensor(a, device="cuda")      # noqa: E731
    args = [cu(rng.integers(0, n_users, R)), cu(rng.integers(0, n_items, R)), cu(seqs), cu(lens),
            cu((rng.random(R) < 0.3).astype(np.float32))]
    for _ in range(3):
        eager.step(*args)
        graph.step_graph(*args)
    t_step = event_ms(lambda: eager.step(*args), reps)
    t_graph = event_ms(lambda: graph.step_graph(*args), reps)
    dims = [eager.F * K + eager.D] + list(HIDDEN)
    fl = flop_per_row(T, eager.D, 1, eager.F, dims)
    res = dict(shape=shape, batch=R, T=T, D=eager.D, n_items=n_items, step_ms=t_step, step_graph_ms=t_graph,
               rows_per_s_step=R / t_step * 1e3, rows_per_s_step_graph=R / t_graph * 1e3, flop_per_row=fl,
               tflops_step_graph=fl * R / t_graph / 1e9, launches_per_step=graph.graph_launches_per_step)
    res.update(kernel_times(eager, R, T, args[3], reps))
    del eager, graph
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="2048,8192")
    ap.add_argument("--shapes", default="c1,item_features")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("profile_transformer_train needs a CUDA device")
    name = card()
    out = dict(card_power_limit_max_sm_clock=name, results=[])
    print(f"card, power.limit, clocks.max.sm: {name}")
    for shape in a.shapes.split(","):
        for R in [int(x) for x in a.batches.split(",")]:
            r = run(shape, R, a.reps)
            out["results"].append(r)
            print(f"{shape} batch {R}: step {r['step_ms']:.3f} ms ({r['rows_per_s_step']:.3g} rows/s), step_graph "
                  f"{r['step_graph_ms']:.3f} ms ({r['rows_per_s_step_graph']:.3g} rows/s, {r['tflops_step_graph']:.3g} "
                  f"TFLOP/s algorithmic, {r['flop_per_row']:.3g} FLOP/row); attention core fwd "
                  f"{r['core_forward_ms']:.3f} / bwd {r['core_backward_ms']:.3f} ms, target attention fwd "
                  f"{r['target_forward_ms']:.3f} / bwd {r['target_backward_ms']:.3f} ms")
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
