"""Time the YouTubeRetrieval training step on the GPU with CUDA events.

Two shapes:
* "c1": the reference's defaults on the C1-like sizes of ``tools/profile_autoint.py`` (6 040 users x 3 200 items,
  the user side's sparse / dense fields), B = S = 256, K = 16, hidden (128, 64, K), T = 10;
* "catalogue": 1 M items, B = S = 8192, K = 64, hidden (128, 64, K), T = 10.
For each shape and loss it reports ``YouTubeRetrievalTrainer.step`` and ``step_graph`` time per batch, rows per
second, the algorithmic FLOP per step computed from the shapes
    6 B S H  (logits U W_s^T, dU = dL W_s, dW_s = dL^T U)  +  6 B sum_l din_l dout_l  (the user tower, forward and
    both backward products)
and the sampler (``b200_unique_candidates``) and loss (``b200_sampled_class_loss``) kernels timed alone.  Prints the
card name and power limit read in the same run.

    python tools/profile_youtube_retrieval_train.py [--shapes c1,catalogue] [--json OUT]
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

T = 10
RUNS = {
    # n_users, n_items, user sparse sizes, user dense, B = S, K
    "c1": (SHAPES["c1"][0], SHAPES["c1"][1], SHAPES["c1"][2], SHAPES["c1"][4], 256, 16),
    "catalogue": (20000, 1_000_000, [2, 30, 100, 1000], 1, 8192, 64),
}


def run(shape, loss_type, reps):
    import torch

    from librecommender_b200 import _lib
    from librecommender_b200 import synthetic as syn
    from librecommender_b200.training import YouTubeRetrievalTrainer

    n_users, n_items, us, ud, B, K = RUNS[shape]
    hidden = (128, 64, K)
    rng = np.random.default_rng(0)
    spec = syn.make_spec(rng, n_users, n_items, us, [], ud, 0)
    emb = syn.make_embeddings(rng, spec, K, linear=False)
    din = (1 + len(us) + ud) * K
    w = dict(seq_embeds=syn._glorot(rng, (n_items, K)), item_embeds=syn._glorot(rng, (n_items, K)),
             item_biases=np.zeros(n_items, np.float32), sparse_embeds=emb["sparse_embeds"],
             dense_embeds=emb["dense_embeds"], mlp=syn.make_mlp(rng, din, hidden, True))
    eager = YouTubeRetrievalTrainer(spec, w, loss_type, batch_size=B)
    graph = YouTubeRetrievalTrainer(spec, w, loss_type, batch_size=B)
    users = torch.as_tensor(rng.integers(0, n_users, B), device="cuda")
    items = torch.as_tensor(rng.integers(0, n_items, B), device="cuda")
    lens = torch.as_tensor(rng.integers(0, T + 1, B).astype(np.int32), device="cuda")
    seqs = torch.as_tensor(rng.integers(0, n_items, (B, T)).astype(np.int32), device="cuda")
    seqs = torch.where(torch.arange(T, device="cuda")[None] < lens[:, None], seqs, torch.full_like(seqs, n_items))
    for _ in range(3):
        eager.step(users, items, seqs, lens)
        graph.step_graph(users, items, seqs, lens)
    t_step, _ = timed(lambda: eager.step(users, items, seqs, lens), reps)
    t_graph, _ = timed(lambda: graph.step_graph(users, items, seqs, lens), reps)
    t_sampler, _ = timed(eager.sample, reps)
    logits = torch.randn((B, B), device="cuda") * 0.1
    scratch = logits.clone()
    true = torch.randn(B, device="cuda") * 0.1
    loss, dtrue = torch.empty((), device="cuda"), torch.empty(B, device="cuda")
    ws = torch.empty(int(_lib.lib.b200_sampled_class_loss_workspace_bytes(B, B)), dtype=torch.uint8, device="cuda")
    P = _lib.ptr

    def loss_kernel():
        scratch.copy_(logits)
        _lib.check(_lib.lib.b200_sampled_class_loss(eager.loss_kind, P(scratch), B, B, B, P(true), P(items),
                                                    P(eager.sampled), P(eager.params["item_biases"]), 0, n_items,
                                                    P(eager.num_tries), P(loss), P(dtrue), P(ws), ws.numel(),
                                                    _lib.current_stream()))
    t_copy, _ = timed(lambda: scratch.copy_(logits), reps)
    t_loss, _ = timed(loss_kernel, reps)
    dims = [din] + list(hidden)
    flop = 6 * B * B * K + 6 * B * sum(dims[i] * dims[i + 1] for i in range(len(hidden)))
    return dict(shape=shape, loss=loss_type, n_items=n_items, batch=B, num_sampled=B, K=K, hidden=list(hidden), T=T,
                step_ms=t_step * 1e3, step_graph_ms=t_graph * 1e3, rows_per_s_step=B / t_step,
                rows_per_s_step_graph=B / t_graph, flop_per_step=flop, tflops_step_graph=flop / t_graph / 1e12,
                launches_per_step=graph.graph_launches_per_step, sampler_ms=t_sampler * 1e3,
                loss_kernel_ms=max(t_loss - t_copy, 0.0) * 1e3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="c1,catalogue")
    ap.add_argument("--losses", default="sampled_softmax,nce")
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("profile_youtube_retrieval_train needs a CUDA device")
    name, power = card()
    out = dict(card=name, power_limit_and_max_sm_clock=power, results=[])
    print(f"card: {name}  power.limit, clocks.max.sm: {power}")
    for shape in a.shapes.split(","):
        for loss_type in a.losses.split(","):
            r = run(shape, loss_type, a.reps)
            out["results"].append(r)
            print(f"{shape} {loss_type}: step {r['step_ms']:.3f} ms ({r['rows_per_s_step']:.3g} rows/s), step_graph "
                  f"{r['step_graph_ms']:.3f} ms ({r['rows_per_s_step_graph']:.3g} rows/s, {r['tflops_step_graph']:.3g} "
                  f"TFLOP/s algorithmic), sampler {r['sampler_ms']:.3f} ms, loss kernel {r['loss_kernel_ms']:.3f} ms")
    print(json.dumps(out))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
