"""Profile SIM training: ``step`` and ``step_graph`` of ``SIMTrainer`` and the SIM training kernels alone.

    python tools/profile_sim_train.py [--steps 20] [--out results/profile_sim_train.json]

Shapes: the reference defaults (K = 16, L = 100, S = 10, search_topk = 10, 2 heads, hidden (200, 80), BN on, keras
attention, cross entropy) at the reference batch (256 positives with 1 negative each: 512 rows) and at 8192 rows;
100 000 users and items, ids only; long lengths uniform in [1, L], short lengths in [1, S].  ``step`` / ``step_graph``
are timed with device events over ``--steps`` steps after warm-up.  On the step's own state, CUDA events time
``b200_sim_gsu_forward``, ``b200_sim_esu_forward`` + ``b200_sim_esu_backward`` and ``b200_sim_long_backward``.

Algorithmic FP32 FLOP of a step (a multiply-add counts 2; the backward of every product counted as twice its
forward, so a step is 3x the forward), set against the data-sheet 67 TFLOP/s:
  per step:  Gp = G Wp over all n_items + 1 rows: 2 (N + 1) K' K;
  per row:   GSU 2 L K + pooled L K; ESU 2 K^2 (Wq) + 2 (2 k K^2) (Wk, Wv) + 4 k K (logits, mix) + 2 K^2 (Wo);
             short attention 4 S K; the two dense_nn stacks 2 (d_in h1 + h1 h2 + h2) with d_in = 2K and (F + 2) K."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from _profile_common import FP32_PEAK, card, event_seconds  # noqa: E402

K, L, S, TOPK, HEADS, HIDDEN = 16, 100, 10, 10, 2, (200, 80)


def step_flop(R, n_items, F=2):
    Kp = K
    mlp = lambda d: 2 * (d * HIDDEN[0] + HIDDEN[0] * HIDDEN[1] + HIDDEN[1])       # noqa: E731
    row = (2 * L * K + L * K + 2 * K * K + 4 * TOPK * K * K + 4 * TOPK * K + 2 * K * K + 4 * S * K + mlp(2 * K) +
           mlp((F + 2) * K))
    return 3 * (2 * (n_items + 1) * Kp * K + R * row)


def case(R, steps, n_users=100_000, n_items=100_000):
    import torch

    from librecommender_b200 import _lib
    from librecommender_b200 import synthetic as syn
    from librecommender_b200.feat_models import ACT_NONE, linear
    from librecommender_b200.training import SIMTrainer

    rng = np.random.default_rng(1)
    spec = syn.make_spec(rng, n_users, n_items, [], [], 0, 0)
    w = syn.make_sim_weights(rng, spec, K, HEADS, HIDDEN, True, "keras")
    tr = SIMTrainer(spec, w, search_topk=TOPK, lr=1e-3)
    ll, sl = rng.integers(1, L + 1, R), rng.integers(1, S + 1, R)
    ls = rng.integers(0, n_items, (R, L)).astype(np.int32)
    ss = rng.integers(0, n_items, (R, S)).astype(np.int32)
    ls[np.arange(L)[None, :] >= ll[:, None]] = n_items
    ss[np.arange(S)[None, :] >= sl[:, None]] = n_items
    cu = lambda a: torch.as_tensor(a).cuda()      # noqa: E731
    args = [cu(rng.integers(0, n_users, R)), cu(rng.integers(0, n_items, R)), cu(ls), cu(ll.astype(np.int32)), cu(ss),
            cu(sl.astype(np.int32)), cu((rng.random(R) < 0.5).astype(np.float32))]
    for _ in range(3):
        tr.step(*args)
        tr.step_graph(*args)
    t_step = event_seconds(lambda: tr.step(*args), steps)
    t_graph = event_seconds(lambda: tr.step_graph(*args), steps)
    # the kernels alone, on the step's own state
    tr.forward(*[a.to(torch.int64) if i < 2 else a for i, a in enumerate(args[:6])])
    c = tr._cache
    Gp = linear(c["G"], tr.params["seq_projT"], None, ACT_NONE, impl="f32")
    lib, st = _lib.lib, _lib.current_stream()
    sel = c["sel"]
    pooled = torch.empty((R, K), device="cuda")
    items, lsd, lld = c["items"], c["long_seqs"], c["long_lens"]

    def gsu():
        _lib.check(lib.b200_sim_gsu_forward(_lib.ptr(Gp), K, K, _lib.ptr(items), _lib.ptr(lsd), L, _lib.ptr(lld), L,
                                            TOPK, R, _lib.ptr(sel), _lib.ptr(pooled), K, st))

    m = c["mha"]
    O, P = torch.empty((R, K), device="cuda"), torch.empty(R * HEADS * TOPK, device="cuda")
    dO = torch.randn((R, K), device="cuda")
    dQ, dKs, dVs = torch.empty((R, K), device="cuda"), *(torch.empty((R * TOPK, K), device="cuda") for _ in range(2))

    def esu():
        _lib.check(lib.b200_sim_esu_forward(_lib.ptr(m["q"]), K, _lib.ptr(m["k"]), _lib.ptr(m["v"]), K, _lib.ptr(sel),
                                            _lib.ptr(lld), R, K, HEADS, TOPK, _lib.ptr(O), K, _lib.ptr(P), st))
        _lib.check(lib.b200_sim_esu_backward(_lib.ptr(m["q"]), K, _lib.ptr(m["k"]), _lib.ptr(m["v"]), K, _lib.ptr(sel),
                                             _lib.ptr(lld), R, K, HEADS, TOPK, _lib.ptr(P), _lib.ptr(dO), K,
                                             _lib.ptr(dQ), K, _lib.ptr(dKs), _lib.ptr(dVs), K, st))

    dGp = torch.zeros((n_items + 1, K), device="cuda")
    dp = torch.randn((R, K), device="cuda")

    def long_bwd():
        _lib.check(lib.b200_sim_long_backward(_lib.ptr(lsd), L, _lib.ptr(lld), L, _lib.ptr(sel), TOPK, R, K,
                                              _lib.ptr(dp), K, _lib.ptr(dKs), K, _lib.ptr(dGp), K, st))

    t_gsu, t_esu, t_long = (event_seconds(f, steps) for f in (gsu, esu, long_bwd))
    flop = step_flop(R, n_items)
    return dict(rows=R, K=K, L=L, S=S, topk=TOPK, heads=HEADS, hidden=list(HIDDEN), n_items=n_items,
                step_ms=t_step * 1e3, step_graph_ms=t_graph * 1e3, rows_per_s_step=R / t_step,
                rows_per_s_graph=R / t_graph, gsu_ms=t_gsu * 1e3, esu_fwd_bwd_ms=t_esu * 1e3,
                long_backward_ms=t_long * 1e3, kernels_share_of_graph_step=(t_gsu + t_esu + t_long) / t_graph,
                algorithmic_tflops_graph_step=flop / t_graph / 1e12, fp32_peak_share_graph_step=flop / t_graph / FP32_PEAK)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default="results/profile_sim_train.json")
    a = ap.parse_args()
    name = card()
    print(f"card, power.limit, clocks.max.sm: {name}")
    out = dict(card_power_limit_max_sm_clock=name, results=[])
    for R in (512, 8192):
        r = case(R, a.steps)
        out["results"].append(r)
        print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()}), flush=True)
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
