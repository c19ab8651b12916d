"""Profile Caser / WaveNet training: ``step`` and ``step_graph`` of ``CaserTrainer`` / ``WaveNetTrainer``, the
save-mode forward kernel alone and the encoder backward alone.

    python tools/profile_conv_train.py [--steps 20] [--out results/profile_conv_train.json]

Shapes: the reference default batch (256 rows per step) and the 8192-row batch of the other trainer profiles;
embed_size K = 16, n_users = n_items = 100 000, cross entropy, T in {10, 50}, lengths uniform in [1, T] (end-padded);
Caser (nh 2, nv 4) and (nh 8, nv 8), WaveNet (F 16, 1 block x 4 layers) and (F 64, 2 blocks x 4 layers), dilated.
``step`` / ``step_graph`` are timed with device events over ``--steps`` steps after warm-up.  On the step's own
saved state, CUDA events time the save-mode forward (``b200_caser_train_forward`` / ``b200_wavenet_train_forward``),
the encoder backward (Caser: ``b200_caser_backward``, its three launches; WaveNet: the position kernels
``b200_wavenet_pool_backward``, ``b200_wavenet_layer_inputs``, ``b200_wavenet_layer_dx`` with the ReLU masks and
the dense products between them) and, for WaveNet, the position kernels alone.

Algorithmic FP32 FLOP per row (a multiply-add counts 2), set against the data-sheet 67 TFLOP/s:
  Caser:   forward 2 K nh sum_{h=1..T} (T-h+1) h + 2 T K nv + 2 D K (D = T nh + K nv); the backward routes each
           horizontal column through ONE window: 2 x (2 K nh sum_h h) + 2 x 2 T K nv + 2 x 2 D K.
  WaveNet: forward sum_l 2 T (2 C_l) F + 2 T F F + 2 F K; backward 2 x the forward (dx and dW of every product)."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from _profile_common import FP32_PEAK, card, event_seconds  # noqa: E402


def flop_per_row(model, T, K, nh=0, nv=0, F=0, n_conv=0):
    if model == "Caser":
        D = T * nh + K * nv
        fwd = 2 * K * nh * sum((T - h + 1) * h for h in range(1, T + 1)) + 2 * T * K * nv + 2 * D * K
        bwd = 2 * 2 * K * nh * sum(range(1, T + 1)) + 2 * 2 * T * K * nv + 2 * 2 * D * K
        return fwd + bwd
    fwd = sum(2 * T * 2 * (K if l == 0 else F) * F for l in range(n_conv)) + 2 * T * F * F + 2 * F * K
    return 3 * fwd


def case(model, B, T, steps, nh=2, nv=4, F=16, n_blocks=1, n_layers=4, n_users=100_000, n_items=100_000, K=16):
    import torch

    from librecommender_b200 import _lib
    from librecommender_b200 import synthetic as syn
    from librecommender_b200.training import CaserTrainer, WaveNetTrainer

    rng = np.random.default_rng(1)
    if model == "Caser":
        raw = syn.make_caser_weights(rng, n_users, n_items, K, T, nh, nv)
        tr = CaserTrainer({"n_users": n_users, "n_items": n_items}, raw, lr=1e-3)
    else:
        raw = syn.make_wavenet_weights(rng, n_users, n_items, K, F, n_blocks, n_layers)
        tr = WaveNetTrainer({"n_users": n_users, "n_items": n_items}, raw, lr=1e-3)
    lens = rng.integers(1, T + 1, B)
    seqs = rng.integers(0, n_items, (B, T)).astype(np.int32)
    seqs[np.arange(T)[None, :] >= lens[:, None]] = n_items
    cu = lambda a: torch.as_tensor(a).cuda()      # noqa: E731
    args = [cu(rng.integers(0, n_users, B)), cu(rng.integers(0, n_items, B)), cu(seqs), cu(lens.astype(np.int32)),
            cu((rng.random(B) < 0.5).astype(np.float32))]
    for _ in range(3):
        tr.step(*args)
        tr.step_graph(*args)
    t_step = event_seconds(lambda: tr.step(*args), steps)
    t_graph = event_seconds(lambda: tr.step_graph(*args), steps)
    # the kernels alone, on the step's own saved state
    _, c = tr.user_vectors(args[0], args[2])
    t_fwd = event_seconds(lambda: tr._encode(c), steps)
    dF = torch.randn(c["feat"].shape, device="cuda")
    t_bwd = event_seconds(lambda: tr._encoder_backward(c, dF), steps)
    res = dict(model=model, batch=B, T=T, K=K, step_ms=t_step * 1e3, step_graph_ms=t_graph * 1e3,
               rows_per_s_step=B / t_step, rows_per_s_graph=B / t_graph, fwd_save_ms=t_fwd * 1e3,
               encoder_backward_ms=t_bwd * 1e3, fwd_share_of_graph_step=t_fwd / t_graph,
               encoder_backward_share_of_graph_step=t_bwd / t_graph)
    if model == "Caser":
        res.update(nh=nh, nv=nv)
        flop = B * flop_per_row(model, T, K, nh=nh, nv=nv)
    else:
        L = n_blocks * n_layers
        res.update(F=F, layers=f"{n_blocks}x{n_layers}")
        flop = B * flop_per_row(model, T, K, F=F, n_conv=L)
        S = B * T
        dZ = torch.empty((S, F), device="cuda")
        xin = torch.empty((S, 2 * max(K, F)), device="cuda")
        P = torch.randn((S, 2 * max(K, F)), device="cuda")
        dx = torch.empty((S, max(K, F)), device="cuda")
        st = _lib.current_stream()

        def position_kernels():
            _lib.check(_lib.lib.b200_wavenet_pool_backward(B, T, F, _lib.ptr(dF), F, _lib.ptr(c["arg"]), _lib.ptr(dZ),
                                                           st))
            for l, d in enumerate(tr.dilations):
                C = K if l == 0 else F
                x = c["X0"] if l == 0 else c["ys"][l - 1]
                _lib.check(_lib.lib.b200_wavenet_layer_inputs(_lib.ptr(x), C, B, T, C, d, _lib.ptr(xin), st))
                _lib.check(_lib.lib.b200_wavenet_layer_dx(_lib.ptr(P), B, T, C, d, _lib.ptr(dx), C, st))

        t_pos = event_seconds(position_kernels, steps)
        res.update(position_kernels_ms=t_pos * 1e3, position_kernels_share_of_graph_step=t_pos / t_graph)
    res.update(algorithmic_tflops_graph_step=flop / t_graph / 1e12, fp32_peak_share_graph_step=flop / t_graph / FP32_PEAK)
    return res


CASES = [("Caser", dict(nh=2, nv=4)), ("Caser", dict(nh=8, nv=8)), ("WaveNet", dict(F=16, n_blocks=1, n_layers=4)),
         ("WaveNet", dict(F=64, n_blocks=2, n_layers=4))]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default="results/profile_conv_train.json")
    a = ap.parse_args()
    name = card()
    print(f"card, power.limit, clocks.max.sm: {name}")
    out = dict(card_power_limit_max_sm_clock=name, results=[])
    for B in (256, 8192):
        for model, kw in CASES:
            for T in (10, 50):
                r = case(model, B, T, a.steps, **kw)
                out["results"].append(r)
                print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()}), flush=True)
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
