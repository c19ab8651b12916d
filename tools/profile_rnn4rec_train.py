"""Profile RNN4Rec training: ``RNN4RecTrainer.step`` and ``step_graph``, and the two recurrent kernels alone.

    python tools/profile_rnn4rec_train.py [--steps 20] [--out results/profile_rnn4rec_train.json]

Shapes: the reference default batch (256 rows per step) and the C1-like 8192-row batch of the other trainer
profiles; embed_size 16, input width hidden_units[0], n_items 100 000, cross entropy; GRU (16,), GRU (128,) and
LSTM (64, 64) (the Keras graph), T in {10, 50}; lengths uniform in [1, T].  ``step`` / ``step_graph`` are timed with
device events over ``--steps`` steps after warm-up; ``b200_rnn_train_forward`` and ``b200_rnn_backward`` (every
layer) are timed with CUDA events over repeated launches on the step's own saved state.  Algorithmic FP32 FLOP:
3 x the forward's 2 G H (in + H) per valid step and layer (G = 3 for GRU, 4 for LSTM), set against the data-sheet
67 TFLOP/s.  The card name and power limit are read in the same run."""
import argparse
import ctypes
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from _profile_common import FP32_PEAK, card  # noqa: E402


def _events(fn, reps):
    import torch

    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps * 1e-3


def case(rnn_type, hidden, B, T, steps, n_items=100_000, K=16):
    import torch

    from librecommender_b200 import _lib
    from librecommender_b200.synthetic import make_rnn4rec_weights
    from librecommender_b200.training import RNN4RecTrainer

    rng = np.random.default_rng(1)
    raw = make_rnn4rec_weights(rng, n_items, K, hidden, rnn_type, False, "keras")
    tr = RNN4RecTrainer({"n_users": 1, "n_items": n_items}, raw, lr=1e-3)
    lens = rng.integers(1, T + 1, B).astype(np.int32)
    seqs = rng.integers(0, n_items, (B, T)).astype(np.int32)
    seqs[np.arange(T)[None, :] >= lens[:, None]] = n_items
    cu = lambda a: torch.as_tensor(a).cuda()      # noqa: E731
    args = [cu(np.zeros(B, np.int64)), cu(rng.integers(0, n_items, B)), cu(seqs), cu(lens),
            cu((rng.random(B) < 0.5).astype(np.float32))]
    for _ in range(3):
        tr.step(*args)
        tr.step_graph(*args)
    t_step = _events(lambda: tr.step(*args), steps)
    t_graph = _events(lambda: tr.step_graph(*args), steps)
    # the kernels alone, on the step's own saved state
    h, c = tr.encode(args[2], args[3])
    ptrs = [t.data_ptr() if t is not None else None for sv in c["saved"] for t in sv]
    table = (ctypes.c_void_p * len(ptrs))(*ptrs)
    E = tr.params["seq_embeds"]

    def fwd():
        _lib.check(_lib.lib.b200_rnn_train_forward(
            _lib.ptr(c["rows"]), B, _lib.ptr(args[3]), _lib.ptr(args[2]), T, T, _lib.ptr(E), E.stride(0), tr.in_dim,
            len(tr.hidden), tr._kinds, tr._hid, tr._acts, _lib.ptr(tr.rnn_w), _lib.ptr(h), h.stride(0), table,
            _lib.current_stream()))

    bufs = []
    for l, (H, kind) in enumerate(zip(tr.hidden, tr.kinds)):
        GH = (4 if kind == 2 else 3) * H
        bufs.append((torch.empty((B * T, GH), device="cuda"), torch.empty((B * T, GH), device="cuda") if kind == 0
                     else None, torch.randn((B, H), device="cuda"), torch.randn((B * T, H), device="cuda")))

    def bwd():
        for l in range(len(tr.hidden) - 1, -1, -1):
            H, kind = tr.hidden[l], tr.kinds[l]
            d = tr.in_dim if l == 0 else tr.hidden[l - 1]
            dgx, dgh, dout, dy = bufs[l]
            top = l == len(tr.hidden) - 1
            t6 = (ctypes.c_void_p * 6)(*ptrs[6 * l:6 * l + 6])
            _lib.check(_lib.lib.b200_rnn_backward(
                _lib.ptr(c["rows"]), B, _lib.ptr(args[3]), T, kind, d, H, 0, _lib.ptr(tr.rnn_w[tr._offs[l]:]),
                _lib.ptr(dout) if top else None, H, None if top else _lib.ptr(dy), t6, _lib.ptr(dgx), _lib.ptr(dgh),
                None, None, _lib.current_stream()))

    fwd()
    bwd()
    t_fwd = _events(fwd, steps)
    t_bwd = _events(bwd, steps)
    valid = float(np.minimum(lens, T).sum())
    flop, d = 0.0, hidden[0]
    for H in hidden:
        G = 3 if rnn_type == "gru" else 4
        flop += 3 * 2 * G * H * (d + H) * valid
        d = H
    return dict(rnn_type=rnn_type, hidden=list(hidden), batch=B, T=T, step_ms=t_step * 1e3, step_graph_ms=t_graph * 1e3,
                rows_per_s_step=B / t_step, rows_per_s_graph=B / t_graph, fwd_save_ms=t_fwd * 1e3,
                bptt_ms=t_bwd * 1e3, fwd_share_of_graph_step=t_fwd / t_graph, bptt_share_of_graph_step=t_bwd / t_graph,
                algorithmic_tflops_graph_step=flop / t_graph / 1e12,
                fp32_peak_share_graph_step=flop / t_graph / FP32_PEAK)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", default="results/profile_rnn4rec_train.json")
    a = ap.parse_args()
    name = card()
    print(f"card, power.limit, clocks.max.sm: {name}")
    out = dict(card_power_limit_max_sm_clock=name, results=[])
    for B in (256, 8192):
        for rt, hidden in (("gru", (16,)), ("gru", (128,)), ("lstm", (64, 64))):
            for T in (10, 50):
                r = case(rt, hidden, B, T, a.steps)
                out["results"].append(r)
                print(json.dumps({k: (round(v, 4) if isinstance(v, float) else v) for k, v in r.items()}), flush=True)
    os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
