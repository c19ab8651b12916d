"""Profile RNN4Rec serving: ``set_embeddings`` over every user, then all-items top-100 retrieval on its tables.

    python tools/profile_rnn4rec.py [--users 10000000] [--items 1000000] [--out results/profile_rnn4rec.json]

Shape: C2 (10 M users, 1 M items, T = 10, embed_size 16), lengths uniform in [0, T].  Cases: GRU and LSTM (the
Keras graph) with hidden_units (16,) (the reference default), (128,) and (64, 64).  The encoder kernel
``b200_rnn_encode`` is timed with CUDA events over repeated launches of one 1 M-user chunk after a warm-up launch;
``set_embeddings`` (encoder, Dense head, serving tables) is timed end to end once.  Algorithmic FLOP:
2 G H (in + H) per user, layer and valid step (G = 3 for GRU, 4 for LSTM), set against the data-sheet FP32 rate
(67 TFLOP/s).  Bytes: the gathered input rows, the sequence rows and the output rows (the weights stay in L2), set
against the data-sheet 3.35 TB/s.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from _profile_common import FP32_PEAK, HBM_PEAK, card, event_seconds, serving_times, write_report  # noqa: E402


def case(rnn_type, hidden, n_users, n_items, T, K, seqs, lens, chunk, reps):
    import torch

    from librecommender_b200.feat_models import RNN4Rec
    from librecommender_b200.synthetic import make_rnn4rec_weights

    rng = np.random.default_rng(1)
    raw = make_rnn4rec_weights(rng, n_items, K, hidden, rnn_type, False, "keras")
    model = RNN4Rec({"n_users": n_users, "n_items": n_items}, raw, seqs, lens)
    ids = torch.arange(min(chunk, n_users), dtype=torch.int64, device=model.device)
    sec = event_seconds(lambda: model.encode(ids), reps)
    n = ids.numel()
    valid = float(lens[:n].clip(0, T).sum())
    G = 3 if rnn_type == "gru" else 4
    flop, d = 0.0, hidden[0]
    for H in hidden:
        flop += 2.0 * G * H * (d + H) * valid
        d = H
    nbytes = valid * hidden[0] * 4 + n * T * 4 + n * hidden[-1] * 4
    serving = serving_times(model, n_users, n_items)
    f_share, b_share = flop / sec / FP32_PEAK, nbytes / sec / HBM_PEAK
    out = dict(rnn_type=rnn_type, hidden_units=list(hidden), encode_users=n, encode_sec=sec, encode_users_per_s=n / sec,
               flop_per_s=flop / sec, share_fp32_peak=f_share, bytes_per_s=nbytes / sec, share_hbm_peak=b_share,
               bound="compute" if f_share >= b_share else "memory", **serving)
    del model
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=10_000_000)
    ap.add_argument("--items", type=int, default=1_000_000)
    ap.add_argument("--T", type=int, default=10)
    ap.add_argument("--K", type=int, default=16)
    ap.add_argument("--chunk", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card(), "users": args.users, "items": args.items, "T": args.T, "K": args.K, "cases": []}
    rng = np.random.default_rng(0)
    n, T = args.users, args.T
    lens = rng.integers(0, T + 1, size=n + 1).astype(np.int32)
    lens[n] = 1
    seqs = rng.integers(0, args.items, size=(n + 1, T), dtype=np.int32)
    seqs[np.arange(T)[None, :] >= lens[:, None]] = args.items
    for rnn_type in ("gru", "lstm"):
        for hidden in ((16,), (128,), (64, 64)):
            r = case(rnn_type, hidden, n, args.items, T, args.K, seqs, lens, args.chunk, args.reps)
            print(json.dumps(r), flush=True)
            res["cases"].append(r)
    write_report(res, args.out)


if __name__ == "__main__":
    main()
