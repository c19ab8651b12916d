"""Profile Caser / WaveNet serving: the encoder kernel, ``set_embeddings`` over every user, then all-items top-100
retrieval on its tables.

    python tools/profile_conv_encoders.py [--users 10000000] [--items 1000000] [--out results/profile_conv.json]

Shape: C2 (10 M users, 1 M items, embed_size K = 32, so the serving width is d = 2K + 1 = 65) at T = 10 and 50,
histories of uniform length in [0, T] right-padded with the pad id.  Cases: the reference defaults (Caser nh = 2,
nv = 4; WaveNet 16 filters, 1 block of 4 layers) and one wider case per model (Caser nh = nv = 8; WaveNet 64
filters, 2 blocks of 4).  The encoder kernel (``b200_caser_encode`` / ``b200_wavenet_encode``) is timed with CUDA
events over repeated launches on one 1 M-user chunk after a warm-up launch; ``set_embeddings`` (OOV row, encoder,
Dense head, user rows, serving tables) is timed end to end once, and top-100 retrieval over 32768 users once after a
warm-up.  Algorithmic FLOP per user: Caser 2 K nh T(T+1)(T+2)/6 + 2 T K nv, WaveNet 2 T F (2 C_in) per causal layer
+ 2 T F F for the 1x1 layer, plus the Dense head 2 D K; set against the data-sheet FP32 rate (67 TFLOP/s).  Bytes:
the gathered rows 4 T K, the sequence row 4 T and the feature row 4 D per user (the weights stay in L2), set against
the data-sheet 3.35 TB/s.  The card name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from _profile_common import FP32_PEAK, HBM_PEAK, card, event_seconds, serving_times, write_report  # noqa: E402

CASES = [("Caser", "default", dict(nh_filters=2, nv_filters=4)), ("Caser", "wide", dict(nh_filters=8, nv_filters=8)),
         ("WaveNet", "default", dict(n_filters=16, n_blocks=1, n_layers_per_block=4)),
         ("WaveNet", "wide", dict(n_filters=64, n_blocks=2, n_layers_per_block=4))]


def algorithmic_flop(model, T, K, cfg):
    """(encoder FLOP, head FLOP, pre-head width D) per user."""
    if model == "Caser":
        nh, nv = cfg["nh_filters"], cfg["nv_filters"]
        D = T * nh + K * nv
        return 2.0 * K * nh * T * (T + 1) * (T + 2) / 6 + 2.0 * T * K * nv, 2.0 * D * K, D
    F, L = cfg["n_filters"], cfg["n_blocks"] * cfg["n_layers_per_block"]
    enc = sum(2.0 * T * F * 2 * (K if i == 0 else F) for i in range(L)) + 2.0 * T * F * F
    return enc, 2.0 * F * K, F


def case(model_name, label, cfg, n_users, n_items, T, K, seqs, lens, chunk, reps):
    import torch

    from librecommender_b200.feat_models import Caser, WaveNet
    from librecommender_b200.synthetic import make_caser_weights, make_wavenet_weights

    rng = np.random.default_rng(1)
    if model_name == "Caser":
        raw = make_caser_weights(rng, n_users, n_items, K, T, **cfg)
        model = Caser({"n_users": n_users, "n_items": n_items}, raw, seqs, lens)
    else:
        raw = make_wavenet_weights(rng, n_users, n_items, K, **cfg)
        model = WaveNet({"n_users": n_users, "n_items": n_items}, raw, seqs, lens)
    del raw
    ids = torch.arange(min(chunk, n_users), dtype=torch.int64, device=model.device)
    sec = event_seconds(lambda: model.encode(ids), reps)
    n = ids.numel()
    enc_flop, head_flop, D = algorithmic_flop(model_name, T, K, cfg)
    flop = enc_flop * n
    nbytes = n * (4.0 * T * K + 4.0 * T + 4.0 * D)
    serving = serving_times(model, n_users, n_items)
    f_share, b_share = flop / sec / FP32_PEAK, nbytes / sec / HBM_PEAK
    out = dict(model=model_name, case=label, T=T, config=cfg, pre_head_width=D,
               serving_width=int(model.item_embeds.shape[1]) + 1,
               encode_users=n, encode_sec=sec, encode_users_per_s=n / sec, encoder_flop_per_user=enc_flop,
               head_flop_per_user=head_flop, flop_per_s=flop / sec, share_fp32_peak=f_share, bytes_per_s=nbytes / sec,
               share_hbm_peak=b_share, bound="compute" if f_share >= b_share else "memory", **serving)
    del model
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=10_000_000)
    ap.add_argument("--items", type=int, default=1_000_000)
    ap.add_argument("--T", type=int, nargs="+", default=[10, 50])
    ap.add_argument("--K", type=int, default=32)
    ap.add_argument("--chunk", type=int, default=1 << 20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    res = {"card": card(), "users": args.users, "items": args.items, "K": args.K, "cases": []}
    n = args.users
    for T in args.T:
        rng = np.random.default_rng(T)
        lens = rng.integers(0, T + 1, size=n + 1).astype(np.int32)
        lens[n] = 1
        seqs = rng.integers(0, args.items, size=(n + 1, T), dtype=np.int32)
        seqs[np.arange(T)[None, :] >= lens[:, None]] = args.items
        for model_name, label, cfg in CASES:
            r = case(model_name, label, cfg, n, args.items, T, args.K, seqs, lens, args.chunk, args.reps)
            print(json.dumps(r), flush=True)
            res["cases"].append(r)
        del seqs, lens
    write_report(res, args.out)


if __name__ == "__main__":
    main()
