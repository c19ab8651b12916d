"""Time skip-gram training on the GPU (``csrc/skipgram.cu``): per mode and corpus, ms per epoch, tokens/s, pairs/s,
the walk kernel's time, bytes per pair from shapes and the share of HBM bandwidth; plus an in-flight sweep.

    python tools/profile_skipgram.py [--large-users 1000000] [--sweep] [--out /tmp/skipgram.json]

Corpora: C1 (``tests/golden/skipgram.npz``: the consumed lists of the chronological 80 % split of the sample
MovieLens ratings) and a seeded synthetic one: ``--large-users`` users, each ``min(Poisson(50), 500)`` items drawn
Zipf(1.1) over ``--large-items`` items.  Bytes per pair: a row touched is read and written (8 d bytes); NS touches
the context row and 1 + negative target rows, HS adds one syn1 row per code, plus 4-byte ids.  Share of HBM bandwidth
is bytes over the epoch kernel's time over 3.35 TB/s (H100 SXM data sheet), with the card's name and power limit read
in the same run.  Recall@10 on C1 is printed for each in-flight count of the sweep.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def synthetic(n_users, n_items, seed=0):
    g = np.random.default_rng(seed)
    lens = np.minimum(g.poisson(50, n_users), 500)
    tokens = (g.zipf(1.1, int(lens.sum())) - 1) % n_items
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    np.cumsum(lens, out=indptr[1:])
    return indptr, tokens.astype(np.int32), n_items


def timed(fn, reps):
    import torch

    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def profile(name, mode, indptr, tokens, n_items, d, reps, max_inflight=0, counts=None):
    """One corpus and mode; ``counts`` (pairs, kept tokens, mean code length) from an earlier call skips the host
    count of the pairs, which does not depend on the schedule."""
    import torch

    from librecommender_b200 import skipgram as sg

    tr = sg.SkipGramTrainer((indptr, tokens), n_items, mode, embed_size=d, seed=42, n_walks=10, walk_length=10,
                            max_inflight=max_inflight)
    ip, tk = tr.epoch_corpus(1)
    kept, sent, klen = sg.subsample(ip, tk, n_items, tr.tables.keep_thr, 42, 1)
    T = int(ip[-1])
    if counts is None:
        counts = pair_counts(tr, ip, kept, sent, klen)
    pairs, kept_total, codelen = counts
    bytes_pair = (2 + sg.NEGATIVE) * 8 * d + codelen * 8 * d + 4 * (2 + sg.NEGATIVE)
    timed(lambda: sg.epoch(ip, kept, sent, klen, n_items, tr.syn0, tr.syn1neg, tr.syn1, tr.tables, tr.window,
                           sg.ALPHA, sg.MIN_ALPHA, 0, T, 42, 1, max_inflight=max_inflight), 1)   # warm-up
    walk_ms = timed(lambda: tr.epoch_corpus(1), 3) if mode == "deepwalk" else 0.0
    sub_ms = timed(lambda: sg.subsample(ip, tk, n_items, tr.tables.keep_thr, 42, 1), reps)
    ep_ms = timed(lambda: sg.epoch(ip, kept, sent, klen, n_items, tr.syn0, tr.syn1neg, tr.syn1, tr.tables, tr.window,
                                   sg.ALPHA, sg.MIN_ALPHA, 0, T, 42, 1, max_inflight=max_inflight), reps)
    full_ms = timed(lambda: tr.epoch(0, 1), reps)
    torch.cuda.synchronize()
    return dict(corpus=name, mode=mode, d=d, max_inflight=max_inflight, raw_tokens=T, kept_tokens=kept_total,
                pairs=pairs, mean_codelen=codelen, walk_ms=walk_ms, subsample_ms=sub_ms, epoch_kernel_ms=ep_ms,
                epoch_ms=full_ms, tokens_per_s=T / full_ms * 1e3, pairs_per_s=pairs / ep_ms * 1e3,
                bytes_per_pair=bytes_pair, hbm_share=pairs * bytes_pair / (ep_ms * 1e-3) / HBM)


def pair_counts(tr, ip, kept, sent, klen):
    """(pairs, kept tokens, mean Huffman code length of the kept centres) of pass 1, counted on the host."""
    from _skipgram_oracle import reduced_windows

    klen_h, ip_h, sent_h = klen.cpu().numpy(), ip.cpu().numpy(), sent.cpu().numpy()
    slots = np.nonzero(sent_h >= 0)[0]
    b = reduced_windows(slots, tr.window, 42, 1)
    i = slots - ip_h[sent_h[slots]]
    n = klen_h[sent_h[slots]]
    reach = tr.window - b
    pairs = int((np.minimum(n - 1, i + reach) - np.maximum(0, i - reach)).sum())
    codelen = 0.0
    if tr.hs:
        hp = tr.tables.hs_ptr.cpu().numpy()
        kt = kept.cpu().numpy()[slots]
        codelen = float((hp[kt + 1] - hp[kt]).mean())
    return pairs, int(klen_h.sum()), codelen


def c1_quality(mode, epochs, max_inflight, n_walks=10):
    import _skipgram_oracle as orc

    from librecommender_b200 import skipgram as sg

    z = np.load(os.path.join(ROOT, "tests", "golden", "skipgram.npz"))
    ip, it, n_i = z["c1_indptr"], z["c1_items"], int(z["c1_shape"][1])
    tr = sg.SkipGramTrainer((ip, it), n_i, mode, embed_size=16, seed=42, n_walks=n_walks, walk_length=10,
                            max_inflight=max_inflight).fit(epochs)
    U, I = tr.embeddings()
    return orc.ranking_metrics(U.cpu().numpy()[:-1], I.cpu().numpy()[:-1], ip, it, z["eval_users"], z["eval_items"])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--large-users", type=int, default=1_000_000)
    ap.add_argument("--large-items", type=int, default=1_000_000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sweep", action="store_true")
    ap.add_argument("--sweep-only", action="store_true", help="skip the per-corpus table")
    ap.add_argument("--sweep-modes", default="item2vec,deepwalk")
    ap.add_argument("--sweep-warps", default="2,4,8,16,32", help="warps of centre groups per SM")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    from librecommender_b200 import skipgram as sg

    torch.cuda.set_device(0)
    res = dict(card=card(), runs=[], sweep=[], quality=[])
    print(res["card"], file=sys.stderr)
    z = np.load(os.path.join(ROOT, "tests", "golden", "skipgram.npz"))
    c1 = (z["c1_indptr"], z["c1_items"], int(z["c1_shape"][1]))
    big = synthetic(a.large_users, a.large_items)
    print("synthetic corpus:", a.large_users, "users,", int(big[0][-1]), "tokens,", a.large_items, "items",
          file=sys.stderr)
    for name, corpus in () if a.sweep_only else (("C1", c1), (f"synthetic {a.large_users}x{a.large_items}", big)):
        for mode in ("item2vec", "deepwalk"):
            r = profile(name, mode, *corpus, 16, a.reps)
            res["runs"].append(r)
            print(json.dumps(r), file=sys.stderr)
    if a.sweep:
        sms = torch.cuda.get_device_properties(0).multi_processor_count
        for mode in a.sweep_modes.split(","):
            counts = None
            for wps in (int(w) for w in a.sweep_warps.split(",")):
                mi = sms * wps * 8              # d = 16: 4 lanes per centre, 8 centres per warp
                r = profile("synthetic", mode, *big, 16, a.reps, max_inflight=mi, counts=counts)
                counts = (r["pairs"], r["kept_tokens"], r["mean_codelen"])
                q = c1_quality(mode, 10, mi)
                row = dict(mode=mode, warps_per_sm=wps, max_inflight=mi, epoch_kernel_ms=r["epoch_kernel_ms"],
                           pairs_per_s=r["pairs_per_s"], c1_recall10=q[0], c1_ndcg10=q[1])
                res["sweep"].append(row)
                print(json.dumps(row), file=sys.stderr)
        for mode in a.sweep_modes.split(","):
            for mi in (0,):
                q = c1_quality(mode, 10, mi)
                res["quality"].append(dict(mode=mode, max_inflight=mi, recall10=q[0], ndcg10=q[1]))
                print(json.dumps(res["quality"][-1]), file=sys.stderr)
    print("default in flight d=16:", sg._lib.lib.b200_skipgram_default_inflight(16), file=sys.stderr)
    if a.out:
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
