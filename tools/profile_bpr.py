"""Profile BPR training epochs (``csrc/bpr.cu``) on a C5-like interaction graph, and the schedule on C1.

    python tools/profile_bpr.py [--scale 1.0] [--reps 2] [--out results/bpr.json]

C5-like graph (seeded, the generator of ``tools/profile_als.py``): 10 M users x 1 M items at scale 1.0, user degrees
min(Poisson(50), 2000), items from Zipf(1.0), about 5e8 interactions; rows are then sorted and de-duplicated (the
canonical CSR the sampler needs), and every interaction is one training sample, in a random order.  For each
optimizer at embed_size 16 and 64, CUDA events time one epoch at the default schedule after a warm-up epoch
(``--c5-sweep``: at embed_size 16 also at the C5_INFLIGHT schedules); each configuration starts from fresh
tables and zero state and reports whether the tables stay finite (lr 0.01, reg 0).

Bytes per sample (the compulsory traffic, from shapes): the ids (8), the user's CSR bounds (16) and the binary
search's probes (4 per probe, ceil(log2(c_u + 1)) probes averaged over the samples), three table rows of 4 D bytes
read and added (2 x 3 x 4 D), and the same again per optimizer state table (momentum 1, adam 2).  The share of peak
is bytes / 3.35 TB/s over the measured time.

C1 (``tests/golden/bpr.npz``: the chronological 80 % split of the sample MovieLens data): three epochs from the
reference's initial tables at the golden learning rates, for max_inflight in {1, 16, 64, 256, 1024, 4096, 16384,
the default and the full occupancy}; each row reports the epoch time and recall@10 / ndcg@10 on the 20 % split.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tests"))

from _profile_common import HBM_PEAK, card, event_seconds, write_report  # noqa: E402

OPTIMIZERS = ("sgd", "momentum", "adam")
STATE_TABLES = {"sgd": 0, "momentum": 1, "adam": 2}
C1_INFLIGHT = (1, 16, 64, 256, 1024, 4096, 16384)
C5_INFLIGHT = (528, 2112, 8448, 33792)       # 1, 4, 16 and 64 warps of 8-lane groups per SM of an H100 SXM


def canonical_graph(n_users, n_items):
    """Users CSR with sorted duplicate-free rows, and the row of every nnz (int32)."""
    import torch

    from profile_als import make_graph

    indptr, indices = make_graph(n_users, n_items)
    rows = torch.repeat_interleave(torch.arange(n_users, device="cuda", dtype=torch.int64), indptr[1:] - indptr[:-1])
    key = rows * n_items + indices.to(torch.int64)
    del rows, indices, indptr
    key = torch.unique(key)                 # sorted and de-duplicated
    users = (key // n_items).to(torch.int32)
    items = (key % n_items).to(torch.int32)
    del key
    indptr = torch.zeros(n_users + 1, dtype=torch.int64, device="cuda")
    indptr[1:] = torch.cumsum(torch.bincount(users, minlength=n_users), 0)
    return indptr, items, users


def search_bytes(indptr):
    """Mean bytes of the negative draw's CSR reads per sample (a user of degree c is sampled c times)."""
    import torch

    deg = (indptr[1:] - indptr[:-1]).double()
    probes = torch.ceil(torch.log2(deg + 1))
    return 16 + 4 * float((deg * probes).sum() / deg.sum())


def bytes_per_sample(D, opt, search):
    return 8 + search + 2 * 3 * 4 * D * (1 + STATE_TABLES[opt])


def run_c5(scale, reps, sweep):
    import torch

    from librecommender_b200 import _lib
    from librecommender_b200.bpr import _launch

    n_users, n_items = int(10_000_000 * scale), int(1_000_000 * scale)
    indptr, indices, users = canonical_graph(n_users, n_items)
    n = int(indices.numel())
    g = torch.Generator(device="cuda").manual_seed(3)
    perm = torch.randperm(n, generator=g, device="cuda")
    s_users, s_items = users[perm].contiguous(), indices[perm].contiguous()
    del perm, users
    search = search_bytes(indptr)
    out = dict(scale=scale, n_users=n_users, n_items=n_items, samples=n, csr_search_bytes=search, configs=[])
    for e in (16, 64):
        D = e + 1
        default = int(_lib.lib.b200_bpr_default_inflight(e))
        for opt in OPTIMIZERS:
            for inflight in (0,) + (C5_INFLIGHT if sweep and e == 16 else ()):
                # every configuration starts from fresh tables and zero state, so a diverging one cannot leak
                U = (torch.randn(n_users, D, generator=g, device="cuda") * 0.03).contiguous()
                U[:, e] = 1.0
                I = (torch.randn(n_items, D, generator=g, device="cuda") * 0.03).contiguous()
                I[:, e] = 0.0
                states = [torch.zeros_like(t) for t in {"sgd": (), "momentum": (U, I), "adam": (U, I, U, I)}[opt]]
                epoch = [0]

                def run():
                    epoch[0] += 1
                    _launch(opt, s_users, s_items, indptr, indices, n_users, n_items, U, I, states, 0.01, 0.0, 0.9,
                            0.9, 0.999, epoch[0], 42, max_inflight=inflight)

                sec = event_seconds(run, reps)
                bps = bytes_per_sample(D, opt, search)
                rec = dict(embed_size=e, optimizer=opt, max_inflight=inflight or default, default=inflight == 0,
                           epochs_run=epoch[0], epoch_sec=sec, samples_per_s=n / sec, bytes_per_sample=bps,
                           gb_per_s=n * bps / sec / 1e9, share_of_hbm=n * bps / HBM_PEAK / sec,
                           finite=bool(torch.isfinite(U).all() and torch.isfinite(I).all()))
                out["configs"].append(rec)
                print(f"C5 e={e} {opt} inflight={rec['max_inflight']}: {sec * 1e3:.1f} ms/epoch, "
                      f"{n / sec / 1e9:.3f} G samples/s, {bps:.0f} B/sample, {rec['share_of_hbm'] * 100:.1f} % of HBM, "
                      f"finite after {epoch[0]} epochs: {rec['finite']}", file=sys.stderr, flush=True)
                del U, I, states
    return out


def run_c1(reps):
    import numpy as np
    import torch

    import _bpr_oracle as orc
    from librecommender_b200 import _lib
    from librecommender_b200.bpr import BPRTrainer
    from test_bpr_cpu import _golden, c1_data, fit_golden

    z = _golden()
    csr, users, items, eu, ei = c1_data(z)
    props = torch.cuda.get_device_properties(0)
    full = props.multi_processor_count * props.max_threads_per_multi_processor // 8      # embed 16: 8 lanes a sample
    default = int(_lib.lib.b200_bpr_default_inflight(16))
    rows = []
    for opt in OPTIMIZERS:
        f = fit_golden(z, opt)
        for inflight in sorted(set(C1_INFLIGHT) | {default, full}):
            tr = BPRTrainer(csr, users, items, optimizer=opt, lr=f["lr"], reg=None, embed_size=16, seed=42)
            tr.max_inflight = inflight
            tr.fit(3)
            U, I = (t.cpu().numpy() for t in tr.embeddings())
            finite = bool(np.isfinite(U).all() and np.isfinite(I).all())
            rec, ndcg = orc.ranking_metrics(U[:-1], I[:-1], csr.indptr, csr.indices, eu, ei) if finite else (0, 0)
            sec = event_seconds(tr.epoch, reps)
            rows.append(dict(optimizer=opt, max_inflight=inflight, default=inflight == default, epoch_sec=sec,
                             samples_per_s=users.size / sec, finite=finite, recall10=rec, ndcg10=ndcg,
                             cython_recall10=float(f["metrics"][0]), cython_ndcg10=float(f["metrics"][1])))
            print(f"C1 {opt} inflight={inflight}{' (default)' if inflight == default else ''}: "
                  f"{sec * 1e3:.2f} ms/epoch recall@10 {rec:.4f} ndcg@10 {ndcg:.4f} "
                  f"(Cython {f['metrics'][0]:.4f} / {f['metrics'][1]:.4f})", file=sys.stderr, flush=True)
    return dict(samples=int(users.size), default_inflight=default, full_occupancy=full, runs=rows)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scale", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--skip-c5", action="store_true")
    ap.add_argument("--c5-sweep", action="store_true", help="also time embed 16 at the C5_INFLIGHT schedules")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("profile_bpr needs a CUDA device")
    res = dict(card=card(), hbm_peak=HBM_PEAK, c1=run_c1(a.reps))
    if not a.skip_c5:
        res["c5"] = run_c5(a.scale, a.reps, a.c5_sweep)
    res["card_after"] = card()
    write_report(res, a.out)


if __name__ == "__main__":
    main()
