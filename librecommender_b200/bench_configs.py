"""``bench.py --config c1|c3|c4|c5``: the other BASELINE.json configurations on ONE GPU, each as a JSON
line with the contract's keys (``metric`` / ``value`` / ``unit`` / ``roofline`` in HBM GB/s where SURVEY.md
§8d says HBM-bound / ``clocks`` / ``cpu_baseline``).  Every timed leg runs ``--warmup`` untimed and
``--steps`` timed calls.  Shapes follow SURVEY.md §8d scaled to one GPU
(the 8-GPU row-sharded variants are exercised by the ``secondary`` legs of the default config at N > 1):

* ``c3``  DeepFM 100 sparse + 10 dense columns, K = 16, hidden (128, 64, 32): training-step
  interactions/s (gather fwd + MLP + loss + backward scatter + TF-Adam on the device) and predict rows/s;
  roofline = the K1 gather against the HBM bandwidth (algorithmic bytes/row of §8d);
* ``c4``  DIN, T = 50, item features (K' = 64): predict rows/s and all-items recommend users/s;
* ``c5``  LightGCN 3-layer propagation over a Zipf bipartite graph: nnz/s and algorithmic GB/s (§8d), then
  top-100 serving over the propagated embeddings;
* ``c1``  FM on the reference's sample_movielens (needs the staged / mounted reference for the data
  pipeline): recommend_user users/s for all users.
"""
from __future__ import annotations

import json
import os
import time

import numpy as np


def _timeit(fn, iters, warm):
    import torch

    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def _hbm_peak(root):
    """(GB/s, source): a measured copy bandwidth from MEASURED_PEAKS.json when present, else the H100 SXM
    data-sheet HBM3 figure."""
    try:
        return (float(json.load(open(os.path.join(root, "MEASURED_PEAKS.json")))["hbm_gbs"]),
                "MEASURED_PEAKS.json hbm_gbs (measured)")
    except Exception:
        return 3350.0, "H100 SXM data-sheet HBM3 bandwidth (not measured)"


def _line(metric, value, unit, steps, warmup, ms, config, roofline, cpu, clocks, extra=None):
    d = {"metric": metric, "value": value, "unit": unit, "n_gpus": 1, "steps": steps, "warmup": warmup,
         "ms_per_step": ms, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "f32",
         "data": "synthetic", "config": config, "clocks": clocks, "roofline": roofline, "cpu_baseline": cpu}
    d.update(extra or {})
    return d


def c3(args, root, sampler):
    import torch

    from . import _lib
    from . import synthetic as syn
    from .feat_models import DeepFM
    from .training import DeepFMTrainer

    rng = np.random.default_rng(5)
    us = [int(x) for x in np.exp(rng.uniform(np.log(10), np.log(2e5), 50))]
    its = [int(x) for x in np.exp(rng.uniform(np.log(10), np.log(2e5), 50))]
    n_users, n_items, K = 1_000_000, 100_000, 16
    spec = syn.make_spec(rng, n_users, n_items, us, its, 5, 5, interleave=False)
    w = syn.make_deepfm_weights(rng, spec, K, (128, 64, 32), True)
    Fs, Fd = spec["n_sparse"], spec["n_dense"]
    F = 2 + Fs + Fd
    # ---- forward gather (K1) + predict
    model = DeepFM(spec, w)
    R = 1 << 20
    users = torch.as_tensor(rng.integers(0, n_users, R)).cuda()
    items = torch.as_tensor(rng.integers(0, n_items, R)).cuda()
    concat = torch.empty((R, F * K), dtype=torch.float32, device="cuda")
    pw = torch.empty((R, K), dtype=torch.float32, device="cuda")
    lin = torch.empty(R, dtype=torch.float32, device="cuda")
    sampler.start()
    ms_g = _timeit(lambda: model._feat_forward(model.spec.layout, users, items, R, 0, concat=concat, pw=pw, lin=lin),
                   args.steps, args.warmup)
    read = R * ((2 + Fs) * (4 * K + 4) + 4 * Fs + 4 * Fd + 16)          # SURVEY 8d: fwd bytes/row
    alg = read + R * (F * K + K + 1) * 4
    up, ip_ = users[:1 << 18].cpu().numpy(), items[:1 << 18].cpu().numpy()
    ms_p = _timeit(lambda: model.logits(up, ip_), args.steps, args.warmup)
    # ---- training step (collate + negatives come from the caller in the reference; here labels are given)
    tr = DeepFMTrainer(spec, w, use_bn=True, lr=1e-3)
    B = 8192
    tu, ti = users[:B].contiguous(), items[:B].contiguous()
    labels = torch.as_tensor((rng.random(B) < 1 / 6).astype(np.float32)).cuda()
    ms_eager = _timeit(lambda: tr.step(tu, ti, labels), args.steps, args.warmup)
    # the same step captured once into a CUDA graph and replayed (launch-bound when issued from Python)
    ms_t = _timeit(lambda: tr.step_graph(tu, ti, labels), args.steps, args.warmup)
    clocks = sampler.stop()
    peak, peak_source = _hbm_peak(root)
    gbs = alg / (ms_g * 1e-3) / 1e9
    roofline = {"bound": "hbm", "kernel": "b200::feat::feat_forward_* (K1 gather + FM sums + deep-input write)",
                "achieved": gbs, "peak": peak, "unit": "GB/s", "frac": gbs / peak, "traffic": None,
                "peak_source": peak_source,
                "avg_launch_ms": ms_g, "algorithmic_bytes_per_row": alg / R}
    config = {"workload": f"C3 DeepFM: {Fs} sparse + {Fd} dense columns, K {K}, hidden (128, 64, 32), "
                          f"{n_users} users x {n_items} items, shared sparse table {spec['sparse_vocab']} rows, "
                          f"batch {B} rows/step, one GPU (tables replicated)",
              "l2": "tables 1.3 GB > L2"}
    return _line("training-step interactions/sec (DeepFM)", B / (ms_t * 1e-3), "interactions/s", args.steps, args.warmup, ms_t, config,
                 roofline, None, clocks,
                 {"predict_rows_per_s": (1 << 18) / (ms_p * 1e-3), "gather_rows_per_s": R / (ms_g * 1e-3),
                  "ms_per_step_eager_launches": ms_eager, "step": "CUDA graph replay (step_graph)",
                  "kernels_per_captured_step": int(getattr(tr, "graph_launches_per_step", 0)),
                  "gpu_launches": int(_lib.launch_count())
                                  + (args.steps + args.warmup) * int(getattr(tr, "graph_launches_per_step", 0))})


def c4(args, root, sampler):
    import torch

    from . import _lib
    from . import synthetic as syn
    from .feat_models import DIN, recent_sequences_csr

    rng = np.random.default_rng(6)
    n_users, n_items, K, T = 200_000, 100_000, 16, 50
    spec = syn.make_spec(rng, n_users, n_items, [50, 7], [1000, 300, 40], 1, 0, interleave=False)
    w = syn.make_seq_weights(rng, spec, K, (128, 64, 32), True, din=True)
    lens = np.minimum(rng.poisson(80, n_users), 1000).clip(min=1)
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    np.cumsum(lens, out=indptr[1:])
    idx = (np.exp(rng.random(int(indptr[-1])) * np.log(n_items)) - 1).astype(np.int32).clip(0, n_items - 1)
    from .consumed import ConsumedCSR

    csr = ConsumedCSR(indptr, idx)
    seqs, slen = recent_sequences_csr(csr, n_items, T)
    model = DIN(spec, w, seqs, slen, csr)
    R = 1 << 18
    users = rng.integers(0, n_users, R)
    items = rng.integers(0, n_items, R)
    sampler.start()
    ms_p = _timeit(lambda: model.logits(users, items), args.steps, args.warmup)
    uids = rng.integers(0, n_users, 16)
    model.recommend(uids[:2], 100, True)
    ms_r = _timeit(lambda: model.recommend(uids, 100, True), args.steps, args.warmup)
    clocks = sampler.stop()
    Kp = model.Kp
    peak, peak_source = _hbm_peak(root)
    alg = R * ((2 + T) * 4 * Kp + 4 * T + 64)                            # SURVEY 8d a7 rows: bytes/row
    gbs = alg / (ms_p * 1e-3) / 1e9
    roofline = {"bound": "hbm", "kernel": "b200::seq::din_attention_kernel + K1 + MLP (predict rows)", "achieved": gbs,
                "peak": peak, "unit": "GB/s", "frac": gbs / peak, "traffic": None, "avg_launch_ms": ms_p,
                "peak_source": peak_source}
    config = {"workload": f"C4 DIN: seq_len {T}, {n_users} users x {n_items} items, K {K}, K' {Kp}, "
                          f"hidden (128, 64, 32), one GPU", "l2": "item feature table 25 MB (L2 resident), rows 13 KB"}
    return _line("DIN predict rows/sec", R / (ms_p * 1e-3), "rows/s", args.steps, args.warmup, ms_p, config, roofline, None, clocks,
                 {"recommend_users_per_s": len(uids) / (ms_r * 1e-3), "recommend_batch": len(uids),
                  "gpu_launches": int(_lib.launch_count())})


def c5(args, root, sampler):
    import torch

    from . import _lib
    from .consumed import ConsumedCSR
    from .engine import EmbedScorer
    from .lightgcn import SpmmGraph, build_laplacian_csr, propagate

    dev = torch.device("cuda")
    g = torch.Generator(device=dev).manual_seed(5)
    n_users, n_items, d, layers = 2_000_000, 200_000, 64, 3
    deg = torch.clamp(torch.poisson(torch.full((n_users,), 50.0, device=dev), generator=g), 1, 2000).long()
    indptr = torch.zeros(n_users + 1, dtype=torch.int64, device=dev)
    indptr[1:] = torch.cumsum(deg, 0)
    u = torch.rand(int(indptr[-1]), device=dev, generator=g)
    idx = (torch.exp(u * np.log(n_items)) - 1).clamp(0, n_items - 1).to(torch.int32)
    csr = ConsumedCSR.from_device_tensors(indptr, idx)
    ip, col, val = build_laplacian_csr(csr, n_users, n_items, dev)
    graph = SpmmGraph(ip, col, val)
    E0 = torch.randn(n_users + n_items, d, device=dev, generator=g) * 0.1
    n, nnz = n_users + n_items, graph.nnz
    sampler.start()
    ms = _timeit(lambda: propagate(graph, E0, layers), args.steps, args.warmup)
    out = propagate(graph, E0, layers)
    scorer = EmbedScorer(out[:n_users], out[n_users:], n_items, csr, n_users=n_users, device=dev)
    uid = torch.randint(0, n_users, (8192,), device=dev, generator=g)
    scorer.recommend_device(uid, 100, True, False)
    ms_s = _timeit(lambda: scorer.recommend_device(uid, 100, True, False), args.steps, args.warmup)
    clocks = sampler.stop()
    alg = layers * (nnz * (8 + 4 * d) + n * (4 * d + 8)) + layers * n * 4 * d      # SURVEY 8d a10 + layer-mean accumulate
    peak, peak_source = _hbm_peak(root)
    gbs = alg / (ms * 1e-3) / 1e9
    roofline = {"bound": "hbm", "kernel": "b200::spmm_* (3 layers, layer mean fused)", "achieved": gbs, "peak": peak,
                "unit": "GB/s", "frac": gbs / peak, "traffic": None, "avg_launch_ms": ms / layers,
                "note": "algorithmic bytes count every gathered row as if it came from HBM; popular rows are served "
                        "by the 50 MB L2, so this can read above 1",
                "peak_source": peak_source}
    config = {"workload": f"C5 LightGCN: {layers}-layer propagation, {n_users} x {n_items} bipartite graph, nnz {nnz}, "
                          f"d {d}; then top-100 over {n_items} items for 8192 users", "l2": "E 563 MB + CSR 2.2 GB > L2"}
    return _line("LightGCN propagation nnz/sec", layers * nnz / (ms * 1e-3), "nnz/s", args.steps, args.warmup, ms, config, roofline, None, clocks,
                 {"serving_users_per_s": 8192 / (ms_s * 1e-3), "gpu_launches": int(_lib.launch_count())})


def c1(args, root, sampler):
    import pandas as pd
    import torch

    from oracle.ref_loader import REFERENCE_ROOT, load_reference, reference_available   # data pipeline only

    if not reference_available():
        return {"config": {"workload": "C1"}, "unavailable": "reference data pipeline neither mounted nor staged"}
    load_reference()
    from libreco.data import DatasetFeat, split_by_ratio_chrono

    from . import _lib
    from . import synthetic as syn
    from .feat_models import FM

    data = pd.read_csv(os.path.join(REFERENCE_ROOT, "examples/sample_data/sample_movielens_merged.csv"))
    train, _ = split_by_ratio_chrono(data, test_size=0.2)
    _, di = DatasetFeat.build_trainset(train, ["sex", "age", "occupation"], ["genre1", "genre2", "genre3"],
                                       ["sex", "occupation", "genre1", "genre2", "genre3"], ["age"])
    spec = dict(n_users=di.n_users, n_items=di.n_items,
                user_sparse_col_index=list(di.user_sparse_col.index), item_sparse_col_index=list(di.item_sparse_col.index),
                user_dense_col_index=list(di.user_dense_col.index), item_dense_col_index=list(di.item_dense_col.index),
                user_sparse_unique=di.user_sparse_unique, item_sparse_unique=di.item_sparse_unique,
                user_dense_unique=di.user_dense_unique.astype(np.float32), item_dense_unique=None,
                sparse_vocab=int(max(di.user_sparse_unique.max(), di.item_sparse_unique.max()) + 1))
    spec["n_sparse"] = len(spec["user_sparse_col_index"]) + len(spec["item_sparse_col_index"])
    spec["n_dense"] = len(spec["user_dense_col_index"]) + len(spec["item_dense_col_index"])
    w = syn.make_fm_weights(np.random.default_rng(42), spec, 16, use_bn=True)
    model = FM(spec, w, di.user_consumed)
    users = np.arange(di.n_users)
    sampler.start()
    for _ in range(args.warmup):
        model.recommend(users, 7, True)
        model.recommend(users, 100, True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    iters = args.steps
    for _ in range(iters):
        model.recommend(users, 7, True)
        model.recommend(users, 100, True)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) / iters * 1e3
    clocks = sampler.stop()
    config = {"workload": f"C1 FM on sample_movielens_merged ({di.n_users} users x {di.n_items} items, embed 16, 5 sparse "
                          "+ 1 dense columns): recommend_user for ALL users, n_rec 7 and 100 (two calls per step)"}
    return _line("recommend_user users/sec (all-items top-K, FM)", 2 * di.n_users / (ms * 1e-3), "users/s", iters, args.warmup, ms,
                 config, None, None, clocks, {"gpu_launches": int(_lib.launch_count())})


CONFIGS = {"c1": c1, "c3": c3, "c4": c4, "c5": c5}
