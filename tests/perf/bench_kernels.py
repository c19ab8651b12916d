"""Secondary kernel measurements (HBM-bound rows of SURVEY.md §8d): achieved GB/s against the
measured copy bandwidth.  CUDA-event timing, 3 warm-ups, inputs larger than L2.
    python tests/perf/bench_kernels.py > gpurun_out/kernels.jsonl
"""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)

PEAK = 3350.0   # H100 SXM data-sheet HBM3 GB/s, used unless MEASURED_PEAKS.json gives a measured copy rate
try:
    PEAK = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"]
except Exception:
    pass


def timeit(fn, iters=10, warm=3):
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


def emit(name, ms, bytes_, extra=None):
    gbs = bytes_ / (ms * 1e-3) / 1e9
    d = {"kernel": name, "ms": ms, "algorithmic_bytes": bytes_, "achieved_gbs": gbs, "peak_gbs": PEAK,
         "frac": gbs / PEAK}
    d.update(extra or {})
    print(json.dumps(d), flush=True)


def bench_spmm():
    from librecommender_b200.lightgcn import SpmmGraph, propagate

    dev = torch.device("cuda")
    g = torch.Generator(device=dev)
    g.manual_seed(5)
    n_users, n_items, d = 2_000_000, 200_000, 64
    counts = torch.poisson(torch.full((n_users,), 50.0, device=dev), generator=g).clamp_(min=1, max=2000).long()
    w = 1.0 / torch.arange(1, n_items + 1, device=dev, dtype=torch.float64)
    cdf = (torch.cumsum(w, 0) / w.sum()).float()
    perm = torch.randperm(n_items, generator=g, device=dev)
    owner = torch.repeat_interleave(torch.arange(n_users, device=dev), counts)
    item = perm[torch.searchsorted(cdf, torch.rand(owner.numel(), generator=g, device=dev)).clamp_(max=n_items - 1)]
    n = n_users + n_items
    shift = (n - 1).bit_length()
    und = torch.unique((owner << shift) | (item + n_users))
    r, c = und >> shift, und & ((1 << shift) - 1)
    key = torch.sort(torch.cat([und, (c << shift) | r])).values
    rows, cols = key >> shift, (key & ((1 << shift) - 1)).to(torch.int32)
    deg = torch.bincount(rows, minlength=n)
    indptr = torch.zeros(n + 1, dtype=torch.int64, device=dev)
    indptr[1:] = torch.cumsum(deg, 0)
    dinv = deg.float().pow(-0.5)
    dinv[torch.isinf(dinv)] = 0
    val = dinv[rows] * dinv[cols.long()]
    graph = SpmmGraph(indptr, cols.contiguous(), val.contiguous())
    E = torch.randn(n, d, device=dev) * 0.1
    out = torch.empty_like(E)
    nnz = graph.nnz
    ms = timeit(lambda: graph.spmm(E, out=out))
    bytes_ = nnz * (4 + 4 + 4 * d) + n * (4 * d + 8)          # SURVEY §8d row a10
    emit("spmm_csr (LightGCN layer)", ms, bytes_, {"nnz": nnz, "rows": n, "d": d, "long_rows": graph.n_long,
                                                  "max_degree": int(deg.max())})
    ms3 = timeit(lambda: propagate(graph, E, 3), iters=5)
    emit("lightgcn propagate 3 layers (fused mean)", ms3, 3 * bytes_ + 3 * n * 4 * d, {"nnz": nnz})
    # one BPR training step exactly as TorchTrainer._compute_loss (full-graph propagation + backward + Adam)
    from librecommender_b200.lightgcn import propagate_autograd

    W = torch.nn.Parameter(E.clone())
    opt = torch.optim.Adam([W], lr=1e-3)
    bs = 2048
    uu = torch.randint(0, n_users, (bs,), device=dev)
    pp = torch.randint(0, n_items, (bs,), device=dev) + n_users
    nn_ = torch.randint(0, n_items, (bs,), device=dev) + n_users

    def step():
        out = propagate_autograd(graph, W, 3)
        loss = -torch.nn.functional.logsigmoid((out[uu] * out[pp]).sum(1) - (out[uu] * out[nn_]).sum(1)).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()

    ms_step = timeit(step, iters=5)
    print(json.dumps({"kernel": "LightGCN BPR training step (3-layer full-graph fwd+bwd, dense Adam), batch 2048",
                      "ms": ms_step, "interactions_per_s": bs / (ms_step * 1e-3), "nodes": n, "nnz": nnz}), flush=True)
    # CPU side: the reference's own op (torch.sparse.mm on a COO Laplacian, lightgcn_module.py:74-88), one layer
    t_rows = torch.repeat_interleave(torch.arange(n, device=dev), deg).cpu()
    Lc = torch.sparse_coo_tensor(torch.stack([t_rows, cols.long().cpu()]), val.cpu(), (n, n)).coalesce()
    Ec = E.cpu()
    torch.set_num_threads(os.cpu_count())
    t0 = time.perf_counter()
    torch.sparse.mm(Lc, Ec)
    cpu_s = time.perf_counter() - t0
    print(json.dumps({"kernel": "cpu_baseline: torch.sparse.mm one layer (reference op)", "seconds": cpu_s,
                      "cores": os.cpu_count(), "kind": "reference-op", "speedup_vs_gpu_layer": cpu_s / (ms * 1e-3)}),
          flush=True)


def bench_feat():
    from librecommender_b200.feat_models import DeepFM, FM
    from oracle import tf_models as tm

    rng = np.random.default_rng(0)
    us = [int(x) for x in np.exp(rng.uniform(np.log(10), np.log(2e5), 50))]
    its = [int(x) for x in np.exp(rng.uniform(np.log(10), np.log(2e5), 50))]
    spec = tm.make_spec(rng, 1_000_000, 100_000, us, its, 5, 5, interleave=False)
    K = 16
    w = tm.make_deepfm_weights(rng, spec, K, (128, 64, 32), True)
    model = DeepFM(spec, w)
    R = 1 << 20
    users = torch.as_tensor(rng.integers(0, 1_000_000, R)).cuda()
    items = torch.as_tensor(rng.integers(0, 100_000, R)).cuda()
    F = 2 + spec["n_sparse"] + spec["n_dense"]
    concat = torch.empty((R, F * K), dtype=torch.float32, device="cuda")
    pw = torch.empty((R, K), dtype=torch.float32, device="cuda")
    lin = torch.empty(R, dtype=torch.float32, device="cuda")
    from librecommender_b200 import _lib

    Fs, Fd = spec["n_sparse"], spec["n_dense"]
    read = R * ((2 + Fs) * (4 * K + 4) + 4 * Fs + 4 * Fd + 16)
    wfm = tm.make_fm_weights(rng, spec, K, True)
    fm = FM(spec, wfm)
    out = torch.empty(R, dtype=torch.float32, device="cuda")
    ref_concat = None
    for tma, tag in ((0, "software-pipelined register gather, K/4 lanes per field (default)"),
                     (8, "cp.async staged, K/4 lanes per field"), (4, "register gather, K/4 lanes per field"),
                     (2, "register gather, lane per field"),
                     (1, "TMA-staged persistent (cp.async.bulk ring)")):
        _lib.check(_lib.lib.b200_feat_forward_tune(tma))
        ms = timeit(lambda: model._feat_forward(model.spec.layout, users, items, R, 0, concat=concat, pw=pw, lin=lin))
        emit(f"feat_forward gather+FM (DeepFM C3 row shape, writes deep input) [{tag}]", ms,
             read + R * (F * K + K + 1) * 4,
             {"rows": R, "F_sparse": Fs, "F_dense": Fd, "K": K, "gather_only_bytes": read, "tma": tma})
        if ref_concat is None:
            ref_concat, ref_pw, ref_lin = concat[:4096].clone(), pw[:4096].clone(), lin[:4096].clone()
        else:   # the two kernels must agree (concat bit-for-bit: pure copies; sums to rounding)
            print(json.dumps({"check": f"variant {tma} vs default kernel", "concat_equal": bool(torch.equal(concat[:4096], ref_concat)),
                              "pw_max_abs_diff": float((pw[:4096] - ref_pw).abs().max()),
                              "lin_max_abs_diff": float((lin[:4096] - ref_lin).abs().max())}), flush=True)
        ms = timeit(lambda: fm._feat_forward(fm.spec.layout, users, items, R, 0, fm_out=out, head=fm.head))
        emit(f"feat_forward FM fused head (no intermediate) [{tag}]", ms, read + R * 4, {"rows": R, "tma": tma})
    _lib.check(_lib.lib.b200_feat_forward_tune(0))
    ms = timeit(lambda: model.logits(users[:1 << 18].cpu().numpy(), items[:1 << 18].cpu().numpy()), iters=3)
    print(json.dumps({"kernel": "DeepFM predict rows/s (gather + fp32 MLP 1792-128-64-32)", "rows_per_s": (1 << 18) / (ms * 1e-3)}))
    # all-items scoring + top-100 (recommend_user of the TfBase models), hoisted kernels
    uids = rng.integers(0, 1_000_000, 256)
    for nm, mdl in (("FM", fm), ("DeepFM", model)):
        mdl.recommend(uids[:8], 100, False)
        ms_r = timeit(lambda: mdl.recommend(uids, 100, False), iters=3, warm=1)
        print(json.dumps({"kernel": f"{nm} recommend_user all-items top-100 (N=100k items, 256 users/call, hoisted)",
                          "ms": ms_r, "users_per_s": len(uids) / (ms_r * 1e-3),
                          "pairs_per_s": len(uids) * 100_000 / (ms_r * 1e-3)}), flush=True)
    # CPU side: numpy restatement of the DeepFM graph (oracle port) on a bounded sample
    nu = 1 << 15
    uh, ih = users[:nu].cpu().numpy(), items[:nu].cpu().numpy()
    sp, de = tm.row_features(spec, uh, ih)
    t0 = time.perf_counter()
    tm.deepfm_forward(w, uh, ih, sp, de)
    cpu_s = time.perf_counter() - t0
    print(json.dumps({"kernel": "cpu_baseline: DeepFM forward (oracle port, numpy)", "rows_per_s": nu / cpu_s,
                      "cores": os.cpu_count(), "kind": "port", "sample": f"{nu} rows"}), flush=True)


def bench_topk_and_sampler():
    import ctypes
    from librecommender_b200 import _lib
    from librecommender_b200.sampling import DeviceNegativeSampler

    B, N, K = 256, 1_000_000, 100
    scores = torch.randn(B, N, device="cuda")
    ids = torch.empty(B, K, dtype=torch.int64, device="cuda")
    nb = ctypes.c_size_t()
    _lib.lib.b200_topk_rows_workspace_bytes(B, N, K, ctypes.byref(nb))
    ws = torch.empty(nb.value, dtype=torch.uint8, device="cuda")
    ms = timeit(lambda: _lib.check(_lib.lib.b200_topk_rows(_lib.ptr(scores), N, B, N, K, _lib.ptr(ids), None,
                                                           _lib.ptr(ws), nb.value, _lib.current_stream())))
    emit("topk_rows radix select (256 x 1M, K=100)", ms, 5 * B * N * 4, {"passes": 5})
    smp = DeviceNegativeSampler(1_000_000, seed=42)
    pos = torch.randint(0, 1_000_000, (1 << 22,), device="cuda")
    ms = timeit(lambda: smp.sample(None, pos, 5, "random"))
    print(json.dumps({"kernel": "sample_negatives random (4M positives x 5)", "ms": ms,
                      "negatives_per_s": (1 << 22) * 5 / (ms * 1e-3)}))
    from librecommender_b200.sampling import negatives_from_random
    ph = pos[:1 << 20].cpu().numpy()
    t0 = time.perf_counter()
    negatives_from_random(np.random.default_rng(462), 1_000_000, ph, 5)
    cpu_s = time.perf_counter() - t0
    print(json.dumps({"kernel": "cpu_baseline: negatives_from_random (reference numpy stream, parity mode)",
                      "negatives_per_s": (1 << 20) * 5 / cpu_s, "cores": 1, "kind": "reference-stream"}))


def bench_linear():
    """Dense layer: exact-fma SIMT kernel vs the wgmma 3xTF32 kernel (fp32-level accuracy)."""
    from librecommender_b200 import _lib

    tc_peak = 989.0   # H100 SXM data-sheet dense BF16 TFLOP/s unless MEASURED_PEAKS.json gives a measured rate
    try:
        tc_peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["bf16_tflops"]
    except Exception:
        pass
    for R, din, dout in ((1 << 20, 1792, 128), (1 << 20, 128, 64), (1 << 18, 512, 256)):
        x = torch.randn(R, din, device="cuda")
        Wt = torch.randn(dout, din, device="cuda") / din ** 0.5
        b = torch.randn(dout, device="cuda")
        y = torch.empty(R, dout, device="cuda")
        ld = int(_lib.lib.b200_linear_tf32x3_split_ld(din))
        ws = torch.empty(2 * dout * ld, device="cuda")
        _lib.check(_lib.lib.b200_linear_tf32x3_split_weights(_lib.ptr(Wt), din, din, dout, _lib.ptr(ws),
                                                             _lib.current_stream()))
        calls = {
            "b200_linear_f32": lambda: _lib.lib.b200_linear_f32(_lib.ptr(x), din, R, _lib.ptr(Wt), din, _lib.ptr(b), din,
                                                                dout, 1, _lib.ptr(y), dout, _lib.current_stream()),
            "b200_linear_tf32x3": lambda: _lib.lib.b200_linear_tf32x3(_lib.ptr(x), din, R, _lib.ptr(Wt), din, None,
                                                                      _lib.ptr(b), din, dout, 1, _lib.ptr(y), dout,
                                                                      _lib.current_stream()),
            "b200_linear_tf32x3 (pre-split weights)": lambda: _lib.lib.b200_linear_tf32x3(
                _lib.ptr(x), din, R, _lib.ptr(Wt), din, _lib.ptr(ws), _lib.ptr(b), din, dout, 1, _lib.ptr(y), dout,
                _lib.current_stream()),
        }
        for name, call in calls.items():
            ms = timeit(lambda: _lib.check(call()), iters=5, warm=3)
            flop = 2.0 * R * din * dout
            byt = 4.0 * (R * din + R * dout + dout * din)
            print(json.dumps({"kernel": f"{name} [{R} x {din}] -> {dout}", "ms": ms,
                              "tflops_effective": flop / (ms * 1e-3) / 1e12,
                              "tensor_tflops_issued": (3 * flop / (ms * 1e-3) / 1e12) if "tf32" in name else None,
                              "tf32_dense_peak_tflops": tc_peak / 2, "achieved_gbs": byt / (ms * 1e-3) / 1e9,
                              "peak_gbs": PEAK, "hbm_frac": byt / (ms * 1e-3) / 1e9 / PEAK}), flush=True)


def bench_seq():
    """Sequence models at a C4-like shape (item sparse fields 3, K = 16 -> K' = 64, T = 50)."""
    from librecommender_b200.consumed import ConsumedCSR
    from librecommender_b200.feat_models import DIN, YouTubeRanking, recent_sequences_csr
    from oracle import tf_models as tm

    rng = np.random.default_rng(0)
    n_users, n_items, T = 200_000, 100_000, 50
    spec = tm.make_spec(rng, n_users, n_items, [50, 1000], [1000, 10000, 100000], 1, 0, interleave=False)
    deg = np.minimum(rng.poisson(80, n_users), 1000).astype(np.int64) + 1
    indptr = np.concatenate([[0], np.cumsum(deg)])
    idx = rng.integers(0, n_items, indptr[-1]).astype(np.int32)
    csr = ConsumedCSR(indptr, idx)
    seqs, lens = recent_sequences_csr(csr, n_items, T)
    R = 1 << 18
    users = rng.integers(0, n_users, R)
    items = rng.integers(0, n_items, R)
    for name, cls, din in (("YouTubeRanking", YouTubeRanking, False), ("DIN", DIN, True)):
        w = tm.make_seq_weights(rng, spec, 16, (128, 64, 32), True, din=din)
        model = cls(spec, w, seqs, lens, csr)
        ms = timeit(lambda: model.logits(users, items), iters=3, warm=1)
        print(json.dumps({"kernel": f"{name} predict rows/s (T={T}, hidden 128-64-32)", "rows_per_s": R / (ms * 1e-3)}),
              flush=True)
        nu = 64 if not din else 4
        uid = rng.integers(0, n_users, nu)
        model.recommend(uid[:2], 100, True)
        ms = timeit(lambda: model.recommend(uid, 100, True), iters=2, warm=1)
        print(json.dumps({"kernel": f"{name} recommend_user all-items top-100 (N={n_items}, {nu} users/call, "
                                    f"{'hoisted' if getattr(model, '_hoistable', lambda: False)() else 'flat grid'})",
                          "ms": ms, "users_per_s": nu / (ms * 1e-3), "pairs_per_s": nu * n_items / (ms * 1e-3)}),
              flush=True)


def bench_train():
    """FM training step (gather fwd, BN, head, loss, backward scatter, TF-Adam over every variable)."""
    from librecommender_b200.training import FMTrainer
    from oracle import fm_train as ft
    from oracle import tf_models as tm

    for tag, n_users, n_items, n_f, R in (("C1-like (6k users x 3.2k items, 5 sparse + 1 dense)", 5958, 3231, 5, 2048),
                                          ("C3-like (1M users x 100k items, 100 sparse + 10 dense)", 1_000_000, 100_000,
                                           100, 8192)):
        rng = np.random.default_rng(0)
        if n_f == 5:
            spec = tm.make_spec(rng, n_users, n_items, [2, 21], [18, 18, 18], 1, 0, interleave=False)
        else:
            us = [int(x) for x in np.exp(rng.uniform(np.log(10), np.log(2e5), 50))]
            its = [int(x) for x in np.exp(rng.uniform(np.log(10), np.log(2e5), 50))]
            spec = tm.make_spec(rng, n_users, n_items, us, its, 5, 5, interleave=False)
        w = tm.make_fm_weights(rng, spec, 16, True)
        tr = FMTrainer(spec, w, use_bn=True, lr=1e-3)
        users = torch.as_tensor(rng.integers(0, n_users, R)).cuda()
        items = torch.as_tensor(rng.integers(0, n_items, R)).cuda()
        labels = torch.as_tensor((rng.random(R) < 0.3).astype(np.float32)).cuda()
        ms = timeit(lambda: tr.step(users, items, labels), iters=10, warm=3)
        n_par = sum(int(v.numel()) for v in tr.params.values())
        print(json.dumps({"kernel": f"FM training step, {tag}, batch {R}", "ms": ms,
                          "interactions_per_s": R / (ms * 1e-3), "trainable_floats": n_par,
                          "adam_dense_bytes_per_step": n_par * 4 * 7,
                          "adam_gbs_if_alone": n_par * 4 * 7 / (ms * 1e-3) / 1e9}), flush=True)
        from librecommender_b200.training import DeepFMTrainer
        from oracle import deepfm_train as dft

        wd = tm.make_deepfm_weights(rng, spec, 16, (128, 64, 32), True)
        trd = DeepFMTrainer(spec, wd, use_bn=True, lr=1e-3)
        ms_d = timeit(lambda: trd.step(users, items, labels), iters=10, warm=3)
        print(json.dumps({"kernel": f"DeepFM training step (128-64-32, BN), {tag}, batch {R}", "ms": ms_d,
                          "interactions_per_s": R / (ms_d * 1e-3),
                          "trainable_floats": sum(int(v.numel()) for v in trd.params.values())}), flush=True)
        if n_users <= 10000:
            std = dft.init_state(wd, True, dtype=np.float32)
            uh, ih, lh = users.cpu().numpy(), items.cpu().numpy(), labels.cpu().numpy()
            sp, de = tm.row_features(spec, uh, ih)
            dft.train_step(std, uh, ih, sp, de, lh, 1e-3)
            t0 = time.perf_counter()
            for _ in range(3):
                dft.train_step(std, uh, ih, sp, de, lh, 1e-3)
            cpu_ms = (time.perf_counter() - t0) / 3 * 1e3
            print(json.dumps({"kernel": f"cpu_baseline: DeepFM training step (oracle port, numpy), {tag}", "ms": cpu_ms,
                              "interactions_per_s": R / (cpu_ms * 1e-3), "cores": os.cpu_count(), "kind": "port"}),
                  flush=True)
        if n_users <= 10000:       # CPU baseline: the numpy restatement of the same step (oracle port)
            st = ft.init_state(w, True, dtype=np.float32)
            uh, ih, lh = users.cpu().numpy(), items.cpu().numpy(), labels.cpu().numpy()
            sp, de = tm.row_features(spec, uh, ih)
            ft.train_step(st, uh, ih, sp, de, lh, 1e-3)
            t0 = time.perf_counter()
            for _ in range(3):
                ft.train_step(st, uh, ih, sp, de, lh, 1e-3)
            cpu_ms = (time.perf_counter() - t0) / 3 * 1e3
            print(json.dumps({"kernel": f"cpu_baseline: FM training step (oracle port, numpy), {tag}", "ms": cpu_ms,
                              "interactions_per_s": R / (cpu_ms * 1e-3), "cores": os.cpu_count(), "kind": "port"}),
                  flush=True)


if __name__ == "__main__":
    which = sys.argv[1:] or ["spmm", "feat", "topk", "linear", "train", "seq"]
    if "train" in which:
        bench_train()
    if "seq" in which:
        bench_seq()
    if "linear" in which:
        bench_linear()
    if "spmm" in which:
        bench_spmm()
    if "feat" in which:
        bench_feat()
    if "topk" in which:
        bench_topk_and_sampler()
