"""The two paths of SURVEY.md §8e that DO have an exchange step, timed for ``bench.py --gpus N``
(N > 1) under the JSON line's ``secondary`` key; each leg checks its own result first.

* ``lightgcn``: 3-layer LightGCN propagation (reference: ``lightgcn_module.py:66-88``) over a C5-shaped
  synthetic bipartite graph (Zipf item popularity, Poisson(50) user degrees), rows sharded over the
  N GPUs, slab exchange per layer — (a) one NCCL all-gather per layer then SpMM, (b) the exchange
  overlapped with per-source-rank block SpMMs, slabs pulled over NVLink peer memory by the copy
  engines (falls back to an NCCL send/recv ring when symmetric memory is unavailable), (c) two
  products per layer: the own column block while the slabs travel, the rest in one product.  Strong
  scaling: ``efficiency = t_single / (N * t_N)`` with the single-GPU time measured in the same run.
* ``row_sharded_lookup``: DeepFM-shaped (K = 16) and DIN-shaped (K' = 64) row gathers from a table
  sharded ``row % N`` — (a) NCCL path (index all-to-all, local gather, row all-to-all), (b) ONE
  kernel that pulls the rows over NVLink from the peer shards (``b200_peer_gather_rows``).
  ``nvlink_gbs`` = bytes that must cross NVLink into one GPU / time; ``frac`` against the H100 SXM
  data-sheet NVLink rate per direction (450 GB/s, not a measured figure).
"""
from __future__ import annotations

import numpy as np

NVLINK_REF_GBS = 450.0   # H100 SXM NVLink 4: 900 GB/s per GPU both directions together (data sheet)


def _timed(fn, iters, max_over_ranks, barrier):
    import torch

    for _ in range(2):
        fn()
    barrier()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    barrier()
    return max_over_ranks(e0.elapsed_time(e1) / iters)


def _lightgcn(rank, world, dev, max_over_ranks, barrier, n_users=2_000_000, n_items=200_000, d=64, n_layers=3):
    import torch

    from .consumed import ConsumedCSR
    from .lightgcn import SpmmGraph, build_laplacian_csr, propagate
    from .parallel import (LightGCNShardPlan, PeerPullExchange, RingExchange, acc_spmm_fn, block_spmm_fn,
                           gather_embeddings, propagate_sharded, propagate_sharded_overlap,
                           propagate_sharded_two_phase, sharded_spmm_fn, split_column_blocks, split_local_remote)

    g = torch.Generator(device=dev).manual_seed(5)
    deg = torch.clamp(torch.poisson(torch.full((n_users,), 50.0, device=dev), generator=g), 1, 2000).long()
    indptr = torch.zeros(n_users + 1, dtype=torch.int64, device=dev)
    indptr[1:] = torch.cumsum(deg, 0)
    nnz_u = int(indptr[-1])
    u = torch.rand(nnz_u, device=dev, generator=g)
    idx = (torch.exp(u * np.log(n_items)) - 1).clamp(0, n_items - 1).to(torch.int32)
    ip, col, val = build_laplacian_csr(ConsumedCSR.from_device_tensors(indptr, idx), n_users, n_items, dev)
    del u, idx, deg
    E0 = torch.randn(n_users + n_items, d, device=dev, generator=g) * 0.1
    nnz = int(col.numel())

    plan = LightGCNShardPlan(n_users, n_items, world)
    lptr, lcol, lval = plan.shard_csr(ip, col, val, rank)
    local_graph = SpmmGraph(lptr, lcol, lval)
    blocks = [SpmmGraph(*b) for b in split_column_blocks(lptr, lcol, lval, plan.slab, world)]
    E0_loc = plan.scatter_rows(E0, rank)
    full_graph = SpmmGraph(ip, col, val)
    ref = propagate(full_graph, E0, n_layers)

    out = {"n_users": n_users, "n_items": n_items, "nnz": nnz, "d": d, "layers": n_layers,
           "nnz_local": int(lval.numel())}
    spmm_local = sharded_spmm_fn(local_graph, plan.slab)

    def run_gather():
        return propagate_sharded(plan, spmm_local, E0_loc, n_layers)

    ue, ie = gather_embeddings(plan, run_gather())
    out["allgather_max_abs_err"] = float((torch.cat([ue, ie]) - ref).abs().max())
    out["ms_allgather_then_spmm"] = _timed(run_gather, 5, max_over_ranks, barrier)

    exchange, kind = None, "peer_pull (symmetric memory, copy engines over NVLink)"
    try:
        exchange = PeerPullExchange(world, rank)
        res = propagate_sharded_overlap(plan, block_spmm_fn(blocks), E0_loc, n_layers, exchange, rank)
        torch.cuda.synchronize()
    except Exception as e:   # symmetric memory not available on this box: NCCL ring
        out["peer_pull_error"] = repr(e)[:300]
        exchange, kind = RingExchange(world, rank), "nccl send/recv ring"
        res = propagate_sharded_overlap(plan, block_spmm_fn(blocks), E0_loc, n_layers, exchange, rank)
    ue, ie = gather_embeddings(plan, res)
    out["overlap_engine"] = kind
    out["overlap_max_abs_err"] = float((torch.cat([ue, ie]) - ref).abs().max())
    out["ref_scale"] = float(ref.abs().max())

    def run_overlap():
        return propagate_sharded_overlap(plan, block_spmm_fn(blocks), E0_loc, n_layers, exchange, rank)

    out["ms_overlapped"] = _timed(run_overlap, 5, max_over_ranks, barrier)
    # (c) two products per layer: the own column block while the slabs travel, every other block in one product
    own, rest = split_local_remote(lptr, lcol, lval, plan.slab, rank)
    g_own, g_rest = SpmmGraph(*own), SpmmGraph(*rest)

    def run_two_phase():
        return propagate_sharded_two_phase(plan, acc_spmm_fn(g_own), acc_spmm_fn(g_rest), E0_loc, n_layers, exchange,
                                           rank)

    ue, ie = gather_embeddings(plan, run_two_phase())
    out["two_phase_max_abs_err"] = float((torch.cat([ue, ie]) - ref).abs().max())
    out["ms_two_phase"] = _timed(run_two_phase, 5, max_over_ranks, barrier)
    out["ms_single_gpu"] = _timed(lambda: propagate(full_graph, E0, n_layers), 3, max_over_ranks, barrier)
    best = min(out["ms_overlapped"], out["ms_allgather_then_spmm"], out["ms_two_phase"])
    out["efficiency_two_phase"] = out["ms_single_gpu"] / (world * out["ms_two_phase"])
    out["efficiency_overlapped"] = out["ms_single_gpu"] / (world * out["ms_overlapped"])
    out["efficiency_allgather"] = out["ms_single_gpu"] / (world * out["ms_allgather_then_spmm"])
    # algorithmic bytes per layer over all ranks (SURVEY 8d): nnz (4 col + 4 val + 4 d gathered row) + rows (4 d + 8)
    alg = n_layers * (nnz * (8 + 4 * d) + (n_users + n_items) * (4 * d + 8))
    out["algorithmic_gbs_aggregate"] = alg / (best * 1e-3) / 1e9
    out["exchange_bytes_per_layer_per_gpu"] = (world - 1) * plan.slab * d * 4
    return out


def _lookup(rank, world, dev, max_over_ranks, barrier):
    import torch

    from .parallel import PeerShardedTable, RowShardedTable

    res = {}
    for name, n_rows, d, n_ids in (("deepfm_k16", 40_000_000, 16, 819_200), ("din_k64", 8_000_000, 64, 2_000_000)):
        rows_loc = -(-n_rows // world)
        # shard content is a cheap function of the global row id, so every rank can check its lookups
        # (integers below 2^24 only: exactly representable in fp32 whatever the row id)
        gid = torch.arange(rows_loc, device=dev, dtype=torch.int64) * world + rank
        cols = torch.arange(d, device=dev, dtype=torch.float32)[None, :]
        local = ((gid % 65521).to(torch.float32)[:, None] + 0.5 * cols).contiguous()
        g = torch.Generator(device=dev).manual_seed(100 + rank)
        ids = torch.randint(0, n_rows, (n_ids,), device=dev, generator=g)
        expect = (ids % 65521).to(torch.float32)[:, None] + 0.5 * cols
        cross = n_ids * (world - 1) / world * (d * 4)            # row bytes that must arrive over NVLink
        leg = {"rows": n_rows, "d": d, "ids_per_gpu": n_ids, "nvlink_row_bytes_per_gpu": cross}
        nccl = RowShardedTable(local, n_rows)
        got = nccl.lookup(ids)
        leg["nccl_exact"] = bool(torch.equal(got, expect))
        ms = _timed(lambda: nccl.lookup(ids), 10, max_over_ranks, barrier)
        leg["nccl_ms"] = ms
        leg["nccl_nvlink_gbs"] = cross / (ms * 1e-3) / 1e9
        try:
            peer = PeerShardedTable(local, n_rows)
            got = peer.lookup(ids)
            torch.cuda.synchronize()
            leg["peer_exact"] = bool(torch.equal(got, expect))
            out = torch.empty((n_ids, d), dtype=torch.float32, device=dev)
            ms = _timed(lambda: peer.lookup(ids, out=out), 20, max_over_ranks, barrier)
            leg["peer_ms"] = ms
            leg["peer_nvlink_gbs"] = cross / (ms * 1e-3) / 1e9
            leg["peer_frac_of_nvlink_ref"] = leg["peer_nvlink_gbs"] / NVLINK_REF_GBS
            leg["peer_rows_per_s_per_gpu"] = n_ids / (ms * 1e-3)
            # gradient path: push float atomics to the owners, then check one owner-side row sum
            grads = torch.ones((n_ids, d), dtype=torch.float32, device=dev)
            before = peer.local.sum(dtype=torch.float64).item()
            peer.sync()
            peer.scatter_add(ids, grads)
            peer.sync()
            torch.cuda.synchronize()
            after = peer.local.sum(dtype=torch.float64).item()
            tot = torch.tensor([after - before], dtype=torch.float64, device=dev)
            import torch.distributed as dist

            dist.all_reduce(tot)
            leg["peer_scatter_add_total_ok"] = bool(abs(tot.item() - world * n_ids * d) < 1e-3 * world * n_ids * d)
            ms = _timed(lambda: peer.scatter_add(ids, grads), 10, max_over_ranks, barrier)
            leg["peer_scatter_add_ms"] = ms
            del peer
        except Exception as e:
            leg["peer_error"] = repr(e)[:300]
        res[name] = leg
        del nccl, local, ids, expect
        torch.cuda.empty_cache()
    return res


def run(rank, world, dev, max_over_ranks, barrier):
    import torch

    out = {"n_gpus": world}
    try:
        out["lightgcn"] = _lightgcn(rank, world, dev, max_over_ranks, barrier)
    except Exception as e:
        out["lightgcn"] = {"error": repr(e)[:400]}
    torch.cuda.empty_cache()
    try:
        out["row_sharded_lookup"] = _lookup(rank, world, dev, max_over_ranks, barrier)
    except Exception as e:
        out["row_sharded_lookup"] = {"error": repr(e)[:400]}
    torch.cuda.empty_cache()
    return out
