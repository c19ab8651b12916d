"""Multi-GPU layout of the recommend path (SURVEY.md §8e row 1): independent users are sharded
across ranks, the item table (+ bf16 catalog) is replicated, there is NO data-path collective.
Only the optional result gather touches the process group.  One process per GPU
(``torchrun``), ``torch.distributed`` for the plumbing (nccl on GPUs, gloo in the CPU tests)."""
from __future__ import annotations

import numpy as np


def shard_bounds(n: int, world: int, rank: int):
    """Contiguous, balanced split of n users: the first n % world ranks take one extra."""
    base, extra = divmod(n, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def shard_users(user_ids, world: int, rank: int):
    user_ids = np.asarray(user_ids)
    lo, hi = shard_bounds(len(user_ids), world, rank)
    return user_ids[lo:hi]


def recommend_sharded(recommend_fn, user_ids, n_rec, group=None, gather=True):
    """Run ``recommend_fn(local_user_ids, n_rec) -> int64[b, n_rec]`` on this rank's shard and
    (optionally) all-gather the ``[B, n_rec]`` result in the original user order on every rank."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group) if dist.is_initialized() else 1
    rank = dist.get_rank(group) if dist.is_initialized() else 0
    local = shard_users(user_ids, world, rank)
    out = recommend_fn(local, n_rec) if len(local) else np.zeros((0, n_rec), dtype=np.int64)
    out = np.asarray(out, dtype=np.int64)
    if world == 1 or not gather:
        return out
    sizes = [shard_bounds(len(user_ids), world, r) for r in range(world)]
    max_rows = max(hi - lo for lo, hi in sizes)
    backend = dist.get_backend(group)
    dev = torch.device("cuda", torch.cuda.current_device()) if backend == "nccl" else torch.device("cpu")
    buf = torch.full((max_rows, n_rec), -1, dtype=torch.int64, device=dev)
    buf[: len(out)] = torch.from_numpy(out).to(dev)
    parts = [torch.empty_like(buf) for _ in range(world)]
    dist.all_gather(parts, buf, group=group)
    rows = [p[: hi - lo].cpu().numpy() for p, (lo, hi) in zip(parts, sizes)]
    return np.concatenate(rows, axis=0)


# ------------------------------------------------------------------------------------------------
# LightGCN propagation over G ranks (SURVEY.md §8e row 3): 1-D row partition of L and E, ONE
# exchange step per layer (all-gather of the [slab, d] blocks), SpMM on the local row block.
# ------------------------------------------------------------------------------------------------
class LightGCNShardPlan:
    """Node -> (rank, slot) layout.  Users and items are dealt round-robin (`id % G`) so that every
    rank owns an equal share of the USERS and of the ITEMS *and* popularity-sorted ids (Zipf heads)
    spread over all ranks: the nnz per rank is balanced without a degree-aware partitioner.  A
    rank's block is ``[su user slots | si item slots]``; the gathered matrix is the concatenation of
    the G blocks (``G * slab`` rows, padding rows are zero and never referenced)."""

    def __init__(self, n_users: int, n_items: int, world: int):
        self.n_users, self.n_items, self.world = int(n_users), int(n_items), int(world)
        self.su = -(-self.n_users // self.world)
        self.si = -(-self.n_items // self.world)
        self.slab = self.su + self.si

    def position(self, nodes):
        """Row of node ids (users 0..n_users-1, items n_users..) in the gathered layout."""
        import torch

        nodes = torch.as_tensor(nodes)
        is_item = nodes >= self.n_users
        u = torch.where(is_item, torch.zeros_like(nodes), nodes)
        i = torch.where(is_item, nodes - self.n_users, torch.zeros_like(nodes))
        pu = (u % self.world) * self.slab + (u // self.world)
        pi = (i % self.world) * self.slab + self.su + (i // self.world)
        return torch.where(is_item, pi, pu)

    def local_nodes(self, rank: int):
        """(node ids owned by `rank` in block order, their slots inside the block)."""
        import torch

        users = torch.arange(min(rank, self.n_users), self.n_users, self.world)   # empty when rank >= n_users
        items = torch.arange(min(rank, self.n_items), self.n_items, self.world)
        nodes = torch.cat([users, self.n_users + items])
        slots = torch.cat([torch.arange(users.numel()), self.su + torch.arange(items.numel())])
        return nodes, slots

    def shard_csr(self, indptr, col, val, rank: int):
        """Rows of `rank` (block order, `slab` rows incl. empty padding rows) of the global CSR, with
        the column ids rewritten to gathered-layout rows.  Tensors stay on the CSR's device."""
        import torch

        dev = indptr.device
        nodes, slots = self.local_nodes(rank)
        nodes, slots = nodes.to(dev), slots.to(dev)
        deg = torch.zeros(self.slab, dtype=torch.int64, device=dev)
        deg[slots] = indptr[nodes + 1] - indptr[nodes]
        lptr = torch.zeros(self.slab + 1, dtype=torch.int64, device=dev)
        lptr[1:] = torch.cumsum(deg, 0)
        # source positions of every local nnz: the owned rows are contiguous runs of the global CSR
        starts = indptr[nodes]
        d_own = indptr[nodes + 1] - starts
        owner = torch.repeat_interleave(torch.arange(nodes.numel(), device=dev), d_own)
        within = torch.arange(int(d_own.sum()), device=dev) - torch.repeat_interleave(
            torch.cumsum(d_own, 0) - d_own, d_own)
        src = starts[owner] + within
        lcol = self.position(col[src].to(torch.int64)).to(torch.int32)
        return lptr, lcol.contiguous(), val[src].contiguous()

    def scatter_rows(self, E_full, rank: int):
        """This rank's `[slab, d]` block of a global `[n_users + n_items, d]` matrix (zeros in padding)."""
        import torch

        nodes, slots = self.local_nodes(rank)
        out = torch.zeros((self.slab, E_full.shape[1]), dtype=E_full.dtype, device=E_full.device)
        out[slots.to(E_full.device)] = E_full[nodes.to(E_full.device)]
        return out

    def unpermute(self, gathered):
        """Gathered layout `[G * slab, d]` -> global node order `[n_users + n_items, d]`."""
        import torch

        pos = self.position(torch.arange(self.n_users + self.n_items)).to(gathered.device)
        return gathered[pos]


def propagate_sharded(plan: LightGCNShardPlan, spmm_local, E0_local, n_layers: int, group=None):
    """mean_{l=0..n_layers} L^l E0 on this rank's row block (lightgcn_module.py:74-88).

    ``spmm_local(E_gathered [G*slab, d], acc [slab, d], final_div) -> out [slab, d]`` multiplies the
    local row block of L (from :meth:`LightGCNShardPlan.shard_csr`) with the gathered layer input,
    adds the product to ``acc`` and divides ``acc`` by ``final_div`` when it is > 0 — exactly the
    fused epilogue of ``b200_spmm_csr`` (:func:`sharded_spmm_fn`).  One ``all_gather_into_tensor``
    per layer is the only collective; the layer mean accumulates locally."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group) if dist.is_initialized() else 1
    assert world == plan.world, (world, plan.world)
    cur = E0_local.contiguous()
    acc = cur.clone()
    if n_layers == 0:
        return acc
    full = torch.empty((plan.world * plan.slab, cur.shape[1]), dtype=cur.dtype, device=cur.device)
    for layer in range(n_layers):
        if world > 1:
            dist.all_gather_into_tensor(full, cur, group=group)
        else:
            full.copy_(cur)
        last = layer == n_layers - 1
        cur = spmm_local(full, acc, float(n_layers + 1) if last else 0.0)
    return acc


def sharded_spmm_fn(local_graph, slab: int):
    """``spmm_local`` for :func:`propagate_sharded` backed by the CUDA SpMM of a local
    :class:`~librecommender_b200.lightgcn.SpmmGraph` (layer-mean epilogue fused)."""
    import torch

    bufs = {}

    def fn(full, acc, final_div):
        key = (full.shape[1], len(bufs) & 1)
        out = bufs.setdefault(key, torch.empty((slab, full.shape[1]), dtype=torch.float32, device=full.device))
        # the last layer's product is only needed inside acc
        local_graph.spmm(full, out=None if final_div > 0 else out, acc=acc, acc_init=False, final_div=final_div)
        return out

    return fn


def gather_embeddings(plan: LightGCNShardPlan, E_local, group=None):
    """All ranks' blocks -> (user_embeds [n_users, d], item_embeds [n_items, d]) on every rank."""
    import torch
    import torch.distributed as dist

    full = torch.empty((plan.world * plan.slab, E_local.shape[1]), dtype=E_local.dtype, device=E_local.device)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_gather_into_tensor(full, E_local.contiguous(), group=group)
    else:
        full.copy_(E_local)
    out = plan.unpermute(full)
    return out[: plan.n_users], out[plan.n_users:]


# ------------------------------------------------------------------------------------------------
# Row-sharded embedding table (SURVEY.md §8e row 2): engaged only when a table exceeds one GPU.
# Row r lives on rank r % G at slot r // G.  A lookup is index all-to-all -> local gather -> row
# all-to-all; the gradient path mirrors it (rows to the owners, local scatter-add).
# ------------------------------------------------------------------------------------------------
def _cuda_gather(local_rows, slots):
    import torch

    from . import _lib

    out = torch.empty((slots.numel(), local_rows.shape[1]), dtype=torch.float32, device=local_rows.device)
    _lib.check(_lib.lib.b200_gather_rows(_lib.ptr(local_rows), local_rows.stride(0), local_rows.shape[1],
                                         _lib.ptr(slots), slots.numel(), _lib.ptr(out), out.stride(0),
                                         _lib.current_stream()))
    return out


def _cuda_scatter_add(local_rows, slots, rows):
    from . import _lib

    _lib.check(_lib.lib.b200_scatter_add_rows(_lib.ptr(local_rows), local_rows.stride(0), local_rows.shape[1],
                                              _lib.ptr(slots), slots.numel(), _lib.ptr(rows), rows.stride(0),
                                              _lib.current_stream()))


class RowShardedTable:
    """One rank's slice ``local_rows [ceil(n_rows / G), d]`` of a table sharded by ``row % G``.

    ``lookup(ids)``: every rank passes ITS OWN ids (its slice of the batch) and gets its rows.
    ``scatter_add(ids, grads)``: the transposed exchange, ``table[ids] += grads`` on the owners.
    ``gather_fn`` / ``scatter_fn`` default to the CUDA kernels; the CPU gloo test injects torch
    stand-ins for exactly these two local operations."""

    def __init__(self, local_rows, n_rows: int, group=None, gather_fn=None, scatter_fn=None):
        import torch.distributed as dist

        self.local, self.n_rows, self.group = local_rows, int(n_rows), group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.gather_fn = gather_fn or _cuda_gather
        self.scatter_fn = scatter_fn or _cuda_scatter_add

    @staticmethod
    def shard(full_table, world: int, rank: int):
        """Rows rank, rank + G, ... of a full table (how a checkpoint is split)."""
        return full_table[rank::world].contiguous()

    def _route(self, ids):
        """Sort the request by owner: (order, per-owner counts sent / received, remote slots received)."""
        import torch
        import torch.distributed as dist

        ids = ids.to(torch.int64)
        owner = ids % self.world
        order = torch.argsort(owner, stable=True)
        send_counts = torch.bincount(owner, minlength=self.world)
        recv_counts = torch.empty_like(send_counts)
        if self.world > 1:
            dist.all_to_all_single(recv_counts, send_counts, group=self.group)
        else:
            recv_counts.copy_(send_counts)
        send_l, recv_l = send_counts.tolist(), recv_counts.tolist()
        slots_out = (ids[order] // self.world).contiguous()
        slots_in = torch.empty(int(sum(recv_l)), dtype=torch.int64, device=ids.device)
        if self.world > 1:
            dist.all_to_all_single(slots_in, slots_out, recv_l, send_l, group=self.group)
        else:
            slots_in.copy_(slots_out)
        return order, send_l, recv_l, slots_in

    def lookup(self, ids):
        import torch
        import torch.distributed as dist

        order, send_l, recv_l, slots_in = self._route(ids)
        rows_out = self.gather_fn(self.local, slots_in)                 # rows other ranks asked this rank for
        d = self.local.shape[1]
        rows_in = torch.empty((int(sum(send_l)), d), dtype=rows_out.dtype, device=rows_out.device)
        if self.world > 1:
            dist.all_to_all_single(rows_in, rows_out.contiguous(), [c for c in send_l], [c for c in recv_l],
                                   group=self.group)
        else:
            rows_in.copy_(rows_out)
        out = torch.empty_like(rows_in)
        out[order] = rows_in                                            # back to the caller's order
        return out

    def scatter_add(self, ids, grads):
        import torch
        import torch.distributed as dist

        order, send_l, recv_l, slots_in = self._route(ids)
        g_out = grads[order].contiguous()
        g_in = torch.empty((int(sum(recv_l)), grads.shape[1]), dtype=grads.dtype, device=grads.device)
        if self.world > 1:
            dist.all_to_all_single(g_in, g_out, recv_l, send_l, group=self.group)
        else:
            g_in.copy_(g_out)
        self.scatter_fn(self.local, slots_in, g_in)


# ------------------------------------------------------------------------------------------------
# Row-sharded table over NVLink PEER MEMORY (SURVEY.md §8e row 2).  Every rank's
# shard lives in symmetric memory (torch.distributed._symmetric_memory: CUDA VMM allocations
# mapped into every process of the node), so one CUDA kernel per direction does the gather AND
# the exchange (`b200_peer_gather_rows` / `b200_peer_scatter_add_rows`): no bucketing by owner, no
# index all-to-all, no row all-to-all, no host synchronisation.
# ------------------------------------------------------------------------------------------------
class PeerShardedTable:
    """``local_rows``: this rank's ``[ceil(n_rows / G), d]`` shard (rows rank, rank + G, ...).
    ``lookup(ids)`` -> ``[len(ids), d]`` rows for ANY global ids; ``scatter_add(ids, grads)`` adds
    into the owners' shards; ``sync()`` is a stream-ordered barrier over all ranks (signal pads in
    the symmetric allocation) — call it between a phase that writes the table and one that reads."""

    def __init__(self, local_rows, n_rows: int, group=None):
        import ctypes

        import torch
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm

        self.group = group if group is not None else dist.group.WORLD
        self.world = dist.get_world_size(self.group)
        self.rank = dist.get_rank(self.group)
        self.n_rows, self.d = int(n_rows), int(local_rows.shape[1])
        rows_loc = -(-self.n_rows // self.world)
        dev = local_rows.device
        self.local = symm.empty((rows_loc, self.d), dtype=torch.float32, device=dev)
        self.local.zero_()
        self.local[: local_rows.shape[0]].copy_(local_rows)
        self.handle = symm.rendezvous(self.local, self.group)
        ptrs = [int(p) for p in self.handle.buffer_ptrs]
        self._shards = (ctypes.c_void_p * self.world)(*ptrs)
        self.sync()

    def sync(self):
        self.handle.barrier(channel=0)

    def lookup(self, ids, out=None):
        import torch

        from . import _lib

        ids = ids.to(torch.int64).contiguous()
        n = int(ids.numel())
        if out is None:
            out = torch.empty((n, self.d), dtype=torch.float32, device=ids.device)
        _lib.check(_lib.lib.b200_peer_gather_rows(self._shards, self.world, self.local.stride(0), self.d,
                                                  _lib.ptr(ids), n, _lib.ptr(out), out.stride(0),
                                                  _lib.current_stream()))
        return out

    def scatter_add(self, ids, grads):
        import torch

        from . import _lib

        ids = ids.to(torch.int64).contiguous()
        grads = grads.contiguous()
        _lib.check(_lib.lib.b200_peer_scatter_add_rows(self._shards, self.world, self.local.stride(0), self.d,
                                                       _lib.ptr(ids), int(ids.numel()), _lib.ptr(grads),
                                                       grads.stride(0), _lib.current_stream()))


# ------------------------------------------------------------------------------------------------
# LightGCN propagation with the exchange OVERLAPPED with the SpMM (SURVEY.md §8e row 3: "chunked so
# SpMM on column block g starts as soon as slab g lands").  The local row block of L is split by
# SOURCE RANK of the column into G sub-matrices; per layer the own block multiplies at once, and
# block g multiplies as soon as slab g has arrived.  Two exchange engines:
#   * ring   — G-1 steps of paired isend / irecv (NCCL on GPUs, gloo in the CPU tests);
#   * peer   — the slabs live in symmetric memory and every rank PULLS its peers' slabs with the
#              copy engines over NVLink (no SM, no NCCL), ordered by one device-side barrier per layer.
# The layer product is accumulated block by block (deterministic order: own block, then source
# ranks r-1, r-2, ...), so it agrees with the single-GPU result to float rounding (not bit-for-bit;
# `propagate_sharded` above is the bit-exact, non-overlapped variant).
# ------------------------------------------------------------------------------------------------
def split_column_blocks(lptr, lcol, lval, slab: int, world: int):
    """Local CSR (columns in the gathered layout, `world * slab` of them) -> one CSR per source rank
    with block-local column ids.  The order of the entries inside a row is preserved."""
    import torch

    dev = lptr.device
    n_rows = lptr.numel() - 1
    deg = lptr[1:] - lptr[:-1]
    rows = torch.repeat_interleave(torch.arange(n_rows, device=dev), deg)
    blk = (lcol.to(torch.int64) // slab)
    out = []
    for g in range(world):
        sel = torch.nonzero(blk == g).flatten()               # ascending: row order and in-row order kept
        ptr = torch.zeros(n_rows + 1, dtype=torch.int64, device=dev)
        ptr[1:] = torch.cumsum(torch.bincount(rows[sel], minlength=n_rows), 0)
        out.append((ptr, (lcol[sel].to(torch.int64) - g * slab).to(torch.int32).contiguous(), lval[sel].contiguous()))
    return out


class RingExchange:
    """Slab exchange by G-1 paired isend / irecv steps; works with nccl (CUDA tensors, on a side
    stream) and gloo (CPU tensors, synchronous)."""

    def __init__(self, world, rank, group=None):
        self.world, self.rank, self.group = world, rank, group
        self._stream = None

    def start(self, cur, slots):
        """Begin the exchange of `cur` [slab, d]; slots[g] receives rank g's slab.  Returns a list of
        (source rank, wait_fn) in arrival order; wait_fn() makes the CURRENT stream wait for that slab."""
        import torch
        import torch.distributed as dist

        arrivals = []
        if self.world == 1:
            return arrivals
        cuda = cur.is_cuda
        if cuda:
            if self._stream is None:
                self._stream = torch.cuda.Stream(device=cur.device)
            ready = torch.cuda.Event()
            ready.record()                               # `cur` is complete on the compute stream here
            self._stream.wait_event(ready)
        for s in range(1, self.world):
            dst, src = (self.rank + s) % self.world, (self.rank - s) % self.world
            ops = [dist.P2POp(dist.isend, cur, dst, self.group), dist.P2POp(dist.irecv, slots[src], src, self.group)]
            if cuda:
                with torch.cuda.stream(self._stream):
                    works = dist.batch_isend_irecv(ops)
                    for w in works:
                        w.wait()                         # side stream waits for the NCCL op
                    ev = torch.cuda.Event()
                    ev.record(self._stream)
                arrivals.append((src, (lambda e=ev: torch.cuda.current_stream().wait_event(e))))
            else:
                works = dist.batch_isend_irecv(ops)
                arrivals.append((src, (lambda ws=works: [w.wait() for w in ws])))
        return arrivals

    def make_slabs(self, slab, d, device, dtype):
        """(list of G receive buffers, 2 ping-pong `cur` buffers)."""
        import torch

        self.gathered = torch.zeros((self.world * slab, d), dtype=dtype, device=device)     # slot g = rank g's slab
        return ([self.gathered[g * slab:(g + 1) * slab] for g in range(self.world)],
                [torch.empty((slab, d), dtype=dtype, device=device) for _ in range(2)])


class PeerPullExchange:
    """Slabs in symmetric memory: after one device-side barrier every rank pulls its peers' slabs with
    cudaMemcpyAsync (copy engines over NVLink) on side streams; the SMs only run the SpMM."""

    def __init__(self, world, rank, group=None):
        self.world, self.rank, self.group = world, rank, group
        self._streams = None
        self._cur_syms = None

    def make_slabs(self, slab, d, device, dtype):
        import torch
        import torch.distributed as dist
        import torch.distributed._symmetric_memory as symm

        grp = self.group if self.group is not None else dist.group.WORLD
        self._cur = [symm.empty((slab, d), dtype=dtype, device=device) for _ in range(2)]
        self._hdl = [symm.rendezvous(t, grp) for t in self._cur]
        self._shape, self._dtype = (slab, d), dtype
        self._streams = [torch.cuda.Stream(device=device) for _ in range(2)]
        self.gathered = torch.zeros((self.world * slab, d), dtype=dtype, device=device)     # slot g = rank g's slab
        return ([self.gathered[g * slab:(g + 1) * slab] for g in range(self.world)], self._cur)

    def start(self, cur, slots):
        import torch

        arrivals = []
        if self.world == 1:
            return arrivals
        which = 0 if cur.data_ptr() == self._cur[0].data_ptr() else 1
        hdl = self._hdl[which]
        hdl.barrier(channel=which)            # every rank's `cur` of this layer is complete (stream-ordered)
        ready = torch.cuda.Event()
        ready.record()
        for s in range(1, self.world):
            src = (self.rank - s) % self.world
            st = self._streams[s & 1]
            st.wait_event(ready)
            with torch.cuda.stream(st):
                remote = hdl.get_buffer(src, self._shape, self._dtype)
                slots[src].copy_(remote, non_blocking=True)          # peer -> local over NVLink (DMA)
                ev = torch.cuda.Event()
                ev.record(st)
            arrivals.append((src, (lambda e=ev: torch.cuda.current_stream().wait_event(e))))
        return arrivals


def propagate_sharded_overlap(plan: LightGCNShardPlan, block_spmm, E0_local, n_layers: int, exchange,
                              rank: int):
    """mean_{l=0..n_layers} L^l E0 on this rank's row block with the slab exchange overlapped with the
    per-source-rank block products.  ``block_spmm(g, E_g [slab, d], acc)`` adds ``L[:, block g] @ E_g``
    to ``acc`` (CUDA: ``SpmmGraph.spmm(..., acc=acc, acc_init=False)`` of the g-th column block from
    :func:`split_column_blocks`)."""
    import torch

    slab, d = E0_local.shape
    if not hasattr(exchange, "_bufs") or exchange._bufs[0][0].shape != (slab, d):
        exchange._bufs = exchange.make_slabs(slab, d, E0_local.device, E0_local.dtype)
    slots, curs = exchange._bufs
    cur = curs[0]
    cur.copy_(E0_local)
    acc = E0_local.clone()
    for layer in range(n_layers):
        nxt = curs[(layer + 1) & 1]
        arrivals = exchange.start(cur, slots)
        nxt.zero_()
        block_spmm(rank, cur, nxt)                       # own block: no communication needed
        for src, wait in arrivals:
            wait()
            block_spmm(src, slots[src], nxt)
        acc.add_(nxt)
        cur = nxt
    acc.div_(float(n_layers + 1))
    return acc


def split_local_remote(lptr, lcol, lval, slab: int, rank: int):
    """Local CSR (columns in the gathered layout) -> (own-block CSR with block-local columns, CSR of every OTHER
    block with the gathered-layout columns kept).  Two products per layer instead of one per source rank: the
    own block needs no communication and runs while the peers' slabs arrive; the rest runs once over the
    gathered buffer.  In-row order preserved."""
    import torch

    dev = lptr.device
    n_rows = lptr.numel() - 1
    deg = lptr[1:] - lptr[:-1]
    rows = torch.repeat_interleave(torch.arange(n_rows, device=dev), deg)
    own = (lcol.to(torch.int64) // slab) == rank
    out = []
    for mask, shift in ((own, rank * slab), (~own, 0)):
        sel = torch.nonzero(mask).flatten()
        ptr = torch.zeros(n_rows + 1, dtype=torch.int64, device=dev)
        ptr[1:] = torch.cumsum(torch.bincount(rows[sel], minlength=n_rows), 0)
        out.append((ptr, (lcol[sel].to(torch.int64) - shift).to(torch.int32).contiguous(), lval[sel].contiguous()))
    return out[0], out[1]


def propagate_sharded_two_phase(plan: LightGCNShardPlan, local_spmm, remote_spmm, E0_local, n_layers: int,
                                exchange, rank: int):
    """mean_{l=0..n_layers} L^l E0 on this rank's row block, two products per layer: ``local_spmm(E_own [slab, d],
    acc)`` adds the own column block while the peers' slabs are in flight, ``remote_spmm(gathered [G * slab, d],
    acc)`` adds every other block once they have all arrived (CSRs from :func:`split_local_remote`)."""
    slab, d = E0_local.shape
    if not hasattr(exchange, "_bufs") or exchange._bufs[0][0].shape != (slab, d):
        exchange._bufs = exchange.make_slabs(slab, d, E0_local.device, E0_local.dtype)
    slots, curs = exchange._bufs
    cur = curs[0]
    cur.copy_(E0_local)
    acc = E0_local.clone()
    for layer in range(n_layers):
        nxt = curs[(layer + 1) & 1]
        arrivals = exchange.start(cur, slots)
        nxt.zero_()
        local_spmm(cur, nxt)
        for _, wait in arrivals:
            wait()
        if arrivals:
            remote_spmm(exchange.gathered, nxt)
        acc.add_(nxt)
        cur = nxt
    acc.div_(float(n_layers + 1))
    return acc


def acc_spmm_fn(graph):
    """``E, acc -> acc += L_part @ E`` backed by the CUDA SpMM of one :class:`SpmmGraph`."""

    def fn(E, acc):
        if graph.nnz:
            graph.spmm(E, out=None, acc=acc, acc_init=False, final_div=0.0)

    return fn


def block_spmm_fn(block_graphs):
    """``block_spmm`` backed by the CUDA SpMM of the per-source-rank :class:`SpmmGraph` objects."""

    def fn(g, E_block, acc):
        if block_graphs[g].nnz:
            block_graphs[g].spmm(E_block, out=None, acc=acc, acc_init=False, final_div=0.0)

    return fn


# ------------------------------------------------------------------------------------------------
# OOV rows of sharded tables (SURVEY.md 8e row 5): the mean row (assign_embedding_oov,
# bases/embed_base.py:257-265; assign_tf_variables_oov, bases/tf_base.py:310-353) of a table whose rows
# live on several ranks = local partial sums + ONE all-reduce.
# ------------------------------------------------------------------------------------------------
def sharded_mean_row(local_rows, n_local_valid: int, n_rows_global: int, group=None):
    """Mean over the `n_rows_global` real rows of a table sharded over the ranks; `local_rows[:n_local_valid]`
    are this rank's real rows (shard padding and the OOV slot itself excluded).  Accumulates in float64."""
    import torch
    import torch.distributed as dist

    part = local_rows[:n_local_valid].sum(dim=0, dtype=torch.float64)
    if dist.is_initialized() and dist.get_world_size(group) > 1:
        dist.all_reduce(part, group=group)
    return (part / float(n_rows_global)).to(local_rows.dtype)


# ------------------------------------------------------------------------------------------------
# Item-sharded recommend (SURVEY.md 8e row 1, the variant for an item table larger than one GPU): the ITEMS are
# split by id range, every rank scores all B users against its shard (the fused tensor-core path on the shard),
# keeps its local top-K with exact scores, and ONE exchange step — an all-gather of (id, score)[B, K] — is followed
# by a K-way merge on the device (b200_topk_rows over the G*K gathered candidates per row).  Exact scores do not
# depend on the sharding and the candidates of a row arrive ordered (shard, score desc, id asc), so the merge
# reproduces the single-GPU total order (score desc, item id asc) bit for bit.
# ------------------------------------------------------------------------------------------------
def restrict_consumed_to_shard(indptr, idx, item_lo: int, item_hi: int):
    """Consumed CSR (numpy ``indptr int64[n_users+1]``, ``idx int32[nnz]``, global item ids, arrival order kept)
    -> the same users' lists restricted to items in ``[item_lo, item_hi)`` with shard-local ids."""
    indptr = np.asarray(indptr, dtype=np.int64)
    idx = np.asarray(idx)
    keep = (idx >= item_lo) & (idx < item_hi)
    counts = np.add.reduceat(keep.astype(np.int64), indptr[:-1]) if len(idx) else np.zeros(len(indptr) - 1, np.int64)
    counts[indptr[:-1] == indptr[1:]] = 0            # reduceat on an empty segment returns the next element
    lptr = np.zeros(len(indptr), dtype=np.int64)
    np.cumsum(counts, out=lptr[1:])
    return lptr, (idx[keep] - item_lo).astype(np.int32)


def merge_topk_shards(ids, scores, n_rec: int):
    """``ids`` int64 ``[G, B, K]`` (global item ids, -1 = no candidate), ``scores`` fp32 ``[G, B, K]`` (device
    tensors, each shard's rows sorted by (score desc, id asc)) -> ``(ids [B, n_rec], scores [B, n_rec])`` of the
    merged order.  One b200_topk_rows over the ``G*K`` candidates of a row; positions index the concatenation
    (shard-major), which is ascending in item id among equal scores."""
    import ctypes

    import torch

    from . import _lib

    G, B, K = ids.shape
    cat_ids = ids.permute(1, 0, 2).reshape(B, G * K).contiguous()
    cat_sc = scores.permute(1, 0, 2).reshape(B, G * K).contiguous().clone()
    cat_sc[cat_ids < 0] = float("-inf")
    ld = (G * K + 3) // 4 * 4
    if ld != G * K:
        pad = torch.full((B, ld), float("-inf"), dtype=torch.float32, device=cat_sc.device)
        pad[:, :G * K] = cat_sc
        cat_sc = pad
    pos = torch.empty((B, n_rec), dtype=torch.int64, device=cat_sc.device)
    out_sc = torch.empty((B, n_rec), dtype=torch.float32, device=cat_sc.device)
    nbytes = ctypes.c_size_t(0)
    _lib.check(_lib.lib.b200_topk_rows_workspace_bytes(B, G * K, n_rec, ctypes.byref(nbytes)))
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=cat_sc.device)
    _lib.check(_lib.lib.b200_topk_rows(_lib.ptr(cat_sc), cat_sc.stride(0), B, G * K, n_rec, _lib.ptr(pos), _lib.ptr(out_sc),
                                       _lib.ptr(ws), nbytes.value, _lib.current_stream()))
    return torch.gather(cat_ids, 1, pos), out_sc


class ItemShardScorer:
    """One rank's shard ``I[item_lo:item_hi]`` of an item-sharded catalogue + the full user table; ``local_topk``
    returns the shard's best ``n_rec`` items per user with GLOBAL ids and exact scores (the fused tensor-core path on
    the shard, flagged rows repaired on the exact path as always)."""

    def __init__(self, user_embeddings, item_shard, item_lo: int, consumed_indptr=None, consumed_idx=None,
                 n_users=None, device=None):
        from .consumed import ConsumedCSR
        from .engine import EmbedScorer

        self.item_lo = int(item_lo)
        self.n_local = int(item_shard.shape[0])
        csr, self.max_consumed = None, 0
        if consumed_indptr is not None:
            indptr = np.asarray(consumed_indptr, dtype=np.int64)
            self.max_consumed = int((indptr[1:] - indptr[:-1]).max()) if len(indptr) > 1 else 0
            lptr, lidx = restrict_consumed_to_shard(indptr, consumed_idx, self.item_lo, self.item_lo + self.n_local)
            csr = ConsumedCSR(lptr, lidx)
        # EmbedScorer wants an [n_items + 1, d] table (last row = the OOV item, never scored)
        import torch

        shard = torch.as_tensor(item_shard) if not isinstance(item_shard, torch.Tensor) else item_shard
        pad = torch.zeros((1, shard.shape[1]), dtype=shard.dtype, device=shard.device)
        self.scorer = EmbedScorer(user_embeddings, torch.cat([shard, pad], dim=0), self.n_local, csr, n_users=n_users,
                                  device=device)

    def local_topk(self, user_ids_d, n_rec: int):
        if n_rec + self.max_consumed > self.n_local:
            raise ValueError(f"item shard of {self.n_local} rows is too small for n_rec {n_rec} + {self.max_consumed} "
                             "consumed items (the consumed-filter rule of ranking.py:38 is evaluated per shard)")
        ids, scores = self.scorer.recommend_device(user_ids_d, n_rec, True, True)
        return ids + self.item_lo, scores


def recommend_item_sharded(shard: ItemShardScorer, user_ids_d, n_rec: int, group=None, all_gather=None, merge=None):
    """All B users against this rank's item shard, all-gather of the ``(id, score)[B, n_rec]`` candidates, K-way merge:
    every rank returns the global ``(ids [B, n_rec], scores [B, n_rec])``.  ``all_gather(t) -> [G, ...]`` defaults to
    ``torch.distributed.all_gather_into_tensor`` (tests inject a stand-in to run several shards in one process);
    ``merge`` defaults to :func:`merge_topk_shards` (CUDA; the gloo CPU test injects a numpy stand-in)."""
    import torch
    import torch.distributed as dist

    ids, scores = shard.local_topk(user_ids_d, n_rec)
    if all_gather is None:
        world = dist.get_world_size(group) if dist.is_initialized() else 1
        if world == 1:
            return ids, scores

        def all_gather(t):
            out = torch.empty((world * t.shape[0],) + tuple(t.shape[1:]), dtype=t.dtype, device=t.device)
            dist.all_gather_into_tensor(out, t.contiguous(), group=group)      # concatenated along dim 0 (nccl and gloo)
            return out.view((world,) + tuple(t.shape))
    return (merge or merge_topk_shards)(all_gather(ids), all_gather(scores), n_rec)
