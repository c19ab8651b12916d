"""Device-resident state for the embed scoring path.

``EmbedScorer`` keeps the user / item embedding tables and the consumed-CSR in
HBM and answers ``recommend`` calls: H2D of the user ids, score → mask → top-K on
the GPU, D2H of the ``[B, n_rec]`` ids.  It is what
``recommend_from_embedding`` (reference: ``libreco/recommendation/recommend.py:57-78``)
runs on; tables are uploaded once per (array object) and cached.
"""
from __future__ import annotations

import ctypes
import os

import numpy as np

from . import _lib
from .consumed import ConsumedCSR, as_csr

_SCORE_WS_BYTES = 1 << 30  # materialised-score workspace of the exact path
FUSED_MAX_D = 256           # limits of b200_recommend_embed (include/b200reco.h)
FUSED_MAX_K = 288
FUSED_ROWS_PER_CALL = 32768    # users per b200_recommend_embed launch on the device path (+3 % per user over 16384)
HOST_ROWS_PER_CALL = 16384     # host seam: smaller launches so that a chunk's D2H / the next chunk's id conversion overlap kernels
NVTX = bool(int(os.environ.get("B200_NVTX", "0")))     # B200_NVTX=1: NVTX ranges around the phases of a recommend call


class _nvtx:
    """``with _nvtx("name"):`` — an NVTX range when B200_NVTX=1 (nsys / ncu --nvtx timelines), free otherwise."""

    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if NVTX:
            import torch

            torch.cuda.nvtx.range_push(self.name)

    def __exit__(self, *exc):
        if NVTX:
            import torch

            torch.cuda.nvtx.range_pop()
        return False



def _as_device_f32(x, device):
    import torch

    if isinstance(x, torch.Tensor):
        t = x.to(device=device, dtype=torch.float32)
    else:
        a = np.asarray(x)
        if a.dtype != np.float32:
            a = a.astype(np.float32)
        t = torch.from_numpy(np.ascontiguousarray(a)).to(device)
    if t.dim() == 1:
        t = t[:, None]
    return t.contiguous()


def masked_topk(owner, scores, user_ids_d, n_rec, filter_consumed, out_ids, out_scores):
    """Consumed filter + top-``n_rec`` of the device fp32 score rows ``scores`` [b, ld] (clobbered by the mask) of
    the users ``user_ids_d`` into ``out_ids`` / ``out_scores`` (nullable).  ``owner`` holds the catalogue size
    ``n_items`` and the consumed CSR (``csr`` with its device arrays ``indptr_d``, ``idx_d``)."""
    import torch

    b, ld = scores.shape[0], scores.stride(0)
    N = owner.n_items
    stream = _lib.current_stream()
    if filter_consumed and owner.csr.nnz > 0:
        _lib.check(_lib.lib.b200_mask_consumed(
            _lib.ptr(scores), ld, _lib.ptr(user_ids_d), b, N, n_rec,
            _lib.ptr(owner.indptr_d), _lib.ptr(owner.idx_d), owner.csr.n_users, stream))
    nbytes = ctypes.c_size_t(0)
    _lib.check(_lib.lib.b200_topk_rows_workspace_bytes(b, N, n_rec, ctypes.byref(nbytes)))
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=scores.device)
    _lib.check(_lib.lib.b200_topk_rows(
        _lib.ptr(scores), ld, b, N, n_rec, _lib.ptr(out_ids), _lib.ptr(out_scores), _lib.ptr(ws), nbytes.value, stream))


class EmbedScorer:
    """Score-all-items + consumed filter + top-K for embedding models (a1 + a2)."""

    def __init__(self, user_embeddings, item_embeddings, n_items, user_consumed=None,
                 n_users=None, device=None):
        import torch

        self.device = device if device is not None else _lib.require_cuda()
        self.U = _as_device_f32(user_embeddings, self.device)
        self.I = _as_device_f32(item_embeddings, self.device)
        if self.U.shape[1] != self.I.shape[1]:
            raise ValueError("user and item embeddings differ in width")
        self.d = int(self.U.shape[1])
        self.n_items = int(n_items)
        if self.n_items > self.I.shape[0]:
            raise ValueError("n_items exceeds rows of item_embeddings")
        self.n_users = int(n_users) if n_users is not None else int(self.U.shape[0])
        self.set_consumed(user_consumed)
        self._torch = torch
        self.events = None  # optional list collecting (start, stop) CUDA events of the sweep kernel
        self.last_fallback_rows = 0   # rows of the latest call that were repaired on the exact path
        self.catalog = None
        if self.d <= FUSED_MAX_D:
            self._prepare_catalog()

    def _prepare_catalog(self):
        """bf16 K-major copy of the item table + max row norm (once per table)."""
        torch = self._torch if hasattr(self, "_torch") else __import__("torch")
        nbytes = ctypes.c_size_t(0)
        _lib.check(_lib.lib.b200_embed_catalog_bytes(self.n_items, self.d, ctypes.byref(nbytes)))
        self.catalog = torch.empty(nbytes.value, dtype=torch.uint8, device=self.device)
        _lib.check(_lib.lib.b200_embed_catalog_prepare(
            _lib.ptr(self.I), self.I.stride(0), self.n_items, self.d, _lib.ptr(self.catalog),
            nbytes.value, _lib.current_stream()))

    def set_consumed(self, user_consumed):
        if user_consumed is None:
            user_consumed = ConsumedCSR(np.zeros(1, dtype=np.int64), np.zeros(0, dtype=np.int32))
        self.csr = as_csr(user_consumed, self.n_users)
        self.indptr_d, self.idx_d = self.csr.device(self.device)

    # ------------------------------------------------------------------------------------
    def topk_scores_inplace(self, scores, user_ids_d, n_rec, filter_consumed, out_ids, out_scores):
        """scores: device fp32 [b, ld] (clobbered by the mask)."""
        masked_topk(self, scores, user_ids_d, n_rec, filter_consumed, out_ids, out_scores)

    def recommend_exact(self, user_ids_d, n_rec, filter_consumed=True, return_scores=False):
        """Exact fp32 path: materialise score row-batches, mask, radix top-K."""
        torch = self._torch
        B = int(user_ids_d.numel())
        N = self.n_items
        if n_rec > N:
            raise ValueError(f"`n_rec` {n_rec} exceeds num of items {N}")
        ld = (N + 3) // 4 * 4
        rows = max(1, min(B, _SCORE_WS_BYTES // (ld * 4), 32768))
        scores = torch.empty((rows, ld), dtype=torch.float32, device=self.device)
        out_ids = torch.empty((B, n_rec), dtype=torch.int64, device=self.device)
        out_scores = torch.empty((B, n_rec), dtype=torch.float32, device=self.device) if return_scores else None
        stream = _lib.current_stream()
        for r0 in range(0, B, rows):
            b = min(rows, B - r0)
            uid = user_ids_d[r0:r0 + b]
            _lib.check(_lib.lib.b200_score_rows_f32(
                _lib.ptr(self.U), self.U.stride(0), _lib.ptr(uid), b,
                _lib.ptr(self.I), self.I.stride(0), N, self.d,
                _lib.ptr(scores), ld, stream))
            self.topk_scores_inplace(
                scores[:b], uid, n_rec, filter_consumed, out_ids[r0:r0 + b],
                out_scores[r0:r0 + b] if return_scores else None)
        return (out_ids, out_scores) if return_scores else out_ids

    def fused_ok(self, n_rec) -> bool:
        return self.catalog is not None and n_rec <= FUSED_MAX_K

    def fused_plan(self, B, n_rec) -> dict:
        """How ``b200_recommend_embed`` will run a call of ``B`` users (``b200_recommend_embed_plan``):
        whether the speculative pre-pass is used, the item splits, the epilogue organisation."""
        out = (ctypes.c_int32 * 8)()
        _lib.check(_lib.lib.b200_recommend_embed_plan(min(int(B), FUSED_ROWS_PER_CALL), self.n_items, self.d,
                                                      int(n_rec), out, 8))
        keys = ("use_pre", "n_splits", "tiles_per_split", "m_tiles", "n_pre_tiles", "tma_stages",
                "cluster_x10_plus_mma_groups", "records_per_list")
        return dict(zip(keys, [int(v) for v in out]))

    def _fused_chunk(self, uid_chunk, n_rec, use_filter, out_ids, out_scores, status, n_flagged=None):
        """One ``b200_recommend_embed`` call (<= FUSED_ROWS_PER_CALL rows) on the current stream; ``n_flagged``:
        address of an int32 that receives the chunk's count of rows with a non-zero status, or None."""
        torch = self._torch
        b = int(uid_chunk.numel())
        nbytes = ctypes.c_size_t(0)
        _lib.check(_lib.lib.b200_recommend_embed_workspace_bytes(b, self.n_items, self.d, n_rec, ctypes.byref(nbytes)))
        ws = self._workspace(nbytes.value)
        ev0 = ev1 = None
        if self.events is not None:
            e0 = torch.cuda.Event(enable_timing=True)
            e1 = torch.cuda.Event(enable_timing=True)
            e0.record()   # creates the cudaEvent_t; re-recorded inside the C-ABI call
            e1.record()
            ev0, ev1 = ctypes.c_void_p(e0.cuda_event), ctypes.c_void_p(e1.cuda_event)
        _lib.check(_lib.lib.b200_recommend_embed(
            _lib.ptr(self.U), self.U.stride(0), _lib.ptr(uid_chunk), b,
            _lib.ptr(self.I), self.I.stride(0), self.n_items, self.d, _lib.ptr(self.catalog),
            _lib.ptr(self.indptr_d), _lib.ptr(self.idx_d), self.csr.n_users, use_filter, n_rec,
            _lib.ptr(out_ids), _lib.ptr(out_scores) if out_scores is not None else None,
            _lib.ptr(status), _lib.ptr(ws), nbytes.value, _lib.current_stream(), ev0, ev1, n_flagged))
        if self.events is not None:
            self.events.append((e0, e1))

    def recommend_fused(self, user_ids_d, n_rec, filter_consumed=True, return_scores=False, on_chunk=None,
                        before_chunk=None, rows_per_call=None, n_flagged=None):
        """Tensor-core path (b200_recommend_embed).  Returns (ids, scores|None, status):
        rows with status != 0 hold -1 ids and must be re-run on the exact path.  ``on_chunk(r0, r1)``
        is called after the kernels of rows [r0, r1) have been enqueued, ``before_chunk(r0, r1)`` just before
        (the host seam fills ``user_ids_d[r0:r1]`` there, so converting the ids of chunk i+1 overlaps the kernels
        of chunk i).  ``n_flagged``: pinned host int32 tensor with a word per chunk, which receives the chunk's
        count of rows with a non-zero status in stream order."""
        torch = self._torch
        B = int(user_ids_d.numel())
        N = self.n_items
        if n_rec > N:
            raise ValueError(f"`n_rec` {n_rec} exceeds num of items {N}")
        out_ids = torch.empty((B, n_rec), dtype=torch.int64, device=self.device)
        out_scores = torch.empty((B, n_rec), dtype=torch.float32, device=self.device) if return_scores else None
        status = torch.empty(B, dtype=torch.int32, device=self.device)
        use_filter = 1 if (filter_consumed and self.csr.nnz > 0) else 0
        step = int(rows_per_call or FUSED_ROWS_PER_CALL)
        for r0 in range(0, B, step):
            r1 = min(B, r0 + step)
            if before_chunk is not None:
                before_chunk(r0, r1)
            self._fused_chunk(user_ids_d[r0:r1], n_rec, use_filter, out_ids[r0:r1],
                              out_scores[r0:r1] if return_scores else None, status[r0:r1],
                              None if n_flagged is None else n_flagged[r0 // step].data_ptr())
            if on_chunk is not None:
                on_chunk(r0, r1)
        return out_ids, out_scores, status

    def _workspace(self, nbytes):
        ws = getattr(self, "_ws", None)
        if ws is None or ws.numel() < nbytes:
            self._ws = None
            ws = self._torch.empty(int(nbytes), dtype=self._torch.uint8, device=self.device)
            self._ws = ws
        return ws

    def recommend_device_async(self, user_ids_d, n_rec, filter_consumed=True, return_scores=False,
                               path="auto"):
        """Enqueue one recommend call on the current stream and return a handle WITHOUT synchronising;
        ``handle.result()`` performs the (rare) exact-path repair of rows the fused path flagged and
        returns the device tensors.  Lets a server keep the next batch in flight while the previous
        one is checked."""
        n_rec = int(n_rec)
        if path == "exact" or (path == "auto" and not self.fused_ok(n_rec)):
            return _Pending(self, user_ids_d, n_rec, filter_consumed, return_scores,
                            self.recommend_exact(user_ids_d, n_rec, filter_consumed, return_scores), None)
        # the flagged-row count of every chunk lands in a pinned word right after the chunk's kernels, so that
        # result() waits for this call only and not for a call enqueued after it
        torch = self._torch
        step = FUSED_ROWS_PER_CALL
        slot = self._pinned("flagged", (max(1, -(-int(user_ids_d.numel()) // step)),), torch.int32)
        slot[0].zero_()
        ids, scores, status = self.recommend_fused(user_ids_d, n_rec, filter_consumed, return_scores,
                                                   rows_per_call=step, n_flagged=slot[0])
        done = torch.cuda.Event()
        done.record()
        return _Pending(self, user_ids_d, n_rec, filter_consumed, return_scores,
                        (ids, scores) if return_scores else ids, status, (self._export(slot), done))

    def recommend_device(self, user_ids_d, n_rec, filter_consumed=True, return_scores=False,
                         path="auto"):
        """Device ids in, device results out; flagged rows are re-run on the exact path."""
        return self.recommend_device_async(user_ids_d, n_rec, filter_consumed, return_scores, path).result()

    def score_rows(self, user_ids_d):
        """Materialised exact fp32 scores [B, n_items] (used by the random_rec branch)."""
        torch = self._torch
        B = int(user_ids_d.numel())
        N = self.n_items
        ld = (N + 3) // 4 * 4
        scores = torch.empty((B, ld), dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_score_rows_f32(
            _lib.ptr(self.U), self.U.stride(0), _lib.ptr(user_ids_d), B,
            _lib.ptr(self.I), self.I.stride(0), N, self.d, _lib.ptr(scores), ld,
            _lib.current_stream()))
        return scores[:, :N]

    def _pinned(self, name, shape, dtype):
        """Pinned host staging buffer for one result.  The reference contract is "a fresh ndarray
        per call": the numpy array handed to the caller VIEWS the pinned buffer, and a buffer is
        recycled only after that array (and every view derived from it) has been garbage collected
        (tracked with a weak reference) — never while the caller can still read it."""
        torch = self._torch
        pool = self.__dict__.setdefault("_pin_pool", {})
        key = (name, tuple(shape), dtype)
        slots = pool.setdefault(key, [])
        for slot in slots:
            if slot[1] is None or slot[1]() is None:
                return slot
        if sum(len(v) for v in pool.values()) >= 64:      # the caller keeps everything: drop dead shapes
            for k in [k for k, v in pool.items() if k != key and all(s[1] is None or s[1]() is None for s in v)]:
                del pool[k]
        slot = [torch.empty(shape, dtype=dtype, pin_memory=True), None]
        slots.append(slot)
        return slot

    @staticmethod
    def _export(slot):
        """numpy view of a pinned slot, registered so that the slot is not reused while it lives."""
        import weakref

        arr = slot[0].numpy()
        slot[1] = weakref.ref(arr)
        return arr

    def recommend(self, user_ids, n_rec, filter_consumed=True, return_scores=False, path="auto"):
        """Host ids in, host ``int64[B, n_rec]`` out (the reference-facing call): one H2D of the
        ids, the kernels, one D2H of ids (+ the per-row status) and a single synchronisation."""
        torch = self._torch
        n_rec = int(n_rec)
        fill = None
        fused = not (path == "exact" or (path == "auto" and not self.fused_ok(n_rec)))
        if isinstance(user_ids, list) and fused and len(user_ids) > HOST_ROWS_PER_CALL:
            # a long python list (the reference's calling convention): converted and uploaded chunk by chunk, the
            # conversion of chunk i+1 runs while the kernels of chunk i execute
            import array

            uid_d = torch.empty(len(user_ids), dtype=torch.int64, device=self.device)

            def fill(r0, r1, _lst=user_ids):
                with _nvtx("b200.recommend.h2d_ids"):
                    uid_d[r0:r1].copy_(torch.frombuffer(array.array("q", _lst[r0:r1]), dtype=torch.int64),
                                       non_blocking=True)
        else:
            if isinstance(user_ids, torch.Tensor):
                uid_h = user_ids.to(torch.int64)
            elif isinstance(user_ids, list):
                # the reference passes a python list of inner ids: array.array's C loop is the fastest way in
                import array

                uid_h = torch.frombuffer(array.array("q", user_ids), dtype=torch.int64) if user_ids else \
                    torch.zeros(0, dtype=torch.int64)
            else:
                uid_h = torch.as_tensor(np.asarray(user_ids, dtype=np.int64))
            with _nvtx("b200.recommend.h2d_ids"):
                uid_d = uid_h.to(self.device, non_blocking=True)
        B = int(uid_d.numel())
        if path == "exact" or (path == "auto" and not self.fused_ok(n_rec)):
            res = self.recommend_exact(uid_d, n_rec, filter_consumed, return_scores)
            if return_scores:
                return res[0].cpu().numpy(), res[1].cpu().numpy()
            return res.cpu().numpy()
        ids_slot = self._pinned("ids", (B, n_rec), torch.int64)
        st_slot = self._pinned("status", (B,), torch.int32)
        sc_slot = self._pinned("scores", (B, n_rec), torch.float32) if return_scores else None
        # the D2H of chunk i runs on a side stream while the kernels of chunk i+1 execute
        main = torch.cuda.current_stream()
        side = self.__dict__.get("_copy_stream")
        if side is None:
            side = self._copy_stream = torch.cuda.Stream(device=self.device)
        res = {}

        def on_chunk(r0, r1):
            ev = torch.cuda.Event()
            ev.record(main)
            res.setdefault("chunks", []).append((r0, r1, ev))

        with _nvtx("b200.recommend.fused_kernels"):
            ids_d, sc_d, status_d = self.recommend_fused(uid_d, n_rec, filter_consumed, return_scores, on_chunk, fill,
                                                         rows_per_call=min(HOST_ROWS_PER_CALL, FUSED_ROWS_PER_CALL))
        with _nvtx("b200.recommend.d2h_results"), torch.cuda.stream(side):
            for r0, r1, ev in res.get("chunks", []):
                side.wait_event(ev)
                ids_slot[0][r0:r1].copy_(ids_d[r0:r1], non_blocking=True)
                st_slot[0][r0:r1].copy_(status_d[r0:r1], non_blocking=True)
                if return_scores:
                    sc_slot[0][r0:r1].copy_(sc_d[r0:r1], non_blocking=True)
        with _nvtx("b200.recommend.sync"):
            side.synchronize()
        for t in (ids_d, sc_d, status_d):            # the side stream used them: keep the allocator informed
            if t is not None:
                t.record_stream(side)
        ids = self._export(ids_slot)
        scores = self._export(sc_slot) if return_scores else None
        bad = np.flatnonzero(st_slot[0].numpy())
        self.last_fallback_rows = int(len(bad))
        if len(bad):                       # rows the fused path could not prove: exact path
            bad_d = torch.as_tensor(bad, device=self.device)
            with _nvtx("b200.recommend.exact_repair"):
                fix = self.recommend_exact(uid_d[bad_d], n_rec, filter_consumed, return_scores)
            if return_scores:
                ids[bad], scores[bad] = fix[0].cpu().numpy(), fix[1].cpu().numpy()
            else:
                ids[bad] = fix.cpu().numpy()
        return (ids, scores) if return_scores else ids

    def predict(self, users, items, mode=0, lo=0.0, hi=0.0):
        """predict_from_embedding (``libreco/prediction/predict.py:36-40``)."""
        torch = self._torch
        u = torch.as_tensor(np.asarray(users, dtype=np.int64)).to(self.device)
        i = torch.as_tensor(np.asarray(items, dtype=np.int64)).to(self.device)
        out = torch.empty(u.numel(), dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_gather_dot(
            _lib.ptr(self.U), self.U.stride(0), _lib.ptr(u), _lib.ptr(self.I), self.I.stride(0),
            _lib.ptr(i), u.numel(), self.d, mode, lo, hi, _lib.ptr(out), _lib.current_stream()))
        return out.cpu().numpy()


class _Pending:
    """Result handle of :meth:`EmbedScorer.recommend_device_async`."""

    def __init__(self, scorer, uid_d, n_rec, filter_consumed, return_scores, res, status, flagged=None):
        self.scorer, self.uid_d, self.n_rec = scorer, uid_d, n_rec
        self.filter_consumed, self.return_scores = filter_consumed, return_scores
        self.res, self.status = res, status
        self.flagged = flagged     # (pinned per-chunk counts of flagged rows, event recorded after the call)

    def result(self):
        if self.status is not None:
            torch = self.scorer._torch
            counts, done = self.flagged
            done.synchronize()            # this call's kernels only; the only synchronisation unless a row is flagged
            self.scorer.last_fallback_rows = int(counts.sum())
            if self.scorer.last_fallback_rows:
                bad = torch.nonzero(self.status).flatten()
                fix = self.scorer.recommend_exact(self.uid_d[bad], self.n_rec, self.filter_consumed,
                                                  self.return_scores)
                if self.return_scores:
                    self.res[0][bad], self.res[1][bad] = fix[0], fix[1]
                else:
                    self.res[bad] = fix
            self.status = self.flagged = None
        return self.res


# ---- cache of scorers: identity of the host arrays + a content fingerprint ----------------------
_scorers: dict = {}


def _fingerprint(a):
    """Cheap content token of a host array: shape, data pointer and the float64 sum of a strided
    sample (<= 64 Ki elements, ends included).  The reference's ALS / BPR update
    ``user_embeds_np`` / ``item_embeds_np`` IN PLACE every epoch (``als.py:153-168``) and call
    ``recommend_user`` in between: such an update changes (practically) every sampled element, so
    the cached device tables are refreshed.  A point edit of a row the sample does not touch is
    not seen — call :func:`invalidate_scorers` after one."""
    if hasattr(a, "data_ptr"):                      # torch tensor (host or device)
        flat = a.detach().reshape(-1)
        n = int(flat.numel())
        step = max(1, n // 65536)
        return (tuple(a.shape), int(a.data_ptr()), float(flat[::step].double().sum()), float(flat[-1]) if n else 0.0)
    arr = np.asarray(a)
    flat = arr.reshape(-1)
    n = flat.size
    step = max(1, n // 65536)
    return (arr.shape, int(arr.ctypes.data), float(flat[::step].sum(dtype=np.float64)), float(flat[-1]) if n else 0.0)


def invalidate_scorers():
    """Drop every cached device copy (after editing embeddings / consumed lists in place)."""
    _scorers.clear()


def scorer_for(model, user_embeddings, item_embeddings) -> EmbedScorer:
    key = (id(user_embeddings), id(item_embeddings), int(model.n_items))
    fp = (_fingerprint(user_embeddings), _fingerprint(item_embeddings))
    hit = _scorers.get(key)
    if (hit is not None and hit[0] is user_embeddings and hit[1] is item_embeddings
            and hit[2] is model.user_consumed and hit[3] == fp):
        return hit[4]
    n_users = getattr(model, "n_users", None)
    sc = EmbedScorer(user_embeddings, item_embeddings, model.n_items, model.user_consumed,
                     n_users=n_users)
    if len(_scorers) > 4:
        _scorers.clear()
    _scorers[key] = (user_embeddings, item_embeddings, model.user_consumed, fp, sc)
    return sc
