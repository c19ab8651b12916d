"""Swing on the device: the ``recfarm.Swing`` engine that ``libreco/algorithms/swing.py`` drives, on the kernels of
``csrc/swing.cu`` and the library's ``b200_topk_rows``.

* :meth:`Swing.compute_swing` builds, per item, its first ``top_k`` swing neighbours by (score desc, id asc) and its
  number of nonzero scores (``b200_swing_scores``).  ``recommend`` and ``predict`` only ever read those first
  ``top_k`` entries (``rust/src/swing.rs:167-168,209-210``), so nothing else is kept.
* :meth:`Swing.recommend` accumulates ``label * score`` per user into dense rows (``b200_swing_recommend``), ranks them
  with ``b200_topk_rows`` and returns ``(recs, additional counts)`` as recfarm does.  With ``random_rec`` a row with
  more than ``n_rec`` candidates draws ``n_rec`` distinct candidates uniformly, keyed by the engine's seed and a call
  counter (Philox4x32-10) instead of recfarm's ``thread_rng``.
* :meth:`Swing.predict` is ``b200_swing_predict``: one warp per (user, item).

``num_threads`` (``compute_swing``) and ``max_cache_num`` (the constructor) are accepted for recfarm's signature and
ignored: the device needs no thread count and caches no common-item lists.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np

from . import _lib

MAX_TOP_K = 4096
_ROW_BYTES = 1 << 28          # recommend: dense score rows per batch


def _host_csr(m, n_rows, n_cols, name):
    """(indptr int64 [n_rows+1], indices int32, data float32) of a scipy CSR or of the reference's ``SparseMatrix``
    (``sparse_indices`` / ``sparse_indptr`` / ``sparse_data``, ``libreco/utils/sparse.py``).  A matrix with fewer rows
    than ``n_rows`` (scipy infers the shape from the largest id) is padded with empty rows.  ``ValueError`` unless
    every row is sorted and duplicate-free with ids in ``[0, n_cols)``."""
    if hasattr(m, "sparse_indptr"):
        indptr, indices, data = m.sparse_indptr, m.sparse_indices, m.sparse_data
    elif hasattr(m, "indptr"):
        indptr, indices, data = m.indptr, m.indices, m.data
    else:
        raise ValueError(f"{name} is neither a CSR matrix nor a SparseMatrix")
    indptr = np.asarray(indptr, dtype=np.int64)
    indices = np.asarray(indices, dtype=np.int64)
    data = np.asarray(data, dtype=np.float32)
    if indptr.ndim != 1 or len(indptr) < 1 or indptr[0] != 0 or indptr[-1] != len(indices) or len(data) != len(
            indices) or np.any(np.diff(indptr) < 0):
        raise ValueError(f"{name} is not a CSR")
    rows = len(indptr) - 1
    if rows > n_rows:
        raise ValueError(f"{name} has {rows} rows, more than {n_rows}")
    if len(indices) and (indices.min() < 0 or indices.max() >= n_cols):
        raise ValueError(f"{name} holds ids outside [0, {n_cols})")
    if len(indices) > 1:
        step = np.diff(indices)
        same_row = np.ones(len(indices) - 1, dtype=bool)
        starts = indptr[1:-1]
        same_row[starts[(starts > 0) & (starts < len(indices))] - 1] = False
        if np.any(step[same_row] <= 0):
            raise ValueError(f"{name} has a row that is not sorted or holds a duplicate")
    indptr = np.concatenate([indptr, np.full(n_rows - rows, indptr[-1], dtype=np.int64)])
    return indptr, indices.astype(np.int32), data


def validate(top_k, alpha):
    if isinstance(top_k, bool) or int(top_k) != top_k or not 1 <= int(top_k) <= MAX_TOP_K:
        raise ValueError(f"top_k must be an integer in [1, {MAX_TOP_K}], got {top_k!r}")
    alpha = float(alpha)
    if not math.isfinite(alpha) or alpha < 0 or alpha > float(np.finfo(np.float32).max):
        raise ValueError(f"alpha must be finite and >= 0, got {alpha!r}")
    return int(top_k), alpha


class Swing:
    """Device engine with the method contract of ``recfarm.Swing`` (``rust/src/swing.rs``)::

        Swing(top_k, alpha, max_cache_num, n_users, n_items, user_interacts, item_interacts, user_consumed,
              default_pred)

    ``user_interacts`` is R (``train_data.sparse_interaction``), ``item_interacts`` its transpose, each a scipy CSR or
    the reference's ``SparseMatrix``; ``user_consumed`` the reference's dict (or a :class:`ConsumedCSR`).  Everything
    is validated on the host, and ``ValueError`` raised, before any launch."""

    def __init__(self, top_k, alpha, max_cache_num, n_users, n_items, user_interacts, item_interacts,
                 user_consumed, default_pred, device=None, seed=42):
        import torch

        from .consumed import as_csr

        self.top_k, self.alpha = validate(top_k, alpha)
        self.max_cache_num = max_cache_num          # no cache on the device
        self.n_users, self.n_items = int(n_users), int(n_items)
        if self.n_users < 1 or self.n_items < 1:
            raise ValueError("n_users and n_items must be >= 1")
        self.default_pred = float(default_pred)
        up, ui, ul = _host_csr(user_interacts, self.n_users, self.n_items, "user_interacts")
        ip, iu, _ = _host_csr(item_interacts, self.n_items, self.n_users, "item_interacts")
        if not (np.array_equal(np.diff(ip), np.bincount(ui, minlength=self.n_items))
                and np.array_equal(_transposed_cols(up, ui), iu)):
            raise ValueError("item_interacts is not the transpose of user_interacts")
        consumed = as_csr(user_consumed, self.n_users)
        cons_ptr = consumed.indptr           # a ConsumedCSR may cover fewer users: pad with empty rows
        cons_ptr = np.concatenate([cons_ptr, np.full(max(0, self.n_users + 1 - len(cons_ptr)), cons_ptr[-1])])
        self.device = device if device is not None else _lib.require_cuda()
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)  # noqa: E731
        self.user_ptr, self.user_items, self.user_labels = dev(up), dev(ui), dev(ul)
        self.item_ptr, self.item_users = dev(ip), dev(iu)
        self.cons_ptr, self.cons_idx = dev(cons_ptr), dev(consumed.idx)
        self.seed = int(seed)
        self._draws = 0
        self.nbr_ids = self.nbr_scores = self.nbr_count = None
        self._n_elements = None
        self.workspace_bytes = None

    # ---- scores --------------------------------------------------------------------------------------------------
    def compute_swing(self, num_threads=1):
        """Swing scores of every item (``num_threads`` is ignored)."""
        import torch

        n = ctypes.c_size_t(0)
        _lib.check(_lib.lib.b200_swing_scores_workspace_bytes(self.n_users, self.n_items, self.top_k,
                                                               ctypes.byref(n)))
        ws = torch.empty(n.value, dtype=torch.uint8, device=self.device)
        ids = torch.empty((self.n_items, self.top_k), dtype=torch.int32, device=self.device)
        scores = torch.empty((self.n_items, self.top_k), dtype=torch.float32, device=self.device)
        count = torch.empty(self.n_items, dtype=torch.int64, device=self.device)
        _lib.check(_lib.lib.b200_swing_scores(
            _lib.ptr(self.user_ptr), _lib.ptr(self.user_items), self.n_users, _lib.ptr(self.item_ptr),
            _lib.ptr(self.item_users), self.n_items, self.alpha, self.top_k, _lib.ptr(ids), _lib.ptr(scores),
            _lib.ptr(count), _lib.ptr(ws), n.value, _lib.current_stream()))
        self.nbr_ids, self.nbr_scores, self.nbr_count = ids, scores, count
        self._n_elements = int(count.sum().item())
        self.workspace_bytes = n.value

    def num_swing_elements(self):
        """Total number of nonzero swing scores.  Like recfarm, ``RuntimeError`` when no item has any (before
        ``compute_swing`` in particular)."""
        if not self._n_elements:
            raise RuntimeError("call `compute_swing` method before calling `num_swing_elements`")
        return self._n_elements

    def _require(self):
        if self.nbr_ids is None:
            raise RuntimeError("call `compute_swing` before `predict` / `recommend`")

    # ---- predict -------------------------------------------------------------------------------------------------
    def predict_device(self, users, items):
        """float32 [n] predictions for int64 device tensors ``users`` / ``items``."""
        import torch

        self._require()
        users = users.to(self.device, torch.int64).contiguous()
        items = items.to(self.device, torch.int64).contiguous()
        if users.shape != items.shape or users.dim() != 1:
            raise ValueError("users and items must be 1-d and of the same length")
        out = torch.empty(users.numel(), dtype=torch.float32, device=self.device)
        _lib.check(_lib.lib.b200_swing_predict(
            _lib.ptr(self.user_ptr), _lib.ptr(self.user_items), self.n_users, _lib.ptr(self.nbr_ids),
            _lib.ptr(self.nbr_scores), _lib.ptr(self.nbr_count), self.n_items, self.top_k, _lib.ptr(users),
            _lib.ptr(items), users.numel(), self.default_pred, _lib.ptr(out), _lib.current_stream()))
        return out

    def predict(self, users, items):
        import torch

        u = torch.as_tensor(np.asarray(users, dtype=np.int64))
        i = torch.as_tensor(np.asarray(items, dtype=np.int64))
        return self.predict_device(u, i).cpu().tolist()

    # ---- recommend -----------------------------------------------------------------------------------------------
    def recommend_device(self, users, n_rec, filter_consumed=True, random_rec=False, seed=None):
        """``(ids int64 [B, k], n int64 [B])`` for an int64 device tensor ``users``, k = min(n_rec, n_items): row r's
        first ``n[r]`` ids are its recommendations, the rest -1.  ``seed`` keys the ``random_rec`` draw (default: the
        engine's seed and a call counter)."""
        self._require()

        def accumulate(ub, rows, counts, stream):
            _lib.check(_lib.lib.b200_swing_recommend(
                _lib.ptr(self.user_ptr), _lib.ptr(self.user_items), _lib.ptr(self.user_labels), self.n_users,
                _lib.ptr(self.nbr_ids), _lib.ptr(self.nbr_scores), _lib.ptr(self.nbr_count), self.n_items, self.top_k,
                _lib.ptr(self.cons_ptr), _lib.ptr(self.cons_idx), 1 if filter_consumed else 0, _lib.ptr(ub),
                ub.numel(), _lib.ptr(rows), self.n_items, _lib.ptr(counts), stream))

        return recommend_rows(self, accumulate, users, n_rec, random_rec, seed)

    def recommend(self, users, n_rec, filter_consumed=True, random_rec=False):
        """recfarm's ``recommend``: ``(recs, additional counts)``, ``recs[r]`` the ids of user r as a list and
        ``additional[r] = n_rec - len(recs[r])``."""
        import torch

        ids, n = self.recommend_device(torch.as_tensor(np.asarray(users, dtype=np.int64)), n_rec, filter_consumed,
                                       random_rec)
        ids, n = ids.cpu().numpy(), n.cpu().numpy()
        recs = [ids[r, :n[r]].tolist() for r in range(len(n))]
        return recs, [int(n_rec) - int(c) for c in n]

    # ---- introspection -------------------------------------------------------------------------------------------
    def neighbors(self):
        """``(ids int32 [n_items, top_k], scores float32 [n_items, top_k], count int64 [n_items])`` on the device."""
        self._require()
        return self.nbr_ids, self.nbr_scores, self.nbr_count


def _transposed_cols(indptr, indices, data=None):
    """Column ids of the transpose's entries in its CSR order (rows of the transpose sorted); with ``data``, also the
    entries' values in that order."""
    rows = np.repeat(np.arange(len(indptr) - 1, dtype=np.int64), np.diff(indptr))
    order = np.lexsort((rows, indices))
    cols = rows[order].astype(np.int32)
    return cols if data is None else (cols, data[order])


def recommend_rows(eng, accumulate, users, n_rec, random_rec=False, seed=None):
    """Batched recommend of a neighbourhood engine ``eng`` (``n_items``, ``device``, ``seed``, the consumed CSR):
    ``accumulate(ub, rows, counts, stream)`` fills the dense score rows [b, n_items] of the users ``ub`` (REMOVED where
    untouched) and their candidate counts; ``random_rec`` rows with more than ``n_rec`` candidates then get
    ``b200_swing_random_keys``, and ``masked_topk`` ranks every row.  Returns ``(ids int64 [B, k], n int64 [B])``,
    k = min(n_rec, n_items), row r's first ``n[r]`` ids its recommendations and the rest -1."""
    import torch

    from .engine import masked_topk

    n_rec = int(n_rec)
    if n_rec < 1:
        raise ValueError("n_rec must be >= 1")
    k = min(n_rec, eng.n_items)
    if k > MAX_TOP_K:
        raise ValueError(f"n_rec above {MAX_TOP_K} is not supported for a catalogue of {eng.n_items} items")
    users = users.to(eng.device, torch.int64).contiguous()
    B = users.numel()
    ids = torch.empty((B, k), dtype=torch.int64, device=eng.device)
    counts = torch.empty(B, dtype=torch.int64, device=eng.device)
    if random_rec and seed is None:
        seed = (eng.seed << 20) + eng._draws
        eng._draws += 1
    chunk = max(1, _ROW_BYTES // (4 * eng.n_items))
    stream = _lib.current_stream()
    for r0 in range(0, B, chunk):
        ub = users[r0:r0 + chunk]
        b = ub.numel()
        rows = torch.empty((b, eng.n_items), dtype=torch.float32, device=eng.device)
        accumulate(ub, rows, counts[r0:r0 + b], stream)
        if random_rec:
            _lib.check(_lib.lib.b200_swing_random_keys(_lib.ptr(rows), eng.n_items, b, eng.n_items, _lib.ptr(ub),
                                                       _lib.ptr(counts[r0:r0 + b]), n_rec,
                                                       int(seed) & 0xFFFFFFFFFFFFFFFF, stream))
        masked_topk(eng, rows, ub, k, False, ids[r0:r0 + b], None)
    n = torch.clamp(counts, max=k)
    ids[torch.arange(k, device=eng.device)[None, :] >= n[:, None]] = -1
    return ids, n


def plan(n_items, top_k):
    """``(shared-memory accumulator?, resident CTAs)`` of ``b200_swing_scores`` on the current device."""
    smem, ctas = ctypes.c_int32(0), ctypes.c_int32(0)
    _lib.check(_lib.lib.b200_swing_plan(int(n_items), int(top_k), ctypes.byref(smem), ctypes.byref(ctas)))
    return bool(smem.value), int(ctas.value)


def fit_reference_model(model, ref_module, train_data, neg_sampling, verbose=1, eval_data=None, metrics=None, k=10,
                        eval_batch_size=8192, eval_user_num=None):
    """``Swing.fit`` of the reference (``libreco/algorithms/swing.py:65-116``) with this engine as ``model.rs_model``
    in place of ``recfarm.Swing``; ``ref_module`` is that module, whose helpers it calls.  A model prepared by
    ``rebuild_model`` (``model.incremental``) raises ``NotImplementedError``: the device engine has no incremental
    update."""
    if model.incremental:
        raise NotImplementedError("the device Swing engine does not update a rebuilt model; fit a new one")
    ref_module.check_fitting(model, train_data, eval_data, neg_sampling, k)
    model.show_start_time()
    R = train_data.sparse_interaction
    model.rs_model = Swing(model.top_k, model.alpha, model.max_cache_num, model.n_users, model.n_items, R,
                           R.T.tocsr(), model.user_consumed, model.default_pred, seed=model.seed)
    with ref_module.time_block("swing computing", verbose=1):
        model.rs_model.compute_swing(model.num_threads)
    num = model.rs_model.num_swing_elements()
    print(f"swing num_elements: {num}, density: {100 * num / (model.n_items * model.n_items):5.4f} %")
    if verbose > 1:
        ref_module.print_metrics(model=model, neg_sampling=neg_sampling, eval_data=eval_data, metrics=metrics,
                                 eval_batch_size=eval_batch_size, k=k, sample_user_num=eval_user_num, seed=model.seed)
        print("=" * 30)
