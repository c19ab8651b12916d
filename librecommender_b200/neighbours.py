"""The host engine shared by the neighbourhood models: Swing (``swing.py``) and UserCF / ItemCF (``cf.py``).

An engine holds R (``user_interacts``), its transpose and the consumed CSR on the device, and a neighbour table that
its subclass computes: ``nbr_ids`` int32 / ``nbr_scores`` float32 [n, k] and ``nbr_count`` int64 [n], row q's first
``min(k, nbr_count[q])`` entries its neighbours by (score desc, id asc).  Serving that table is the same for every
engine (``csrc/neighbours.cu``):

* :meth:`NeighbourEngine.recommend_device` accumulates per user into dense rows (``b200_nbr_recommend``), optionally
  draws ``random_rec`` keys (``b200_nbr_random_keys``) and ranks the rows with ``b200_topk_rows``;
* :meth:`NeighbourEngine.predict_device` is ``b200_nbr_predict``: the query's neighbours intersected with a row of R
  (item-based engines) or of R^T (user-based), then recfarm's compute_pred of the engine's task.
"""
from __future__ import annotations

import numpy as np

from . import _lib

MAX_TOP_K = 4096
TASKS = {"rating": 0, "ranking": 1}
_ROW_BYTES = 1 << 28          # recommend: dense score rows per batch


def check_top_k(k, name):
    """``k`` as an int, ``ValueError`` unless it is an integer in [1, MAX_TOP_K]."""
    if isinstance(k, bool) or int(k) != k or not 1 <= int(k) <= MAX_TOP_K:
        raise ValueError(f"{name} must be an integer in [1, {MAX_TOP_K}], got {k!r}")
    return int(k)


def host_csr(m, n_rows, n_cols, name):
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


def transposed_cols(indptr, indices, data=None):
    """Column ids of the transpose's entries in its CSR order (rows of the transpose sorted); with ``data``, also the
    entries' values in that order."""
    rows = np.repeat(np.arange(len(indptr) - 1, dtype=np.int64), np.diff(indptr))
    order = np.lexsort((rows, indices))
    cols = rows[order].astype(np.int32)
    return cols if data is None else (cols, data[order])


class NeighbourEngine:
    """Constructor body and serving of a neighbourhood engine.  A subclass validates its own parameters, calls this
    constructor, computes the table through :meth:`_compute`, and sets:

    * ``user_based``: the table is over users (UserCF) rather than items.  Recommend then walks the user's neighbours'
      rows of R, and predict intersects the user's neighbours with the item's row of R^T;
    * ``uses_item_labels``: the engine reads ``item_interacts``' labels (ItemCF's similarities, UserCF's predict).
      The transpose check then compares them bit for bit, and they are uploaded as ``item_labels``;
    * ``task``: ``"rating"`` or ``"ranking"``, the compute_pred of predict.

    ``user_interacts`` is R (``train_data.sparse_interaction``), ``item_interacts`` its transpose, each a scipy CSR or
    the reference's ``SparseMatrix``; ``user_consumed`` the reference's dict (or a :class:`ConsumedCSR`).  Everything
    is validated on the host, and ``ValueError`` raised, before any launch."""

    user_based = False
    uses_item_labels = True

    def __init__(self, n_users, n_items, user_interacts, item_interacts, user_consumed, default_pred, device, seed):
        import torch

        from .consumed import as_csr

        self.n_users, self.n_items = int(n_users), int(n_items)
        if self.n_users < 1 or self.n_items < 1:
            raise ValueError("n_users and n_items must be >= 1")
        self.default_pred = float(default_pred)
        up, ui, ul = host_csr(user_interacts, self.n_users, self.n_items, "user_interacts")
        ip, iu, il = host_csr(item_interacts, self.n_items, self.n_users, "item_interacts")
        cols, vals = transposed_cols(up, ui, ul)
        if not (np.array_equal(np.diff(ip), np.bincount(ui, minlength=self.n_items)) and np.array_equal(cols, iu)
                and (not self.uses_item_labels or np.array_equal(vals.view(np.uint32), il.view(np.uint32)))):
            raise ValueError("item_interacts is not the transpose of user_interacts")
        consumed = as_csr(user_consumed, self.n_users)
        cons_ptr = consumed.indptr           # a ConsumedCSR may cover fewer users: pad with empty rows
        cons_ptr = np.concatenate([cons_ptr, np.full(max(0, self.n_users + 1 - len(cons_ptr)), cons_ptr[-1])])
        self.device = device if device is not None else _lib.require_cuda()
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)  # noqa: E731
        self.user_ptr, self.user_items, self.user_labels = dev(up), dev(ui), dev(ul)
        self.item_ptr, self.item_users = dev(ip), dev(iu)
        self.item_labels = dev(il) if self.uses_item_labels else None
        self.cons_ptr, self.cons_idx = dev(cons_ptr), dev(consumed.idx)
        self.seed = int(seed)
        self._draws = 0
        self.nbr_ids = self.nbr_scores = self.nbr_count = None
        self._n_elements = 0
        self.workspace_bytes = None

    def _compute(self, n, k, ws_bytes, launch):
        """Compute a new table of ``n`` rows of ``k``: ``launch(ws, ids, scores, count)``, ``ws`` of ``ws_bytes``."""
        import torch

        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.device)
        ids = torch.empty((n, k), dtype=torch.int32, device=self.device)
        scores = torch.empty((n, k), dtype=torch.float32, device=self.device)
        count = torch.empty(n, dtype=torch.int64, device=self.device)
        launch(ws, ids, scores, count)
        self.nbr_ids, self.nbr_scores, self.nbr_count = ids, scores, count
        self._n_elements = int(count.sum().item())
        self.workspace_bytes = ws_bytes

    def _require(self):
        if self.nbr_ids is None:
            raise RuntimeError("compute the neighbours (`compute_swing` / `compute_similarities`) before `predict` / "
                               "`recommend`")

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
        if self.user_based:      # the user's neighbours intersected with the item's row of R^T
            ptr, idx, lab, n_rows, rows, n_q, queries = (self.item_ptr, self.item_users, self.item_labels,
                                                         self.n_items, items, self.n_users, users)
        else:                    # the item's neighbours intersected with the user's row of R
            ptr, idx, lab, n_rows, rows, n_q, queries = (self.user_ptr, self.user_items, self.user_labels,
                                                         self.n_users, users, self.n_items, items)
        _lib.check(_lib.lib.b200_nbr_predict(
            _lib.ptr(ptr), _lib.ptr(idx), _lib.ptr(lab), n_rows, _lib.ptr(self.nbr_ids), _lib.ptr(self.nbr_scores),
            _lib.ptr(self.nbr_count), n_q, self.nbr_ids.shape[1], _lib.ptr(rows), _lib.ptr(queries), users.numel(),
            TASKS[self.task], self.default_pred, _lib.ptr(out), _lib.current_stream()))
        return out

    def predict(self, users, items):
        import torch

        u = torch.as_tensor(np.asarray(users, dtype=np.int64))
        i = torch.as_tensor(np.asarray(items, dtype=np.int64))
        return self.predict_device(u, i).cpu().tolist()

    # ---- recommend -----------------------------------------------------------------------------------------------
    def recommend_device(self, users, n_rec, filter_consumed=True, random_rec=False, seed=None):
        """``(ids int64 [B, k], n int64 [B])`` for an int64 device tensor ``users``, k = min(n_rec, n_items): row r's
        first ``n[r]`` ids are its recommendations, the rest -1.  ``random_rec`` rows with more than ``n_rec``
        candidates draw ``n_rec`` of them uniformly, keyed by ``seed`` (default: the engine's seed and a call
        counter; Philox4x32-10 instead of recfarm's ``thread_rng``)."""
        import torch

        from .engine import masked_topk

        self._require()
        n_rec = int(n_rec)
        if n_rec < 1:
            raise ValueError("n_rec must be >= 1")
        k = min(n_rec, self.n_items)
        if k > MAX_TOP_K:
            raise ValueError(f"n_rec above {MAX_TOP_K} is not supported for a catalogue of {self.n_items} items")
        users = users.to(self.device, torch.int64).contiguous()
        B = users.numel()
        ids = torch.empty((B, k), dtype=torch.int64, device=self.device)
        counts = torch.empty(B, dtype=torch.int64, device=self.device)
        if random_rec and seed is None:
            seed = (self.seed << 20) + self._draws
            self._draws += 1
        chunk = max(1, _ROW_BYTES // (4 * self.n_items))
        stream = _lib.current_stream()
        for r0 in range(0, B, chunk):
            ub = users[r0:r0 + chunk]
            b = ub.numel()
            rows = torch.empty((b, self.n_items), dtype=torch.float32, device=self.device)
            _lib.check(_lib.lib.b200_nbr_recommend(
                _lib.ptr(self.user_ptr), _lib.ptr(self.user_items), _lib.ptr(self.user_labels), self.n_users,
                _lib.ptr(self.nbr_ids), _lib.ptr(self.nbr_scores), _lib.ptr(self.nbr_count), self.n_items,
                self.nbr_ids.shape[1], 1 if self.user_based else 0, _lib.ptr(self.cons_ptr), _lib.ptr(self.cons_idx),
                1 if filter_consumed else 0, _lib.ptr(ub), b, _lib.ptr(rows), self.n_items,
                _lib.ptr(counts[r0:r0 + b]), stream))
            if random_rec:
                _lib.check(_lib.lib.b200_nbr_random_keys(_lib.ptr(rows), self.n_items, b, self.n_items, _lib.ptr(ub),
                                                         _lib.ptr(counts[r0:r0 + b]), n_rec,
                                                         int(seed) & 0xFFFFFFFFFFFFFFFF, stream))
            masked_topk(self, rows, ub, k, False, ids[r0:r0 + b], None)
        n = torch.clamp(counts, max=k)
        ids[torch.arange(k, device=self.device)[None, :] >= n[:, None]] = -1
        return ids, n

    def _recommend_lists(self, users, n_rec, filter_consumed, random_rec):
        """Host lists of :meth:`recommend_device`'s recommendations for the ids ``users``."""
        import torch

        ids, n = self.recommend_device(torch.as_tensor(np.asarray(users, dtype=np.int64)), n_rec, filter_consumed,
                                       random_rec)
        ids, n = ids.cpu().numpy(), n.cpu().numpy()
        return [ids[r, :n[r]].tolist() for r in range(len(n))]

    # ---- introspection -------------------------------------------------------------------------------------------
    def neighbors(self):
        """``(ids int32 [n, k], scores float32 [n, k], count int64 [n])`` on the device: the neighbour table."""
        self._require()
        return self.nbr_ids, self.nbr_scores, self.nbr_count
