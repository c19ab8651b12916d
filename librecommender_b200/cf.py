"""UserCF and ItemCF on the device: the ``recfarm.UserCF`` / ``recfarm.ItemCF`` engines that
``libreco/bases/cf_base_rs.py`` drives (``RsUserCF`` / ``RsItemCF``), on the kernels of ``csrc/cf.cu``, Swing's serving
kernels (``csrc/swing.cu``) and the library's ``b200_topk_rows``.

* :meth:`compute_similarities` builds, per row of the "sim side" (items for ItemCF, users for UserCF), its first
  ``k_sim`` cosine neighbours by (cosine desc, id asc) and its kept count: every other row sharing at least
  ``min_common`` interactions, zero cosines included (``b200_cf_cosine``).  ``recommend`` and ``predict`` only ever
  read those first ``k_sim`` entries (``item_cf.rs:375,421``, ``user_cf.rs:828,870``), so nothing else is kept.
* :meth:`recommend` accumulates ``sim * label`` per user into dense rows (ItemCF: ``b200_swing_recommend`` on the
  item neighbour table; UserCF: ``b200_user_cf_recommend``), ranks them with ``b200_topk_rows`` and returns
  ``(recs, no_rec_indices)`` as recfarm does.  With ``random_rec`` a row with more than ``n_rec`` candidates draws
  ``n_rec`` distinct candidates uniformly (Philox4x32-10 instead of recfarm's ``thread_rng``).
* :meth:`predict` is ``b200_cf_predict``: the query's neighbours intersected with the other CSR's row, then
  compute_pred of the engine's task.

``invert`` and ``num_threads`` (``compute_similarities``) are accepted for recfarm's signature and ignored: both
recfarm modes compute the same similarities, and the device runs one algorithm.
"""
from __future__ import annotations

import ctypes

import numpy as np

from . import _lib
from .swing import MAX_TOP_K, _host_csr, _transposed_cols, recommend_rows

TASKS = {"rating": 0, "ranking": 1}


def validate(task, k_sim, min_common):
    if task not in TASKS:
        raise ValueError(f"task must be 'rating' or 'ranking', got {task!r}")
    if isinstance(k_sim, bool) or int(k_sim) != k_sim or not 1 <= int(k_sim) <= MAX_TOP_K:
        raise ValueError(f"k_sim must be an integer in [1, {MAX_TOP_K}], got {k_sim!r}")
    if isinstance(min_common, bool) or int(min_common) != min_common or int(min_common) < 1:
        raise ValueError(f"min_common must be an integer >= 1, got {min_common!r}")
    return task, int(k_sim), int(min_common)


def workspace_bytes(n_x, k_sim):
    """Bytes of ``b200_cf_cosine``'s workspace for ``n_x`` sim-side rows on the current device."""
    n = ctypes.c_size_t(0)
    _lib.check(_lib.lib.b200_cf_cosine_workspace_bytes(int(n_x), int(k_sim), ctypes.byref(n)))
    return n.value


def plan(n_x, k_sim):
    """``(shared-memory accumulator?, resident CTAs)`` of ``b200_cf_cosine`` on the current device."""
    smem, ctas = ctypes.c_int32(0), ctypes.c_int32(0)
    _lib.check(_lib.lib.b200_cf_plan(int(n_x), int(k_sim), ctypes.byref(smem), ctypes.byref(ctas)))
    return bool(smem.value), int(ctas.value)


class _CfEngine:
    """Shared body of :class:`ItemCF` and :class:`UserCF`, recfarm's constructor::

        ItemCF(task, k_sim, n_users, n_items, min_common, user_interacts, item_interacts, user_consumed, default_pred)

    ``user_interacts`` is R (``train_data.sparse_interaction``), ``item_interacts`` its transpose, each a scipy CSR or
    the reference's ``SparseMatrix``; ``user_consumed`` the reference's dict (or a :class:`ConsumedCSR`).  Everything
    is validated on the host, and ``ValueError`` raised, before any launch."""

    user_based = False

    def __init__(self, task, k_sim, n_users, n_items, min_common, user_interacts, item_interacts, user_consumed,
                 default_pred, device=None, seed=42):
        import torch

        from .consumed import as_csr

        self.task, self.k_sim, self.min_common = validate(task, k_sim, min_common)
        self.n_users, self.n_items = int(n_users), int(n_items)
        if self.n_users < 1 or self.n_items < 1:
            raise ValueError("n_users and n_items must be >= 1")
        self.default_pred = float(default_pred)
        up, ui, ul = _host_csr(user_interacts, self.n_users, self.n_items, "user_interacts")
        ip, iu, il = _host_csr(item_interacts, self.n_items, self.n_users, "item_interacts")
        cols, vals = _transposed_cols(up, ui, ul)
        if not (np.array_equal(np.diff(ip), np.bincount(ui, minlength=self.n_items)) and np.array_equal(cols, iu)
                and np.array_equal(vals.view(np.uint32), il.view(np.uint32))):
            raise ValueError("item_interacts is not the transpose of user_interacts")
        consumed = as_csr(user_consumed, self.n_users)
        cons_ptr = consumed.indptr           # a ConsumedCSR may cover fewer users: pad with empty rows
        cons_ptr = np.concatenate([cons_ptr, np.full(max(0, self.n_users + 1 - len(cons_ptr)), cons_ptr[-1])])
        self.device = device if device is not None else _lib.require_cuda()
        dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(self.device)  # noqa: E731
        self.user_ptr, self.user_items, self.user_labels = dev(up), dev(ui), dev(ul)
        self.item_ptr, self.item_users, self.item_labels = dev(ip), dev(iu), dev(il)
        self.cons_ptr, self.cons_idx = dev(cons_ptr), dev(consumed.idx)
        self.seed = int(seed)
        self._draws = 0
        self.nbr_ids = self.nbr_scores = self.nbr_count = None
        self._n_elements = 0
        self.workspace_bytes = None

    # the CSR whose rows are compared, and its transpose
    def _sides(self):
        users = (self.user_ptr, self.user_items, self.user_labels, self.n_users)
        items = (self.item_ptr, self.item_users, self.item_labels, self.n_items)
        return (users, items) if self.user_based else (items, users)

    # ---- similarities --------------------------------------------------------------------------------------------
    def compute_similarities(self, invert=True, num_threads=1):
        """Cosine neighbours of every sim-side row (``invert`` and ``num_threads`` are ignored).  ``ValueError`` when
        the workspace does not fit in the device's free memory."""
        import torch

        (sp_, si, sv, n_x), (mp, mi, mv, n_y) = self._sides()
        n = workspace_bytes(n_x, self.k_sim)
        out_bytes = n_x * self.k_sim * 8 + n_x * 8
        free = torch.cuda.mem_get_info(self.device)[0]
        if n + out_bytes > free:
            raise ValueError(f"the similarity workspace of {n_x} rows needs {n + out_bytes} bytes, more than the "
                             f"{free} free on {self.device}")
        ws = torch.empty(n, dtype=torch.uint8, device=self.device)
        ids = torch.empty((n_x, self.k_sim), dtype=torch.int32, device=self.device)
        scores = torch.empty((n_x, self.k_sim), dtype=torch.float32, device=self.device)
        count = torch.empty(n_x, dtype=torch.int64, device=self.device)
        _lib.check(_lib.lib.b200_cf_cosine(
            _lib.ptr(sp_), _lib.ptr(si), _lib.ptr(sv), n_x, _lib.ptr(mp), _lib.ptr(mi), _lib.ptr(mv), n_y,
            min(self.min_common, 1 << 62), self.k_sim, _lib.ptr(ids), _lib.ptr(scores), _lib.ptr(count), _lib.ptr(ws), n,
            _lib.current_stream()))
        self.nbr_ids, self.nbr_scores, self.nbr_count = ids, scores, count
        self._n_elements = int(count.sum().item())
        self.workspace_bytes = n

    def _require(self):
        if self.nbr_ids is None:
            raise RuntimeError("call `compute_similarities` before `predict` / `recommend`")

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
        # the query's neighbours intersected with the other CSR's row: ItemCF items over R, UserCF users over R^T
        (_, _, _, n_q), (ptr, idx, lab, n_rows) = self._sides()
        rows, queries = (items, users) if self.user_based else (users, items)
        _lib.check(_lib.lib.b200_cf_predict(
            _lib.ptr(ptr), _lib.ptr(idx), _lib.ptr(lab), n_rows, _lib.ptr(self.nbr_ids), _lib.ptr(self.nbr_scores),
            _lib.ptr(self.nbr_count), n_q, self.k_sim, _lib.ptr(rows), _lib.ptr(queries), users.numel(),
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
        first ``n[r]`` ids are its recommendations, the rest -1.  ``seed`` keys the ``random_rec`` draw (default: the
        engine's seed and a call counter)."""
        self._require()
        fn = _lib.lib.b200_user_cf_recommend if self.user_based else _lib.lib.b200_swing_recommend

        def accumulate(ub, rows, counts, stream):
            _lib.check(fn(
                _lib.ptr(self.user_ptr), _lib.ptr(self.user_items), _lib.ptr(self.user_labels), self.n_users,
                _lib.ptr(self.nbr_ids), _lib.ptr(self.nbr_scores), _lib.ptr(self.nbr_count), self.n_items, self.k_sim,
                _lib.ptr(self.cons_ptr), _lib.ptr(self.cons_idx), 1 if filter_consumed else 0, _lib.ptr(ub),
                ub.numel(), _lib.ptr(rows), self.n_items, _lib.ptr(counts), stream))

        return recommend_rows(self, accumulate, users, n_rec, random_rec, seed)

    def recommend(self, users, n_rec, filter_consumed=True, random_rec=False):
        """recfarm CF's ``recommend``: ``(recs, no_rec_indices)``, ``recs[r]`` the ids of user r as a list (empty for
        a user without candidates) and ``no_rec_indices`` the positions r of those users."""
        import torch

        ids, n = self.recommend_device(torch.as_tensor(np.asarray(users, dtype=np.int64)), n_rec, filter_consumed,
                                       random_rec)
        ids, n = ids.cpu().numpy(), n.cpu().numpy()
        recs = [ids[r, :n[r]].tolist() for r in range(len(n))]
        return recs, [r for r in range(len(n)) if n[r] == 0]

    # ---- introspection -------------------------------------------------------------------------------------------
    def neighbors(self):
        """``(ids int32 [n_x, k_sim], cosines float32 [n_x, k_sim], kept count int64 [n_x])`` on the device."""
        self._require()
        return self.nbr_ids, self.nbr_scores, self.nbr_count


class ItemCF(_CfEngine):
    """``recfarm.ItemCF`` (``rust/src/item_cf.rs``) on the device: item-item cosines over the users' labels."""

    def num_sim_elements(self):
        """Total kept similarities.  Like recfarm, ``ValueError`` when no item kept any (before
        ``compute_similarities`` in particular)."""
        if not self._n_elements:
            raise ValueError("call `compute_similarities` first")
        return self._n_elements


class UserCF(_CfEngine):
    """``recfarm.UserCF`` (``rust/src/user_cf.rs``) on the device: user-user cosines over the items' labels."""

    user_based = True

    def num_sim_elements(self):
        """Total kept similarities; 0 when there are none, as in recfarm."""
        return self._n_elements


def fit_reference_model(model, ref_module, train_data, neg_sampling, verbose=1, eval_data=None, metrics=None, k=10,
                        eval_batch_size=8192, eval_user_num=None):
    """``RsCfBase.fit`` of the reference (``libreco/bases/cf_base_rs.py:64-122``) with :class:`UserCF` /
    :class:`ItemCF` as ``model.rs_model`` in place of recfarm's; ``ref_module`` is that module, whose helpers it
    calls.  A model prepared by ``rebuild_model`` (``model.incremental``) raises ``NotImplementedError``: the device
    engines have no incremental update."""
    if model.incremental:
        raise NotImplementedError("the device CF engines do not update a rebuilt model; fit a new one")
    ref_module.check_fitting(model, train_data, eval_data, neg_sampling, k)
    model.show_start_time()
    R = train_data.sparse_interaction
    user_based = "user" in model.model_name.lower()
    cls = UserCF if user_based else ItemCF
    model.rs_model = cls(model.task, model.k_sim, model.n_users, model.n_items, model.min_common, R, R.T.tocsr(),
                         model.user_consumed, model.default_pred, seed=model.seed)
    with ref_module.time_block("similarity", verbose=1):
        model.rs_model.compute_similarities(model.mode == "invert", model.num_threads)
    num = model.rs_model.num_sim_elements()
    n = model.n_users if user_based else model.n_items
    print(f"similarity num_elements: {num}, density: {100 * num / (n * n):5.4f} %")
    if verbose > 1:
        ref_module.print_metrics(model=model, neg_sampling=neg_sampling, eval_data=eval_data, metrics=metrics,
                                 eval_batch_size=eval_batch_size, k=k, sample_user_num=eval_user_num, seed=model.seed)
        print("=" * 30)
