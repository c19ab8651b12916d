"""UserCF and ItemCF on the device: the ``recfarm.UserCF`` / ``recfarm.ItemCF`` engines that
``libreco/bases/cf_base_rs.py`` drives (``RsUserCF`` / ``RsItemCF``), on the kernels of ``csrc/cf.cu`` and the
neighbourhood serving of ``neighbours.py``.

* :meth:`compute_similarities` builds, per row of the "sim side" (items for ItemCF, users for UserCF), its first
  ``k_sim`` cosine neighbours by (cosine desc, id asc) and its kept count: every other row sharing at least
  ``min_common`` interactions, zero cosines included (``b200_cf_cosine``).  ``recommend`` and ``predict`` only ever
  read those first ``k_sim`` entries (``item_cf.rs:375,421``, ``user_cf.rs:828,870``), so nothing else is kept.
* :meth:`recommend` accumulates ``sim * label`` per user into dense rows (ItemCF over the item neighbour table, UserCF
  over the user's neighbours' rows), ranks them with ``b200_topk_rows`` and returns ``(recs, no_rec_indices)`` as
  recfarm does.  With ``random_rec`` a row with more than ``n_rec`` candidates draws ``n_rec`` distinct candidates
  uniformly (Philox4x32-10 instead of recfarm's ``thread_rng``).
* :meth:`predict`: the query's neighbours intersected with the other CSR's row, then compute_pred of the engine's
  task.

``invert`` and ``num_threads`` (``compute_similarities``) are accepted for recfarm's signature and ignored: both
recfarm modes compute the same similarities, and the device runs one algorithm.
"""
from __future__ import annotations

import ctypes

from . import _lib
from .neighbours import TASKS, NeighbourEngine, check_top_k


def validate(task, k_sim, min_common):
    if task not in TASKS:
        raise ValueError(f"task must be 'rating' or 'ranking', got {task!r}")
    k_sim = check_top_k(k_sim, "k_sim")
    if isinstance(min_common, bool) or int(min_common) != min_common or int(min_common) < 1:
        raise ValueError(f"min_common must be an integer >= 1, got {min_common!r}")
    return task, k_sim, int(min_common)


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


class _CfEngine(NeighbourEngine):
    """Shared body of :class:`ItemCF` and :class:`UserCF`, recfarm's constructor::

        ItemCF(task, k_sim, n_users, n_items, min_common, user_interacts, item_interacts, user_consumed, default_pred)

    The arguments other than ``task``, ``k_sim`` and ``min_common`` are :class:`NeighbourEngine`'s."""

    def __init__(self, task, k_sim, n_users, n_items, min_common, user_interacts, item_interacts, user_consumed,
                 default_pred, device=None, seed=42):
        self.task, self.k_sim, self.min_common = validate(task, k_sim, min_common)
        super().__init__(n_users, n_items, user_interacts, item_interacts, user_consumed, default_pred, device, seed)

    def compute_similarities(self, invert=True, num_threads=1):
        """Cosine neighbours of every sim-side row (``invert`` and ``num_threads`` are ignored).  ``ValueError`` when
        the workspace does not fit in the device's free memory."""
        import torch

        # the CSR whose rows are compared, and its transpose
        users = (self.user_ptr, self.user_items, self.user_labels, self.n_users)
        items = (self.item_ptr, self.item_users, self.item_labels, self.n_items)
        (sp_, si, sv, n_x), (mp, mi, mv, n_y) = (users, items) if self.user_based else (items, users)
        n = workspace_bytes(n_x, self.k_sim)
        out_bytes = n_x * self.k_sim * 8 + n_x * 8
        free = torch.cuda.mem_get_info(self.device)[0]
        if n + out_bytes > free:
            raise ValueError(f"the similarity workspace of {n_x} rows needs {n + out_bytes} bytes, more than the "
                             f"{free} free on {self.device}")

        def launch(ws, ids, scores, count):
            _lib.check(_lib.lib.b200_cf_cosine(
                _lib.ptr(sp_), _lib.ptr(si), _lib.ptr(sv), n_x, _lib.ptr(mp), _lib.ptr(mi), _lib.ptr(mv), n_y,
                min(self.min_common, 1 << 62), self.k_sim, _lib.ptr(ids), _lib.ptr(scores), _lib.ptr(count),
                _lib.ptr(ws), n, _lib.current_stream()))

        self._compute(n_x, self.k_sim, n, launch)

    def recommend(self, users, n_rec, filter_consumed=True, random_rec=False):
        """recfarm CF's ``recommend``: ``(recs, no_rec_indices)``, ``recs[r]`` the ids of user r as a list (empty for
        a user without candidates) and ``no_rec_indices`` the positions r of those users."""
        recs = self._recommend_lists(users, n_rec, filter_consumed, random_rec)
        return recs, [r for r, rec in enumerate(recs) if not rec]


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
