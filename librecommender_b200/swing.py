"""Swing on the device: the ``recfarm.Swing`` engine that ``libreco/algorithms/swing.py`` drives, on the kernels of
``csrc/swing.cu`` and the neighbourhood serving of ``neighbours.py``.

* :meth:`Swing.compute_swing` builds, per item, its first ``top_k`` swing neighbours by (score desc, id asc) and its
  number of nonzero scores (``b200_swing_scores``).  ``recommend`` and ``predict`` only ever read those first
  ``top_k`` entries (``rust/src/swing.rs:167-168,209-210``), so nothing else is kept.
* :meth:`Swing.recommend` accumulates ``label * score`` per user into dense rows over the item neighbour table, ranks
  them with ``b200_topk_rows`` and returns ``(recs, additional counts)`` as recfarm does.  With ``random_rec`` a row
  with more than ``n_rec`` candidates draws ``n_rec`` distinct candidates uniformly, keyed by the engine's seed and a
  call counter (Philox4x32-10) instead of recfarm's ``thread_rng``.
* :meth:`Swing.predict` is compute_pred "ranking": one warp per (user, item).

``num_threads`` (``compute_swing``) and ``max_cache_num`` (the constructor) are accepted for recfarm's signature and
ignored: the device needs no thread count and caches no common-item lists.
"""
from __future__ import annotations

import ctypes
import math

import numpy as np

from . import _lib
from .neighbours import NeighbourEngine, check_top_k


def validate(top_k, alpha):
    top_k = check_top_k(top_k, "top_k")
    alpha = float(alpha)
    if not math.isfinite(alpha) or alpha < 0 or alpha > float(np.finfo(np.float32).max):
        raise ValueError(f"alpha must be finite and >= 0, got {alpha!r}")
    return top_k, alpha


class Swing(NeighbourEngine):
    """Device engine with the method contract of ``recfarm.Swing`` (``rust/src/swing.rs``)::

        Swing(top_k, alpha, max_cache_num, n_users, n_items, user_interacts, item_interacts, user_consumed,
              default_pred)

    The arguments after ``max_cache_num`` are :class:`NeighbourEngine`'s.  Swing never reads item labels, so
    ``item_interacts`` needs only the transpose's pattern."""

    uses_item_labels = False
    task = "ranking"

    def __init__(self, top_k, alpha, max_cache_num, n_users, n_items, user_interacts, item_interacts,
                 user_consumed, default_pred, device=None, seed=42):
        self.top_k, self.alpha = validate(top_k, alpha)
        self.max_cache_num = max_cache_num          # no cache on the device
        super().__init__(n_users, n_items, user_interacts, item_interacts, user_consumed, default_pred, device, seed)

    def compute_swing(self, num_threads=1):
        """Swing scores of every item (``num_threads`` is ignored)."""
        n = ctypes.c_size_t(0)
        _lib.check(_lib.lib.b200_swing_scores_workspace_bytes(self.n_users, self.n_items, self.top_k,
                                                               ctypes.byref(n)))

        def launch(ws, ids, scores, count):
            _lib.check(_lib.lib.b200_swing_scores(
                _lib.ptr(self.user_ptr), _lib.ptr(self.user_items), self.n_users, _lib.ptr(self.item_ptr),
                _lib.ptr(self.item_users), self.n_items, self.alpha, self.top_k, _lib.ptr(ids), _lib.ptr(scores),
                _lib.ptr(count), _lib.ptr(ws), n.value, _lib.current_stream()))

        self._compute(self.n_items, self.top_k, n.value, launch)

    def num_swing_elements(self):
        """Total number of nonzero swing scores.  Like recfarm, ``RuntimeError`` when no item has any (before
        ``compute_swing`` in particular)."""
        if not self._n_elements:
            raise RuntimeError("call `compute_swing` method before calling `num_swing_elements`")
        return self._n_elements

    def recommend(self, users, n_rec, filter_consumed=True, random_rec=False):
        """recfarm's ``recommend``: ``(recs, additional counts)``, ``recs[r]`` the ids of user r as a list and
        ``additional[r] = n_rec - len(recs[r])``."""
        recs = self._recommend_lists(users, n_rec, filter_consumed, random_rec)
        return recs, [int(n_rec) - len(r) for r in recs]


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
