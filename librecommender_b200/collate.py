"""Device-side batch collation (SURVEY.md §8a row a11) — the part of
``libreco/batch/collators.py`` that sits between the interaction arrays and the model forward:

* ``PointwiseCollator.__call__`` (:225-252): users / items repeated ``num_neg + 1`` times, labels
  ``1, 0, 0, …``, the ``num_neg`` negatives of positive ``j`` interleaved right after it (:231-232);
* ``PairwiseCollator.__call__`` (:277-299): ``(users, items_pos, items_neg)`` with the positives
  repeated ``num_neg`` times when ``repeat_positives``.

Negatives come from :class:`~librecommender_b200.sampling.DeviceNegativeSampler` (fast mode) or from
a host array produced by the parity samplers.  The per-row FEATURE gathering of the reference
(``get_pointwise_feats`` / ``get_sampled_item_feats``, :254-267,460-490) has no counterpart here on
purpose: the feature kernels (``b200_feat_forward``) read the per-user / per-item unique tables
themselves from ``(user, item)``, so a collated batch is just the three id / label vectors.
Index bookkeeping only (repeat / interleave on device tensors); the sampling itself is the CUDA
kernel."""
from __future__ import annotations

import numpy as np


def adjust_batch_size(batch_size: int, num_neg: int, pairwise: bool) -> int:
    """libreco/batch/batch_data.py:93-105 — positives per step."""
    return max(1, int(batch_size / (num_neg if pairwise else num_neg + 1)))


class DevicePointwiseCollator:
    def __init__(self, sampler, num_neg: int, sampler_name: str = "random"):
        self.sampler, self.num_neg, self.sampler_name = sampler, int(num_neg), sampler_name

    def __call__(self, users_d, items_d, negatives_d=None):
        import torch

        r = self.num_neg + 1
        n = users_d.numel()
        if negatives_d is None:
            negatives_d = self.sampler.sample(users_d, items_d, self.num_neg, self.sampler_name)
        users = users_d.repeat_interleave(r)
        items = torch.empty(n * r, dtype=torch.int64, device=users_d.device)
        items.view(n, r)[:, 0] = items_d
        items.view(n, r)[:, 1:] = negatives_d.view(n, self.num_neg)
        labels = torch.zeros(n * r, dtype=torch.float32, device=users_d.device)
        labels[::r] = 1.0
        return users, items, labels


class DevicePairwiseCollator:
    def __init__(self, sampler, num_neg: int, sampler_name: str = "random", repeat_positives: bool = True):
        self.sampler, self.num_neg = sampler, int(num_neg)
        self.sampler_name, self.repeat_positives = sampler_name, repeat_positives

    def __call__(self, users_d, items_d, negatives_d=None):
        if negatives_d is None:
            negatives_d = self.sampler.sample(users_d, items_d, self.num_neg, self.sampler_name)
        if self.repeat_positives and self.num_neg > 1:
            return users_d.repeat_interleave(self.num_neg), items_d.repeat_interleave(self.num_neg), negatives_d
        return users_d, items_d, negatives_d


def interacted_positions_host(user_consumed, user_indices, item_indices):
    """PARITY mode helper: the positions ``get_interacted_seqs`` (libreco/batch/sequence.py:44-55)
    would draw for samples whose item is not in the user's history, consuming Python's global
    ``random`` stream exactly like the reference (one ``random.randrange(0, len)`` per such
    sample, in batch order).  Returns int64[n] (-1 where the item is in the list: the kernel finds
    the first occurrence itself)."""
    import random

    out = np.full(len(user_indices), -1, dtype=np.int64)
    sets = {}
    for j, (u, i) in enumerate(zip(user_indices, item_indices)):
        u = int(u)
        s = sets.get(u)
        if s is None:
            s = sets[u] = set(user_consumed[u])
        if int(i) not in s:
            out[j] = random.randrange(0, len(user_consumed[u]))
    return out


class DeviceSequenceBuilder:
    """``get_interacted_seqs`` (libreco/batch/sequence.py:33-71, ``mode="recent"``) on the device:
    the per-sample history window the sequence models (DIN, YouTubeRanking, …) train on
    (``batch/collators.py:207-222``).  ``consumed`` is a :class:`~librecommender_b200.consumed.ConsumedCSR`
    in arrival order; ``pad_index`` is ``n_items`` in the reference (``bases/tf_base.py`` seq models)."""

    def __init__(self, consumed, max_seq_len: int, pad_index: int, seed: int = 42, device="cuda"):
        self.consumed, self.max_seq_len, self.pad_index = consumed, int(max_seq_len), int(pad_index)
        self.seed, self.step, self.device = int(seed), 0, device

    def __call__(self, users_d, items_d, rand_pos_d=None):
        import torch

        from . import _lib

        indptr, idx = self.consumed.device(users_d.device)
        n = users_d.numel()
        seqs = torch.empty((n, self.max_seq_len), dtype=torch.int32, device=users_d.device)
        lens = torch.empty(n, dtype=torch.int32, device=users_d.device)
        users_d = users_d.to(torch.int64).contiguous()
        items_d = items_d.to(torch.int64).contiguous()
        if rand_pos_d is not None:
            rand_pos_d = rand_pos_d.to(torch.int64).contiguous()
        _lib.check(_lib.lib.b200_interacted_seqs(
            _lib.ptr(indptr), _lib.ptr(idx), self.consumed.n_users, _lib.ptr(users_d), _lib.ptr(items_d), n,
            self.max_seq_len, self.pad_index, _lib.ptr(rand_pos_d), self.seed, self.step, _lib.ptr(seqs),
            _lib.ptr(lens), _lib.current_stream()))
        self.step += 1
        return seqs, lens


class DeviceDualSequenceBuilder:
    """``get_dual_seqs`` (libreco/batch/sequence.py:94-147) on the device: SIM's per-sample long and short windows
    (``batch/collators.py:114-116``), the dual counterpart of :class:`DeviceSequenceBuilder` with the same position
    rule and draw stream.  Parity mode passes the positions of :func:`interacted_positions_host`: ``get_dual_seqs``
    draws from the same ``random.randrange`` stream.  A user with no items gets position 0 (two all-pad rows of length
    1) where the reference raises.  Returns (long_seqs [n, L], long_lens, short_seqs [n, S], short_lens), int32."""

    def __init__(self, consumed, long_max_len: int, short_max_len: int, pad_index: int, seed: int = 42,
                 device="cuda"):
        self.consumed, self.pad_index = consumed, int(pad_index)
        self.long_max_len, self.short_max_len = int(long_max_len), int(short_max_len)
        self.seed, self.step, self.device = int(seed), 0, device

    def __call__(self, users_d, items_d, rand_pos_d=None):
        import torch

        from . import _lib

        indptr, idx = self.consumed.device(users_d.device)
        n, L, S = users_d.numel(), self.long_max_len, self.short_max_len
        dev = users_d.device
        long_seqs = torch.empty((n, L), dtype=torch.int32, device=dev)
        short_seqs = torch.empty((n, S), dtype=torch.int32, device=dev)
        long_lens = torch.empty(n, dtype=torch.int32, device=dev)
        short_lens = torch.empty(n, dtype=torch.int32, device=dev)
        users_d = users_d.to(torch.int64).contiguous()
        items_d = items_d.to(torch.int64).contiguous()
        if rand_pos_d is not None:
            rand_pos_d = rand_pos_d.to(torch.int64).contiguous()
        _lib.check(_lib.lib.b200_interacted_dual_seqs(
            _lib.ptr(indptr), _lib.ptr(idx), self.consumed.n_users, _lib.ptr(users_d), _lib.ptr(items_d), n, L, S,
            self.pad_index, _lib.ptr(rand_pos_d), self.seed, self.step, _lib.ptr(long_seqs), _lib.ptr(long_lens),
            _lib.ptr(short_seqs), _lib.ptr(short_lens), _lib.current_stream()))
        self.step += 1
        return long_seqs, long_lens, short_seqs, short_lens
