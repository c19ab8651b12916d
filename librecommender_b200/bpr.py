"""BPR training on the device: the reference's Cython ``libreco/algorithms/_bpr.pyx`` (``bpr_update``) and the
``BPR.fit`` loop with ``use_tf=False`` (``libreco/algorithms/bpr.py:296-379``) on the kernel of ``csrc/bpr.cu``.

* :func:`bpr_update` has the Cython function's signature and contract: the tables and every optimizer state array
  (host float32) are updated in place for one epoch over the given samples.  ``dropin.install(libreco, bpr=True)``
  registers it as ``libreco.algorithms._bpr.bpr_update``, so the reference's own ``BPR(use_tf=False).fit`` runs here.
* :class:`BPRTrainer` keeps the CSR, both tables and the optimizer state on the device for the whole fit; its
  :meth:`~BPRTrainer.embeddings` feed ``recommend_from_embedding`` / ``EmbedScorer`` with no host copy.

Negatives are uniform over the items the user did not consume, as the reference draws them, from a Philox stream
keyed by (seed, epoch, sample index) rather than the reference's ``mt19937`` streams.  Updates are atomic adds of
deltas with about ``b200_bpr_default_inflight()`` samples in flight; like the reference's OpenMP path, that is not
bit-reproducible.  The serial schedule (one sample in flight) is, and it is what the tests compare bit for bit.
"""
from __future__ import annotations

import numpy as np

from . import _lib
from .als import truncated_normal

MAX_EMBED = 128
OPTIMIZERS = {"sgd": 0, "momentum": 1, "adam": 2}


def initial_tables(n_users, n_items, embed_size, seed=42):
    """``BPR._build_model_cython`` (``bpr.py:143-159``): users, then items, from one ``default_rng(seed)``; the last
    column is the item bias, 1.0 in the user table and 0.0 in the item table."""
    rng = np.random.default_rng(seed)
    U = truncated_normal(rng, [n_users, embed_size + 1], 0.0, 0.03)
    U[:, embed_size] = 1.0
    I = truncated_normal(rng, [n_items, embed_size + 1], 0.0, 0.03)
    I[:, embed_size] = 0.0
    return U, I


def state_names(optimizer):
    """The ``bpr_update`` keyword arrays an optimizer reads and writes, users' first."""
    return {"sgd": (), "momentum": ("u_velocity", "i_velocity"),
            "adam": ("u_1st_mom", "i_1st_mom", "u_2nd_mom", "i_2nd_mom")}[optimizer]


def _check_optimizer(optimizer):
    if optimizer not in OPTIMIZERS:
        raise ValueError(f"optimizer must be one of these: (`sgd`, `momentum`, `adam`), got {optimizer!r}")


def _check_table(name, a, rows, width=None):
    if not isinstance(a, np.ndarray) or a.ndim != 2 or a.dtype != np.float32 or not a.flags.c_contiguous:
        raise ValueError(f"`{name}` must be a C-contiguous 2-D float32 numpy array")
    if not a.flags.writeable:
        raise ValueError(f"`{name}` must be writeable")
    if a.shape[0] != rows or (width is not None and a.shape[1] != width):
        want = f"({rows}, {width})" if width is not None else f"({rows}, D)"
        raise ValueError(f"`{name}` has shape {a.shape}, expected {want}")


def _check_ids(name, a, n):
    if not isinstance(a, np.ndarray) or a.ndim != 1 or a.dtype != np.int32:
        raise ValueError(f"`{name}` must be a 1-D int32 numpy array")
    if a.size and (a.min() < 0 or a.max() >= n):
        raise ValueError(f"`{name}` holds ids outside [0, {n})")


def check_csr(indptr, indices, n_users, n_items):
    """A canonical CSR of the users' consumed items: ``n_users`` rows, ids in range, every row sorted and
    duplicate-free (the reference's ``binary_search`` is undefined otherwise).  Returns the row lengths."""
    indptr, indices = np.asarray(indptr), np.asarray(indices)
    if not (np.issubdtype(indptr.dtype, np.integer) and np.issubdtype(indices.dtype, np.integer)):
        raise ValueError("indptr and indices must be integer arrays")
    if indptr.ndim != 1 or indptr.shape[0] != n_users + 1:
        raise ValueError(f"indptr has {indptr.shape[0]} entries, expected n_users + 1 = {n_users + 1}")
    if indptr[0] != 0 or np.any(np.diff(indptr) < 0):
        raise ValueError("indptr must start at 0 and be non-decreasing")
    if indices.shape != (int(indptr[-1]),):
        raise ValueError(f"indices must hold indptr[-1] = {int(indptr[-1])} entries")
    if indices.size and (indices.min() < 0 or indices.max() >= n_items):
        raise ValueError(f"item index outside [0, {n_items})")
    deg = np.diff(indptr)
    step = np.diff(indices.astype(np.int64))
    first = np.zeros(indices.size, dtype=bool)
    first[indptr[:-1][deg > 0]] = True
    if np.any((step <= 0) & ~first[1:]):
        raise ValueError("every CSR row must be sorted and duplicate-free (call sort_indices / sum_duplicates)")
    return deg


def validate(optimizer, user_indices, item_indices, sparse_interaction, user_embed, item_embed, n_users, n_items,
             epoch, states):
    """Every check ``bpr_update`` makes before it touches the device; returns (indptr, indices)."""
    _check_optimizer(optimizer)
    n_users, n_items = int(n_users), int(n_items)
    if n_users < 1 or n_items < 1:
        raise ValueError("n_users and n_items must be positive")
    _check_table("user_embed", user_embed, n_users)
    D = user_embed.shape[1]
    if not 1 <= D - 1 <= MAX_EMBED:
        raise ValueError(f"embed size {D - 1} outside [1, {MAX_EMBED}]")
    _check_table("item_embed", item_embed, n_items, D)
    for name in state_names(optimizer):
        if states.get(name) is None:
            raise ValueError(f"optimizer {optimizer!r} needs `{name}`")
        _check_table(name, states[name], n_users if name.startswith("u_") else n_items, D)
    if optimizer == "adam" and (int(epoch) != epoch or epoch < 1):
        raise ValueError(f"`epoch` must be an integer >= 1 for adam, got {epoch}")
    _check_ids("user_indices", user_indices, n_users)
    _check_ids("item_indices", item_indices, n_items)
    if user_indices.shape != item_indices.shape:
        raise ValueError("user_indices and item_indices differ in length")
    try:
        indptr, indices = np.asarray(sparse_interaction.indptr), np.asarray(sparse_interaction.indices)
    except AttributeError:
        raise ValueError("`sparse_interaction` must be a scipy CSR matrix") from None
    deg = check_csr(indptr, indices, n_users, n_items)
    full = deg[user_indices] >= n_items
    if np.any(full):
        raise ValueError(f"user {int(user_indices[np.argmax(full)])} consumed every item: no negative exists")
    return indptr, indices


def _launch(optimizer, users, items, indptr, indices, n_users, n_items, U, I, states, lr, reg, momentum, rho1,
            rho2, epoch, seed, items_neg=None, neg_out=None, max_inflight=0):
    """One epoch on device tensors: ``states`` the optimizer's state tensors in ``state_names`` order."""
    st = list(states) + [None] * (4 - len(states))
    _lib.check(_lib.lib.b200_bpr_update(
        OPTIMIZERS[optimizer], _lib.ptr(users), _lib.ptr(items), int(users.numel()), _lib.ptr(indptr),
        _lib.ptr(indices), int(n_users), int(n_items), _lib.ptr(U), _lib.ptr(I), int(U.shape[1]) - 1,
        *(_lib.ptr(t) for t in st), float(lr), float(reg), float(momentum), float(rho1), float(rho2), int(epoch),
        int(seed) & 0xFFFFFFFFFFFFFFFF, _lib.ptr(items_neg), _lib.ptr(neg_out), int(max_inflight),
        _lib.current_stream()))


def _update(optimizer, user_indices, item_indices, sparse_interaction, user_embed, item_embed, lr, reg, n_users,
            n_items, seed, epoch, momentum=0.9, rho1=0.9, rho2=0.999, items_neg=None, neg_out=False, max_inflight=0,
            **states):
    """:func:`bpr_update` with the schedule and the negatives exposed: ``items_neg`` (int32 [n]) replaces the
    draw, ``neg_out=True`` returns the negatives used, ``max_inflight`` bounds the samples in flight (1: serial)."""
    import torch

    indptr, indices = validate(optimizer, user_indices, item_indices, sparse_interaction, user_embed, item_embed,
                               n_users, n_items, epoch, states)
    n = int(user_indices.shape[0])
    if items_neg is not None:
        _check_ids("items_neg", items_neg, int(n_items))
        if items_neg.shape != (n,):
            raise ValueError("items_neg must hold one negative per sample")
    dev = _lib.require_cuda()
    names = state_names(optimizer)
    host = [user_embed, item_embed] + [states[k] for k in names]
    dv = [torch.as_tensor(a, device=dev) for a in host]
    neg = torch.full((n,), -1, dtype=torch.int32, device=dev) if neg_out else None
    _launch(optimizer, torch.as_tensor(user_indices, device=dev), torch.as_tensor(item_indices, device=dev),
            torch.as_tensor(indptr.astype(np.int64), device=dev), torch.as_tensor(indices.astype(np.int32), device=dev),
            n_users, n_items, dv[0], dv[1], dv[2:], lr, reg, momentum, rho1, rho2, epoch, seed,
            None if items_neg is None else torch.as_tensor(items_neg, device=dev), neg, max_inflight)
    for h, d in zip(host, dv):
        h[...] = d.cpu().numpy()
    return None if neg is None else neg.cpu().numpy()


def bpr_update(optimizer, user_indices, item_indices, sparse_interaction, user_embed, item_embed, lr, reg, n_users,
               n_items, num_threads, seed, epoch, u_velocity=None, i_velocity=None, momentum=0.9, u_1st_mom=None,
               i_1st_mom=None, u_2nd_mom=None, i_2nd_mom=None, rho1=0.9, rho2=0.999):
    """``libreco.algorithms._bpr.bpr_update`` on the GPU: one epoch over ``(user_indices, item_indices)`` in that
    order, tables and optimizer state updated in place.  ``num_threads`` is accepted and ignored."""
    del num_threads
    states = dict(u_velocity=u_velocity, i_velocity=i_velocity, u_1st_mom=u_1st_mom, i_1st_mom=i_1st_mom,
                  u_2nd_mom=u_2nd_mom, i_2nd_mom=i_2nd_mom)
    _update(optimizer, user_indices, item_indices, sparse_interaction, user_embed, item_embed, lr, reg, n_users,
            n_items, seed, epoch, momentum=momentum, rho1=rho1, rho2=rho2, **states)


class BPRTrainer:
    """``BPR(use_tf=False).fit`` with the CSR, both tables and the optimizer state resident on the device.

    ``interaction``: ``train_data.sparse_interaction`` (scipy CSR, users x items, canonical rows).
    ``user_indices`` / ``item_indices``: the training samples; each epoch visits them in a fresh permutation drawn
    on the device from a generator seeded with ``seed`` (``shuffle=False``: in the given order).
    ``user_embeds`` / ``item_embeds``: initial tables (host or device, D = embed_size + 1 columns); drawn as
    ``_build_model_cython`` does from ``seed`` when not given."""

    def __init__(self, interaction, user_indices, item_indices, optimizer="adam", lr=0.001, reg=0.0, embed_size=16,
                 momentum=0.9, rho1=0.9, rho2=0.999, user_embeds=None, item_embeds=None, seed=42, shuffle=True,
                 device=None):
        import torch

        _check_optimizer(optimizer)
        self.optimizer, self.lr, self.reg = optimizer, float(lr), float(reg or 0.0)
        self.momentum, self.rho1, self.rho2 = float(momentum), float(rho1), float(rho2)
        self.seed, self.shuffle, self.epochs_done = int(seed), bool(shuffle), 0
        self.max_inflight = 0       # the library default; 1 runs the serial schedule
        self.device = torch.device(device) if device is not None else _lib.require_cuda()
        self.n_users, self.n_items = (int(v) for v in interaction.shape)
        if user_embeds is None or item_embeds is None:
            user_embeds, item_embeds = initial_tables(self.n_users, self.n_items, embed_size, seed)
        self.U = torch.as_tensor(user_embeds, dtype=torch.float32, device=self.device).clone().contiguous()
        self.I = torch.as_tensor(item_embeds, dtype=torch.float32, device=self.device).clone().contiguous()
        D = int(self.U.shape[1])
        if self.U.shape != (self.n_users, D) or self.I.shape != (self.n_items, D):
            raise ValueError(f"tables {tuple(self.U.shape)} / {tuple(self.I.shape)} do not fit the "
                             f"{self.n_users} x {self.n_items} interaction matrix")
        if not 1 <= D - 1 <= MAX_EMBED:
            raise ValueError(f"embed size {D - 1} outside [1, {MAX_EMBED}]")
        users, items = np.asarray(user_indices), np.asarray(item_indices)
        if users.shape != items.shape or users.ndim != 1:
            raise ValueError("user_indices and item_indices must be 1-D and of equal length")
        _check_ids("user_indices", users.astype(np.int32), self.n_users)
        _check_ids("item_indices", items.astype(np.int32), self.n_items)
        deg = check_csr(interaction.indptr, interaction.indices, self.n_users, self.n_items)
        if users.size and np.any(deg[users] >= self.n_items):
            raise ValueError("a sampled user consumed every item: no negative exists")
        self.indptr = torch.as_tensor(np.asarray(interaction.indptr, dtype=np.int64), device=self.device)
        self.indices = torch.as_tensor(np.asarray(interaction.indices, dtype=np.int32), device=self.device)
        self.users = torch.as_tensor(users.astype(np.int32), device=self.device)
        self.items = torch.as_tensor(items.astype(np.int32), device=self.device)
        self.states = [torch.zeros_like(t) for name in state_names(optimizer)
                       for t in ((self.U,) if name.startswith("u_") else (self.I,))]
        self.generator = torch.Generator(device=self.device).manual_seed(self.seed)

    def order(self):
        """The next epoch's sample permutation (consumes the generator)."""
        import torch

        return torch.randperm(self.users.numel(), generator=self.generator, device=self.device)

    def epoch(self):
        """One epoch: shuffle, then one kernel over every sample; epochs count from 1 (Adam's bias correction)."""
        self.epochs_done += 1
        users, items = self.users, self.items
        if self.shuffle:
            perm = self.order()
            users, items = users[perm], items[perm]
        _launch(self.optimizer, users, items, self.indptr, self.indices, self.n_users, self.n_items, self.U, self.I,
                self.states, self.lr, self.reg, self.momentum, self.rho1, self.rho2, self.epochs_done, self.seed,
                max_inflight=self.max_inflight)

    def fit(self, n_epochs):
        for _ in range(int(n_epochs)):
            self.epoch()
        return self

    def embeddings(self):
        """Device ``(U, I)`` with the mean row appended (``assign_embedding_oov``)."""
        import torch

        return (torch.cat([self.U, self.U.mean(0, keepdim=True)]),
                torch.cat([self.I, self.I.mean(0, keepdim=True)]))
