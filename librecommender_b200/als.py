"""ALS training on the device: the reference's ``libreco/algorithms/_als.pyx`` (``als_update``) and the
``ALS.fit`` loop (``libreco/algorithms/als.py:134-181``) on the kernels of ``csrc/als.cu``.

* :func:`als_update` has the Cython function's signature and contract: ``X`` (host float32) is updated in
  place from the fixed ``Y`` and the (already alpha-scaled) scipy CSR.  ``dropin.install(libreco, als=True)``
  registers it as ``libreco.algorithms._als.als_update``, so the reference's own ``ALS.fit`` runs here.
* :class:`ALSTrainer` keeps both CSR orientations and both tables on the device for the whole fit; its
  :meth:`~ALSTrainer.embeddings` feed ``recommend_from_embedding`` / ``EmbedScorer`` with no host copy.

A half-epoch is ``A0`` (``Y^T Y + reg I`` for ranking, ``reg I`` for rating) on the split-K dense product,
then one call of ``b200_als_cg`` or ``b200_als_direct``.
"""
from __future__ import annotations

import ctypes

import numpy as np

from . import _lib

MAX_EMBED = 128
# Y^T Y is accumulated over row chunks of Y so the transposed copy stays bounded; chunk sums add in order
GRAM_ROWS = 1 << 22


def _posv_error(err, row):
    return ValueError(f"cython_lapack.posv failed (err={err}) on row {row}. "
                      "Try increasing the regularization parameter.")


def truncated_normal(rng, shape, mean=0.0, scale=0.05, tolerance=5):
    """``libreco.utils.initializers.truncated_normal``: normal draws, out-of-band ones redrawn up to 5 times."""
    n = int(np.prod(shape))
    a = rng.normal(mean, scale, n).astype(np.float32)
    hi, lo = mean + 2 * scale, mean - 2 * scale
    for _ in range(tolerance):
        bad = np.logical_or(a > hi, a < lo)
        k = int(bad.sum())
        if k == 0:
            break
        a[bad] = rng.normal(mean, scale, k)
    return a.reshape(*shape)


def initial_tables(n_users, n_items, embed_size, seed=42):
    """``ALS.build_model`` (``als.py:84-91``): users, then items, from one ``default_rng(seed)``."""
    rng = np.random.default_rng(seed)
    U = truncated_normal(rng, [n_users, embed_size], 0.0, 0.03)
    I = truncated_normal(rng, [n_items, embed_size], 0.0, 0.03)
    return U, I


class RowPlan:
    """A device CSR (``indptr`` int64, ``indices`` int32, ``data`` float32) and its row classes: rows of at most
    ``b200_als_long_row_threshold()`` nnz, and the longer rows split into ``b200_als_chunk()``-nnz chunks."""

    def __init__(self, indptr, indices, data, n_cols):
        import torch

        self.indptr, self.indices, self.data = indptr, indices, data
        self.n_rows, self.n_cols = indptr.numel() - 1, int(n_cols)
        dev = indptr.device
        thr, chunk = _lib.lib.b200_als_long_row_threshold(), _lib.lib.b200_als_chunk()
        deg = indptr[1:] - indptr[:-1]
        is_long = deg > thr
        self.short_rows = torch.nonzero(~is_long).flatten().to(torch.int32)
        long_rows = torch.nonzero(is_long).flatten()
        self.n_short, self.n_long = int(self.short_rows.numel()), int(long_rows.numel())
        self.long_rows = long_rows.to(torch.int32)
        nch = (deg[long_rows] + chunk - 1) // chunk
        self.long_chunk_ptr = torch.zeros(self.n_long + 1, dtype=torch.int64, device=dev)
        self.long_chunk_ptr[1:] = torch.cumsum(nch, 0)
        self.n_chunks = int(self.long_chunk_ptr[-1]) if self.n_long else 0
        owner = torch.repeat_interleave(torch.arange(self.n_long, device=dev), nch)
        self.chunk_long = owner.to(torch.int32)
        self.chunk_k = (torch.arange(self.n_chunks, device=dev) - self.long_chunk_ptr[owner]).to(torch.int32)
        self._ws = {}

    @classmethod
    def from_scipy(cls, csr, device, n_cols):
        import torch

        return cls(torch.as_tensor(np.asarray(csr.indptr, dtype=np.int64), device=device),
                   torch.as_tensor(np.asarray(csr.indices, dtype=np.int32), device=device),
                   torch.as_tensor(np.asarray(csr.data, dtype=np.float32), device=device), n_cols)

    def workspace(self, d, use_cg):
        import torch

        key = (int(d), bool(use_cg))
        if key not in self._ws:
            n = ctypes.c_size_t(0)
            _lib.check(_lib.lib.b200_als_workspace_bytes(int(d), int(use_cg), self.n_long, self.n_chunks,
                                                         ctypes.byref(n)))
            self._ws[key] = torch.empty((n.value + 15) // 16 * 4, dtype=torch.float32, device=self.indptr.device)
        return self._ws[key]


def gram(Y, reg, implicit):
    """A0 [d, d] float32: ``Y^T Y + reg I`` (implicit) or ``reg I``, as ``_als.pyx:114-117,187-190`` form it
    (the float32 ``reg`` added to the float32 diagonal).  Y^T Y runs on ``b200_linear_tf32x3_splitk`` over
    transposed row chunks of Y, whose results add in chunk order."""
    import torch

    n_y, d = int(Y.shape[0]), int(Y.shape[1])
    A0 = torch.zeros((d, d), dtype=torch.float32, device=Y.device)
    if implicit:
        stream = _lib.current_stream()
        for r0 in range(0, n_y, GRAM_ROWS):
            rows = min(GRAM_ROWS, n_y - r0)
            ld = (rows + 3) // 4 * 4
            Yt = torch.zeros((d, ld), dtype=torch.float32, device=Y.device)
            Yt[:, :rows] = Y[r0:r0 + rows].t()
            splits = max(1, min(64, rows // 4096))
            part = torch.empty(splits * d * d, dtype=torch.float32, device=Y.device)
            out = torch.empty((d, d), dtype=torch.float32, device=Y.device)
            _lib.check(_lib.lib.b200_linear_tf32x3_splitk(_lib.ptr(Yt), ld, d, _lib.ptr(Yt), ld, None, rows, d, 0,
                                                          splits, _lib.ptr(part), part.numel() * 4, _lib.ptr(out),
                                                          d, stream))
            A0 += out
    A0.diagonal().add_(torch.tensor(float(reg), dtype=torch.float32, device=Y.device))
    return A0


def solve(plan: RowPlan, X, Y, A0, implicit, use_cg=True, cg_steps=3):
    """One half-epoch in place on device tables: every row of X [plan.n_rows, d] against Y [plan.n_cols, d]."""
    d = int(X.shape[1])
    ws = plan.workspace(d, use_cg)
    args = (_lib.ptr(plan.indptr), _lib.ptr(plan.indices), _lib.ptr(plan.data), plan.n_rows, _lib.ptr(X),
            _lib.ptr(Y), int(Y.shape[0]), d, _lib.ptr(A0), int(bool(implicit)))
    plan_args = (_lib.ptr(plan.short_rows), plan.n_short, _lib.ptr(plan.long_rows), _lib.ptr(plan.long_chunk_ptr),
                 plan.n_long, _lib.ptr(plan.chunk_long), _lib.ptr(plan.chunk_k), plan.n_chunks, _lib.ptr(ws),
                 ws.numel() * 4)
    if use_cg:
        _lib.check(_lib.lib.b200_als_cg(*args, int(cg_steps), *plan_args, _lib.current_stream()))
        return
    row, info = ctypes.c_int64(-1), ctypes.c_int32(0)
    _lib.check(_lib.lib.b200_als_direct(*args, *plan_args, ctypes.byref(row), ctypes.byref(info),
                                        _lib.current_stream()))
    if info.value != 0:
        raise _posv_error(info.value, row.value)


def _check_table(name, a):
    if not isinstance(a, np.ndarray) or a.ndim != 2 or a.dtype != np.float32 or not a.flags.c_contiguous:
        raise ValueError(f"`{name}` must be a C-contiguous 2-D float32 numpy array")


def _check_task(task, cg_steps):
    if task not in ("rating", "ranking"):
        raise ValueError(f"`task` must be 'rating' or 'ranking', got {task!r}")
    if int(cg_steps) != cg_steps or cg_steps < 0:
        raise ValueError(f"`cg_steps` must be a non-negative integer, got {cg_steps}")


def _check_embed(d):
    if not 1 <= d <= MAX_EMBED:
        raise ValueError(f"embed size {d} outside [1, {MAX_EMBED}]")


def validate(interaction, X, Y, task, cg_steps):
    """Every check ``als_update`` makes before it touches the device; returns (indptr, indices, data)."""
    _check_task(task, cg_steps)
    _check_table("X", X)
    _check_table("Y", Y)
    if X.shape[1] != Y.shape[1]:
        raise ValueError(f"X and Y widths differ: {X.shape[1]} vs {Y.shape[1]}")
    _check_embed(X.shape[1])
    try:
        indptr, indices, data = (np.asarray(interaction.indptr), np.asarray(interaction.indices),
                                 np.asarray(interaction.data))
    except AttributeError:
        raise ValueError("`interaction` must be a scipy CSR matrix") from None
    if indptr.ndim != 1 or indptr.shape[0] != X.shape[0] + 1:
        raise ValueError(f"indptr has {indptr.shape[0]} entries, expected n_x + 1 = {X.shape[0] + 1}")
    if not (np.issubdtype(indptr.dtype, np.integer) and np.issubdtype(indices.dtype, np.integer)):
        raise ValueError("indptr and indices must be integer arrays")
    if data.dtype != np.float32:
        raise ValueError(f"interaction data must be float32, got {data.dtype}")
    if indptr[0] != 0 or np.any(np.diff(indptr) < 0):
        raise ValueError("indptr must start at 0 and be non-decreasing")
    nnz = int(indptr[-1])
    if indices.shape != (nnz,) or data.shape != (nnz,):
        raise ValueError(f"indices / data must hold indptr[-1] = {nnz} entries")
    if nnz and (indices.min() < 0 or indices.max() >= Y.shape[0]):
        raise ValueError(f"column index outside [0, {Y.shape[0]})")
    return indptr, indices, data


def als_update(interaction, X, Y, reg, task, use_cg=True, num_threads=1, cg_steps=3):
    """``libreco.algorithms._als.als_update`` on the GPU: solve every row of ``X`` in place against ``Y``.
    ``num_threads`` is accepted and ignored."""
    import torch

    del num_threads
    indptr, indices, data = validate(interaction, X, Y, task, cg_steps)
    dev = _lib.require_cuda()
    plan = RowPlan(torch.as_tensor(indptr.astype(np.int64), device=dev),
                   torch.as_tensor(indices.astype(np.int32), device=dev), torch.as_tensor(data, device=dev),
                   Y.shape[0])
    Xd, Yd = torch.as_tensor(X, device=dev), torch.as_tensor(Y, device=dev)
    implicit = task == "ranking"
    A0 = gram(Yd, reg, implicit)
    try:
        solve(plan, Xd, Yd, A0, implicit, use_cg, cg_steps)
    finally:
        X[...] = Xd.cpu().numpy()


class ALSTrainer:
    """``ALS.fit`` with both tables and both CSR orientations resident on the device.

    ``interaction``: the unscaled ``train_data.sparse_interaction`` (scipy CSR, users x items; never mutated).
    ``user_embeds`` / ``item_embeds``: initial tables (host or device); drawn as ``ALS.build_model`` does from
    ``seed`` when not given."""

    def __init__(self, interaction, task, reg, alpha=10, use_cg=True, cg_steps=3, embed_size=16,
                 user_embeds=None, item_embeds=None, seed=42, device=None):
        import torch

        _check_task(task, cg_steps)
        self.task, self.reg, self.alpha = task, float(reg), alpha
        self.use_cg, self.cg_steps = bool(use_cg), int(cg_steps)
        self.device = torch.device(device) if device is not None else _lib.require_cuda()
        n_users, n_items = interaction.shape
        if user_embeds is None or item_embeds is None:
            user_embeds, item_embeds = initial_tables(n_users, n_items, embed_size, seed)
        self.U = torch.as_tensor(user_embeds, dtype=torch.float32, device=self.device).clone().contiguous()
        self.I = torch.as_tensor(item_embeds, dtype=torch.float32, device=self.device).clone().contiguous()
        if self.U.shape != (n_users, self.U.shape[1]) or self.I.shape != (n_items, self.U.shape[1]):
            raise ValueError(f"tables {tuple(self.U.shape)} / {tuple(self.I.shape)} do not fit the "
                             f"{n_users} x {n_items} interaction matrix")
        _check_embed(int(self.U.shape[1]))
        indptr = torch.as_tensor(np.asarray(interaction.indptr, dtype=np.int64), device=self.device)
        indices = torch.as_tensor(np.asarray(interaction.indices, dtype=np.int32), device=self.device)
        data = torch.as_tensor(np.asarray(interaction.data, dtype=np.float32), device=self.device).clone()
        if task == "ranking":   # als.py:148-150: two float32 roundings, as numpy does them
            data = data * alpha
            data = data + 1
        self.users = RowPlan(indptr, indices, data, n_items)
        # the item orientation: a stable sort by item keeps each item's users in ascending order (= .T.tocsr())
        rows = torch.repeat_interleave(torch.arange(n_users, device=self.device, dtype=torch.int32),
                                       indptr[1:] - indptr[:-1])
        order = torch.sort(indices, stable=True).indices
        iptr = torch.zeros(n_items + 1, dtype=torch.int64, device=self.device)
        iptr[1:] = torch.cumsum(torch.bincount(indices, minlength=n_items), 0)
        self.items = RowPlan(iptr, rows[order].contiguous(), data[order].contiguous(), n_users)

    def epoch(self):
        """Users half, then items half, each against the just-updated other table (``als.py:153-168``)."""
        implicit = self.task == "ranking"
        solve(self.users, self.U, self.I, gram(self.I, self.reg, implicit), implicit, self.use_cg, self.cg_steps)
        solve(self.items, self.I, self.U, gram(self.U, self.reg, implicit), implicit, self.use_cg, self.cg_steps)

    def fit(self, n_epochs):
        for _ in range(int(n_epochs)):
            self.epoch()
        return self

    def embeddings(self):
        """Device ``(U, I)`` with the mean row appended (``assign_embedding_oov``)."""
        import torch

        return (torch.cat([self.U, self.U.mean(0, keepdim=True)]),
                torch.cat([self.I, self.I.mean(0, keepdim=True)]))
