"""``rank_recommendations`` on the GPU — drop-in for
``libreco/recommendation/ranking.py:10-56`` (same signature, same errors).

* consumed filter incl. the "cannot filter" rule of ``ranking.py:38``  → ``b200_mask_consumed``
* ``partition_select`` + descending ``argsort`` (``:48-49,:76-78``)      → ``b200_topk_rows``
  with the total order (score desc, item id asc) where the reference leaves ties unspecified.
  In that order -0.0 equals +0.0 and every NaN ranks above +inf (numpy's sort puts NaN last, so
  the reference's reversed ``argsort`` returns it first).  Consumed items are removed, as
  ``filter_items`` does: they are overwritten with the REMOVED pattern, which ranks below every
  score, so a consumed item never comes back even where the answer reaches ``-inf`` scores.
  Returned scores write -0.0 as +0.0 and every NaN as one NaN.
* ``random_rec`` (``:65-73``: sample ``n_rec`` without replacement with
  p ∝ softmax(preds)^0.75 + 1e-8) → Gumbel-top-K over ``log p`` through the same
  kernel (the reference's own RNG here is unseeded, so only the distribution is defined).
  A ``-inf`` prediction keeps the ``1e-8`` floor and can be drawn; a consumed item cannot.
"""
from __future__ import annotations

import ctypes

import numpy as np

from .. import _lib
from ..consumed import as_csr


def _expit(x):
    return 1.0 / (1.0 + np.exp(-x))


def rank_recommendations(
    task,
    user_ids,
    model_preds,
    n_rec,
    n_items,
    user_consumed,
    filter_consumed=True,
    random_rec=False,
    return_scores=False,
):
    import torch

    if n_rec > n_items:
        raise ValueError(f"`n_rec` {n_rec} exceeds num of items {n_items}")
    device = _lib.require_cuda()
    if isinstance(model_preds, torch.Tensor):
        preds = model_preds.to(device=device, dtype=torch.float32)
    else:
        preds = torch.from_numpy(np.ascontiguousarray(model_preds, dtype=np.float32)).to(device)
    if preds.dim() == 1:
        assert preds.numel() % n_items == 0
        preds = preds.reshape(-1, n_items)
    B = preds.shape[0]
    uid = torch.as_tensor(np.asarray(list(user_ids), dtype=np.int64)).to(device)
    assert uid.numel() == B
    n_users = int(uid.max().item()) + 1 if B else 0
    if not hasattr(user_consumed, "device"):
        n_users = max(n_users, (max(user_consumed) + 1) if len(user_consumed) else 0)
    csr = as_csr(user_consumed, n_users)
    indptr_d, idx_d = csr.device(device)
    stream = _lib.current_stream()
    lib = _lib.lib

    # a copy (never clobber caller data) with one NaN pattern: a caller's NaN must not read as REMOVED
    work = preds.masked_fill(torch.isnan(preds), float("nan")).contiguous()
    ld = work.stride(0)
    if filter_consumed and csr.nnz > 0:
        _lib.check(lib.b200_mask_consumed(_lib.ptr(work), ld, _lib.ptr(uid), B, n_items, n_rec,
                                          _lib.ptr(indptr_d), _lib.ptr(idx_d), csr.n_users, stream))
    select_on = work
    if random_rec:
        # log p = log(softmax^0.75 + 1e-8) (unnormalised is enough); Gumbel-top-K samples without replacement
        # from p.  Removed (consumed) entries stay removed; the softmax sees them as -inf, i.e. it runs over the
        # kept items only, like the reference's after filter_items.
        removed = work.view(torch.int32) == _lib.REMOVED_BITS
        logp = torch.log(torch.softmax(work.double().masked_fill(removed, float("-inf")), dim=1).pow(0.75) + 1e-8)
        g = -torch.log(-torch.log(torch.rand_like(logp).clamp_min(1e-300)))
        select_on = (logp + g).float().contiguous()
        select_on.view(torch.int32).masked_fill_(removed, _lib.REMOVED_BITS)
    out_ids = torch.empty((B, n_rec), dtype=torch.int64, device=device)
    out_scores = torch.empty((B, n_rec), dtype=torch.float32, device=device)
    nbytes = ctypes.c_size_t(0)
    _lib.check(lib.b200_topk_rows_workspace_bytes(B, n_items, n_rec, ctypes.byref(nbytes)))
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=device)
    _lib.check(lib.b200_topk_rows(_lib.ptr(select_on), select_on.stride(0), B, n_items, n_rec,
                                  _lib.ptr(out_ids), _lib.ptr(out_scores), _lib.ptr(ws),
                                  nbytes.value, stream))
    if random_rec:  # reference sorts the sampled items by their true scores (ranking.py:47-49)
        true = torch.gather(preds, 1, out_ids)
        order = torch.argsort(true, dim=1, descending=True, stable=True)
        out_ids = torch.gather(out_ids, 1, order)
        out_scores = torch.gather(true, 1, order)
    ids = out_ids.cpu().numpy()
    if return_scores:
        scores = out_scores.cpu().numpy()
        if task == "ranking":
            scores = _expit(scores)
        return ids, scores
    return ids
