"""Training losses of the hot path (SURVEY.md §8a row a13) on the device: the reference's function
names and argument meaning, value + gradient from one fused CUDA pass (``csrc/loss.cu``).

* ``libreco/torchops/loss.py:5-60``: ``binary_cross_entropy_loss``, ``focal_loss``, ``bpr_loss``,
  ``max_margin_loss``, ``pairwise_bce_loss``, ``pairwise_focal_loss``; ``compute_pair_scores`` (:63-90)
* ``libreco/tfops/loss.py:4-71``: sigmoid CE / focal / MSE of the TF models, ``max_margin_loss`` on
  embeddings, ``softmax_cross_entropy`` with ``TwoTower.adjust_logits``
  (``algorithms/two_tower.py:458-479``).

Every function takes fp32 CUDA tensors and returns a 0-d CUDA tensor that participates in torch
autograd (a ``torch.autograd.Function`` whose backward scales the gradient the kernel already
produced), so it drops into ``TorchTrainer._compute_loss`` (``training/torch_trainer.py:140-161``)
unchanged.  torch is used for memory and the autograd tape only.
"""
from __future__ import annotations

from . import _lib

_WS = {}


def _workspace(device):
    import torch

    key = (device.type, device.index)
    if key not in _WS:
        _WS[key] = torch.empty(int(_lib.lib.b200_loss_workspace_bytes()), dtype=torch.uint8, device=device)
    return _WS[key]


def _f32(t):
    import torch

    if not t.is_cuda:
        raise _lib.B200Error("losses need CUDA tensors (no CPU fallback)")
    return t.detach().to(torch.float32).contiguous()


def _make_functions():
    import torch

    class _Pointwise(torch.autograd.Function):
        @staticmethod
        def forward(ctx, logits, labels, kind, alpha, gamma):
            x, y = _f32(logits).reshape(-1), _f32(labels).reshape(-1)
            if x.numel() != y.numel():
                raise ValueError(f"logits and labels length doesn't match, got {x.numel()} and {y.numel()}")
            out = torch.empty((), dtype=torch.float32, device=x.device)
            grad = torch.empty_like(x)
            ws = _workspace(x.device)
            _lib.check(_lib.lib.b200_pointwise_loss(_lib.ptr(x), _lib.ptr(y), x.numel(), kind, alpha, gamma,
                                                    _lib.ptr(out), _lib.ptr(grad), _lib.ptr(ws), ws.numel(),
                                                    _lib.current_stream()))
            ctx.save_for_backward(grad)
            ctx.shape = logits.shape
            return out

        @staticmethod
        def backward(ctx, g):
            (grad,) = ctx.saved_tensors
            return (grad * g).reshape(ctx.shape), None, None, None, None

    class _Pairwise(torch.autograd.Function):
        @staticmethod
        def forward(ctx, pos, neg, kind, margin, alpha, gamma, mean):
            p, n = _f32(pos).reshape(-1), _f32(neg).reshape(-1)
            out = torch.empty((), dtype=torch.float32, device=p.device)
            gp, gn = torch.empty_like(p), torch.empty_like(n)
            ws = _workspace(p.device)
            _lib.check(_lib.lib.b200_pairwise_loss(_lib.ptr(p), p.numel(), _lib.ptr(n), n.numel(), kind, margin,
                                                   alpha, gamma, 1 if mean else 0, _lib.ptr(out), _lib.ptr(gp),
                                                   _lib.ptr(gn), _lib.ptr(ws), ws.numel(), _lib.current_stream()))
            ctx.save_for_backward(gp, gn)
            ctx.shapes = (pos.shape, neg.shape)
            return out

        @staticmethod
        def backward(ctx, g):
            gp, gn = ctx.saved_tensors
            return (gp * g).reshape(ctx.shapes[0]), (gn * g).reshape(ctx.shapes[1]), None, None, None, None, None

    class _InBatchSoftmax(torch.autograd.Function):
        @staticmethod
        def forward(ctx, user_embeds, item_embeds, temperature, correction, item_ids):
            from .feat_models import linear

            U, I = _f32(user_embeds), _f32(item_embeds)
            if U.shape != I.shape:
                raise ValueError(f"user and item embeds shape doesn't match, got {tuple(U.shape)} and {tuple(I.shape)}")
            S = linear(U, I, None, False, cache_split=False)                    # [B, B] = U I^T on the library's GEMM
            B = S.shape[0]
            out = torch.empty((), dtype=torch.float32, device=U.device)
            ws = _workspace(U.device)
            corr = _f32(correction) if correction is not None else None
            ids = item_ids.detach().to(torch.int64).contiguous() if item_ids is not None else None
            _lib.check(_lib.lib.b200_softmax_inbatch_loss(_lib.ptr(S), S.stride(0), B, float(temperature),
                                                          _lib.ptr(corr), _lib.ptr(ids), 1, _lib.ptr(out),
                                                          _lib.ptr(ws), ws.numel(), _lib.current_stream()))
            ctx.save_for_backward(S, U, I)                   # S now holds dloss/dS
            return out

        @staticmethod
        def backward(ctx, g):
            from .feat_models import linear

            G, U, I = ctx.saved_tensors
            # dU = G I, dI = G^T U: the same dense-layer kernel with the transposed operands
            dU = linear(G, I.t().contiguous(), None, False, cache_split=False)
            dI = linear(G.t().contiguous(), U.t().contiguous(), None, False, cache_split=False)
            return dU * g, dI * g, None, None, None

    return _Pointwise, _Pairwise, _InBatchSoftmax


_FNS = None


def _fns():
    global _FNS
    if _FNS is None:
        _FNS = _make_functions()
    return _FNS


# ---------------------------------------------------------------- pointwise
def binary_cross_entropy_loss(logits, labels):
    """torchops/loss.py:5-6; tfops/loss.py:14-18 (`cross_entropy`)."""
    return _fns()[0].apply(logits, labels, 0, 0.25, 2.0)


def focal_loss(logits, labels, alpha=0.25, gamma=2.0):
    """torchops/loss.py:10-19 with mean=True; tfops/loss.py:52-58 + reduce_mean."""
    return _fns()[0].apply(logits, labels, 1, float(alpha), float(gamma))


def mean_squared_error(predictions, labels):
    """tfops/loss.py:5-8 (task == "rating")."""
    return _fns()[0].apply(predictions, labels, 2, 0.25, 2.0)


# ---------------------------------------------------------------- pairwise
def bpr_loss(pos_scores, neg_scores):
    """torchops/loss.py:22-24."""
    return _fns()[1].apply(pos_scores, neg_scores, 0, 0.0, 0.25, 2.0, True)


def max_margin_loss(pos_scores, neg_scores, margin):
    """torchops/loss.py:27-30 (margin_ranking_loss with target 1) = tfops/loss.py:61-64 + reduce_mean.

    The value is the same for both.  The gradient follows torch: a pair exactly on the hinge
    (``pos - neg == margin``) passes gradient -1/n to ``pos`` and 1/n to ``neg``, where TF's relu gives 0."""
    return _fns()[1].apply(pos_scores, neg_scores, 1, float(margin), 0.25, 2.0, True)


def pairwise_bce_loss(pos_scores, neg_scores, mean=True):
    """torchops/loss.py:33-46."""
    return _fns()[1].apply(pos_scores, neg_scores, 2, 0.0, 0.25, 2.0, bool(mean))


def pairwise_focal_loss(pos_scores, neg_scores, mean=True):
    """torchops/loss.py:49-60 (alpha 0.25, gamma 2)."""
    return _fns()[1].apply(pos_scores, neg_scores, 3, 0.0, 0.25, 2.0, bool(mean))


def compute_pair_scores(targets, items_pos, items_neg, repeat_positives=True):
    """torchops/loss.py:63-90 — row dot products; negatives may be `factor` per positive."""
    import torch

    if len(targets) == len(items_pos) == len(items_neg):
        return (targets * items_pos).sum(1), (targets * items_neg).sum(1)
    if len(targets) != len(items_pos):
        raise ValueError(f"targets and items_pos length doesn't match, got {len(targets)} and {len(items_pos)}")
    pos_len, neg_len = len(items_pos), len(items_neg)
    if neg_len % pos_len != 0:
        raise ValueError(f"negatives length is not a multiple of positives length, got {neg_len} and {pos_len}")
    factor = neg_len // pos_len
    pos_scores = (targets * items_pos).sum(1)
    if repeat_positives:
        pos_scores = pos_scores.repeat_interleave(factor)
    neg_scores = (targets.unsqueeze(1) * items_neg.view(pos_len, factor, -1)).sum(2).reshape(-1)
    return pos_scores, neg_scores


# ---------------------------------------------------------------- in-batch softmax (TwoTower)
def softmax_cross_entropy(user_embeds, item_embeds, temperature=1.0, correction=None, item_indices=None):
    """tfops/loss.py:67-71 with ``adjust_logits(all_adjust=True)`` (two_tower.py:458-479):
    ``correction`` = sampling probabilities of the batch items (``use_correction``), ``item_indices``
    enables ``remove_accidental_hits``.  Returns the mean over the batch."""
    return _fns()[2].apply(user_embeds, item_embeds, float(temperature), correction, item_indices)
