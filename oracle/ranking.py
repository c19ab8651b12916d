"""Numpy restatement of the reference's score-all-items + top-K path.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

Follows (reference @ 7463d9d):
* ``libreco/recommendation/recommend.py:57-78``  recommend_from_embedding
* ``libreco/recommendation/ranking.py:10-78``    rank_recommendations,
  filter_items, partition_select, get_reco_probs
* ``libreco/prediction/predict.py:18-40``        predict_from_embedding,
  normalize_prediction
* ``libreco/bases/embed_base.py:257-265``        assign_embedding_oov
* ``rust/src/utils.rs:8-35``                     build_consumed_unique
  (consecutive de-duplication; pinned by ``tests/test_consumed.py:12-25`` and the
  Rust unit test ``rust/src/utils.rs:41-59``)

Pinned against ``tests/test_rank_reco.py:7-87`` (known-answer IDs) and against
the unmodified reference on random inputs (``tests/golden/gen_ranking.py``).

Tie rule.  The reference leaves the order of equal scores unspecified
(``np.argpartition`` + reversed unstable ``np.argsort``, ranking.py:48,76-78).
The restatement uses the total order (score descending, item id ascending);
it equals the reference wherever the reference's answer is unique.  Special values
follow the reference's numpy order: -0.0 == +0.0, and every NaN ranks above +inf.
"""
from __future__ import annotations

import numpy as np


def build_consumed_unique(user_indices, item_indices):
    """rust/src/utils.rs:8-35 — group by key in arrival order, then drop
    CONSECUTIVE repeats inside every list (``Vec::dedup``)."""
    user_consumed: dict[int, list[int]] = {}
    item_consumed: dict[int, list[int]] = {}
    for u, i in zip(np.asarray(user_indices).tolist(), np.asarray(item_indices).tolist()):
        lu = user_consumed.setdefault(u, [])
        if not lu or lu[-1] != i:
            lu.append(i)
        li = item_consumed.setdefault(i, [])
        if not li or li[-1] != u:
            li.append(u)
    return user_consumed, item_consumed


def _row_topk(scores: np.ndarray, ids: np.ndarray, n_rec: int):
    """Top ``n_rec`` of one row under (score desc, id asc), where -0.0 == +0.0 and every NaN ranks
    above +inf: numpy sorts NaN last, so the reference's reversed ``argsort`` returns it first."""
    # lexsort: last key is primary.  -scores ascending == scores descending.
    n = len(scores)
    nan = np.isnan(scores)
    if nan.any():
        neg = np.where(nan, 0.0, -scores.astype(np.float64))
        order = np.lexsort((ids, neg, ~nan))[:n_rec]
    elif n > 4 * n_rec + 1024:
        # same answer, less sorting: every item of the top n_rec has a score >= the n_rec-th largest
        # value v, so only the items with score >= v (ties at v included) need the full ordering
        v = np.partition(scores, n - n_rec)[n - n_rec]
        sel = np.nonzero(scores >= v)[0]
        order = sel[np.lexsort((ids[sel], -scores[sel].astype(np.float64)))][:n_rec]
    else:
        order = np.lexsort((ids, -scores.astype(np.float64)))[:n_rec]
    return ids[order], scores[order]


def rank_recommendations(
    task,
    user_ids,
    model_preds,
    n_rec,
    n_items,
    user_consumed,
    filter_consumed=True,
    return_scores=False,
):
    """ranking.py:10-56 without the ``random_rec`` branch (unseeded RNG there,
    SURVEY.md H4).  ``user_consumed`` is the reference's ``dict[int, list]``."""
    if n_rec > n_items:  # ranking.py:21-22
        raise ValueError(f"`n_rec` {n_rec} exceeds num of items {n_items}")
    preds = np.asarray(model_preds)
    if preds.ndim == 1:  # ranking.py:23-26
        assert len(preds) % n_items == 0
        preds = preds.reshape(len(preds) // n_items, n_items)
    out_ids = np.empty((len(preds), n_rec), dtype=np.int64)
    out_scores = np.empty((len(preds), n_rec), dtype=preds.dtype)
    base_ids = np.arange(n_items, dtype=np.int64)
    for r, user in enumerate(user_ids):
        consumed = user_consumed[user] if user in user_consumed else []
        row, ids = preds[r], base_ids
        # ranking.py:38 — the filter is skipped unless K + len(consumed) <= N,
        # where len() counts duplicates left by the consecutive-only dedup.  ``filter_items``
        # (np.isin) removes the listed ids that exist; ids outside [0, n_items) match nothing.
        if filter_consumed and len(consumed) > 0 and n_rec + len(consumed) <= n_items:
            keep = np.ones(n_items, dtype=bool)
            c = np.asarray(consumed, dtype=np.int64)
            keep[c[(c >= 0) & (c < n_items)]] = False
            row, ids = row[keep], ids[keep]
        out_ids[r], out_scores[r] = _row_topk(row, ids, n_rec)
    if return_scores:
        if task == "ranking":  # ranking.py:52-53
            out_scores = 1.0 / (1.0 + np.exp(-out_scores.astype(np.float64)))
            out_scores = out_scores.astype(preds.dtype)
        return out_ids, out_scores
    return out_ids


def embed_scores(user_embeddings, item_embeddings, user_ids, n_items):
    """recommend.py:66-68 — fp32 ``U[user_ids] @ I[:n_items].T``."""
    u = np.asarray(user_embeddings)[np.asarray(user_ids, dtype=np.int64)]
    return u @ np.asarray(item_embeddings)[:n_items].T


def recommend_from_embedding(
    task,
    user_ids,
    n_rec,
    user_embeddings,
    item_embeddings,
    n_items,
    user_consumed,
    filter_consumed=True,
    return_scores=False,
):
    """recommend.py:57-78."""
    preds = embed_scores(user_embeddings, item_embeddings, user_ids, n_items)
    return rank_recommendations(
        task, user_ids, preds, n_rec, n_items, user_consumed, filter_consumed, return_scores
    )


def predict_from_embedding(user_embeddings, item_embeddings, users, items, task="ranking",
                           lower_bound=None, upper_bound=None):
    """predict.py:36-40 + normalize_prediction (:18-23): row-wise dot, then
    expit (ranking) or clip (rating)."""
    u = np.asarray(user_embeddings)[np.asarray(users, dtype=np.int64)]
    i = np.asarray(item_embeddings)[np.asarray(items, dtype=np.int64)]
    preds = np.sum(u * i, axis=1)
    if task == "rating":
        return np.clip(preds, lower_bound, upper_bound)
    return (1.0 / (1.0 + np.exp(-preds.astype(np.float64)))).astype(preds.dtype)


def assign_embedding_oov(embed):
    """embed_base.py:257-265 — append the column-mean row (mean scalar for 1-D)."""
    embed = np.asarray(embed)
    if embed.ndim == 1:
        return np.append(embed, np.mean(embed))
    return np.vstack([embed, np.mean(embed, axis=0)])


def reco_probs(preds):
    """ranking.py:65-67 — ``softmax(preds)**0.75 + 1e-8`` normalised; the
    distribution ``random_rec=True`` samples from without replacement."""
    x = np.asarray(preds, dtype=np.float64)
    e = np.exp(x - x.max())
    p = np.power(e / e.sum(), 0.75) + 1e-8
    return p / p.sum()


def near_tie_mask(ref_ids, got_ids, full_scores, rel_tol=1e-6):
    """Positions where ``got_ids`` differs from ``ref_ids`` only because the
    oracle's own scores of the two items are within ``rel_tol`` (relative to
    the row's max |score|) — the parity contract of SURVEY.md §7.2(2)."""
    ref_ids = np.asarray(ref_ids)
    got_ids = np.asarray(got_ids)
    ok = np.ones(ref_ids.shape, dtype=bool)
    for r in range(ref_ids.shape[0]):
        diff = np.nonzero(ref_ids[r] != got_ids[r])[0]
        if len(diff) == 0:
            continue
        scale = max(float(np.abs(full_scores[r]).max()), 1e-30)
        a = full_scores[r, ref_ids[r, diff]].astype(np.float64)
        b = full_scores[r, got_ids[r, diff]].astype(np.float64)
        ok[r, diff] = np.abs(a - b) <= rel_tol * scale
    return ok


# ---------------------------------------------------------------------------------------------
# Cost-faithful variant for the CPU-baseline leg of bench.py: the same numpy primitives, in the
# same order, as the reference (tile of int64 ids, per-user isin filter, argpartition, then a
# reversed argsort) — ranking.py:30-49,59-61,76-78.  Tie order is whatever numpy gives, like the
# reference; `rank_recommendations` above is the deterministic checker.
# ---------------------------------------------------------------------------------------------
def rank_recommendations_numpy_path(user_ids, preds, n_rec, n_items, user_consumed, filter_consumed=True):
    if n_rec > n_items:
        raise ValueError(f"`n_rec` {n_rec} exceeds num of items {n_items}")
    preds = np.asarray(preds)
    if preds.ndim == 1:
        preds = preds.reshape(len(preds) // n_items, n_items)
    id_matrix = np.tile(np.arange(n_items), (len(preds), 1))           # ranking.py:30
    picked_ids, picked_scores = [], []
    for r, user in enumerate(user_ids):                                 # ranking.py:33-45
        ids, row = id_matrix[r], preds[r]
        consumed = user_consumed[user] if user in user_consumed else []
        if filter_consumed and consumed and n_rec + len(consumed) <= n_items:
            keep = np.isin(ids, consumed, assume_unique=True, invert=True)   # ranking.py:60
            ids, row = ids[keep], row[keep]
        top = np.argpartition(row, -n_rec)[-n_rec:]                     # ranking.py:77
        picked_ids.append(ids[top])
        picked_scores.append(row[top])
    picked_ids, picked_scores = np.array(picked_ids), np.array(picked_scores)
    order = np.argsort(picked_scores, axis=1)[:, ::-1]                  # ranking.py:48
    return np.take_along_axis(picked_ids, order, axis=1)


def recommend_from_embedding_numpy_path(user_ids, n_rec, user_rows, item_embeddings, n_items,
                                        user_consumed, filter_consumed=True):
    """recommend.py:66-77 with ``user_rows = user_embeddings[user_ids]`` already gathered."""
    preds = user_rows @ item_embeddings[:n_items].T
    return rank_recommendations_numpy_path(user_ids, preds, n_rec, n_items, user_consumed, filter_consumed)
