"""Host-side pieces of the reference's inference plumbing that the engines need for the cases the
device tables do not cover (SURVEY.md §8 a3 / a15):

* :func:`assign_oov_rows`      — ``TfBase.assign_tf_variables_oov`` (``bases/tf_base.py:310-353``): after
  training the OOV rows (user ``n_users``, item ``n_items``, each sparse field's oov slot) become the
  mean of the field's real rows;
* :func:`dynamic_feature_rows` — the per-row feature matrices of "one user x every item" with the
  user's features overridden for one call (``recommendation/preprocess.py:104-148,160-212`` +
  ``prediction/preprocess.py:58-104``); nothing of ``data_info`` is modified;
* :func:`build_rec_seq`        — a caller-supplied behaviour sequence turned into the padded
  ``[1, max_seq_len]`` row the sequence models read (``recommendation/preprocess.py:36-45,215-220``).
"""
from __future__ import annotations

import numpy as np


def assign_oov_rows(weights, n_users, n_items, sparse_oov=None):
    """Returns a copy of the weight dict with the OOV rows assigned as the reference does.
    user variables: ``user_embeds`` / ``user_linear`` (row ``n_users`` = mean of rows ``[0, n_users)``);
    item variables likewise; sparse variables ``sparse_embeds`` / ``sparse_linear``: for every oov index
    in ``data_info.sparse_oov`` (ascending) the mean of the rows since the previous oov index
    (a multi-sparse field repeats its oov: ``start >= oov`` entries are skipped, ``tf_base.py:340-342``)."""
    out = dict(weights)

    def mean_row(name, n):
        v = out.get(name)
        if v is None:
            return
        v = np.array(v, dtype=np.float32, copy=True)
        v[n] = v[:n].mean(axis=0, dtype=np.float32) if v.ndim > 1 else np.float32(v[:n].mean(dtype=np.float32))
        out[name] = v

    for name in ("user_embeds", "user_linear"):
        mean_row(name, n_users)
    for name in ("item_embeds", "item_linear"):
        mean_row(name, n_items)
    if sparse_oov is not None:
        for name in ("sparse_embeds", "sparse_linear"):
            v = out.get(name)
            if v is None:
                continue
            v = np.array(v, dtype=np.float32, copy=True)
            start = 0
            for oov in [int(o) for o in sparse_oov]:
                if start >= oov:
                    continue
                v[oov] = v[start:oov].mean(axis=0, dtype=np.float32)
                start = oov + 1
            out[name] = v
    return out


def _extract(user_row, n_items, user_col, item_col, item_unique):
    """``recommendation/preprocess.py:201-212`` for one user: tile the user's row, drop the items' OOV
    row, restore the original column order."""
    user_feats = np.tile(user_row, (n_items, 1)) if user_col else None
    item_feats = item_unique[:-1] if item_col else None
    if user_col and item_col:
        orig_cols = list(user_col) + list(item_col)
        col_reindex = np.arange(len(orig_cols))[np.argsort(orig_cols)]
        return np.concatenate([user_feats, item_feats], axis=1)[:, col_reindex]
    return user_feats if user_col else item_feats


def dynamic_feature_rows(data_info, user, user_feats=None):
    """(sparse_indices int[N, F_s] | None, dense_values f32[N, F_d] | None) for user ``user`` against
    every item, with ``user_feats`` ({column name: value}) applied the way ``set_temp_feats`` does:
    unknown columns and unseen sparse values are ignored, dense values are written as given."""
    n_items = data_info.n_items
    sparse = dense = None
    if data_info.user_sparse_unique is not None or data_info.item_sparse_unique is not None:
        ucol, icol = data_info.user_sparse_col.index, data_info.item_sparse_col.index
        urow = data_info.user_sparse_unique[user] if ucol else None
        sparse = _extract(urow, n_items, ucol, icol, data_info.item_sparse_unique)
    if data_info.user_dense_unique is not None or data_info.item_dense_unique is not None:
        ucol, icol = data_info.user_dense_col.index, data_info.item_dense_col.index
        urow = data_info.user_dense_unique[user] if ucol else None
        dense = _extract(urow, n_items, ucol, icol, data_info.item_dense_unique)
    if user_feats is not None:
        if not isinstance(user_feats, dict):
            raise AssertionError("`user_feats` must be `dict`.")
        cm = data_info.col_name_mapping
        if sparse is not None:
            sparse = sparse.copy()
            if "sparse_col" in cm:
                for col, val in user_feats.items():
                    if col not in cm["sparse_col"]:
                        continue
                    if "multi_sparse" in cm and col in cm["multi_sparse"]:
                        idx_mapping = data_info.sparse_idx_mapping[cm["multi_sparse"][col]]
                    else:
                        idx_mapping = data_info.sparse_idx_mapping[col]
                    if val in idx_mapping:
                        f = cm["sparse_col"][col]
                        sparse[:, f] = idx_mapping[val] + data_info.sparse_offset[f]
        if dense is not None:
            dense = dense.copy()
            if "dense_col" in cm:
                for col, val in user_feats.items():
                    if col in cm["dense_col"]:
                        dense[:, cm["dense_col"][col]] = val
    return sparse, dense


def build_rec_seq(seq, n_items, max_seq_len, item2id=None, inner_id=False):
    """(recent_seq int32[1, max_seq_len] padded with ``n_items``, seq_len int32[1]): the LAST
    ``max_seq_len`` items of ``seq``; original ids are mapped through ``item2id`` (unknown -> ``n_items``)."""
    if not isinstance(seq, (list, np.ndarray)):
        raise AssertionError("`seq` must be list or numpy.ndarray.")
    if not inner_id:
        seq = [item2id.get(i, n_items) for i in seq]
    seq_len = min(int(max_seq_len), len(seq))
    out = np.full((1, int(max_seq_len)), n_items, dtype=np.int32)
    if seq_len > 0:
        out[0, :seq_len] = np.asarray(seq[-seq_len:], dtype=np.int32)
    return out, np.array([seq_len], dtype=np.int32)


def build_dual_seq(seq, n_items, long_max_len, short_max_len, item2id=None, inner_id=False):
    """(long_seq int32[1, long_max_len], long_len int32[1], short_seq int32[1, short_max_len], short_len int32[1])
    of a caller-supplied sequence for SIM (``recommendation/preprocess.py:49-76``): the last ``short_max_len`` items
    and up to ``long_max_len`` items before them, padded with ``n_items``; a sequence of at most ``short_max_len``
    items gets long length 1 over an all-pad row.  Original ids go through ``item2id`` (unknown -> ``n_items``)."""
    if not isinstance(seq, (list, np.ndarray)):
        raise AssertionError("`seq` must be list or numpy.ndarray.")
    if not inner_id:
        seq = [item2id.get(i, n_items) for i in seq]
    seq = np.asarray(seq, dtype=np.int32).reshape(-1)
    n, L, S = len(seq), int(long_max_len), int(short_max_len)
    long_seq = np.full((1, L), n_items, dtype=np.int32)
    if n >= L + S:
        long_len = L
        long_seq[0] = seq[n - L - S:n - S]
    elif n > S:
        long_len = n - S
        long_seq[0, :long_len] = seq[:long_len]
    else:
        long_len = 1
    short_seq = np.full((1, S), n_items, dtype=np.int32)
    short_len = min(S, n)
    if short_len > 0:
        short_seq[0, :short_len] = seq[n - short_len:]
    return long_seq, np.array([long_len], dtype=np.int32), short_seq, np.array([short_len], dtype=np.int32)
