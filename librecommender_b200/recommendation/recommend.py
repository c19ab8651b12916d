"""``recommend_from_embedding`` / ``construct_rec`` — drop-ins for
``libreco/recommendation/recommend.py:8-18,57-78``."""
from __future__ import annotations

import numpy as np

from ..engine import scorer_for
from .ranking import rank_recommendations


_ID_LOOKUP = {}


def _lookup_array(mapping, name, data_info):
    """dict inner id -> original id as one numpy array (built once per data_info object)."""
    key = (id(data_info), name, len(mapping))
    hit = _ID_LOOKUP.get(key)
    if hit is None or hit[0] is not mapping:
        n = (max(mapping) + 1) if len(mapping) else 0
        sample = next(iter(mapping.values())) if len(mapping) else 0
        arr = np.empty(n, dtype=object if isinstance(sample, str) else np.asarray(sample).dtype)
        for k, v in mapping.items():
            arr[k] = v
        if len(_ID_LOOKUP) > 16:
            _ID_LOOKUP.clear()
        hit = _ID_LOOKUP[key] = (mapping, arr)
    return hit[1]


def construct_rec(data_info, user_ids, computed_recs, inner_id):
    """recommend.py:8-18 — inner ids -> original ids.  The reference walks a Python dict per
    recommended item; here the item map becomes one lookup array (cached per data_info), so a
    batch of B x n_rec ids is a single fancy-index (SURVEY.md 8f-3)."""
    out = {}
    if inner_id:
        for r, u in enumerate(user_ids):
            out[u] = np.array(computed_recs[r])
        return out
    items = _lookup_array(data_info.id2item, "item", data_info)
    recs = np.asarray(computed_recs)
    for r, u in enumerate(user_ids):
        out[data_info.id2user[u]] = items[recs[r]]
    return out


def check_dynamic_rec_feats(model_name, user, user_feats, seq):
    """Argument validation of recommend.py:39-54 (same conditions, same exception type)."""
    sequence_models = ("YouTubeRetrieval", "YouTubeRanking", "DIN", "RNN4Rec", "Caser", "WaveNet", "Transformer",
                       "SIM")
    if seq is not None and model_name not in sequence_models:
        raise ValueError(f"`{model_name}` doesn't support arbitrary seq inference.")
    if not np.isscalar(user):
        if user_feats is not None:
            raise ValueError(f"Batch inference doesn't support assigning arbitrary features: {user}")
        if seq is not None:
            raise ValueError(f"Batch inference doesn't support arbitrary item sequence: {user}")
    if seq is not None and not isinstance(seq, (list, np.ndarray)):
        raise ValueError("`seq` must be list or numpy.ndarray.")
    if user_feats is not None and not isinstance(user_feats, dict):
        raise ValueError("`user_feats` must be `dict`.")


def recommend_tf_feat(model, user_ids, n_rec, user_feats, seq, filter_consumed, random_rec, inner_id=False):
    """recommend.py:81-105 for the feature models.  The reference tiles a B*N-row feed
    (``process_tf_feat``) and runs the TF graph; here ``model.b200_engine`` — a
    :mod:`librecommender_b200.feat_models` engine (FM / DeepFM / DIN / YouTubeRanking / AutoInt / Transformer / SIM) built from the
    model's saved variables — scores the implicit (user, item) grid on the GPU and the consumed
    filter + top-K run on the score rows.  A single-user call with ``user_feats`` / ``seq`` goes through
    ``engine.recommend_dynamic`` (explicit per-row feature matrix / replaced sequence row; both of SIM's rows)."""
    from .. import _lib

    engine = getattr(model, "b200_engine", None)
    if engine is None:
        raise _lib.B200Error("recommend_tf_feat: attach a feat_models engine as `model.b200_engine` first")
    if user_feats is not None or (seq is not None and len(seq) > 0):
        # single-user call with features / sequence supplied for this request (recommend.py:39-54)
        if len(user_ids) != 1:
            raise ValueError(f"Batch inference doesn't support assigning arbitrary features: {user_ids}")
        return engine.recommend_dynamic(user_ids[0], n_rec, model.data_info, user_feats, seq, filter_consumed,
                                        inner_id)
    if n_rec > model.n_items:
        raise ValueError(f"`n_rec` {n_rec} exceeds num of items {model.n_items}")
    if random_rec:
        import torch

        uid = torch.as_tensor(np.asarray(user_ids, dtype=np.int64)).to(engine.device)
        rows = engine.score_all_items(uid)
        return rank_recommendations(model.task, user_ids, rows, n_rec, model.n_items, engine.csr,
                                    filter_consumed, True)
    out = engine.recommend(user_ids, n_rec, filter_consumed)
    return out[0] if isinstance(out, tuple) else out


def recommend_from_embedding(
    model,
    user_ids,
    n_rec,
    user_embeddings,
    item_embeddings,
    filter_consumed,
    random_rec,
):
    """Same contract as the reference: ``int64[B, n_rec]`` inner item ids."""
    if n_rec > model.n_items:
        raise ValueError(f"`n_rec` {n_rec} exceeds num of items {model.n_items}")
    scorer = scorer_for(model, user_embeddings, item_embeddings)
    if random_rec:
        import torch

        uid = torch.as_tensor(np.asarray(user_ids, dtype=np.int64)).to(scorer.device)
        rows = scorer.score_rows(uid)
        return rank_recommendations(model.task, user_ids, rows, n_rec, model.n_items,
                                    scorer.csr, filter_consumed, True)
    return scorer.recommend(user_ids, n_rec, filter_consumed)
