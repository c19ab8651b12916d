"""Drop-in wiring: patch an imported reference package (``libreco``) so that its OWN classes run the
hot path on this library — the code form of INTEGRATION.md ("What a reference maintainer changes").

    import libreco
    from librecommender_b200 import dropin
    dropin.install(libreco)            # LightGCN(...).fit(...); model.recommend_user(...) now run on the GPU
    dropin.uninstall()                 # the reference's numpy / torch-CPU path again

What is patched (seams of SURVEY.md §8b; nothing else of the reference changes):

* ``libreco.recommendation.{rank_recommendations, recommend_from_embedding, construct_rec}`` and the
  copies of those names that ``bases/embed_base.py:10``, ``bases/dyn_embed_base.py:8`` and
  ``recommendation/recommend.py`` hold — so ``EmbedBase.fit`` (default_recs, ``embed_base.py:153-161``),
  ``EmbedBase.recommend_user`` (``:190-251``) and ``DynEmbedBase.recommend_user`` call the CUDA path;
* ``libreco.algorithms.lightgcn.LightGCNModel`` (``algorithms/lightgcn.py:4,117-127``) → the
  differentiable K6 module with the reference's constructor / ``forward(use_dropout)`` contract;
* optionally the loss functions ``TorchTrainer._compute_loss`` uses
  (``training/torch_trainer.py:15-23,140-161``);
* optionally (``als=True``) the Cython extension ``libreco.algorithms._als``: a module whose ``als_update``
  is ``librecommender_b200.als.als_update`` is registered in ``sys.modules`` and as the package attribute,
  so ``ALS.fit``'s ``from ._als import als_update`` (``algorithms/als.py:135``) resolves to the GPU solver
  whether or not a Cython build exists;
* optionally (``bpr=True``) the Cython extension ``libreco.algorithms._bpr`` in the same way, with
  ``librecommender_b200.bpr.bpr_update``, so ``BPR(use_tf=False).fit``'s ``from ._bpr import bpr_update``
  (``algorithms/bpr.py:309``) trains on the GPU;
* optionally (``gensim=True``) the ``Word2Vec`` name that ``bases/gensim_base.py:5``, ``algorithms/item2vec.py:2``
  and ``algorithms/deepwalk.py:6`` bound at import → ``librecommender_b200.skipgram.Word2Vec``, and
  ``GensimBase.set_embeddings`` (``gensim_base.py:96-108``, a per-user Python loop) → the device pooling, so
  ``Item2Vec(...).fit`` / ``DeepWalk(...).fit`` train on the GPU whether or not gensim is installed;
* optionally (``sage=True``) ``SageBase.set_embeddings`` (``bases/sage_base.py:136-173``, a Python neighbour walk
  and a torch encoder per batch) → ``librecommender_b200.sage.set_embeddings`` for the non-DGL ``GraphSage`` /
  ``PinSage``; the DGL classes keep the reference's method;
* optionally (``swing=True``) ``Swing.fit`` (``algorithms/swing.py:65-116``, which imports ``recfarm``) → a ``fit``
  that builds ``librecommender_b200.swing.Swing`` into ``self.rs_model``, so the reference's own ``predict`` and
  ``recommend_user`` run on the device engine whether or not ``recfarm`` is installed.  No ``recfarm`` module is
  registered: ``data/consumed.py`` catches only ``ModuleNotFoundError`` on ``from recfarm import ...``;
* optionally (``cf=True``) ``RsCfBase.fit`` (``bases/cf_base_rs.py:64-122``, which imports ``recfarm``) → a ``fit``
  that builds ``librecommender_b200.cf.UserCF`` / ``ItemCF`` into ``self.rs_model``, so the reference's own
  ``RsUserCF`` / ``RsItemCF`` ``predict``, ``recommend_user`` and ``evaluate`` run on the device engines; again no
  ``recfarm`` module is registered.
"""
from __future__ import annotations

import importlib
import sys
import types

_saved: list = []
_MISSING = object()


def _patch(mod, name, value):
    if hasattr(mod, name):
        _saved.append((mod, name, getattr(mod, name)))
        setattr(mod, name, value)


def _register_cython(base, name, func):
    """Put a module holding the GPU ``func`` at ``{base}.algorithms.{name}`` in place of the reference's Cython
    extension; remember what was there (or that nothing was)."""
    full = f"{base}.algorithms.{name}"
    pkg = importlib.import_module(f"{base}.algorithms")
    mod = types.ModuleType(full, f"{func.__module__}.{func.__name__} registered as the reference's {name}")
    setattr(mod, func.__name__, func)
    _saved.append((sys.modules, full, sys.modules.get(full, _MISSING)))
    sys.modules[full] = mod
    _saved.append((pkg, name, getattr(pkg, name, _MISSING)))
    setattr(pkg, name, mod)


def install(libreco=None, losses: bool = True, lightgcn: bool = True, als: bool = False,
            bpr: bool = False, gensim: bool = False, sage: bool = False, swing: bool = False,
            cf: bool = False) -> None:
    """Patch the reference package in place (idempotent: a second call re-installs)."""
    from . import recommendation as rec

    if libreco is None:
        libreco = importlib.import_module("libreco")
    uninstall()
    base = libreco.__name__
    mods = {}
    for sub in ("recommendation", "recommendation.recommend", "bases.embed_base", "bases.dyn_embed_base",
                "algorithms.lightgcn", "training.torch_trainer", "torchops"):
        try:
            mods[sub] = importlib.import_module(f"{base}.{sub}")
        except Exception:                      # a sub-module the installed reference cannot import
            mods[sub] = None
    for sub in ("recommendation", "recommendation.recommend", "bases.embed_base", "bases.dyn_embed_base"):
        m = mods[sub]
        if m is None:
            continue
        _patch(m, "rank_recommendations", rec.rank_recommendations)
        _patch(m, "recommend_from_embedding", rec.recommend_from_embedding)
        _patch(m, "construct_rec", rec.construct_rec)
    if lightgcn and mods["algorithms.lightgcn"] is not None:
        from .lightgcn import make_lightgcn_model_class

        _patch(mods["algorithms.lightgcn"], "LightGCNModel", make_lightgcn_model_class())
    if losses:
        from . import losses as L

        for sub in ("training.torch_trainer", "torchops"):
            m = mods[sub]
            if m is None:
                continue
            for name in ("binary_cross_entropy_loss", "bpr_loss", "compute_pair_scores", "focal_loss",
                         "max_margin_loss", "pairwise_bce_loss", "pairwise_focal_loss"):
                if hasattr(L, name):
                    _patch(m, name, getattr(L, name))
    if als:
        from .als import als_update

        _register_cython(base, "_als", als_update)
    if bpr:
        from .bpr import bpr_update

        _register_cython(base, "_bpr", bpr_update)
    if gensim:
        from . import skipgram

        for sub in ("bases.gensim_base", "algorithms.item2vec", "algorithms.deepwalk"):
            m = importlib.import_module(f"{base}.{sub}")
            _patch(m, "Word2Vec", skipgram.Word2Vec)
        gb = importlib.import_module(f"{base}.bases.gensim_base")
        _patch(gb.GensimBase, "set_embeddings", skipgram.set_embeddings)
    if sage:
        from . import sage as sage_engine

        sb = importlib.import_module(f"{base}.bases.sage_base")
        reference_set_embeddings = sb.SageBase.set_embeddings

        def set_embeddings(model):
            if model.use_dgl:
                return reference_set_embeddings(model)
            return sage_engine.set_embeddings(model)

        _patch(sb.SageBase, "set_embeddings", set_embeddings)
    if swing:
        from . import swing as swing_engine

        sw = importlib.import_module(f"{base}.algorithms.swing")

        def fit(model, train_data, neg_sampling, verbose=1, eval_data=None, metrics=None, k=10, eval_batch_size=8192,
                eval_user_num=None):
            return swing_engine.fit_reference_model(model, sw, train_data, neg_sampling, verbose, eval_data, metrics,
                                                    k, eval_batch_size, eval_user_num)

        _patch(sw.Swing, "fit", fit)
    if cf:
        from . import cf as cf_engine

        cb = importlib.import_module(f"{base}.bases.cf_base_rs")

        def cf_fit(model, train_data, neg_sampling, verbose=1, eval_data=None, metrics=None, k=10,
                   eval_batch_size=8192, eval_user_num=None):
            return cf_engine.fit_reference_model(model, cb, train_data, neg_sampling, verbose, eval_data, metrics, k,
                                                 eval_batch_size, eval_user_num)

        _patch(cb.RsCfBase, "fit", cf_fit)


def uninstall() -> None:
    """Restore every patched name."""
    while _saved:
        mod, name, old = _saved.pop()
        if mod is sys.modules:
            if old is _MISSING:
                sys.modules.pop(name, None)
            else:
                sys.modules[name] = old
        elif old is _MISSING:
            if hasattr(mod, name):
                delattr(mod, name)
        else:
            setattr(mod, name, old)


def installed() -> bool:
    return bool(_saved)
