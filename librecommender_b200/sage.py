"""GraphSage and PinSage inference on the device: what ``SageBase.set_embeddings`` (``libreco/bases/sage_base.py:136-173``)
does for the reference's non-DGL ``GraphSage`` / ``PinSage``, on the kernels of ``csrc/sage.cu`` and the library's
gather and dense-layer kernels.

* Neighbour sampling (``NeighborWalker.sample_graphsage`` / ``sample_pinsage``, ``libreco/graph/neighbor_walk.py``)
  runs per level on the device over CSRs of ``item_consumed`` / ``user_consumed`` kept with list order and
  multiplicity.  The reference's rules are kept; its Python ``random`` streams are not: every draw is Philox4x32-10
  keyed by (seed, root item, path, level, draw), so a seed gives the same neighbours however the items are batched.
* The item encoder (eval mode) hoists the per-item work once over the catalogue: ``P = item_proj(raw(i))`` (K1 gather
  + :func:`feat_models.linear`) and, for PinSage, ``Q0 = relu(q_linears[0](P))``.  Then layer by layer over the sampled
  nodes: ``b200_sage_aggregate`` writes ``[h_self, mean]`` (GraphSage) or ``[h_self, sum w relu(q(h_nb))]`` (PinSage)
  and ``linear`` applies ``w_linears[l]`` with its activation (PinSage: ReLU, the row L2 normalisation, and
  ``G2(relu(G1(.)))`` at the end).
* User rows: i2i, the mean of the consumed item rows with multiplicity (``b200_spmm_csr``); u2i, ``user_proj`` of
  the raw user features (PinSage: then ``U2(relu(U1(.)))``).  Both tables get the mean OOV row
  (``assign_embedding_oov``) and serve through :class:`engine.EmbedScorer`.
* Training (:class:`GraphSageTrainer`, GraphSage only): ``GraphTrainer`` + ``GraphCollator`` on the device, i2i walk
  pairs and negatives from ``csrc/sage_train.cu``, the encoder's backward through ``b200_sage_aggregate_backward``,
  ``torch.optim.Adam`` as TF-Adam; :meth:`GraphSageTrainer.state_dict` loads into :class:`GraphSage`.
"""
from __future__ import annotations

import math

import numpy as np

from . import _lib
from .consumed import ConsumedCSR
from .feat_models import (ACT_NONE, ACT_RELU, FeatSpec, _dev, _spec_get, feat_backward, feat_forward, linear,
                          tables_struct)
from .training import _weight_grad

MAX_LAYERS = 3
MAX_NEIGHBORS = 32
MAX_VISITS = 256
MAX_EMBED = 128
ROWS_PER_CHUNK = 1 << 22      # sampled nodes of the deepest level per encoder chunk
HOIST_CHUNK = 1 << 20


def cont_threshold(termination_prob):
    """Step s > 0 of a PinSage walk is taken when its 32-bit termination word is >= this value, which is
    ``random.random() >= termination_prob`` for u = word / 2^32."""
    return min(1 << 32, max(0, math.ceil(float(termination_prob) * 2.0 ** 32)))


def _csr(consumed, n, n_cols, name):
    """(indptr int64, idx int32) of the reference's dict of lists (or an (indptr, idx) pair), order and multiplicity
    kept; ``ValueError`` for an id outside ``[0, n_cols)``."""
    if isinstance(consumed, tuple):
        indptr, idx = (np.asarray(a) for a in consumed)
    else:
        from .consumed import as_csr

        c = as_csr(consumed, n)
        indptr, idx = c.indptr, c.idx
    indptr = np.ascontiguousarray(indptr, dtype=np.int64)
    if indptr.shape != (n + 1,) or indptr[0] != 0 or np.any(np.diff(indptr) < 0) or indptr[-1] != len(idx):
        raise ValueError(f"{name} is not a CSR over {n} rows")
    idx = np.ascontiguousarray(idx)
    if idx.size and (idx.min() < 0 or idx.max() >= n_cols):
        raise ValueError(f"{name} holds ids outside [0, {n_cols})")
    return indptr, idx.astype(np.int32)


class _SageEngine:
    """Shared host path of :class:`GraphSage` and :class:`PinSage`.

    ``data_info``: the reference's ``DataInfo`` or a dict with ``n_users``, ``n_items``, ``user_consumed``,
    ``item_consumed`` and the feature layout ``FeatSpec`` reads (``item_sparse_col_index``, ``item_sparse_unique``,
    ...).  ``state_dict``: the reference model's ``torch_model.state_dict()`` or the ``model_state_dict`` entry of
    ``<name>_torch.pt`` (torch tensors or numpy arrays).  ``ValueError`` before any launch for keys or shapes that do
    not match the paradigm and layer count, or parameters outside the envelope (layers 1..3, neighbours 1..32,
    embed 1..128)."""

    KIND = ""

    def __init__(self, data_info, state_dict, paradigm="i2i", num_layers=2, num_neighbors=3, seed=42, device=None):
        import torch

        self._torch = torch
        g = _spec_get(data_info)
        self.n_users, self.n_items = int(g("n_users")), int(g("n_items"))
        if paradigm not in ("i2i", "u2i"):
            raise ValueError("`paradigm` must either be `u2i` or `i2i`")
        if not 1 <= int(num_layers) <= MAX_LAYERS:
            raise ValueError(f"num_layers {num_layers} outside [1, {MAX_LAYERS}]")
        if not 1 <= int(num_neighbors) <= MAX_NEIGHBORS:
            raise ValueError(f"num_neighbors {num_neighbors} outside [1, {MAX_NEIGHBORS}]")
        self.paradigm, self.num_layers, self.num_neighbors = paradigm, int(num_layers), int(num_neighbors)
        self.seed = int(seed) & ((1 << 64) - 1)
        self.item_ptr, self.item_users = _csr(g("item_consumed"), self.n_items, self.n_users, "item_consumed")
        self.user_ptr, self.user_items = _csr(g("user_consumed"), self.n_users, self.n_items, "user_consumed")
        self.user_consumed = ConsumedCSR(self.user_ptr, self.user_items)
        sd = {k: (v.detach().cpu().numpy() if hasattr(v, "detach") else np.asarray(v)) for k, v in state_dict.items()}
        self.d = self._check_state(sd, g)
        self.device = torch.device(device) if device is not None else _lib.require_cuda()
        f32 = torch.float32
        self.spec = FeatSpec(data_info, self.d, self.device)
        self.t = {"item_embeds": _dev(sd["item_embeds.weight"], self.device, f32),
                  "user_embeds": _dev(sd.get("user_embeds.weight"), self.device, f32),
                  "sparse_embeds": _dev(sd.get("sparse_embeds.weight"), self.device, f32),
                  "dense_embeds": _dev(sd.get("dense_embeds"), self.device, f32)}
        self.tables = tables_struct(self.t)
        self.w = {k: _dev(self._side_order(k, v), self.device, f32) for k, v in sd.items() if not k.endswith("embeds")
                  and not k.endswith("embeds.weight")}
        self.graph = [torch.as_tensor(a).to(self.device) for a in (self.item_ptr, self.item_users, self.user_ptr,
                                                                     self.user_items)]
        self.item_deg = np.diff(self.item_ptr)
        self.P = self.Q0 = None
        self.tables_d = self.scorer = None

    # ---- weights -----------------------------------------------------------------------------------------------------
    def _expected(self, g, d):
        """{key: shape} of the state dict the model's paradigm and layer count give (embed size d)."""
        width = {s: len(list(g(f"{s}_sparse_col_index") or [])) + len(list(g(f"{s}_dense_col_index") or []))
                 for s in ("user", "item")}
        shapes = {"item_embeds.weight": (self.n_items, d), "item_proj.weight": (d, (width["item"] + 1) * d),
                  "item_proj.bias": (d,)}
        if self.paradigm == "u2i":
            shapes.update({"user_embeds.weight": (self.n_users, d), "user_proj.bias": (d,),
                           "user_proj.weight": (d, (width["user"] + 1) * d)})
        for layer in range(self.num_layers):
            shapes[f"w_linears.{layer}.weight"] = (d, 2 * d)
            shapes[f"w_linears.{layer}.bias"] = (d,)
        return shapes

    def _check_state(self, sd, g):
        if "item_embeds.weight" not in sd or np.ndim(sd["item_embeds.weight"]) != 2:
            raise ValueError(f"{self.KIND} state dict: no 2-D item_embeds.weight")
        d = int(np.shape(sd["item_embeds.weight"])[1])
        if not 1 <= d <= MAX_EMBED:
            raise ValueError(f"embed size {d} outside [1, {MAX_EMBED}]")
        shapes = self._expected(g, d)
        optional = {"sparse_embeds.weight", "dense_embeds"}
        missing = sorted(set(shapes) - set(sd))
        extra = sorted(set(sd) - set(shapes) - optional)
        if missing or extra:
            raise ValueError(f"{self.KIND} {self.paradigm} state dict: missing {missing}, unexpected {extra}")
        for k, want in shapes.items():
            if tuple(np.shape(sd[k])) != want:
                raise ValueError(f"{k} has shape {tuple(np.shape(sd[k]))}, expected {want}")
        for k in optional & set(sd):
            if np.ndim(sd[k]) != 2 or np.shape(sd[k])[1] != d:
                raise ValueError(f"{k} has shape {tuple(np.shape(sd[k]))}, expected (n, {d})")
        for s in ("item", "user") if self.paradigm == "u2i" else ("item",):
            if list(g(f"{s}_sparse_col_index") or []) and "sparse_embeds.weight" not in sd:
                raise ValueError("the data has sparse features but the state dict no sparse_embeds.weight")
            if list(g(f"{s}_dense_col_index") or []) and "dense_embeds" not in sd:
                raise ValueError("the data has dense features but the state dict no dense_embeds")
        return d

    def _side_order(self, key, w):
        """The projections read [sparse.., dense.., id] (get_raw_features); the K1 side gather writes [id, sparse..,
        dense..]: move the id block of the weight's columns first."""
        w = np.asarray(w, dtype=np.float32)
        if key in ("item_proj.weight", "user_proj.weight"):
            d = self.d
            w = np.concatenate([w[:, -d:], w[:, :-d]], axis=1)
        return np.ascontiguousarray(w)

    def _lin(self, x, name, act, bias=True):
        return linear(x, self.w[f"{name}.weight"], self.w[f"{name}.bias"] if bias else None, act)

    # ---- raw features -----------------------------------------------------------------------------------------------
    def _project(self, which, ids_d):
        """``{which}_proj(raw features)`` of the ids: K1 side gather, then the projection."""
        torch = self._torch
        L, pos = self.spec.side(which)
        n = int(ids_d.numel())
        x = torch.empty((n, len(pos) * self.d), dtype=torch.float32, device=self.device)
        feat_forward(L, self.tables, ids_d, ids_d, n, concat=x)
        return self._lin(x, f"{which}_proj", ACT_NONE)

    def _hoist(self):
        """P = item_proj(raw(i)) over the catalogue (and PinSage's Q0 = relu(q_linears[0](P))), once."""
        if self.P is not None:
            return
        torch = self._torch
        parts = []
        for i0 in range(0, self.n_items, HOIST_CHUNK):
            ids = torch.arange(i0, min(self.n_items, i0 + HOIST_CHUNK), dtype=torch.int64, device=self.device)
            parts.append(self._project("item", ids))
        self.P = torch.cat(parts) if len(parts) > 1 else parts[0]
        if self.KIND == "PinSage":
            self.Q0 = self._lin(self.P, "q_linears.0", ACT_RELU)

    # ---- sampling ---------------------------------------------------------------------------------------------------
    def _check_items(self, items):
        items = np.asarray(items).reshape(-1)
        if items.size and (not np.issubdtype(items.dtype, np.integer) or items.min() < 0
                           or items.max() >= self.n_items):
            raise ValueError(f"item ids outside [0, {self.n_items})")
        items = items.astype(np.int64)
        if items.size and np.any(self.item_deg[items] == 0):
            bad = int(items[self.item_deg[items] == 0][0])
            raise ValueError(f"item {bad} has no consumer to walk from")
        return items

    def _sample_level(self, roots_d, nodes_d, per_root, level):
        raise NotImplementedError

    def _sample(self, roots_d):
        """Device levels for the roots: a list of (ids [n_l, nn], weights or None, lens or None)."""
        nodes, per_root, out = roots_d, 1, []
        for level in range(self.num_layers):
            res = self._sample_level(roots_d, nodes, per_root, level)
            out.append(res)
            nodes, per_root = res[0].reshape(-1), per_root * self.num_neighbors
        return out

    def neighbors(self, items):
        """The sampled message of the items, per level on host: GraphSage ``ids`` [n_l, num_neighbors]; PinSage
        ``(ids, weights, lens)``, padded with -1 / 0 past each length.  Level l+1 samples for every slot of level l
        (flattened), so level l has ``len(items) * num_neighbors ** l`` rows."""
        torch = self._torch
        items = self._check_items(items)
        levels = self._sample(torch.as_tensor(items.astype(np.int32)).to(self.device))
        host = [tuple(None if a is None else a.cpu().numpy() for a in lv) for lv in levels]
        return [h[0] for h in host] if self.KIND == "GraphSage" else host

    # ---- encoder ----------------------------------------------------------------------------------------------------
    def _encode(self, ids, bags):
        """Item rows of the roots ``ids[0]``: ``ids[k]`` int32 device node ids of level k (k = 0..L; a negative id is
        an empty padded slot), ``bags[k] = (offsets int64 [n_k + 1] or None, lens int32 [n_k] or None, weights float
        [n_{k+1}] or None)``, the neighbour rows of level k (``offsets`` None: ``num_neighbors`` per row)."""
        torch = self._torch
        self._hoist()
        L, d = self.num_layers, self.d
        pin = self.KIND == "PinSage"
        H = None
        for layer in range(L):
            nxt = []
            for k in range(L - layer):
                n_k = int(ids[k].numel())
                if layer == 0:
                    S, sidx, N, nidx = self.P, ids[k], (self.Q0 if pin else self.P), ids[k + 1]
                else:
                    S, sidx, nidx = H[k], None, None
                    N = self._lin(H[k + 1], f"q_linears.{layer}", ACT_RELU) if pin else H[k + 1]
                offs, lens, wts = bags[k]
                agg = torch.empty((n_k, 2 * d), dtype=torch.float32, device=self.device)
                _lib.check(_lib.lib.b200_sage_aggregate(
                    _lib.ptr(S), S.stride(0), _lib.ptr(sidx), n_k, _lib.ptr(N), N.stride(0), _lib.ptr(nidx),
                    _lib.ptr(offs), _lib.ptr(lens), self.num_neighbors, _lib.ptr(wts), d, _lib.ptr(agg), agg.stride(0),
                    _lib.current_stream()))
                act = ACT_RELU if pin or layer != L - 1 else ACT_NONE
                h = self._lin(agg, f"w_linears.{layer}", act)
                if pin:
                    _lib.check(_lib.lib.b200_l2_normalize_rows(_lib.ptr(h), h.stride(0), n_k, d,
                                                               _lib.current_stream()))
                nxt.append(h)
            H = nxt
        out = H[0]
        if pin:
            out = self._lin(self._lin(out, "G1", ACT_RELU), "G2", ACT_NONE, bias=False)
        return out

    def encode_message(self, items, neighbors, offsets, weights=None):
        """Item rows (device [n, d]) of a message in the reference's form (``ItemMessage``: per-level neighbour ids,
        per-level offsets into them, PinSage's per-level weights), e.g. one recorded from ``NeighborWalker``."""
        torch = self._torch
        items = self._check_items(items)
        if len(neighbors) != self.num_layers or len(offsets) != self.num_layers:
            raise ValueError(f"the message must have {self.num_layers} levels")
        if (weights is None) != (self.KIND == "GraphSage"):
            raise ValueError("PinSage messages carry weights, GraphSage messages none")
        ids = [torch.as_tensor(items.astype(np.int32)).to(self.device)]
        bags = []
        for k in range(self.num_layers):
            nb = self._check_items(neighbors[k]) if len(neighbors[k]) else np.zeros(0, np.int64)
            off = np.asarray(offsets[k], dtype=np.int64).reshape(-1)
            if off.size != ids[k].numel() or (off.size and (off[0] != 0 or np.any(np.diff(off) < 0)
                                                            or off[-1] > nb.size)):
                raise ValueError(f"offsets of level {k} do not split its {nb.size} neighbours over "
                                 f"{ids[k].numel()} rows")
            off = torch.as_tensor(np.append(off, nb.size)).to(self.device)
            w = None
            if weights is not None:
                w = torch.as_tensor(np.asarray(weights[k], dtype=np.float32).reshape(-1)).to(self.device)
                if w.numel() != nb.size:
                    raise ValueError(f"weights of level {k} do not match its neighbours")
            ids.append(torch.as_tensor(nb.astype(np.int32)).to(self.device))
            bags.append((off, None, w))
        return self._encode(ids, bags)

    def _encode_roots(self, roots_d):
        levels = self._sample(roots_d)
        ids = [roots_d] + [lv[0].reshape(-1) for lv in levels]
        bags = [(None, lv[2], None if lv[1] is None else lv[1].reshape(-1)) for lv in levels]
        return self._encode(ids, bags)

    def item_embeddings(self):
        """Device ``[n_items, d]``: every item through the sampler and the encoder, in chunks of roots."""
        torch = self._torch
        self._check_items(np.arange(self.n_items))
        chunk = max(1, ROWS_PER_CHUNK // self.num_neighbors ** self.num_layers)
        out = torch.empty((self.n_items, self.d), dtype=torch.float32, device=self.device)
        for i0 in range(0, self.n_items, chunk):
            roots = torch.arange(i0, min(self.n_items, i0 + chunk), dtype=torch.int32, device=self.device)
            out[i0:i0 + roots.numel()] = self._encode_roots(roots)
        return out

    def user_embeddings(self, item_embeds=None):
        """Device ``[n_users, d]``: i2i, the mean of each user's consumed item rows of ``item_embeds`` (default
        :meth:`item_embeddings`), duplicates included; u2i, the user tower over the raw user features."""
        torch = self._torch
        if self.paradigm == "i2i":
            from .skipgram import pool_users

            I = self.item_embeddings() if item_embeds is None else item_embeds
            return pool_users(self.user_ptr, self.user_items, I)
        parts = []
        for u0 in range(0, self.n_users, HOIST_CHUNK):
            ids = torch.arange(u0, min(self.n_users, u0 + HOIST_CHUNK), dtype=torch.int64, device=self.device)
            x = self._project("user", ids)
            if self.KIND == "PinSage":
                x = self._lin(self._lin(x, "U1", ACT_RELU), "U2", ACT_NONE, bias=False)
            parts.append(x)
        return torch.cat(parts) if len(parts) > 1 else parts[0]

    def set_embeddings(self):
        """Device ``(U [n_users + 1, d], I [n_items + 1, d])``, the last row of each the mean row
        (``assign_embedding_oov``); they also back :meth:`recommend_user` and :meth:`predict`."""
        from .engine import EmbedScorer

        torch = self._torch
        I = self.item_embeddings()
        U = self.user_embeddings(I)
        U = torch.cat([U, U.mean(dim=0, keepdim=True)])
        I = torch.cat([I, I.mean(dim=0, keepdim=True)])
        self.tables_d = (U, I)
        self.scorer = EmbedScorer(U, I, self.n_items, self.user_consumed, n_users=self.n_users, device=self.device)
        return U, I

    def _ready(self):
        if self.scorer is None:
            self.set_embeddings()
        return self.scorer

    def recommend_user(self, users, n_rec, filter_consumed=True, return_scores=False):
        """Top ``n_rec`` item ids per user (inner ids; ``n_users`` is the OOV user) over the device tables."""
        users = np.asarray(users, dtype=np.int64).reshape(-1)
        if users.size and (users.min() < 0 or users.max() > self.n_users):
            raise ValueError(f"user ids outside [0, {self.n_users}]")
        return self._ready().recommend(users.tolist(), int(n_rec), filter_consumed, return_scores)

    def predict(self, users, items):
        """expit of the dot product of the user and item rows (``predict_from_embedding`` +
        ``normalize_prediction`` for ranking); ids up to ``n_users`` / ``n_items`` (the OOV rows)."""
        users = np.asarray(users, dtype=np.int64).reshape(-1)
        items = np.asarray(items, dtype=np.int64).reshape(-1)
        if users.shape != items.shape:
            raise ValueError("users and items differ in length")
        if users.size and (users.min() < 0 or users.max() > self.n_users or items.min() < 0
                           or items.max() > self.n_items):
            raise ValueError("user or item ids out of range")
        return self._ready().predict(users, items, mode=1)


class GraphSage(_SageEngine):
    """``GraphSage`` (``libreco/algorithms/graphsage.py``) inference: ``num_neighbors`` one-walk neighbours per node
    and level, mean aggregation, ReLU on every layer but the last."""

    KIND = "GraphSage"

    def _sample_level(self, roots_d, nodes_d, per_root, level):
        torch = self._torch
        n = int(nodes_d.numel())
        out = torch.empty((n, self.num_neighbors), dtype=torch.int32, device=self.device)
        _lib.check(_lib.lib.b200_sage_neighbors(*[_lib.ptr(a) for a in self.graph], _lib.ptr(roots_d),
                                                _lib.ptr(nodes_d), n, per_root, level, self.num_neighbors, self.seed,
                                                _lib.ptr(out), _lib.current_stream()))
        return out, None, None


class PinSage(_SageEngine):
    """``PinSage`` (``libreco/algorithms/pinsage.py``) inference: ``num_walks`` random walks of at most
    ``neighbor_walk_len`` one-walks per node and level, the ``num_neighbors`` most visited with visit-count weights,
    the q / w layers with the row L2 normalisation, ``G2(relu(G1(.)))`` at the end.  ``num_walks *
    neighbor_walk_len`` must be at most 256."""

    KIND = "PinSage"

    def __init__(self, data_info, state_dict, paradigm="i2i", num_layers=2, num_neighbors=3, num_walks=10,
                 neighbor_walk_len=2, termination_prob=0.5, seed=42, device=None):
        if not (int(num_walks) >= 1 and int(neighbor_walk_len) >= 1
                and int(num_walks) * int(neighbor_walk_len) <= MAX_VISITS):
            raise ValueError(f"num_walks * neighbor_walk_len must lie in [1, {MAX_VISITS}]")
        if not 0.0 <= float(termination_prob) <= 1.0:
            raise ValueError(f"termination_prob {termination_prob} outside [0, 1]")
        self.num_walks, self.walk_len = int(num_walks), int(neighbor_walk_len)
        self.threshold = cont_threshold(termination_prob)
        super().__init__(data_info, state_dict, paradigm, num_layers, num_neighbors, seed, device)

    def _expected(self, g, d):
        shapes = super()._expected(g, d)
        for layer in range(self.num_layers):
            shapes[f"q_linears.{layer}.weight"] = (d, d)
            shapes[f"q_linears.{layer}.bias"] = (d,)
        shapes.update({"G1.weight": (d, d), "G1.bias": (d,), "G2.weight": (d, d)})
        if self.paradigm == "u2i":
            shapes.update({"U1.weight": (d, d), "U1.bias": (d,), "U2.weight": (d, d)})
        return shapes

    def _sample_level(self, roots_d, nodes_d, per_root, level):
        torch = self._torch
        n, nn = int(nodes_d.numel()), self.num_neighbors
        ids = torch.empty((n, nn), dtype=torch.int32, device=self.device)
        wts = torch.empty((n, nn), dtype=torch.float32, device=self.device)
        lens = torch.empty(n, dtype=torch.int32, device=self.device)
        _lib.check(_lib.lib.b200_pinsage_neighbors(*[_lib.ptr(a) for a in self.graph], _lib.ptr(roots_d),
                                                   _lib.ptr(nodes_d), n, per_root, level, nn, self.num_walks,
                                                   self.walk_len, self.threshold, self.seed, _lib.ptr(ids),
                                                   _lib.ptr(wts), _lib.ptr(lens), _lib.current_stream()))
        return ids, wts, lens


def engine_for(model):
    """The device engine of a fitted reference ``GraphSage`` / ``PinSage`` (non-DGL) model."""
    kw = dict(paradigm=model.paradigm, num_layers=model.num_layers, num_neighbors=model.num_neighbors,
              seed=model.seed)
    sd = model.torch_model.state_dict()
    if "PinSage" in model.model_name:
        return PinSage(model.data_info, sd, num_walks=model.num_walks, neighbor_walk_len=model.neighbor_walk_len,
                       termination_prob=model.termination_prob, **kw)
    return GraphSage(model.data_info, sd, **kw)


def set_embeddings(model):
    """``SageBase.set_embeddings`` on the device for the non-DGL classes: sets ``item_embeds_np`` /
    ``user_embeds_np`` (without the OOV rows, which ``fit`` appends)."""
    eng = engine_for(model)
    I = eng.item_embeddings()
    U = eng.user_embeddings(I)
    model.item_embeds_np = I.cpu().numpy()
    model.user_embeds_np = U.cpu().numpy()


# ---- GraphSage training ---------------------------------------------------------------------------------------------
BETA1, BETA2 = 0.9, 0.999                    # torch.optim.Adam defaults (training/torch_trainer.py:63-68)
LOSS_KINDS = {"bpr": 0, "max_margin": 1, "cross_entropy": 2, "focal": 3}    # b200_pairwise_loss kinds
NEG_TOLERANCE = 10                           # negatives_from_random's tolerance
_M64 = (1 << 64) - 1


def adam_step_constants(lr, epsilon, t):
    """``torch.optim.Adam`` step t (from 1) as TF-Adam: ``p -= lr_t m / (sqrt(v) + eps_hat)`` with ``lr_t = lr
    sqrt(1 - beta2^t) / (1 - beta1^t)`` and ``eps_hat = eps sqrt(1 - beta2^t)``.  torch divides sqrt(v) by
    sqrt(1 - beta2^t) before adding eps; multiplying through by that factor gives the TF form exactly."""
    c2 = math.sqrt(1.0 - BETA2 ** t)
    return lr * c2 / (1.0 - BETA1 ** t), epsilon * c2


def _mix(seed, step, role):
    """splitmix64 of (seed, step, role): one sampler seed per step and use, so each step draws fresh neighbours."""
    x = (int(seed) + 0x9E3779B97F4A7C15 * (2 * int(step) + 1) + 0xD1B54A32D192ED03 * (int(role) + 1)) & _M64
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & _M64
    return x ^ (x >> 31)


def _xavier(rng, shape, gain=1.0):
    """nn.init.xavier_uniform_ of a 2-D weight (fan_in = shape[1], fan_out = shape[0])."""
    bound = gain * math.sqrt(6.0 / (shape[0] + shape[1]))
    return rng.uniform(-bound, bound, size=shape).astype(np.float32)


def init_state_dict(data_info, paradigm="i2i", embed_size=16, num_layers=2, seed=42):
    """A fresh ``GraphSageModel`` state dict as ``init_parameters`` draws it (graphsage_module.py:38-49, 91-99):
    xavier-uniform tables and projections, ``w_linears`` with the relu gain on every layer but the last, zero biases.
    The shapes are the reference's; the values come from numpy's generator seeded by ``seed``."""
    g = _spec_get(data_info)
    d = int(embed_size)
    rng = np.random.default_rng(seed)
    n_users, n_items = int(g("n_users")), int(g("n_items"))
    sides = ("user", "item") if paradigm == "u2i" else ("item",)
    width = {s: len(list(g(f"{s}_sparse_col_index") or [])) + len(list(g(f"{s}_dense_col_index") or []))
             for s in ("user", "item")}
    sd = {}
    for s in sides:
        sd[f"{s}_embeds.weight"] = _xavier(rng, ((n_users if s == "user" else n_items), d))
        sd[f"{s}_proj.weight"] = _xavier(rng, (d, (width[s] + 1) * d))
        sd[f"{s}_proj.bias"] = np.zeros(d, np.float32)
    uniq = [np.asarray(g(f"{s}_sparse_unique")) for s in ("user", "item")
            if list(g(f"{s}_sparse_col_index") or []) and g(f"{s}_sparse_unique") is not None]
    if uniq:                                  # sparse_feat_size: the largest index + 1
        sd["sparse_embeds.weight"] = _xavier(rng, (int(max(int(u.max()) for u in uniq)) + 1, d))
    n_dense = len(list(g("user_dense_col_index") or [])) + len(list(g("item_dense_col_index") or []))
    if n_dense:
        sd["dense_embeds"] = _xavier(rng, (n_dense, d))
    relu_gain = math.sqrt(2.0)
    for layer in range(num_layers):
        sd[f"w_linears.{layer}.weight"] = _xavier(rng, (d, 2 * d), relu_gain if layer != num_layers - 1 else 1.0)
        sd[f"w_linears.{layer}.bias"] = np.zeros(d, np.float32)
    return sd


def _check_train_options(paradigm, loss_type, sampler, start_node, lr_decay, amsgrad, dropout_rate, remove_edges):
    if paradigm not in ("i2i", "u2i"):
        raise ValueError("`paradigm` must either be `u2i` or `i2i`")
    if loss_type not in LOSS_KINDS:
        raise ValueError(f"unsupported `loss_type` {loss_type!r}, expected one of {sorted(LOSS_KINDS)}")
    if lr_decay:
        raise ValueError("lr_decay (CosineAnnealingWarmRestarts) is not supported by GraphSageTrainer")
    if amsgrad:
        raise ValueError("amsgrad is not supported by GraphSageTrainer")
    if dropout_rate:
        raise ValueError("dropout_rate > 0 is not supported by GraphSageTrainer")
    if remove_edges:
        raise ValueError("remove_edges is not supported by GraphSageTrainer")
    if sampler in ("popular", "out-batch"):
        raise ValueError(f"the {sampler!r} sampler is not supported by GraphSageTrainer")
    allowed = ("random", "unconsumed") if paradigm == "u2i" else ("random",)
    if sampler not in allowed:
        raise ValueError(f"`sampler` must be one of {allowed} for {paradigm}, got {sampler!r}")
    if start_node == "unpopular":
        raise ValueError("start_node='unpopular' is not supported by GraphSageTrainer")
    if start_node != "random":
        raise ValueError(f"`start_node` must be 'random', got {start_node!r}")


class GraphSageTrainer:
    """Device training of the non-DGL ``GraphSage`` (``GraphSageModel``, graphsage_module.py:82-140) with
    ``GraphTrainer`` (training/torch_trainer.py:170-282) and ``GraphCollator`` (batch/collators.py:338-386).

    One :meth:`step` per mini-batch, every piece on the device:

        i2i: b200_sage_walk_pairs (start items, walk pairs) -> b200_sage_i2i_negatives;  u2i: the batch's (user, item)
        pairs -> b200_sample_negatives -> b200_sage_neighbors per level for the query, positive and negative items
        (one encoder pass over all three) -> K1 gather + item_proj -> per layer b200_sage_aggregate + w_linears ->
        pair scores -> b200_pairwise_loss -> the same chain backward (b200_sage_aggregate_backward, the dense-layer
        kernel for dX / dW, b200_feat_backward into the tables) -> torch.optim.Adam as TF-Adam (b200_adam_dense_dev
        with eps_hat = eps sqrt(1 - beta2^t), weight_decay = reg added to the gradient by b200_axpy).

    The only device-to-host copy inside a step is the number of i2i walk pairs, which sizes the batch.  Neighbour
    draws are keyed by (seed, step, encoder row, path, level), so every occurrence of an item in a batch draws its
    own neighbours, as the reference's per-call ``random.choice`` does; the streams themselves are not the
    reference's.

    ``state_dict``: a ``GraphSageModel`` state dict to start from, else :func:`init_state_dict`.  The options are the
    reference's; ``lr_decay``, ``amsgrad``, ``dropout_rate > 0``, ``remove_edges``, the ``popular`` / ``out-batch``
    samplers and ``start_node='unpopular'`` raise ``ValueError``."""

    def __init__(self, data_info, state_dict=None, paradigm="i2i", loss_type="cross_entropy", embed_size=16,
                 num_layers=2, num_neighbors=3, num_neg=1, lr=1e-3, epsilon=1e-8, reg=None, margin=1.0,
                 sampler="random", num_walks=10, sample_walk_len=5, start_node="random", focus_start=False,
                 lr_decay=False, amsgrad=False, dropout_rate=0.0, remove_edges=False, seed=42, device=None):
        _check_train_options(paradigm, loss_type, sampler, start_node, lr_decay, amsgrad, dropout_rate, remove_edges)
        g = _spec_get(data_info)
        n_items = int(g("n_items"))
        if not 0 < int(num_neg) < n_items:
            raise ValueError(f"`num_neg` should be positive and smaller than total items, got {num_neg}, {n_items}")
        if not (1 <= int(num_walks) <= 1024 and 1 <= int(sample_walk_len) <= 1024):
            raise ValueError("num_walks and sample_walk_len must lie in [1, 1024]")
        if reg is not None and not (isinstance(reg, float) and reg > 0.0):
            raise ValueError("reg must be float and positive...")
        import torch

        self._torch = torch
        if state_dict is None:
            state_dict = init_state_dict(data_info, paradigm, embed_size, num_layers, seed)
        self.data_info = data_info
        self.eng = GraphSage(data_info, state_dict, paradigm, num_layers, num_neighbors, seed, device)
        e = self.eng
        if paradigm == "i2i" and np.any(e.item_deg == 0):
            raise ValueError(f"item {int(np.flatnonzero(e.item_deg == 0)[0])} has no consumer to walk from")
        self.device, self.d, self.paradigm = e.device, e.d, paradigm
        self.n_users, self.n_items = e.n_users, e.n_items
        self.num_layers, self.num_neighbors, self.seed = e.num_layers, e.num_neighbors, e.seed
        self.loss_type, self.kind = loss_type, LOSS_KINDS[loss_type]
        self.num_neg, self.margin, self.sampler = int(num_neg), float(margin), sampler
        self.num_walks, self.walk_len, self.focus_start = int(num_walks), int(sample_walk_len), bool(focus_start)
        self.lr, self.epsilon, self.reg = float(lr), float(epsilon), float(reg or 0.0)
        # the trainable tensors are the engine's own device copies, updated in place
        self.params = {k: v for k, v in e.t.items() if v is not None}
        self.params.update(e.w)
        self.grads = {k: torch.zeros_like(v) for k, v in self.params.items()}
        self.m = {k: torch.zeros_like(v) for k, v in self.params.items()}
        self.v = {k: torch.zeros_like(v) for k, v in self.params.items()}
        # torch's Adam skips a parameter without a gradient: the feature tables no side of the paradigm reads
        sides = ("user", "item") if paradigm == "u2i" else ("item",)
        reads = {"sparse_embeds": any(getattr(e.spec, f"{s}_sparse_cols") for s in sides),
                 "dense_embeds": any(getattr(e.spec, f"{s}_dense_cols") for s in sides)}
        self.frozen = {k for k, used in reads.items() if k in self.params and not used}
        self.t = 0
        self._step_dev = torch.zeros(1, dtype=torch.int64, device=self.device)
        self._lr_t = torch.zeros(1, dtype=torch.float32, device=self.device)
        self._lws = torch.empty(int(_lib.lib.b200_loss_workspace_bytes()), dtype=torch.uint8, device=self.device)
        self._sorted = None
        if sampler == "unconsumed":          # b200_sample_negatives reads each user's items sorted
            row = np.repeat(np.arange(self.n_users), np.diff(e.user_ptr))
            idx = e.user_items[np.lexsort((e.user_items, row))]
            self._sorted = (torch.as_tensor(e.user_ptr).to(self.device),
                            torch.as_tensor(np.ascontiguousarray(idx)).to(self.device))
        self.last = None

    # ---- sampling ---------------------------------------------------------------------------------------------------
    def walk_pairs(self, n_starts, step=None):
        """(starts, items, items_pos) int32 device tensors of one i2i batch: ``n_starts`` start items and their
        random-walk pairs.  The pair count is the one device-to-host copy of a step."""
        torch = self._torch
        step = self.t if step is None else int(step)
        dev, n = self.device, int(n_starts)
        slots = n * (self.num_walks + 1)
        starts = torch.empty(n, dtype=torch.int32, device=dev)
        counts = torch.empty(slots, dtype=torch.int64, device=dev)
        offsets = torch.empty(slots + 1, dtype=torch.int64, device=dev)
        args = [_lib.ptr(a) for a in self.eng.graph] + [self.n_items, n, self.num_walks, self.walk_len,
                                                         int(self.focus_start), self.seed, step, _lib.ptr(starts)]
        _lib.check(_lib.lib.b200_sage_walk_pairs(*args, _lib.ptr(counts), _lib.ptr(offsets), None, None,
                                                 _lib.current_stream()))
        total = int(offsets[slots].item())
        items = torch.empty(total, dtype=torch.int32, device=dev)
        items_pos = torch.empty(total, dtype=torch.int32, device=dev)
        if total:
            _lib.check(_lib.lib.b200_sage_walk_pairs(*args, None, _lib.ptr(offsets), _lib.ptr(items),
                                                     _lib.ptr(items_pos), _lib.current_stream()))
        return starts, items, items_pos

    def negatives(self, items_pos, items=None, users=None, step=None):
        """int32 device [n * num_neg]: i2i (``items`` given) excludes each pair's item and positive; u2i draws
        with the ``random`` or ``unconsumed`` rule of b200_sample_negatives."""
        torch = self._torch
        step = self.t if step is None else int(step)
        n, f = int(items_pos.numel()), self.num_neg
        if items is not None:
            out = torch.empty(n * f, dtype=torch.int32, device=self.device)
            _lib.check(_lib.lib.b200_sage_i2i_negatives(_lib.ptr(items), _lib.ptr(items_pos), n, f, self.n_items,
                                                        NEG_TOLERANCE, self.seed, step, _lib.ptr(out),
                                                        _lib.current_stream()))
            return out
        out = torch.empty(n * f, dtype=torch.int64, device=self.device)
        pos64 = items_pos.to(torch.int64)
        users64 = users.to(torch.int64)
        mode = 1 if self.sampler == "unconsumed" else 0
        indptr, idx = self._sorted if mode == 1 else (None, None)
        _lib.check(_lib.lib.b200_sample_negatives(_lib.ptr(users64), _lib.ptr(pos64), n, f, self.n_items, mode,
                                                  NEG_TOLERANCE, self.seed, step, _lib.ptr(indptr), _lib.ptr(idx),
                                                  self.n_users, None, _lib.ptr(out), _lib.current_stream()))
        return out.to(torch.int32)

    def levels(self, items, step=None):
        """Node ids per level (int32 device): level 0 the items, level l+1 ``num_neighbors`` per node of level l.
        Each row of ``items`` roots its own draws (keyed by its position), so a repeated item draws anew."""
        torch = self._torch
        step = self.t if step is None else int(step)
        nn, seed = self.num_neighbors, _mix(self.seed, step, 0)
        keys = torch.arange(int(items.numel()), dtype=torch.int32, device=self.device)
        ids, nodes, per_root = [items], items, 1
        for level in range(self.num_layers):
            n = int(nodes.numel())
            out = torch.empty(n * nn, dtype=torch.int32, device=self.device)
            _lib.check(_lib.lib.b200_sage_neighbors(*[_lib.ptr(a) for a in self.eng.graph], _lib.ptr(keys),
                                                    _lib.ptr(nodes), n, per_root, level, nn, seed, _lib.ptr(out),
                                                    _lib.current_stream()))
            ids.append(out)
            nodes, per_root = out, per_root * nn
        return ids

    # ---- encoder ----------------------------------------------------------------------------------------------------
    def _project(self, which, ids64):
        torch = self._torch
        L, pos = self.eng.spec.side(which)
        n = int(ids64.numel())
        x = torch.empty((n, len(pos) * self.d), dtype=torch.float32, device=self.device)
        feat_forward(L, self.eng.tables, ids64, ids64, n, concat=x)
        p = self.params
        return x, linear(x, p[f"{which}_proj.weight"], p[f"{which}_proj.bias"], ACT_NONE, cache_split=False)

    def _project_backward(self, which, ids64, x, dy):
        p, g = self.params, self.grads
        g[f"{which}_proj.weight"] += _weight_grad(dy, x)
        _col_sum(dy, g[f"{which}_proj.bias"])
        dx = linear(dy, p[f"{which}_proj.weight"].t().contiguous(), None, ACT_NONE, cache_split=False)
        feat_backward(self.eng.spec.side(which)[0], self.eng.tables, ids64, ids64, int(ids64.numel()), g, dconcat=dx)

    def encode(self, ids):
        """GraphSageModel.forward over the levels ``ids`` (from :meth:`levels`): (rows [n_0, d], cache).  Every level
        is projected in one gather and one GEMM; the levels of a layer are aggregated into one buffer and go through
        one GEMM."""
        torch = self._torch
        d, L, nn = self.d, self.num_layers, self.num_neighbors
        sizes = [int(a.numel()) for a in ids]
        offs = np.concatenate([[0], np.cumsum(sizes)]).tolist()
        ids64 = torch.cat(ids).to(torch.int64)
        x, H = self._project("item", ids64)
        c = dict(ids64=ids64, x=x, offs=offs, aggs=[], outs=[])
        for layer in range(L):
            depth = L - layer
            agg = torch.empty((offs[depth], 2 * d), dtype=torch.float32, device=self.device)
            for k in range(depth):
                S, N, out = H[offs[k]:offs[k + 1]], H[offs[k + 1]:offs[k + 2]], agg[offs[k]:offs[k + 1]]
                _lib.check(_lib.lib.b200_sage_aggregate(
                    _lib.ptr(S), d, None, sizes[k], _lib.ptr(N), d, None, None, None, nn, None, d, _lib.ptr(out),
                    2 * d, _lib.current_stream()))
            H = linear(agg, self.params[f"w_linears.{layer}.weight"], self.params[f"w_linears.{layer}.bias"],
                       ACT_RELU if layer != L - 1 else ACT_NONE, cache_split=False)
            c["aggs"].append(agg)
            c["outs"].append(H)
        return H, c

    def encode_backward(self, c, dH):
        """Gradients of :meth:`encode`'s parameters ADDED into ``grads`` given d loss / d rows."""
        torch = self._torch
        lib, st = _lib.lib, _lib.current_stream()
        d, L, nn, offs = self.d, self.num_layers, self.num_neighbors, c["offs"]
        p, g = self.params, self.grads
        G = dH.contiguous()
        for layer in range(L - 1, -1, -1):
            depth = L - layer
            if layer != L - 1:
                dz = torch.empty_like(G)
                _lib.check(lib.b200_relu_backward(_lib.ptr(G), _lib.ptr(c["outs"][layer]), G.numel(), _lib.ptr(dz),
                                                  st))
                G = dz
            g[f"w_linears.{layer}.weight"] += _weight_grad(G, c["aggs"][layer])
            _col_sum(G, g[f"w_linears.{layer}.bias"])
            dagg = linear(G, p[f"w_linears.{layer}.weight"].t().contiguous(), None, ACT_NONE, cache_split=False)
            dprev = torch.zeros((offs[depth + 1], d), dtype=torch.float32, device=self.device)
            for k in range(depth):
                dA, dS, dN = dagg[offs[k]:offs[k + 1]], dprev[offs[k]:offs[k + 1]], dprev[offs[k + 1]:offs[k + 2]]
                _lib.check(lib.b200_sage_aggregate_backward(
                    _lib.ptr(dA), 2 * d, None, offs[k + 1] - offs[k], _lib.ptr(dS), d, None, None, None, nn, d,
                    _lib.ptr(dN), d, st))
            G = dprev
        self._project_backward("item", c["ids64"], c["x"], G)

    # ---- step -------------------------------------------------------------------------------------------------------
    def _scores(self, Q, P, N):
        """compute_pair_scores (torchops/loss.py:67-90): pos [n], neg [n num_neg] with negatives of row i at
        i num_neg ..; the positives are repeated by the loss kernel for bpr / max-margin."""
        torch = self._torch
        n, f, d = int(Q.shape[0]), self.num_neg, self.d
        rows = torch.arange(n * f, dtype=torch.int64, device=self.device)
        pos = torch.empty(n, dtype=torch.float32, device=self.device)
        neg = torch.empty(n * f, dtype=torch.float32, device=self.device)
        st = _lib.current_stream()
        _lib.check(_lib.lib.b200_gather_dot(_lib.ptr(Q), d, _lib.ptr(rows), _lib.ptr(P), d, _lib.ptr(rows), n, d, 0,
                                            0.0, 0.0, _lib.ptr(pos), st))
        qrows = torch.div(rows, f, rounding_mode="floor")
        _lib.check(_lib.lib.b200_gather_dot(_lib.ptr(Q), d, _lib.ptr(qrows), _lib.ptr(N), d, _lib.ptr(rows), n * f, d,
                                            0, 0.0, 0.0, _lib.ptr(neg), st))
        return pos, neg

    def forward_backward(self, users=None, items=None, batch_size=None):
        """One batch's loss (device scalar) with every gradient buffer filled, no optimizer step.  u2i: ``users`` /
        ``items`` the batch's pairs; i2i: ``batch_size`` start items (or ``len(items)``).  The sampled batch is kept
        in ``last`` (device tensors).  None when an i2i batch yields no pair."""
        torch = self._torch
        dev, f = self.device, self.num_neg
        if self.paradigm == "u2i":
            users = torch.as_tensor(users).to(dev).to(torch.int64).reshape(-1)
            q_items = None
            pos_items = torch.as_tensor(items).to(dev).to(torch.int32).reshape(-1)
            if users.numel() != pos_items.numel():
                raise ValueError("users and items differ in length")
            neg_items = self.negatives(pos_items, users=users)
            roots = torch.cat([pos_items, neg_items])
        else:
            n_starts = int(batch_size if batch_size is not None else len(items))
            _, q_items, pos_items = self.walk_pairs(n_starts)
            if q_items.numel() == 0:
                self.last = None
                return None
            neg_items = self.negatives(pos_items, items=q_items)
            roots = torch.cat([q_items, pos_items, neg_items])
        n = int(pos_items.numel())
        ids = self.levels(roots)
        R, c = self.encode(ids)
        if self.paradigm == "u2i":
            xu, Q = self._project("user", users)
            P, N = R[:n], R[n:]
        else:
            Q, P, N = R[:n], R[n:2 * n], R[2 * n:]
        pos, neg = self._scores(Q, P, N)
        loss = torch.empty((), dtype=torch.float32, device=dev)
        dpos, dneg = torch.empty_like(pos), torch.empty_like(neg)
        mean = 1 if self.paradigm == "u2i" else 0
        _lib.check(_lib.lib.b200_pairwise_loss(_lib.ptr(pos), n, _lib.ptr(neg), n * f, self.kind, self.margin, 0.25,
                                               2.0, mean, _lib.ptr(loss), _lib.ptr(dpos), _lib.ptr(dneg),
                                               _lib.ptr(self._lws), self._lws.numel(), _lib.current_stream()))
        # d loss / d rows of the pair scores (elementwise; the reductions over the batch happen in the GEMMs above)
        dneg3 = dneg.view(n, f, 1)
        dQ = dpos[:, None] * P + (dneg3 * N.view(n, f, self.d)).sum(1)
        dR = torch.cat([dpos[:, None] * Q, (dneg3 * Q[:, None, :]).reshape(n * f, self.d)])
        if self.paradigm == "u2i":
            self._project_backward("user", users, xu, dQ)
        else:
            dR = torch.cat([dQ, dR])
        self.encode_backward(c, dR)
        self.last = dict(users=users, items=q_items, items_pos=pos_items, items_neg=neg_items, levels=ids, pos=pos,
                         neg=neg)
        return loss

    def adam_update(self):
        """torch.optim.Adam(lr, eps=epsilon, weight_decay=reg) over every parameter; zeroes the gradients."""
        lib, st = _lib.lib, _lib.current_stream()
        self.t += 1
        _, eps_hat = adam_step_constants(self.lr, self.epsilon, self.t)
        _lib.check(lib.b200_adam_begin_step(_lib.ptr(self._step_dev), self.lr, BETA1, BETA2, 1.0, 0,
                                            _lib.ptr(self._lr_t), st))
        for k, p in self.params.items():
            if k in self.frozen:
                continue
            if self.reg:
                _lib.check(lib.b200_axpy(_lib.ptr(self.grads[k]), _lib.ptr(p), self.reg, p.numel(), st))
            _lib.check(lib.b200_adam_dense_dev(_lib.ptr(p), _lib.ptr(self.m[k]), _lib.ptr(self.v[k]),
                                               _lib.ptr(self.grads[k]), p.numel(), _lib.ptr(self._lr_t), BETA1, BETA2,
                                               eps_hat, st))

    def step(self, users=None, items=None, batch_size=None):
        """One mini-batch: sampling, forward, backward and the Adam update.  Returns the device loss (None for an
        i2i batch without pairs, which leaves the parameters and the step count alone)."""
        loss = self.forward_backward(users, items, batch_size)
        if loss is not None:
            self.adam_update()
        return loss

    def fit(self, users, items, n_epochs=1, batch_size=256, shuffle=True):
        """Epochs over the training pairs in mini-batches of ``batch_size`` (shuffled per epoch as the reference's
        DataLoader does); an i2i batch takes its size from the pairs.  Returns the mean batch loss per epoch."""
        torch = self._torch
        users, items = np.asarray(users).reshape(-1), np.asarray(items).reshape(-1)
        rng = np.random.default_rng(self.seed)
        means = []
        for _ in range(int(n_epochs)):
            order = rng.permutation(users.size) if shuffle else np.arange(users.size)
            losses = []
            for b0 in range(0, users.size, int(batch_size)):
                sel = order[b0:b0 + int(batch_size)]
                loss = self.step(users[sel], items[sel]) if self.paradigm == "u2i" else self.step(batch_size=sel.size)
                if loss is not None:
                    losses.append(loss)
            means.append(float(torch.stack(losses).mean().item()) if losses else float("nan"))
        return means

    # ---- export -----------------------------------------------------------------------------------------------------
    def state_dict(self):
        """The parameters as ``GraphSageModel.state_dict()`` holds them: the reference's keys, shapes and column
        order, float32 CPU tensors."""
        out = {}
        for k, v in self.params.items():
            a = v.detach().cpu()
            if k in ("item_proj.weight", "user_proj.weight"):       # the side gather's [id, ...] back to [..., id]
                a = self._torch.cat([a[:, self.d:], a[:, :self.d]], dim=1)
            key = k if k in ("dense_embeds",) or "." in k else f"{k}.weight"
            out[key] = a.contiguous()
        return out

    def engine(self):
        """A :class:`GraphSage` inference engine on the current parameters."""
        return GraphSage(self.data_info, self.state_dict(), self.paradigm, self.num_layers, self.num_neighbors,
                         self.seed, self.device)


def _col_sum(X, out):
    """out += the column sums of X (b200_col_reduce, deterministic)."""
    _lib.check(_lib.lib.b200_col_reduce(_lib.ptr(X), X.stride(0), X.shape[0], X.shape[1], None, None, 0, _lib.ptr(out),
                                        _lib.current_stream()))
