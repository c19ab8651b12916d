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
"""
from __future__ import annotations

import math

import numpy as np

from . import _lib
from .consumed import ConsumedCSR
from .feat_models import ACT_NONE, ACT_RELU, FeatSpec, _dev, _spec_get, feat_forward, linear, tables_struct

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
