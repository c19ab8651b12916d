"""Restatement of GraphSage / PinSage inference (``csrc/sage.cu``, ``librecommender_b200.sage``; DESIGN.md §4,
"GraphSage / PinSage inference") for checking the kernels.

* The sampling rules of ``libreco/sampling/random_walks.py`` written once, over a draw provider: :class:`KeyedDraws`
  gives the library's Philox4x32-10 streams keyed by (seed, root, path, level, draw), :class:`PythonDraws` the
  reference's ``random`` calls in the reference's order, so the same rule code is checked against the reference
  functions and then gives the kernels' expected output bit for bit.
* :func:`encode`: the float64 item encoder of ``graphsage_module.py`` / ``pinsage_module.py`` over a message in the
  reference's form (per-level ids, offsets, weights); :func:`raw_features` is ``get_raw_features``.
"""
import random
from collections import Counter

import numpy as np

from oracle.sampling import philox4x32_10

TAG_SAGE, TAG_PIN_STEP, TAG_PIN_STOP = 0, 1, 2
ATTEMPTS = 12


def csr(consumed, n):
    """(indptr int64, idx int32) of a dict of lists, order and multiplicity kept."""
    lens = np.array([len(consumed.get(k, ())) for k in range(n)], dtype=np.int64)
    indptr = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=indptr[1:])
    idx = np.fromiter((x for k in range(n) for x in consumed.get(k, ())), dtype=np.int64, count=int(indptr[-1]))
    return indptr, idx.astype(np.int32)


def cont_threshold(termination_prob):
    """Step s > 0 is taken when the termination word is >= this: random.random() >= p with u = word / 2^32."""
    import math

    return min(1 << 32, max(0, math.ceil(float(termination_prob) * 2.0 ** 32)))


def bounded(hi, lo, n):
    """philox.cuh ``bounded``: high 64 bits of ((hi << 32) | lo) * n, exact for n < 2^31."""
    hi, lo, n = (np.asarray(x, dtype=np.uint64) for x in (hi, lo, n))
    return ((hi * n + ((lo * n) >> np.uint64(32))) >> np.uint64(32)).astype(np.int64)


class Graph:
    def __init__(self, user_consumed, item_consumed, n_users, n_items):
        self.item_ptr, self.item_users = csr(item_consumed, n_items)
        self.user_ptr, self.user_items = csr(user_consumed, n_users)
        self.user_consumed, self.item_consumed = user_consumed, item_consumed

    def one_walk(self, v, r):
        """Vectorised one-walk from items ``v`` with the four Philox words ``r``."""
        v = np.asarray(v, dtype=np.int64)
        i0 = self.item_ptr[v]
        u = self.item_users[i0 + bounded(r[0], r[1], self.item_ptr[v + 1] - i0)].astype(np.int64)
        u0 = self.user_ptr[u]
        return self.user_items[u0 + bounded(r[2], r[3], self.user_ptr[u + 1] - u0)].astype(np.int64)

    def has_no_neighbor(self, v):
        users = self.item_users[self.item_ptr[v]:self.item_ptr[v + 1]]
        return bool(np.all(self.user_ptr[users + 1] - self.user_ptr[users] <= 1))


def keyed(root, path, level, idx, tag, seed):
    c2 = (np.asarray(level, dtype=np.uint64) << np.uint64(24)) | np.asarray(idx, dtype=np.uint64)
    return philox4x32_10(np.asarray(root, dtype=np.uint32), np.asarray(path, dtype=np.uint32), c2.astype(np.uint32),
                         np.uint32(tag), seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)


class KeyedDraws:
    """The library's streams for the nodes of one level (roots [n_roots], per_root nodes each)."""

    def __init__(self, graph, seed, roots, nodes, per_root, level, nn, walks=None):
        self.g, self.seed, self.level, self.nn = graph, int(seed), int(level), int(nn)
        self.nodes = np.asarray(nodes, dtype=np.int64)
        r = np.arange(self.nodes.size)
        self.root = np.asarray(roots, dtype=np.int64)[r // per_root]
        self.path = r % per_root
        if walks is None:          # GraphSage: every attempt of every slot, [n, nn, 12]
            j = np.arange(nn)[None, :, None]
            a = np.arange(ATTEMPTS)[None, None, :]
            shape = (self.nodes.size, nn, ATTEMPTS)
            words = keyed(np.broadcast_to(self.root[:, None, None], shape),
                          np.broadcast_to(self.path[:, None, None] * nn + j, shape), self.level,
                          np.broadcast_to(a, shape), TAG_SAGE, self.seed)
            v = np.broadcast_to(np.maximum(self.nodes, 0)[:, None, None], shape)
            self.cand = self.g.one_walk(v, words)
        else:                      # PinSage: termination words and walks, [n, num_walks * walk_len]
            num_walks, walk_len, self.thr = walks
            V = num_walks * walk_len
            shape = (self.nodes.size, V)
            idx = np.broadcast_to(np.arange(V)[None, :], shape)
            root = np.broadcast_to(self.root[:, None], shape)
            path = np.broadcast_to(self.path[:, None], shape)
            self.stop_word = keyed(root, path, self.level, idx, TAG_PIN_STOP, self.seed)[0]
            self.step_words = keyed(root, path, self.level, idx, TAG_PIN_STEP, self.seed)
            self.walk_len = walk_len

    def for_node(self, r):
        keyed_self = self

        class One:
            def attempt(self, j, a):
                return int(keyed_self.cand[r, j, a])

            def cont(self, w, s):
                return int(keyed_self.stop_word[r, w * keyed_self.walk_len + s]) >= keyed_self.thr

            def step(self, w, s, cur):
                q = w * keyed_self.walk_len + s
                return int(keyed_self.g.one_walk(cur, [x[r, q] for x in keyed_self.step_words]))

        return One()


class PythonDraws:
    """The reference's ``random`` calls, in the order the reference makes them."""

    def __init__(self, graph, termination_prob=0.5):
        self.g, self.p = graph, termination_prob

    def _walk(self, v):
        user = random.choice(self.g.item_consumed[v])
        return random.choice(self.g.user_consumed[user])

    def for_node(self, v):
        outer = self

        class One:
            def attempt(self, j, a):
                return outer._walk(v)

            def cont(self, w, s):
                return random.random() >= outer.p

            def step(self, w, s, cur):
                return outer._walk(cur)

        return One()


def sage_node(v, nn, d):
    """bipartite_neighbors' rules for one node over the draw provider ``d`` (attempt(slot, a))."""
    taken = []
    for j in range(nn):
        n = d.attempt(j, 0)
        if n == v or n in taken:
            ok = False
            for a in range(1, 6):
                n = d.attempt(j, a)
                if n != v and n not in taken:
                    ok = True
                    break
            if not ok:
                for a in range(6, 11):
                    n = d.attempt(j, a)
                    if n != v:
                        ok = True
                        break
            if not ok:
                n = d.attempt(j, 11)
        taken.append(n)
    return taken


def pinsage_node(g, v, nn, num_walks, walk_len, d):
    """bipartite_neighbors_with_weights' rules for one node (items_pos None): (ids, float64 weights)."""
    if g.has_no_neighbor(v):
        return [v], [1.0]
    visits = []
    for w in range(num_walks):
        walk = []
        for s in range(walk_len):
            if not walk:
                walk.append(d.step(w, s, v))
            elif d.cont(w, s):
                walk.append(d.step(w, s, walk[-1]))
            else:
                break
        visits.extend(walk)
    kept = [x for x in visits if x != v]
    if not kept:
        return [v], [1.0]
    if len(kept) == 1:
        return kept, [1.0]
    top = Counter(kept).most_common(nn)
    total = sum(c for _, c in top)
    return [n for n, _ in top], [c / total for _, c in top]


def sample_level(kind, graph, seed, roots, nodes, per_root, level, nn, num_walks=0, walk_len=0, thr=0):
    """The kernels' padded output for one level: ids int32 [n, nn] (and for PinSage float32 weights, int32 lens)."""
    nodes = np.asarray(nodes, dtype=np.int64)
    walks = None if kind == "graphsage" else (num_walks, walk_len, thr)
    draws = KeyedDraws(graph, seed, roots, nodes, per_root, level, nn, walks)
    ids = np.full((nodes.size, nn), -1, dtype=np.int32)
    if kind == "graphsage":
        for r, v in enumerate(nodes):
            if v >= 0:
                ids[r] = sage_node(int(v), nn, draws.for_node(r))
        return ids
    wts = np.zeros((nodes.size, nn), dtype=np.float32)
    lens = np.zeros(nodes.size, dtype=np.int32)
    for r, v in enumerate(nodes):
        if v < 0:
            continue
        n, w = pinsage_node(graph, int(v), nn, num_walks, walk_len, draws.for_node(r))
        ids[r, :len(n)], wts[r, :len(n)], lens[r] = n, np.asarray(w, dtype=np.float32), len(n)
    return ids, wts, lens


def sample(kind, graph, seed, items, num_layers, nn, num_walks=0, walk_len=0, termination_prob=0.5):
    """Every level for the roots ``items``: a list of per-level outputs of :func:`sample_level`."""
    thr = cont_threshold(termination_prob)
    items = np.asarray(items, dtype=np.int64)
    nodes, per_root, out = items, 1, []
    for level in range(num_layers):
        res = sample_level(kind, graph, seed, items, nodes, per_root, level, nn, num_walks, walk_len, thr)
        out.append(res)
        nodes = (res if kind == "graphsage" else res[0]).reshape(-1).astype(np.int64)
        per_root *= nn
    return out


def padded_to_message(kind, items, levels):
    """The padded levels in the reference's message form: per level the neighbour ids of the real nodes, flattened,
    their offsets (and weights).  A padded slot (id -1) is no node of the reference's message."""
    nbs, offs, wts = [], [], []
    real = np.ones(len(items), dtype=bool)
    for res in levels:
        ids, w, lens = (res, None, np.full(res.shape[0], res.shape[1], np.int32)) if kind == "graphsage" else res
        keep = np.arange(ids.shape[1])[None, :] < lens[:, None]
        nbs.append(ids[keep].astype(np.int64))
        if w is not None:
            wts.append(w[keep])
        offs.append(np.concatenate([[0], np.cumsum(lens[real])[:-1]]).astype(np.int64))
        real = ids.reshape(-1) >= 0
    return nbs, offs, (None if kind == "graphsage" else wts)


# ---- float64 encoder ------------------------------------------------------------------------------------------------
def raw_features(sd, ids, sparse_unique, dense_unique, dense_cols, prefix="item"):
    """get_raw_features (graphsage_module.py:54-78) in float64, before the projection."""
    ids = np.asarray(ids, dtype=np.int64)
    parts = []
    if sparse_unique is not None:
        parts.append(sd["sparse_embeds.weight"][np.asarray(sparse_unique)[ids]].reshape(ids.size, -1))
    if dense_unique is not None:
        vals = np.asarray(dense_unique, dtype=np.float64)[ids]
        parts.append((sd["dense_embeds"][list(dense_cols)][None, :, :] * vals[:, :, None]).reshape(ids.size, -1))
    parts.append(sd[f"{prefix}_embeds.weight"][ids])
    return np.concatenate(parts, axis=1)


def project(sd, ids, feats, prefix="item"):
    x = raw_features(sd, ids, *feats, prefix=prefix)
    return x @ sd[f"{prefix}_proj.weight"].T + sd[f"{prefix}_proj.bias"]


def _dense(sd, name, x, bias=True):
    y = x @ sd[f"{name}.weight"].T
    return y + sd[f"{name}.bias"] if bias else y


def _bag(rows, offsets, weights=None):
    n = len(offsets)
    ends = list(offsets[1:]) + [rows.shape[0]]
    out = np.zeros((n, rows.shape[1]))
    for r in range(n):
        seg = rows[offsets[r]:ends[r]]
        if seg.shape[0] == 0:
            continue
        out[r] = seg.mean(axis=0) if weights is None else (seg * weights[offsets[r]:ends[r], None]).sum(axis=0)
    return out


def encode(kind, sd, items, nbs, offsets, weights, num_layers, feats):
    """The item encoder's forward in eval mode, float64, on a message in the reference's form."""
    sd = {k: np.asarray(v, dtype=np.float64) for k, v in sd.items()}
    hidden = [project(sd, items, feats)] + [project(sd, n, feats) for n in nbs]
    for layer in range(num_layers):
        nxt = []
        for k in range(num_layers - layer):
            if kind == "graphsage":
                h = np.concatenate([hidden[k], _bag(hidden[k + 1], offsets[k])], axis=1)
                h = _dense(sd, f"w_linears.{layer}", h)
                nxt.append(h if layer == num_layers - 1 else np.maximum(h, 0))
            else:
                q = np.maximum(_dense(sd, f"q_linears.{layer}", hidden[k + 1]), 0)
                z = np.concatenate([hidden[k], _bag(q, offsets[k], np.asarray(weights[k], np.float64))], axis=1)
                z = np.maximum(_dense(sd, f"w_linears.{layer}", z), 0)
                norm = np.linalg.norm(z, axis=1, keepdims=True)
                nxt.append(z / np.where(norm == 0, 1.0, norm))
        hidden = nxt
    out = hidden[0]
    if kind == "pinsage":
        out = _dense(sd, "G2", np.maximum(_dense(sd, "G1", out), 0), bias=False)
    return out


def user_rows(kind, sd, users, feats):
    """user_repr (graphsage_module.py:51-52, pinsage_module.py:28-32) in float64."""
    sd = {k: np.asarray(v, dtype=np.float64) for k, v in sd.items()}
    x = project(sd, users, feats, prefix="user")
    if kind == "pinsage":
        x = _dense(sd, "U2", np.maximum(_dense(sd, "U1", x), 0), bias=False)
    return x
