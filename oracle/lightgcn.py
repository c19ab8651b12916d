"""Numpy/scipy restatement of LightGCN propagation.  TEST INFRASTRUCTURE ONLY.

Follows ``libreco/algorithms/torch_modules/lightgcn_module.py`` (reference @ 7463d9d):
* ``_build_laplacian_matrix`` (:36-61): R binary from ``user_consumed`` (duplicates collapse to
  1.0), A = [[0, R], [R^T, 0]], L = D^-1/2 A D^-1/2 in float32, isolated nodes -> 0.
* ``embedding_propagation`` (:66-88): E^{l+1} = L E^l, output = mean over the n_layers+1 terms,
  split into users / items.

* ``propagate64`` / ``propagate64_grad``: the same layer mean in float64 for any value array
  (including the non-symmetric values edge dropout leaves, :90-96), and its gradient
  ``mean_l (L^T)^l G``.

Pinned against the unmodified reference module run in the build container
(``tests/golden/gen_lightgcn.py`` -> ``tests/golden/lightgcn_*.npz``).
"""
from __future__ import annotations

import numpy as np
from scipy import sparse as sp


def build_laplacian(n_users, n_items, user_consumed):
    rows, cols = [], []
    for u in range(n_users):
        items = np.unique(np.asarray(user_consumed.get(u, []), dtype=np.int64))
        rows.append(np.full(len(items), u, dtype=np.int64))
        cols.append(items)
    rows = np.concatenate(rows) if rows else np.zeros(0, np.int64)
    cols = np.concatenate(cols) if cols else np.zeros(0, np.int64)
    n = n_users + n_items
    ones = np.ones(len(rows), dtype=np.float32)
    A = sp.coo_matrix((np.concatenate([ones, ones]),
                       (np.concatenate([rows, cols + n_users]), np.concatenate([cols + n_users, rows]))),
                      shape=(n, n), dtype=np.float32).tocsr()
    deg = np.asarray(A.sum(axis=1)).reshape(-1).astype(np.float32)
    with np.errstate(divide="ignore"):
        dinv = np.power(deg, np.float32(-0.5)).astype(np.float32)
    dinv[np.isinf(dinv)] = 0.0
    D = sp.diags(dinv)
    return D.dot(A).dot(D).tocsr().astype(np.float32)


def propagate(L, user_embeds, item_embeds, n_layers):
    E = np.concatenate([user_embeds, item_embeds], axis=0).astype(np.float32)
    layers = [E]
    for _ in range(n_layers):
        layers.append((L @ layers[-1]).astype(np.float32))
    out = np.mean(np.stack(layers, axis=1), axis=1, dtype=np.float32)
    return out[: len(user_embeds)], out[len(user_embeds):]


def propagate64(L, E0, n_layers):
    """mean over l = 0..n_layers of L^l E0 in float64; ``L`` is any scipy sparse matrix."""
    L = sp.csr_matrix(L, dtype=np.float64)
    cur = np.asarray(E0, dtype=np.float64)
    total = cur.copy()
    for _ in range(n_layers):
        cur = L @ cur
        total += cur
    return total / (n_layers + 1)


def propagate64_grad(L, G, n_layers):
    """Gradient of ``(propagate64(L, E0, n_layers) * G).sum()`` w.r.t. E0: mean_l (L^T)^l G."""
    return propagate64(sp.csr_matrix(L, dtype=np.float64).T, G, n_layers)
