"""Float64 numpy restatement of NGCF propagation.  TEST INFRASTRUCTURE ONLY.

Follows ``libreco/algorithms/torch_modules/ngcf_module.py`` (reference @ 7463d9d):
* ``_build_laplacian_matrix`` (:61-85): R binary from ``user_consumed`` (duplicates collapse to
  1.0), A = [[0, R], [R^T, 0]], L = D^-1 (A + I) with D the row sums of A + I.
* ``embedding_propagation`` (:87-124) without dropout: per layer k
  ``side = L E``, ``self = side W_self_k + b_self_k``, ``pair = (side * E) W_pair_k + b_pair_k``,
  ``E' = normalize(leaky_relu(self + pair, 0.2))`` with F.normalize's ``max(||m||_2, 1e-12)``;
  the output is the concatenation of E^0 .. E^K, split into users / items.

Pinned against the unmodified reference module run in the build container
(``tests/golden/gen_ngcf.py`` -> ``tests/golden/ngcf_*.npz``).
"""
from __future__ import annotations

import numpy as np
from scipy import sparse as sp


def build_laplacian(n_users, n_items, user_consumed):
    """D^-1 (A + I) in float64 (scipy CSR)."""
    rows, cols = [], []
    for u in range(n_users):
        items = np.unique(np.asarray(user_consumed.get(u, []), dtype=np.int64))
        rows.append(np.full(len(items), u, dtype=np.int64))
        cols.append(items)
    rows = np.concatenate(rows) if rows else np.zeros(0, np.int64)
    cols = np.concatenate(cols) if cols else np.zeros(0, np.int64)
    n = n_users + n_items
    ones = np.ones(len(rows), dtype=np.float64)
    A = sp.coo_matrix((np.concatenate([ones, ones]),
                       (np.concatenate([rows, cols + n_users]), np.concatenate([cols + n_users, rows]))),
                      shape=(n, n), dtype=np.float64).tocsr()
    A = A + sp.eye(n, dtype=np.float64, format="csr")
    deg = np.asarray(A.sum(axis=1)).reshape(-1)
    return (sp.diags(1.0 / deg) @ A).tocsr()


def combine64(self_part, pair_part, negative_slope=0.2, eps=1e-12):
    """normalize(leaky_relu(self + pair)) in float64 (ngcf_module.py:116-121)."""
    m = np.asarray(self_part, np.float64) + np.asarray(pair_part, np.float64)
    m = np.where(m > 0, m, negative_slope * m)
    norm = np.sqrt((m * m).sum(axis=1, keepdims=True))
    return m / np.maximum(norm, eps)


def propagate64(L, user_embed, item_embed, weights):
    """(user_out, item_out) float64; ``weights`` holds ``W_self_k`` [d_in, d_out], ``b_self_k``,
    ``W_pair_k``, ``b_pair_k`` (the reference's ParameterDict names)."""
    L = sp.csr_matrix(L, dtype=np.float64)
    E = np.concatenate([user_embed, item_embed]).astype(np.float64)
    outs = [E]
    k = 0
    while f"W_self_{k}" in weights:
        w = {name: np.asarray(weights[f"{name}_{k}"], np.float64) for name in ("W_self", "b_self", "W_pair", "b_pair")}
        side = L @ E
        self_part = side @ w["W_self"] + w["b_self"].reshape(1, -1)
        pair_part = (side * E) @ w["W_pair"] + w["b_pair"].reshape(1, -1)
        E = combine64(self_part, pair_part)
        outs.append(E)
        k += 1
    full = np.concatenate(outs, axis=1)
    n_users = len(user_embed)
    return full[:n_users], full[n_users:]
