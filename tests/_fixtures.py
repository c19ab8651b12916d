"""Loaders of committed golden fixtures shared by several test modules."""
import os

import numpy as np

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
GOLD = os.path.join(GOLDEN, "movielens_multi_sparse.npz")


def load_multi_sparse_spec():
    g = np.load(GOLD)
    spec = dict(
        n_users=int(g["n_users"]), n_items=int(g["n_items"]),
        user_sparse_col_index=g["user_sparse_col_index"].tolist(), item_sparse_col_index=g["item_sparse_col_index"].tolist(),
        user_dense_col_index=g["user_dense_col_index"].tolist(), item_dense_col_index=g["item_dense_col_index"].tolist(),
        user_sparse_unique=g["user_sparse_unique"], item_sparse_unique=g["item_sparse_unique"],
        user_dense_unique=g["user_dense_unique"].astype(np.float32), item_dense_unique=None,
        sparse_vocab=int(g["sparse_vocab"]),
        multi_sparse_combine_info=dict(field_offset=g["field_offset"].tolist(), field_len=g["field_len"].tolist(),
                                       feat_oov=g["feat_oov"]))
    spec["n_sparse"] = len(spec["user_sparse_col_index"]) + len(spec["item_sparse_col_index"])
    spec["n_dense"] = len(spec["user_dense_col_index"]) + len(spec["item_dense_col_index"])
    return g, spec


# seeded inputs of the randomized comparisons with the reference; golden/live_reference.npz holds the
# reference's answers for them (golden/gen_live_reference.py)

def rank_cases():
    rng = np.random.default_rng(5)
    for _ in range(20):
        B, N = int(rng.integers(1, 6)), int(rng.integers(5, 400))
        K = int(rng.integers(1, N + 1))
        preds = rng.standard_normal((B, N)).astype(np.float32)
        consumed = {u: rng.choice(N, size=int(rng.integers(0, N)), replace=False).tolist() for u in range(B)}
        consumed = {u: v for u, v in consumed.items() if v}
        yield list(range(B)), preds, K, N, consumed


def sampling_cases():
    gen = np.random.default_rng(9)
    for trial in range(5):
        n_items = int(gen.integers(20, 3000))
        pos = gen.integers(0, n_items, size=int(gen.integers(1, 500)))
        num_neg = int(gen.integers(1, 6))
        yield trial, n_items, pos, num_neg
