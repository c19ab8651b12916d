"""Golden vectors for SIM's collate-time dual (long + short) sequences from the UNMODIFIED reference
(libreco/batch/sequence.py: get_dual_seqs, called from batch/collators.py:114-116).

    python tests/golden/gen_dual_sequences.py
"""
import os
import random
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.ref_loader import load_reference  # noqa: E402

load_reference()
from libreco.batch.sequence import get_dual_seqs  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
SHAPES = ((20, 5), (100, 10), (8, 8))        # (long_max_len, short_max_len)

if __name__ == "__main__":
    g = np.random.default_rng(91)
    n_users, n_items = 80, 300
    consumed = {}
    for u in range(n_users):
        ln = int(g.integers(1, 140))                      # every length class of every shape; get_dual_seqs needs >= 1
        consumed[u] = g.integers(0, n_items, ln).tolist()  # repeats allowed: the first occurrence is the position
    n = 900
    users = g.integers(0, n_users, n)
    items = np.array([consumed[u][int(g.integers(0, len(consumed[u])))] if g.random() < 0.6
                      else int(g.integers(0, n_items)) for u in users])
    sets = {u: set(v) for u, v in consumed.items()}
    data = {"users": users, "items": items}
    for L, S in SHAPES:
        random.seed(4321)
        ls, ll, ss, sl = get_dual_seqs(users, items, consumed, n_items, L, S, sets)
        data[f"long_{L}_{S}"], data[f"long_lens_{L}_{S}"] = ls, ll
        data[f"short_{L}_{S}"], data[f"short_lens_{L}_{S}"] = ss, sl
    indptr = np.zeros(n_users + 1, dtype=np.int64)
    for u in range(n_users):
        indptr[u + 1] = indptr[u] + len(consumed[u])
    data["indptr"] = indptr
    data["idx"] = np.concatenate([np.asarray(consumed[u], dtype=np.int32) for u in range(n_users)])
    data["n_items"] = n_items
    data["shapes"] = np.asarray(SHAPES, dtype=np.int64)
    np.savez_compressed(os.path.join(OUT, "dual_sequences.npz"), **data)
    print("wrote dual_sequences.npz", {k: np.shape(v) for k, v in data.items()})
