"""Golden data for skip-gram training (Item2Vec / DeepWalk): the C1 corpus and the float64 oracle's fits on it.

    python tests/golden/gen_skipgram.py

C1 comes from the reference's own data pipeline (gensim / TensorFlow stubbed by ``oracle.ref_loader``):
``sample_movielens_rating.dat`` -> ``split_by_ratio_chrono(test_size=0.2)`` -> ``DatasetPure.build_trainset``.
Stored: the consumed lists in ``user_consumed`` iteration order (``c1_indptr``, ``c1_items``), the held-out pairs
(``eval_users``, ``eval_items``), and for each mode the float64 oracle fit's recall@10 / ndcg@10 and those of its
initial vectors (``{mode}_metrics``, ``{mode}_initial_metrics``).  Sizes: embed 16, window 5, seed 42; Item2Vec
2 epochs; DeepWalk n_walks = 2, walk_length = 10, 1 epoch.  A small case (``small_*``: the first 60 users, embed
8, one epoch of each mode) keeps the oracle's output tables (syn0 as its change from the initial vectors) so the CPU suite can reproduce them.  Data only: no
reference source.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle.ref_loader import load_reference, sample_data_path  # noqa: E402
import _skipgram_oracle as orc  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "skipgram.npz")
EPOCHS = {"item2vec": 2, "deepwalk": 1}
N_WALKS, WALK_LENGTH, SEED, WINDOW, EMBED = 2, 10, 42, 5, 16
SMALL_USERS, SMALL_EMBED = 60, 8


def c1():
    import pandas as pd

    load_reference()
    from libreco.data import DatasetPure, split_by_ratio_chrono

    data = pd.read_csv(sample_data_path(), sep="::", names=["user", "item", "label", "time"], engine="python")
    train, test = split_by_ratio_chrono(data, test_size=0.2)
    train_data, data_info = DatasetPure.build_trainset(train)
    eval_data = DatasetPure.build_evalset(test)
    n_u, n_i = data_info.n_users, data_info.n_items
    rows = list(data_info.user_consumed.values())
    indptr = np.zeros(len(rows) + 1, dtype=np.int64)
    np.cumsum([len(r) for r in rows], out=indptr[1:])
    items = np.concatenate(rows).astype(np.int32)
    keep = (eval_data.user_indices < n_u) & (eval_data.item_indices < n_i)
    assert list(data_info.user_consumed.keys()) == list(range(n_u))
    return indptr, items, n_u, n_i, eval_data.user_indices[keep], eval_data.item_indices[keep]


def oracle_fit(mode, indptr, items, n_items, d, epochs, n_walks=N_WALKS):
    """The float64 serial fit: (syn0, syn1neg, syn1, vocab_items, initial syn0)."""
    from librecommender_b200 import skipgram as sg

    hs = mode == "deepwalk"
    if hs:
        g_indptr, g_dst = sg.walk_graph(indptr, items, n_items)

        def corpus(p):
            w = orc.walks(g_indptr, g_dst, n_items, n_walks, WALK_LENGTH, SEED, p)
            return sg.corpus_csr(w)
        vocab_tokens = corpus(0)[1]
        corpora = [corpus(e + 1) for e in range(epochs)]
    else:
        vocab_tokens = items
        corpora = [(indptr, items)] * epochs
    vocab_items, counts = orc.vocab_first_appearance(vocab_tokens)
    init = sg.initial_vectors(vocab_items, n_items, d, SEED)
    thr = sg.keep_thresholds(vocab_items, counts, n_items)
    syn1 = np.zeros((max(len(vocab_items) - 1, 1), d)) if hs else None
    s0, s1n, s1 = orc.train(np.float64, corpora, init, np.zeros_like(init), syn1, vocab_items, counts, thr, hs,
                            WINDOW, SEED, vocab_tokens.size)
    return s0, s1n, s1, init


def main():
    indptr, items, n_u, n_i, ev_u, ev_i = c1()
    out = dict(c1_indptr=indptr, c1_items=items, c1_shape=np.array([n_u, n_i]),
               eval_users=ev_u.astype(np.int32), eval_items=ev_i.astype(np.int32))
    for mode, epochs in EPOCHS.items():
        out[f"{mode}_epochs"] = np.int64(epochs)
        s0, _, _, init = oracle_fit(mode, indptr, items, n_i, EMBED, epochs)
        for key, table in ((f"{mode}_metrics", s0), (f"{mode}_initial_metrics", init)):
            U = np.stack([table[items[indptr[u]:indptr[u + 1]]].mean(0) for u in range(n_u)])
            out[key] = np.array(orc.ranking_metrics(U, table, indptr, items, ev_u, ev_i))
        print(mode, "recall/ndcg@10 initial", out[f"{mode}_initial_metrics"], "fit", out[f"{mode}_metrics"],
              file=sys.stderr)
        assert out[f"{mode}_metrics"][0] > out[f"{mode}_initial_metrics"][0], mode
        sp, si = indptr[:SMALL_USERS + 1], items[:indptr[SMALL_USERS]]
        s0, s1n, s1, init = oracle_fit(mode, sp, si, n_i, SMALL_EMBED, 1, n_walks=1)
        out[f"small_{mode}_syn0_delta"], out[f"small_{mode}_syn1neg"] = s0 - init, s1n
        if s1 is not None:
            out[f"small_{mode}_syn1"] = s1
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), file=sys.stderr)


if __name__ == "__main__":
    main()
