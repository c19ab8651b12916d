"""Skip-gram training without a GPU: the host tables of ``librecommender_b200.skipgram`` against the restatement in
``tests/_skipgram_oracle.py``, the oracle against its golden fits, every validation error and C-ABI rejection, the
``Word2Vec`` subset and the ``gensim=True`` drop-in wiring."""
import ctypes
import os
import types

import numpy as np
import pytest
from scipy import stats

import _skipgram_oracle as orc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "skipgram.npz")


def _zipf_counts(g, V):
    return np.maximum(1, (1e4 / np.arange(1, V + 1) ** 1.1 * g.uniform(0.5, 1.5, V)).astype(np.int64))


@pytest.mark.parametrize("mode", ["item2vec", "deepwalk"])
def test_oracle_reproduces_the_small_golden_fit(mode):
    import importlib.util

    spec = importlib.util.spec_from_file_location(
        "gen_skipgram", os.path.join(os.path.dirname(GOLDEN), "gen_skipgram.py"))
    gen = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(gen)
    z = np.load(GOLDEN)
    ip, it = z["c1_indptr"], z["c1_items"]
    n_i = int(z["c1_shape"][1])
    sp, si = ip[:gen.SMALL_USERS + 1], it[:ip[gen.SMALL_USERS]]
    s0, s1n, s1, init = gen.oracle_fit(mode, sp, si, n_i, gen.SMALL_EMBED, 1, n_walks=1)
    np.testing.assert_allclose(s0 - init, z[f"small_{mode}_syn0_delta"], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(s1n, z[f"small_{mode}_syn1neg"], rtol=1e-9, atol=1e-12)
    if mode == "deepwalk":
        np.testing.assert_allclose(s1, z["small_deepwalk_syn1"], rtol=1e-9, atol=1e-12)
    for m in ("item2vec", "deepwalk"):
        assert z[f"{m}_metrics"][0] > z[f"{m}_initial_metrics"][0]


@pytest.mark.parametrize("V", [1, 2, 3, 17, 500])
def test_huffman_codes_are_optimal_prefix_codes(V):
    from librecommender_b200 import skipgram as sg

    counts = _zipf_counts(np.random.default_rng(V), V)
    ptr, points, codes = sg.huffman(counts)
    paths = orc.huffman_paths(counts)
    words = []
    for v in range(V):
        assert points[ptr[v]:ptr[v + 1]].tolist() == paths[v][0]
        assert codes[ptr[v]:ptr[v + 1]].tolist() == paths[v][1]
        words.append("".join(map(str, paths[v][1])))
    if V == 1:
        return
    assert all(0 <= p < V - 1 for p in points.tolist()) and np.all(points[ptr[:-1][np.diff(ptr) > 0]] == V - 2)
    for a in words:
        assert not any(b != a and b.startswith(a) for b in words)
    lens = np.array([len(w) for w in words])
    assert abs(np.sum(2.0 ** -lens) - 1.0) < 1e-12
    # optimal total length: sum over merges of the merged counts
    import heapq

    h = [int(c) for c in counts]
    heapq.heapify(h)
    cost = 0
    while len(h) > 1:
        s = heapq.heappop(h) + heapq.heappop(h)
        cost += s
        heapq.heappush(h, s)
    assert int((lens * counts).sum()) == cost


def test_negative_table_matches_the_restatement_and_its_draws_follow_c_075():
    from librecommender_b200 import skipgram as sg

    g = np.random.default_rng(1)
    counts = _zipf_counts(g, 40)
    cum = sg.negative_table(counts)
    assert np.array_equal(cum.astype(np.int64), orc.cum_table(counts))
    guide, buckets = sg.negative_guide(cum, 64)
    r = g.integers(0, int(cum[-1]), size=2000)
    want = np.searchsorted(cum.astype(np.int64), r, side="left")
    step = -(-int(cum[-1]) // buckets)
    for x, w in zip(r.tolist(), want.tolist()):
        b = x // step
        assert guide[b] <= w <= guide[b + 1]
    items = np.arange(40, dtype=np.int32)
    negs = orc.negative_draws(7, np.arange(-5, 6), 5, 5, cum, items, 42, 1)
    draws = np.concatenate([orc.negative_draws(q, np.arange(-5, 6), 5, 5, cum, items, 42, 1).ravel()
                            for q in range(400)])
    assert negs.shape == (11, 5)
    p = counts ** 0.75 / np.sum(counts ** 0.75)
    obs = np.bincount(draws, minlength=40)
    assert stats.chisquare(obs, p * obs.sum()).pvalue > 1e-3


def test_keep_rate_matches_the_probability():
    from librecommender_b200 import skipgram as sg

    counts = np.array([20000, 5000, 800, 100, 3], dtype=np.int64)
    items = np.arange(5, dtype=np.int32)
    thr = sg.keep_thresholds(items, counts, 5)
    tokens = np.repeat(items, counts)
    keep = orc.keep_decisions(tokens, thr, 42, 1)
    p = orc.keep_probability(counts)
    for w in range(5):
        k = keep[tokens == w]
        assert abs(k.mean() - p[w]) <= 5 * np.sqrt(p[w] * (1 - p[w]) / k.size) + 1e-12
    assert np.all(keep[tokens == 4]) and p[4] == 1.0


def test_walks_follow_edge_multiplicities_and_stop():
    from librecommender_b200 import skipgram as sg

    indptr = np.array([0, 4, 7, 9], dtype=np.int64)
    items = np.array([0, 1, 0, 1, 0, 2, 0, 3, 4], dtype=np.int32)      # 0->1 x2, 1->0 x1, 0->2, 2->0, 3->4
    g_indptr, g_dst = sg.walk_graph(indptr, items, 6)
    assert g_indptr.tolist() == [0, 3, 4, 5, 6, 6, 6] and g_dst.tolist() == [1, 1, 2, 0, 0, 4]
    ws = orc.walks(g_indptr, g_dst, 6, 300, 6, 42, 1)
    assert all(w[0] == k % 6 for k, w in enumerate(ws))
    trans = np.zeros((6, 6))
    for w in ws:
        assert len(w) == 6 or int(g_indptr[w[-1] + 1] - g_indptr[w[-1]]) == 0
        for a, b in zip(w[:-1], w[1:]):
            trans[a, b] += 1
    assert trans[0, 1] > 0 and trans[0, 2] > 0 and trans[0].sum() > 0
    assert stats.chisquare(trans[0, [1, 2]], trans[0, [1, 2]].sum() * np.array([2 / 3, 1 / 3])).pvalue > 1e-3
    assert all(len(w) == 1 for w in ws[4::6]) and all(len(w) == 2 and w[1] == 4 for w in ws[3::6])


def test_vocabulary_and_initial_vectors():
    from librecommender_b200 import skipgram as sg

    tokens = np.array([5, 3, 5, 9, 3, 3, 0], dtype=np.int32)
    items, counts = sg.vocabulary(tokens)
    assert items.tolist() == [5, 3, 9, 0] and counts.tolist() == [2, 3, 1, 1]
    oi, oc = orc.vocab_first_appearance(tokens)
    assert np.array_equal(items, oi) and np.array_equal(counts, oc)
    v = sg.initial_vectors(items, 10, 4, 42)
    want = (np.random.default_rng(42).random((4, 4), dtype=np.float32) * 2 - 1) / 4
    assert np.allclose(v[items], want, atol=1e-8) and not v[[1, 2, 4]].any()
    ip, tk = sg.truncate_csr(np.array([0, 12000, 12003]), np.arange(12003) % 7)
    assert ip.tolist() == [0, 10000, 10003] and tk[10000:].tolist() == [12000 % 7, 12001 % 7, 12002 % 7]


def _lib():
    from librecommender_b200 import _lib

    return _lib


def test_cabi_rejections_return_minus_two():
    L = _lib()
    lib, P = L.lib, ctypes.c_void_p
    nz = P(16)
    ep = lambda d=8, w=5, neg=5, hs=0, p=nz, syn1=None: lib.b200_skipgram_epoch(  # noqa: E731
        p, 1, nz, nz, nz, 4, 10, nz, nz, syn1, d, hs, None, None, None, nz, nz, 5, 100, nz, 4, w, neg, 0.025, 1e-4,
        0.0, 4.0, 1, 1, None, None, 0, None)
    for rc in (ep(d=0), ep(d=129), ep(w=0), ep(w=4097), ep(neg=0), ep(neg=17), ep(hs=2), ep(p=None), ep(hs=1)):
        assert rc == -2
    assert lib.b200_skipgram_subsample(None, nz, 1, 10, nz, 1, 1, nz, nz, nz, None, None) == -2
    assert lib.b200_skipgram_subsample(nz, nz, -1, 10, nz, 1, 1, nz, nz, nz, None, None) == -2
    assert lib.b200_item_walks(nz, nz, 10, 2, 0, 1, 0, nz, None, None, None) == -2
    assert lib.b200_item_walks(nz, nz, 10, 2, 10001, 1, 0, nz, None, None, None) == -2
    assert lib.b200_item_walks(nz, nz, 10, 2, 5, 1, 0, nz, nz, nz, None) == -2          # both outputs
    assert lib.b200_item_walks(nz, nz, 10, 2, 5, 1, 0, None, None, nz, None) == -2      # tokens without indptr
    assert lib.b200_item_walks(None, nz, 10, 2, 5, 1, 0, nz, None, None, None) == -2
    assert lib.b200_skipgram_default_inflight(0) == 0 and lib.b200_skipgram_default_inflight(129) == 0
    assert "b200_item_walks" in L.lib.b200_last_error().decode()
    assert lib.b200_version() == 100


def test_trainer_validation_errors():
    from librecommender_b200 import skipgram as sg

    ok = (np.array([0, 2]), np.array([0, 1]))
    for kw, msg in ((dict(mode="cbow"), "mode"), (dict(embed_size=0), "embed_size"), (dict(embed_size=129), "embed"),
                    (dict(window=0), "window"), (dict(n_epochs=-1), ">= 0"),
                    (dict(mode="deepwalk", n_walks=0), "n_walks")):
        with pytest.raises(ValueError, match=msg):
            sg.SkipGramTrainer(ok, 2, device="cpu", **kw)
    with pytest.raises(ValueError, match="outside"):
        sg.SkipGramTrainer((np.array([0, 2]), np.array([0, 5])), 2, device="cpu")
    with pytest.raises(ValueError, match="CSR"):
        sg.SkipGramTrainer((np.array([0, 3]), np.array([0, 1])), 2, device="cpu")
    with pytest.raises(ValueError, match="n_items"):
        sg.SkipGramTrainer(ok, 0, device="cpu")


def test_word2vec_subset_rejects_what_it_does_not_implement():
    from librecommender_b200.skipgram import Word2Vec

    kw = dict(vector_size=8, window=5, sg=1, hs=0, negative=5, seed=1, min_count=1, workers=4, sorted_vocab=0)
    w = Word2Vec(**kw)
    with pytest.raises(TypeError, match="unsupported corpus"):
        w.build_vocab([["1", "2"], ["2", "3"]])
    with pytest.raises(NotImplementedError, match="update=True"):
        w.build_vocab(types.SimpleNamespace(item_seqs=[[1, 2]]), update=True)
    with pytest.raises(RuntimeError, match="build_vocab"):
        w.train(None, total_examples=1, epochs=1)
    for bad in (dict(sg=0), dict(min_count=5), dict(sorted_vocab=1), dict(negative=0), dict(cbow_mean=1)):
        with pytest.raises(NotImplementedError):
            Word2Vec(**{**kw, **bad})


def test_dropin_patches_and_restores_the_gensim_names():
    from oracle.ref_loader import load_reference, reference_available

    if not reference_available():
        pytest.skip("reference tree not present")
    libreco = load_reference()
    import importlib

    from librecommender_b200 import dropin, skipgram

    mods = [importlib.import_module(f"libreco.{m}") for m in
            ("bases.gensim_base", "algorithms.item2vec", "algorithms.deepwalk")]
    before = [m.Word2Vec for m in mods]
    gb = mods[0].GensimBase
    set_before = gb.set_embeddings
    dropin.install(libreco, gensim=True)
    try:
        assert all(m.Word2Vec is skipgram.Word2Vec for m in mods)
        assert gb.set_embeddings is skipgram.set_embeddings
    finally:
        dropin.uninstall()
    assert [m.Word2Vec for m in mods] == before and gb.set_embeddings is set_before
    dropin.install(libreco)
    try:
        assert [m.Word2Vec for m in mods] == before
    finally:
        dropin.uninstall()
