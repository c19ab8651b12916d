"""Skip-gram training on the GPU (``csrc/skipgram.cu``, ``librecommender_b200.skipgram``) against the serial
restatement (``tests/_skipgram_oracle.py``).

Tolerance: in the serial schedule, per row the device's max-norm distance to the float64 oracle may be at most 4x the
float32 oracle's own distance plus a floor of 2e-6 (1 + |x|) — the BPR bound, with the float32 oracle in place of
the Cython build."""
import os

import numpy as np
import pytest

import _skipgram_oracle as orc

pytestmark = pytest.mark.gpu

FLOOR = 2e-6
QUALITY_MARGIN = 0.15
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "skipgram.npz")


def _torch():
    import torch

    return torch


def _corpus(g, n_sent, n_items, max_len, zipf=True):
    lens = g.integers(0, max_len + 1, size=n_sent)
    lens[:3] = (0, 1, max_len)
    p = 1.0 / np.arange(1, n_items + 1) if zipf else np.ones(n_items)
    p /= p.sum()
    seqs = [g.choice(n_items, size=int(k), p=p) for k in lens]
    indptr = np.zeros(n_sent + 1, dtype=np.int64)
    np.cumsum(lens, out=indptr[1:])
    return indptr, np.concatenate(seqs).astype(np.int32)


def _device_fit(indptr, tokens, n_items, d, hs, window, seed, epochs, max_inflight, record=False, syn0=None):
    """Serial/default device epochs over a fixed corpus; returns host tables and the recorded streams."""
    from librecommender_b200 import skipgram as sg

    torch = _torch()
    dev = torch.device("cuda")
    vocab_items, counts = sg.vocabulary(tokens)
    tables = sg.Tables(vocab_items, counts, n_items, hs, dev)
    s0 = sg.initial_vectors(vocab_items, n_items, d, seed) if syn0 is None else syn0
    S0 = torch.as_tensor(s0, device=dev).clone()
    S1n = torch.zeros_like(S0)
    S1 = torch.zeros((max(len(vocab_items) - 1, 1), d), device=dev) if hs else None
    ip, tk = torch.as_tensor(indptr, device=dev), torch.as_tensor(np.r_[tokens, 0].astype(np.int32), device=dev)
    rec = []
    for e in range(epochs):
        kept, sent, klen, keep = sg.subsample(ip, tk[:tokens.size], n_items, tables.keep_thr, seed, e + 1, record=True)
        out = sg.epoch(ip, kept, sent, klen, n_items, S0, S1n, S1, tables, window, sg.ALPHA, sg.MIN_ALPHA,
                       e * tokens.size, epochs * tokens.size, seed, e + 1, max_inflight=max_inflight, record=record)
        rec.append((keep.cpu().numpy().astype(bool), kept.cpu().numpy(), sent.cpu().numpy(), klen.cpu().numpy(),
                    None if out is None else (out[0].cpu().numpy(), out[1].cpu().numpy())))
    torch.cuda.synchronize()
    return (S0.cpu().numpy(), S1n.cpu().numpy(), None if S1 is None else S1.cpu().numpy(), tables, rec, s0)


@pytest.mark.parametrize("max_inflight", [1, 7, 0])
def test_device_streams_equal_the_restatement(max_inflight):
    from librecommender_b200 import skipgram as sg

    g = np.random.default_rng(3)
    n_items, window, seed = 60, 5, (1 << 40) + 9
    indptr, tokens = _corpus(g, 40, n_items, 30)
    *_, tables, rec, _ = _device_fit(indptr, tokens, n_items, 8, 1, window, seed, 2, max_inflight, record=True)
    cum = sg.negative_table(tables.counts)
    for e, (keep, kept, sent, klen, (wout, nout)) in enumerate(rec):
        want_keep = orc.keep_decisions(tokens, tables.keep_thr.cpu().numpy(), seed, e + 1)
        assert np.array_equal(keep, want_keep)
        for s, (beg, items) in enumerate(orc.compact(indptr, tokens, want_keep)):
            n = items.size
            assert klen[s] == n and np.array_equal(kept[beg:beg + n], items)
            assert np.all(sent[beg:beg + n] == s) and np.all(sent[beg + n:indptr[s + 1]] == -1)
            if n == 0:
                continue
            b = orc.reduced_windows(beg + np.arange(n), window, seed, e + 1)
            assert np.array_equal(wout[beg:beg + n], b)
            for i in range(n):
                reach = window - int(b[i])
                js = [j for j in range(max(0, i - reach), min(n - 1, i + reach) + 1) if j != i]
                if js:
                    want = orc.negative_draws(beg + i, np.array(js) - i, window, 5, cum, tables.vocab_items, seed,
                                              e + 1)
                    assert np.array_equal(nout[beg + i][np.array(js) - i + window], want)


@pytest.mark.parametrize("max_inflight", [1, 7, 0])
def test_device_walks_equal_the_restatement(max_inflight):
    from librecommender_b200 import skipgram as sg

    torch = _torch()
    g = np.random.default_rng(5)
    n_items = 50
    indptr, tokens = _corpus(g, 30, n_items, 12)
    g_indptr, g_dst = sg.walk_graph(indptr, tokens, n_items)
    dev = torch.device("cuda")
    for pass_, L in ((0, 10), (3, 1), (7, 25)):
        ip, tk = sg.walks(torch.as_tensor(g_indptr, device=dev), torch.as_tensor(np.r_[g_dst, 0], device=dev),
                          n_items, 3, L, 42, pass_)
        want = orc.walks(g_indptr, g_dst, n_items, 3, L, 42, pass_)
        ip, tk = ip.cpu().numpy(), tk.cpu().numpy()
        assert [tk[ip[w]:ip[w + 1]].tolist() for w in range(len(want))] == want


@pytest.mark.parametrize("hs", [0, 1])
@pytest.mark.parametrize("d", [1, 7, 16, 64, 128])
def test_serial_schedule_equals_the_oracle(hs, d):
    from librecommender_b200 import skipgram as sg

    g = np.random.default_rng(100 + d + hs)
    n_items, window, seed = 40, 3, 11
    indptr, tokens = _corpus(g, 24, n_items, 14)
    epochs = 1 + (d % 2)
    s0, s1n, s1, tables, _, init = _device_fit(indptr, tokens, n_items, d, hs, window, seed, epochs, 1)
    syn1 = np.zeros((max(tables.V - 1, 1), d)) if hs else None
    args = ([(indptr, tokens)] * epochs, init, np.zeros_like(init), syn1, tables.vocab_items, tables.counts,
            tables.keep_thr.cpu().numpy(), hs, window, seed, tokens.size)
    ref = orc.train(np.float64, *args)
    f32 = orc.train(np.float32, *args)
    for got, r, u in zip((s0, s1n, s1), ref, f32):
        if r is None:
            continue
        unit = np.abs(u.astype(np.float64) - r).max(axis=1)
        dist = np.abs(got.astype(np.float64) - r).max(axis=1)
        bound = 4 * unit + FLOOR * (1 + np.abs(r).max(axis=1))
        assert np.all(dist <= bound), (d, hs, dist.max(), bound[np.argmax(dist - bound)])
    assert np.abs(s0 - init).max() > 0


def test_default_schedule_equals_serial_on_disjoint_rows():
    """Length-2 sentences over distinct items, and every negative mapped to one wall row whose |f| >= 6 always skips
    it: no two in-flight centres write the same row, so the default schedule is bit-identical to the serial one."""
    from librecommender_b200 import skipgram as sg

    torch = _torch()
    dev = torch.device("cuda")
    n_pairs, d = 4000, 16
    n_items = 2 * n_pairs + 1
    wall = n_items - 1
    tokens = np.arange(2 * n_pairs, dtype=np.int32)
    indptr = np.arange(0, 2 * n_pairs + 1, 2, dtype=np.int64)
    tables = sg.Tables(np.r_[tokens, wall].astype(np.int32), np.ones(2 * n_pairs + 1, dtype=np.int64), n_items, 0,
                       dev)
    tables.keep_thr.fill_(1 << 32)
    tables.neg_items.fill_(wall)                  # every negative draw lands on the wall row
    g = np.random.default_rng(0)
    s0 = (0.5 + 0.5 * g.random((n_items, d))).astype(np.float32)
    outs = []
    for mi in (1, 0):
        S0 = torch.as_tensor(s0, device=dev).clone()
        S1n = torch.zeros_like(S0)
        S1n[wall] = 100.0
        ip, tk = torch.as_tensor(indptr, device=dev), torch.as_tensor(tokens, device=dev)
        kept, sent, klen = sg.subsample(ip, tk, n_items, tables.keep_thr, 1, 1)
        sg.epoch(ip, kept, sent, klen, n_items, S0, S1n, None, tables, 5, 0.025, 1e-4, 0, tokens.size, 1, 1,
                 max_inflight=mi)
        outs.append((S0.cpu().numpy(), S1n.cpu().numpy()))
    assert np.array_equal(outs[0][0], outs[1][0]) and np.array_equal(outs[0][1], outs[1][1])
    assert np.abs(outs[0][1][:wall]).max() > 0 and outs[0][1][wall].min() == 100.0


@pytest.mark.parametrize("norm", [False, True])
def test_device_pooling_equals_the_mean_loop(norm):
    import types

    from librecommender_b200 import skipgram as sg

    g = np.random.default_rng(9)
    n_users, n_items, d = 300, 120, 16
    consumed = {u: g.integers(0, n_items, size=int(g.integers(1, 700 if u == 0 else 30))).tolist()
                for u in range(n_users)}
    vecs = g.standard_normal((n_items, d)).astype(np.float32)
    model = types.SimpleNamespace(gensim_model=types.SimpleNamespace(wv=types.SimpleNamespace(vectors=vecs)),
                                  n_items=n_items, n_users=n_users, user_consumed=consumed, norm_embed=norm)
    sg.set_embeddings(model)
    items = vecs / np.linalg.norm(vecs, axis=1, keepdims=True) if norm else vecs
    users = np.array([np.mean(items[consumed[u]], axis=0) for u in range(n_users)])
    assert np.allclose(model.item_embeds_np, items, rtol=1e-6, atol=1e-7)
    assert np.allclose(model.user_embeds_np, users, rtol=1e-5, atol=1e-6)


@pytest.mark.parametrize("mode", ["item2vec", "deepwalk"])
def test_trainer_equals_an_epoch_loop_and_serves(mode):
    from librecommender_b200 import recommend_from_embedding
    from librecommender_b200 import skipgram as sg

    torch = _torch()
    g = np.random.default_rng(21)
    n_users, n_items = 200, 150
    indptr, tokens = _corpus(g, n_users, n_items, 25)
    kw = dict(embed_size=16, window=5, seed=7, n_walks=2, walk_length=8, max_inflight=1)
    a = sg.SkipGramTrainer((indptr, tokens), n_items, mode, **kw).fit(2)
    b = sg.SkipGramTrainer((indptr, tokens), n_items, mode, **kw)
    for e in range(2):
        b.epoch(e, 2)
    assert torch.equal(a.syn0, b.syn0) and torch.equal(a.syn1neg, b.syn1neg)
    U, I = a.embeddings()
    assert U.shape == (n_users + 1, 16) and I.shape == (n_items + 1, 16)
    import types

    consumed = {u: tokens[indptr[u]:indptr[u + 1]].tolist() for u in range(n_users)}
    model = types.SimpleNamespace(task="ranking", n_items=n_items, n_users=n_users, user_consumed=consumed)
    users = list(range(3, 40))
    rec = recommend_from_embedding(model, users, 10, U.cpu().numpy(), I.cpu().numpy(), True, False)
    assert rec.shape == (len(users), 10)
    for r, u in enumerate(users):
        assert not set(rec[r].tolist()) & set(consumed[u])


def _c1():
    z = np.load(GOLDEN)
    return z, (z["c1_indptr"], z["c1_items"]), int(z["c1_shape"][1]), z["eval_users"], z["eval_items"]


@pytest.mark.parametrize("mode", ["item2vec", "deepwalk"])
def test_default_schedule_reaches_the_oracle_quality_on_c1(mode):
    from librecommender_b200 import skipgram as sg

    z, (indptr, items), n_items, ev_u, ev_i = _c1()
    epochs = int(z[f"{mode}_epochs"])
    tr = sg.SkipGramTrainer((indptr, items), n_items, mode, embed_size=16, window=5, seed=42, n_walks=2,
                            walk_length=10).fit(epochs)
    U, I = tr.embeddings()
    csr_ptr, csr_idx = z["c1_indptr"], z["c1_items"]
    r = orc.ranking_metrics(U.cpu().numpy()[:-1], I.cpu().numpy()[:-1], csr_ptr, csr_idx, ev_u, ev_i)
    want = z[f"{mode}_metrics"]
    assert r[0] >= (1 - QUALITY_MARGIN) * want[0] and r[1] >= (1 - QUALITY_MARGIN) * want[1], (r, want)


def _reference_fit(cls_name, tmp_path, **kw):
    import pandas as pd

    from oracle.ref_loader import load_reference, reference_available, sample_data_path

    if not reference_available():
        pytest.skip("reference tree not staged")
    libreco = load_reference()
    from librecommender_b200 import dropin

    dropin.install(libreco, gensim=True)
    try:
        import libreco.algorithms as algos
        from libreco.data import DatasetPure, split_by_ratio_chrono

        data = pd.read_csv(sample_data_path(), sep="::", names=["user", "item", "label", "time"], engine="python")
        train, test = split_by_ratio_chrono(data, test_size=0.2)
        train_data, data_info = DatasetPure.build_trainset(train)
        model = getattr(algos, cls_name)("ranking", data_info, embed_size=16, n_epochs=2, **kw)
        model.fit(train_data, neg_sampling=True, verbose=0)
        users = list(range(min(200, model.n_users)))
        rec = model.recommend_user(users, 10, inner_id=True)
        for u in users:
            got = np.asarray(rec[u])
            assert got.size == 10 and not set(got.tolist()) & set(model.user_consumed[u])
        assert np.all(np.isfinite(model.predict(users[:50], users[:50])))
        assert model.default_recs is not None and len(model.default_recs) > 0
        model.save(str(tmp_path), "m", inference_only=True)
        loaded = getattr(algos, cls_name).load(str(tmp_path), "m", data_info)
        rec2 = loaded.recommend_user(users, 10, inner_id=True)
        assert all(np.array_equal(rec[u], rec2[u]) for u in users)
        model.save(str(tmp_path), "full", inference_only=False)
        from librecommender_b200.skipgram import Word2Vec

        w2v = Word2Vec.load(os.path.join(str(tmp_path), "full_gensim.pkl"))
        assert np.array_equal(w2v.wv.get_vector("3"), model.gensim_model.wv.get_vector("3"))
    finally:
        dropin.uninstall()


def test_reference_item2vec_fit_under_the_dropin(tmp_path):
    _reference_fit("Item2Vec", tmp_path)


def test_reference_deepwalk_fit_under_the_dropin(tmp_path):
    _reference_fit("DeepWalk", tmp_path, n_walks=2, walk_length=10)
