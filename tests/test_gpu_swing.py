"""GPU: Swing's device engine (``csrc/swing.cu``, ``librecommender_b200.swing``) against the float64 oracles of
``_swing_oracle``: the known answer, random graphs on every dispatch path of ``b200_swing_scores`` (shared-memory and
global accumulators, split heavy items in one and in several rounds), recommend and predict on C1, and the reference's
own ``Swing`` under ``dropin.install(swing=True)``."""
import numpy as np
import pytest
import scipy.sparse as sp

import _swing_oracle as orc
from oracle.ref_loader import reference_available, sample_data_path
from test_swing_cpu import known_graph, known_item0

pytestmark = pytest.mark.gpu


def engine(R, top_k=20, alpha=1.0, consumed=None, **kw):
    from librecommender_b200.swing import Swing

    R = sp.csr_matrix(R)
    if consumed is None:
        consumed = {u: R.indices[R.indptr[u]:R.indptr[u + 1]].tolist() for u in range(R.shape[0])}
    eng = Swing(top_k, alpha, 100_000_000, R.shape[0], R.shape[1], R, R.T.tocsr(), consumed, 0.0, **kw)
    eng.compute_swing(1)
    return eng


def graph(rows, n_items, labels=None):
    indptr = np.cumsum([0] + [len(r) for r in rows])
    idx = np.concatenate([np.sort(np.asarray(r, dtype=np.int64)) for r in rows])
    data = np.ones(len(idx), np.float32) if labels is None else labels
    return sp.csr_matrix((data, idx, indptr), shape=(len(rows), n_items))


def check_lists(eng, R, alpha, top_k, tol=1e-5, atol=0.0):
    S = orc.matrix_scores(R, alpha).tocsr()
    lists, count = orc.topk_lists(S, top_k)
    ids, sc, cnt = (t.cpu().numpy() for t in eng.neighbors())
    np.testing.assert_array_equal(cnt, count)
    assert eng.num_swing_elements() == int(count.sum())
    for i in range(R.shape[1]):
        k = min(top_k, int(count[i]))
        assert (ids[i, k:] == -1).all() and (sc[i, k:] == 0).all()
        if k == 0:
            continue
        got = ids[i, :k]
        assert len(set(got.tolist())) == k and (got >= 0).all()
        assert (np.diff(sc[i, :k]) <= 0).all()
        row = S.getrow(i)
        ref_of_got = row[:, got].toarray().ravel()
        np.testing.assert_allclose(sc[i, :k], ref_of_got, rtol=tol, atol=atol)
        want_ids, want_s = lists[i]
        diff = got != want_ids
        if diff.any():       # ids may differ only inside the near-tie band at equal ranks
            scale = float(want_s[0])
            assert np.all(np.abs(ref_of_got[diff] - want_s[diff]) <= tol * scale + 2 * atol), (i, got, want_ids)


def test_known_answer_on_the_device():
    eng = engine(known_graph(), top_k=10)
    ids, sc, cnt = (t.cpu().numpy() for t in eng.neighbors())
    want = known_item0()
    assert cnt[0] == 3 and ids[0, :4].tolist() == [3, 1, 2, -1]
    np.testing.assert_allclose(sc[0, :3], [s for _, s in want], rtol=1e-6)
    assert cnt[4] == 0 and (ids[4] == -1).all()
    assert eng.num_swing_elements() == int(cnt.sum())


def random_rows(rng, n_users, n_items, deg_max, zipf=None):
    p = None
    if zipf is not None:
        p = 1.0 / np.arange(1, n_items + 1) ** zipf
        p /= p.sum()
    rows = []
    for u in range(n_users):
        k = 1 if u % 17 == 0 else int(rng.integers(2, deg_max + 1))      # some users with one item
        rows.append(rng.choice(n_items, size=k, replace=False, p=p))
    return rows


@pytest.mark.parametrize("top_k", [1, 7, 20, 300])
@pytest.mark.parametrize("alpha", [0.0, 1.0])
def test_random_graph_shared_accumulator(top_k, alpha):
    from librecommender_b200.swing import plan

    rng = np.random.default_rng(top_k)
    n_items = 400
    rows = random_rows(rng, 300, n_items - 20, 30, zipf=0.6)   # the last 20 items have no user
    rows.append([n_items - 5])                                 # ... but one has a single user
    R = graph(rows, n_items)
    assert plan(n_items, top_k)[0]
    check_lists(engine(R, top_k, alpha), R, alpha, top_k)


def test_random_graph_global_accumulator():
    from librecommender_b200.swing import plan

    rng = np.random.default_rng(5)
    n_items = 60_000
    R = graph(random_rows(rng, 1500, n_items, 25, zipf=1.0), n_items)
    assert not plan(n_items, 20)[0]
    check_lists(engine(R, 20, 1.0), R, 1.0, 20)


def test_split_heavy_item():
    rng = np.random.default_rng(6)
    n_items = 500
    rows = random_rows(rng, 800, n_items, 12)
    rows = [np.union1d(r, [7]) if u < 700 else r for u, r in enumerate(rows)]      # item 7: >= 700 users
    R = graph(rows, n_items)
    assert np.diff(R.tocsc().indptr)[7] >= 700       # 244 650 pairs: split into pieces
    check_lists(engine(R, 50, 1.0), R, 1.0, 50)


def test_split_items_over_several_rounds():
    rng = np.random.default_rng(7)
    n_items = 400
    # 70 items of about 300 users each (> 32768 pairs: split), more than the 64 split slots of a round; each user
    # holds 10 of them, so a score sums about C(40, 2) terms and its fp32 rounding stays far below 1e-5
    rows = [np.concatenate([rng.choice(70, 10, replace=False), rng.choice(np.arange(70, n_items), 3, replace=False)])
            for _ in range(2100)]
    R = graph(rows, n_items)
    assert (np.diff(R.tocsc().indptr)[:70] >= 257).sum() > 64
    check_lists(engine(R, 20, 0.5), R, 0.5, 20)


def test_subnormal_terms_on_the_global_and_split_paths():
    """alpha = 1e38 makes every term subnormal (at most 0.5 / alpha).  The adds keep them, as recfarm's fp32 sums do:
    the nonzero counts are exact and the scores match the float64 oracle to a few subnormal ulps per term."""
    from librecommender_b200.swing import plan

    rng = np.random.default_rng(8)
    n_items = 60_000
    rows = random_rows(rng, 1500, n_items, 25)
    # item 7: 300 users (> 32768 pairs: split), each also holding 3 of 40 pool items, so a score of item 7 sums a few
    # hundred terms and its fp32 rounding stays well below 1e-5
    rows = [np.union1d(r, np.concatenate([[7], 100 + rng.choice(40, 3, replace=False)])) if u < 300 else r
            for u, r in enumerate(rows)]
    R = graph(rows, n_items)
    assert not plan(n_items, 20)[0] and np.diff(R.tocsc().indptr)[7] >= 257
    eng = engine(R, 20, 1e38)
    sc = eng.neighbors()[1].cpu().numpy()
    assert 0 < sc[sc > 0].min() < np.finfo(np.float32).tiny           # single-term scores stay subnormal
    # a term is at least 0.2^2 / 1e38 = 4e-40; each rounding is at most 2^-150, so relative errors stay below 1e-5
    check_lists(eng, R, 1e38, 20, tol=1e-5, atol=2.0 ** -149 * 64)


def test_recommend_zero_and_fractional_labels_on_the_device():
    """Labels 0, 0.5, 1 and 2.5: a candidate reached only through zero labels has score 0 and still counts; the
    consumed CSR covers half of the users only (the rest have nothing to filter)."""
    from librecommender_b200.consumed import ConsumedCSR

    rng = np.random.default_rng(9)
    n_users, n_items = 240, 150
    rows = random_rows(rng, n_users, n_items, 12)
    labels = rng.choice(np.array([0.0, 0.5, 1.0, 2.5], np.float32), sum(len(r) for r in rows))
    R = graph(rows, n_items, labels)
    half = n_users // 2
    consumed = {u: R.indices[R.indptr[u]:R.indptr[u + 1]].tolist() for u in range(half)}
    eng = engine(R, 8, 1.0, ConsumedCSR.from_dict(consumed, half))
    ids, sc, cnt = (t.cpu().numpy() for t in eng.neighbors())
    lists = [(ids[i, :min(8, cnt[i])].astype(np.int64), sc[i, :min(8, cnt[i])].astype(np.float64))
             for i in range(n_items)]
    users = list(range(n_users))
    zero_seen = False
    for n_rec in (5, n_items):
        for filt in (True, False):
            recs, extra = eng.recommend(users, n_rec, filt, False)
            want, want_extra, dicts = orc.recommend(R, lists, 8, consumed, users, n_rec, filt)
            assert extra == want_extra
            for g, w, d in zip(recs, want, dicts):
                assert len(g) == len(w)
                if g != w:
                    scale = max(abs(v) for v in d.values())
                    assert all(abs(d[a] - d[b]) <= 1e-5 * scale for a, b in zip(g, w)), (g, w)
                if n_rec == n_items:
                    assert set(g) == set(d)
                    zero_seen |= any(v == 0.0 for v in d.values())
    assert zero_seen


# ---- C1 ------------------------------------------------------------------------------------------------------------
def c1():
    import pandas as pd

    if not reference_available():
        pytest.skip("reference neither mounted nor staged: no C1 data")
    df = pd.read_csv(sample_data_path(), sep="::", names=["user", "item", "label", "time"], engine="python")
    u, _ = pd.factorize(df["user"])
    i, _ = pd.factorize(df["item"])
    df = pd.DataFrame({"u": u, "i": i, "label": df["label"].astype(np.float32)})
    consumed = df.groupby("u")["i"].apply(list).to_dict()
    df = df.drop_duplicates(subset=["u", "i"], keep="last")
    R = sp.csr_matrix((df["label"].to_numpy(), (df["u"].to_numpy(), df["i"].to_numpy())), dtype=np.float32)
    R.sort_indices()
    return R, consumed


@pytest.fixture(scope="module")
def c1_engine():
    R, consumed = c1()
    eng = engine(R, 20, 1.0, consumed)
    ids, sc, cnt = (t.cpu().numpy() for t in eng.neighbors())
    lists = [(ids[i, :min(20, cnt[i])].astype(np.int64), sc[i, :min(20, cnt[i])].astype(np.float64))
             for i in range(R.shape[1])]
    return R, consumed, eng, lists


def test_c1_lists_against_the_matrix_oracle(c1_engine):
    R, _, eng, _ = c1_engine
    check_lists(eng, R, 1.0, 20)


@pytest.mark.parametrize("n_rec", [10, 100])
@pytest.mark.parametrize("filter_consumed", [True, False])
def test_c1_recommend(c1_engine, n_rec, filter_consumed):
    R, consumed, eng, lists = c1_engine
    users = list(range(R.shape[0])) + [R.shape[0], -1]
    recs, extra = eng.recommend(users, n_rec, filter_consumed, False)
    want, want_extra, dicts = orc.recommend(R, lists, 20, consumed, users, n_rec, filter_consumed)
    assert extra == want_extra
    for r, (g, w, sc) in enumerate(zip(recs, want, dicts)):
        assert len(g) == len(w) == min(n_rec, len(sc))
        if g != w:
            scale = max(abs(v) for v in sc.values())
            for a, b in zip(g, w):
                assert abs(sc[a] - sc[b]) <= 1e-5 * scale, (r, g, w)
        if filter_consumed and r < R.shape[0]:
            assert not set(g) & set(consumed.get(r, []))
    rnd, rnd_extra = eng.recommend(users, n_rec, filter_consumed, True)
    assert rnd_extra == want_extra
    for g, w, sc in zip(rnd, want, dicts):
        assert len(g) == len(set(g)) == len(w) and set(g) <= set(sc)
        if len(sc) <= n_rec:
            assert set(g) == set(w)


def test_c1_predict(c1_engine):
    R, _, eng, lists = c1_engine
    rng = np.random.default_rng(0)
    n_users, n_items = R.shape
    users = np.concatenate([rng.integers(0, n_users, 4000), R.nonzero()[0][:500], [n_users, 0, n_users + 3, -1]])
    items = np.concatenate([rng.integers(0, n_items, 4000), R.nonzero()[1][:500], [0, n_items, 2, 1]])
    got = eng.predict(users.tolist(), items.tolist())
    want = orc.predict(R, lists, 20, n_users, n_items, users, items, 0.0)
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=0)
    assert got[-4:] == [0.0] * 4
    assert sum(g != 0 for g in got) > 100


def test_dropin_reference_swing():
    if not reference_available():
        pytest.skip("reference neither mounted nor staged")
    from oracle.ref_loader import load_reference

    load_reference()
    import sys

    import pandas as pd

    import libreco
    from libreco.algorithms import Swing
    from libreco.data import DatasetPure, split_by_ratio_chrono

    from librecommender_b200 import dropin

    df = pd.read_csv(sample_data_path(), sep="::", names=["user", "item", "label", "time"], engine="python")
    train, _ = split_by_ratio_chrono(df, test_size=0.2)
    train_data, di = DatasetPure.build_trainset(train)
    original = Swing.fit
    model = Swing("ranking", di, top_k=20, alpha=1.0)
    dropin.install(libreco, losses=False, lightgcn=False, swing=True)
    try:
        model.fit(train_data, neg_sampling=True, verbose=0)
        assert "recfarm" not in sys.modules
    finally:
        dropin.uninstall()
    assert Swing.fit is original
    R = train_data.sparse_interaction
    S = orc.matrix_scores(R, 1.0)
    _, count = orc.topk_lists(S, 20)
    assert model.rs_model.num_swing_elements() == int(count.sum())
    popular = {di.item2id[i] for i in di.popular_items}
    ids, sc, cnt = (t.cpu().numpy() for t in model.rs_model.neighbors())
    lists = [(ids[i, :min(20, cnt[i])].astype(np.int64), sc[i, :min(20, cnt[i])].astype(np.float64))
             for i in range(di.n_items)]
    users = list(range(0, di.n_users, 7))
    recs = model.recommend_user(users, 10, inner_id=True)
    want, extra, dicts = orc.recommend(R, lists, 20, di.user_consumed, users, 10, True)
    for u, w, e, sc_u in zip(users, want, extra, dicts):
        g = list(recs[u])
        assert len(g) == 10
        head = g[:len(w)]
        if head != w:
            scale = max(abs(v) for v in sc_u.values())
            assert all(abs(sc_u[a] - sc_u[b]) <= 1e-5 * scale for a, b in zip(head, w))
        assert set(g[len(w):]) <= popular          # the reference's popular fill of the additional count
    cold = model.recommend_user("no-such-user", 10)
    assert len(cold["no-such-user"]) == 10 and set(cold["no-such-user"]) <= set(di.popular_items)
    pu = [di.id2user[u] for u in users[:300]]
    pi = [di.id2item[int(i)] for i in np.random.default_rng(1).integers(0, di.n_items, len(pu))]
    got = model.predict(pu, pi)
    want_p = orc.predict(R, lists, 20, di.n_users, di.n_items, users[:300],
                         [di.item2id[x] for x in pi], model.default_pred)
    np.testing.assert_allclose(got, want_p, rtol=1e-5, atol=0)
    assert model.predict("no-such-user", pi[0]) == model.default_pred
