"""GPU: the UserCF / ItemCF device engines (``csrc/cf.cu``, ``librecommender_b200.cf``) against the float64 oracles of
``_cf_oracle``: the known answer, random graphs on every dispatch path of ``b200_cf_cosine`` for both engines
(shared-memory and global accumulators, one split heavy row, splits over several rounds), ``min_common``, zero and
negative labels, recommend, ``random_rec`` and predict, both engines on C1, and the reference's own ``RsItemCF`` /
``RsUserCF`` under ``dropin.install(cf=True)``.

Labels are multiples of 0.5 of small magnitude, so every product and partial sum of a cosine's ``prod`` is exact in
fp32: the device's atomic order cannot change it, zero cosines are exactly zero, and the cosines match the float64
oracle to a few fp32 ulps.  Ties at the ``k_sim`` cut are compared as sets of values."""
import numpy as np
import pytest
import scipy.sparse as sp

import _cf_oracle as orc
from oracle.ref_loader import reference_available, sample_data_path
from test_cf_cpu import KNOWN_NEIGHBOURS, known_matrix

pytestmark = pytest.mark.gpu

LABELS = np.array([-1.5, -0.5, 0.0, 0.5, 1.0, 2.5], np.float32)


def engine(R, user_based, k_sim=20, min_common=1, task="ranking", consumed=None, default_pred=0.0):
    from librecommender_b200.cf import ItemCF, UserCF

    R = sp.csr_matrix(R)
    if consumed is None:
        consumed = {u: R.indices[R.indptr[u]:R.indptr[u + 1]].tolist() for u in range(R.shape[0])}
    cls = UserCF if user_based else ItemCF
    eng = cls(task, k_sim, R.shape[0], R.shape[1], min_common, R, R.T.tocsr(), consumed, default_pred)
    eng.compute_similarities(True, 1)
    return eng


def graph(rows, n_items, labels=None):
    indptr = np.cumsum([0] + [len(r) for r in rows])
    idx = np.concatenate([np.sort(np.asarray(r, dtype=np.int64)) for r in rows]) if len(rows) else np.zeros(0, int)
    data = np.ones(len(idx), np.float32) if labels is None else np.asarray(labels, np.float32)
    return sp.csr_matrix((data, idx, indptr), shape=(len(rows), n_items))


def random_rows(rng, n_rows, n_cols, deg_max, zipf=None):
    p = None
    if zipf is not None:
        p = 1.0 / np.arange(1, n_cols + 1) ** zipf
        p /= p.sum()
    return [rng.choice(n_cols, size=0 if r % 23 == 0 else int(rng.integers(1, deg_max + 1)), replace=False, p=p)
            for r in range(n_rows)]


def labelled(rng, rows, n_items, labels=LABELS):
    return graph(rows, n_items, rng.choice(labels, sum(len(r) for r in rows)))


def device_lists(eng):
    ids, sc, cnt = (t.cpu().numpy() for t in eng.neighbors())
    k = eng.k_sim
    return [(ids[x, :min(k, cnt[x])].astype(np.int64), sc[x, :min(k, cnt[x])].astype(np.float64))
            for x in range(len(cnt))]


def check_lists(eng, R, user_based, min_common, rtol=1e-6, atol=1e-6):
    x1, x2, cos = orc.matrix_sims(orc.sim_side(R, user_based), min_common)
    n_x = R.shape[0] if user_based else R.shape[1]
    lists, count = orc.topk_lists((x1, x2, cos), n_x, eng.k_sim)
    ids, sc, cnt = (t.cpu().numpy() for t in eng.neighbors())
    np.testing.assert_array_equal(cnt, count)
    assert eng.num_sim_elements() == int(count.sum())
    starts = np.concatenate([[0], np.cumsum(count)])
    for x in range(n_x):
        k = min(eng.k_sim, int(count[x]))
        assert (ids[x, k:] == -1).all() and (sc[x, k:] == 0).all()
        if k == 0:
            continue
        got = ids[x, :k]
        assert len(set(got.tolist())) == k and (got >= 0).all()
        assert (np.diff(sc[x, :k]) <= 0).all()
        ref = dict(zip(x2[starts[x]:starts[x + 1]].tolist(), cos[starts[x]:starts[x + 1]].tolist()))
        ref_of_got = np.array([ref[int(j)] for j in got])
        np.testing.assert_allclose(sc[x, :k], ref_of_got, rtol=rtol, atol=atol)
        # the same values as the oracle's first k (ids may differ only among equal values at the cut)
        np.testing.assert_allclose(np.sort(ref_of_got)[::-1], lists[x][1], rtol=rtol, atol=atol)
        row = cos[starts[x]:starts[x + 1]]      # a value tied with any other of the row, inside the cut or not
        unique = (np.abs(lists[x][1][:, None] - row[None, :]) <= atol + rtol * np.abs(row[None, :])).sum(axis=1) == 1
        np.testing.assert_array_equal(got[unique], lists[x][0][unique])
    return x1, x2, cos


def test_known_answer_on_the_device():
    M = known_matrix()
    for user_based, R in ((False, M.T.tocsr()), (True, M)):
        eng = engine(R, user_based, k_sim=10)
        ids, _, cnt = (t.cpu().numpy() for t in eng.neighbors())
        assert cnt.tolist() == [4] * 5
        assert ids[:, :4].tolist() == KNOWN_NEIGHBOURS and (ids[:, 4:] == -1).all()
        assert eng.num_sim_elements() == 20


@pytest.mark.parametrize("user_based", [False, True])
@pytest.mark.parametrize("k_sim", [1, 7, 20, 300])
@pytest.mark.parametrize("min_common", [1, 2])
def test_random_graph_shared_accumulator(user_based, k_sim, min_common):
    from librecommender_b200.cf import plan

    rng = np.random.default_rng(k_sim + 10 * min_common)
    n_users, n_items = 300, 400
    R = labelled(rng, random_rows(rng, n_users, n_items - 20, 30, zipf=0.6), n_items)  # the last 20 items: no user
    assert plan(n_users if user_based else n_items, k_sim)[0]
    check_lists(engine(R, user_based, k_sim, min_common), R, user_based, min_common)


@pytest.mark.parametrize("user_based", [False, True])
def test_random_graph_global_accumulator(user_based):
    from librecommender_b200.cf import plan

    rng = np.random.default_rng(5)
    if user_based:
        R = labelled(rng, random_rows(rng, 30_000, 3000, 4, zipf=0.8), 3000)
    else:
        R = labelled(rng, random_rows(rng, 1500, 40_000, 25, zipf=1.0), 40_000)
    assert not plan(R.shape[0] if user_based else R.shape[1], 20)[0]
    check_lists(engine(R, user_based, 20, 1), R, user_based, 1)


def work_of(R, user_based):
    """Per sim-side row: the summed length of the middle rows it walks (what the task plan splits on)."""
    M = orc.sim_side(R, user_based)
    deg = np.diff(sp.csr_matrix(M.T).indptr)
    return np.array([deg[M.indices[M.indptr[x]:M.indptr[x + 1]]].sum() for x in range(M.shape[0])])


@pytest.mark.parametrize("user_based", [False, True])
def test_split_heavy_row(user_based):
    rng = np.random.default_rng(6)
    n_users, n_items = 800, 500
    rows = random_rows(rng, n_users, n_items, 250)
    if user_based:         # user 7 holds every item: about 500 x 200 walked entries
        rows[7] = np.arange(n_items)
    else:                  # item 7: >= 700 users of about 125 items each
        rows = [np.union1d(r, [7]) if u < 700 else r for u, r in enumerate(rows)]
    R = labelled(rng, rows, n_items)
    work = work_of(R, user_based)
    assert work[7] > 65536 and (work > 65536).sum() <= 64        # split, within one round
    check_lists(engine(R, user_based, 50, 1), R, user_based, 1)


@pytest.mark.parametrize("user_based", [False, True])
def test_splits_over_several_rounds(user_based):
    rng = np.random.default_rng(7)
    if user_based:         # 400 users of 300 items out of 400: each walks about 300 x 300 entries
        R = labelled(rng, [rng.choice(400, 300, replace=False) for _ in range(400)] + random_rows(rng, 50, 400, 5),
                     400)
    else:                  # 2100 users of 250 items out of 400: each item walks about 1300 x 250 entries
        R = labelled(rng, [rng.choice(400, 250, replace=False) for _ in range(2100)], 400)
    assert (work_of(R, user_based) > 65536).sum() > 64
    check_lists(engine(R, user_based, 20, 2), R, user_based, 2)


@pytest.mark.parametrize("user_based", [False, True])
def test_zero_labels_keep_zero_cosines(user_based):
    rng = np.random.default_rng(8)
    R = labelled(rng, random_rows(rng, 200, 150, 10), 150, labels=np.array([0.0, 0.0, 1.0], np.float32))
    eng = engine(R, user_based, 500, 1)
    _, _, cos = check_lists(eng, R, user_based, 1)
    assert (cos == 0).sum() > 100
    sc, cnt = eng.neighbors()[1].cpu().numpy(), eng.neighbors()[2].cpu().numpy()
    kept = np.arange(sc.shape[1])[None, :] < cnt[:, None]
    assert (sc[kept] == 0).sum() == (cos == 0).sum()        # every zero cosine is kept, within k_sim = 500


# ---- serving -------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module", params=[False, True], ids=["item", "user"])
def served(request):
    user_based = request.param
    rng = np.random.default_rng(9)
    n_users, n_items = 240, 150
    R = labelled(rng, random_rows(rng, n_users, n_items, 12), n_items)
    half = n_users // 2
    consumed = {u: R.indices[R.indptr[u]:R.indptr[u + 1]].tolist() for u in range(half)}
    from librecommender_b200.consumed import ConsumedCSR

    eng = engine(R, user_based, 8, 1, consumed=ConsumedCSR.from_dict(consumed, half))
    return user_based, R, consumed, eng, device_lists(eng)


def check_recs(got, want, dicts, tol=1e-5):
    for g, w, d in zip(got, want, dicts):
        assert len(g) == len(w)
        if g != w:
            scale = max(abs(v) for v in d.values())
            assert all(abs(d[a] - d[b]) <= tol * scale for a, b in zip(g, w)), (g, w)


@pytest.mark.parametrize("filter_consumed", [True, False])
def test_recommend(served, filter_consumed):
    user_based, R, consumed, eng, lists = served
    users = list(range(R.shape[0])) + [R.shape[0], -1]
    for n_rec in (5, R.shape[1]):
        recs, no_rec = eng.recommend(users, n_rec, filter_consumed, False)
        want, want_no, dicts = orc.recommend(R, lists, 8, consumed, users, n_rec, filter_consumed, user_based)
        assert no_rec == want_no and len(no_rec) > 2
        check_recs(recs, want, dicts)
        if n_rec == R.shape[1]:
            assert all(set(g) == set(d) for g, d in zip(recs, dicts))
            assert any(v < 0 for d in dicts for v in d.values())
        if filter_consumed:
            assert all(not set(g) & set(consumed.get(r, [])) for r, g in enumerate(recs))


def test_random_rec(served):
    import torch

    user_based, R, consumed, eng, lists = served
    users = torch.arange(R.shape[0])
    a = eng.recommend_device(users, 3, True, True, seed=11)
    b = eng.recommend_device(users, 3, True, True, seed=11)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])
    ids, n = a[0].cpu().numpy(), a[1].cpu().numpy()
    _, _, dicts = orc.recommend(R, lists, 8, consumed, list(range(R.shape[0])), 3, True, user_based)
    for r, d in enumerate(dicts):
        g = ids[r, :n[r]].tolist()
        assert n[r] == min(3, len(d)) and len(set(g)) == len(g) and set(g) <= set(d)
    c = eng.recommend_device(users, 3, True, True, seed=12)[0]
    assert not torch.equal(a[0], c)


@pytest.mark.parametrize("task", ["rating", "ranking"])
def test_predict(served, task):
    user_based, R, _, eng, lists = served
    eng.task = task
    try:
        rng = np.random.default_rng(0)
        n_users, n_items = R.shape
        users = np.concatenate([rng.integers(0, n_users, 3000), R.nonzero()[0][:500], [n_users, 0, -1, 3]])
        items = np.concatenate([rng.integers(0, n_items, 3000), R.nonzero()[1][:500], [0, n_items, 2, -4]])
        got = eng.predict(users.tolist(), items.tolist())
        want = orc.predict(R, lists, 8, task, users, items, 0.0, user_based)
        np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6)
        assert got[-4:] == [0.0] * 4
        assert sum(g != 0 for g in got) > 100
    finally:
        eng.task = "ranking"


@pytest.mark.parametrize("user_based", [False, True])
def test_predict_zero_sum_of_sims_is_nan(user_based):
    # users 0 and 1 share item 0; user 1's only label is 0, so sq = 0 and every cosine of user 1 (and of item 0 with
    # item 1 for ItemCF) is 0: rating predict divides 0 by a zero sum
    R = graph([[0], [0, 1]], 3, [1.0, 1.0, 0.0]) if not user_based else graph([[0], [0]], 3, [1.0, 0.0])
    eng = engine(R, user_based, 5, 1, task="rating", default_pred=7.0)
    if user_based:   # user 0's neighbour 1 (sim 0: user 1's sq is 0) holds item 0 with label 0
        q = ([0, 0, 2], [0, 1, 0])
    else:            # item 1's neighbour 0 (sim 0: item 1's sq is 0) is in row 1 with label 1
        q = ([1, 0, 0], [1, 2, 3])
    got = eng.predict(*q)
    assert np.isnan(got[0]) and got[1:] == [7.0, 7.0]
    eng.task = "ranking"
    assert eng.predict(q[0][:1], q[1][:1]) == [0.0]


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


@pytest.mark.parametrize("user_based", [False, True])
def test_c1(user_based):
    R, consumed = c1()
    eng = engine(R, user_based, 20, 1, task="rating", consumed=consumed, default_pred=3.5)
    check_lists(eng, R, user_based, 1, rtol=1e-5, atol=1e-6)
    lists = device_lists(eng)
    users = list(range(0, R.shape[0], 3))
    for filt in (True, False):
        recs, no_rec = eng.recommend(users, 10, filt, False)
        want, want_no, dicts = orc.recommend(R, lists, 20, consumed, users, 10, filt, user_based)
        assert no_rec == want_no
        check_recs(recs, want, dicts)
    rng = np.random.default_rng(0)
    pu = np.concatenate([rng.integers(0, R.shape[0], 3000), R.nonzero()[0][:500]])
    pi = np.concatenate([rng.integers(0, R.shape[1], 3000), R.nonzero()[1][:500]])
    got = eng.predict(pu.tolist(), pi.tolist())
    want = orc.predict(R, lists, 20, "rating", pu, pi, 3.5, user_based)
    np.testing.assert_allclose(got, want, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("name", ["RsItemCF", "RsUserCF"])
def test_dropin_reference_cf(name):
    if not reference_available():
        pytest.skip("reference neither mounted nor staged")
    from oracle.ref_loader import load_reference

    load_reference()
    import sys

    import pandas as pd

    import libreco
    from libreco import algorithms
    from libreco.bases.cf_base_rs import RsCfBase
    from libreco.data import DatasetPure, split_by_ratio_chrono
    from libreco.evaluation import evaluate

    from librecommender_b200 import dropin

    cls = getattr(algorithms, name)
    user_based = name == "RsUserCF"
    df = pd.read_csv(sample_data_path(), sep="::", names=["user", "item", "label", "time"], engine="python")
    train, test = split_by_ratio_chrono(df, test_size=0.2)
    train_data, di = DatasetPure.build_trainset(train)
    eval_data = DatasetPure.build_testset(test)
    original = RsCfBase.fit
    model = cls("rating", di, k_sim=20)
    dropin.install(libreco, losses=False, lightgcn=False, cf=True)
    try:
        model.fit(train_data, neg_sampling=False, verbose=2, eval_data=eval_data, metrics=["rmse", "mae"])
        assert "recfarm" not in sys.modules
    finally:
        dropin.uninstall()
    assert RsCfBase.fit is original
    R = train_data.sparse_interaction
    x1, _, _ = orc.matrix_sims(orc.sim_side(R, user_based), 1)
    assert model.rs_model.num_sim_elements() == len(x1)
    lists = device_lists(model.rs_model)
    users = list(range(0, di.n_users, 7))
    recs = model.recommend_user(users, 10, inner_id=True)
    want, _, dicts = orc.recommend(R, lists, 20, di.user_consumed, users, 10, True, user_based)
    popular = {di.item2id[i] for i in di.popular_items}
    for u, w, sc_u in zip(users, want, dicts):
        g = list(recs[u])
        assert len(g) == (min(10, len(sc_u)) if w else 10)
        head = g[:len(w)]
        if head != w:
            scale = max(abs(v) for v in sc_u.values())
            assert all(abs(sc_u[a] - sc_u[b]) <= 1e-5 * scale for a, b in zip(head, w))
        if not w:
            assert set(g) <= popular        # the reference's popular fill of a user without candidates
    pu = [di.id2user[u] for u in users[:300]]
    pi = [di.id2item[int(i)] for i in np.random.default_rng(1).integers(0, di.n_items, len(pu))]
    got = model.predict(pu, pi)
    want_p = orc.predict(R, lists, 20, "rating", users[:300], [di.item2id[x] for x in pi], model.default_pred,
                         user_based)
    np.testing.assert_allclose(got, want_p, rtol=1e-4, atol=1e-5)
    assert model.predict("no-such-user", pi[0]) == np.float32(model.default_pred)     # recfarm keeps it in f32
    res = evaluate(model, eval_data, False, metrics=["rmse", "mae"])
    assert np.isfinite(res["rmse"]) and np.isfinite(res["mae"])
