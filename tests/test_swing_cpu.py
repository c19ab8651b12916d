"""CPU: the Swing oracles on the known answer of recfarm's unit test, against each other, and on serving edge cases;
the device engine's host validation and the drop-in wiring (no launch)."""
import math

import numpy as np
import pytest
import scipy.sparse as sp

import _swing_oracle as orc


def known_graph():
    # rust/src/swing.rs tests: users {0,1,2,3}, {0,1,3}, {0,2,3,4}; 5 items
    rows = [[0, 1, 2, 3], [0, 1, 3], [0, 2, 3, 4]]
    indptr = np.cumsum([0] + [len(r) for r in rows])
    idx = np.concatenate(rows)
    return sp.csr_matrix((np.ones(len(idx), np.float32), idx, indptr), shape=(3, 5))


def known_item0(dtype=np.float64):
    w = [1 / math.sqrt(4), 1 / math.sqrt(3), 1 / math.sqrt(4)]
    s01, s02, s12 = w[0] * w[1] / 3, w[0] * w[2] / 3, w[1] * w[2] / 2
    return [(3, s01 + s02 + s12), (1, s01), (2, s02)]


def random_graph(rng, n_users, n_items, max_deg, labels=False):
    rows, data = [], []
    for _ in range(n_users):
        k = int(rng.integers(1, max_deg + 1))
        rows.append(np.sort(rng.choice(n_items, size=min(k, n_items), replace=False)))
        data.append(rng.choice([0.0, 1.0, 2.5], size=len(rows[-1])) if labels else np.ones(len(rows[-1])))
    indptr = np.cumsum([0] + [len(r) for r in rows])
    return sp.csr_matrix((np.concatenate(data).astype(np.float32), np.concatenate(rows), indptr),
                         shape=(n_users, n_items))


def test_known_answer_both_oracles():
    R = known_graph()
    want = known_item0()
    lists, count = orc.topk_lists(orc.matrix_scores(R, 1.0), 10)
    assert count[0] == 3
    assert lists[0][0].tolist() == [j for j, _ in want]
    np.testing.assert_allclose(lists[0][1], [s for _, s in want], rtol=1e-15)
    lit = orc.literal_scores(R, 1.0)
    np.testing.assert_allclose(lit[0, [3, 1, 2]], [s for _, s in want], rtol=1e-6)
    assert lit[0, 0] == 0 and lit[0, 4] == 0
    assert count[4] == 0 and lists[4][0].size == 0       # item 4 has one user: no pair


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("alpha", [0.0, 1.0, 3.5])
def test_literal_loop_and_matrix_oracle_agree(seed, alpha):
    rng = np.random.default_rng(seed)
    R = random_graph(rng, 25, 18, 9, labels=True)
    lit = orc.literal_scores(R, alpha, dtype=np.float64)
    mat = orc.matrix_scores(R, alpha).toarray()
    assert (lit != 0).sum() == (mat != 0).sum() > 0
    np.testing.assert_allclose(lit, mat, rtol=1e-12, atol=0)
    lit32 = orc.literal_scores(R, alpha)
    np.testing.assert_allclose(lit32, mat, rtol=1e-5, atol=0)


def serving_case():
    # labels != 1, a zero label, an empty user row (user 3)
    # row 0 holds an explicit zero label at item 3: stored, so it still sends terms
    R = sp.csr_matrix((np.array([2.0, 1.0, 0.0, 1.0, 1.0, 0.5], np.float32), np.array([0, 2, 3, 1, 3, 0]),
                       np.array([0, 3, 5, 6, 6])), shape=(4, 4))
    lists = [(np.array([1, 2]), np.array([0.5, 0.25])), (np.array([0, 3]), np.array([1.0, 0.75])),
             (np.array([0]), np.array([0.125])), (np.array([1, 2, 0]), np.array([0.5, 0.4, 0.3]))]
    consumed = {0: [0, 2, 3], 1: [1, 3], 2: [0], 3: []}
    return R, lists, consumed


def test_recommend_restatement_edge_cases():
    R, lists, consumed = serving_case()
    assert R.nnz == 6
    recs, extra, sc = orc.recommend(R, lists, 2, consumed, [0, 1, 2, 3, 99], 3, False)
    # user 0: items 0 (2.0), 2 (1.0), 3 (0.0 explicit): 0 -> {1: 1.0, 2: 0.5}; 2 -> {0: 0.125}; 3 -> {1: 0, 2: 0}
    assert sc[0] == {1: 1.0, 2: 0.5, 0: 0.125}
    assert recs[0] == [1, 2, 0] and extra[0] == 0
    assert recs[3] == [] and extra[3] == 3 and recs[4] == [] and extra[4] == 3
    recs, extra, sc = orc.recommend(R, lists, 2, consumed, [0, 2], 3, True)
    assert sc[0] == {1: 1.0} and recs[0] == [1] and extra[0] == 2
    # user 2: item 0 (0.5) -> {1: 0.25, 2: 0.125}; item 0 is consumed but is not a neighbour anyway
    assert sc[1] == {1: 0.25, 2: 0.125}
    # a zero label still makes a candidate (score 0)
    R2 = sp.csr_matrix((np.array([0.0], np.float32), np.array([2]), np.array([0, 1])), shape=(1, 4))
    recs, extra, sc = orc.recommend(R2, lists, 2, {0: [2]}, [0], 5, True)
    assert sc[0] == {0: 0.0} and recs[0] == [0] and extra[0] == 4


def test_predict_restatement_edge_cases():
    R, lists, _ = serving_case()
    got = orc.predict(R, lists, 2, 4, 4, [0, 0, 1, 3, 4, 0, 2], [3, 1, 0, 0, 0, 4, 1], default_pred=0.0)
    # (0, 3): neighbours 1 (not in row 0), 2 (in) -> 0.4;  (0, 1): 0 and 3 both in row 0 -> mean(1, .75)
    # (1, 0): 1 in row 1 -> 0.5;  (3, 0): empty row;  (4, 0): unknown user;  (0, 4): unknown item;  (2, 1): 0 -> 1.0
    np.testing.assert_allclose(got, [0.4, 0.875, 0.5, 0.0, 0.0, 0.0, 1.0])
    got = orc.predict(R, lists, 1, 4, 4, [0], [3])
    assert got == [0.0]               # top_k 1: only neighbour 1, not in row 0 -> default


def _engine(**kw):
    from librecommender_b200.swing import Swing

    R = known_graph()
    args = dict(top_k=10, alpha=1.0, max_cache_num=100, n_users=3, n_items=5, user_interacts=R,
                item_interacts=R.T.tocsr(), user_consumed={0: [0, 1], 1: [0, 1], 2: [0, 1, 2]}, default_pred=0.0)
    args.update(kw)
    return Swing(**args)


@pytest.mark.parametrize("kw, msg", [
    (dict(top_k=0), "top_k"), (dict(top_k=4097), "top_k"), (dict(top_k=2.5), "top_k"), (dict(top_k=True), "top_k"),
    (dict(alpha=-1.0), "alpha"), (dict(alpha=float("nan")), "alpha"), (dict(alpha=float("inf")), "alpha"),
    (dict(alpha=1e39), "alpha"), (dict(n_users=2), "rows"), (dict(n_items=3), "outside"),
])
def test_validation_errors(kw, msg):
    with pytest.raises(ValueError, match=msg):
        _engine(**kw)


def test_validation_of_the_csrs():
    R = known_graph()
    bad = R.copy()
    bad.indices[[0, 1]] = bad.indices[[1, 0]]            # row 0 unsorted
    with pytest.raises(ValueError, match="sorted"):
        _engine(user_interacts=bad)
    dup = sp.csr_matrix((np.ones(3, np.float32), np.array([1, 1, 2]), np.array([0, 2, 3, 3])), shape=(3, 5))
    with pytest.raises(ValueError, match="sorted"):
        _engine(user_interacts=dup, item_interacts=sp.csr_matrix(dup.T))
    other = sp.csr_matrix(np.eye(3, 5, dtype=np.float32))
    with pytest.raises(ValueError, match="transpose"):
        _engine(item_interacts=other.T.tocsr())
    with pytest.raises(ValueError, match="not a CSR"):
        _engine(user_interacts=type("M", (), {"sparse_indptr": [0, 2], "sparse_indices": [0], "sparse_data": [1]})())


def test_dropin_wiring_without_launch():
    import sys

    from oracle.ref_loader import load_reference, reference_available

    if not reference_available():
        pytest.skip("reference neither mounted nor staged")
    load_reference()
    import libreco
    from libreco.algorithms import swing as ref_swing

    from librecommender_b200 import dropin

    original = ref_swing.Swing.fit
    dropin.install(libreco, losses=False, lightgcn=False, swing=True)
    try:
        assert ref_swing.Swing.fit is not original
        assert "recfarm" not in sys.modules
        model = type("M", (), {"incremental": True})()
        with pytest.raises(NotImplementedError):
            ref_swing.Swing.fit(model, None, False)
    finally:
        dropin.uninstall()
    assert ref_swing.Swing.fit is original
