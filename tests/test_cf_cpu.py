"""CPU: the UserCF / ItemCF oracles on the known answers of recfarm's unit tests, against each other, and on serving
edge cases; the device engines' host validation, return contracts that need no launch, and the drop-in wiring."""
import numpy as np
import pytest
import scipy.sparse as sp

import _cf_oracle as orc


def known_matrix():
    # rust/src/item_cf.rs and user_cf.rs tests: the sim-side matrix
    # [[1, 1, 0, 0], [2, 1, 0, 0], [0, 1, 1, 0], [2, 1, 1, 0], [0, 1, 2, 0]]
    return sp.csr_matrix((np.array([1., 1., 2., 1., 1., 1., 2., 1., 1., 1., 2.], np.float32),
                          np.array([0, 1, 0, 1, 1, 2, 0, 1, 2, 1, 2]), np.array([0, 2, 4, 6, 9, 11])), shape=(5, 4))


KNOWN_NEIGHBOURS = [[1, 3, 2, 4], [0, 3, 2, 4], [4, 3, 0, 1], [1, 0, 2, 4], [2, 3, 0, 1]]


def random_matrix(rng, n_rows, n_cols, max_deg, values=(1.0,)):
    rows, data = [], []
    for _ in range(n_rows):
        k = int(rng.integers(0, max_deg + 1))
        rows.append(np.sort(rng.choice(n_cols, size=min(k, n_cols), replace=False)))
        data.append(rng.choice(values, size=len(rows[-1])))
    indptr = np.cumsum([0] + [len(r) for r in rows])
    return sp.csr_matrix((np.concatenate(data).astype(np.float32), np.concatenate(rows).astype(np.int64), indptr),
                         shape=(n_rows, n_cols))


@pytest.mark.parametrize("oracle", ["matrix", "literal"])
def test_known_answers(oracle):
    M = known_matrix()
    pairs = orc.matrix_sims(M, 1) if oracle == "matrix" else orc.literal_sims(M, 1)
    lists, count = orc.topk_lists(pairs, 5, 10)
    assert [ids.tolist() for ids, _ in lists] == KNOWN_NEIGHBOURS
    assert count.tolist() == [4] * 5
    # item 0 = (1, 1, 0, 0), item 1 = (2, 1, 0, 0): 3 / (sqrt 2 sqrt 5)
    np.testing.assert_allclose(lists[0][1][0], 3 / np.sqrt(10), rtol=1e-6)


def test_known_answer_of_compute_pred():
    # rust/src/inference.rs tests
    assert abs(orc.compute_pred("rating", [0.1, 0.2, 0.3], [2.0, 4.0, 1.0], np.float32) - 2.1666667) < 1e-4
    assert orc.compute_pred("ranking", [0.1, 0.2, 0.3], [2.0, 4.0, 1.0], np.float32) == np.float32(0.2)
    assert np.isnan(orc.compute_pred("rating", [0.0, 0.0], [1.0, 2.0]))      # a zero sum of sims


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("min_common", [1, 2, 3])
def test_literal_loop_and_matrix_oracle_agree(seed, min_common):
    rng = np.random.default_rng(seed)
    M = random_matrix(rng, 24, 15, 9, values=(-1.5, 0.0, 1.0, 2.5))
    a1, a2, ac = orc.literal_sims(M, min_common, dtype=np.float64)
    b1, b2, bc = orc.matrix_sims(M, min_common)
    assert len(a1) > 0 and (ac < 0).any()
    np.testing.assert_array_equal(a1, b1)
    np.testing.assert_array_equal(a2, b2)
    np.testing.assert_allclose(ac, bc, rtol=1e-12, atol=1e-15)
    _, _, c32 = orc.literal_sims(M, min_common)
    np.testing.assert_allclose(c32, bc, rtol=1e-5, atol=1e-6)


def serving_case():
    # R: 3 users x 4 items with a negative and a zero label; user 2 has an empty row
    R = sp.csr_matrix((np.array([2.0, -1.0, 0.0, 1.0], np.float32), np.array([0, 2, 1, 3]), np.array([0, 2, 4, 4])),
                      shape=(3, 4))
    item_lists = [(np.array([2, 1]), np.array([0.5, 0.0])), (np.array([3]), np.array([-0.25])),
                  (np.array([0]), np.array([0.5])), (np.array([1, 0]), np.array([0.75, -0.5]))]
    user_lists = [(np.array([1]), np.array([0.0])), (np.array([0]), np.array([0.0])), (np.array([]), np.array([]))]
    return R, item_lists, user_lists, {0: [0, 2], 1: [1, 3], 2: []}


def test_recommend_restatement_edge_cases():
    R, il, ul, consumed = serving_case()
    recs, no_rec, sc = orc.recommend(R, il, 2, consumed, [0, 1, 2, 9], 3, False, user_based=False)
    # user 0: item 0 (2.0) -> {2: 1.0, 1: 0.0}; item 2 (-1.0) -> {0: -0.5}
    assert sc[0] == {2: 1.0, 1: 0.0, 0: -0.5} and recs[0] == [2, 1, 0]
    # user 1: item 1 (0.0) -> {3: -0.0}; item 3 (1.0) -> {1: 0.75, 0: -0.5}
    assert sc[1] == {3: 0.0, 1: 0.75, 0: -0.5} and recs[1] == [1, 3, 0]
    assert no_rec == [2, 3]
    recs, no_rec, sc = orc.recommend(R, il, 2, consumed, [0, 1], 3, True, user_based=False)
    assert sc[0] == {1: 0.0} and sc[1] == {0: -0.5} and no_rec == []
    # UserCF: user 0's neighbour 1 has similarity 0: its items are candidates with score 0
    recs, no_rec, sc = orc.recommend(R, ul, 2, consumed, [0, 2], 5, False, user_based=True)
    assert sc[0] == {1: 0.0, 3: 0.0} and recs[0] == [1, 3] and no_rec == [1]


def test_predict_restatement_edge_cases():
    R, il, ul, _ = serving_case()
    # ItemCF (0, 3): neighbours 1 (not in row 0) and 0 (label 2, sim -0.5) -> rating 2, ranking -0.5
    assert orc.predict(R, il, 2, "rating", [0], [3], 9.0, False) == [2.0]
    assert orc.predict(R, il, 2, "ranking", [0], [3], 9.0, False) == [-0.5]
    # (0, 0): neighbours 2 (label -1, sim 0.5) and 1 (not in row 0) -> rating -1
    assert orc.predict(R, il, 2, "rating", [0], [0], 9.0, False) == [-1.0]
    # k_sim 1 cuts item 3's list to neighbour 1: empty intersection with row 0 -> default; OOV -> default
    assert orc.predict(R, il, 1, "rating", [0, 3, 0], [3, 0, 4], 9.0, False) == [9.0, 9.0, 9.0]
    # UserCF (0, 1): user 0's neighbour 1 holds item 1 (label 0) with sim 0 -> rating 0 * 0 / 0 = NaN
    got = orc.predict(R, ul, 2, "rating", [0, 0], [1, 0], 9.0, True)
    assert np.isnan(got[0]) and got[1] == 9.0


def _engine(cls="ItemCF", **kw):
    from librecommender_b200 import cf

    M = known_matrix()        # the item x user matrix of item_cf.rs's test: R is its transpose
    R = M.T.tocsr()
    args = dict(task="ranking", k_sim=10, n_users=4, n_items=5, min_common=1, user_interacts=R, item_interacts=M,
                user_consumed={0: [0, 1], 1: [0, 1]}, default_pred=0.0)
    args.update(kw)
    return getattr(cf, cls)(**args)


@pytest.mark.parametrize("cls", ["ItemCF", "UserCF"])
@pytest.mark.parametrize("kw, msg", [
    (dict(task="regression"), "task"), (dict(k_sim=0), "k_sim"), (dict(k_sim=4097), "k_sim"),
    (dict(k_sim=2.5), "k_sim"), (dict(k_sim=True), "k_sim"), (dict(min_common=0), "min_common"),
    (dict(min_common=1.5), "min_common"), (dict(n_users=3), "rows"), (dict(n_items=4), "outside"),
])
def test_validation_errors(cls, kw, msg):
    with pytest.raises(ValueError, match=msg):
        _engine(cls, **kw)


def test_validation_of_the_csrs():
    M = known_matrix()
    R = M.T.tocsr()
    bad = R.copy()
    bad.indices[[0, 1]] = bad.indices[[1, 0]]            # row 0 unsorted
    with pytest.raises(ValueError, match="sorted"):
        _engine(user_interacts=bad)
    relabelled = M.copy()
    relabelled.data[0] = 7.0                             # same pattern, another label
    with pytest.raises(ValueError, match="transpose"):
        _engine(item_interacts=relabelled)
    with pytest.raises(ValueError, match="outside"):
        _engine(user_interacts=sp.csr_matrix((np.ones(1, np.float32), [9], [0, 1, 1, 1, 1]), shape=(4, 10)))


def test_dropin_wiring_without_launch():
    import sys

    from oracle.ref_loader import load_reference, reference_available

    if not reference_available():
        pytest.skip("reference neither mounted nor staged")
    load_reference()
    import libreco
    from libreco.bases import cf_base_rs

    from librecommender_b200 import dropin

    original = cf_base_rs.RsCfBase.fit
    dropin.install(libreco, losses=False, lightgcn=False, cf=True)
    try:
        assert cf_base_rs.RsCfBase.fit is not original
        from libreco.algorithms import RsItemCF, RsUserCF

        assert RsItemCF.fit is cf_base_rs.RsCfBase.fit and RsUserCF.fit is cf_base_rs.RsCfBase.fit
        assert "recfarm" not in sys.modules
        model = type("M", (), {"incremental": True})()
        with pytest.raises(NotImplementedError):
            cf_base_rs.RsCfBase.fit(model, None, False)
    finally:
        dropin.uninstall()
    assert cf_base_rs.RsCfBase.fit is original
