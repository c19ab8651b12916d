"""CPU checks of BPR training: the float64 oracle and the negative-stream replay against the Cython goldens
(``tests/golden/bpr.npz``), the device sampler's restatement, the initial tables, the host-side validation of
``bpr_update``, the C-ABI's rejections and the drop-in's module registration.  No device needed."""
import ctypes
import os
import sys

import numpy as np
import pytest
import scipy.sparse as sp

import _bpr_oracle as orc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "bpr.npz")


def _golden():
    return np.load(GOLDEN)


def golden_case(z, i):
    k = f"c{i}_"
    o, e, nt, epochs, seed = (int(v) for v in z[k + "meta"])
    opt = orc.OPTIMIZERS[o]
    U0, I0 = z[k + "U0"], z[k + "I0"]
    indptr, indices = z[k + "indptr"].astype(np.int32), z[k + "indices"].astype(np.int32)
    csr = sp.csr_matrix((np.ones(indices.size, np.float32), indices, indptr), shape=(U0.shape[0], I0.shape[0]))
    lr, reg = (float(v) for v in z[k + "lr_reg"])
    samples = [(z[f"{k}users{ep}"].astype(np.int32), z[f"{k}items{ep}"].astype(np.int32))
               for ep in range(1, epochs + 1)]
    states = {name: z[k + name] for name in orc.STATE_NAMES[opt]}
    return dict(opt=opt, embed=e, num_threads=nt, seed=seed, csr=csr, U0=U0, I0=I0, states=states, lr=lr, reg=reg,
                samples=samples, U=z[k + "U"], I=z[k + "I"], u_dev=z[k + "u_dev"], i_dev=z[k + "i_dev"])


def oracle_case(c):
    """The float64 oracle on a golden case, fed the Cython's replayed negatives; returns (U, I)."""
    U, I, st = c["U0"], c["I0"], c["states"]
    for ep, (users, items) in enumerate(c["samples"], start=1):
        negs = orc.reference_negatives(users, c["csr"].indptr, c["csr"].indices, c["I0"].shape[0], c["seed"],
                                       c["num_threads"])
        U, I, st = orc.update(c["opt"], users, items, negs, U, I, c["lr"], c["reg"], ep, st)
    return U, I


def fit_rows(z, n):
    return np.unique(np.r_[np.arange(0, n, int(z["fit_stride"])), n - 1])


def c1_data(z):
    """(train CSR, training users, items in the reference's order, eval users, eval items) of the C1 fits."""
    n_u, n_i = (int(v) for v in z["fit_shape"])
    users, items = z["fit_users"].astype(np.int32), z["fit_items"].astype(np.int32)
    csr = sp.csr_matrix((np.ones(users.size, np.float32), (users, items)), shape=(n_u, n_i))
    csr.sort_indices()
    return csr, users, items, z["fit_eval_users"].astype(np.int64), z["fit_eval_items"].astype(np.int64)


def reference_orders(z, users, items):
    """The reference's per-epoch sample orders: successive ``default_rng(42).permutation`` (``shuffle_data``)."""
    rng = np.random.default_rng(int(z["fit_rng_seed"]))
    out = []
    for _ in range(int(z["fit_epochs"])):
        perm = rng.permutation(range(users.size))
        out.append((users[perm], items[perm]))
    return out


def fit_golden(z, opt):
    k = f"fit_{opt}_"
    return dict(lr=float(z[k + "lr"]), user_dev=z[k + "user_dev"].astype(np.float64),
                item_dev=z[k + "item_dev"].astype(np.float64), user_rows=z[k + "user_rows"],
                item_rows=z[k + "item_rows"], default_recs=z[k + "default_recs"].astype(np.int64),
                metrics=z[k + "metrics"])


def oracle_fit(z, opt):
    """The float64 fit of the C1 golden from ``_build_model_cython``'s initial tables (seed 42, embed 16), with the
    mean rows appended."""
    from librecommender_b200.bpr import initial_tables

    csr, users, items, _, _ = c1_data(z)
    U0, I0 = initial_tables(csr.shape[0], csr.shape[1], 16, seed=42)
    U, I = U0, I0
    st = {name: np.zeros(U0.shape if name.startswith("u_") else I0.shape) for name in orc.STATE_NAMES[opt]}
    for ep, (u, it) in enumerate(reference_orders(z, users, items), start=1):
        negs = orc.reference_negatives(u, csr.indptr, csr.indices, csr.shape[1], 42, 1)
        U, I, st = orc.update(opt, u, it, negs, U, I, fit_golden(z, opt)["lr"], 0.0, ep, st)
    return np.vstack([U, U.mean(0)]), np.vstack([I, I.mean(0)])


def test_goldens_cover_the_issue_grid():
    z = _golden()
    cases = [golden_case(z, i) for i in range(int(z["n_cases"]))]
    assert {(c["opt"], c["embed"]) for c in cases} == {(o, e) for o in orc.OPTIMIZERS for e in (1, 7, 16, 64, 128)}
    assert {c["num_threads"] for c in cases} == {1, 3} and {len(c["samples"]) for c in cases} == {1, 2}
    for c in cases:
        deg = np.diff(c["csr"].indptr)
        users = np.concatenate([u for u, _ in c["samples"]])
        n_items = c["I0"].shape[0]
        assert deg[0] == 0 and deg[1] == n_items - 1 and {0, 1} <= set(users.tolist())
    assert os.path.getsize(GOLDEN) <= 600 * 1024


@pytest.mark.parametrize("i", range(15))
def test_oracle_reproduces_golden_case(i):
    c = golden_case(_golden(), i)
    U, I = oracle_case(c)
    for got, ref, dev in ((c["U"], U, c["u_dev"]), (c["I"], I, c["i_dev"])):
        dist = np.abs(got.astype(np.float64) - ref).max(axis=1)
        # the stored tolerance unit is the Cython's own float32 deviation from this oracle
        np.testing.assert_allclose(dist, dev, rtol=1e-9, atol=0)
        # float32-rounding distance: a wrong negative would move rows by the size of an update
        assert (dist <= 1e-5 * (1 + np.abs(ref).max(axis=1))).all(), dist
    assert np.all(c["U"][:, -1] == 1.0)


@pytest.mark.parametrize("opt", orc.OPTIMIZERS)
def test_oracle_fit_reproduces_the_c1_goldens(opt):
    z = _golden()
    f = fit_golden(z, opt)
    U, I = oracle_fit(z, opt)
    for ref, rows, dev in ((U, f["user_rows"], f["user_dev"]), (I, f["item_rows"], f["item_dev"])):
        assert dev.shape == (ref.shape[0],)
        keep = fit_rows(z, ref.shape[0])
        np.testing.assert_allclose(np.abs(rows.astype(np.float64) - ref[keep]).max(axis=1), dev[keep], rtol=1e-6,
                                   atol=0)
        assert (dev <= 1e-4 * (1 + np.abs(ref).max(axis=1))).all(), dev.max()
    recs = f["default_recs"]
    assert len(set(recs.tolist())) == recs.size == min(2000, I.shape[0] - 1)


@pytest.mark.parametrize("opt", orc.OPTIMIZERS)
def test_c1_golden_metrics_recompute_and_move(opt):
    from librecommender_b200.bpr import initial_tables

    z = _golden()
    csr, _, _, eu, ei = c1_data(z)
    f = fit_golden(z, opt)
    U, I = oracle_fit(z, opt)
    rec, ndcg = orc.ranking_metrics(U[:-1], I[:-1], csr.indptr, csr.indices, eu, ei)
    # the oracle tables give the Cython tables' metrics up to a swapped near-tie or two
    assert abs(rec - f["metrics"][0]) < 2e-3 and abs(ndcg - f["metrics"][1]) < 2e-3
    U0, I0 = initial_tables(csr.shape[0], csr.shape[1], 16, seed=42)
    r0 = orc.ranking_metrics(U0, I0, csr.indptr, csr.indices, eu, ei)
    assert np.allclose(r0, f["metrics"][2:], rtol=0, atol=1e-12)
    assert f["metrics"][0] > 1.5 * f["metrics"][2]          # three epochs visibly move recall@10


def test_reference_stream_replay_interleaves_generators():
    """Generator t = i % num_threads; every generator is mt19937((seed + 11 t) % 7) restarted per call."""
    indptr = np.array([0, 0, 3], dtype=np.int64)
    indices = np.array([1, 4, 5], dtype=np.int32)
    users = np.array([0, 1, 0, 0, 1, 1, 0], dtype=np.int32)
    a = orc.reference_negatives(users, indptr, indices, 9, seed=5, num_threads=3)
    for t in range(3):
        sub = users[t::3]
        ref = orc.reference_negatives(sub, indptr, indices, 9, seed=(5 + 11 * t) % 7, num_threads=1)
        assert np.array_equal(a[t::3], ref)
    assert not np.isin(a[users == 1], indices).any()
    # seeds that agree mod 7 give the same stream
    assert np.array_equal(orc.reference_negatives(users, indptr, indices, 9, 2, 1),
                          orc.reference_negatives(users, indptr, indices, 9, 9, 1))


def test_device_sampler_never_returns_a_consumed_item_and_is_uniform():
    from scipy.stats import chisquare

    g = np.random.default_rng(7)
    n_items = 40
    rows = [np.sort(g.choice(n_items, size=k, replace=False)) for k in (0, 1, 5, 20, 39, 12)]
    rows[4] = np.delete(np.arange(n_items), 17)         # misses one item: always item 17
    indptr = np.concatenate([[0], np.cumsum([r.size for r in rows])])
    indices = np.concatenate(rows).astype(np.int32)
    users = np.repeat(np.arange(len(rows)), 4000)
    negs = orc.device_negatives(users, indptr, indices, n_items, seed=123, epoch=2)
    for u, r in enumerate(rows):
        got = negs[users == u]
        assert not np.isin(got, r).any()
        free = np.setdiff1d(np.arange(n_items), r)
        assert np.isin(got, free).all()
        if free.size > 1:
            counts = np.array([(got == x).sum() for x in free])
            assert chisquare(counts).pvalue > 1e-3, (u, counts)
    assert (negs[users == 4] == 17).all()
    # the key is (seed, epoch, sample index): another epoch or seed gives another stream
    assert not np.array_equal(negs, orc.device_negatives(users, indptr, indices, n_items, seed=123, epoch=3))
    full = orc.device_negatives([0], np.array([0, 3]), np.array([0, 1, 2]), 3, seed=1, epoch=1)
    assert full.tolist() == [-1]


def test_device_draws_match_the_scalar_philox_restatement():
    from oracle.sampling import _draw

    m = np.array([7, 1, 3231, 10 ** 6, 2 ** 31 - 1, 5, 17, 99])
    got = orc.device_draws(m.size, seed=(1 << 40) + 77, epoch=3, m=m)
    want = [_draw(0, None, int(m[s]), (1 << 40) + 77, 3, s, 0) for s in range(m.size)]
    assert got.tolist() == want


def test_initial_tables_restate_build_model_cython():
    from librecommender_b200.bpr import initial_tables
    from oracle.ref_loader import load_reference, reference_available

    if not reference_available():
        pytest.skip("reference neither mounted nor staged")
    load_reference()
    from libreco.utils.initializers import truncated_normal

    rng = np.random.default_rng(42)
    U_ref = truncated_normal(rng, shape=(300, 17), mean=0.0, scale=0.03)
    U_ref[:, 16] = 1.0
    I_ref = truncated_normal(rng, shape=(200, 17), mean=0.0, scale=0.03)
    I_ref[:, 16] = 0.0
    U, I = initial_tables(300, 200, 16, seed=42)
    assert np.array_equal(U, U_ref) and np.array_equal(I, I_ref)


def _case(n_users=5, n_items=7, D=5):
    g = np.random.default_rng(0)
    rows = [[0, 2], [1], [], [3, 4, 6], [5]]
    indices = np.concatenate([np.asarray(r, dtype=np.int32) for r in rows])
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    csr = sp.csr_matrix((np.ones(indices.size, np.float32), indices, indptr), shape=(n_users, n_items))
    U = g.standard_normal((n_users, D)).astype(np.float32)
    I = g.standard_normal((n_items, D)).astype(np.float32)
    users = np.array([0, 1, 3, 4], dtype=np.int32)
    items = np.array([2, 1, 6, 5], dtype=np.int32)
    return csr, U, I, users, items


BAD = ["optimizer", "user_dtype", "item_dtype", "ids_len", "user_range", "item_range", "table_dtype", "table_order",
       "table_rows", "width", "embed0", "embed129", "momentum_state", "adam_state", "state_shape", "state_dtype",
       "adam_epoch", "indptr_len", "index_range", "unsorted", "duplicate", "full_row", "not_csr"]


@pytest.mark.parametrize("bad", BAD)
def test_bpr_update_rejects_bad_input_before_any_launch(bad):
    from librecommender_b200.bpr import bpr_update

    csr, U, I, users, items = _case()
    n_users, n_items = U.shape[0], I.shape[0]
    opt, kw, epoch = "sgd", {}, 1
    if bad == "optimizer":
        opt = "rmsprop"
    elif bad == "user_dtype":
        users = users.astype(np.int64)
    elif bad == "item_dtype":
        items = items.astype(np.float32)
    elif bad == "ids_len":
        items = items[:-1].copy()
    elif bad == "user_range":
        users[0] = n_users
    elif bad == "item_range":
        items[0] = -1
    elif bad == "table_dtype":
        U = U.astype(np.float64)
    elif bad == "table_order":
        I = np.asfortranarray(I)
    elif bad == "table_rows":
        U = U[:-1].copy()
    elif bad == "width":
        I = np.zeros((n_items, 4), np.float32)
    elif bad == "embed0":
        U, I = U[:, :1].copy(), I[:, :1].copy()
    elif bad == "embed129":
        U, I = np.zeros((n_users, 130), np.float32), np.zeros((n_items, 130), np.float32)
    elif bad == "momentum_state":
        opt, kw = "momentum", dict(u_velocity=np.zeros_like(U))
    elif bad == "adam_state":
        opt, kw = "adam", dict(u_1st_mom=np.zeros_like(U), i_1st_mom=np.zeros_like(I), u_2nd_mom=np.zeros_like(U))
    elif bad == "state_shape":
        opt, kw = "momentum", dict(u_velocity=np.zeros_like(U), i_velocity=np.zeros_like(U))
    elif bad == "state_dtype":
        opt, kw = "momentum", dict(u_velocity=np.zeros_like(U), i_velocity=np.zeros(I.shape))
    elif bad == "adam_epoch":
        opt, epoch = "adam", 0
        kw = dict(u_1st_mom=np.zeros_like(U), i_1st_mom=np.zeros_like(I), u_2nd_mom=np.zeros_like(U),
                  i_2nd_mom=np.zeros_like(I))
    elif bad == "indptr_len":
        csr = sp.csr_matrix(csr[:-1])
    elif bad == "index_range":
        csr = sp.csr_matrix((np.ones(2, np.float32), np.array([0, 9]), np.array([0, 2, 2, 2, 2, 2])),
                            shape=(n_users, 10))
    elif bad == "unsorted":
        csr = csr.copy()
        csr.indices[0], csr.indices[1] = csr.indices[1], csr.indices[0]
    elif bad == "duplicate":
        csr = csr.copy()
        csr.indices[1] = csr.indices[0]
    elif bad == "full_row":
        rows = [[0, 2], list(range(n_items)), [], [3, 4, 6], [5]]
        indices = np.concatenate([np.asarray(r, dtype=np.int32) for r in rows])
        indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
        csr = sp.csr_matrix((np.ones(indices.size, np.float32), indices, indptr), shape=(n_users, n_items))
    elif bad == "not_csr":
        csr = csr.toarray()
    before = [a.copy() for a in (U, I)]
    with pytest.raises(ValueError):
        bpr_update(opt, users, items, csr, U, I, 0.1, 0.01, n_users, n_items, 1, 42, epoch, **kw)
    assert all(np.array_equal(a, b) for a, b in zip((U, I), before))


def test_cabi_rejects_bad_arguments_without_a_device():
    from librecommender_b200 import _lib

    L = _lib.lib
    P, vp = ctypes.cast, ctypes.c_void_p
    ids = (ctypes.c_int32 * 2)(0, 1)
    ip = (ctypes.c_int64 * 3)(0, 1, 2)
    U = (ctypes.c_float * 600)()
    I = (ctypes.c_float * 600)()

    def call(opt=0, embed=4, users=True, table=True, s1=None, s2=None, epoch=1, inflight=0):
        return L.b200_bpr_update(opt, P(ids, vp) if users else None, P(ids, vp), 2, P(ip, vp), P(ids, vp), 2, 3,
                                 P(U, vp) if table else None, P(I, vp), embed, s1, s1, s2, s2, 0.1, 0.0, 0.9, 0.9,
                                 0.999, epoch, 42, None, None, inflight, None)

    for e in (0, 129, -1):
        assert call(embed=e) == -2
        assert b"embed size" in L.b200_last_error()
        assert L.b200_bpr_default_inflight(e) == 0
    assert call(opt=3) == -2 and b"optimizer" in L.b200_last_error()
    assert call(opt=-1) == -2
    assert call(users=False) == -2 and b"null" in L.b200_last_error()
    assert call(table=False) == -2
    assert call(opt=1) == -2 and b"momentum" in L.b200_last_error()
    assert call(opt=2, s1=P(U, vp)) == -2 and b"adam" in L.b200_last_error()
    assert call(opt=2, s1=P(U, vp), s2=P(U, vp), epoch=0) == -2
    assert call(inflight=-1) == -2


def test_dropin_registers_and_restores_the_bpr_and_als_modules():
    from oracle.ref_loader import load_reference, reference_available

    if not reference_available():
        pytest.skip("reference neither mounted nor staged")
    from librecommender_b200 import als as gpu_als
    from librecommender_b200 import bpr as gpu_bpr
    from librecommender_b200 import dropin

    libreco = load_reference()
    import libreco.algorithms as algos

    names = {"_als": gpu_als.als_update, "_bpr": gpu_bpr.bpr_update}
    before = {n: (sys.modules.get(f"libreco.algorithms.{n}"), getattr(algos, n, None)) for n in names}
    for flags in (dict(bpr=True), dict(als=True, bpr=True)):
        dropin.install(libreco, **flags)
        try:
            from libreco.algorithms._bpr import bpr_update       # what BPR._fit_cython does (bpr.py:309)

            assert bpr_update is gpu_bpr.bpr_update
            assert algos._bpr is sys.modules["libreco.algorithms._bpr"]
            if flags.get("als"):
                assert sys.modules["libreco.algorithms._als"].als_update is gpu_als.als_update
            else:
                assert sys.modules.get("libreco.algorithms._als") is before["_als"][0]
        finally:
            dropin.uninstall()
        for n in names:
            assert sys.modules.get(f"libreco.algorithms.{n}") is before[n][0]
            assert getattr(algos, n, None) is before[n][1]
