"""CPU checks of ALS training: the float64 oracle against the Cython goldens (``tests/golden/als.npz``), the
host-side validation of ``als_update``, the C-ABI's rejections and the row plan.  No device needed."""
import ctypes
import os
import types

import numpy as np
import pytest
import scipy.sparse as sp

import _als_oracle as orc

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "als.npz")


def _golden():
    return np.load(GOLDEN)


def golden_case(z, i):
    j, use_cg, steps = (int(v) for v in z[f"c{i}_meta"])
    g = f"g{j}_"
    d, implicit, reg = z[g + "meta"]
    X0, Y = z[g + "X0"], z[g + "Y"]
    csr = sp.csr_matrix((z[g + "data"], z[g + "indices"], z[g + "indptr"]), shape=(X0.shape[0], Y.shape[0]))
    return dict(csr=csr, X0=X0, Y=Y, X=z[f"c{i}_X"], cy_dev=z[f"c{i}_cy_dev"], d=int(d),
                task="ranking" if implicit else "rating", use_cg=bool(use_cg), steps=steps, reg=float(reg))


def fit_rows(z, n):
    """Rows of a fitted table the goldens keep: every ``fit_stride``-th one and the OOV (last) row."""
    return np.unique(np.r_[np.arange(0, n, int(z["fit_stride"])), n - 1])


def fit_golden(z, task, use_cg):
    """The C1 fit case: (unscaled CSR, per-row Cython distance to the float64 oracle for U and I, the kept rows
    of the Cython's U and I, default_recs)."""
    key = f"fit_{task}_{'cg' if use_cg else 'direct'}_"
    n_u, n_i = (int(v) for v in z["fit_shape"])
    indptr = z["fit_indptr"].astype(np.int64)
    planes = z["fit_index_gaps"].astype(np.int64)
    gaps = planes[0] + 256 * planes[1]
    csum = np.cumsum(gaps)
    deg = np.diff(indptr)
    starts = indptr[:-1][deg > 0]
    base = np.repeat(csum[starts] - gaps[starts], deg[deg > 0])   # running sum before each row's first gap
    indices = (csum - base).astype(np.int32)
    csr = sp.csr_matrix((z["fit_data"].astype(np.float32), indices, indptr.astype(np.int32)), shape=(n_u, n_i))
    return (csr, z[key + "user_dev"].astype(np.float64), z[key + "item_dev"].astype(np.float64),
            z[key + "user_rows"], z[key + "item_rows"], z[key + "default_recs"].astype(np.int64))


def oracle_fit(csr, task, use_cg):
    """The float64 fit from ``ALS.build_model``'s initial tables (seed 42, embed 16)."""
    from librecommender_b200.als import initial_tables

    U0, I0 = initial_tables(csr.shape[0], csr.shape[1], 16, seed=42)
    return orc.fit(csr, task, use_cg, U0, I0)


def test_goldens_cover_the_issue_grid():
    z = _golden()
    cases = [golden_case(z, i) for i in range(int(z["n_cases"]))]
    assert {c["d"] for c in cases} == {1, 7, 16, 64}
    assert {(c["task"], c["use_cg"], c["steps"]) for c in cases} >= {
        (t, cg, s) for t in ("ranking", "rating") for cg, s in ((False, 0), (True, 0), (True, 1), (True, 3))}
    degs = np.diff(cases[0]["csr"].indptr)
    assert 0 in degs and 1 in degs and degs.max() >= 200
    # the rsold exit: a CG case whose row 3 (started at its own solution) is left bitwise unchanged
    assert any(c["use_cg"] and c["steps"] > 0 and np.array_equal(c["X"][3], c["X0"][3]) for c in cases)


@pytest.mark.parametrize("i", range(32))
def test_oracle_reproduces_golden_case(i):
    z = _golden()
    c = golden_case(z, i)
    ref, _ = orc.als_update(c["csr"], c["X0"], c["Y"], c["reg"], c["task"], c["use_cg"], c["steps"])
    dev = np.abs(c["X"].astype(np.float64) - ref).max(axis=1)
    # the stored tolerance unit is the Cython's own float32 deviation from this oracle
    np.testing.assert_allclose(dev, c["cy_dev"], rtol=1e-9, atol=0)
    scale = 1 + np.abs(ref).max(axis=1)
    assert (dev <= 2e-5 * scale).all()
    if c["use_cg"] and c["steps"] == 0:
        assert np.array_equal(c["X"], c["X0"])


@pytest.mark.parametrize("task,use_cg", [("ranking", True), ("ranking", False), ("rating", True)])
def test_oracle_fit_reproduces_the_c1_goldens(task, use_cg):
    z = _golden()
    csr, dev_u, dev_i, rows_u, rows_i, recs = fit_golden(z, task, use_cg)
    assert csr.has_sorted_indices and csr.nnz > 50_000 and csr.data.min() >= 1
    U, I = oracle_fit(csr, task, use_cg)
    assert dev_u.shape == (U.shape[0],) and dev_i.shape == (I.shape[0],)
    for ref, rows, dev in ((U, rows_u, dev_u), (I, rows_i, dev_i)):
        keep = fit_rows(z, ref.shape[0])
        np.testing.assert_allclose(np.abs(rows.astype(np.float64) - ref[keep]).max(axis=1), dev[keep], rtol=1e-6,
                                   atol=0)
        assert (dev <= 2e-4 * (1 + np.abs(ref).max(axis=1))).all()
    assert recs.shape == (min(2000, csr.shape[1]),) and len(set(recs.tolist())) == recs.size


def test_oracle_raises_the_reference_posv_error():
    z = _golden()
    X0, Y = z["fail_X0"], z["fail_Y"]
    csr = sp.csr_matrix((z["fail_data"], z["fail_indices"], z["fail_indptr"]), shape=(X0.shape[0], Y.shape[0]))
    with pytest.raises(ValueError) as e:
        orc.als_update(csr, X0, Y, 0.0, "rating", use_cg=False)
    assert str(e.value) == str(z["fail_msg"])
    assert "err=1) on row 2." in str(e.value)


def test_initial_tables_restate_build_model():
    from librecommender_b200.als import initial_tables
    from oracle.ref_loader import load_reference, reference_available

    if not reference_available():
        pytest.skip("reference neither mounted nor staged")
    load_reference()
    from libreco.utils.initializers import truncated_normal

    rng = np.random.default_rng(42)
    U_ref = truncated_normal(rng, shape=[300, 16], mean=0.0, scale=0.03)
    I_ref = truncated_normal(rng, shape=[200, 16], mean=0.0, scale=0.03)
    U, I = initial_tables(300, 200, 16, seed=42)
    assert np.array_equal(U, U_ref) and np.array_equal(I, I_ref)


def _case(n_x=5, n_y=7, d=4):
    g = np.random.default_rng(0)
    csr = sp.random(n_x, n_y, density=0.5, format="csr", dtype=np.float32, random_state=1)
    return csr, g.standard_normal((n_x, d)).astype(np.float32), g.standard_normal((n_y, d)).astype(np.float32)


@pytest.mark.parametrize("bad", ["task", "steps", "x_dtype", "x_order", "width", "d0", "d129", "indptr_len",
                                 "indptr_order", "index_range", "data_dtype", "nnz"])
def test_als_update_rejects_bad_input_before_any_launch(bad):
    from librecommender_b200.als import als_update

    csr, X, Y = _case()
    kw = dict(reg=1.0, task="ranking", use_cg=True, cg_steps=3)
    if bad == "task":
        kw["task"] = "ranked"
    elif bad == "steps":
        kw["cg_steps"] = -1
    elif bad == "x_dtype":
        X = X.astype(np.float64)
    elif bad == "x_order":
        X = np.asfortranarray(X)
    elif bad == "width":
        Y = np.zeros((Y.shape[0], 5), np.float32)
    elif bad == "d0":
        X, Y = X[:, :0].copy(), Y[:, :0].copy()
    elif bad == "d129":
        X, Y = np.zeros((X.shape[0], 129), np.float32), np.zeros((Y.shape[0], 129), np.float32)
    elif bad == "indptr_len":
        X = np.zeros((X.shape[0] + 1, X.shape[1]), np.float32)
    elif bad == "indptr_order":
        csr = csr.copy()
        csr.indptr[2], csr.indptr[3] = csr.indptr[3], csr.indptr[2]
    elif bad == "index_range":
        Y = Y[:3].copy()
    elif bad == "data_dtype":
        csr = csr.astype(np.float64)
    elif bad == "nnz":
        csr = types.SimpleNamespace(indptr=csr.indptr, indices=csr.indices[:-1], data=csr.data[:-1])
    X_before = X.copy()
    with pytest.raises(ValueError):
        als_update(csr, X, Y, **kw)
    assert np.array_equal(X, X_before)


def test_cabi_rejects_unsupported_shapes_without_a_device():
    from librecommender_b200 import _lib

    L = _lib.lib
    n = ctypes.c_size_t(0)
    for d in (0, 129, -3):
        assert L.b200_als_workspace_bytes(d, 1, 0, 0, ctypes.byref(n)) == -2
        assert L.b200_als_stage_rows(d) == 0
    assert L.b200_als_workspace_bytes(16, 1, 2, 9, ctypes.byref(n)) == 0
    assert n.value >= (9 * 16 + 2 * (3 * 16 + 2)) * 4
    assert L.b200_als_workspace_bytes(16, 0, 2, 9, ctypes.byref(n)) == 0
    assert n.value >= 9 * (16 * 16 + 16) * 4 + 8
    assert L.b200_als_stage_rows(64) >= 32 and L.b200_als_chunk() > 0
    assert L.b200_als_long_row_threshold() >= L.b200_als_chunk()
    ws = (ctypes.c_float * 64)()
    ip = (ctypes.c_int64 * 3)(0, 0, 0)
    rows = (ctypes.c_int32 * 2)(0, 1)
    A0 = (ctypes.c_float * 4)()
    X = (ctypes.c_float * 4)()
    row, info = ctypes.c_int64(0), ctypes.c_int32(0)
    P = ctypes.cast
    vp = ctypes.c_void_p
    common = lambda d, n_x, n_short: (P(ip, vp), None, None, n_x, P(X, vp), P(X, vp), 2, d, P(A0, vp), 1)  # noqa: E731
    plan = (P(rows, vp), 2, None, None, 0, None, None, 0, P(ws, vp), 256)
    for d in (0, 129):
        assert L.b200_als_cg(*common(d, 2, 2), 3, *plan, None) == -2
        assert L.b200_als_direct(*common(d, 2, 2), *plan, ctypes.byref(row), ctypes.byref(info), None) == -2
        assert b"embed size" in L.b200_last_error()
    # the row plan must cover every row: n_short + n_long == n_x
    assert L.b200_als_cg(*common(2, 3, 2), 3, *plan, None) == -2
    assert b"row counts" in L.b200_last_error()
    # a long row without its chunk lists
    bad_plan = (P(rows, vp), 1, P(rows, vp), None, 1, None, None, 0, P(ws, vp), 256)
    assert L.b200_als_cg(*common(2, 2, 1), 3, *bad_plan, None) == -2
    # negative step count, workspace too small
    assert L.b200_als_cg(*common(2, 2, 2), -1, *plan, None) == -2
    small = (P(rows, vp), 2, None, None, 0, None, None, 0, P(ws, vp), 8)
    assert L.b200_als_direct(*common(2, 2, 2), *small, ctypes.byref(row), ctypes.byref(info), None) == -2


def test_row_plan_classes_and_chunks():
    import torch

    from librecommender_b200 import _lib
    from librecommender_b200.als import RowPlan

    thr, chunk = _lib.lib.b200_als_long_row_threshold(), _lib.lib.b200_als_chunk()
    degs = np.array([0, 3, thr, thr + 1, 0, 5 * chunk + 7, 2 * thr])
    indptr = np.concatenate([[0], np.cumsum(degs)]).astype(np.int64)
    nnz = int(indptr[-1])
    plan = RowPlan(torch.as_tensor(indptr), torch.zeros(nnz, dtype=torch.int32), torch.ones(nnz), 10)
    assert plan.short_rows.tolist() == [0, 1, 2, 4]
    assert plan.long_rows.tolist() == [3, 5, 6]
    want = [-(-int(degs[r]) // chunk) for r in (3, 5, 6)]
    assert np.diff(plan.long_chunk_ptr.numpy()).tolist() == want and plan.n_chunks == sum(want)
    owner = np.repeat(np.arange(3), want)
    assert plan.chunk_long.tolist() == owner.tolist()
    assert plan.chunk_k.tolist() == [k for n in want for k in range(n)]
    for c in range(plan.n_chunks):    # the chunks of a long row tile its nnz exactly
        r = int(plan.long_rows[owner[c]])
        beg = indptr[r] + plan.chunk_k[c].item() * chunk
        assert indptr[r] <= beg < indptr[r + 1]


def test_dropin_registers_and_restores_the_als_module():
    import sys

    from oracle.ref_loader import load_reference, reference_available

    if not reference_available():
        pytest.skip("reference neither mounted nor staged")
    from librecommender_b200 import als as gpu_als
    from librecommender_b200 import dropin

    libreco = load_reference()
    import libreco.algorithms as algos

    name = "libreco.algorithms._als"
    before_mod, before_attr = sys.modules.get(name), getattr(algos, "_als", None)
    dropin.install(libreco, als=True)
    try:
        assert sys.modules[name].als_update is gpu_als.als_update
        assert algos._als is sys.modules[name]
        from libreco.algorithms._als import als_update      # what ALS.fit does (als.py:135)

        assert als_update is gpu_als.als_update
    finally:
        dropin.uninstall()
    assert sys.modules.get(name) is before_mod
    assert getattr(algos, "_als", None) is before_attr
