"""ALS training on the GPU (``csrc/als.cu``, ``librecommender_b200.als``) against the Cython goldens
(``tests/golden/als.npz``) and the float64 oracle (``tests/_als_oracle.py``).

Tolerances: per row, the GPU's max-norm distance to the float64 oracle may be at most 4x the Cython float32
build's own distance on the same case, plus a floor of 2e-6 (1 + |x|).  The larger seeded cases (every row
class, d = 128) have no Cython run; their systems are well conditioned (Gaussian Y with n_y >> d) and the bound
there is 2e-5 (1 + |x|)."""
import numpy as np
import pytest
import scipy.sparse as sp

import _als_oracle as orc
from test_als_cpu import _golden, fit_golden, fit_rows, golden_case, oracle_fit

pytestmark = pytest.mark.gpu


def _lib_consts():
    from librecommender_b200 import _lib

    L = _lib.lib
    return L.b200_als_long_row_threshold(), L.b200_als_chunk(), L.b200_als_stage_rows


def _row_ok(got, ref, unit, floor=2e-6):
    dist = np.abs(got.astype(np.float64) - ref).max(axis=1)
    bound = 4 * unit + floor * (1 + np.abs(ref).max(axis=1))
    return dist <= bound, dist, bound


def test_base_matrix_within_float32_summation_bound():
    import torch

    from librecommender_b200.als import gram

    g = np.random.default_rng(5)
    for n_y, d in ((1, 1), (50, 7), (5000, 16), (70001, 64), (20000, 128)):
        Y = (g.standard_normal((n_y, d)) * 0.2).astype(np.float32)
        A0 = gram(torch.as_tensor(Y, device="cuda"), 0.75, True).cpu().numpy().astype(np.float64)
        Y64 = Y.astype(np.float64)
        ref = Y64.T @ Y64 + np.float32(0.75) * np.eye(d)
        # split-K tf32x3 products (relative error <= 2^-21 each) summed in float32 over n_y terms
        bound = (n_y + 16) * 2.0 ** -22 * (np.abs(Y64).T @ np.abs(Y64)) + 2.0 ** -22 * 0.75 + 1e-30
        assert (np.abs(A0 - ref) <= bound).all(), (n_y, d, np.abs(A0 - ref).max())
        expl = gram(torch.as_tensor(Y, device="cuda"), 0.75, False).cpu().numpy()
        assert np.array_equal(expl, np.float32(0.75) * np.eye(d, dtype=np.float32))


@pytest.mark.parametrize("i", range(32))
def test_golden_case(i):
    from librecommender_b200.als import als_update

    c = golden_case(_golden(), i)
    X = c["X0"].copy()
    als_update(c["csr"], X, c["Y"], c["reg"], c["task"], use_cg=c["use_cg"], cg_steps=c["steps"])
    ref, _ = orc.als_update(c["csr"], c["X0"], c["Y"], c["reg"], c["task"], c["use_cg"], c["steps"])
    ok, dist, bound = _row_ok(X, ref, c["cy_dev"])
    assert ok.all(), (dist, bound)
    if c["use_cg"] and c["steps"] == 0:     # no CG step: X is never written
        assert np.array_equal(X, c["X0"])


@pytest.mark.parametrize("task", ["ranking", "rating"])
def test_rsold_exit_leaves_rows_bitwise_unchanged(task):
    """Rows whose start is their exact solution in float32 arithmetic (unit-vector Y, values whose halves are
    exact): r = b - A x is exactly 0 in any summation order, so the rsold < 1e-10 exit must leave them alone."""
    from librecommender_b200.als import als_update

    d = 8
    Y = np.eye(d, dtype=np.float32)
    rows = [[0, 3], [1, 2, 5, 7], [4], [], [0, 1, 2, 3, 4, 5, 6, 7], [6, 2]]
    indices = np.concatenate([np.asarray(r, dtype=np.int32) for r in rows])
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int32)
    g = np.random.default_rng(3)
    if task == "ranking":      # c = 1, reg = 1: A = 2 I on the row's items, x = 1/2 there
        data = np.ones(indices.size, dtype=np.float32)
    else:                      # reg = 1: A = I + sum e_k e_k^T, x_k = r_k / 2
        data = g.integers(1, 6, size=indices.size).astype(np.float32)
    csr = sp.csr_matrix((data, indices, indptr), shape=(len(rows), d))
    X0 = np.zeros((len(rows), d), dtype=np.float32)
    for m, r in enumerate(rows):
        for j, k in enumerate(r):
            X0[m, k] = 0.5 if task == "ranking" else data[indptr[m] + j] / 2
    moved = [1, 4]                            # two rows start elsewhere and must move
    X0[moved] += np.float32(0.25)
    X = X0.copy()
    als_update(csr, X, Y, 1.0, task, use_cg=True, cg_steps=3)
    keep = [m for m in range(len(rows)) if m not in moved]
    assert np.array_equal(X[keep], X0[keep])
    assert not np.array_equal(X[moved], X0[moved])


def test_posv_failure_raises_the_reference_error():
    from librecommender_b200.als import als_update

    z = _golden()
    X0, Y = z["fail_X0"], z["fail_Y"]
    csr = sp.csr_matrix((z["fail_data"], z["fail_indices"], z["fail_indptr"]), shape=(X0.shape[0], Y.shape[0]))
    X = X0.copy()
    with pytest.raises(ValueError) as e:
        als_update(csr, X, Y, 0.0, "rating", use_cg=False)
    assert str(e.value) == str(z["fail_msg"])
    assert np.array_equal(X[2], X0[2])       # the failing row is not written


def _big_case(d, task, seed):
    thr, chunk, stage_rows = _lib_consts()
    g = np.random.default_rng(seed)
    n_y = 6000
    degs = [0, 1, 3, 17, stage_rows(d), stage_rows(d) + 1, stage_rows(d) + 40, thr - 1, thr, thr + 1,
            2 * chunk + 5, 5000, 9, 120, 0, 777]
    idx = [np.sort(g.choice(n_y, size=n, replace=False)).astype(np.int32) for n in degs]
    indptr = np.concatenate([[0], np.cumsum(degs)]).astype(np.int32)
    indices = np.concatenate(idx).astype(np.int32)
    if task == "ranking":
        data = (g.integers(1, 6, size=indices.size).astype(np.float32) * 10 + 1).astype(np.float32)
    else:
        data = g.integers(1, 6, size=indices.size).astype(np.float32)
    csr = sp.csr_matrix((data, indices, indptr), shape=(len(degs), n_y))
    X = (g.standard_normal((len(degs), d)) * 0.05).astype(np.float32)
    Y = (g.standard_normal((n_y, d)) * 0.1).astype(np.float32)
    return csr, X, Y


# (d, cg_steps): at d = 5 one step, because more steps bring some rows' residuals near the 1e-10 exit
@pytest.mark.parametrize("d,steps", [(5, 1), (12, 3), (32, 3), (64, 3), (128, 3)])
@pytest.mark.parametrize("task,use_cg", [("ranking", True), ("ranking", False), ("rating", True), ("rating", False)])
def test_every_row_class_against_the_oracle(d, steps, task, use_cg):
    from librecommender_b200.als import als_update

    csr, X0, Y = _big_case(d, task, seed=d)
    reg = 3.0
    ref, tested = orc.als_update(csr, X0, Y, reg, task, use_cg, steps)
    # no residual the exits test sits near 1e-10, where float32 and float64 could take different branches
    assert not np.any((tested > 1e-11) & (tested < 1e-9))
    X = X0.copy()
    als_update(csr, X, Y, reg, task, use_cg=use_cg, cg_steps=steps)
    ok, dist, bound = _row_ok(X, ref, 0.0, floor=2e-5)
    assert ok.all(), (dist, bound)
    X2 = X0.copy()                           # deterministic: the same call gives the same bits
    als_update(csr, X2, Y, reg, task, use_cg=use_cg, cg_steps=steps)
    assert np.array_equal(X, X2)


def _check_fit(z, csr, task, use_cg, U, I, dev_u, dev_i, rows_u, rows_i):
    """A fit's tables against the float64 oracle fit, per row within 4x the Cython fit's own distance plus
    1e-5 (1 + |x|); returns the oracle tables."""
    Uo, Io = oracle_fit(csr, task, use_cg)
    for got, ref, unit, rows in ((U, Uo, dev_u, rows_u), (I, Io, dev_i, rows_i)):
        ok, dist, bound = _row_ok(got, ref, unit, floor=1e-5)
        assert ok.all(), (dist.max(), bound[~ok][:5], dist[~ok][:5])
        # and the kept rows of the Cython's table within the same distance of ours
        keep = fit_rows(z, ref.shape[0])
        near = np.abs(got[keep] - rows).max(axis=1) <= 5 * unit[keep] + 1e-5 * (1 + np.abs(ref[keep]).max(axis=1))
        assert near.all()
    return Uo, Io


@pytest.mark.parametrize("task,use_cg", [("ranking", True), ("ranking", False), ("rating", True)])
def test_trainer_matches_update_loop_and_c1_golden(task, use_cg):
    import torch

    from librecommender_b200.als import ALSTrainer, als_update, initial_tables

    z = _golden()
    csr, dev_u, dev_i, rows_u, rows_i, _ = fit_golden(z, task, use_cg)
    data_before = csr.data.copy()
    tr = ALSTrainer(csr, task, 5.0, alpha=10, use_cg=use_cg, cg_steps=3, embed_size=16, seed=42).fit(2)
    assert np.array_equal(csr.data, data_before)          # the caller's matrix is never mutated
    U, I = (t.cpu().numpy() for t in tr.embeddings())
    # the same bits as the drop-in's host loop (ALS.fit with als_update)
    users = csr.copy()
    items = users.T.tocsr()
    if task == "ranking":
        users.data = users.data * 10 + 1
        items.data = items.data * 10 + 1
    Uh, Ih = initial_tables(csr.shape[0], csr.shape[1], 16, seed=42)
    for _ in range(2):
        als_update(users, Uh, Ih, 5.0, task, use_cg=use_cg)
        als_update(items, Ih, Uh, 5.0, task, use_cg=use_cg)
    assert np.array_equal(U[:-1], Uh) and np.array_equal(I[:-1], Ih)
    assert isinstance(tr.embeddings()[0], torch.Tensor) and tr.embeddings()[0].is_cuda
    _check_fit(z, csr, task, use_cg, U, I, dev_u, dev_i, rows_u, rows_i)


def test_trainer_rejects_bad_arguments():
    from librecommender_b200.als import ALSTrainer

    csr = sp.random(20, 10, density=0.3, format="csr", dtype=np.float32, random_state=0)
    with pytest.raises(ValueError):
        ALSTrainer(csr, "ranked", 1.0)
    with pytest.raises(ValueError):
        ALSTrainer(csr, "ranking", 1.0, cg_steps=-1)
    with pytest.raises(ValueError):
        ALSTrainer(csr, "ranking", 1.0, embed_size=200)
    with pytest.raises(ValueError):
        ALSTrainer(csr, "ranking", 1.0, user_embeds=np.zeros((19, 8), np.float32),
                   item_embeds=np.zeros((10, 8), np.float32))


def test_trainer_embeddings_serve_and_save(tmp_path):
    import types

    from librecommender_b200 import recommend_from_embedding, weights_io
    from librecommender_b200.als import ALSTrainer
    from oracle import ranking as rk

    csr, *_ = fit_golden(_golden(), "ranking", True)
    tr = ALSTrainer(csr, "ranking", 5.0).fit(1)
    U, I = tr.embeddings()
    n_u, n_i = csr.shape
    consumed = {u: csr.indices[csr.indptr[u]:csr.indptr[u + 1]].tolist() for u in range(n_u)}
    model = types.SimpleNamespace(task="ranking", n_items=n_i, n_users=n_u, user_consumed=consumed)
    users = list(range(0, n_u, 37))
    got = recommend_from_embedding(model, users, 10, U, I, True, False)
    Un, In = U.cpu().numpy(), I.cpu().numpy()
    ref = rk.recommend_from_embedding("ranking", users, 10, Un, In, n_i, consumed, True)
    assert rk.near_tie_mask(ref, got, rk.embed_scores(Un, In, users, n_i), 1e-6).all()
    weights_io.save_embed_model(str(tmp_path), "als", Un, In)
    Ul, Il = weights_io.load_embed_model(str(tmp_path), "als")
    assert np.array_equal(Ul, Un) and np.array_equal(Il, In)


def test_reference_als_fit_runs_on_the_dropin():
    """The reference's own ``ALS.fit`` / ``recommend_user`` with ``dropin.install(libreco, als=True)``."""
    import sys

    from oracle.ref_loader import load_reference, reference_available, sample_data_path

    if not reference_available():
        pytest.skip("reference neither mounted nor staged")
    import pandas as pd

    from librecommender_b200 import dropin
    from librecommender_b200 import als as gpu_als
    from oracle import ranking as rk

    libreco = load_reference()
    from libreco.data import DatasetPure, split_by_ratio_chrono

    before = sys.modules.get("libreco.algorithms._als")
    data = pd.read_csv(sample_data_path(), sep="::", names=["user", "item", "label", "time"], engine="python")
    train, _ = split_by_ratio_chrono(data, test_size=0.2)
    z = _golden()
    dropin.install(libreco, als=True)
    try:
        assert sys.modules["libreco.algorithms._als"].als_update is gpu_als.als_update
        from libreco.algorithms import ALS

        for task, use_cg in (("ranking", True), ("ranking", False), ("rating", True)):
            train_data, data_info = DatasetPure.build_trainset(train)
            csr, dev_u, dev_i, rows_u, rows_i, recs_cy = fit_golden(z, task, use_cg)
            model = ALS(task, data_info, embed_size=16, n_epochs=2, reg=5.0, alpha=10, use_cg=use_cg, seed=42)
            model.fit(train_data, neg_sampling=task == "ranking", verbose=0)
            # the oracle tables (float64 fit, OOV rows included) stand in for the Cython's tables: the goldens keep
            # only the Cython's distance to them per row
            Uo, Io = _check_fit(z, csr, task, use_cg, model.user_embeds_np, model.item_embeds_np, dev_u, dev_i,
                                rows_u, rows_i)
            n_i = data_info.n_items
            full = rk.embed_scores(Uo, Io, [model.n_users], n_i)
            assert rk.near_tie_mask(recs_cy[None, :], model.default_recs[None, :], full, 1e-4).all()
            if task != "ranking" or not use_cg:
                continue
            users = list(range(data_info.n_users))
            scores = rk.embed_scores(Uo, Io, users, n_i)
            for n in (7, 100):
                got = model.recommend_user(users, n, inner_id=True)
                g = np.stack([got[u] for u in users])
                ref = rk.recommend_from_embedding("ranking", users, n, Uo, Io, n_i, data_info.user_consumed, True)
                assert rk.near_tie_mask(ref, g, scores, 1e-4).all()
    finally:
        dropin.uninstall()
    assert sys.modules.get("libreco.algorithms._als") is before
