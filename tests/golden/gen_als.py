"""Golden vectors for ALS training from the UNMODIFIED reference: ``libreco/algorithms/_als.pyx`` compiled with
Cython (serial: no OpenMP, so ``prange`` is a plain loop; every row is solved independently, so the result does
not depend on the thread count) into a temporary directory, and the reference's own ``ALS.fit`` on C1.

    python tests/golden/gen_als.py

Groups ``g{j}_*``: a seeded CSR with rows of 0, 1, a few and a few hundred nnz, X0 and Y, for d in {1, 7, 16, 64}
and both tasks.  Cases ``c{i}_*``: ``als_update`` on one group with the direct solve or CG with cg_steps in
{0, 1, 3}: the output and, per row, its distance to the float64 oracle.  Row 3 starts at its own
solution (the rsold exit of CG).  ``fail_*``: the direct explicit solve with reg = 0 and an empty row 2 (posv
info = 1 there), with the exception text.  ``fit_*``: ``ALS(embed_size=16, n_epochs=2, reg=5.0, seed=42).fit``
on C1's chronological 80 % split for ranking/CG, ranking/direct and rating/CG: per row of the final tables (OOV
rows included) the distance to the float64 oracle fit from the same initial tables, every 8th row of the tables
themselves, and ``default_recs``.  The C1 matrix is stored as the byte planes of the uint16 gaps between item ids within a row and uint8 labels (all integers).  Only outputs are written: no source, no binary.
"""
import importlib
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np
import scipy.sparse as sp

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle.ref_loader import REFERENCE_ROOT, load_reference, sample_data_path  # noqa: E402
import _als_oracle  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
DIMS = (1, 7, 16, 64)
FIT_CASES = (("ranking", True), ("ranking", False), ("rating", True))
FIT_STRIDE = 32


def fit_rows(n):
    """Rows of a fitted table kept in the file: every FIT_STRIDE-th one and the OOV (last) row."""
    return np.unique(np.r_[np.arange(0, n, FIT_STRIDE), n - 1])


def model_initial_tables(shape, seed):
    """``ALS.build_model``'s tables (``als.py:84-91``), drawn with the reference's own initializer."""
    from libreco.utils.initializers import truncated_normal

    rng = np.random.default_rng(seed)
    return (truncated_normal(rng, shape=[shape[0], 16], mean=0.0, scale=0.03),
            truncated_normal(rng, shape=[shape[1], 16], mean=0.0, scale=0.03))


def build_cython(tmp):
    """Compile the reference's _als.pyx (no OpenMP) in ``tmp``; return the imported module."""
    shutil.copy(os.path.join(REFERENCE_ROOT, "libreco", "algorithms", "_als.pyx"), tmp)
    setup = ("from setuptools import setup, Extension\nfrom Cython.Build import cythonize\nimport numpy\n"
             "setup(ext_modules=cythonize([Extension('_als', ['_als.pyx'], include_dirs=[numpy.get_include()])],"
             " quiet=True), script_args=['build_ext', '--inplace'])\n")
    with open(os.path.join(tmp, "setup_als.py"), "w") as f:
        f.write(setup)
    subprocess.run([sys.executable, "setup_als.py"], cwd=tmp, check=True, capture_output=True)
    sys.path.insert(0, tmp)
    return importlib.import_module("_als")


def quantize(a):
    return (np.round(np.asarray(a) * 4096) / 4096).astype(np.float32)


def encode_indices(csr):
    """Column ids as gaps within each row (the first gap of a row is its first id), uint16 stored as its low and
    high byte planes [2, nnz], which compress far better than the interleaved bytes."""
    gaps = np.diff(csr.indices.astype(np.int64), prepend=0)
    gaps[csr.indptr[:-1][np.diff(csr.indptr) > 0]] = csr.indices[csr.indptr[:-1][np.diff(csr.indptr) > 0]]
    assert gaps.min() >= 0 and gaps.max() < 1 << 16
    return np.stack([gaps & 0xFF, gaps >> 8]).astype(np.uint8)


def make_case(g, d, task, n_x=12, n_y=400):
    degs = np.array([0, 1, 5, 5, 300, 37, 2, 250, 0, 64, 3, 180])[:n_x]
    rows = []
    for n in degs:
        rows.append(np.sort(g.choice(n_y, size=int(n), replace=False)).astype(np.int32))
    indptr = np.concatenate([[0], np.cumsum(degs)]).astype(np.int32)
    indices = np.concatenate(rows).astype(np.int32)
    if task == "ranking":
        raw = g.integers(1, 6, size=indices.size).astype(np.float32)
        data = raw * 10 + 1
    else:
        data = g.integers(1, 6, size=indices.size).astype(np.float32)
    csr = sp.csr_matrix((data.astype(np.float32), indices, indptr), shape=(n_x, n_y))
    # inputs on a 2^-12 grid: exact float32 values whose zero low mantissa bits keep the file small
    X = quantize(g.standard_normal((n_x, d)) * 0.03)
    Y = quantize(g.standard_normal((n_y, d)) * (0.3 if task == "ranking" else 0.6))
    reg = 2.0 if task == "ranking" else 1.5
    # row 3 starts at its own solution: r = b - A x is rounding noise, below the 1e-10 exit
    implicit = task == "ranking"
    A0 = _als_oracle.base_matrix(Y, reg, implicit)
    idx, val = csr.indices[csr.indptr[3]:csr.indptr[4]], csr.data[csr.indptr[3]:csr.indptr[4]].astype(np.float64)
    Yr = Y[idx].astype(np.float64)
    w = val - 1 if implicit else np.ones_like(val)
    X[3] = np.linalg.solve(A0 + (Yr * w[:, None]).T @ Yr, Yr.T @ val).astype(np.float32)
    return csr, X, Y, reg


def update_cases(cy):
    """Group j (one per (d, task)) holds the inputs; case i holds one solver's output on its group."""
    g = np.random.default_rng(2024)
    out, i, j = {}, 0, 0
    for d in DIMS:
        for task in ("ranking", "rating"):
            csr, X0, Y, reg = make_case(g, d, task)
            out.update({f"g{j}_indptr": csr.indptr, f"g{j}_indices": csr.indices, f"g{j}_data": csr.data,
                        f"g{j}_X0": X0, f"g{j}_Y": Y,
                        f"g{j}_meta": np.array([d, task == "ranking", reg], dtype=np.float64)})
            for use_cg, steps in ((False, 0), (True, 0), (True, 1), (True, 3)):
                X = X0.copy()
                cy.als_update(csr, X, Y, reg, task, use_cg=use_cg, num_threads=1, cg_steps=steps)
                ref, _ = _als_oracle.als_update(csr, X0, Y, reg, task, use_cg, steps)
                out.update({f"c{i}_X": X, f"c{i}_cy_dev": np.abs(X.astype(np.float64) - ref).max(axis=1),
                            f"c{i}_meta": np.array([j, use_cg, steps], dtype=np.int64)})
                i += 1
            j += 1
    out["n_cases"] = np.int64(i)
    # posv failure: explicit, direct, reg = 0, row 2 empty -> A = 0 -> info = 1
    d, n_x, n_y = 16, 6, 100
    degs = [30, 25, 0, 40, 20, 33]
    indices = np.concatenate([np.sort(g.choice(n_y, size=n, replace=False)) for n in degs]).astype(np.int32)
    indptr = np.concatenate([[0], np.cumsum(degs)]).astype(np.int32)
    data = g.integers(1, 6, size=indices.size).astype(np.float32)
    csr = sp.csr_matrix((data, indices, indptr), shape=(n_x, n_y))
    X0 = quantize(g.standard_normal((n_x, d)) * 0.03)
    Y = quantize(g.standard_normal((n_y, d)))
    try:
        cy.als_update(csr, X0.copy(), Y, 0.0, "rating", use_cg=False)
        raise SystemExit("expected the posv failure")
    except ValueError as e:
        msg = str(e)
    out.update({"fail_indptr": indptr, "fail_indices": indices, "fail_data": data, "fail_X0": X0, "fail_Y": Y,
                "fail_msg": np.array(msg)})
    return out


def fit_cases(cy):
    import pandas as pd

    load_reference()
    import libreco.algorithms as algos

    sys.modules["libreco.algorithms._als"] = cy
    algos._als = cy
    from libreco.algorithms import ALS
    from libreco.data import DatasetPure, split_by_ratio_chrono

    out = {}
    data = pd.read_csv(sample_data_path(), sep="::", names=["user", "item", "label", "time"], engine="python")
    train, _ = split_by_ratio_chrono(data, test_size=0.2)
    for task, use_cg in FIT_CASES:
        train_data, data_info = DatasetPure.build_trainset(train)   # fit rescales sparse_interaction in place
        key = f"fit_{task}_{'cg' if use_cg else 'direct'}_"
        csr = train_data.sparse_interaction.copy()      # the same unscaled matrix for every case
        assert csr.shape[1] < 1 << 16 and np.array_equal(csr.data, np.round(csr.data)) and csr.data.max() < 256
        out.update({"fit_indptr": csr.indptr.astype(np.int32), "fit_index_gaps": encode_indices(csr),
                    "fit_data": csr.data.astype(np.uint8), "fit_shape": np.array(csr.shape, dtype=np.int64)})
        model = ALS(task, data_info, embed_size=16, n_epochs=2, reg=5.0, alpha=10, use_cg=use_cg, n_threads=1,
                    seed=42)
        model.fit(train_data, neg_sampling=task == "ranking", verbose=0)
        U0, I0 = model_initial_tables(csr.shape, model.seed)
        Uo, Io = _als_oracle.fit(csr, task, use_cg, U0, I0)
        for side, cy, ref in (("user", model.user_embeds_np, Uo), ("item", model.item_embeds_np, Io)):
            # every row's distance to the float64 oracle (the tolerance unit), and every FIT_STRIDE-th row of the
            # table itself plus the OOV row
            out[key + side + "_dev"] = np.abs(cy.astype(np.float64) - ref).max(axis=1).astype(np.float32)
            out[key + side + "_rows"] = cy[fit_rows(cy.shape[0])]
        out[key + "default_recs"] = model.default_recs.astype(np.int32)
    out["fit_stride"] = np.int64(FIT_STRIDE)
    return out


if __name__ == "__main__":
    tmp = tempfile.mkdtemp(prefix="als_cython_")
    try:
        cy = build_cython(tmp)
        out = update_cases(cy)
        out.update(fit_cases(cy))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    np.savez_compressed(os.path.join(OUT, "als.npz"), **out)
    print("wrote als.npz", len(out), "arrays")
