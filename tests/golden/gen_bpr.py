"""Golden vectors for BPR training from the UNMODIFIED reference: ``libreco/algorithms/_bpr.pyx`` compiled with
Cython and g++ 13.3 (serial: no OpenMP, so ``prange`` is a plain loop and sample i draws from generator
i % num_threads; the result is deterministic) into a temporary directory, and the reference's own
``BPR(use_tf=False).fit`` on C1.  Other compilers are refused: the negatives come from libstdc++'s
``uniform_int_distribution``, which ``tests/_bpr_oracle.py`` restates for this version.

    python tests/golden/gen_bpr.py

Cases ``c{i}_*``: ``bpr_update`` for each optimizer and embed size in {1, 7, 16, 64, 128}, with num_threads in
{1, 3} and 1 or 2 epochs in rotation, on a seeded CSR of 8 users x 24 items where user 0's row is empty and user 1's
misses one item; inputs on a 2^-12 grid.  Stored: the inputs, the output tables and, per row, their distance to
the float64 oracle fed the replayed negatives.  ``fit_{opt}_*``: ``BPR(use_tf=False, embed_size=16, n_epochs=3,
lr=lr_o, optimizer=o, seed=42).fit`` on C1's chronological 80 % split: per row the distance to the oracle fit,
every ``fit_stride``-th row, ``default_recs``, ``lr``, and recall@10 / ndcg@10 on the 20 % split
(``_bpr_oracle.ranking_metrics``).  The training rows in the order the reference feeds them (``fit_users``,
``fit_items``; its per-epoch shuffles are ``default_rng(fit_rng_seed).permutation``, checked here) and the
evaluation pairs are stored as integers.  Only outputs are written: no source, no binary.
"""
import importlib
import os
import shutil
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle.ref_loader import REFERENCE_ROOT, load_reference, sample_data_path  # noqa: E402
import _bpr_oracle as orc  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
GXX = "13.3.0"
DIMS = (1, 7, 16, 64, 128)
SCHEDULES = ((1, 1), (3, 2), (1, 2), (3, 1))       # (num_threads, epochs), in rotation over the cases
CASE_LR = {"sgd": 0.0625, "momentum": 0.03125, "adam": 0.015625}
REG = 0.0078125
FIT_LR = {"sgd": 0.05, "momentum": 0.01, "adam": 0.005}
FIT_EPOCHS = 3
FIT_STRIDE = 64
N_USERS, N_ITEMS, N_SAMPLES = 8, 24, 48


def fit_rows(n):
    """Rows of a fitted table kept in the file: every FIT_STRIDE-th one and the OOV (last) row."""
    return np.unique(np.r_[np.arange(0, n, FIT_STRIDE), n - 1])


def build_cython(tmp):
    """Compile the reference's _bpr.pyx (no OpenMP) in ``tmp``; return the imported module."""
    ver = subprocess.run(["g++", "-dumpfullversion"], capture_output=True, text=True, check=True).stdout.strip()
    if ver != GXX:
        raise SystemExit(f"g++ {ver}: the negative-stream replay is written for g++ {GXX}'s libstdc++")
    shutil.copy(os.path.join(REFERENCE_ROOT, "libreco", "algorithms", "_bpr.pyx"), tmp)
    setup = ("from setuptools import setup, Extension\nfrom Cython.Build import cythonize\nimport numpy\n"
             "setup(ext_modules=cythonize([Extension('_bpr', ['_bpr.pyx'], language='c++',"
             " include_dirs=[numpy.get_include()])], quiet=True), script_args=['build_ext', '--inplace'])\n")
    with open(os.path.join(tmp, "setup_bpr.py"), "w") as f:
        f.write(setup)
    env = dict(os.environ, CC="gcc", CXX="g++")
    subprocess.run([sys.executable, "setup_bpr.py"], cwd=tmp, check=True, capture_output=True, env=env)
    sys.path.insert(0, tmp)
    return importlib.import_module("_bpr")


def quantize(a):
    return (np.round(np.asarray(a) * 4096) / 4096).astype(np.float32)


def make_csr(g):
    rows = [np.array([], dtype=np.int32), np.delete(np.arange(N_ITEMS), g.integers(N_ITEMS)).astype(np.int32)]
    for _ in range(N_USERS - 2):
        rows.append(np.sort(g.choice(N_ITEMS, size=int(g.integers(2, 9)), replace=False)).astype(np.int32))
    indptr = np.concatenate([[0], np.cumsum([r.size for r in rows])]).astype(np.int32)
    return indptr, np.concatenate(rows).astype(np.int32)


def make_samples(g, indptr, indices, seed, num_threads):
    """Samples over every user (user 0 and 1 included); a positive is in the user's row, except for the empty user 0,
    whose positive is any item but the one its negative will be (so no sample updates one item row twice)."""
    users = g.integers(0, N_USERS, size=N_SAMPLES).astype(np.int32)
    users[:2] = (0, 1)
    g.shuffle(users)
    negs = orc.reference_negatives(users, indptr, indices, N_ITEMS, seed, num_threads)
    items = np.empty(N_SAMPLES, dtype=np.int32)
    for i, u in enumerate(users.tolist()):
        row = indices[indptr[u]:indptr[u + 1]]
        if row.size:
            items[i] = g.choice(row)
        else:
            items[i] = g.choice(np.setdiff1d(np.arange(N_ITEMS), [negs[i]]))
    return users, items


def update_cases(cy):
    import scipy.sparse as sp

    g = np.random.default_rng(2025)
    out, i = {}, 0
    for opt in orc.OPTIMIZERS:
        for e in DIMS:
            nt, epochs = SCHEDULES[i % len(SCHEDULES)]
            D, seed = e + 1, int(g.integers(0, 100))
            indptr, indices = make_csr(g)
            csr = sp.csr_matrix((np.ones(indices.size, np.float32), indices, indptr), shape=(N_USERS, N_ITEMS))
            U0 = quantize(g.standard_normal((N_USERS, D)) * 0.1)
            U0[:, e] = 1.0
            I0 = quantize(g.standard_normal((N_ITEMS, D)) * 0.1)
            st0 = {}
            for name in orc.STATE_NAMES[opt]:
                rows = N_USERS if name.startswith("u_") else N_ITEMS
                a = g.standard_normal((rows, D)) * 0.01
                # second moments at least 1e-3: sqrt(h) stays well above the size of a moment update
                st0[name] = quantize(1e-3 + np.abs(a) * 0.2 if "2nd" in name else a)
                if name.startswith("u_"):
                    st0[name][:, e] = 0.0
            U, I, st = U0.copy(), I0.copy(), {k: v.copy() for k, v in st0.items()}
            Uo, Io, sto = U0, I0, st0
            key = f"c{i}_"
            for ep in range(1, epochs + 1):
                users, items = make_samples(g, indptr, indices, seed, nt)
                cy.bpr_update(opt, users, items, csr, U, I, CASE_LR[opt], REG, N_USERS, N_ITEMS, nt, seed, ep,
                              **st)
                negs = orc.reference_negatives(users, indptr, indices, N_ITEMS, seed, nt)
                Uo, Io, sto = orc.update(opt, users, items, negs, Uo, Io, CASE_LR[opt], REG, ep, sto)
                out.update({f"{key}users{ep}": users.astype(np.uint8), f"{key}items{ep}": items.astype(np.uint8)})
            assert np.all(U[:, e] == 1.0)
            out.update({key + "indptr": indptr.astype(np.uint8), key + "indices": indices.astype(np.uint8),
                        key + "U0": U0, key + "I0": I0, key + "U": U, key + "I": I,
                        key + "u_dev": np.abs(U - Uo).max(axis=1), key + "i_dev": np.abs(I - Io).max(axis=1),
                        key + "meta": np.array([orc.OPTIMIZERS.index(opt), e, nt, epochs, seed], dtype=np.int64),
                        key + "lr_reg": np.array([CASE_LR[opt], REG])})
            out.update({key + name: v for name, v in st0.items()})
            i += 1
    out["n_cases"] = np.int64(i)
    return out


def fit_cases(cy):
    import pandas as pd

    load_reference()
    import libreco.algorithms as algos

    sys.modules["libreco.algorithms._bpr"] = cy
    algos._bpr = cy
    from libreco.algorithms import BPR
    from libreco.data import DatasetPure, split_by_ratio_chrono

    data = pd.read_csv(sample_data_path(), sep="::", names=["user", "item", "label", "time"], engine="python")
    train, test = split_by_ratio_chrono(data, test_size=0.2)
    out = {}
    for opt in orc.OPTIMIZERS:
        train_data, data_info = DatasetPure.build_trainset(train)
        eval_data = DatasetPure.build_evalset(test)
        csr = train_data.sparse_interaction
        n_u, n_i = csr.shape
        users0, items0 = train_data.user_indices.astype(np.int32), train_data.item_indices.astype(np.int32)
        keep = (eval_data.user_indices < n_u) & (eval_data.item_indices < n_i)
        ev_u, ev_i = eval_data.user_indices[keep], eval_data.item_indices[keep]
        assert n_u < 1 << 16 and n_i < 1 << 16 and csr.has_sorted_indices
        calls = []

        def spy(*args, **kw):
            calls.append((kw["user_indices"].copy(), kw["item_indices"].copy()))
            return cy.bpr_update(*args, **kw)

        model = BPR("ranking", data_info, embed_size=16, n_epochs=FIT_EPOCHS, lr=FIT_LR[opt], optimizer=opt,
                    use_tf=False, seed=42)
        mod = types_module(spy)
        sys.modules["libreco.algorithms._bpr"] = mod
        algos._bpr = mod
        model.fit(train_data, neg_sampling=True, verbose=0)
        sys.modules["libreco.algorithms._bpr"] = cy
        algos._bpr = cy
        # the reference's per-epoch shuffles are successive permutations of data_info.np_rng = default_rng(42)
        rng = np.random.default_rng(42)
        orders = []
        for ep, (u, it) in enumerate(calls):
            perm = rng.permutation(range(len(users0)))
            assert np.array_equal(u, users0[perm]) and np.array_equal(it, items0[perm]), ep
            orders.append((u, it))
        from librecommender_b200.bpr import initial_tables

        U0, I0 = initial_tables(n_u, n_i, 16, seed=42)
        Uo, Io = oracle_fit(opt, orders, csr.indptr, csr.indices, U0, I0, FIT_LR[opt])
        key = f"fit_{opt}_"
        for side, got, ref in (("user", model.user_embeds_np, Uo), ("item", model.item_embeds_np, Io)):
            out[key + side + "_dev"] = np.abs(got.astype(np.float64) - ref).max(axis=1).astype(np.float32)
            out[key + side + "_rows"] = got[fit_rows(got.shape[0])]
        out[key + "default_recs"] = model.default_recs.astype(np.int32)
        r0 = orc.ranking_metrics(U0, I0, csr.indptr, csr.indices, ev_u, ev_i)
        r = orc.ranking_metrics(model.user_embeds_np[:-1], model.item_embeds_np[:-1], csr.indptr, csr.indices,
                                ev_u, ev_i)
        out[key + "metrics"] = np.array([r[0], r[1], r0[0], r0[1]])
        out[key + "lr"] = np.float64(FIT_LR[opt])
        print(opt, "recall/ndcg@10 initial", r0, "after", r, file=sys.stderr)
        out.update({"fit_users": users0.astype(np.uint16), "fit_items": items0.astype(np.uint16),
                    "fit_eval_users": ev_u.astype(np.uint16), "fit_eval_items": ev_i.astype(np.uint16),
                    "fit_shape": np.array([n_u, n_i], dtype=np.int64)})
    out["fit_stride"] = np.int64(FIT_STRIDE)
    out["fit_rng_seed"] = np.int64(42)
    out["fit_epochs"] = np.int64(FIT_EPOCHS)
    return out


def types_module(fn):
    import types

    mod = types.ModuleType("libreco.algorithms._bpr")
    mod.bpr_update = fn
    return mod


def oracle_fit(opt, orders, indptr, indices, U0, I0, lr):
    """``_fit_cython``'s loop in float64: the given per-epoch orders, the reference's negatives (num_threads 1,
    seed 42, the same stream every epoch), zero optimizer state; returns (U, I) with the mean row appended."""
    U, I = U0, I0
    st = {name: np.zeros_like(U0 if name.startswith("u_") else I0, dtype=np.float64)
          for name in orc.STATE_NAMES[opt]}
    for ep, (users, items) in enumerate(orders, start=1):
        negs = orc.reference_negatives(users, indptr, indices, I0.shape[0], 42, 1)
        U, I, st = orc.update(opt, users, items, negs, U, I, lr, 0.0, ep, st)
    return np.vstack([U, U.mean(0)]), np.vstack([I, I.mean(0)])


if __name__ == "__main__":
    tmp = tempfile.mkdtemp(prefix="bpr_cython_")
    try:
        cy = build_cython(tmp)
        out = update_cases(cy)
        out.update(fit_cases(cy))
    finally:
        shutil.rmtree(tmp, ignore_errors=True)
    np.savez_compressed(os.path.join(OUT, "bpr.npz"), **out)
    print("wrote bpr.npz", len(out), "arrays")
