"""CPU checks of the host side of the graph propagation and of its float64 oracles:
* ``SpmmGraph``'s long-row chunk plan against the numpy restatement (tests/_spmm_plan.py) at the chunk boundaries;
* ``SpmmGraph.transpose_perm``, which the LightGCN backward under edge dropout uses to reach L^T's values;
* the edge-dropout goldens (tests/golden/lightgcn_drop_*.npz): the mask stream and the non-zero order it indexes;
* ``oracle.ngcf`` and ``oracle.lightgcn.propagate64`` against every NGCF / LightGCN golden of the reference."""
import glob
import os

import numpy as np
import pytest
import torch
from scipy import sparse as sp

from _spmm_plan import long_row_plan

GOLD = os.path.join(os.path.dirname(__file__), "golden")
DROP = sorted(glob.glob(os.path.join(GOLD, "lightgcn_drop_*.npz")))
PLAIN = sorted(set(glob.glob(os.path.join(GOLD, "lightgcn_*.npz"))) - set(DROP))


def _consumed(g):
    return {u: g["idx"][g["indptr"][u]:g["indptr"][u + 1]].tolist() for u in range(int(g["n_users"]))}


def _laplacian_cpu(g):
    from librecommender_b200.lightgcn import build_laplacian_csr

    nu, ni = int(g["n_users"]), int(g["n_items"])
    return [t.numpy() for t in build_laplacian_csr(_consumed(g), nu, ni, device=torch.device("cpu"))]


@pytest.mark.parametrize("long_deg", [1024, 1025, 2048, 2049, 16385])
def test_spmm_graph_plan_matches_numpy(long_deg):
    """The chunk plan SpmmGraph builds for b200_spmm_csr: rows above the threshold, ceil(nnz / chunk) chunks each,
    chunk_row / chunk_k / long_chunk_ptr exactly as the numpy restatement (1024 is the last short degree)."""
    from librecommender_b200 import _lib
    from librecommender_b200.lightgcn import SpmmGraph

    thr, chunk = _lib.lib.b200_spmm_long_row_threshold(), _lib.lib.b200_spmm_chunk()
    assert (thr, chunk) == (1024, 1024)
    deg = np.array([long_deg, 3, 0, long_deg, 1100, 7, long_deg], dtype=np.int64)
    indptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    nnz = int(indptr[-1])
    g = SpmmGraph(torch.as_tensor(indptr), torch.zeros(nnz, dtype=torch.int32), torch.zeros(nnz))
    p = long_row_plan(indptr, thr, chunk)
    assert g.n_long == p["n_long"] and g.n_chunks == p["n_chunks"]
    assert p["n_long"] == (4 if long_deg > 1024 else 1)
    for k in ("long_rows", "long_chunk_ptr", "chunk_row", "chunk_k"):
        got = getattr(g, k)
        assert got.dtype == torch.as_tensor(p[k]).dtype, k
        np.testing.assert_array_equal(got.numpy(), p[k])
    # every non-zero of a long row lies in exactly one chunk
    covered = np.zeros(nnz, dtype=np.int64)
    for r, k in zip(p["chunk_row"], p["chunk_k"]):
        beg = indptr[r] + k * chunk
        covered[beg: min(beg + chunk, indptr[r + 1])] += 1
    long_nz = np.repeat(deg > thr, deg)
    assert (covered[long_nz] == 1).all() and (covered[~long_nz] == 0).all()


@pytest.mark.parametrize("path", PLAIN[:2] + DROP, ids=os.path.basename)
def test_transpose_perm_gives_transpose_values(path):
    """val[transpose_perm()] are the values of L^T in CSR order, bit for bit, for a non-symmetric value array on the
    symmetric Laplacian structure (what the backward of edge dropout multiplies by)."""
    from librecommender_b200.lightgcn import SpmmGraph

    indptr, col, val = _laplacian_cpu(np.load(path))
    n = len(indptr) - 1
    vals = np.random.default_rng(n).standard_normal(len(col)).astype(np.float32)
    g = SpmmGraph(torch.as_tensor(indptr), torch.as_tensor(col), torch.as_tensor(vals))
    LT = sp.csr_matrix((vals, col, indptr), shape=(n, n)).T.tocsr()
    LT.sort_indices()
    np.testing.assert_array_equal(LT.indptr, indptr)                    # symmetric structure
    np.testing.assert_array_equal(LT.indices, col)
    got = vals[g.transpose_perm().numpy()]
    assert np.array_equal(got.view(np.int32), LT.data.view(np.int32))
    assert not np.array_equal(got, vals)


@pytest.mark.parametrize("path", DROP, ids=os.path.basename)
def test_dropout_golden_mask_and_order(path):
    """torch.manual_seed(seed) then floor(rand(nnz) + keep) reproduces the reference's mask, and our CSR order of
    the Laplacian is the reference COO order the mask indexes (so our model drops the same edges)."""
    g = np.load(path)
    keep = 1 - float(g["dropout"])
    torch.manual_seed(int(g["seed"]))
    mask = torch.floor(torch.rand(int(g["nnz"])) + keep).bool().numpy()
    np.testing.assert_array_equal(mask, g["mask"])
    assert 0 < mask.mean() < 1
    indptr, col, val = _laplacian_cpu(g)
    rows = np.repeat(np.arange(len(indptr) - 1), np.diff(indptr))
    np.testing.assert_array_equal(rows, g["lap_row"])
    np.testing.assert_array_equal(col, g["lap_col"])
    assert np.array_equal(val.view(np.int32), g["lap_val"].view(np.int32))
    deg = np.diff(indptr)
    nu = int(g["n_users"])
    assert deg.max() > 1024                       # the head item's row takes the chunked path
    assert deg[nu - 1] == 0 and deg[-1] == 0      # isolated user, unconsumed item


def _drop_matrix(g):
    """The reference's L after sparse_dropout: kept values / keep in float32, dropped ones removed."""
    keep = np.float32(1 - float(g["dropout"]))
    n = int(g["n_users"]) + int(g["n_items"])
    m = g["mask"]
    v = g["lap_val"][m] / keep
    return sp.csr_matrix((v.astype(np.float64), (g["lap_row"][m], g["lap_col"][m])), shape=(n, n))


def _mag(L, X, n_layers):
    from oracle.lightgcn import propagate64

    return propagate64(abs(L), np.abs(X), n_layers)


@pytest.mark.parametrize("path", PLAIN + DROP, ids=os.path.basename)
def test_propagate64_reproduces_lightgcn_goldens(path):
    """propagate64 (and its gradient on the dropout goldens) matches the reference's float32 outputs within
    1e-5 * mag + 1e-7 per element, mag = mean_l |L|^l |E0| (|L^T| and |W| for the gradient)."""
    from oracle.lightgcn import propagate64, propagate64_grad

    g = np.load(path)
    n_layers = int(g["n_layers"])
    n = int(g["n_users"]) + int(g["n_items"])
    if "mask" in g.files:
        L = _drop_matrix(g)
    else:
        L = sp.csr_matrix((g["lap_val"].astype(np.float64), (g["lap_row"], g["lap_col"])), shape=(n, n))
    E0 = np.concatenate([g["user_init"], g["item_init"]])
    ref = propagate64(L, E0, n_layers)
    got = np.concatenate([g["user_out"], g["item_out"]])
    assert (np.abs(got - ref) <= 1e-5 * _mag(L, E0, n_layers) + 1e-7).all()
    if "W" in g.files:
        grad = propagate64_grad(L, g["W"], n_layers)
        got = np.concatenate([g["user_grad"], g["item_grad"]])
        assert (np.abs(got - grad) <= 1e-5 * _mag(L.T, g["W"], n_layers) + 1e-7).all()


@pytest.mark.parametrize("name", ["ngcf_d16.npz", "ngcf_d64.npz", "ngcf_d10.npz", "ngcf_d36.npz"])
def test_ngcf_oracle_reproduces_goldens(name):
    """oracle.ngcf in float64 against the reference's float32 run: the Laplacian within one float32 rounding, the
    propagated embeddings within the GPU test's rtol 2e-5, atol 2e-6 (a float32 forward of the same graph)."""
    from oracle import ngcf as on

    g = np.load(os.path.join(GOLD, name))
    nu, ni = int(g["n_users"]), int(g["n_items"])
    L = on.build_laplacian(nu, ni, _consumed(g)).tocoo()
    ref_L = sp.csr_matrix((g["lap_val"].astype(np.float64), (g["lap_row"], g["lap_col"])), shape=L.shape)
    np.testing.assert_allclose((sp.csr_matrix(L) - ref_L).toarray(), 0, atol=2 ** -24)
    weights = {k: g[k] for k in g.files if k.startswith(("W_", "b_"))}
    ue, ie = on.propagate64(L, g["user_embed"], g["item_embed"], weights)
    np.testing.assert_allclose(g["user_out"], ue, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(g["item_out"], ie, rtol=2e-5, atol=2e-6)
    assert ue.shape[1] == g["user_embed"].shape[1] + sum(g[f"W_self_{k}"].shape[1] for k in range(len(weights) // 4))
