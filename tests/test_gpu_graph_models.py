"""The graph models end to end on the GPU against float64 oracles and the reference's goldens:
* LightGCN edge dropout (``forward(use_dropout=True)``): L stops being symmetric, so the backward multiplies by L^T
  through ``SpmmGraph.transpose_perm``; forward and init-embedding gradients are checked;
* ``propagate`` at several depths and widths with a per-element bound that sees one dropped edge;
* ``NGCFPropagator`` at widths that change per layer in odd steps, with a row above the long-row threshold."""
import glob
import os

import numpy as np
import pytest
from scipy import sparse as sp

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")
DROP = sorted(glob.glob(os.path.join(GOLD, "lightgcn_drop_*.npz")))


def _consumed(g):
    return {u: g["idx"][g["indptr"][u]:g["indptr"][u + 1]].tolist() for u in range(int(g["n_users"]))}


def _mag(L, X, n_layers):
    """mean_l |L|^l |X|: the scale of each element's summation error."""
    from oracle.lightgcn import propagate64

    return propagate64(abs(L), np.abs(X), n_layers)


@pytest.mark.parametrize("path", DROP, ids=os.path.basename)
def test_lightgcn_edge_dropout_forward_and_gradients(path):
    """Edge dropout with the reference's mask stream (CPU torch.rand after torch.manual_seed): outputs and the
    init-embedding gradients of (cat(out) * W).sum() against the golden and against float64 on the stored mask,
    within 1e-5 * mag + 1e-7 per element.  The dropout is strong enough that a backward multiplying by L instead of
    L^T (val instead of val[transpose_perm]) is far outside that bound."""
    import torch

    from librecommender_b200.lightgcn import make_lightgcn_model_class
    from oracle.lightgcn import propagate64, propagate64_grad

    g = np.load(path)
    nu, ni, n_layers, p = int(g["n_users"]), int(g["n_items"]), int(g["n_layers"]), float(g["dropout"])
    d = g["user_init"].shape[1]
    m = make_lightgcn_model_class()(nu, ni, d, n_layers, p, _consumed(g), "cuda")
    assert m.graph.n_long >= 1
    with torch.no_grad():
        m.user_init_embeds.weight.copy_(torch.from_numpy(g["user_init"]))
        m.item_init_embeds.weight.copy_(torch.from_numpy(g["item_init"]))
    torch.manual_seed(int(g["seed"]))
    ue, ie = m(use_dropout=True)
    out = torch.cat([ue, ie])
    (out * torch.from_numpy(g["W"]).cuda()).sum().backward()
    got = out.detach().cpu().numpy()
    grad = torch.cat([m.user_init_embeds.weight.grad, m.item_init_embeds.weight.grad]).cpu().numpy()

    keep = np.float32(1 - p)
    mask = g["mask"]
    L = sp.csr_matrix(((g["lap_val"][mask] / keep).astype(np.float64), (g["lap_row"][mask], g["lap_col"][mask])),
                      shape=(nu + ni, nu + ni))
    E0 = np.concatenate([g["user_init"], g["item_init"]])
    ref, mag = propagate64(L, E0, n_layers), _mag(L, E0, n_layers)
    assert (np.abs(got - ref) <= 1e-5 * mag + 1e-7).all()
    gold = np.concatenate([g["user_out"], g["item_out"]])
    assert (np.abs(got - gold) <= 2e-5 * mag + 2e-7).all()

    ref_g, mag_g = propagate64_grad(L, g["W"], n_layers), _mag(L.T, g["W"], n_layers)
    bound_g = 1e-5 * mag_g + 1e-7
    assert (np.abs(grad - ref_g) <= bound_g).all()
    gold_g = np.concatenate([g["user_grad"], g["item_grad"]])
    assert (np.abs(grad - gold_g) <= 2 * bound_g).all()
    wrong = propagate64(L, g["W"], n_layers)            # backward through L instead of L^T
    assert (np.abs(wrong - ref_g) > 100 * bound_g).mean() > 0.5


def _graph(nu, ni, seed):
    """Zipf consumption, item 0 consumed by half the users (a long row), an isolated user and an unconsumed item."""
    rng = np.random.default_rng(seed)
    w = 1.0 / np.arange(1, ni) ** 1.1
    w /= w.sum()
    consumed = {}
    for u in range(nu):
        items = set(rng.choice(ni - 1, size=int(rng.integers(1, 15)), replace=False, p=w).tolist())
        if u % 2 == 0:
            items.add(0)
        consumed[u] = sorted(items)
    consumed[nu - 1] = []
    return consumed


@pytest.mark.parametrize("d", [3, 16, 64, 132])
@pytest.mark.parametrize("n_layers", [0, 1, 2, 4])
def test_propagate_per_element_bound(n_layers, d):
    """mean_l L^l E0 for the scalar (3, 132) and vec4 (16, 64) SpMM branches and the fused layer-mean epilogue
    (acc_init on the first layer, final_div on the last; n_layers = 0 copies E0): |got - ref64| <= 1e-5 mag + 1e-7
    per element, where one dropped edge changes an element by about mag / deg.  Isolated nodes are exactly
    E0 / (n_layers + 1)."""
    import torch

    from librecommender_b200.lightgcn import SpmmGraph, build_laplacian_csr, propagate
    from oracle.lightgcn import propagate64

    nu, ni = 2600, 200
    indptr, col, val = build_laplacian_csr(_graph(nu, ni, 60 + d), nu, ni)
    graph = SpmmGraph(indptr, col, val)
    assert graph.n_long >= 1
    rng = np.random.default_rng(d * 7 + n_layers)
    E0 = rng.normal(0, 0.1, (nu + ni, d)).astype(np.float32)
    got = propagate(graph, torch.from_numpy(E0).cuda(), n_layers).cpu().numpy()
    n = nu + ni
    ip = indptr.cpu().numpy()
    L = sp.csr_matrix((val.cpu().numpy().astype(np.float64), col.cpu().numpy(), ip), shape=(n, n))
    ref, mag = propagate64(L, E0, n_layers), _mag(L, E0, n_layers)
    assert (np.abs(got - ref) <= 1e-5 * mag + 1e-7).all()
    iso = np.flatnonzero(np.diff(ip) == 0)
    assert set(iso) >= {nu - 1, n - 1}
    np.testing.assert_array_equal(got[iso], E0[iso] / np.float32(n_layers + 1))


@pytest.mark.parametrize("name", ["ngcf_d10.npz", "ngcf_d36.npz"])
def test_ngcf_odd_widths_golden_and_float64(name):
    """Layer-input widths 10 / 24 (d10: layers (24, 7)) and 36 / 132 (d36: layers (132, 20)) drive the SpMM's scalar
    lpr 16, vec4 LPR 8 / 16 and scalar T = 5 branches and ngcf_combine at 24 / 7 / 132 / 20, with the head item's
    row on the long-row path: the golden at rtol 2e-5, atol 2e-6 and oracle.ngcf in float64 at the same bound."""
    from librecommender_b200.consumed import ConsumedCSR
    from librecommender_b200.ngcf import NGCFPropagator
    from oracle import ngcf as on

    g = np.load(os.path.join(GOLD, name))
    nu, ni = int(g["n_users"]), int(g["n_items"])
    csr = ConsumedCSR(g["indptr"], g["idx"])
    weights = {k: g[k] for k in g.files if k.startswith(("W_", "b_")) or k in ("user_embed", "item_embed")}
    prop = NGCFPropagator(nu, ni, csr, weights)
    assert prop.graph.n_long >= 1
    ue, ie = (t.cpu().numpy() for t in prop.forward())
    np.testing.assert_allclose(ue, g["user_out"], rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(ie, g["item_out"], rtol=2e-5, atol=2e-6)
    ru, ri = on.propagate64(on.build_laplacian(nu, ni, csr.to_dict()), g["user_embed"], g["item_embed"], weights)
    np.testing.assert_allclose(ue, ru, rtol=2e-5, atol=2e-6)
    np.testing.assert_allclose(ie, ri, rtol=2e-5, atol=2e-6)
