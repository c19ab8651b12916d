"""GPU parity of the CSR SpMM / LightGCN propagation against the reference-generated golden
vectors (tests/golden/lightgcn_*.npz) and the oracle; float tolerance 1e-5 relative."""
import glob
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")


def _consumed(g):
    return {u: g["idx"][g["indptr"][u]:g["indptr"][u + 1]].tolist() for u in range(int(g["n_users"]))}


@pytest.mark.parametrize("path", sorted(set(glob.glob(os.path.join(GOLD, "lightgcn_*.npz")))
                                        - set(glob.glob(os.path.join(GOLD, "lightgcn_drop_*.npz")))))
def test_laplacian_and_propagation_golden(path):
    """Goldens without edge dropout (the dropout ones are checked in test_gpu_graph_models.py)."""
    import torch
    from librecommender_b200.lightgcn import SpmmGraph, build_laplacian_csr, propagate

    g = np.load(path)
    nu, ni, L = int(g["n_users"]), int(g["n_items"]), int(g["n_layers"])
    indptr, col, val = build_laplacian_csr(_consumed(g), nu, ni)
    rows = np.repeat(np.arange(nu + ni), np.diff(indptr.cpu().numpy()))
    np.testing.assert_array_equal(rows, g["lap_row"])            # same (row, col) order as the reference COO
    np.testing.assert_array_equal(col.cpu().numpy(), g["lap_col"])
    np.testing.assert_array_equal(val.cpu().numpy(), g["lap_val"])   # bit-exact fp32 values
    graph = SpmmGraph(indptr, col, val)
    E0 = torch.from_numpy(np.concatenate([g["user_init"], g["item_init"]])).cuda()
    out = propagate(graph, E0, L).cpu().numpy()
    np.testing.assert_allclose(out[:nu], g["user_out"], rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(out[nu:], g["item_out"], rtol=1e-5, atol=1e-7)


def test_long_rows_and_widths_vs_oracle():
    import torch
    from librecommender_b200.lightgcn import SpmmGraph, build_laplacian_csr, propagate
    from oracle import lightgcn as og

    rng = np.random.default_rng(4)
    nu, ni = 6000, 300
    consumed = {}
    for u in range(nu):
        items = set(rng.choice(ni, size=int(rng.integers(1, 20)), replace=False).tolist())
        if u % 2 == 0:
            items.add(0)            # item 0: ~3000 edges  -> chunked long row
        if u % 3 == 0:
            items.add(1)            # item 1: ~2000 edges
        consumed[u] = sorted(items)
    Lm = og.build_laplacian(nu, ni, consumed)
    for d in (64, 16, 100, 3):
        indptr, col, val = build_laplacian_csr(consumed, nu, ni)
        graph = SpmmGraph(indptr, col, val)
        assert graph.n_long >= 2
        ue = rng.normal(0, 0.1, (nu, d)).astype(np.float32)
        ie = rng.normal(0, 0.1, (ni, d)).astype(np.float32)
        out = propagate(graph, torch.from_numpy(np.concatenate([ue, ie])).cuda(), 3).cpu().numpy()
        ru, ri = og.propagate(Lm, ue, ie, 3)
        ref = np.concatenate([ru, ri])
        scale = np.abs(ref).max()
        assert np.abs(out - ref).max() <= 1e-5 * scale


def test_module_forward_backward_matches_torch_sparse():
    import torch
    from librecommender_b200.lightgcn import make_lightgcn_model_class

    rng = np.random.default_rng(2)
    nu, ni, d, L = 300, 200, 16, 3
    consumed = {u: rng.choice(ni, size=int(rng.integers(1, 30)), replace=False).tolist() for u in range(nu)}
    Model = make_lightgcn_model_class()
    torch.manual_seed(0)
    m = Model(nu, ni, d, L, 0.0, consumed, "cuda")
    ue, ie = m(use_dropout=False)
    # reference formulation with torch.sparse.mm on the same device
    g = m.graph
    rows = torch.repeat_interleave(torch.arange(g.n, device="cuda"), g.indptr[1:] - g.indptr[:-1])
    Lt = torch.sparse_coo_tensor(torch.stack([rows, g.col.long()]), g.val, (g.n, g.n))
    E0 = torch.cat([m.user_init_embeds.weight, m.item_init_embeds.weight]).detach().clone().requires_grad_(True)
    layers = [E0]
    for _ in range(L):
        layers.append(torch.sparse.mm(Lt, layers[-1]))
    ref = torch.stack(layers, 1).mean(1)
    torch.testing.assert_close(torch.cat([ue, ie]), ref, rtol=1e-5, atol=1e-7)
    w = torch.randn_like(ref)
    (ref * w).sum().backward()
    (torch.cat([ue, ie]) * w).sum().backward()
    got = torch.cat([m.user_init_embeds.weight.grad, m.item_init_embeds.weight.grad])
    torch.testing.assert_close(got, E0.grad, rtol=1e-4, atol=1e-6)


def test_bpr_training_steps_reduce_loss():
    """A few BPR steps exactly as TorchTrainer._compute_loss does them
    (libreco/training/torch_trainer.py:140-161: full-graph propagation, gather, bpr_loss of
    libreco/torchops/loss.py:22-24, Adam) through the CUDA propagation and its backward."""
    import torch
    from librecommender_b200.lightgcn import make_lightgcn_model_class
    from librecommender_b200.sampling import DeviceNegativeSampler

    rng = np.random.default_rng(5)
    nu, ni, d = 400, 300, 16
    consumed = {u: rng.choice(ni, size=int(rng.integers(3, 25)), replace=False).tolist() for u in range(nu)}
    Model = make_lightgcn_model_class()
    torch.manual_seed(1)
    m = Model(nu, ni, d, 2, 0.0, consumed, "cuda")
    opt = torch.optim.Adam(m.parameters(), lr=0.05)
    sampler = DeviceNegativeSampler(ni, consumed, nu, seed=42)
    users = torch.as_tensor(np.repeat(np.arange(nu), 3)).cuda()
    pos = torch.as_tensor(np.array([consumed[u][j] for u in range(nu) for j in range(3)])).cuda()
    losses = []
    for step in range(8):
        neg = sampler.sample(users, pos, 1, "unconsumed")
        ue, ie = m(use_dropout=False)
        s_pos = (ue[users] * ie[pos]).sum(1)
        s_neg = (ue[users] * ie[neg]).sum(1)
        loss = -torch.nn.functional.logsigmoid(s_pos - s_neg).mean()
        opt.zero_grad()
        loss.backward()
        opt.step()
        losses.append(float(loss))
    assert losses[-1] < losses[0] * 0.9, losses
