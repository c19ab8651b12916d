"""SIM training without a GPU: the float64 step oracle against the inference restatement and central differences,
the dual-sequence collation against the reference's golden vectors, the float32 calibration of the GPU bounds, the
C-ABI envelope of the training kernels and the trainer's argument checks."""
import os
import random

import numpy as np
import pytest
import torch

import _sim_oracle as so
import _sim_train_oracle as sto

G = np.load(os.path.join(os.path.dirname(__file__), "golden", "dual_sequences.npz"))

LAYOUTS = [("ids", 16, 2, True, "keras"), ("feat", 8, 4, True, "legacy"), ("multi", 16, 1, False, "keras")]


def _case(c, **kw):
    spec, w, consumed, rows = sto.make_train_case(*c, **kw)
    return spec, w, consumed, rows


@pytest.mark.parametrize("c", LAYOUTS, ids=so.case_id)
def test_second_stage_in_inference_mode_is_the_inference_graph(c):
    """alpha = 0, beta = 1 and BN on the moving statistics: the oracle's logits are _sim_oracle.sim_forward's."""
    from librecommender_b200.feat_models import recent_dual_sequences
    from oracle import tf_models as tm

    spec, w, consumed, rows = _case(c)
    users, items = rows[0], rows[1]
    L, S, k = 24, 6, 6
    tabs = recent_dual_sequences(consumed, spec["n_users"], spec["n_items"], L, S)
    sparse, dense = tm.row_features(spec, users, items)
    want, sel, _, _ = so.sim_forward(dict(w, multi_sparse=None) if c[0] == "multi" else w, spec, users, items, *tabs,
                                     k, sparse, dense)
    st = sto.init_state(w, c[3], k, alpha=0.0, beta=1.0)
    t = {n: torch.tensor(v) for n, v in st["params"].items()}
    z, _, _, sel2, _, _ = sto.logits(st, t, spec, users, items, tabs[0][users], tabs[1][users], tabs[2][users],
                                     tabs[3][users], sparse, dense, bn_frozen=True)
    np.testing.assert_array_equal(sel2, sel)
    np.testing.assert_allclose(z.numpy(), want, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("scheme", ["keras", "legacy"])
def test_torch_esu_is_the_inference_restatement(scheme):
    from librecommender_b200 import synthetic as syn

    rng = np.random.default_rng(5)
    spec = syn.make_spec(rng, 5, 9, [], [], 0, 0)
    w = syn.make_sim_weights(rng, spec, 16, 4, (8, 4), False, scheme)
    q, rows = rng.standard_normal((7, 16)), rng.standard_normal((7, 5, 16))
    valid = rng.random((7, 5)) < 0.6
    valid[:, 0] = True
    st = sto.init_state(w, False, 5)
    t = {n: torch.tensor(v) for n, v in st["params"].items()}
    got = sto.esu(t, torch.tensor(q), torch.tensor(rows), valid, w["sim_scheme"], 4).numpy()
    np.testing.assert_allclose(got, so.esu(w, q, rows, valid, np.float64), rtol=1e-12, atol=1e-12)


def test_alpha_zero_gives_zero_first_stage_gradients():
    spec, w, _, rows = _case(LAYOUTS[0])
    st = sto.init_state(w, True, 6, alpha=0.0, beta=1.0)
    _, _, g, _, _, _, _ = sto.forward_backward(st, spec, *rows)
    fs = [k for k in g if k.startswith(("fs_", "first_stage_out"))]
    assert fs and all(not np.any(g[k]) for k in fs)
    assert np.any(g["seq_proj"]) and np.any(g["out_kernel"])


@pytest.mark.parametrize("loss_type", ["cross_entropy", "focal"])
@pytest.mark.parametrize("c", [LAYOUTS[0], LAYOUTS[1]], ids=so.case_id)
def test_oracle_gradients_against_central_differences(c, loss_type):
    spec, w, _, rows = _case(c, R=24)
    st = sto.init_state(w, c[3], 6, alpha=0.3, beta=0.8, loss_type=loss_type)
    _, _, g, _, sel, _, _ = sto.forward_backward(st, spec, *rows)
    rng = np.random.default_rng(1)
    for name in ("seq_proj", "item_embeds", f"sim_{sto.tto.att_names(c[4])[1]}", "fs_W0", "W0", "out_bias"):
        p = st["params"][name]
        for _ in range(3):
            i = tuple(int(rng.integers(0, s)) for s in p.shape)
            old = p[i]
            f = []
            for h in (1e-6, -1e-6):
                p[i] = old + h
                t = {n: torch.tensor(v) for n, v in st["params"].items()}
                z = sto.logits(st, t, spec, *rows[:8], sel=sel)[0]
                f.append(float(sto.loss_of(z, rows[8], loss_type)))
            p[i] = old
            fd = (f[0] - f[1]) / 2e-6
            assert abs(fd - g[name][i]) <= 1e-6 + 1e-5 * abs(fd), (name, i, fd, g[name][i])


# ---- the GPU bound: float32 against float64 on float64's selection ------------------------------------------------
GPU_RTOL = 2e-3            # test_gpu_sim_train: |gpu - f64| <= GPU_RTOL * max|f64| per gradient


@pytest.mark.parametrize("c", LAYOUTS, ids=so.case_id)
def test_float32_meets_the_gpu_gradient_bound_with_margin(c):
    spec, w, _, rows = _case(c)
    st = sto.init_state(w, c[3], 6, alpha=0.3, beta=0.8)
    l64, z64, g64, _, sel, _, _ = sto.forward_backward(st, spec, *rows)
    l32, z32, g32, _, _, _, _ = sto.forward_backward(st, spec, *rows, sel=sel, dtype=torch.float32)
    assert abs(l32 - l64) <= 0.25 * GPU_RTOL * abs(l64)
    for k in g64:
        scale = max(np.abs(g64[k]).max(), 1e-30)
        assert np.abs(g32[k] - g64[k]).max() <= 0.25 * GPU_RTOL * scale, k


# ---- dual sequences ------------------------------------------------------------------------------------------
def test_dual_windows_reproduce_the_reference_golden_vectors():
    """get_dual_seqs at the positions of interacted_positions_host (the same random.randrange stream)."""
    from librecommender_b200.collate import interacted_positions_host

    indptr, idx = G["indptr"], G["idx"]
    cons = {u: [int(i) for i in idx[indptr[u]:indptr[u + 1]]] for u in range(len(indptr) - 1)}
    users, items = G["users"], G["items"]
    for L, S in G["shapes"]:
        random.seed(4321)
        pos = interacted_positions_host(cons, users, items)
        pos = np.array([cons[int(u)].index(int(i)) if p < 0 else p for u, i, p in zip(users, items, pos)])
        ls, ll, ss, sl = sto.dual_windows(cons, users, pos, int(G["n_items"]), int(L), int(S))
        for got, key in ((ls, "long"), (ll, "long_lens"), (ss, "short"), (sl, "short_lens")):
            np.testing.assert_array_equal(got, G[f"{key}_{L}_{S}"])


# ---- C ABI and argument checks ------------------------------------------------------------------------------
def test_cabi_rejects_out_of_envelope_shapes_before_launch():
    from librecommender_b200 import _lib

    lib, x = _lib.lib, np.zeros(64, dtype=np.float32)
    P = _lib.ptr(x)
    n0 = _lib.launch_count()
    for K, H, L, k in [(65, 1, 100, 10), (0, 1, 100, 10), (16, 3, 100, 10), (16, 2, 257, 10), (16, 2, 100, 33),
                       (16, 2, 8, 9), (16, 2, 100, 0)]:
        if H == 2 or K % H == 0:      # the GSU and the long backward take no heads
            assert lib.b200_sim_gsu_forward(P, 64, K, P, P, 300, P, L, k, 4, P, P, 64, None) == -2, (K, L, k)
            assert lib.b200_sim_long_backward(P, 300, P, L, P, k, 4, K, P, 64, P, 64, P, 64, None) == -2, (K, L, k)
        if L != 257 and (L, k) != (8, 9):
            assert lib.b200_sim_esu_forward(P, 64, P, P, 64, P, P, 4, K, H, k, P, 64, P, None) == -2, (K, H, k)
            assert lib.b200_sim_esu_backward(P, 64, P, P, 64, P, P, 4, K, H, k, P, P, 64, P, 64, P, P, 64,
                                             None) == -2, (K, H, k)
    assert lib.b200_interacted_dual_seqs(P, P, 1, P, P, 4, 0, 5, 9, None, 0, 0, P, P, P, P, None) == -2
    assert _lib.launch_count() == n0


@pytest.mark.parametrize("bad", ["alpha", "beta", "loss", "task", "combiner"])
def test_trainer_argument_errors_need_no_device(bad):
    from librecommender_b200 import synthetic as syn
    from librecommender_b200.training import SIMTrainer

    rng = np.random.default_rng(2)
    if bad == "combiner":
        spec = syn.make_multi_sparse_spec(rng, 10, 12, [9], [12, 6], [("user", 17, 3), ("item", 23, 2)], 1, 1)
    else:
        spec = syn.make_spec(rng, 10, 12, [], [], 0, 0)
    w = syn.make_sim_weights(rng, spec, 8, 2, (8, 4), True, "keras")
    kw = dict(alpha=dict(alpha=1.5), beta=dict(beta=-0.1), loss=dict(loss_type="bpr"), task=dict(task="rating"),
              combiner={})[bad]
    with pytest.raises(ValueError):
        SIMTrainer(spec, w, **kw)
