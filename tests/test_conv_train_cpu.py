"""Caser / WaveNet training without a GPU: the float64 autograd oracle (tests/_conv_train_oracle.py) against the
inference restatement and central differences, the first-index tie rule of the max-pools, which table rows get
gradient, the float32 calibration of the GPU bounds, the export round trip through the TF variable names and the
C-ABI envelope of the new entry points."""
import numpy as np
import pytest
import torch

import _conv_encoder_oracle as inf
import _conv_train_oracle as co
from librecommender_b200 import synthetic as syn
from librecommender_b200 import weights_io as wio

N_USERS, N_ITEMS = 12, 20


def raw_weights(model, K=4, T=6, seed=0, dilated=True):
    rng = np.random.default_rng(seed)
    if model == "Caser":
        return syn.make_caser_weights(rng, N_USERS, N_ITEMS, K, T, 3, 2)
    return syn.make_wavenet_weights(rng, N_USERS, N_ITEMS, K, 5, 2, 2, dilated)


def batch(rng, R, T):
    """users (never the OOV row n_users, nor user 0), items, end-padded seqs with one all-pad row, labels."""
    lens = rng.integers(1, T + 1, R)
    lens[0] = 0
    seqs = rng.integers(0, N_ITEMS, (R, T))
    seqs[np.arange(T)[None, :] >= lens[:, None]] = N_ITEMS
    return rng.integers(1, N_USERS, R), rng.integers(0, N_ITEMS, R), seqs, (rng.random(R) < 0.5).astype(np.float64)


CASES = [("Caser", True), ("WaveNet", True), ("WaveNet", False)]


@pytest.mark.parametrize("model,dilated", CASES)
@pytest.mark.parametrize("T", [1, 2, 7])
def test_oracle_forward_equals_inference_restatement(model, dilated, T):
    raw = raw_weights(model, T=T, dilated=dilated)
    users, _, seqs, _ = batch(np.random.default_rng(1), 9, T)
    got = co.user_vectors(co.init_params(raw), co.meta_of(raw), users, seqs).detach().numpy()
    np.testing.assert_allclose(got, inf.user_vectors(raw, users, seqs), rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize("model,dilated", CASES)
@pytest.mark.parametrize("loss_type", ["cross_entropy", "focal"])
def test_gradients_match_central_differences(model, dilated, loss_type):
    raw = raw_weights(model, K=3, T=5, dilated=dilated)
    users, items, seqs, labels = batch(np.random.default_rng(2), 7, 5)
    meta = co.meta_of(raw)
    P = co.init_params(raw)
    arg, gap = co.pool_argmax(P, meta, seqs)
    assert gap.min() > 1e-4          # the data keeps a margin from ties (exact ties of identical windows are inf)
    _, g = co.forward_backward(P, meta, users, items, seqs, labels, loss_type, norm_embed=True)
    rng = np.random.default_rng(3)
    for k, v in P.items():
        flat = v.reshape(-1)
        for i in rng.choice(flat.numel(), min(6, flat.numel()), replace=False):
            old = float(flat[i])
            h = 1e-6
            flat[i] = old + h
            lp = float(co.loss(P, meta, users, items, seqs, labels, loss_type, True))
            flat[i] = old - h
            lm = float(co.loss(P, meta, users, items, seqs, labels, loss_type, True))
            flat[i] = old
            assert abs((lp - lm) / (2 * h) - g[k].reshape(-1)[i]) <= 1e-6 * max(1.0, abs(g[k]).max()), (k, i)


@pytest.mark.parametrize("model", ["Caser", "WaveNet"])
def test_tied_pad_windows_send_the_gradient_to_the_lowest_position(model):
    """A long all-pad tail makes the windows inside it bitwise identical; with the pad row pointing along a filter
    they tie at a positive maximum, and the whole gradient goes to the first of them."""
    T = 12
    raw = raw_weights(model, K=4, T=T, seed={"Caser": 5, "WaveNet": 7}[model], dilated=False)
    first = raw["convs"][0]["kernel"][-1]                     # [C_in = K, filters]: h = 1 (Caser), W[1] (WaveNet)
    if model == "WaveNet":                                     # a positive causal output, then a positive 1x1 output
        raw["out_conv"]["kernel"][0] = np.abs(raw["out_conv"]["kernel"][0])
    raw["seq_embeds"][N_ITEMS] = 3.0 * first[:, 0] / np.linalg.norm(first[:, 0])
    users, items, seqs, labels = batch(np.random.default_rng(6), 6, T)
    seqs[1:3, 3:] = N_ITEMS                                    # rows 1, 2: a pad tail from position 3
    meta = co.meta_of(raw)
    P = co.init_params(raw)
    keep = []
    f = co.features({k: v.clone().requires_grad_(True) for k, v in P.items()}, meta, seqs, keep=keep)
    for pre, _ in keep:
        pre.retain_grad()
    f.sum().backward()
    tied = 0
    for pre, a in keep:
        for r in (1, 2):
            for col in range(pre.shape[2]):
                v, g = pre[r, :, col].detach(), pre.grad[r, :, col]
                if v.max() <= 0:
                    assert torch.all(g == 0)
                    continue
                top = torch.nonzero(v == v.max()).reshape(-1)
                assert int(a[r, col]) == int(top[0])
                assert g[top[0]] == 1 and torch.count_nonzero(g) == 1
                tied += int(top.numel() > 1)
    assert tied >= 2


@pytest.mark.parametrize("model", ["Caser", "WaveNet"])
def test_pad_row_and_used_user_rows_get_gradient_unused_rows_none(model):
    raw = raw_weights(model)
    users, items, seqs, labels = batch(np.random.default_rng(4), 8, 6)
    _, g = co.forward_backward(co.init_params(raw), co.meta_of(raw), users, items, seqs, labels)
    assert np.any(g["seq_embeds"][N_ITEMS] != 0)              # the pad row is an ordinary trainable row
    for u in range(N_USERS + 1):                               # the OOV row n_users and user 0 are never used
        assert np.any(g["user_embeds"][u] != 0) == (u in set(users.tolist())), u
    unused = [r for r in range(N_ITEMS) if r not in set(seqs.reshape(-1).tolist())]
    assert np.all(g["seq_embeds"][unused] == 0)


def test_float32_restatement_meets_gpu_bounds():
    """The GPU bounds of test_gpu_conv_train.py hold for a float32 restatement with 4x to spare and are not more
    than 1000x loose.  Near-tied pooled columns follow the float32 choice, as the GPU tests follow the device's."""
    import test_gpu_conv_train as gt

    worst = 0.0
    for model, dilated in CASES:
        for loss_type in ("cross_entropy", "focal"):
            raw = raw_weights(model, K=8, T=10, seed=7, dilated=dilated)
            users, items, seqs, labels = batch(np.random.default_rng(8), 128, 10)
            meta = co.meta_of(raw)
            P64, P32 = co.init_params(raw), co.init_params(raw, torch.float32)
            arg32, _ = co.pool_argmax(P32, meta, seqs)
            pick = co.near_tie_pick(P64, meta, seqs, arg32, gt.GAP)
            l64, g64 = co.forward_backward(P64, meta, users, items, seqs, labels, loss_type, True, pick)
            l32, g32 = co.forward_backward(P32, meta, users, items, seqs, labels, loss_type, True)
            assert abs(l32 - l64) * 4 <= 2e-5 * max(1.0, abs(l64))
            gmax = max(np.abs(v).max() for v in g64.values())
            for k in g64:
                bound = gt.GRAD_REL * np.abs(g64[k]).max() + gt.GRAD_ABS * gmax
                err = np.abs(g32[k].astype(np.float64) - g64[k]).max()
                assert err * 4 <= bound, (model, loss_type, k, err, bound)
                worst = max(worst, err / bound)
    assert worst * 1000 >= 1.0, worst


@pytest.mark.parametrize("model,dilated", CASES)
def test_export_round_trip_is_exact(model, dilated, tmp_path):
    """An exported trainer state (the raw layout of ``co.raw_of``, float32) goes through ``*_tf_variables`` and
    ``load_reference_tf_model`` unchanged."""
    raw = raw_weights(model, dilated=dilated)
    users, items, seqs, labels = batch(np.random.default_rng(9), 8, 6)
    st = co.init_state(raw)
    co.train_step(st, co.meta_of(raw), users, items, seqs, labels, 1e-2, 1e-5)
    exp = co.raw_of(st["P"], raw)
    to32 = lambda a: np.asarray(a, np.float32)      # noqa: E731
    exp = {k: ([{n: to32(x) for n, x in c.items()} for c in v] if k == "convs" else
               {n: to32(x) for n, x in v.items()} if isinstance(v, dict) else v if k == "dilations" else to32(v))
           for k, v in exp.items()}
    np.savez(tmp_path / "m_tf_variables.npz", **wio._conv_tf_variables(exp))
    if model == "Caser":
        back, ref = wio.load_reference_tf_model(str(tmp_path), "m", "Caser", None, False), wio.caser_weights(exp)
    else:
        back = wio.load_reference_tf_model(str(tmp_path), "m", "WaveNet", None, False, n_filters=5, n_blocks=2,
                                           n_layers_per_block=2, dilated=dilated)
        ref = wio.wavenet_weights(exp)
    assert back.keys() == ref.keys()
    for k, v in ref.items():
        if isinstance(v, np.ndarray):
            np.testing.assert_array_equal(back[k], v, err_msg=k)
        else:
            assert back[k] == v, k


def test_cabi_rejects_out_of_envelope_before_launch():
    import ctypes

    from librecommender_b200 import _lib

    lib = _lib.lib
    n0 = _lib.launch_count()
    for T, K, nh, nv in ((0, 8, 2, 2), (65, 8, 2, 2), (10, 129, 2, 2), (10, 8, 33, 2), (10, 8, 2, 0)):
        assert lib.b200_caser_train_forward(None, 4, None, T, T, None, K, K, nh, nv, None, None, 100, None,
                                            None) == -2
        assert lib.b200_caser_backward_workspace_floats(4, T, K, nh, nv) == -2
        assert lib.b200_caser_backward(4, T, K, nh, nv, None, 10000, None, 10000, None, None, K, None, None, K, None,
                                       None, 0, None) == -2
    one = (ctypes.c_int32 * 17)(*([1] * 17))
    for T, K, L, F in ((0, 8, 2, 8), (65, 8, 2, 8), (10, 129, 2, 8), (10, 8, 17, 8), (10, 8, 2, 129)):
        assert lib.b200_wavenet_train_forward(None, 4, None, T, T, None, K, K, L, F, one, None, None, F, None, None,
                                              None) == -2
    zero = (ctypes.c_int32 * 2)(1, 0)
    assert lib.b200_wavenet_train_forward(None, 4, None, 10, 10, None, 8, 8, 2, 8, zero, None, None, 8, None, None,
                                          None) == -2
    for T, F in ((0, 8), (65, 8), (10, 0), (10, 129)):
        assert lib.b200_wavenet_pool_backward(4, T, F, None, F, None, None, None) == -2
    for T, C, d in ((0, 8, 1), (65, 8, 1), (10, 129, 1), (10, 8, 0)):
        assert lib.b200_wavenet_layer_inputs(None, C, 4, T, C, d, None, None) == -2
        assert lib.b200_wavenet_layer_dx(None, 4, T, C, d, None, C, None) == -2
    # n = 0 launches nothing
    assert lib.b200_caser_backward(0, 10, 8, 2, 2, None, 100, None, 100, None, None, 8, None, None, 8, None, None, 0,
                                   None) == 0
    assert lib.b200_caser_backward_workspace_floats(0, 10, 8, 2, 2) == 0
    assert lib.b200_wavenet_pool_backward(0, 10, 8, None, 8, None, None, None) == 0
    assert lib.b200_wavenet_layer_inputs(None, 8, 0, 10, 8, 1, None, None) == 0
    assert lib.b200_wavenet_layer_dx(None, 0, 10, 8, 1, None, 8, None) == 0
    assert _lib.launch_count() == n0
