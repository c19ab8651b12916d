"""Caser / WaveNet without a GPU: the float64 oracle against an independent restatement on torch's conv1d /
max_pool1d, the missing length mask, the TF1 dilation hazard, the OOV user row, the float32 error bound the GPU
tests use, the weight files and the C-ABI envelope."""
import numpy as np
import pytest

from _conv_encoder_oracle import assign_user_oov, caser_features, user_vectors, wavenet_features
from librecommender_b200.synthetic import make_caser_weights, make_wavenet_weights
from librecommender_b200.weights_io import wavenet_dilations

N_USERS, N_ITEMS = 30, 40


def _seqs(rng, n, T, n_items=N_ITEMS):
    """Right-padded rows as get_recent_seqs makes them: lens 0, 1, T and random."""
    lens = rng.integers(0, T + 1, n)
    lens[:3] = [0, 1, T]
    seqs = np.full((n, T), n_items, np.int32)
    for r, ln in enumerate(lens):
        seqs[r, :ln] = rng.integers(0, n_items, ln)
    return seqs, lens.astype(np.int32)


def _torch_caser(raw, seqs):
    """Caser's concat on torch.nn.functional (channels first): Keras kernel [w, in, out] -> torch [out, in, w]."""
    import torch
    import torch.nn.functional as F

    t = lambda a: torch.as_tensor(np.asarray(a, np.float64))      # noqa: E731
    X = t(raw["seq_embeds"])[torch.as_tensor(seqs, dtype=torch.int64)]      # [n, T, K]
    x = X.permute(0, 2, 1)                                                  # [n, K, T]
    outs = []
    for layer in raw["convs"]:
        y = F.relu(F.conv1d(x, t(layer["kernel"]).permute(2, 1, 0), t(layer["bias"])))   # [n, nh, T-h+1]
        outs.append(F.max_pool1d(y, y.shape[2]).squeeze(2))
    # the vertical layer reads x^T [n, K steps, T channels]: channels first that is X itself
    v = F.relu(F.conv1d(X, t(raw["vertical"]["kernel"]).permute(2, 1, 0), t(raw["vertical"]["bias"])))   # [n, nv, K]
    outs.append(v.permute(0, 2, 1).reshape(len(seqs), -1))
    return torch.cat(outs, dim=1).numpy()


def _torch_wavenet(raw, seqs, dilations):
    import torch
    import torch.nn.functional as F

    t = lambda a: torch.as_tensor(np.asarray(a, np.float64))      # noqa: E731
    x = t(raw["seq_embeds"])[torch.as_tensor(seqs, dtype=torch.int64)].permute(0, 2, 1)
    for layer, d in zip(raw["convs"], dilations):
        w = t(layer["kernel"]).permute(2, 1, 0)                                 # [F, C, 2]
        x = F.relu(F.conv1d(F.pad(x, ((w.shape[2] - 1) * d, 0)), w, t(layer["bias"]), dilation=d))
    z = F.relu(F.conv1d(x, t(raw["out_conv"]["kernel"]).permute(2, 1, 0), t(raw["out_conv"]["bias"])))
    return F.max_pool1d(z, z.shape[2]).squeeze(2).numpy()


@pytest.mark.parametrize("T", [1, 2, 10, 50])
@pytest.mark.parametrize("K,nh,nv", [(8, 2, 4), (16, 1, 1), (5, 3, 7)])
def test_caser_oracle_matches_torch(T, K, nh, nv):
    rng = np.random.default_rng(T * 100 + K)
    raw = make_caser_weights(rng, N_USERS, N_ITEMS, K, T, nh, nv)
    seqs, _ = _seqs(rng, 23, T)
    got = caser_features(raw, seqs)
    assert got.shape == (23, T * nh + K * nv)
    np.testing.assert_allclose(got, _torch_caser(raw, seqs), rtol=0, atol=1e-12)
    assert (got == 0).any() and (got > 0).any()           # ReLU zeros and live features both occur


@pytest.mark.parametrize("T", [1, 2, 10, 50])
@pytest.mark.parametrize("K,F,blocks,per_block", [(8, 16, 1, 4), (16, 4, 2, 3), (5, 9, 3, 1)])
@pytest.mark.parametrize("dilated", [True, False])
def test_wavenet_oracle_matches_torch(T, K, F, blocks, per_block, dilated):
    rng = np.random.default_rng(T * 100 + K + dilated)
    raw = make_wavenet_weights(rng, N_USERS, N_ITEMS, K, F, blocks, per_block, dilated)
    assert raw["dilations"] == wavenet_dilations(blocks, per_block, dilated)
    seqs, _ = _seqs(rng, 23, T)
    got = wavenet_features(raw, seqs)
    assert got.shape == (23, F)
    np.testing.assert_allclose(got, _torch_wavenet(raw, seqs, raw["dilations"]), rtol=0, atol=1e-12)


def test_tf1_graph_is_dilation_one():
    """A TF1-built WaveNet has dilation 1 in every layer; it agrees with the TF2 graph only while no dilated tap
    reaches back into the sequence differently (T = 1) and differs once it does."""
    assert wavenet_dilations(2, 4, True) == [1, 2, 4, 8, 1, 2, 4, 8]
    assert wavenet_dilations(2, 4, False) == [1] * 8
    rng = np.random.default_rng(5)
    raw = make_wavenet_weights(rng, N_USERS, N_ITEMS, 8, 8, 1, 4, True)
    for T in (1, 3, 10):
        seqs, _ = _seqs(rng, 20, T)
        tf1 = wavenet_features(raw, seqs, wavenet_dilations(1, 4, False))
        np.testing.assert_array_equal(tf1, wavenet_features(raw, seqs, [1, 1, 1, 1]))
        if T == 1:
            np.testing.assert_array_equal(tf1, wavenet_features(raw, seqs))
        else:
            assert np.abs(tf1 - wavenet_features(raw, seqs)).max() > 1e-6


@pytest.mark.parametrize("model", ["Caser", "WaveNet"])
def test_no_length_mask_pad_row_counts(model):
    """Neither graph reads the length: the pad positions go through the convolutions, so changing the pad row moves
    a short-history user's vector and leaves a full-length one alone."""
    rng = np.random.default_rng(11)
    T = 10
    raw = (make_caser_weights(rng, N_USERS, N_ITEMS, 8, T) if model == "Caser"
           else make_wavenet_weights(rng, N_USERS, N_ITEMS, 8, 8))
    seqs, lens = _seqs(rng, 12, T)
    ids = np.arange(12)
    before = user_vectors(raw, ids, seqs)
    moved = dict(raw, seq_embeds=np.array(raw["seq_embeds"]))
    moved["seq_embeds"][N_ITEMS] += 0.5
    after = user_vectors(moved, ids, seqs)
    short, full = lens < T, lens == T
    assert short.any() and full.any()
    assert (np.abs(after - before).max(axis=1)[short] > 0).all()
    np.testing.assert_array_equal(after[full], before[full])


def test_oov_user_row_is_the_mean():
    rng = np.random.default_rng(2)
    raw = make_caser_weights(rng, N_USERS, N_ITEMS, 8, 4)
    oov = assign_user_oov(raw)
    np.testing.assert_allclose(oov["user_embeds"][N_USERS], np.asarray(raw["user_embeds"][:N_USERS], np.float64).mean(0))
    np.testing.assert_array_equal(oov["user_embeds"][:N_USERS], raw["user_embeds"][:N_USERS])
    seqs, _ = _seqs(rng, 3, 4)
    v = user_vectors(oov, [N_USERS, 3, 0], seqs)
    np.testing.assert_allclose(v[0, :8], oov["user_embeds"][N_USERS])


GPU_ATOL = 2e-5       # the bound of tests/test_gpu_caser_wavenet.py


@pytest.mark.parametrize("model,T,shape", [("Caser", 50, (32, 8, 8)), ("Caser", 64, (128, 32, 32)),
                                           ("WaveNet", 50, (32, 64, 2, 4)), ("WaveNet", 64, (128, 128, 4, 4))])
def test_float32_restatement_within_gpu_bound(model, T, shape):
    """The same graphs in float32 stay well inside the tolerance the GPU tests apply (largest shapes tested)."""
    rng = np.random.default_rng(3)
    if model == "Caser":
        K, nh, nv = shape
        raw = make_caser_weights(rng, N_USERS, N_ITEMS, K, T, nh, nv)
    else:
        K, F, blocks, per_block = shape
        raw = make_wavenet_weights(rng, N_USERS, N_ITEMS, K, F, blocks, per_block)
    seqs, _ = _seqs(rng, 16, T)
    ids = np.arange(16)
    ref = user_vectors(raw, ids, seqs)
    f32 = user_vectors(raw, ids, seqs, dtype=np.float32)
    err = np.abs(f32 - ref).max() / max(1.0, np.abs(ref).max())
    assert err < GPU_ATOL / 4, err


def _same_weights(a, b):
    assert a.keys() == b.keys()
    for k in a:
        if isinstance(a[k], np.ndarray):
            np.testing.assert_array_equal(a[k], b[k])
        else:
            assert a[k] == b[k], k


@pytest.mark.parametrize("T", [1, 7])
def test_caser_npz_round_trip(tmp_path, T):
    from librecommender_b200.weights_io import _conv_raw, caser_tf_variables, caser_weights, load_reference_tf_model

    rng = np.random.default_rng(T)
    raw = make_caser_weights(rng, N_USERS, N_ITEMS, 6, T, 3, 2)
    tfv = caser_tf_variables(raw)
    assert f"conv1d_{T}/kernel:0" in tfv and tfv[f"conv1d_{T}/kernel:0"].shape == (1, T, 2)
    assert len([n for n in tfv if n.startswith("conv1d")]) == 2 * (T + 1)
    np.savez(tmp_path / "m_tf_variables.npz", **tfv)
    w = load_reference_tf_model(str(tmp_path), "m", "Caser", None, False)     # T is read off the file
    assert w["T"] == T and w["nh"] == 3 and w["nv"] == 2
    _same_weights(w, caser_weights(raw))
    back = caser_tf_variables(_conv_raw(np.load(tmp_path / "m_tf_variables.npz"), "Caser"))
    assert back.keys() == tfv.keys()
    for n, a in back.items():
        np.testing.assert_array_equal(a, tfv[n])


@pytest.mark.parametrize("dilated", [True, False])
def test_wavenet_npz_round_trip(tmp_path, dilated):
    from librecommender_b200.weights_io import load_reference_tf_model, wavenet_tf_variables, wavenet_weights

    rng = np.random.default_rng(4)
    raw = make_wavenet_weights(rng, N_USERS, N_ITEMS, 6, 5, 2, 3, dilated)
    tfv = wavenet_tf_variables(raw)
    assert tfv["conv1d_6/kernel:0"].shape == (1, 5, 5) and tfv["conv1d/kernel:0"].shape == (2, 6, 5)
    np.savez(tmp_path / "m_tf_variables.npz", **tfv)
    w = load_reference_tf_model(str(tmp_path), "m", "WaveNet", None, False, n_filters=5, n_blocks=2,
                                n_layers_per_block=3, dilated=dilated)
    assert w["dilations"] == ([1, 2, 4] * 2 if dilated else [1] * 6)
    _same_weights(w, wavenet_weights(raw))


def test_loader_reports_missing_and_misshaped(tmp_path):
    from librecommender_b200.weights_io import caser_tf_variables, load_reference_tf_model, wavenet_tf_variables

    rng = np.random.default_rng(9)
    tfv = caser_tf_variables(make_caser_weights(rng, N_USERS, N_ITEMS, 6, 5))
    for i, (name, value) in enumerate([("conv1d_2/kernel:0", None), ("conv1d_2/kernel:0", np.zeros((2, 6, 2))),
                                       ("dense/bias:0", np.zeros(7)), ("embedding/user_embeds_var:0", None),
                                       ("embedding/seq_embeds_var:0", np.zeros((N_ITEMS, 6)))]):
        bad = {k: v for k, v in tfv.items() if k != name}
        if value is not None:
            bad[name] = value.astype(np.float32)
        np.savez(tmp_path / f"c{i}_tf_variables.npz", **bad)
        with pytest.raises(KeyError, match=name):
            load_reference_tf_model(str(tmp_path), f"c{i}", "Caser", None, False)
    no_vertical = {k: v for k, v in tfv.items() if not k.startswith("conv1d_5/")}
    np.savez(tmp_path / "cv_tf_variables.npz", **no_vertical)
    with pytest.raises(KeyError, match="vertical"):
        load_reference_tf_model(str(tmp_path), "cv", "Caser", None, False)
    tfv = wavenet_tf_variables(make_wavenet_weights(rng, N_USERS, N_ITEMS, 6, 5, 1, 4))
    np.savez(tmp_path / "w_tf_variables.npz", **tfv)
    with pytest.raises(KeyError, match="conv1d_4/kernel:0"):           # five causal layers: the 1x1 has the wrong shape
        load_reference_tf_model(str(tmp_path), "w", "WaveNet", None, False, n_filters=5, n_blocks=1,
                                n_layers_per_block=5)
    with pytest.raises(KeyError, match="shape"):                        # a wrong filter count
        load_reference_tf_model(str(tmp_path), "w", "WaveNet", None, False, n_filters=6, n_blocks=1,
                                n_layers_per_block=4)
    # a layer named differently is overridden through extra_names
    ren = {k.replace("conv1d_4/", "out/"): v for k, v in tfv.items()}
    np.savez(tmp_path / "r_tf_variables.npz", **ren)
    w = load_reference_tf_model(str(tmp_path), "r", "WaveNet", None, False, n_filters=5, n_blocks=1,
                                n_layers_per_block=4, extra_names={"out_conv": {"kernel": "out/kernel:0",
                                                                                "bias": "out/bias:0"}})
    assert w["F"] == 5


def test_constructors_reject_out_of_envelope_shapes():
    """ValueError before any device work (the checks run ahead of the device lookup)."""
    from librecommender_b200 import _lib
    from librecommender_b200.feat_models import Caser, WaveNet

    rng = np.random.default_rng(0)
    n0 = _lib.launch_count()
    info = {"n_users": 4, "n_items": 20}

    def seqs(T):
        return np.full((5, T), 20, np.int32), np.ones(5, np.int32)
    for kw, T, match in [(dict(max_seq_len=65), 65, "max_seq_len"), (dict(nh_filters=33), 4, "nh_filters"),
                         (dict(nv_filters=33), 4, "nv_filters")]:
        with pytest.raises(ValueError, match=match):
            Caser(info, make_caser_weights(rng, 4, 20, 4, **{"max_seq_len": 4, **kw}), *seqs(T))
    with pytest.raises(ValueError, match="horizontal"):
        Caser(info, make_caser_weights(rng, 4, 20, 4, 5), *seqs(4))
    with pytest.raises(ValueError, match="embed_size"):
        Caser(info, make_caser_weights(rng, 4, 20, 129, 2, 1, 1), *seqs(2))
    for kw, match in [(dict(n_filters=129), "n_filters"), (dict(n_blocks=17, n_layers_per_block=1), "dilations")]:
        with pytest.raises(ValueError, match=match):
            WaveNet(info, make_wavenet_weights(rng, 4, 20, 4, **kw), *seqs(10))
    raw = make_wavenet_weights(rng, 4, 20, 4, 4)
    with pytest.raises(ValueError, match="dilations"):
        WaveNet(info, dict(raw, dilations=[1, 0, 1, 1]), *seqs(10))
    with pytest.raises(ValueError, match="recent sequences"):
        WaveNet(info, raw, np.zeros((4, 10), np.int32), np.ones(4, np.int32))
    assert _lib.launch_count() == n0


def test_cabi_envelope():
    import ctypes

    from librecommender_b200 import _lib

    lib = _lib.lib
    assert lib.b200_caser_weight_floats(10, 16, 2, 4) == 16 * 2 * 55 + 10 * 2 + 10 * 4 + 4
    assert lib.b200_caser_weight_floats(1, 3, 1, 1) == 3 + 1 + 1 + 1
    assert lib.b200_wavenet_weight_floats(16, 16, 4) == (2 * 16 * 16 + 16) * 4 + 16 * 16 + 16
    assert lib.b200_wavenet_weight_floats(8, 4, 1) == 2 * 8 * 4 + 4 + 16 + 4
    for args in [(0, 16, 2, 4), (65, 16, 2, 4), (10, 0, 2, 4), (10, 129, 2, 4), (10, 16, 0, 4), (10, 16, 33, 4),
                 (10, 16, 2, 0), (10, 16, 2, 33)]:
        assert lib.b200_caser_weight_floats(*args) == -2, args
    for args in [(0, 16, 4), (129, 16, 4), (16, 0, 4), (16, 129, 4), (16, 16, 0), (16, 16, 17)]:
        assert lib.b200_wavenet_weight_floats(*args) == -2, args
    n0 = _lib.launch_count()
    x = np.zeros(64, np.float32)
    users = np.zeros(4, np.int64)
    seqs = np.zeros(4 * 100, np.int32)
    P = _lib.ptr
    for T, K, nh, nv in [(0, 16, 2, 4), (65, 16, 2, 4), (10, 129, 2, 4), (10, 16, 33, 4), (10, 16, 2, 0)]:
        assert lib.b200_caser_encode(P(users), 4, P(seqs), 100, T, P(x), 200, K, nh, nv, P(x), P(x), 10000,
                                     None) == -2
    for T, K, L, F, dil in [(65, 16, 1, 16, [1]), (10, 129, 1, 16, [1]), (10, 16, 1, 129, [1]),
                            (10, 16, 17, 16, [1] * 17), (10, 16, 0, 16, [1]), (10, 16, 2, 16, [1, 0])]:
        arr = (ctypes.c_int32 * len(dil))(*dil)
        assert lib.b200_wavenet_encode(P(users), 4, P(seqs), 100, T, P(x), 200, K, L, F, arr, P(x), P(x), 200,
                                       None) == -2
    assert lib.b200_wavenet_encode(P(users), 4, P(seqs), 100, 10, P(x), 200, 16, 1, 16, None, P(x), P(x), 200,
                                   None) == -2
    # n = 0 launches nothing
    assert lib.b200_caser_encode(None, 0, None, 100, 10, None, 200, 16, 2, 4, None, None, 10000, None) == 0
    assert _lib.launch_count() == n0
