"""RNN4Rec without a GPU: the float64 oracle of both TensorFlow graphs against an explicit per-step scalar loop over
the engine's canonical weights, the legacy / keras LSTM equivalence, the masking rules, the float32 bound the GPU
tests use, weight interchange through ``.npz`` and the C-ABI's envelope."""
import math

import numpy as np
import pytest

from _rnn4rec_oracle import rnn_states, user_vectors
from librecommender_b200.synthetic import make_rnn4rec_weights
from librecommender_b200.weights_io import rnn4rec_weights

N_ITEMS, K = 40, 8
CASES = [(typ, scheme, hu, ln) for typ in ("gru", "lstm") for scheme in ("keras", "legacy")
         for hu in ((6,), (5, 7)) for ln in ((False, True) if scheme == "keras" else (False,))]


def _seqs(rng, n, T, n_items=N_ITEMS):
    seqs = rng.integers(0, n_items + 1, size=(n, T)).astype(np.int32)
    lens = rng.integers(0, T + 1, size=n).astype(np.int32)
    lens[:3] = [0, 1, T]
    return seqs, lens


def _scalar_encode(w, seq, ln):
    """The cell formulas of b200_rnn_encode written as scalar loops over the canonical W / U / bx / bh layout."""
    sig = lambda v: 1.0 / (1.0 + math.exp(-v))      # noqa: E731
    layers = w["rnn_layers"]
    hs = [[0.0] * lw["U"].shape[0] for lw in layers]
    cs = [[0.0] * lw["U"].shape[0] for lw in layers]
    E = w["seq_embeds"].astype(np.float64)
    out = None
    for t in range(ln):
        x = list(E[seq[t]])
        for li, lw in enumerate(layers):
            W, U = lw["W"].astype(np.float64), lw["U"].astype(np.float64)
            bx, bh = lw["bx"].astype(np.float64), lw["bh"].astype(np.float64)
            H, h = U.shape[0], hs[li]
            act = (lambda v: v) if lw["act"] == 1 else math.tanh

            def pre(col, vec, M, b):
                return sum(vec[k] * M[k, col] for k in range(len(vec))) + b[col]
            nh, nc = [0.0] * H, list(cs[li])
            if lw["kind"] == 1:
                z = [sig(pre(j, x, W, bx) + pre(j, h, U, bh)) for j in range(H)]
                r = [sig(pre(H + j, x, W, bx) + pre(H + j, h, U, bh)) for j in range(H)]
                rh = [r[j] * h[j] for j in range(H)]
                for j in range(H):
                    cc = act(pre(2 * H + j, x, W, bx) + pre(2 * H + j, rh, U, bh))
                    nh[j] = z[j] * h[j] + (1 - z[j]) * cc
            for j in range(H):
                if lw["kind"] == 0:
                    z = sig(pre(j, x, W, bx) + pre(j, h, U, bh))
                    r = sig(pre(H + j, x, W, bx) + pre(H + j, h, U, bh))
                    hh = act(pre(2 * H + j, x, W, bx) + r * pre(2 * H + j, h, U, bh))
                    nh[j] = z * h[j] + (1 - z) * hh
                elif lw["kind"] == 2:
                    g = [pre(q * H + j, x, W, bx) + pre(q * H + j, h, U, bh) for q in range(4)]
                    nc[j] = sig(g[1]) * cs[li][j] + sig(g[0]) * act(g[2])
                    nh[j] = sig(g[3]) * act(nc[j])
            hs[li], cs[li] = nh, nc
            x = _ln_tanh(nh, lw) if lw["act"] == 1 else nh
        out = x
    last = layers[-1]
    if out is None or ln == 0:
        out = _ln_tanh(hs[-1], last) if last["act"] == 1 else hs[-1]
    return np.array(out)


def _ln_tanh(h, lw):
    H = len(h)
    mean = sum(h) / H
    var = sum((v - mean) ** 2 for v in h) / H
    return [math.tanh((h[j] - mean) / math.sqrt(var + 1e-3) * float(lw["gamma"][j]) + float(lw["beta"][j]))
            for j in range(H)]


@pytest.mark.parametrize("typ,scheme,hu,ln", CASES)
def test_oracle_matches_scalar_loop(typ, scheme, hu, ln):
    rng = np.random.default_rng(CASES.index((typ, scheme, hu, ln)))
    raw = make_rnn4rec_weights(rng, N_ITEMS, K, hu, typ, ln, scheme)
    w = rnn4rec_weights(raw)
    assert [lw["kind"] for lw in w["rnn_layers"]] == [{"gru": 0 if scheme == "keras" else 1, "lstm": 2}[typ]] * len(hu)
    T = 6
    seqs, lens = _seqs(rng, 12, T)
    ref = rnn_states(raw, seqs, lens)
    # the legacy LSTM's forget_bias 1.0 is folded into a float32 bias: one rounding of bias + 1 (< 6e-8)
    atol = 1e-7 if (typ, scheme) == ("lstm", "legacy") else 1e-12
    for i in range(len(seqs)):
        np.testing.assert_allclose(_scalar_encode(w, seqs[i], int(lens[i])), ref[i], rtol=0, atol=atol)


def test_legacy_and_keras_lstm_agree():
    rng = np.random.default_rng(5)
    leg = make_rnn4rec_weights(rng, N_ITEMS, K, (6, 4), "lstm", False, "legacy")
    ker = dict(leg, rnn_scheme="keras", rnn_layers=[])
    d = leg["seq_embeds"].shape[1]
    for lw in leg["rnn_layers"]:
        k, b = lw["kernel"].astype(np.float64), lw["bias"].astype(np.float64)
        H = k.shape[1] // 4
        perm = np.r_[0:H, 2 * H:3 * H, H:2 * H, 3 * H:4 * H]        # i | j | f | o -> i | f | c | o
        bias = b[perm].copy()
        bias[H:2 * H] += 1.0
        ker["rnn_layers"].append(dict(kernel=k[:d, perm], recurrent_kernel=k[d:, perm], bias=bias))
        d = H
    seqs, lens = _seqs(rng, 20, 7)
    np.testing.assert_allclose(rnn_states(ker, seqs, lens), rnn_states(leg, seqs, lens), rtol=0, atol=1e-9)


@pytest.mark.parametrize("typ,scheme,ln", [("gru", "keras", False), ("gru", "keras", True), ("gru", "legacy", False),
                                           ("lstm", "keras", True), ("lstm", "legacy", False)])
def test_masking_rules(typ, scheme, ln):
    rng = np.random.default_rng(11)
    raw = make_rnn4rec_weights(rng, N_ITEMS, K, (6, 5), typ, ln, scheme)
    T = 8
    seqs, lens = _seqs(rng, 30, T)
    ref = user_vectors(raw, seqs, lens)
    garbage = seqs.copy()
    for i, n in enumerate(lens):
        garbage[i, n:] = rng.integers(0, N_ITEMS + 1, T - n)
    np.testing.assert_array_equal(user_vectors(raw, garbage, lens), ref)
    if not ln:       # len 0: zero state, so the user vector is the Dense bias
        np.testing.assert_allclose(ref[lens == 0], np.broadcast_to(raw["dense_bias"], ref[lens == 0].shape), atol=1e-15)
    # the OOV row of recent_sequences: all pad with len 1 = one step over the pad row
    oov = user_vectors(raw, np.full((1, T), N_ITEMS, np.int32), np.array([1]))
    one = user_vectors(raw, np.array([[N_ITEMS] + [0] * (T - 1)], np.int32), np.array([1]))
    np.testing.assert_array_equal(oov, one)
    assert not np.allclose(oov, user_vectors(raw, np.full((1, T), N_ITEMS, np.int32), np.array([0])))


# The GPU tests compare float32 device results with the float64 oracle at this bound; the float32 restatement of the
# same graphs must stay within a quarter of it at the GPU tests' shapes (4x margin).
GPU_ATOL = 2e-5


@pytest.mark.parametrize("typ,scheme,ln", [("gru", "keras", False), ("gru", "keras", True), ("gru", "legacy", False),
                                           ("lstm", "keras", False), ("lstm", "keras", True), ("lstm", "legacy", False)])
@pytest.mark.parametrize("hu,T", [((16,), 10), ((32, 64), 50)])
def test_float32_meets_gpu_bound(typ, scheme, ln, hu, T):
    rng = np.random.default_rng(3)
    raw = make_rnn4rec_weights(rng, 300, 16, hu, typ, ln, scheme)
    seqs, lens = _seqs(rng, 200, T, 300)
    for norm in (False, True):
        ref = user_vectors(raw, seqs, lens, norm)
        got = user_vectors(raw, seqs, lens, norm, dtype=np.float32)
        err = np.abs(got - ref).max() / max(1.0, np.abs(ref).max())
        assert err < GPU_ATOL / 4, err


@pytest.mark.parametrize("typ,scheme,ln", [("gru", "keras", True), ("gru", "legacy", False), ("lstm", "keras", False),
                                           ("lstm", "legacy", False)])
def test_npz_round_trip(tmp_path, typ, scheme, ln):
    from librecommender_b200.weights_io import load_reference_tf_model, rnn4rec_tf_variables

    rng = np.random.default_rng(7)
    hu = (6, 5)
    raw = make_rnn4rec_weights(rng, N_ITEMS, K, hu, typ, ln, scheme)
    tfv = rnn4rec_tf_variables(raw)
    np.savez(tmp_path / "m_tf_variables.npz", **tfv)
    w = load_reference_tf_model(str(tmp_path), "m", "RNN4Rec", None, False, rnn_type=typ, hidden_units=hu,
                                use_layer_norm=ln)
    ref = rnn4rec_weights(raw)
    for k in ("seq_embeds", "item_embeds", "item_biases", "dense_kernel", "dense_bias"):
        np.testing.assert_array_equal(w[k], ref[k])
    for a, b in zip(w["rnn_layers"], ref["rnn_layers"]):
        assert a["kind"] == b["kind"] and a["act"] == b["act"]
        for k in ("W", "U", "bx", "bh", "gamma", "beta"):
            np.testing.assert_array_equal(a[k], b[k])
    # the scheme comes from the names
    names = set(tfv)
    if scheme == "legacy":
        assert any(n.startswith(f"rnn/multi_rnn_cell/cell_1/{typ}_cell/") for n in names)
    else:
        assert f"{typ}_1/{typ}_cell/recurrent_kernel:0" in names
        assert ("layer_normalization_1/gamma:0" in names) == ln
    # raw -> names -> raw round trip
    from librecommender_b200.weights_io import _rnn4rec_raw
    back = _rnn4rec_raw(np.load(tmp_path / "m_tf_variables.npz"), typ, hu, ln)
    assert rnn4rec_tf_variables(back).keys() == tfv.keys()
    for n, a in rnn4rec_tf_variables(back).items():
        np.testing.assert_array_equal(a, tfv[n])


def test_loader_reports_missing_and_misshaped(tmp_path):
    from librecommender_b200.weights_io import load_reference_tf_model, rnn4rec_tf_variables

    rng = np.random.default_rng(9)
    raw = make_rnn4rec_weights(rng, N_ITEMS, K, (6,), "gru", False, "keras")
    tfv = rnn4rec_tf_variables(raw)
    miss = {k: v for k, v in tfv.items() if k != "gru/gru_cell/recurrent_kernel:0"}
    np.savez(tmp_path / "a_tf_variables.npz", **miss)
    with pytest.raises(KeyError, match="gru/gru_cell/recurrent_kernel:0"):
        load_reference_tf_model(str(tmp_path), "a", "RNN4Rec", None, False, rnn_type="gru", hidden_units=(6,))
    bad = dict(tfv)
    bad["dense/kernel:0"] = np.zeros((7, K), np.float32)
    np.savez(tmp_path / "b_tf_variables.npz", **bad)
    with pytest.raises(KeyError, match="dense/kernel:0"):
        load_reference_tf_model(str(tmp_path), "b", "RNN4Rec", None, False, rnn_type="gru", hidden_units=(6,))
    # a wrong hidden size shows up as a misshaped variable
    np.savez(tmp_path / "c_tf_variables.npz", **tfv)
    with pytest.raises(KeyError, match="shape"):
        load_reference_tf_model(str(tmp_path), "c", "RNN4Rec", None, False, rnn_type="gru", hidden_units=(8,))
    # a Keras cell scope another Keras version names differently is overridden through extra_names
    ren = {k.replace("gru/gru_cell/", "gru/"): v for k, v in tfv.items()}
    np.savez(tmp_path / "d_tf_variables.npz", **ren)
    names = {"rnn_layers": [{k: f"gru/{k}:0" for k in ("kernel", "recurrent_kernel", "bias")}]}
    w = load_reference_tf_model(str(tmp_path), "d", "RNN4Rec", None, False, rnn_type="gru", hidden_units=(6,),
                                extra_names=names)
    np.testing.assert_array_equal(w["rnn_layers"][0]["W"], raw["rnn_layers"][0]["kernel"])


def test_cabi_rejects_out_of_envelope_shapes_before_launch():
    import ctypes

    from librecommender_b200 import _lib

    lib = _lib.lib
    n0 = _lib.launch_count()
    x = np.zeros(64, np.float32)
    users = np.zeros(4, np.int64)
    lens = np.ones(4, np.int32)
    seqs = np.zeros(4 * 200, np.int32)

    def call(T, in_dim, kinds, hidden, acts, n=4):
        L = len(hidden)
        arr = lambda v: (ctypes.c_int32 * max(1, L))(*v)      # noqa: E731
        return lib.b200_rnn_encode(_lib.ptr(users), n, _lib.ptr(lens), _lib.ptr(seqs), 200, T, _lib.ptr(x), 300,
                                   in_dim, L, arr(kinds), arr(hidden), arr(acts), _lib.ptr(x), _lib.ptr(x), 300, None)
    for args in [(0, 16, [0], [16], [0]), (129, 16, [0], [16], [0]), (10, 0, [0], [16], [0]), (10, 257, [0], [16], [0]),
                 (10, 16, [0], [257], [0]), (10, 16, [0, 0], [16, 0], [0, 0]), (10, 16, [3], [16], [0]),
                 (10, 16, [0], [16], [2]), (10, 16, [0] * 5, [16] * 5, [0] * 5), (10, 16, [], [], [])]:
        assert call(*args) == -2, args
    assert _lib.launch_count() == n0
    assert lib.b200_rnn_layer_floats(0, 16, 32) == 16 * 96 + 32 * 96 + 2 * 96 + 64
    assert lib.b200_rnn_layer_floats(2, 8, 4) == 8 * 16 + 4 * 16 + 32 + 8
    assert lib.b200_rnn_layer_floats(3, 8, 4) == -2
