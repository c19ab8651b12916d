"""CPU: Transformer training without a GPU.

* the float64 training restatement (``tests/_transformer_train_oracle.py``) with the BN frozen computes the logits of
  the inference restatement (``tests/_transformer_oracle.py``) for both graphs;
* its autograd gradients match central differences (causal on and off, rows of len 1 holding the pad id, rows with
  len < T), padded positions get exactly zero gradient, and a few TF-Adam steps reduce the loss;
* the raw variables round-trip through ``weights_io.transformer_tf_variables`` -> ``load_reference_tf_model`` for
  both graphs;
* calibration of the GPU bounds of ``test_gpu_transformer_train.py`` (the rule of ``test_din_kernel_bounds_cpu.py``):
  a float32 restatement meets each with 4x to spare, and its worst error uses at least 1/1000 of it;
* the new kernels' C-ABI rejects unsupported shapes before launching anything."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _transformer_oracle as to  # noqa: E402
import _transformer_train_oracle as tto  # noqa: E402
import test_gpu_transformer_train as gt  # noqa: E402


@pytest.mark.parametrize("c", gt.TRAIN_CASES, ids=gt.train_case_id)
def test_training_forward_with_frozen_bn_equals_inference_oracle(c):
    layout, K, H, L, causal, pos, bn, version, T = c
    rng, spec, w, seqs, lens = to.make_case((layout, K, "concat", H, L, causal, pos, bn, version), T=T)
    lens = np.maximum(lens, 1)                   # a training row has len >= 1
    users, items, sparse, dense = to.case_rows(rng, spec, R=60)
    st = tto.init_state(w, bn)
    t = {k: torch.tensor(v) for k, v in st["params"].items()}
    with torch.no_grad():
        out = tto.logits(st, t, spec, users, items, seqs[users], lens[users], sparse, dense, bn_frozen=True).numpy()
    ref = to.transformer_forward(w, spec, users, items, seqs, lens, sparse, dense)
    np.testing.assert_allclose(out, ref, rtol=1e-9, atol=1e-9 * np.abs(ref).max())


def _tiny(scheme, causal, pos="trainable", seed=5):
    """A case small enough for central differences: D = 8 (K = 2, one item sparse and one item dense field),
    T = 4, two heads, rows with len 1 holding the pad id, len < T and len = T."""
    from librecommender_b200 import synthetic as syn
    from oracle import tf_models as tm

    rng = np.random.default_rng(seed)
    n_users, n_items, T = 6, 7, 4
    spec = syn.make_spec(rng, n_users, n_items, [3], [4], 1, 1)
    w = syn.make_transformer_weights(rng, spec, 2, 2, 1, T, (4, 3), True, pos, causal, "concat", scheme)
    users, items = np.array([0, 3, 5, 2, 1]), np.array([1, 6, 4, 4, 0])
    lens = np.array([1, 2, 4, 3, 1], np.int32)
    seqs = rng.integers(0, n_items, (5, T)).astype(np.int32)
    seqs[np.arange(T)[None, :] >= lens[:, None]] = n_items
    seqs[0, 0] = n_items                          # the first position of a history: len 1, the pad id
    sparse, dense = tm.row_features(spec, users, items)
    return spec, w, (users, items, seqs, lens, sparse, dense, np.array([1, 0, 0, 1, 1], np.float32))


@pytest.mark.parametrize("scheme", ["keras", "legacy"])
@pytest.mark.parametrize("causal", [False, True])
def test_gradients_match_central_differences(scheme, causal):
    spec, w, batch = _tiny(scheme, causal)
    st = tto.init_state(w, True)
    _, _, g, _ = tto.forward_backward(st, spec, *batch)
    rng = np.random.default_rng(1)

    def loss_at(k, idx, delta):
        p = st["params"][k]
        old = p[idx]
        p[idx] = old + delta
        loss, _, _, _ = tto.forward_backward(st, spec, *batch)
        p[idx] = old
        return loss

    h = 1e-6
    for k, p in st["params"].items():
        flat = list(np.ndindex(p.shape))
        if k.startswith("tfm") or k in ("positional_encoding", "rms_last", "rms_item"):
            picks = flat                 # every entry: legacy Wk through the scores AND V = (X Wk) Wv'
        else:
            picks = [flat[i] for i in rng.choice(len(flat), size=min(6, len(flat)), replace=False)]
        for idx in picks:
            fd = (loss_at(k, idx, h) - loss_at(k, idx, -h)) / (2 * h)
            assert abs(fd - g[k][idx]) <= 1e-7 + 1e-5 * abs(fd), (k, idx, fd, g[k][idx])


@pytest.mark.parametrize("causal", [False, True])
def test_padded_positions_get_exactly_zero_gradient(causal):
    """The pad id fills only padded positions here (no len-1 row): its item-embedding row gets exactly 0, and so do
    the inputs of the padded positions."""
    spec, w, batch = _tiny("keras", causal)
    users, items, seqs, lens, sparse, dense, labels = batch
    lens = lens.copy()
    lens[0] = 2
    seqs = seqs.copy()
    seqs[0, :2] = [3, 5]
    st = tto.init_state(w, True)
    _, _, g, _ = tto.forward_backward(st, spec, users, items, seqs, lens, sparse, dense, labels)
    n_items = spec["n_items"]
    assert not g["item_embeds"][n_items].any()
    assert np.abs(g["item_embeds"][:n_items]).max() > 0
    # a trainable position appears padded in some rows and live in others; the sum over rows of the padded ones is 0:
    # position T-1 is live only in the len = T row, so changing that row's label moves it and nothing else does
    T = seqs.shape[1]
    only_padded = [t for t in range(T) if (lens <= t).all()]
    for t in only_padded:
        assert not g["positional_encoding"][t].any()


def test_steps_reduce_the_loss():
    spec, w, batches = gt.train_batch(gt.TRAIN_CASES[1], R=256, n_batches=1)
    users, items, seqs, lens, sparse, dense, labels = batches[0]
    st = tto.init_state(w, True)
    losses = [tto.train_step(st, spec, users, items, seqs, lens, sparse, dense, labels, 1e-2) for _ in range(6)]
    assert losses[-1] < losses[0] - 1e-3, losses


@pytest.mark.parametrize("scheme", ["keras", "legacy"])
@pytest.mark.parametrize("pos", ["trainable", "sinusoidal"])
def test_tf_variables_round_trip(tmp_path, scheme, pos):
    from librecommender_b200 import synthetic as syn
    from librecommender_b200 import weights_io as wio

    rng = np.random.default_rng(3)
    spec = syn.make_spec(rng, 30, 40, [5], [7, 3], 1, 1)
    w = syn.make_transformer_weights(rng, spec, 8, 2, 2, 12, (16, 8), True, pos, True, "concat", scheme)
    st = tto.init_state(w, True)
    raw = tto.raw_weights(st, w)                 # the raw layout a trained model exports
    np.savez(tmp_path / "m_tf_variables.npz", **wio.transformer_tf_variables(raw))
    got = wio.load_reference_tf_model(str(tmp_path), "m", "Transformer", 2, True, num_heads=2, num_tfm_layers=2,
                                      positional_embedding=pos, use_causal_mask=True)
    ref = wio.transformer_weights(raw)
    for lg, lr in zip(got["tfm_layers"], ref["tfm_layers"]):
        for k in lr:
            np.testing.assert_array_equal(lg[k], lr[k])
    for k in ("rms_last", "rms_item", "out_kernel", "out_bias", "user_embeds", "item_embeds", "sparse_embeds",
              "dense_embeds"):
        np.testing.assert_array_equal(got[k], ref[k])
    assert ("positional_encoding" in got) == (pos == "trainable")
    for i in range(2):
        np.testing.assert_array_equal(got["mlp"]["kernels"][i], raw["mlp"]["kernels"][i])
    np.testing.assert_array_equal(got["mlp"]["bn_in"]["mean"], raw["mlp"]["bn_in"]["mean"])


def _calibrate(ratios, what):
    worst = max(ratios)
    print(f"{what}: float32 uses {worst:.3g} of the bound")
    assert 4.0 * worst <= 1.0, f"{what}: float32 error is not 4x inside the bound ({worst:.3g})"
    assert worst >= 1e-3, f"{what}: bound is over 1000x looser than float32 needs ({worst:.3g})"


def _ratio(got, ref, bound):
    return float((np.abs(np.asarray(got, dtype=np.float64) - ref) / bound).max())


def test_attention_core_bounds():
    ratios = {n: [] for n in ("O", "lse", "dQ", "dK", "dV")}
    cases = [(c, False) for c in gt.KERNEL_CASES if c[0] * c[1] <= 2000] + [((37, 10, 2, 16, True), True),
                                                                           ((9, 64, 1, 128, False), True)]
    for c, large in cases:
        q, k, v, do, lens = gt.make_kernel_case(c, large)
        H, causal = c[2], c[4]
        ref = gt.reference(q, k, v, do, lens, H, causal, torch.float64)
        got = gt.reference(q, k, v, do, lens, H, causal, torch.float32)
        for name, g, r, b in zip(ratios, got, ref, gt.bounds(q, k, v, do, lens, H, causal)):
            ratios[name].append(_ratio(g, r, b))
    for name, r in ratios.items():
        _calibrate(r, name)


def test_rms_activation_and_target_attention_bounds():
    ratios = {n: [] for n in ("rms y", "rms rstd", "rms dx", "rms dscale", "swish y", "swish dy", "gelu y", "gelu dy",
                              "ta dq", "ta dS")}
    for R, D in gt.RMS_CASES:
        x, s, dy = gt.make_rms_case(R, D)
        ref, got = gt.rms_reference(x, s, dy, torch.float64), gt.rms_reference(x, s, dy, torch.float32)
        for name, g, r, b in zip(("rms y", "rms rstd", "rms dx", "rms dscale"), got, ref, gt.rms_bounds(x, s, dy)):
            ratios[name].append(_ratio(g, r, b))
    x = gt.act_inputs()
    for act in gt.ACT_CODES:
        ref = [np.nan_to_num(a) for a in gt.act_reference(x, act, torch.float64)]
        got = gt.act_reference(x, act, torch.float32)
        for name, g, r, b in zip((f"{act} y", f"{act} dy"), got, ref, gt.act_bounds(x, act)):
            ratios[name].append(_ratio(np.nan_to_num(g), r, b))
    for R, T, D in gt.TA_CASES:
        for large in (False, True):
            q, S, lens, dout = gt.make_ta_case(R, T, D, large=large)
            ref, got = gt.ta_reference(q, S, lens, dout, torch.float64), gt.ta_reference(q, S, lens, dout, torch.float32)
            for name, g, r, b in zip(("ta dq", "ta dS"), got, ref, gt.ta_bounds(q, S, lens, dout)):
                ratios[name].append(_ratio(g, r, b))
    for name, r in ratios.items():
        _calibrate(r, name)


def test_trainer_bounds():
    ratios = {"logits": [], "loss": [], "gradients": []}
    for c in gt.TRAIN_CASES:
        spec, w, batches = gt.train_batch(c, n_batches=1)
        batch = batches[0]
        st = tto.init_state(w, c[6])
        l64, o64, g64, _ = tto.forward_backward(st, spec, *batch)
        l32, o32, g32, _ = tto.forward_backward(st, spec, *batch, dtype=torch.float32)
        ratios["logits"].append(float((np.abs(o32 - o64) / (3e-5 + 3e-5 * np.abs(o64))).max()))
        ratios["loss"].append(abs(l32 - l64) / 2e-5)
        gmax = max(np.abs(v).max() for v in g64.values())
        bound = {k: gt.GRAD_REL * np.abs(g64[k]).max() + gt.GRAD_ABS * gmax for k in g64}
        ratios["gradients"].append(max(float(np.abs(g32[k] - g64[k]).max() / bound[k]) for k in g64))
    for name, r in ratios.items():
        _calibrate(r, name)


def test_cabi_rejects_unsupported_shapes_before_launch():
    from librecommender_b200 import _lib

    lib = _lib.lib
    x = np.zeros(256, np.float32)
    p = _lib.ptr(x)
    lens = np.ones(4, np.int32)
    pl = _lib.ptr(lens)
    n0 = _lib.launch_count()
    # (R, T, H, hd, ld): T outside [1, 64], no heads, empty heads, H * hd > 128, a stride below H * hd, R < 0
    for R, T, H, hd, ld in ((4, 65, 1, 8, 8), (4, 0, 1, 8, 8), (4, 8, 0, 8, 8), (4, 8, 2, 0, 8), (4, 8, 3, 43, 129),
                            (4, 8, 2, 8, 15), (-1, 8, 1, 8, 8)):
        assert lib.b200_transformer_attention_forward(p, ld, p, ld, p, ld, pl, R, T, H, hd, 1, 0.5, p, ld, p,
                                                      None) == -2
        assert b"b200_transformer_attention_forward" in lib.b200_last_error()
        assert lib.b200_transformer_attention_backward(p, ld, p, ld, p, ld, p, ld, p, p, ld, pl, R, T, H, hd, 0, 0.5, p,
                                                       p, p, ld, None) == -2
        assert b"b200_transformer_attention_backward" in lib.b200_last_error()
    assert lib.b200_transformer_attention_forward(p, 8, p, 8, p, 8, pl, 4, 8, 1, 8, 0, float("inf"), p, 8, p, None) == -2
    assert lib.b200_transformer_attention_forward(p, 8, p, 8, p, 8, None, 4, 8, 1, 8, 0, 0.5, p, 8, p, None) == -2
    # rms_norm: D < 1, a stride below D, R < 0
    for R, D, ld in ((4, 0, 8), (4, 8, 7), (-1, 8, 8)):
        assert lib.b200_rms_norm_forward(p, ld, R, D, p, p, ld, p, None) == -2
        assert lib.b200_rms_norm_backward(p, ld, p, ld, p, R, D, p, p, ld, None) == -2
    # activations: codes other than relu / swish / gelu, n < 0
    for act, n in ((0, 4), (4, 4), (2, -1)):
        assert lib.b200_activation_forward(p, n, act, p, None) == -2
        assert lib.b200_activation_backward(p, p, n, act, p, None) == -2
    # target-attention backward: T outside [1, 64], D outside [1, 128], a stride below D
    for T, D, ld in ((65, 8, 8), (0, 8, 8), (8, 129, 129), (8, 0, 8), (8, 16, 15)):
        assert lib.b200_transformer_target_attention_backward(p, ld, p, T, D, pl, p, ld, 4, p, ld, p, None) == -2
        assert b"b200_transformer_target_attention_backward" in lib.b200_last_error()
    assert _lib.launch_count() == n0
