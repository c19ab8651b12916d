"""CPU: AutoInt training without a GPU.

* the float64 training restatement (``tests/_autoint_train_oracle.py``) computes, before any step, the logits of
  the inference restatement (``tests/_autoint_oracle.py``) for both graphs, and its autograd gradients match
  central differences on a tiny case, the legacy value kernel Wv' and key kernel (both of its paths) included;
* a few TF-Adam steps reduce the loss;
* ``weights_io.autoint_tf_variables`` -> ``load_reference_tf_model`` round-trips both schemes;
* calibration of the GPU bounds of ``test_gpu_autoint_train.py`` (the rule of ``test_din_kernel_bounds_cpu.py``): a
  float32 restatement meets each with 4x to spare, and its worst error uses at least 1/1000 of it;
* the attention kernels' C-ABI rejects unsupported shapes before launching anything."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _autoint_oracle as ao  # noqa: E402
import _autoint_train_oracle as ato  # noqa: E402
import test_gpu_autoint_train as gt  # noqa: E402


@pytest.mark.parametrize("c", gt.TRAIN_CASES, ids=ao.case_id)
def test_training_forward_equals_inference_oracle(c):
    rng, spec, w = ao.make_case(c)
    users, items, sparse, dense = ao.case_rows(rng, spec, R=60)
    st = ato.init_state(w)
    _, out, _ = ato.forward_backward(st, users, items, sparse, dense, np.zeros(60, np.float32))
    ref = ao.autoint_forward(w, users, items, sparse, dense, np.float64)
    np.testing.assert_allclose(out, ref, rtol=1e-9, atol=1e-9 * np.abs(ref).max())


@pytest.mark.parametrize("scheme", ["keras", "legacy"])
@pytest.mark.parametrize("residual", [True, False])
def test_gradients_match_central_differences(scheme, residual):
    from librecommender_b200 import synthetic as syn
    from oracle import tf_models as tm

    rng = np.random.default_rng(5)
    spec = syn.make_spec(rng, 6, 7, [3], [4], 1, 1)
    w = syn.make_autoint_weights(rng, spec, 3, (2, 3), 2, residual, scheme)
    users, items = np.array([0, 3, 6, 2]), np.array([1, 7, 4, 4])
    sparse, dense = tm.row_features(spec, users, items)
    labels = np.array([1, 0, 0, 1], np.float32)
    st = ato.init_state(w)
    _, _, g = ato.forward_backward(st, users, items, sparse, dense, labels)

    def loss_at(k, idx, delta):
        p = st["params"][k]
        old = p[idx]
        p[idx] = old + delta
        loss, _, _ = ato.forward_backward(st, users, items, sparse, dense, labels)
        p[idx] = old
        return loss

    h = 1e-6
    for k, p in st["params"].items():
        flat = list(np.ndindex(p.shape))
        if k.startswith("mha"):      # every entry of the layer kernels: legacy Wk through the scores AND V = (X Wk) Wv'
            picks = flat
        else:
            picks = [flat[i] for i in rng.choice(len(flat), size=min(6, len(flat)), replace=False)]
        for idx in picks:
            fd = (loss_at(k, idx, h) - loss_at(k, idx, -h)) / (2 * h)
            assert abs(fd - g[k][idx]) <= 1e-7 + 1e-5 * abs(fd), (k, idx, fd, g[k][idx])


def test_steps_reduce_the_loss():
    rng, spec, w = ao.make_case(gt.TRAIN_CASES[1])
    users, items, sparse, dense = ao.case_rows(rng, spec, R=256)
    labels = (rng.random(256) < 0.35).astype(np.float32)
    st = ato.init_state(w)
    losses = [ato.train_step(st, users, items, sparse, dense, labels, 1e-2) for _ in range(6)]
    assert losses[-1] < losses[0] - 1e-3, losses


@pytest.mark.parametrize("scheme", ["keras", "legacy"])
def test_tf_variables_round_trip(tmp_path, scheme):
    from librecommender_b200 import synthetic as syn
    from librecommender_b200 import weights_io as wio

    rng = np.random.default_rng(3)
    spec = syn.make_spec(rng, 30, 40, [5], [7, 3], 1, 1)
    att, H = (4, 8), 2
    w = syn.make_autoint_weights(rng, spec, 8, att, H, False, scheme)
    v = wio.autoint_tf_variables(w)
    names = wio.default_tf_names("AutoInt", None, False, n_layers=2, scheme=scheme)
    assert names["out_kernel"] in v and v[names["out_kernel"]].shape == (np.size(w["out_kernel"]), 1)
    assert all(n in v for ln in names["autoint_mha"] for n in ln.values())
    np.savez(tmp_path / "m_tf_variables.npz", **v)
    got = wio.load_reference_tf_model(str(tmp_path), "m", "AutoInt", None, False, num_heads=H, att_embed_size=att,
                                      use_residual=False)
    ref = wio.autoint_weights(w)
    assert set(got) == set(ref)
    for a, b in zip(got["autoint_layers"], ref["autoint_layers"]):
        for k in ("wq", "wk", "wv", "wo"):
            np.testing.assert_array_equal(a[k], b[k])
    for k in ("user_embeds", "item_embeds", "sparse_embeds", "dense_embeds", "out_kernel"):
        np.testing.assert_array_equal(got[k], ref[k])
    assert got["out_bias"] == ref["out_bias"] and got["num_heads"] == H and got["use_residual"] is False


def _calibrate(ratios, what):
    worst = max(ratios)
    print(f"{what}: float32 uses {worst:.3g} of the bound")
    assert 4.0 * worst <= 1.0, f"{what}: float32 error is not 4x inside the bound ({worst:.3g})"
    assert worst >= 1e-3, f"{what}: bound is over 1000x looser than float32 needs ({worst:.3g})"


def test_attention_kernel_bounds():
    ratios = {n: [] for n in ("O", "lse", "dQ", "dK", "dV")}
    cases = [(gt.make_kernel_case(c), c[2]) for c in gt.KERNEL_CASES]
    cases += [(gt.make_kernel_case(c, large=True), c[2]) for c in [(37, 8, 2, 8), (37, 33, 1, 3)]]
    for (q, k, v, do), H in cases:
        ref = gt.reference(q, k, v, do, H, torch.float64)
        got = gt.reference(q, k, v, do, H, torch.float32)
        for name, g, r, b in zip(ratios, got, ref, gt.bounds(q, k, v, do, H)):
            ratios[name].append(float((np.abs(g.astype(np.float64) - r) / b).max()))
    for name, r in ratios.items():
        _calibrate(r, name)


def test_trainer_bounds():
    ratios = {"logits": [], "loss": [], "gradients": []}
    for c in gt.TRAIN_CASES:
        spec, w, batches = gt.train_batch(c)
        users, items, sparse, dense, labels = batches[0]
        st = ato.init_state(w)
        l64, o64, g64 = ato.forward_backward(st, users, items, sparse, dense, labels)
        l32, o32, g32 = ato.forward_backward(st, users, items, sparse, dense, labels, dtype=torch.float32)
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
    x = np.zeros(64, np.float32)
    p = _lib.ptr(x)
    n0 = _lib.launch_count()
    # (R, F, H, hd, ld): F outside [2, 130], no heads, empty heads, H * hd > 64, a stride below H * hd, R < 0
    for R, F, H, hd, ld in ((4, 131, 1, 8, 8), (4, 1, 1, 8, 8), (4, 8, 0, 8, 8), (4, 8, 2, 0, 8), (4, 8, 5, 13, 65),
                            (4, 8, 2, 8, 15), (-1, 8, 1, 8, 8)):
        assert lib.b200_autoint_attention_forward(p, ld, p, ld, p, ld, R, F, H, hd, 0.5, p, ld, p, None) == -2
        assert b"b200_autoint_attention_forward" in lib.b200_last_error()
        assert lib.b200_autoint_attention_backward(p, ld, p, ld, p, ld, p, ld, p, p, ld, R, F, H, hd, 0.5, p, p, p, ld,
                                                   None) == -2
        assert b"b200_autoint_attention_backward" in lib.b200_last_error()
    assert lib.b200_autoint_attention_forward(p, 8, p, 8, p, 8, 4, 8, 1, 8, float("inf"), p, 8, p, None) == -2
    assert _lib.launch_count() == n0
