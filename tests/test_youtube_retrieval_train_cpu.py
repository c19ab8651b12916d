"""CPU: YouTubeRetrieval training without a GPU.

* the host restatement of the unique candidate sampler: ids distinct and in range, ``num_tries == S`` when no draw
  collides, ``S = n_items`` yields every id, the log-uniform probabilities sum to 1, expected counts;
* the float64 training restatement (``tests/_youtube_retrieval_train_oracle.py``): autograd against central
  differences; with the uniform sampler, ``S = n_items`` and no BN, the sampled softmax equals the full-catalogue
  softmax cross entropy built from ``oracle.tf_models.youtube_retrieval_user_vectors``;
* calibration of the GPU bounds of ``test_gpu_youtube_retrieval_train.py``: a float32 restatement meets each with 4x
  to spare and uses at least 1/1000 of it;
* the ``weights_io`` round trip and its rejections; the C-ABI rejects calls outside the envelope before launching."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _youtube_retrieval_train_oracle as yo  # noqa: E402
import test_gpu_youtube_retrieval_train as gt  # noqa: E402


@pytest.mark.parametrize("kind", [0, 1])
@pytest.mark.parametrize("S,n_items", [(1, 1), (7, 7), (64, 1000), (500, 600), (2000, 1 << 30)])
def test_sampler_restatement_properties(kind, S, n_items):
    ids, tries, _ = yo.unique_candidates(kind, n_items, S, 11, 5)
    assert len(ids) == S and len(np.unique(ids)) == S and ids.min() >= 0 and ids.max() < n_items
    assert tries >= S
    all_draws, _ = yo.draws(kind, n_items, 11, 5, np.arange(tries))
    assert all_draws[-1] == ids[-1] and set(all_draws.tolist()) == set(ids.tolist())
    if len(np.unique(all_draws[:S])) == S:
        assert tries == S
    if S == n_items:
        assert sorted(ids.tolist()) == list(range(n_items))
    nxt, _, _ = yo.unique_candidates(kind, n_items, S, 11, 6)
    assert S == n_items or not np.array_equal(nxt, ids)


def test_uniform_draws_are_uniform_and_log_uniform_probabilities_sum_to_one():
    ids, _ = yo.draws(0, 10, 1, 0, np.arange(200_000))
    np.testing.assert_allclose(np.bincount(ids, minlength=10) / 2e5, 0.1, atol=4e-3)
    for n in (1, 10, 3200, 1_000_000):
        assert abs(yo.probabilities(1, np.arange(n), n).sum() - 1.0) < 1e-9
    ids, _ = yo.draws(1, 50, 2, 0, np.arange(400_000))
    np.testing.assert_allclose(np.bincount(ids, minlength=50) / 4e5, yo.probabilities(1, np.arange(50), 50), atol=3e-3)


def test_expected_counts():
    e = yo.expected_counts(0, np.arange(5), 100, 10, 10)
    np.testing.assert_allclose(e, 0.1, rtol=1e-12)                    # p S without collisions
    e = yo.expected_counts(0, np.arange(5), 100, 10, 13)
    np.testing.assert_allclose(e, 1 - (1 - 0.01) ** 13, rtol=1e-12)   # P(drawn at least once in 13 tries)
    e32 = yo.expected_counts(1, np.arange(5), 100, 10, 13, np.float32)
    assert e32.dtype == np.float32
    np.testing.assert_allclose(e32, yo.expected_counts(1, np.arange(5), 100, 10, 13), rtol=1e-6)


@pytest.mark.parametrize("loss_type", ["sampled_softmax", "nce"])
@pytest.mark.parametrize("norm", [False, True])
def test_gradients_match_central_differences(loss_type, norm):
    spec, w, consumed, (users, items) = gt.make_case(5, n_users=12, n_items=15, K=3, hidden=(5, 4), B=9, T=3)
    seqs, lens = gt.reference_windows(consumed, users, items, 3, 15)
    sampled, tries, _ = yo.unique_candidates(1, 15, 6, 3, 0)
    sampled[0] = items[0]                                  # an accidental hit
    st = yo.init_state(w, True)
    args = (spec, users, items, seqs, lens, sampled, tries, loss_type, 1, norm)
    _, g, _, _ = yo.forward_backward(st, *args)
    rng = np.random.default_rng(0)

    def loss_at(k, idx, delta):
        p = st["params"][k]
        old = p[idx]
        p[idx] = old + delta
        loss = yo.forward_backward(st, *args)[0]
        p[idx] = old
        return loss

    h = 1e-6
    for k, p in st["params"].items():
        flat = list(np.ndindex(p.shape))
        picks = [flat[i] for i in rng.choice(len(flat), size=min(6, len(flat)), replace=False)]
        if k == "item_embeds":
            picks += [(int(items[0]), 0), (int(sampled[1]), 1)]
        for idx in picks:
            fd = (loss_at(k, idx, h) - loss_at(k, idx, -h)) / (2 * h)
            assert abs(fd - g[k][idx]) <= 1e-7 + 1e-5 * abs(fd), (k, idx, fd, g[k][idx])


def test_full_catalogue_sampled_softmax_is_full_softmax():
    from oracle import tf_models as tm

    n_items, T = 40, 4
    spec, w, consumed, (users, items) = gt.make_case(8, n_users=30, n_items=n_items, use_bn=False, B=30, T=T)
    users = np.arange(30)
    items = np.array([consumed[u][-1] for u in users])
    seqs, lens = gt.reference_windows(consumed, users, items, T, n_items)
    sampled, tries, _ = yo.unique_candidates(0, n_items, n_items, 1, 0)
    assert tries > n_items                                  # collisions: the -expm1 branch of the expected count
    st = yo.init_state(w, False)
    loss, _, _, _ = yo.forward_backward(st, spec, users, items, seqs, lens, sampled, tries)
    U = tm.youtube_retrieval_user_vectors(w, spec, users, seqs, lens, dtype=np.float64)   # seqs / lens per row here
    z = U @ w["item_embeds"].astype(np.float64).T + w["item_biases"].astype(np.float64)[None]
    ref = np.mean(np.log(np.exp(z - z.max(1, keepdims=True)).sum(1)) + z.max(1) - z[np.arange(30), items])
    assert abs(loss - ref) <= 1e-10 * max(1.0, abs(ref)), (loss, ref)


def _calibrate(ratios, what):
    worst = max(ratios)
    print(f"{what}: float32 uses {worst:.3g} of the bound")
    assert 4.0 * worst <= 1.0, f"{what}: float32 error is not 4x inside the bound ({worst:.3g})"
    assert worst >= 1e-3, f"{what}: bound is over 1000x looser than float32 needs ({worst:.3g})"


def test_gpu_bounds_calibration():
    ratios = {"loss": [], "gradients": []}
    for loss_type, norm, use_bn, fields, kind, S in gt.CASES:
        T, n_items = 5, 300
        spec, w, consumed, (users, items) = gt.make_case(7 + S, use_bn=use_bn, fields=fields, T=T, n_items=n_items)
        seqs, lens = gt.reference_windows(consumed, users, items, T, n_items)
        sampled, tries, _ = yo.unique_candidates(kind, n_items, S, 42, 0)
        st = yo.init_state(w, use_bn)
        args = (spec, users, items, seqs, lens, sampled, tries, loss_type, kind, norm)
        l64, g64, _, _ = yo.forward_backward(st, *args)
        l32, g32, _, _ = yo.forward_backward(st, *args, dtype=torch.float32)
        ratios["loss"].append(abs(l32 - l64) / (gt.LOSS_REL * max(1.0, abs(l64))))
        gmax = max(np.abs(v).max() for v in g64.values())
        ratios["gradients"].append(max(float(np.abs(g32[k] - g64[k]).max()
                                             / (gt.GRAD_REL * np.abs(g64[k]).max() + gt.GRAD_ABS * gmax)) for k in g64))
    for name, r in ratios.items():
        _calibrate(r, name)


def test_tf_variables_round_trip_and_rejections(tmp_path):
    from librecommender_b200 import weights_io as wio

    spec, w, _, _ = gt.make_case(4, hidden=(24, 12, 16))
    v = wio.youtube_retrieval_tf_variables(w)
    for name in ("embedding/seq_embeds_var:0", "embedding/item_embeds_var:0", "embedding/item_bias_var:0",
                 "embedding/sparse_embeds_var:0", "embedding/dense_embeds_var:0", "mlp/mlp_layer3/kernel:0",
                 "mlp/batch_normalization_2/moving_variance:0"):
        assert name in v, name
    assert v["embedding/item_bias_var:0"].shape == (300,)
    np.savez(tmp_path / "m_tf_variables.npz", **v)
    got = wio.load_reference_tf_model(str(tmp_path), "m", "YouTubeRetrieval", 3, True)
    for k in ("seq_embeds", "item_embeds", "item_biases", "sparse_embeds", "dense_embeds"):
        np.testing.assert_array_equal(got[k], w[k])
    for i in range(3):
        np.testing.assert_array_equal(got["mlp"]["kernels"][i], w["mlp"]["kernels"][i])
        np.testing.assert_array_equal(got["mlp"]["biases"][i], w["mlp"]["biases"][i])
    np.testing.assert_array_equal(got["mlp"]["bns"][1]["var"], w["mlp"]["bns"][1]["var"])
    with pytest.raises(KeyError, match="mlp_layer4"):
        wio.load_reference_tf_model(str(tmp_path), "m", "YouTubeRetrieval", 4, True)
    with pytest.raises(KeyError, match="batch_normalization"):
        np.savez(tmp_path / "nobn_tf_variables.npz", **{k: a for k, a in v.items() if "batch_norm" not in k})
        wio.load_reference_tf_model(str(tmp_path), "nobn", "YouTubeRetrieval", 3, True)
    bad = dict(v)
    bad["embedding/item_embeds_var:0"] = bad["embedding/item_embeds_var:0"][:, :-1]
    np.savez(tmp_path / "bad_tf_variables.npz", **bad)
    with pytest.raises(KeyError, match="item_embeds_var"):
        wio.load_reference_tf_model(str(tmp_path), "bad", "YouTubeRetrieval", 3, True)
    bad = dict(v)
    bad["embedding/item_bias_var:0"] = bad["embedding/item_bias_var:0"][:-1]
    np.savez(tmp_path / "bad2_tf_variables.npz", **bad)
    with pytest.raises(KeyError, match="item_bias_var"):
        wio.load_reference_tf_model(str(tmp_path), "bad2", "YouTubeRetrieval", 3, True)


def test_cabi_rejects_outside_the_envelope_before_launch():
    from librecommender_b200 import _lib

    lib = _lib.lib
    x = np.zeros(64, np.int64)
    p = _lib.ptr(x)
    n0 = _lib.launch_count()
    # (kind, n_items, S, workspace bytes)
    for kind, n, S, wsb in ((2, 100, 10, 400), (0, 0, 1, 400), (0, 1 << 31, 10, 1 << 40), (0, 100, 0, 400),
                            (1, 100, 101, 400), (0, 100_000, 65_537, 400_000), (0, 100, 10, 399)):
        assert lib.b200_unique_candidates(kind, n, S, 1, p, p, wsb, p, p, None) == -2
        assert b"b200_unique_candidates" in lib.b200_last_error()
    assert lib.b200_unique_candidates(0, 100, 10, 1, p, None, 400, p, p, None) == -2
    wsb = lib.b200_sampled_class_loss_workspace_bytes(8, 4)
    # (loss kind, sampler kind, B, S, ld, n_items)
    for lk, sk, B, S, ld, n in ((2, 0, 8, 4, 4, 100), (0, 2, 8, 4, 4, 100), (0, 0, 0, 4, 4, 100), (1, 0, 8, 4, 3, 100),
                                (0, 1, 8, 4, 4, 3), (0, 0, 8, 65_537, 65_537, 100_000)):
        assert lib.b200_sampled_class_loss(lk, p, ld, B, S, p, p, p, p, sk, n, p, p, p, p, 1 << 30, None) == -2
        assert b"b200_sampled_class_loss" in lib.b200_last_error()
    assert lib.b200_sampled_class_loss(0, p, 4, 8, 4, p, p, p, p, 0, 100, p, p, p, p, wsb - 1, None) == -2
    assert _lib.launch_count() == n0
