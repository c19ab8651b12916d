"""RNN4Rec training without a GPU: the float64 autograd oracle (tests/_rnn4rec_train_oracle.py) against the
inference restatement and central differences, the BPR / norm_embed quirk, the export round trip, the float32
calibration of the GPU bounds and the C-ABI envelope of the new entry points."""
import numpy as np
import pytest
import torch

import _rnn4rec_oracle as inf
import _rnn4rec_train_oracle as ro
from librecommender_b200 import synthetic as syn
from librecommender_b200 import weights_io as wio

N_ITEMS = 20


def raw_weights(scheme, rt, ln, hidden=(6, 5), K=4, seed=0):
    return syn.make_rnn4rec_weights(np.random.default_rng(seed), N_ITEMS, K, hidden, rt, ln, scheme)


def batch(rng, R, T):
    lens = rng.integers(0, T + 1, R)
    lens[0], lens[1], lens[2] = 0, 1, T
    seqs = rng.integers(0, N_ITEMS, (R, T))
    seqs[np.arange(T)[None, :] >= lens[:, None]] = N_ITEMS
    lens[3] = 1
    seqs[3] = N_ITEMS             # a first history position: len 1 holding the pad id
    return seqs, lens, rng.integers(0, N_ITEMS, R), (rng.random(R) < 0.5).astype(np.float64), rng.integers(0, N_ITEMS, R)


GRAPHS = [(s, t, ln) for s in ("keras", "legacy") for t in ("gru", "lstm") for ln in (False, True)
          if not (ln and s == "legacy")]


@pytest.mark.parametrize("scheme,rt,ln", GRAPHS)
def test_oracle_forward_equals_inference_restatement(scheme, rt, ln):
    raw = raw_weights(scheme, rt, ln)
    seqs, lens, *_ = batch(np.random.default_rng(1), 9, 7)
    got = ro.user_vectors(ro.init_params(raw), ro.meta_of(raw), seqs, lens).detach().numpy()
    np.testing.assert_allclose(got, inf.user_vectors(raw, seqs, lens), rtol=1e-12, atol=1e-13)


@pytest.mark.parametrize("scheme,rt,ln", GRAPHS)
@pytest.mark.parametrize("loss_type", ["cross_entropy", "focal", "bpr"])
def test_gradients_match_central_differences(scheme, rt, ln, loss_type):
    raw = raw_weights(scheme, rt, ln, hidden=(3, 2), K=3)
    seqs, lens, items, labels, neg = batch(np.random.default_rng(2), 6, 4)
    y = neg if loss_type == "bpr" else labels
    meta = ro.meta_of(raw)
    P = ro.init_params(raw)
    _, g = ro.forward_backward(P, meta, seqs, lens, items, y, loss_type, norm_embed=True)
    rng = np.random.default_rng(3)
    for k, v in P.items():
        flat = v.reshape(-1)
        for i in rng.choice(flat.numel(), min(6, flat.numel()), replace=False):
            old = float(flat[i])
            h = 1e-6
            flat[i] = old + h
            lp = float(ro.loss(P, meta, seqs, lens, items, y, loss_type, True))
            flat[i] = old - h
            lm = float(ro.loss(P, meta, seqs, lens, items, y, loss_type, True))
            flat[i] = old
            assert abs((lp - lm) / (2 * h) - g[k].reshape(-1)[i]) <= 1e-6 * max(1.0, abs(g[k]).max()), (k, i)


def test_steps_past_len_and_unused_rows_get_zero_gradient():
    raw = raw_weights("keras", "lstm", True)
    T = 6
    seqs, lens, items, labels, _ = batch(np.random.default_rng(4), 8, T)
    meta = ro.meta_of(raw)
    P = ro.init_params(raw)
    _, g = ro.forward_backward(P, meta, seqs, lens, items, labels)
    used = set(seqs[np.arange(T)[None, :] < np.maximum(lens, 0)[:, None]].tolist())
    unused = [r for r in range(N_ITEMS + 1) if r not in used]
    assert unused and np.all(g["seq_embeds"][unused] == 0)
    assert np.any(g["seq_embeds"][N_ITEMS] != 0)        # the pad row of a len-1 first position is trained
    assert np.all(g["item_embeds"][[r for r in range(N_ITEMS) if r not in set(items.tolist())]] == 0)
    # the input at a step past len gets exactly zero gradient
    X = P["seq_embeds"][torch.as_tensor(seqs)].detach().requires_grad_(True)
    P2 = dict(P)
    P2["seq_embeds"] = P["seq_embeds"]
    out = ro.rnn({**P2, "seq_embeds": X.reshape(-1, X.shape[-1])},
                 meta, np.arange(seqs.size).reshape(seqs.shape), lens)
    (gx,) = torch.autograd.grad(out.sum(), X)
    assert np.all(gx.numpy()[np.arange(T)[None, :] >= lens[:, None]] == 0)


def test_bpr_norm_embed_scores_normalised_items_against_the_raw_user():
    raw = raw_weights("keras", "gru", False)
    seqs, lens, items, _, neg = batch(np.random.default_rng(5), 7, 5)
    meta = ro.meta_of(raw)
    P = ro.init_params(raw)
    u = ro.user_vectors(P, meta, seqs, lens)
    n = lambda x: x / torch.linalg.norm(x, dim=1, keepdim=True)    # noqa: E731
    ip, in_ = n(P["item_embeds"][items]), n(P["item_embeds"][neg])
    b = P["item_biases"]
    quirk = -torch.nn.functional.logsigmoid((b[items] - b[neg]) + (u * (ip - in_)).sum(1)).mean()
    both = -torch.nn.functional.logsigmoid((b[items] - b[neg]) + (n(u) * (ip - in_)).sum(1)).mean()
    got = ro.loss(P, meta, seqs, lens, items, neg, "bpr", True)
    assert float(got) == float(quirk) and abs(float(got) - float(both)) > 1e-3


@pytest.mark.parametrize("scheme,rt,ln", GRAPHS)
def test_export_round_trip_is_exact(scheme, rt, ln):
    raw = raw_weights(scheme, rt, ln)
    can = wio.rnn_layers(raw["rnn_layers"], scheme, rt, 6, raw["use_layer_norm"])
    back = wio.rnn_raw_layers(can, scheme, rt, 6)
    for a, b in zip(raw["rnn_layers"], back):
        assert set(a) == set(b)
        for k in a:
            a32 = np.asarray(a[k], np.float32).reshape(b[k].shape)
            if scheme == "legacy" and rt == "lstm" and k == "bias":
                H = b[k].size // 4
                f = slice(2 * H, 3 * H)            # the folded forget bias: fl32(fl32(b + 1) - 1)
                np.testing.assert_array_equal(b[k][f], (a32[f] + np.float32(1)) - np.float32(1))
                keep = np.r_[0:2 * H, 3 * H:4 * H]
                np.testing.assert_array_equal(b[k][keep], a32[keep])
            else:
                np.testing.assert_array_equal(b[k], a32)


def test_float32_restatement_meets_gpu_bounds():
    """The GPU bounds of test_gpu_rnn4rec_train.py hold for a float32 restatement with 4x to spare and are not more
    than 1000x loose."""
    import test_gpu_rnn4rec_train as gt

    worst = 0.0
    for scheme, rt, ln in GRAPHS:
        for loss_type in ("cross_entropy", "bpr"):
            raw = raw_weights(scheme, rt, ln, hidden=(16, 8), K=8)
            seqs, lens, items, labels, neg = batch(np.random.default_rng(6), 64, 20)
            y = neg if loss_type == "bpr" else labels
            meta = ro.meta_of(raw)
            _, g64 = ro.forward_backward(ro.init_params(raw), meta, seqs, lens, items, y, loss_type, True)
            _, g32 = ro.forward_backward(ro.init_params(raw, torch.float32), meta, seqs, lens, items, y, loss_type,
                                         True)
            gmax = max(np.abs(v).max() for v in g64.values())
            for k in g64:
                bound = gt.GRAD_REL * np.abs(g64[k]).max() + gt.GRAD_ABS * gmax
                err = np.abs(g32[k].astype(np.float64) - g64[k]).max()
                assert err * 4 <= bound, (scheme, rt, ln, k, err, bound)
                worst = max(worst, err / bound)
    assert worst * 1000 >= 1.0, worst


def test_cabi_rejects_out_of_envelope_before_launch():
    import ctypes

    from librecommender_b200 import _lib

    L = lambda *v: (ctypes.c_int32 * len(v))(*v)      # noqa: E731
    n0 = _lib.launch_count()
    fwd = _lib.lib.b200_rnn_train_forward
    for T, d, hid, kind, act in ((0, 8, 8, 0, 0), (129, 8, 8, 0, 0), (10, 257, 8, 0, 0), (10, 8, 257, 0, 0),
                                 (10, 8, 8, 3, 0), (10, 8, 8, 0, 2)):
        assert fwd(None, 4, None, None, T, T, None, d, d, 1, L(kind), L(hid), L(act), None, None, hid, None, None) == -2
        assert _lib.lib.b200_rnn_backward(None, 4, None, T, kind, d, hid, act, None, None, hid, None, None, None, None,
                                          None, None, None) == -2
    five = L(0, 0, 0, 0, 0)
    assert fwd(None, 4, None, None, 10, 10, None, 8, 8, 5, five, L(8, 8, 8, 8, 8), five, None, None, 8, None,
               None) == -2
    assert _lib.lib.b200_rnn_backward(None, 0, None, 10, 0, 8, 8, 0, None, None, 8, None, None, None, None, None, None,
                                      None) == 0
    assert _lib.launch_count() == n0
