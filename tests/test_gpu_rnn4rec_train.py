"""RNN4Rec training on the GPU: the training forward against b200_rnn_encode (bit for bit) and its saved tensors
against float64, the BPTT backward and one full step against the float64 autograd oracle
(tests/_rnn4rec_train_oracle.py), Adam steps, CUDA-graph replay, export into the serving model, the regulariser and
the errors raised before any launch."""
import ctypes

import numpy as np
import pytest

import _rnn4rec_train_oracle as ro

pytestmark = pytest.mark.gpu

# gradients: |got - ref| <= GRAD_REL * max|ref of the variable| + GRAD_ABS * (largest gradient of the batch), calibrated
# in test_rnn4rec_train_cpu.py::test_float32_restatement_meets_gpu_bounds
GRAD_REL, GRAD_ABS = 5e-4, 1e-5
SAVED_ATOL = 2e-4


def _cu(a):
    import torch

    return torch.as_tensor(np.asarray(a)).cuda()


def make_batch(rng, n_items, R, T):
    """seqs [R, T] padded with n_items, lens with 0, 1 and T present; rows 0..3 are a first history position (len 1,
    the pad id); items / labels / negatives."""
    lens = rng.integers(0, T + 1, R).astype(np.int32)
    lens[4:6] = T
    lens[6:8] = 0
    lens[8:10] = 1
    seqs = rng.integers(0, n_items, (R, T)).astype(np.int32)
    seqs[np.arange(T)[None, :] >= lens[:, None]] = n_items
    lens[:4] = 1
    seqs[:4] = n_items
    items = rng.integers(0, n_items, R)
    return seqs, lens, items, (rng.random(R) < 0.4).astype(np.float32), rng.integers(0, n_items, R)


def raw_weights(scheme, rnn_type, ln, hidden, n_items=60, K=8, seed=0):
    from librecommender_b200 import synthetic as syn

    return syn.make_rnn4rec_weights(np.random.default_rng(seed), n_items, K, hidden, rnn_type, ln, scheme)


def trainer(raw, n_items=60, **kw):
    from librecommender_b200.training import RNN4RecTrainer

    return RNN4RecTrainer({"n_users": 10, "n_items": n_items}, raw, **kw)


# ---------------------------------------------------------------------------------------------------------------
# the training forward
# ---------------------------------------------------------------------------------------------------------------
def _sig(x):
    return 1.0 / (1.0 + np.exp(-x))


def canonical_saved(layers, X, lens):
    """float64 restatement of what b200_rnn_train_forward saves, per layer [n, T, .]: h_{t-1}, y_t, the gates, the
    cell block, x^ and rstd (rows t >= len are 0)."""
    n, T, _ = X.shape
    seq, out = X, []
    for lw in layers:
        kind, act = int(lw["kind"]), int(lw["act"])
        W, U, bx, bh = (np.asarray(lw[k], np.float64) for k in ("W", "U", "bx", "bh"))
        H = U.shape[0]
        G = 4 if kind == 2 else 3
        a = (lambda v: v) if act else np.tanh
        h, c = np.zeros((n, H)), np.zeros((n, H))
        sv = dict(hp=np.zeros((n, T, H)), y=np.zeros((n, T, H)), g=np.zeros((n, T, G * H)), x=np.zeros((n, T, H)),
                  xh=np.zeros((n, T, H)), rs=np.zeros((n, T)))
        ys = np.zeros((n, T, H))
        for t in range(T):
            live = t < lens
            ax = seq[:, t] @ W + bx
            if kind == 2:
                m = ax + h @ U + bh
                i, f, o = _sig(m[:, :H]), _sig(m[:, H:2 * H]), _sig(m[:, 3 * H:])
                g = a(m[:, 2 * H:3 * H])
                nc = f * c + i * g
                nh, gates, blk = o * a(nc), np.hstack([i, f, g, o]), nc
            elif kind == 0:
                ah = h @ U + bh
                z, r = _sig(ax[:, :H] + ah[:, :H]), _sig(ax[:, H:2 * H] + ah[:, H:2 * H])
                hh = a(ax[:, 2 * H:] + r * ah[:, 2 * H:])
                nh, nc, gates, blk = z * h + (1 - z) * hh, c, np.hstack([z, r, hh]), ah[:, 2 * H:]
            else:
                ah = h @ U[:, :2 * H] + bh[:2 * H]
                z, r = _sig(ax[:, :H] + ah[:, :H]), _sig(ax[:, H:2 * H] + ah[:, H:])
                rh = r * h
                cc = a(ax[:, 2 * H:] + rh @ U[:, 2 * H:] + bh[2 * H:])
                nh, nc, gates, blk = z * h + (1 - z) * cc, c, np.hstack([z, r, cc]), rh
            hp = h
            h = np.where(live[:, None], nh, h)
            c = np.where(live[:, None], nc, c)
            if act:
                mean = h.mean(1, keepdims=True)
                rs = 1 / np.sqrt(((h - mean) ** 2).mean(1, keepdims=True) + 1e-3)
                xh = (h - mean) * rs
                y = np.tanh(xh * np.asarray(lw["gamma"], np.float64) + np.asarray(lw["beta"], np.float64))
            else:
                y = h
            ys[:, t] = y
            L = live
            sv["hp"][L, t], sv["y"][L, t], sv["g"][L, t], sv["x"][L, t] = hp[L], y[L], gates[L], blk[L]
            if act:
                sv["xh"][L, t], sv["rs"][L, t] = xh[L], rs[L, 0]
        out.append(sv)
        seq = ys
    return out


FWD_CASES = [  # (scheme, rnn_type, ln, hidden, T)
    ("keras", "gru", False, (16,), 1), ("keras", "gru", True, (16, 12), 10), ("keras", "lstm", False, (24,), 50),
    ("keras", "lstm", True, (8, 8, 8), 128), ("legacy", "gru", False, (16, 16), 10), ("legacy", "gru", False, (32,), 128),
    ("legacy", "lstm", False, (16,), 10), ("legacy", "lstm", False, (12, 20), 50), ("keras", "gru", True, (40,), 50),
    ("legacy", "lstm", False, (8, 8, 8, 8), 1),
]


@pytest.mark.parametrize("c", FWD_CASES, ids=lambda c: "-".join(map(str, c)))
def test_training_forward_equals_encode_and_saves_float64(c):
    import torch

    from librecommender_b200 import _lib
    from librecommender_b200.feat_models import RNN4Rec

    scheme, rt, ln, hidden, T = c
    raw = raw_weights(scheme, rt, ln, hidden)
    rng = np.random.default_rng(1)
    seqs, lens, *_ = make_batch(rng, 60, 203, T)
    tr = trainer(raw)
    h, cache = tr.encode(_cu(seqs), _cu(lens))
    model = RNN4Rec({"n_users": 203, "n_items": 60}, raw, seqs, lens)
    ref = model.encode(torch.arange(203, device="cuda"))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(h.cpu().numpy(), ref.cpu().numpy())
    X = np.asarray(raw["seq_embeds"], np.float64)[seqs]
    exp = canonical_saved(tr.canonical_layers(), X, np.clip(lens, 0, T))
    for l, (sv, e) in enumerate(zip(cache["saved"], exp)):
        for k, got in zip(("hp", "y", "g", "x", "xh", "rs"), sv):
            if got is None:
                continue
            g = got.cpu().numpy().reshape(e[k].shape)
            np.testing.assert_allclose(g, e[k], rtol=0, atol=SAVED_ATOL * max(1.0, np.abs(e[k]).max()),
                                       err_msg=f"layer {l} {k}")
            assert np.all(g[np.arange(T)[None, :] >= lens[:, None]] == 0)
    assert _lib.lib.b200_rnn_train_forward(None, 0, None, None, T, T, None, 16, 16, len(hidden), tr._kinds, tr._hid,
                                           tr._acts, None, None, 16, None, None) == 0


# ---------------------------------------------------------------------------------------------------------------
# gradients of one step against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------
def trainer_grads(tr, raw):
    """The trainer's gradients in the raw layout of its graph."""
    from librecommender_b200.weights_io import rnn_raw_layers

    g = {k: v.cpu().numpy().astype(np.float64) for k, v in tr.grads.items()}
    canon = []
    for l, lw in enumerate(tr.canonical_layers()):
        pre = f"rnn{l}_"
        canon.append(dict(kind=lw["kind"], act=lw["act"], W=g[pre + "W"], U=g[pre + "U"], bx=g[pre + "bx"],
                          bh=g.get(pre + "bh", np.zeros_like(g[pre + "bx"])),
                          gamma=g.get(pre + "gamma", np.zeros(lw["U"].shape[0])),
                          beta=g.get(pre + "beta", np.zeros(lw["U"].shape[0]))))
    out = {k: g[k] for k in ro.TABLES}
    out["dense_kernel"], out["dense_bias"] = g["dense_Wt"].T, g["dense_b"]
    for i, lw in enumerate(rnn_raw_layers(canon, tr.scheme, tr.rnn_type, tr.in_dim, forget_bias=0.0)):
        for k, v in lw.items():
            out[f"rnn{i}_{k}"] = v
    return out


def check_grads(got, ref):
    gmax = max(np.abs(v).max() for v in ref.values())
    assert set(got) == set(ref)
    for k, r in ref.items():
        a = np.asarray(got[k], np.float64).reshape(r.shape)
        err = np.abs(a - r).max()
        assert err <= GRAD_REL * np.abs(r).max() + GRAD_ABS * gmax, (k, float(err), float(np.abs(r).max()), gmax)


STEP_CASES = [  # (scheme, rnn_type, ln, hidden, T, loss, norm_embed)
    ("keras", "gru", False, (16,), 10, "cross_entropy", False), ("keras", "gru", True, (16, 8), 10, "focal", True),
    ("keras", "lstm", True, (16,), 20, "bpr", False), ("keras", "lstm", False, (12, 12), 10, "bpr", True),
    ("legacy", "gru", False, (16, 8), 10, "cross_entropy", True), ("legacy", "gru", False, (16,), 30, "bpr", True),
    ("legacy", "lstm", False, (16,), 10, "focal", False), ("legacy", "lstm", False, (8, 16), 10, "bpr", False),
    ("keras", "gru", False, (16,), 1, "cross_entropy", False), ("keras", "lstm", True, (16,), 10, "cross_entropy", True),
]


@pytest.mark.parametrize("c", STEP_CASES, ids=lambda c: "-".join(map(str, c)))
def test_gradients_of_one_step_match_oracle(c):
    import torch

    scheme, rt, ln, hidden, T, loss_type, ne = c
    raw = raw_weights(scheme, rt, ln, hidden)
    seqs, lens, items, labels, neg = make_batch(np.random.default_rng(2), 60, 203, T)
    y = neg if loss_type == "bpr" else labels
    tr = trainer(raw, loss_type=loss_type, norm_embed=ne)
    loss = tr.forward_backward(_cu(items), _cu(seqs), _cu(lens), _cu(y))
    torch.cuda.synchronize()
    meta = ro.meta_of(raw)
    ref_loss, ref = ro.forward_backward(ro.init_params(raw), meta, seqs, lens, items, y, loss_type, ne)
    assert abs(float(loss) - ref_loss) <= 2e-5 * max(1.0, abs(ref_loss))
    check_grads(trainer_grads(tr, raw), ref)


def test_backward_kernel_at_the_envelope_maximum():
    """Four LSTM layers of 256 with layer norm, T = 128, a few rows."""
    import torch

    raw = raw_weights("keras", "lstm", True, (256, 256, 256, 256), K=8)
    seqs, lens, items, labels, _ = make_batch(np.random.default_rng(3), 60, 12, 128)
    tr = trainer(raw)
    loss = tr.forward_backward(_cu(items), _cu(seqs), _cu(lens), _cu(labels))
    torch.cuda.synchronize()
    ref_loss, ref = ro.forward_backward(ro.init_params(raw), ro.meta_of(raw), seqs, lens, items, labels)
    assert abs(float(loss) - ref_loss) <= 2e-5 * max(1.0, abs(ref_loss))
    check_grads(trainer_grads(tr, raw), ref)


def test_backward_kernel_is_bit_identical_on_repeat_and_zero_past_len():
    import torch

    from librecommender_b200 import _lib

    raw = raw_weights("legacy", "gru", False, (16, 16))
    seqs, lens, *_ = make_batch(np.random.default_rng(4), 60, 77, 20)
    tr = trainer(raw)
    h, c = tr.encode(_cu(seqs), _cu(lens))
    dout = torch.randn(h.shape, device="cuda")
    outs = []
    for _ in range(2):
        H, S = 16, 77 * 20
        dgx = torch.full((S, 48), 7.0, device="cuda")
        table = (ctypes.c_void_p * 6)(*[t.data_ptr() if t is not None else None for t in c["saved"][1]])
        _lib.check(_lib.lib.b200_rnn_backward(_lib.ptr(c["rows"]), 77, _lib.ptr(c["lens"]), 20, 1, H, H, 0,
                                              _lib.ptr(tr.rnn_w[tr._offs[1]:]), _lib.ptr(dout), dout.stride(0), None,
                                              table, _lib.ptr(dgx), None, None, None, _lib.current_stream()))
        outs.append(dgx.cpu().numpy().reshape(77, 20, 48))
    np.testing.assert_array_equal(outs[0], outs[1])
    assert np.all(outs[0][np.arange(20)[None, :] >= lens[:, None]] == 0)
    assert np.all(np.isfinite(outs[0]))


# ---------------------------------------------------------------------------------------------------------------
# steps, graphs, export, regulariser, errors
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", [STEP_CASES[1], STEP_CASES[4], STEP_CASES[7]], ids=lambda c: "-".join(map(str, c)))
def test_adam_steps_track_oracle_and_loss_falls(c):
    scheme, rt, ln, hidden, T, loss_type, ne = c
    raw = raw_weights(scheme, rt, ln, hidden)
    rng = np.random.default_rng(5)
    batches = [make_batch(rng, 60, 256, T) for _ in range(3)]
    lr, eps = 1e-2, 1e-5
    tr = trainer(raw, loss_type=loss_type, norm_embed=ne, lr=lr, epsilon=eps)
    st = ro.init_state(raw)
    meta = ro.meta_of(raw)
    for step, (seqs, lens, items, labels, neg) in enumerate(batches):
        y = neg if loss_type == "bpr" else labels
        ref_loss = ro.train_step(st, meta, seqs, lens, items, y, lr, eps, loss_type, ne)
        loss = float(tr.step(_cu(np.zeros(256, np.int64)), _cu(items), _cu(seqs), _cu(lens), _cu(y)))
        assert abs(loss - ref_loss) <= 1e-3 * max(1.0, abs(ref_loss)) * (step + 1), (step, loss, ref_loss)
    exported = tr.export_weights()
    ref_raw = ro.raw_of(st["P"], raw)
    for k in ro.TABLES + ("dense_kernel", "dense_bias"):
        assert np.abs(np.asarray(exported[k], np.float64).reshape(np.shape(ref_raw[k])) - ref_raw[k]).max() <= 3e-2 * lr
    for a, b in zip(exported["rnn_layers"], ref_raw["rnn_layers"]):
        for k in b:
            assert np.abs(a[k].astype(np.float64).reshape(b[k].shape) - b[k]).max() <= 3e-2 * lr, k
    # on one repeated synthetic batch the loss goes down
    seqs, lens, items, labels, neg = batches[0]
    y = neg if loss_type == "bpr" else labels
    first = float(tr.step(_cu(items), _cu(items), _cu(seqs), _cu(lens), _cu(y)))
    for _ in range(30):
        last = float(tr.step(_cu(items), _cu(items), _cu(seqs), _cu(lens), _cu(y)))
    assert last < first


def test_graph_replay_and_fresh_trainers_agree():
    raw = raw_weights("keras", "gru", True, (16, 8))
    rng = np.random.default_rng(6)
    batches = [make_batch(rng, 60, 200, 10) for _ in range(3)]
    a, b, c = (trainer(raw, lr=1e-2) for _ in range(3))
    for i, (seqs, lens, items, labels, _) in enumerate(batches):
        args = [_cu(x) for x in (np.zeros(200, np.int64), items, seqs, lens, labels)]
        la, lb, lc = float(a.step(*args)), float(b.step_graph(*args)), float(c.step(*args))
        assert abs(la - lb) <= 1e-5 * max(1.0, abs(la)) and abs(la - lc) <= 1e-5 * max(1.0, abs(la))
        if i == 0:
            # after one step everything but the atomically scattered tables is bit-identical
            for k in a.params:
                if k not in ro.TABLES:
                    np.testing.assert_array_equal(a.params[k].cpu().numpy(), b.params[k].cpu().numpy(), err_msg=k)
                    np.testing.assert_array_equal(a.params[k].cpu().numpy(), c.params[k].cpu().numpy(), err_msg=k)
    assert b.graph_launches_per_step > 20 and int(b._step_dev.item()) == 3
    for k in a.params:
        assert (a.params[k] - b.params[k]).abs().max().item() <= 2e-4, k      # float atomics in the table scatters
        assert (a.params[k] - c.params[k]).abs().max().item() <= 2e-4, k


@pytest.mark.parametrize("scheme,rt,ln", [("keras", "gru", False), ("keras", "lstm", True), ("legacy", "gru", False),
                                          ("legacy", "lstm", False)])
def test_export_serves_bit_identically_and_round_trips_tf_variables(scheme, rt, ln, tmp_path):
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import RNN4Rec

    raw = raw_weights(scheme, rt, ln, (16, 12))
    seqs, lens, items, labels, _ = make_batch(np.random.default_rng(7), 60, 120, 10)
    tr = trainer(raw, lr=1e-2, norm_embed=True)
    for _ in range(2):
        tr.step(_cu(items), _cu(items), _cu(seqs), _cu(lens), _cu(labels))
    exp = tr.export_weights()
    model = RNN4Rec({"n_users": 120, "n_items": 60}, exp, seqs, lens, norm_embed=False)
    u, _ = tr.user_vectors(_cu(seqs), _cu(lens))
    np.testing.assert_array_equal(model.user_vectors(np.arange(120)).cpu().numpy(), u.cpu().numpy())
    np.savez(tmp_path / "m_tf_variables.npz", **wio.rnn4rec_tf_variables(exp))
    back = wio.load_reference_tf_model(str(tmp_path), "m", "RNN4Rec", 0, False, rnn_type=rt, hidden_units=(16, 12),
                                       use_layer_norm=ln)
    ref = wio.rnn4rec_weights(exp)
    for k in ("seq_embeds", "item_embeds", "item_biases", "dense_kernel", "dense_bias"):
        np.testing.assert_array_equal(back[k], ref[k])
    for a, b in zip(back["rnn_layers"], ref["rnn_layers"]):
        for k in ("W", "U", "bx", "bh", "gamma", "beta"):
            np.testing.assert_array_equal(a[k], b[k])
    # served end to end with no TensorFlow: embeddings, then retrieval
    U, I = RNN4Rec({"n_users": 120, "n_items": 60}, exp, seqs, lens, norm_embed=True).set_embeddings()
    assert U.shape == (121, 9) and I.shape == (61, 9) and bool(U.isfinite().all())


def test_regularisation_adds_2_reg_w_to_the_tables_only():
    from librecommender_b200.training import set_regularisation

    raw = raw_weights("keras", "gru", False, (16,))
    seqs, lens, items, labels, _ = make_batch(np.random.default_rng(8), 60, 100, 10)
    args = [_cu(x) for x in (items, items, seqs, lens, labels)]
    lr, eps, reg = 1e-2, 1e-5, 3e-3
    plain = trainer(raw, lr=lr, epsilon=eps)
    tr = set_regularisation(trainer(raw, lr=lr, epsilon=eps), reg=reg)
    assert tr.reg_vars == ("seq_embeds", "item_embeds", "item_biases")
    st = ro.init_state(raw)
    ro.train_step(st, ro.meta_of(raw), seqs, lens, items, labels, lr, eps, reg=reg)
    tr.step(*args)
    plain.step(*args)
    ref = ro.raw_of(st["P"], raw)
    for k in ro.TABLES:
        got = tr.params[k].cpu().numpy().astype(np.float64).reshape(np.shape(ref[k]))
        assert np.abs(got - ref[k]).max() <= 2e-2 * lr, k
        assert (tr.params[k] - plain.params[k]).abs().max().item() > 0.1 * lr or k == "item_biases"
    for k in tr.params:         # the other variables see the same gradients: the same bits after one step
        if k not in ro.TABLES:
            np.testing.assert_array_equal(tr.params[k].cpu().numpy(), plain.params[k].cpu().numpy(), err_msg=k)


@pytest.mark.parametrize("what", ["loss", "rnn_type", "scheme", "rows", "rating", "T", "width", "layers", "memory"])
def test_trainer_rejects_before_launch(what):
    from librecommender_b200 import _lib

    raw = raw_weights("keras", "gru", False, (16,))
    kw, T = {}, 10
    if what == "loss":
        kw["loss_type"] = "softmax"
    elif what == "rnn_type":
        raw["rnn_type"] = "rnn"
    elif what == "scheme":
        raw["rnn_scheme"] = "tf3"
    elif what == "rows":
        raw["seq_embeds"] = raw["seq_embeds"][:-1]
    elif what == "rating":
        kw["task"] = "rating"
    elif what == "width":
        raw = raw_weights("keras", "gru", False, (16, 300))
    elif what == "layers":
        raw = raw_weights("keras", "gru", False, (8,) * 5)
    elif what == "T":
        T = 129
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        tr = trainer(raw, **kw)
        B = 4 if what != "memory" else 1 << 40
        if what == "memory":
            tr._check_batch(B, T)
        seqs = np.zeros((4, T), np.int32)
        tr.step(_cu(np.zeros(4, np.int64)), _cu(np.zeros(4, np.int64)), _cu(seqs), _cu(np.ones(4, np.int32)),
                _cu(np.zeros(4, np.float32)))
    assert _lib.launch_count() == n0
