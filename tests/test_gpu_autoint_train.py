"""GPU: AutoInt training.

* The attention-core kernels (``b200_autoint_attention_forward`` / ``_backward``) through the C-ABI against torch
  float64 autograd: O, lse, dQ, dK and dV within per-element bounds (below; ``test_autoint_train_cpu.py`` shows a
  float32 restatement meets them with 4x to spare and uses at least 1/1000 of them), bit-identical repeats,
  strided inputs, attention logits around +-100, shape rejections before any launch.
* ``training.AutoIntTrainer`` against the float64 restatement in ``tests/_autoint_train_oracle.py`` (parity
  unpinned, see its header) with the bounds of ``test_gpu_din_train.py``: logits, loss and every raw gradient of
  one batch, parameters after a step, the loss over two steps, ``step_graph``, ``set_regularisation``, and the
  exported weights in the inference engine and through a ``_tf_variables.npz`` round trip."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _autoint_oracle as ao  # noqa: E402
import _autoint_train_oracle as ato  # noqa: E402

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24

# ---------------------------------------------------------------------------------------------------------------
# attention core: cases and bounds (shared with the CPU calibration)
# ---------------------------------------------------------------------------------------------------------------
# (R, F, H, hd)
KERNEL_CASES = [
    (37, 2, 1, 1), (37, 8, 2, 8), (37, 33, 5, 3), (37, 130, 1, 64), (1, 130, 5, 8), (37, 8, 5, 1),
    (37, 33, 2, 3), (1, 2, 1, 64), (5000, 8, 2, 8), (5000, 2, 5, 3), (37, 130, 2, 3), (1, 33, 1, 64),
]
C_O, C_LSE, C_DV, C_DQK = 8.0, 16.0, 8.0, 8.0


def kernel_case_id(c):
    return "R{}-F{}-H{}-hd{}".format(*c)


def make_kernel_case(c, large=False, seed=0):
    """float32 Q, K, V, dO [R, F, D] (D = H * hd); ``large`` scales Q so the largest logit is about 100."""
    R, F, H, hd = c
    rng = np.random.default_rng(seed + 1000 * F + 10 * hd + H)
    D = H * hd
    q, k, v, do = (rng.standard_normal((R, F, D)).astype(np.float32) for _ in range(4))
    if large:
        s = np.abs(np.einsum("rfhd,rghd->rhfg", q.reshape(R, F, H, hd), k.reshape(R, F, H, hd))).max() / np.sqrt(hd)
        q = (q * (100.0 / s)).astype(np.float32)
    return q, k, v, do


def reference(q, k, v, do, H, dtype):
    """torch autograd of the core in ``dtype``: numpy (O, lse, dQ, dK, dV)."""
    import torch

    hd = q.shape[2] // H
    t = [torch.tensor(a, dtype=dtype, requires_grad=True) for a in (q, k, v)]
    o, lse = ato.attention_core(*t, H, 1.0 / np.sqrt(hd) if dtype == torch.float64 else np.float32(1.0 / np.sqrt(hd)))
    (o * torch.as_tensor(do, dtype=dtype)).sum().backward()
    return [a.detach().numpy() for a in (o, lse)] + [a.grad.numpy() for a in t]


def bounds(q, k, v, do, H):
    """Per-element bounds of (O, lse, dQ, dK, dV): C * u32 * (F + hd + A) * G, per (row, head) A = the largest
    scale * sum_j |q_fj k_gj| and G the magnitude each output is built from (float64)."""
    R, F, D = q.shape
    hd = D // H
    sc = 1.0 / np.sqrt(hd)
    sp = lambda a: a.astype(np.float64).reshape(R, F, H, hd).transpose(0, 2, 1, 3)      # noqa: E731
    Q, K, V, dO = sp(q), sp(k), sp(v), sp(do)
    s = Q @ K.transpose(0, 1, 3, 2) * sc
    P = np.exp(s - s.max(-1, keepdims=True))
    P /= P.sum(-1, keepdims=True)
    O = P @ V
    dP = dO @ V.transpose(0, 1, 3, 2)
    Dr = (dO * O).sum(-1, keepdims=True)
    A = (np.abs(Q) @ np.abs(K).transpose(0, 1, 3, 2) * sc).max(axis=(2, 3))           # [R, H]
    amp = U32 * (F + hd + A)[:, :, None, None]
    W = P * (np.abs(dP) + np.abs(Dr))                                                   # |dS| / scale before cancels
    mx = lambda a: np.abs(a).max(axis=(2, 3), keepdims=True)                            # noqa: E731
    back = lambda a: np.broadcast_to(a, (R, H, F, hd)).transpose(0, 2, 1, 3).reshape(R, F, D)   # noqa: E731
    bO = back(C_O * amp * mx(V))
    bL = C_LSE * amp[:, :, :, 0] * np.ones((R, H, F))
    bdV = back(C_DV * amp * P.sum(2).max(-1)[:, :, None, None] * mx(dO))
    bdQ = back(C_DQK * amp * sc * W.sum(-1).max(-1)[:, :, None, None] * mx(K))
    bdK = back(C_DQK * amp * sc * W.sum(2).max(-1)[:, :, None, None] * mx(Q))
    return bO, bL, bdQ, bdK, bdV


def _run_kernels(q, k, v, do, H, strided=False):
    """The two kernels on device copies; returns numpy (O, lse, dQ, dK, dV) and the launch count they took."""
    import torch

    from librecommender_b200 import _lib

    R, F, D = q.shape
    hd = D // H
    dev = torch.device("cuda")
    if strided:                         # Q / K / V as column slices of one [R*F, 3D] buffer
        buf = torch.as_tensor(np.concatenate([q, k, v], axis=2).reshape(R * F, 3 * D), device=dev)
        Q, K, V = buf[:, :D], buf[:, D:2 * D], buf[:, 2 * D:]
    else:
        Q, K, V = (torch.as_tensor(a.reshape(R * F, D), device=dev) for a in (q, k, v))
    dO = torch.as_tensor(do.reshape(R * F, D), device=dev)
    O = torch.full((R * F, D), float("nan"), device=dev)
    lse = torch.full((R * H * F,), float("nan"), device=dev)
    dQ, dK, dV = (torch.full((R * F, D), float("nan"), device=dev) for _ in range(3))
    sc = float(np.float32(1.0 / np.sqrt(hd)))
    st = _lib.current_stream()
    n0 = _lib.launch_count()
    _lib.check(_lib.lib.b200_autoint_attention_forward(_lib.ptr(Q), Q.stride(0), _lib.ptr(K), K.stride(0), _lib.ptr(V),
                                                       V.stride(0), R, F, H, hd, sc, _lib.ptr(O), O.stride(0),
                                                       _lib.ptr(lse), st))
    _lib.check(_lib.lib.b200_autoint_attention_backward(_lib.ptr(Q), Q.stride(0), _lib.ptr(K), K.stride(0), _lib.ptr(V),
                                                        V.stride(0), _lib.ptr(O), O.stride(0), _lib.ptr(lse),
                                                        _lib.ptr(dO), dO.stride(0), R, F, H, hd, sc, _lib.ptr(dQ),
                                                        _lib.ptr(dK), _lib.ptr(dV), D, st))
    torch.cuda.synchronize()
    out = [O.cpu().numpy().reshape(R, F, D), lse.cpu().numpy().reshape(R, H, F)]
    out += [a.cpu().numpy().reshape(R, F, D) for a in (dQ, dK, dV)]
    return out, _lib.launch_count() - n0


def _check_kernels(q, k, v, do, H, strided=False):
    import torch

    got, n = _run_kernels(q, k, v, do, H, strided)
    assert n == 2
    ref = reference(q, k, v, do, H, torch.float64)
    for name, g, r, b in zip(("O", "lse", "dQ", "dK", "dV"), got, ref, bounds(q, k, v, do, H)):
        assert np.isfinite(g).all(), name
        err = np.abs(g.astype(np.float64) - r)
        assert (err <= b).all(), (name, float((err / b).max()))
    return got


@pytest.mark.parametrize("c", KERNEL_CASES, ids=kernel_case_id)
def test_attention_kernels_match_fp64_autograd(c):
    _check_kernels(*make_kernel_case(c), H=c[2])


@pytest.mark.parametrize("c", [(37, 8, 2, 8), (37, 33, 5, 3), (1, 130, 1, 64)], ids=kernel_case_id)
def test_attention_kernels_strided_rows_and_bit_identical_repeats(c):
    a = _check_kernels(*make_kernel_case(c), H=c[2], strided=True)
    b, _ = _run_kernels(*make_kernel_case(c), H=c[2], strided=True)
    for x, y in zip(a, b):
        np.testing.assert_array_equal(x, y)
    contiguous, _ = _run_kernels(*make_kernel_case(c), H=c[2])
    for x, y in zip(a, contiguous):
        np.testing.assert_array_equal(x, y)


@pytest.mark.parametrize("c", [(37, 8, 2, 8), (37, 33, 1, 3)], ids=kernel_case_id)
def test_attention_kernels_large_logits(c):
    q, k, v, do = make_kernel_case(c, large=True)
    R, F, H, hd = c
    s = np.einsum("rfhd,rghd->rhfg", q.reshape(R, F, H, hd).astype(np.float64),
                  k.reshape(R, F, H, hd).astype(np.float64)) / np.sqrt(hd)
    assert np.abs(s).max() > 80
    _check_kernels(q, k, v, do, H)


def test_attention_kernels_reject_shapes_before_launch():
    from librecommender_b200 import _lib

    lib = _lib.lib
    x = np.zeros(64, np.float32)
    p = _lib.ptr(x)
    n0 = _lib.launch_count()
    # (R, F, H, hd, ld)
    for R, F, H, hd, ld in ((4, 131, 1, 8, 8), (4, 1, 1, 8, 8), (4, 8, 0, 8, 8), (4, 8, 2, 0, 8), (4, 8, 5, 13, 65),
                            (4, 8, 2, 8, 15), (-1, 8, 1, 8, 8)):
        assert lib.b200_autoint_attention_forward(p, ld, p, ld, p, ld, R, F, H, hd, 0.5, p, ld, p, None) == -2
        assert b"b200_autoint_attention_forward" in lib.b200_last_error()
        assert lib.b200_autoint_attention_backward(p, ld, p, ld, p, ld, p, ld, p, p, ld, R, F, H, hd, 0.5, p, p, p, ld,
                                                   None) == -2
        assert b"b200_autoint_attention_backward" in lib.b200_last_error()
    assert _lib.launch_count() == n0


# ---------------------------------------------------------------------------------------------------------------
# the trainer against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------
TRAIN_CASES = [c for c in ao.CASES if c[0] != "multi"]
# logits rtol = atol = 3e-5 and loss 2e-5 as in test_gpu_din_train.py; gradients
# <= GRAD_REL * max|ref| + GRAD_ABS * (largest gradient of the batch), 10x tighter than there: its
# 1e-3 / 2e-5 would be over 1000x looser than float32 needs here (test_autoint_train_cpu.py::test_trainer_bounds)
GRAD_REL, GRAD_ABS = 1e-4, 2e-6


def train_batch(c, seed=0, R=1024):
    """(spec, raw weights, [(users, items, sparse, dense, labels)] x 2) of a case."""
    rng, spec, w = ao.make_case(c, seed)
    batches = []
    for _ in range(2):
        users, items, sparse, dense = ao.case_rows(rng, spec, R)
        batches.append((users, items, sparse, dense, (rng.random(R) < 0.35).astype(np.float32)))
    return spec, w, batches


def _cu(a):
    import torch

    return torch.as_tensor(np.asarray(a)).cuda()


@pytest.mark.parametrize("c", TRAIN_CASES, ids=ao.case_id)
def test_gradients_of_one_batch_match_oracle(c):
    import torch

    from librecommender_b200.training import AutoIntTrainer

    spec, w, batches = train_batch(c)
    users, items, sparse, dense, labels = batches[0]
    tr = AutoIntTrainer(spec, w)
    st = ato.init_state(w)
    ref_loss, ref_out, ref_g = ato.forward_backward(st, users, items, sparse, dense, labels)
    logits = tr.forward(_cu(users), _cu(items))
    np.testing.assert_allclose(logits.cpu().numpy(), ref_out, rtol=3e-5, atol=3e-5)
    loss = tr.backward(_cu(labels))
    torch.cuda.synchronize()
    assert abs(float(loss) - ref_loss) < 2e-5
    assert set(tr.grads) == set(ref_g)
    gmax = max(np.abs(v).max() for v in ref_g.values())
    for k, ref in ref_g.items():
        got = tr.grads[k].cpu().numpy().astype(np.float64).reshape(ref.shape)
        scale = np.abs(ref).max()
        assert np.abs(got - ref).max() <= GRAD_REL * scale + GRAD_ABS * gmax, (k, float(np.abs(got - ref).max()), scale, gmax)


@pytest.mark.parametrize("c", [TRAIN_CASES[0], TRAIN_CASES[1]], ids=ao.case_id)
def test_training_steps_match_oracle_and_export(c, tmp_path):
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import AutoInt
    from librecommender_b200.training import AutoIntTrainer

    spec, w, batches = train_batch(c, 11)
    lr, eps = 1e-2, 1e-5
    tr = AutoIntTrainer(spec, w, lr=lr, epsilon=eps)
    st = ato.init_state(w)
    for step, (users, items, sparse, dense, labels) in enumerate(batches):
        ref_loss = ato.train_step(st, users, items, sparse, dense, labels, lr, eps)
        loss = tr.step(_cu(users), _cu(items), _cu(labels))
        assert abs(float(loss) - ref_loss) <= 1e-3 * max(1.0, abs(ref_loss)) * (step + 1), (step, float(loss), ref_loss)
        if step == 0:
            for k, ref in st["params"].items():
                got = tr.params[k].cpu().numpy().astype(np.float64).reshape(ref.shape)
                assert np.abs(got - ref).max() <= 2e-2 * lr + 1e-6, (k, float(np.abs(got - ref).max()))
    # export: the raw layout of the same scheme, straight into the inference engine
    raw = tr.export_weights()
    assert raw["autoint_scheme"] == w["autoint_scheme"]
    for a, b in zip(raw["autoint_mha"], w["autoint_mha"]):
        assert {k: v.shape for k, v in a.items()} == {k: np.shape(v) for k, v in b.items()}
    model = AutoInt(spec, wio.autoint_weights(raw))
    rng = np.random.default_rng(3)
    users, items, sparse, dense = ao.case_rows(rng, spec, R=300)
    got = model.logits(users, items).cpu().numpy()
    ao.close(got, ao.autoint_forward(raw, users, items, sparse, dense, np.float64))
    # a save as the reference's <name>_tf_variables.npz and a reload give the same logits bit for bit
    np.savez(tmp_path / "m_tf_variables.npz", **wio.autoint_tf_variables(raw))
    hds = [lw["query"].shape[-1] if raw["autoint_scheme"] == "keras" else lw["query"].shape[1] // raw["num_heads"]
           for lw in raw["autoint_mha"]]
    back = wio.load_reference_tf_model(str(tmp_path), "m", "AutoInt", None, False, num_heads=raw["num_heads"],
                                       att_embed_size=hds, use_residual=raw["use_residual"])
    np.testing.assert_array_equal(AutoInt(spec, back).logits(users, items).cpu().numpy(), got)


def test_graph_replay_equals_eager_steps():
    from librecommender_b200.training import AutoIntTrainer

    spec, w, batches = train_batch(TRAIN_CASES[4], 21)
    a = AutoIntTrainer(spec, w, lr=1e-2)
    b = AutoIntTrainer(spec, w, lr=1e-2)
    for users, items, _, _, labels in batches + batches[:1]:
        u, i, y = _cu(users), _cu(items), _cu(labels)
        la = float(a.step(u, i, y))
        lb = float(b.step_graph(u, i, y))
        assert abs(la - lb) <= 1e-5 * max(1.0, abs(la)), (la, lb)
    assert a.t == b.t == 3 and int(b._step_dev.item()) == 3
    assert b.graph_launches_per_step > 10
    for k in a.params:
        d = (a.params[k] - b.params[k]).abs().max().item()
        assert d <= 2e-4, (k, d)          # float atomics in the table scatter: order differs run to run


def test_regularisation_and_lr_decay_match_oracle():
    from librecommender_b200.training import AutoIntTrainer, set_regularisation

    spec, w, batches = train_batch(TRAIN_CASES[1], 31)
    lr, eps, reg = 1e-2, 1e-5, 3e-3
    tr = set_regularisation(AutoIntTrainer(spec, w, lr=lr, epsilon=eps), reg=reg, lr_decay=True, decay_steps=2,
                            decay_rate=0.5)
    plain = AutoIntTrainer(spec, w, lr=lr, epsilon=eps)
    st = ato.init_state(w)
    seq = batches + batches
    for step, (users, items, sparse, dense, labels) in enumerate(seq):
        ref_loss = ato.train_step(st, users, items, sparse, dense, labels, lr, eps, reg=reg, decay_steps=2,
                                  decay_rate=0.5)
        u, i, y = _cu(users), _cu(items), _cu(labels)
        loss = tr.step(u, i, y)
        plain.step(u, i, y)
        assert abs(float(loss) - ref_loss) <= 2e-3 * max(1.0, abs(ref_loss)) * (step + 1), (step, float(loss), ref_loss)
    moved = 0.0
    for k in ato.TABLES:
        ref = st["params"][k]
        got = tr.params[k].cpu().numpy().astype(np.float64).reshape(ref.shape)
        # the decayed step sizes bound the total movement: lr (1 + 1 + .5 + .5) = 3 lr per weight
        assert np.abs(got - ref).max() <= 0.12 * lr * 3, (k, float(np.abs(got - ref).max()))
        assert np.median(np.abs(got - ref)) <= 0.01 * lr, (k, float(np.median(np.abs(got - ref))))
        moved = max(moved, float((tr.params[k] - plain.params[k]).abs().max()))
    assert moved > 0.5 * lr          # the regulariser + decay changed the trajectory


@pytest.mark.parametrize("what", ["multi_sparse", "K", "layers", "width", "heads", "fields", "out_kernel"])
def test_trainer_rejects_before_launch(what):
    from librecommender_b200 import _lib
    from librecommender_b200 import synthetic as syn
    from librecommender_b200.training import AutoIntTrainer

    rng = np.random.default_rng(8)
    spec = syn.make_spec(rng, 20, 30, [3], [4], 1, 1)
    K, att, H = 16, (8, 8), 2
    if what == "multi_sparse":
        spec = syn.make_multi_sparse_spec(rng, 20, 30, [9, 30], [12, 6, 25], [("user", 17, 3), ("item", 23, 4)], 1, 1)
    elif what == "K":
        K = 65
    elif what == "layers":
        att = (4, 4, 4, 4, 4)
    elif what == "width":
        att = (40,)                      # D = 80
    elif what == "fields":
        spec = syn.make_spec(rng, 20, 30, [3] * 64, [3] * 64, 1, 0)      # F = 131
    w = syn.make_autoint_weights(rng, spec, K, att, H, True, "legacy")
    if what == "heads":
        w["num_heads"] = 3               # D = 16 is not a multiple of 3
    elif what == "out_kernel":
        w["out_kernel"] = w["out_kernel"][:-1]
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        AutoIntTrainer(spec, w)
    assert _lib.launch_count() == n0


def test_multi_sparse_normal_combiner_trains():
    """Multi-sparse members as separate fields (combiner "normal") need no pooling backward."""
    import torch

    from librecommender_b200 import synthetic as syn
    from librecommender_b200.training import AutoIntTrainer
    from oracle import tf_models as tm

    rng = np.random.default_rng(9)
    spec = syn.make_multi_sparse_spec(rng, 60, 80, [9, 30], [12, 6, 25], [("user", 17, 3), ("item", 23, 4)], 1, 1)
    w = syn.make_autoint_weights(rng, spec, 8, (4, 4), 2, True, "keras", combiner="normal")
    w["multi_sparse_combiner"] = "normal"
    users, items = rng.integers(0, 61, 512), rng.integers(0, 81, 512)
    sparse, dense = tm.row_features(spec, users, items)
    labels = (rng.random(512) < 0.4).astype(np.float32)
    tr = AutoIntTrainer(spec, w)
    st = ato.init_state(w)
    ref_loss, ref_out, ref_g = ato.forward_backward(st, users, items, sparse, dense, labels)
    np.testing.assert_allclose(tr.forward(_cu(users), _cu(items)).cpu().numpy(), ref_out, rtol=3e-5, atol=3e-5)
    loss = tr.backward(_cu(labels))
    torch.cuda.synchronize()
    assert abs(float(loss) - ref_loss) < 2e-5
    gmax = max(np.abs(v).max() for v in ref_g.values())
    for k, ref in ref_g.items():
        got = tr.grads[k].cpu().numpy().astype(np.float64).reshape(ref.shape)
        assert np.abs(got - ref).max() <= GRAD_REL * np.abs(ref).max() + GRAD_ABS * gmax, k
    assert tr.export_weights()["multi_sparse_combiner"] == "normal"
