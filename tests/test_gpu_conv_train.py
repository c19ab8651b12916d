"""Caser / WaveNet training on the GPU: the training forward against b200_caser_encode / b200_wavenet_encode (bit for
bit) and its saved argmax against float64, one step's loss and gradients against the float64 autograd oracle
(tests/_conv_train_oracle.py), bit-identical repeats of the backward kernels, Adam steps, CUDA-graph replay, export
into the serving models, the regulariser and the errors raised before any launch."""
import numpy as np
import pytest

import _conv_train_oracle as co

pytestmark = pytest.mark.gpu

# gradients: |got - ref| <= GRAD_REL * max|ref of the variable| + GRAD_ABS * (largest gradient of the batch), calibrated
# in test_conv_train_cpu.py::test_float32_restatement_meets_gpu_bounds
GRAD_REL, GRAD_ABS = 5e-4, 1e-5
# a pooled column whose float64 maximum is closer than this to its runner-up (or to 0) may legitimately pick another
# position in float32; every other column's saved argmax must equal the oracle's
GAP = 1e-4
N_ITEMS = 60


def _cu(a):
    import torch

    return torch.as_tensor(np.asarray(a)).cuda()


def make_batch(rng, n_users, R, T, n_items=N_ITEMS):
    """users, items, seqs [R, T] end-padded with n_items (a quarter of the rows keep a long pad tail, one row is all
    padding), lens, labels."""
    lens = rng.integers(1, T + 1, R)
    lens[: R // 4] = rng.integers(0, max(1, T // 3) + 1, R // 4)
    lens[-1] = 0
    seqs = rng.integers(0, n_items, (R, T)).astype(np.int32)
    seqs[np.arange(T)[None, :] >= lens[:, None]] = n_items
    return (rng.integers(0, n_users, R), rng.integers(0, n_items, R), seqs, lens.astype(np.int32),
            (rng.random(R) < 0.4).astype(np.float32))


def raw_weights(model, n_users, K, seed=0, T=10, nh=2, nv=4, F=16, n_blocks=1, n_layers=4, dilated=True):
    from librecommender_b200 import synthetic as syn

    rng = np.random.default_rng(seed)
    if model == "Caser":
        return syn.make_caser_weights(rng, n_users, N_ITEMS, K, T, nh, nv)
    return syn.make_wavenet_weights(rng, n_users, N_ITEMS, K, F, n_blocks, n_layers, dilated)


def trainer(raw, n_users, **kw):
    from librecommender_b200.training import CaserTrainer, WaveNetTrainer

    cls = CaserTrainer if "vertical" in raw else WaveNetTrainer
    return cls({"n_users": n_users, "n_items": N_ITEMS}, raw, **kw)


# ---------------------------------------------------------------------------------------------------------------
# the training forward
# ---------------------------------------------------------------------------------------------------------------
FWD_CASES = [  # (model, T, K, nh / F, nv / layers per block, blocks, dilated)
    ("Caser", 1, 8, 2, 4, 1, True), ("Caser", 2, 7, 3, 1, 1, True), ("Caser", 10, 16, 2, 4, 1, True),
    ("Caser", 50, 13, 8, 8, 1, True), ("Caser", 64, 32, 4, 2, 1, True),
    ("WaveNet", 1, 8, 16, 4, 1, True), ("WaveNet", 2, 9, 5, 2, 1, True), ("WaveNet", 10, 16, 16, 4, 1, True),
    ("WaveNet", 50, 31, 64, 4, 2, True), ("WaveNet", 64, 16, 33, 3, 1, False), ("WaveNet", 10, 16, 16, 4, 2, False),
]


def _raw_of_case(c, n_users, seed=0):
    model, T, K, a, b, blocks, dil = c
    if model == "Caser":
        return raw_weights(model, n_users, K, seed, T=T, nh=a, nv=b)
    return raw_weights(model, n_users, K, seed, F=a, n_blocks=blocks, n_layers=b, dilated=dil)


@pytest.mark.parametrize("c", FWD_CASES, ids=lambda c: "-".join(map(str, c)))
def test_training_forward_equals_encode_and_saves_the_first_argmax(c):
    import torch

    from librecommender_b200 import feat_models as fm

    T, R = c[1], 150
    raw = _raw_of_case(c, R - 1)
    users, items, seqs, lens, labels = make_batch(np.random.default_rng(1), R - 1, R, T)
    tr = trainer(raw, R - 1)
    u0, cache = tr.user_vectors(_cu(users), _cu(seqs))
    model = (fm.Caser if c[0] == "Caser" else fm.WaveNet)({"n_users": R - 1, "n_items": N_ITEMS}, raw, seqs, lens)
    ref = model.encode(torch.arange(R, device="cuda"))
    torch.cuda.synchronize()
    feat = cache["feat"].cpu().numpy()
    np.testing.assert_array_equal(feat, ref.cpu().numpy())
    np.testing.assert_array_equal(u0.cpu().numpy(), model.user_vectors(users, seqs).cpu().numpy())
    arg = cache["arg"].cpu().numpy()
    pooled = feat[:, :arg.shape[1]]
    assert np.array_equal(arg == -1, pooled == 0)                     # -1 exactly where the max is <= 0
    P, meta = co.init_params(raw), co.meta_of(raw)
    ref_arg, _ = co.pool_argmax(P, meta, seqs)
    clear = co.near_tie_pick(P, meta, seqs, arg, GAP) == -1
    assert clear.mean() > 0.95
    np.testing.assert_array_equal(arg[clear], ref_arg[clear])
    if c[0] == "WaveNet":                                              # every causal layer's output, float64-close
        P = co.init_params(raw)
        x = P["seq_embeds"][torch.as_tensor(seqs.astype(np.int64))]
        for i, d in enumerate(co.meta_of(raw)["dilations"]):
            W = P[f"conv{i}_kernel"]
            prev = torch.cat([torch.zeros_like(x[:, :d]), x[:, :-d]], 1) if d < T else torch.zeros_like(x)
            x = torch.relu(prev @ W[0] + x @ W[1] + P[f"conv{i}_bias"])
            got = cache["ys"][i].cpu().numpy().reshape(x.shape)
            np.testing.assert_allclose(got, x.numpy(), rtol=0, atol=2e-5 * max(1.0, float(x.abs().max())))


# ---------------------------------------------------------------------------------------------------------------
# gradients of one step against the float64 oracle
# ---------------------------------------------------------------------------------------------------------------
def trainer_grads(tr):
    g = {k: v.cpu().numpy().astype(np.float64) for k, v in tr.grads.items()}
    g["dense_kernel"], g["dense_bias"] = g.pop("dense_Wt").T, g.pop("dense_b")
    return g


def check_grads(got, ref):
    gmax = max(np.abs(v).max() for v in ref.values())
    assert set(got) == set(ref)
    for k, r in ref.items():
        a = np.asarray(got[k], np.float64).reshape(r.shape)
        err = np.abs(a - r).max()
        assert err <= GRAD_REL * np.abs(r).max() + GRAD_ABS * gmax, (k, float(err), float(np.abs(r).max()), gmax)


STEP_CASES = [  # (model, T, K, nh / F, nv / layers per block, blocks, dilated, loss, norm_embed, rows)
    ("Caser", 10, 16, 2, 4, 1, True, "cross_entropy", False, 200), ("Caser", 10, 16, 2, 4, 1, True, "focal", True, 200),
    ("Caser", 20, 9, 8, 8, 1, True, "cross_entropy", True, 300), ("Caser", 5, 16, 3, 2, 1, True, "focal", False, 700),
    ("WaveNet", 10, 16, 16, 4, 1, True, "cross_entropy", False, 200),
    ("WaveNet", 10, 16, 16, 4, 1, True, "focal", True, 200),
    ("WaveNet", 30, 12, 24, 4, 2, True, "cross_entropy", True, 300),
    ("WaveNet", 10, 16, 16, 3, 1, False, "focal", False, 300),
    ("Caser", 64, 128, 32, 32, 1, True, "cross_entropy", True, 4),      # the envelope maxima
    ("WaveNet", 64, 16, 128, 16, 1, False, "cross_entropy", True, 6),
    ("WaveNet", 64, 128, 128, 4, 4, True, "focal", False, 4),
]


def _step_case(c, seed=2):
    raw = _raw_of_case(c[:7], 40)
    batch = make_batch(np.random.default_rng(seed), 40, c[9], c[1])
    return raw, batch


@pytest.mark.parametrize("c", STEP_CASES, ids=lambda c: "-".join(map(str, c)))
def test_gradients_of_one_step_match_oracle(c):
    import torch

    loss_type, ne = c[7], c[8]
    raw, (users, items, seqs, lens, labels) = _step_case(c)
    P, meta = co.init_params(raw), co.meta_of(raw)
    tr = trainer(raw, 40, loss_type=loss_type, norm_embed=ne)
    _, cache = tr.user_vectors(_cu(users), _cu(seqs))
    pick = co.near_tie_pick(P, meta, seqs, cache["arg"].cpu().numpy(), GAP)
    loss = tr.forward_backward(_cu(users), _cu(items), _cu(seqs), _cu(lens), _cu(labels))
    torch.cuda.synchronize()
    ref_loss, ref = co.forward_backward(P, meta, users, items, seqs, labels, loss_type, ne, pick)
    assert abs(float(loss) - ref_loss) <= 2e-5 * max(1.0, abs(ref_loss))
    check_grads(trainer_grads(tr), ref)


@pytest.mark.parametrize("model", ["Caser", "WaveNet"])
def test_backward_kernels_repeat_bit_for_bit(model):
    import torch

    c = STEP_CASES[2] if model == "Caser" else STEP_CASES[6]
    raw, (users, items, seqs, lens, labels) = _step_case(c)
    tr = trainer(raw, 40)
    _, cache = tr.user_vectors(_cu(users), _cu(seqs))
    dF = torch.randn(cache["feat"].shape, device="cuda")
    outs = []
    for _ in range(2):
        tr.conv_g.fill_(7.0)
        dX = tr._encoder_backward(cache, dF)
        outs.append((dX.cpu().numpy(), tr.conv_g.cpu().numpy()))
    for a, b in zip(*outs):
        np.testing.assert_array_equal(a, b)
        assert np.all(np.isfinite(a))


# ---------------------------------------------------------------------------------------------------------------
# steps, graphs, export, regulariser, errors
# ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("c", [STEP_CASES[1], STEP_CASES[2], STEP_CASES[5], STEP_CASES[7]],
                         ids=lambda c: "-".join(map(str, c)))
def test_adam_steps_track_oracle_and_loss_falls(c):
    loss_type, ne = c[7], c[8]
    raw = _raw_of_case(c[:7], 40)
    rng = np.random.default_rng(5)
    batches = [make_batch(rng, 40, 256, c[1]) for _ in range(3)]
    lr, eps = 1e-2, 1e-5
    tr = trainer(raw, 40, loss_type=loss_type, norm_embed=ne, lr=lr, epsilon=eps)
    st, meta = co.init_state(raw), co.meta_of(raw)
    for step, (users, items, seqs, lens, labels) in enumerate(batches):
        _, cache = tr.user_vectors(_cu(users), _cu(seqs))
        pick = co.near_tie_pick(st["P"], meta, seqs, cache["arg"].cpu().numpy(), GAP)
        ref_loss = co.train_step(st, meta, users, items, seqs, labels, lr, eps, loss_type, ne, pick=pick)
        loss = float(tr.step(_cu(users), _cu(items), _cu(seqs), _cu(lens), _cu(labels)))
        assert abs(loss - ref_loss) <= 1e-3 * max(1.0, abs(ref_loss)) * (step + 1), (step, loss, ref_loss)
    exported, ref_raw = tr.export_weights(), co.raw_of(st["P"], raw)
    for k in co.TABLES + ("dense_kernel", "dense_bias"):
        assert np.abs(np.asarray(exported[k], np.float64).reshape(np.shape(ref_raw[k])) - ref_raw[k]).max() <= 3e-2 * lr
    last = co.last_layer(raw)
    for a, b in zip(exported["convs"] + [exported[last]], ref_raw["convs"] + [ref_raw[last]]):
        for k in ("kernel", "bias"):
            assert np.abs(a[k].astype(np.float64) - b[k]).max() <= 3e-2 * lr, k
    users, items, seqs, lens, labels = batches[0]
    args = [_cu(x) for x in (users, items, seqs, lens, labels)]
    first = float(tr.step(*args))
    for _ in range(30):
        last_loss = float(tr.step(*args))
    assert last_loss < first


@pytest.mark.parametrize("model", ["Caser", "WaveNet"])
def test_graph_replay_and_fresh_trainers_agree(model):
    c = STEP_CASES[0] if model == "Caser" else STEP_CASES[4]
    raw = _raw_of_case(c[:7], 40)
    rng = np.random.default_rng(6)
    batches = [make_batch(rng, 40, 200, c[1]) for _ in range(3)]
    a, b, d = (trainer(raw, 40, lr=1e-2) for _ in range(3))
    for i, batch in enumerate(batches):
        args = [_cu(x) for x in batch]
        la, lb, ld = float(a.step(*args)), float(b.step_graph(*args)), float(d.step(*args))
        assert abs(la - lb) <= 1e-5 * max(1.0, abs(la)) and abs(la - ld) <= 1e-5 * max(1.0, abs(la))
        if i == 0:
            # after one step everything but the atomically scattered tables is bit-identical
            for k in a.params:
                if k not in co.TABLES:
                    np.testing.assert_array_equal(a.params[k].cpu().numpy(), b.params[k].cpu().numpy(), err_msg=k)
                    np.testing.assert_array_equal(a.params[k].cpu().numpy(), d.params[k].cpu().numpy(), err_msg=k)
            for k in co.TABLES:
                assert (a.params[k] - b.params[k]).abs().max().item() <= 1e-6, k
                assert (a.params[k] - d.params[k]).abs().max().item() <= 1e-6, k
    assert b.graph_launches_per_step > 20 and int(b._step_dev.item()) == 3
    for k in a.params:
        assert (a.params[k] - b.params[k]).abs().max().item() <= 2e-4, k      # float atomics in the table scatters


@pytest.mark.parametrize("model", ["Caser", "WaveNet"])
def test_export_serves_bit_identically(model):
    from librecommender_b200 import feat_models as fm

    c = STEP_CASES[2] if model == "Caser" else STEP_CASES[6]
    raw = _raw_of_case(c[:7], 40)
    users, items, seqs, lens, labels = make_batch(np.random.default_rng(7), 40, 41, c[1])
    tr = trainer(raw, 40, lr=1e-2, norm_embed=True)
    for _ in range(2):
        tr.step(_cu(users), _cu(items), _cu(seqs), _cu(lens), _cu(labels))
    exp = tr.export_weights()
    cls = fm.Caser if model == "Caser" else fm.WaveNet
    served = cls({"n_users": 40, "n_items": N_ITEMS}, exp, seqs, lens, norm_embed=False)
    u, _ = tr.user_vectors(_cu(users), _cu(seqs))
    np.testing.assert_array_equal(served.user_vectors(users, seqs).cpu().numpy(), u.cpu().numpy())
    U, I = cls({"n_users": 40, "n_items": N_ITEMS}, exp, seqs, lens, norm_embed=True).set_embeddings()
    K = tr.K
    assert U.shape == (41, 2 * K + 1) and I.shape == (N_ITEMS + 1, 2 * K + 1)
    assert bool(U.isfinite().all()) and bool(I.isfinite().all())


@pytest.mark.parametrize("model", ["Caser", "WaveNet"])
def test_regularisation_changes_the_three_tables_only(model):
    from librecommender_b200.training import set_regularisation

    c = STEP_CASES[0] if model == "Caser" else STEP_CASES[4]
    raw = _raw_of_case(c[:7], 40)
    users, items, seqs, lens, labels = make_batch(np.random.default_rng(8), 40, 100, c[1])
    args = [_cu(x) for x in (users, items, seqs, lens, labels)]
    lr, eps, reg = 1e-2, 1e-5, 3e-3
    plain = trainer(raw, 40, lr=lr, epsilon=eps)
    tr = set_regularisation(trainer(raw, 40, lr=lr, epsilon=eps), reg=reg)
    assert tr.reg_vars == co.REG_VARS
    st = co.init_state(raw)
    _, cache = tr.user_vectors(args[0], args[2])
    pick = co.near_tie_pick(st["P"], co.meta_of(raw), seqs, cache["arg"].cpu().numpy(), GAP)
    co.train_step(st, co.meta_of(raw), users, items, seqs, labels, lr, eps, reg=reg, pick=pick)
    tr.step(*args)
    plain.step(*args)
    ref = co.raw_of(st["P"], raw)
    for k in co.REG_VARS:
        got = tr.params[k].cpu().numpy().astype(np.float64)
        assert np.abs(got - ref[k]).max() <= 2e-2 * lr, k
        assert (tr.params[k] - plain.params[k]).abs().max().item() > 0.1 * lr, k
    for k in tr.params:         # every other variable sees the same gradients: the same bits after one step
        if k not in co.TABLES:
            np.testing.assert_array_equal(tr.params[k].cpu().numpy(), plain.params[k].cpu().numpy(), err_msg=k)
    # item_biases is not regularised; its scatter is atomic, so it agrees to the rounding of the summation order
    assert (tr.params["item_biases"] - plain.params["item_biases"]).abs().max().item() <= 1e-7


@pytest.mark.parametrize("what", ["bpr", "loss", "rating", "rows", "K", "filters", "layers", "T", "memory"])
@pytest.mark.parametrize("model", ["Caser", "WaveNet"])
def test_trainer_rejects_before_launch(model, what):
    from librecommender_b200 import _lib

    caser = model == "Caser"
    kw, K, T = {}, 8, 10
    raw = raw_weights(model, 5, K)
    if what == "bpr":
        kw["loss_type"] = "bpr"
    elif what == "loss":
        kw["loss_type"] = "softmax"
    elif what == "rating":
        kw["task"] = "rating"
    elif what == "rows":
        raw["seq_embeds"] = raw["seq_embeds"][:-1]
    elif what == "K":
        raw = raw_weights(model, 5, 129)
    elif what == "filters":
        raw = raw_weights(model, 5, K, nh=33) if caser else raw_weights(model, 5, K, F=129)
    elif what == "layers":
        raw = raw_weights(model, 5, K, T=65) if caser else raw_weights(model, 5, K, n_layers=17)
    elif what == "T":
        T = 9 if caser else 65
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        tr = trainer(raw, 5, **kw)
        B = 4 if what != "memory" else 1 << 40
        if what == "memory":
            tr._check_batch(B, T)
        tr.step(_cu(np.zeros(4, np.int64)), _cu(np.zeros(4, np.int64)), _cu(np.zeros((4, T), np.int32)),
                _cu(np.ones(4, np.int32)), _cu(np.zeros(4, np.float32)))
    assert _lib.launch_count() == n0
