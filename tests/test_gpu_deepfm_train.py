"""GPU parity of the device DeepFM training step (librecommender_b200/training.py::DeepFMTrainer)
against oracle/deepfm_train.py (numpy float64; gradient math pinned to torch autograd by
tests/test_deepfm_train_cpu.py; TensorFlow conventions unpinned): raw gradients of one batch,
parameters after 1 and 3 steps, BN moving statistics, exported weights in the inference engine."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _case(seed, use_bn, hidden, R=1536, K=16):
    from oracle import tf_models as tm

    rng = np.random.default_rng(seed)
    spec = tm.make_spec(rng, 300, 500, [7, 30, 12], [11, 5, 40, 8], 1, 2)
    w = tm.make_deepfm_weights(rng, spec, K, hidden, use_bn)
    batches = []
    for _ in range(3):
        users, items = rng.integers(0, 300, R), rng.integers(0, 500, R)
        batches.append((users, items, (rng.random(R) < 0.35).astype(np.float32)))
    return spec, w, batches


def _map_params(st_params):
    """oracle names (W{i} = [din, dout]) -> trainer names (Wt{i} = [dout, din])."""
    out = {}
    for k, v in st_params.items():
        if k.startswith("W") and k[1:].isdigit():
            out["Wt" + k[1:]] = v.T
        else:
            out[k] = v
    return out


@pytest.mark.parametrize("use_bn,hidden", [(True, (128, 64, 32)), (False, (64, 32)), (True, (48,))])
def test_gradients_of_one_batch_match_oracle(use_bn, hidden):
    import torch

    from librecommender_b200.training import DeepFMTrainer
    from oracle import deepfm_train as dt_
    from oracle import tf_models as tm

    spec, w, batches = _case(5, use_bn, hidden)
    users, items, labels = batches[0]
    tr = DeepFMTrainer(spec, w, use_bn=use_bn)
    st = dt_.init_state(w, use_bn)
    sparse, dense = tm.row_features(spec, users, items)
    ref_loss, ref_out, ref_g, _ = dt_.forward_backward(st, users, items, sparse, dense, labels)
    u, i, y = torch.as_tensor(users).cuda(), torch.as_tensor(items).cuda(), torch.as_tensor(labels).cuda()
    logits = tr.forward(u, i)
    np.testing.assert_allclose(logits.cpu().numpy(), ref_out, rtol=3e-5, atol=3e-5)
    tr._cache["users"], tr._cache["items"] = u, i
    loss = tr.backward(y)
    torch.cuda.synchronize()
    assert abs(float(loss) - ref_loss) < 2e-5
    for k, ref in _map_params(ref_g).items():
        got = tr.grads[k].cpu().numpy().astype(np.float64).reshape(ref.shape)
        scale = max(np.abs(ref).max(), 1e-8)
        assert np.abs(got - ref).max() <= 5e-4 * scale + 1e-9, (k, float(np.abs(got - ref).max()), scale)


@pytest.mark.parametrize("use_bn", [True, False])
def test_training_steps_match_oracle(use_bn):
    import torch

    from librecommender_b200.feat_models import DeepFM
    from librecommender_b200.training import DeepFMTrainer
    from oracle import deepfm_train as dt_
    from oracle import tf_models as tm

    spec, w, batches = _case(11, use_bn, (128, 64, 32))
    lr, eps = 1e-2, 1e-5
    tr = DeepFMTrainer(spec, w, use_bn=use_bn, lr=lr, epsilon=eps)
    st = dt_.init_state(w, use_bn)
    for step, (users, items, labels) in enumerate(batches):
        sparse, dense = tm.row_features(spec, users, items)
        ref_loss = dt_.train_step(st, users, items, sparse, dense, labels, lr, eps)
        loss = tr.step(torch.as_tensor(users).cuda(), torch.as_tensor(items).cuda(), torch.as_tensor(labels).cuda())
        assert abs(float(loss) - ref_loss) <= 1e-3 * max(1.0, abs(ref_loss)) * (step + 1), (step, float(loss), ref_loss)
        if step == 0:
            for k, ref in _map_params(st["params"]).items():
                got = tr.params[k].cpu().numpy().astype(np.float64).reshape(ref.shape)
                err = np.abs(got - ref).max()
                assert err <= 2e-2 * lr + 1e-6, (k, err)       # first Adam step moves every touched weight by ~lr
    if use_bn:
        assert sorted(tr.moving) == sorted(st["moving"])
        for name, (mm, mv) in tr.moving.items():
            np.testing.assert_allclose(mm.cpu().numpy(), st["moving"][name][0], rtol=2e-3, atol=2e-4)
            np.testing.assert_allclose(mv.cpu().numpy(), st["moving"][name][1], rtol=2e-3, atol=2e-4)
    users, items, _ = batches[0]
    got = DeepFM(spec, tr.export_weights()).logits(users, items).cpu().numpy()
    sparse, dense = tm.row_features(spec, users, items)
    ref = tm.deepfm_forward(dt_.export_weights(st), users, items, sparse, dense, dtype=np.float64)
    assert np.abs(got - ref).max() <= 3e-2 * max(1.0, np.abs(ref).max())


def test_graph_replay_equals_eager_steps():
    """step_graph (one CUDA-graph capture, then replays with the Adam step counter on the device) must produce
    the same parameters as the eager step loop, for every trainer family."""
    import torch

    from librecommender_b200.training import DeepFMTrainer, FMTrainer
    from oracle import tf_models as tm

    spec, w, batches = _case(21, True, (64, 32))
    rng = np.random.default_rng(0)
    wf = tm.make_fm_weights(rng, spec, 16, True)
    for cls, weights in ((DeepFMTrainer, w), (FMTrainer, wf)):
        a = cls(spec, weights, use_bn=True, lr=1e-2)
        b = cls(spec, weights, use_bn=True, lr=1e-2)
        for users, items, labels in batches + batches:
            u, i, y = torch.as_tensor(users).cuda(), torch.as_tensor(items).cuda(), torch.as_tensor(labels).cuda()
            la = float(a.step(u, i, y))
            lb = float(b.step_graph(u, i, y))
            assert abs(la - lb) <= 1e-5 * max(1.0, abs(la)), (cls.__name__, la, lb)
        assert a.t == b.t == 6 and int(b._step_dev.item()) == 6
        assert b.graph_launches_per_step > 10
        for k in a.params:
            da = (a.params[k] - b.params[k]).abs().max().item()
            assert da <= 2e-4, (cls.__name__, k, da)       # float atomics in the scatter: order differs run to run


def test_l2_regulariser_and_lr_decay_match_oracle():
    """set_regularisation: reg (2 reg w added to the table gradients) + staircase exponential lr decay, 5 steps."""
    import torch

    from librecommender_b200.training import DeepFMTrainer, set_regularisation
    from oracle import deepfm_train as dt_
    from oracle import tf_models as tm

    spec, w, batches = _case(31, True, (64, 32))
    lr, eps, reg = 1e-2, 1e-5, 3e-3
    tr = set_regularisation(DeepFMTrainer(spec, w, use_bn=True, lr=lr, epsilon=eps), reg=reg, lr_decay=True,
                            decay_steps=2, decay_rate=0.5)
    plain = DeepFMTrainer(spec, w, use_bn=True, lr=lr, epsilon=eps)
    st = dt_.init_state(w, True)
    seq = batches + batches[:2]
    for step, (users, items, labels) in enumerate(seq):
        sparse, dense = tm.row_features(spec, users, items)
        ref_loss = dt_.train_step(st, users, items, sparse, dense, labels, lr, eps, reg=reg, decay_steps=2, decay_rate=0.5)
        u, i, y = torch.as_tensor(users).cuda(), torch.as_tensor(items).cuda(), torch.as_tensor(labels).cuda()
        loss = tr.step(u, i, y)
        plain.step(u, i, y)
        assert abs(float(loss) - ref_loss) <= 2e-3 * max(1.0, abs(ref_loss)) * (step + 1), (step, float(loss), ref_loss)
    moved = 0.0
    for k, ref in _map_params(st["params"]).items():
        got = tr.params[k].cpu().numpy().astype(np.float64).reshape(ref.shape)
        # the decayed step sizes bound the total movement: lr (1 + 1 + .5 + .5 + .25) = 3.25 lr per weight
        assert np.abs(got - ref).max() <= 0.12 * lr * 3.25, (k, float(np.abs(got - ref).max()))
        assert np.median(np.abs(got - ref)) <= 0.01 * lr, (k, float(np.median(np.abs(got - ref))))
        moved = max(moved, float((tr.params[k] - plain.params[k]).abs().max()))
    assert moved > 0.5 * lr          # the regulariser + decay changed the trajectory
    with pytest.raises(ValueError, match="reg must be float and positive"):
        set_regularisation(plain, reg=-1.0)
