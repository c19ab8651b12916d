"""GraphSage training on the device: ``b200_sage_aggregate_backward`` against float64 over the layer chain of the
encoder (empty bags, ``-1`` ids, bit-identical reruns), ``b200_sage_walk_pairs`` against the restated rule on the same
keyed draws, the i2i negatives, one full ``GraphSageTrainer`` step per paradigm and loss against the float64 oracle of
``tests/_sage_train_oracle.py`` on the step's own sampled batch (every gradient and every updated parameter), and a
few epochs on the MovieLens fixture served through the existing ``GraphSage`` inference path."""
import os

import numpy as np
import pytest

import _sage_oracle as sorc
import _sage_train_oracle as orc
from test_sage_cpu import data_info, feats, golden

pytestmark = pytest.mark.gpu
GPU_RTOL = 2e-3                # |gpu - f64| <= GPU_RTOL * max|f64| per gradient (test_gpu_sim_train's bar)
MOVIELENS = os.path.join(os.path.dirname(__file__), "golden", "movielens_feat.npz")


def _agg_backward(dout, dS, dN, n, d, nn, self_idx=None, nb_idx=None, offsets=None, lens=None):
    from librecommender_b200 import _lib

    _lib.check(_lib.lib.b200_sage_aggregate_backward(
        _lib.ptr(dout), dout.stride(0), _lib.ptr(self_idx), n, _lib.ptr(dS), dS.stride(0), _lib.ptr(nb_idx),
        _lib.ptr(offsets), _lib.ptr(lens), nn, d, _lib.ptr(dN), dN.stride(0), _lib.current_stream()))


@pytest.mark.parametrize("d", [1, 7, 16, 64, 128])
@pytest.mark.parametrize("layers", [1, 2, 3])
def test_aggregate_backward_over_the_layer_chain_matches_float64(d, layers):
    """The encoder's use: levels of n * nn^k rows, one call per level k < depth adding into one zeroed buffer
    (level k as self rows, level k + 1 as neighbour rows)."""
    import torch

    nn, n0 = 3, 37
    sizes = [n0 * nn ** k for k in range(layers + 1)]
    offs = np.concatenate([[0], np.cumsum(sizes)])
    rng = np.random.default_rng(d * 10 + layers)
    dagg = rng.standard_normal((offs[layers], 2 * d)).astype(np.float32)
    want = np.zeros((offs[-1], d))
    for k in range(layers):
        g = dagg[offs[k]:offs[k + 1]].astype(np.float64)
        want[offs[k]:offs[k + 1]] += g[:, :d]
        want[offs[k + 1]:offs[k + 2]] += np.repeat(g[:, d:] * np.float64(np.float32(1.0 / nn)), nn, axis=0)
    runs = []
    for _ in range(2):
        dA = torch.as_tensor(dagg).cuda()
        out = torch.zeros((offs[-1], d), dtype=torch.float32, device="cuda")
        for k in range(layers):
            _agg_backward(dA[offs[k]:offs[k + 1]], out[offs[k]:offs[k + 1]], out[offs[k + 1]:offs[k + 2]], sizes[k],
                          d, nn)
        runs.append(out.cpu().numpy())
    np.testing.assert_allclose(runs[0], want, rtol=1e-6, atol=1e-6)
    assert np.array_equal(runs[0].view(np.uint32), runs[1].view(np.uint32))


@pytest.mark.parametrize("d", [1, 7, 16, 64, 128])
def test_aggregate_backward_with_indices_empty_bags_and_negative_ids(d):
    import torch

    rng = np.random.default_rng(d)
    n, n_nb, ld = 50, 160, d + 3
    lens = rng.integers(0, 6, size=n).astype(np.int32)
    lens[:4] = 0
    offsets = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    m = int(offsets[-1])
    nb_idx = rng.permutation(n_nb)[:m].astype(np.int32)               # distinct neighbour rows
    nb_idx[rng.random(m) < 0.2] = -1
    self_idx = rng.permutation(n + 10)[:n].astype(np.int32)            # distinct self rows
    self_idx[::7] = -1
    dout = rng.standard_normal((n, 2 * d + 1)).astype(np.float32)
    dS0 = rng.standard_normal((n + 10, ld)).astype(np.float32)
    dN0 = rng.standard_normal((n_nb, ld)).astype(np.float32)
    wS, wN = dS0.astype(np.float64), dN0.astype(np.float64)
    for r in range(n):
        if self_idx[r] >= 0:
            wS[self_idx[r], :d] += dout[r, :d]
        for j in range(offsets[r], offsets[r] + lens[r]):
            if nb_idx[j] >= 0:
                wN[nb_idx[j], :d] += dout[r, d:2 * d] * np.float64(np.float32(1.0 / lens[r]))
    T = lambda a: torch.as_tensor(a).cuda()     # noqa: E731
    dS, dN = T(dS0), T(dN0)
    _agg_backward(T(dout), dS, dN, n, d, 0, T(self_idx), T(nb_idx), T(offsets), T(lens))
    np.testing.assert_allclose(dS.cpu().numpy(), wS, rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(dN.cpu().numpy(), wN, rtol=1e-6, atol=1e-6)


def _trainer(paradigm="i2i", data="pure", **kw):
    from librecommender_b200.sage import GraphSageTrainer

    z = golden()
    di = data_info(z, data)
    return GraphSageTrainer(di, paradigm=paradigm, **kw), di, z


@pytest.mark.parametrize("focus_start", [False, True])
def test_walk_pairs_match_the_restated_rule_on_the_same_draws(focus_start):
    tr, di, _ = _trainer(num_walks=6, sample_walk_len=4, focus_start=focus_start, seed=1234567890123)
    g = sorc.Graph(di["user_consumed"], di["item_consumed"], di["n_users"], di["n_items"])
    for step in (0, 5):
        starts, items, pos = (a.cpu().numpy() for a in tr.walk_pairs(300, step))
        w_starts, w_items, w_pos, _ = orc.keyed_walk_pairs(g, di["n_items"], 300, 6, 4, focus_start,
                                                           1234567890123, step)
        np.testing.assert_array_equal(starts, w_starts)
        np.testing.assert_array_equal(items, w_items)
        np.testing.assert_array_equal(pos, w_pos)
        if not focus_start:                      # (cur, next): one item -> consumer -> item move
            for a, b in zip(items.tolist(), pos.tolist()):
                assert any(b in g.user_consumed[u] for u in g.item_consumed[a]), (a, b)


def test_i2i_negatives_exclude_the_item_and_its_positive():
    import torch

    tr, di, _ = _trainer(num_neg=4)
    items = torch.randint(0, di["n_items"], (5000,), dtype=torch.int32, device="cuda")
    pos = torch.randint(0, di["n_items"], (5000,), dtype=torch.int32, device="cuda")
    neg = tr.negatives(pos, items=items).view(5000, 4).cpu().numpy()
    assert neg.min() >= 0 and neg.max() < di["n_items"]
    assert not np.any(neg == items.cpu().numpy()[:, None]) and not np.any(neg == pos.cpu().numpy()[:, None])
    assert len(np.unique(neg)) > 0.5 * di["n_items"]


def _internal_to_reference(tr, name, a):
    if name in ("item_proj.weight", "user_proj.weight"):
        a = np.concatenate([a[:, tr.d:], a[:, :tr.d]], axis=1)
    return (name if name == "dense_embeds" or "." in name else f"{name}.weight"), a


@pytest.mark.parametrize("paradigm,data", [("i2i", "pure"), ("u2i", "feat"), ("i2i", "feat")])
@pytest.mark.parametrize("loss_type", ["cross_entropy", "focal", "bpr", "max_margin"])
def test_full_step_matches_the_float64_oracle(paradigm, data, loss_type):
    from librecommender_b200.sage import init_state_dict

    z = golden()
    di = data_info(z, data)
    num_neg = 2 if loss_type in ("bpr", "focal") else 1
    sd = init_state_dict(di, paradigm, embed_size=16, num_layers=2, seed=3)
    cfg = dict(paradigm=paradigm, loss_type=loss_type, num_layers=2, num_neighbors=3, margin=0.8, lr=1e-3,
               epsilon=1e-8, reg=0.01 if loss_type != "focal" else None)
    tr, di, _ = _trainer(paradigm, data, state_dict=sd, loss_type=loss_type, num_neg=num_neg, margin=0.8,
                         reg=cfg["reg"], num_walks=2, sample_walk_len=3, seed=7)
    before = {k: v.detach().cpu().numpy().copy() for k, v in tr.params.items()}
    rng = np.random.default_rng(0)
    users = rng.integers(0, di["n_users"], 64)
    items = rng.integers(0, di["n_items"], 64)
    loss = tr.forward_backward(users, items) if paradigm == "u2i" else tr.forward_backward(batch_size=24)
    last = {k: (v.cpu().numpy() if hasattr(v, "cpu") else v) for k, v in tr.last.items() if k != "levels"}
    batch = dict(last, levels=[a.cpu().numpy() for a in tr.last["levels"]])
    l64, g64, p64 = orc.step(sd, batch, cfg, feats(di), feats(di, "user"))
    assert abs(float(loss) - l64) <= GPU_RTOL * max(abs(l64), 1e-3)
    grads = dict(_internal_to_reference(tr, k, v.cpu().numpy()) for k, v in tr.grads.items())
    for k, want in g64.items():
        scale = max(np.abs(want).max(), 1e-4)      # a gradient that cancels in float64 (bpr: the last bias)
        assert np.abs(grads[k] - want).max() <= GPU_RTOL * scale, (k, np.abs(grads[k] - want).max(), scale)
    tr.adam_update()
    lr = cfg["lr"]
    for k, v in tr.params.items():
        key, got = _internal_to_reference(tr, k, v.cpu().numpy())
        _, old = _internal_to_reference(tr, k, before[k])
        want, g = p64[key], g64[key] + (cfg["reg"] or 0.0) * old
        step_got, step_want = got - old, want - old
        assert np.abs(step_got).max() <= lr * 1.001 + 1e-7, key
        # Adam's first step is lr * sign(g): compare where g is well above the float32 gradient error
        sure = np.abs(g) > 10 * GPU_RTOL * max(np.abs(g).max(), 1e-4)
        np.testing.assert_allclose(step_got[sure], step_want[sure], rtol=0, atol=2e-2 * lr, err_msg=key)
        assert not np.any(tr.grads[k].cpu().numpy()), k                 # the update zeroes the gradients


def _movielens():
    """The fixture's user -> items lists split into train and held-out: a user's last item is held out when the
    user keeps two items and the item keeps a consumer."""
    g = np.load(MOVIELENS)
    n_users, n_items = int(g["n_users"]), int(g["n_items"])
    ip, idx = g["consumed_indptr"], g["consumed_idx"]
    item_count = np.bincount(idx, minlength=n_items)
    train, eval_u, eval_i = {}, [], []
    for u in range(n_users):
        items = idx[ip[u]:ip[u + 1]].tolist()
        if len(items) >= 3 and item_count[items[-1]] > 1:
            item_count[items[-1]] -= 1
            eval_u.append(u)
            eval_i.append(items[-1])
            items = items[:-1]
        train[u] = items
    item_consumed = {i: [] for i in range(n_items)}
    for u, items in train.items():
        for i in items:
            item_consumed[i].append(u)
    di = dict(n_users=n_users, n_items=n_items, user_consumed=train, item_consumed=item_consumed,
              user_sparse_col_index=g["user_sparse_col_index"].tolist(),
              item_sparse_col_index=g["item_sparse_col_index"].tolist(),
              user_dense_col_index=g["user_dense_col_index"].tolist(), item_dense_col_index=[],
              user_sparse_unique=g["user_sparse_unique"], item_sparse_unique=g["item_sparse_unique"],
              user_dense_unique=g["user_dense_unique"].astype(np.float32), item_dense_unique=None)
    return di, np.asarray(eval_u), np.asarray(eval_i)


@pytest.mark.parametrize("paradigm", ["i2i", "u2i"])
def test_movielens_epochs_lower_the_loss_and_raise_recall(paradigm):
    import torch

    from _bpr_oracle import ranking_metrics
    from librecommender_b200.sage import GraphSage, GraphSageTrainer, init_state_dict

    di, eval_u, eval_i = _movielens()
    sd0 = init_state_dict(di, paradigm, embed_size=16, num_layers=2, seed=0)
    tr = GraphSageTrainer(di, state_dict=sd0, paradigm=paradigm, num_neg=1, lr=3e-3, seed=0)
    users = np.repeat(np.arange(di["n_users"]), [len(di["user_consumed"][u]) for u in range(di["n_users"])])
    items = np.concatenate([di["user_consumed"][u] for u in range(di["n_users"])])
    losses = tr.fit(users, items, n_epochs=3, batch_size=512)
    assert losses[-1] < losses[0], losses
    indptr = np.concatenate([[0], np.cumsum([len(di["user_consumed"][u]) for u in range(di["n_users"])])])

    def recall(sd):
        eng = GraphSage(di, sd, paradigm=paradigm, num_layers=2, num_neighbors=3, seed=0)
        U, I = (t.cpu().numpy() for t in eng.set_embeddings())
        return ranking_metrics(U[:-1], I[:-1], indptr, items, eval_u, eval_i)[0], eng

    sd = tr.state_dict()
    assert all(isinstance(v, torch.Tensor) and v.dtype == torch.float32 for v in sd.values())
    assert {k: tuple(v.shape) for k, v in sd.items()} == {k: v.shape for k, v in sd0.items()}
    r0, _ = recall(sd0)
    r1, eng = recall(sd)
    assert r1 > r0, (r0, r1)
    assert np.asarray(eng.recommend_user(eval_u[:8], 10)).shape == (8, 10)
