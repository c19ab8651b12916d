"""GraphSage training without a GPU: the walk-pair rule of ``tests/_sage_train_oracle.py`` (fed the kernel's keyed
draws on the GPU) against the reference's ``pairs_from_random_walk`` on the same Python ``random`` stream and on a
hand-built graph (order, ``focus_start``, the no-neighbour pair), the float64 oracle against the reference's own
``GraphSageModel`` and losses, the torch-Adam-as-TF-Adam mapping against ``torch.optim.Adam``, the trainer's
``ValueError`` for every option it does not build, the initial state dict, and the C-ABI rejections."""
import random

import numpy as np
import pytest
import torch

import _sage_oracle as sorc
import _sage_train_oracle as orc
from test_sage_cpu import data_info, feats, golden, message, state_dict


def _graph(z, data="pure"):
    di = data_info(z, data)
    return di, sorc.Graph(di["user_consumed"], di["item_consumed"], di["n_users"], di["n_items"])


def _python_one_walk(g):
    def one_walk(i, w, t, cur):
        user = random.choice(g.item_consumed[cur])
        return random.choice(g.user_consumed[user])
    return one_walk


@pytest.mark.parametrize("focus_start", [False, True])
def test_walk_rule_matches_the_reference_on_its_random_stream(focus_start):
    from oracle.ref_loader import load_reference, reference_available

    if not reference_available():
        pytest.skip("reference not importable")
    load_reference()
    from libreco.sampling.random_walks import pairs_from_random_walk

    z = golden()
    di, g = _graph(z)
    starts = np.random.default_rng(3).integers(0, di["n_items"], size=40).tolist()
    # an item whose only consumer consumed nothing else: has_no_neighbor
    lonely = [v for v in range(di["n_items"]) if g.has_no_neighbor(v)]
    starts += lonely[:2]
    random.seed(11)
    want_i, want_p = pairs_from_random_walk(starts, g.user_consumed, g.item_consumed, 4, 3, focus_start)
    random.seed(11)
    got_i, got_p, counts = orc.walk_rule(starts, g.has_no_neighbor, _python_one_walk(g), 4, 3, focus_start)
    np.testing.assert_array_equal(got_i, want_i)
    np.testing.assert_array_equal(got_p, want_p)
    assert counts.sum() == got_i.size and counts.size == len(starts) * 5


def test_walk_rule_order_focus_start_and_the_lonely_pair():
    # items 0..3; user 0: [0, 1], user 1: [1, 2], user 2: [3] (item 3 has no neighbour)
    user_consumed = {0: [0, 1], 1: [1, 2], 2: [3]}
    item_consumed = {0: [0], 1: [0, 1], 2: [1], 3: [2]}
    g = sorc.Graph(user_consumed, item_consumed, 3, 4)
    script = {(0, 0, 0): 1, (0, 0, 1): 1, (0, 1, 0): 0, (0, 1, 1): 1, (1, 0, 0): 3, (1, 0, 1): 3,
              (1, 1, 0): 3, (1, 1, 1): 3}

    def one_walk(i, w, t, cur):
        return script[(i, w, t)]

    items, pos, counts = orc.walk_rule([0, 3], g.has_no_neighbor, one_walk, 2, 2, False)
    # start 0: walk 0 0->1 (pair), 1->1 (none); walk 1 0->0 (none), 0->1 (pair); start 3: (3, 3) once, walks stay
    np.testing.assert_array_equal(items, [0, 0, 3])
    np.testing.assert_array_equal(pos, [1, 1, 3])
    np.testing.assert_array_equal(counts, [0, 1, 1, 1, 0, 0])
    items, pos, counts = orc.walk_rule([0, 3], g.has_no_neighbor, one_walk, 2, 2, True)
    # focus_start: (start, next) whenever next != start, 1->1 included
    np.testing.assert_array_equal(items, [0, 0, 0, 3])
    np.testing.assert_array_equal(pos, [1, 1, 1, 3])
    np.testing.assert_array_equal(counts, [0, 2, 1, 1, 0, 0])


def test_keyed_walk_pairs_are_two_hop_moves():
    z = golden()
    di, g = _graph(z)
    starts, items, pos, counts = orc.keyed_walk_pairs(g, di["n_items"], 30, 5, 4, False, 1234567890123, 7)
    assert counts.sum() == items.size == pos.size
    assert np.all((starts >= 0) & (starts < di["n_items"]))
    for a, b in zip(items.tolist(), pos.tolist()):
        users = set(g.item_consumed[a])
        assert any(b in g.user_consumed[u] for u in users), (a, b)
    again = orc.keyed_walk_pairs(g, di["n_items"], 30, 5, 4, False, 1234567890123, 8)
    assert not np.array_equal(again[0], starts)          # the step keys the starts


def test_adam_mapping_matches_torch_adam():
    from librecommender_b200.sage import BETA1, BETA2, adam_step_constants

    rng = np.random.default_rng(0)
    lr, eps, reg = 3e-3, 1e-8, 0.01
    p0 = rng.standard_normal(64)
    grads = [rng.standard_normal(64) * 10.0 ** -k for k in range(6)]
    p_t = torch.tensor(p0, requires_grad=True)
    opt = torch.optim.Adam([p_t], lr=lr, eps=eps, weight_decay=reg)
    p, m, v = p0.copy(), np.zeros(64), np.zeros(64)
    for t, gr in enumerate(grads, start=1):
        p_t.grad = torch.tensor(gr)
        opt.step()
        g = gr + reg * p                              # weight_decay: reg * p on the gradient (b200_axpy)
        lr_t, eps_hat = adam_step_constants(lr, eps, t)
        m = BETA1 * m + (1 - BETA1) * g               # b200_adam_dense_dev
        v = BETA2 * v + (1 - BETA2) * g * g
        p = p - lr_t * m / (np.sqrt(v) + eps_hat)
        np.testing.assert_allclose(p, p_t.detach().numpy(), rtol=1e-12, atol=1e-15)


@pytest.mark.parametrize("kw,name", [
    (dict(lr_decay=True), "lr_decay"), (dict(amsgrad=True), "amsgrad"), (dict(dropout_rate=0.1), "dropout_rate"),
    (dict(remove_edges=True), "remove_edges"), (dict(sampler="popular"), "popular"),
    (dict(sampler="out-batch"), "out-batch"), (dict(start_node="unpopular"), "unpopular"),
    (dict(paradigm="u2i", sampler="popular"), "popular"), (dict(sampler="unconsumed"), "sampler"),
    (dict(loss_type="softmax"), "loss_type"), (dict(paradigm="x"), "paradigm"), (dict(num_neg=0), "num_neg"),
])
def test_out_of_scope_options_raise_value_error(kw, name):
    from librecommender_b200.sage import GraphSageTrainer

    di = data_info(golden(), "pure")
    with pytest.raises(ValueError, match=name):
        GraphSageTrainer(di, **kw)


@pytest.mark.parametrize("data,paradigm", [("pure", "i2i"), ("feat", "u2i"), ("feat", "i2i")])
def test_init_state_dict_has_the_reference_keys_and_shapes(data, paradigm):
    from librecommender_b200.sage import init_state_dict

    z = golden()
    di = data_info(z, data)
    want = {k: tuple(np.shape(v)) for k, v in state_dict(z, f"{data}_graphsage_{paradigm}").items()}
    d0 = want["item_embeds.weight"][1]
    got = {k: v.shape for k, v in init_state_dict(di, paradigm, embed_size=d0, num_layers=2, seed=1).items()}
    assert got == want
    sd = init_state_dict(di, paradigm, embed_size=8, num_layers=3, seed=1)
    assert {k for k in sd if k.startswith("w_linears")} == {f"w_linears.{i}.{p}" for i in range(3)
                                                           for p in ("weight", "bias")}
    bound = lambda shp, gain=1.0: gain * np.sqrt(6.0 / (shp[0] + shp[1]))   # noqa: E731
    assert np.abs(sd["w_linears.0.weight"]).max() <= bound((8, 16), np.sqrt(2.0))
    assert np.abs(sd["w_linears.2.weight"]).max() <= bound((8, 16))
    assert not np.any(sd["w_linears.1.bias"]) and not np.any(sd["item_proj.bias"])


@pytest.mark.parametrize("data,paradigm", [("pure", "i2i"), ("feat", "i2i"), ("feat", "u2i")])
def test_oracle_matches_the_reference_module_forward_and_gradients(data, paradigm):
    from oracle.ref_loader import load_reference, reference_available

    if not reference_available():
        pytest.skip("reference not importable")
    load_reference()
    z = golden()
    di = data_info(z, data)
    case = f"{data}_graphsage_{paradigm}"
    sd = state_dict(z, case)
    items, nbs, offs, _ = message(z, case, "graphsage")
    d = sd["item_embeds.weight"].shape[1]
    ref = orc.reference_model(di, paradigm, d, 2).double()
    ref.load_state_dict({k: torch.as_tensor(np.asarray(v, np.float64)) for k, v in sd.items()})

    def side(ids, s="item"):
        sp = di[f"{s}_sparse_unique"]
        dn = di[f"{s}_dense_unique"]
        return (torch.as_tensor(np.asarray(sp)[ids]) if sp is not None else None,
                torch.as_tensor(np.asarray(dn, np.float64)[ids]) if dn is not None else None)

    sp, dn = side(items)
    nsp, ndn = zip(*[side(n) for n in nbs])
    out_ref = ref(torch.as_tensor(items), sp, dn, [torch.as_tensor(n) for n in nbs], list(nsp), list(ndn),
                  [torch.as_tensor(o) for o in offs])
    P = orc.params(sd)
    out = orc.item_repr(P, items, nbs, offs, 2, feats(di))
    np.testing.assert_allclose(out.detach().numpy(), out_ref.detach().numpy(), rtol=1e-12, atol=1e-12)
    w = torch.as_tensor(np.random.default_rng(0).standard_normal(out.shape))
    (out * w).sum().backward()
    (out_ref * w).sum().backward()
    ref_grads = dict(ref.named_parameters())
    for k, v in P.items():
        if (k.startswith("user") and paradigm == "u2i") or v.grad is None:     # the user tower / an unused table
            assert ref_grads[k].grad is None or not ref_grads[k].grad.any(), k
            continue
        np.testing.assert_allclose(v.grad.numpy(), ref_grads[k].grad.numpy(), rtol=1e-10, atol=1e-12, err_msg=k)
    if paradigm == "u2i":
        users = np.arange(min(5, di["n_users"]))
        usp, udn = side(users, "user")
        np.testing.assert_allclose(orc.user_repr(P, users, feats(di, "user")).detach().numpy(),
                                   ref.user_repr(torch.as_tensor(users), usp, udn).detach().numpy(), rtol=1e-12,
                                   atol=1e-12)


@pytest.mark.parametrize("f", [1, 3])
def test_oracle_losses_match_the_reference_functions(f):
    from oracle.ref_loader import load_reference, reference_available

    if not reference_available():
        pytest.skip("reference not importable")
    load_reference()
    from libreco.torchops.loss import (bpr_loss, compute_pair_scores, max_margin_loss, pairwise_bce_loss,
                                       pairwise_focal_loss)

    rng = np.random.default_rng(1)
    q, p, n = (torch.as_tensor(rng.standard_normal(s)) for s in ((6, 4), (6, 4), (6 * f, 4)))
    for loss_type in ("cross_entropy", "focal", "bpr", "max_margin"):
        repeat = loss_type in ("bpr", "max_margin")
        pos, neg = orc.pair_scores(q, p, n, repeat)
        rpos, rneg = compute_pair_scores(q, p, n, repeat)
        np.testing.assert_allclose(pos.numpy(), rpos.numpy(), rtol=1e-14)
        np.testing.assert_allclose(neg.numpy(), rneg.numpy(), rtol=1e-14)
        for paradigm in ("i2i", "u2i"):
            mean = paradigm == "u2i"
            want = {"cross_entropy": lambda: pairwise_bce_loss(rpos, rneg, mean=mean),
                    "focal": lambda: pairwise_focal_loss(rpos, rneg, mean=mean),
                    "bpr": lambda: bpr_loss(rpos, rneg),
                    "max_margin": lambda: max_margin_loss(rpos, rneg, 0.7)}[loss_type]()
            got = orc.loss(loss_type, pos, neg, paradigm, 0.7)
            np.testing.assert_allclose(float(got), float(want), rtol=1e-13)


def test_cabi_rejections_return_minus_two():
    import ctypes

    from librecommender_b200 import _lib

    lib, p = _lib.lib, ctypes.c_void_p(8)
    assert lib.b200_sage_aggregate_backward(p, 2, None, 4, p, 1, None, None, None, 3, 0, p, 1, None) == -2
    assert lib.b200_sage_aggregate_backward(p, 2, None, 4, p, 1, None, None, None, 3, 129, p, 129, None) == -2
    assert lib.b200_sage_aggregate_backward(p, 3, None, 4, p, 2, None, None, None, 3, 2, p, 2, None) == -2
    assert lib.b200_sage_aggregate_backward(None, 4, None, 4, p, 2, None, None, None, 3, 2, p, 2, None) == -2
    assert lib.b200_sage_walk_pairs(p, p, p, p, 10, 4, 0, 5, 0, 1, 0, p, p, p, None, None, None) == -2
    assert lib.b200_sage_walk_pairs(p, p, p, p, 10, 4, 10, 1025, 0, 1, 0, p, p, p, None, None, None) == -2
    assert lib.b200_sage_walk_pairs(p, p, p, p, 10, 4, 10, 5, 0, 1, 0, p, None, p, None, None, None) == -2
    assert lib.b200_sage_i2i_negatives(p, p, 4, 0, 10, 10, 1, 0, p, None) == -2
    assert lib.b200_sage_i2i_negatives(p, None, 4, 1, 10, 10, 1, 0, p, None) == -2
