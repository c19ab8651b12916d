"""GPU: the SIM engine (csrc/sim.cu through feat_models.SIM) against the float64 restatement of the reference graph in
tests/_sim_oracle.py (parity unpinned, see its header).

Rows-mode logits are held to the bound of test_gpu_feat_models._close (1e-5 relative) on every pair, with the oracle
evaluated on the kernel's own GSU selection; test_sim_cpu.py shows float32 meets it with 4x to spare on the same cases.
The selection itself must equal float64's wherever float64's top-k boundary is not a near tie.  Grid mode (all-items
scoring through the pair kernel) re-associates the first MLP layer, so it is held to rows mode by the same bound, and
each mode repeats bit for bit."""
import os
import sys
import types

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _sim_oracle as so  # noqa: E402
import _transformer_oracle as to  # noqa: E402

from oracle import tf_models as tm  # noqa: E402

pytestmark = pytest.mark.gpu
K_SEL = so.TOPK_DEFAULT


def _engine(spec, w, seqs, consumed=None, k=K_SEL):
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import SIM

    return SIM(spec, wio.sim_weights(w), *seqs, user_consumed=consumed, search_topk=k)


def _oracle(w, spec, users, items, seqs, k=K_SEL, sel=None):
    sparse, dense = tm.row_features(spec, users, items)
    return so.sim_forward(w, spec, users, items, *seqs, k, sparse, dense, sel=sel)


def _oracle_grid(w, spec, seqs, user_ids, N, k=K_SEL):
    uu, ii = np.repeat(user_ids, N), np.tile(np.arange(N), len(user_ids))
    return _oracle(w, spec, uu, ii, seqs, k)[0].reshape(len(user_ids), N)


def _rows_grid(model, user_ids):
    N = model.n_items
    return model.logits(np.repeat(user_ids, N), np.tile(np.arange(N), len(user_ids))).cpu().numpy().reshape(-1, N)


def _check_selection(pos, ref_sel, margin, sk):
    """The kernel's selection equals float64's on every row whose boundary gap exceeds 1e-4 max(1, |s_k|); fewer than
    2 % of the rows may be excluded."""
    clear = margin > 1e-4 * np.maximum(1.0, sk)
    assert (~clear).mean() < 0.02, (~clear).mean()
    bad = np.nonzero(clear & (pos != ref_sel).any(axis=1))[0]
    assert bad.size == 0, (bad[:5], pos[bad[:2]], ref_sel[bad[:2]])


@pytest.mark.parametrize("c", so.CASES, ids=so.case_id)
def test_rows_logits_and_selection_match_fp64(c):
    import torch

    rng, spec, w, _, seqs = so.make_case(c)
    model = _engine(spec, w, seqs)
    users, items, _, _ = so.case_rows(rng, spec, R=600)
    _, pos = model.attention_rows(users, items)
    pos = pos.cpu().numpy()
    assert (np.diff(pos, axis=1) > 0).all()
    z = model.logits(users, items)
    ref, ref_sel, margin, sk = _oracle(w, spec, users, items, seqs)
    _check_selection(pos, ref_sel, margin, sk)
    ref_own, _, _, _ = _oracle(w, spec, users, items, seqs, sel=pos)
    to.close(z.cpu().numpy(), ref_own)
    np.testing.assert_array_equal(model.predict(users, items), torch.sigmoid(z).cpu().numpy())


def test_exact_ties_resolve_to_the_lower_position():
    """A long sequence of one repeated item next to others: every copy scores the same, the lowest copies win."""
    c = so.CASES[0]
    rng, spec, w, consumed, _ = so.make_case(c)
    from librecommender_b200.feat_models import recent_dual_sequences

    nu, N = spec["n_users"], spec["n_items"]
    for u in range(nu):
        consumed[u] = [3] * 40 + [int(i) for i in rng.integers(0, N, size=30)] + [3] * 40 + list(range(10))
    seqs = recent_dual_sequences(consumed, nu, N, so.L_DEFAULT, so.S_DEFAULT)
    model = _engine(spec, w, seqs)
    users = np.repeat(np.arange(4), N)
    items = np.tile(np.arange(N), 4)
    _, pos = model.attention_rows(users, items)
    pos = pos.cpu().numpy()
    _, ref_sel, margin, sk = _oracle(w, spec, users, items, seqs)
    _check_selection(pos, ref_sel, margin, sk)
    # the rows whose selection contains a copy of item 3 but not all of them took the lowest copies
    ls = seqs[0][users]
    copies = np.take_along_axis(ls, pos, axis=1) == 3
    part = copies.any(axis=1) & ~copies.all(axis=1)
    assert part.any()
    for r in np.nonzero(part)[0]:
        chosen = pos[r][copies[r]]
        all_copies = np.nonzero(ls[r] == 3)[0]
        assert (chosen == all_copies[:len(chosen)]).all()


@pytest.mark.parametrize("c", so.CASES, ids=so.case_id)
def test_grid_matches_rows_and_repeats_bit_for_bit(c):
    import torch

    # at K = 32 the default hidden (200, 80) needs more shared memory than the opt-in: a narrower MLP there
    rng, spec, w, _, seqs = so.make_case(c, hidden=(200, 80) if c[1] <= 16 else (128, 64))
    model = _engine(spec, w, seqs)
    assert model._hoistable()
    uid = np.array([0, 1, 2, spec["n_users"], 17, 5, 9, 10])
    u = torch.as_tensor(uid, device=model.device)
    a = model.score_all_items(u).cpu().numpy()
    np.testing.assert_array_equal(a, model.score_all_items(u).cpu().numpy())
    rows = _rows_grid(model, uid)
    np.testing.assert_array_equal(rows, _rows_grid(model, uid))
    to.close(a.reshape(-1), rows.reshape(-1).astype(np.float64))
    # the grid's pairs select what rows mode selects: scoring rows mode on its own selection reproduces it
    N = spec["n_items"]
    uu, ii = np.repeat(uid, N), np.tile(np.arange(N), len(uid))
    _, pos = model.attention_rows(uu, ii)
    ref_own = _oracle(w, spec, uu, ii, seqs, sel=pos.cpu().numpy())[0]
    to.close(a.reshape(-1), ref_own)


@pytest.mark.parametrize("c", [so.CASES[0], so.CASES[3]], ids=so.case_id)
def test_recommend_matches_oracle_and_excludes_consumed(c):
    from oracle import ranking as orc

    rng, spec, w, consumed, seqs = so.make_case(c, n_items=300)
    N = spec["n_items"]
    model = _engine(spec, w, seqs, consumed)
    user_ids = rng.choice(spec["n_users"], size=12, replace=False)
    got = model.recommend(user_ids, 10, True)
    preds = _oracle_grid(w, spec, seqs, user_ids, N).astype(np.float32)
    ref = orc.rank_recommendations("ranking", user_ids.tolist(), preds.reshape(-1), 10, N, consumed, True)
    assert orc.near_tie_mask(ref, got, preds, 1e-5).all()
    for r, u in enumerate(user_ids.tolist()):
        assert not set(got[r].tolist()) & set(consumed[u])


def test_envelope_edge_rows_mode():
    """K = 64, L = 256, S = 64, search_topk = 32, 4 heads: past the pair kernel's shared memory, so all-items scoring
    runs in rows mode."""
    import torch

    c = ("feat", 64, 4, True, "keras")
    rng, spec, w, _, seqs = so.make_case(c, n_users=18, n_items=60, L=256, S=64, k=32, hidden=(64, 32))
    model = _engine(spec, w, seqs, k=32)
    assert (model.K, model.L, model.S, model.topk) == (64, 256, 64, 32) and not model._hoistable()
    users, items, _, _ = so.case_rows(rng, spec, R=200)
    _, pos = model.attention_rows(users, items)
    pos = pos.cpu().numpy()
    ref, ref_sel, margin, sk = _oracle(w, spec, users, items, seqs, k=32)
    _check_selection(pos, ref_sel, margin, sk)
    to.close(model.logits(users, items).cpu().numpy(), _oracle(w, spec, users, items, seqs, k=32, sel=pos)[0])
    uid = np.array([0, 1, 18])
    got = model.score_all_items(torch.as_tensor(uid, device=model.device)).cpu().numpy()
    to.close(got.reshape(-1), _rows_grid(model, uid).reshape(-1).astype(np.float64))


def test_grid_with_a_wide_three_layer_mlp():
    """H1 = 256, H2 = 96 (past the 64-unit second layer of the other pair kernels), H3 = 48 at K = 16 fits the pair
    kernel's shared memory; the widest MLP of its envelope, (256, 128, 64), does not and is scored in rows mode."""
    import torch

    c = ("ids", 16, 2, True, "legacy")
    rng, spec, w, _, seqs = so.make_case(c, hidden=(256, 96, 48))
    model = _engine(spec, w, seqs)
    assert model._hoistable()
    wide = _engine(spec, so.make_case(c, hidden=(256, 128, 64))[2], seqs)
    assert not wide._hoistable()
    uid = np.array([0, 1, 2, 3, spec["n_users"]])
    a = model.score_all_items(torch.as_tensor(uid, device=model.device)).cpu().numpy()
    to.close(a.reshape(-1), _rows_grid(model, uid).reshape(-1).astype(np.float64))


def test_non_hoistable_mlp_falls_back_to_rows():
    import torch

    c = ("feat", 16, 2, True, "keras")
    rng, spec, w, _, seqs = so.make_case(c, hidden=(32, 80, 16, 8))     # 4 layers: outside the pair kernel
    model = _engine(spec, w, seqs)
    assert not model._hoistable()
    uid = np.array([0, 7, spec["n_users"]])
    got = model.score_all_items(torch.as_tensor(uid, device=model.device)).cpu().numpy()
    rows = _rows_grid(model, uid)
    np.testing.assert_array_equal(got, rows)
    N = spec["n_items"]
    uu, ii = np.repeat(uid, N), np.tile(np.arange(N), len(uid))
    _, pos = model.attention_rows(uu, ii)
    to.close(got.reshape(-1), _oracle(w, spec, uu, ii, seqs, sel=pos.cpu().numpy())[0])


@pytest.mark.parametrize("what", ["K", "heads", "L", "S", "topk", "topk_over_L", "mlp_in"])
def test_unsupported_shapes_raise_before_launch(what):
    from librecommender_b200 import _lib
    from librecommender_b200 import synthetic as syn
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import SIM

    rng = np.random.default_rng(9)
    spec = syn.make_spec(rng, 20, 30, [3], [4], 1, 1)
    K, L, S, k = 16, 100, 10, 10
    if what == "K":
        K = 72
    elif what == "L":
        L = 257
    elif what == "S":
        S = 65
    elif what == "topk":
        k = 33
    elif what == "topk_over_L":
        L, k = 8, 9
    w = wio.sim_weights(syn.make_sim_weights(rng, spec, K, 2, (32, 16)))
    if what == "heads":
        w["num_heads"] = 3
    elif what == "mlp_in":
        w["mlp"] = dict(w["mlp"], kernels=[w["mlp"]["kernels"][0][:-1]] + w["mlp"]["kernels"][1:],
                        bn_in={kk: v[:-1] for kk, v in w["mlp"]["bn_in"].items()})
    seqs = (np.full((21, L), 30, dtype=np.int32), np.ones(21, dtype=np.int32), np.full((21, S), 30, dtype=np.int32),
            np.ones(21, dtype=np.int32))
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        SIM(spec, w, *seqs, search_topk=k)
    assert _lib.launch_count() == n0


def _data_info(spec, names_dense):
    col = lambda idx: types.SimpleNamespace(index=list(idx))      # noqa: E731
    return types.SimpleNamespace(
        n_items=spec["n_items"], user_sparse_unique=spec["user_sparse_unique"],
        item_sparse_unique=spec["item_sparse_unique"], user_sparse_col=col(spec["user_sparse_col_index"]),
        item_sparse_col=col(spec["item_sparse_col_index"]), user_dense_unique=spec["user_dense_unique"],
        item_dense_unique=spec["item_dense_unique"], user_dense_col=col(spec["user_dense_col_index"]),
        item_dense_col=col(spec["item_dense_col_index"]), item2id={i: i for i in range(spec["n_items"])},
        col_name_mapping={"dense_col": names_dense, "sparse_col": {}}, sparse_idx_mapping={}, sparse_offset=[])


def test_recommend_dynamic_default_recs_and_assign_oov():
    import torch

    from librecommender_b200.dynamic_feats import assign_oov_rows, build_dual_seq
    from oracle import ranking as orc

    c = ("feat", 16, 2, True, "keras")
    rng, spec, w, consumed, seqs = so.make_case(c, n_items=200)
    N, nu = spec["n_items"], spec["n_users"]
    model = _engine(spec, w, seqs, consumed)
    u = 7
    # a behaviour sequence supplied for the call (grid mode); the cached rows are restored afterwards
    seq = [int(i) for i in rng.integers(0, N, size=60)]
    got = model.recommend_dynamic(u, 12, _data_info(spec, {}), seq=seq, inner_id=True)
    s2 = [a.copy() for a in seqs]
    for a, v in zip(s2, build_dual_seq(seq, N, so.L_DEFAULT, so.S_DEFAULT, inner_id=True)):
        a[u] = v[0]
    preds = _oracle_grid(w, spec, s2, np.array([u]), N).astype(np.float32)
    ref = orc.rank_recommendations("ranking", [u], preds.reshape(-1), 12, N, consumed, True)
    assert orc.near_tie_mask(ref, got, preds, 1e-5).all()
    assert model.long_lens[u].item() == seqs[1][u] and model.lens[u].item() == seqs[3][u]
    assert (model.long_seqs[u].cpu().numpy() == seqs[0][u]).all()
    # a user dense feature supplied for the call: rows mode over the flat grid
    g = spec["user_dense_col_index"][0]
    got = model.recommend_dynamic(u, 12, _data_info(spec, {"age": g}), user_feats={"age": 3.5})
    uu, ii = np.repeat(u, N), np.arange(N)
    sparse, dense = tm.row_features(spec, uu, ii)
    dense[:, g] = 3.5
    preds = so.sim_forward(w, spec, uu, ii, *seqs, K_SEL, sparse, dense)[0].astype(np.float32)
    ref = orc.rank_recommendations("ranking", [u], preds, 12, N, consumed, True)
    assert orc.near_tie_mask(ref, got, preds.reshape(1, N), 1e-5).all()
    # default_recs: the OOV user, no consumed filter
    dr = model.default_recs(30)
    pre = _oracle_grid(w, spec, seqs, np.array([nu]), N).astype(np.float32)
    ref = orc.rank_recommendations("ranking", [nu], pre.reshape(-1), 30, N, {}, False)
    assert orc.near_tie_mask(ref, dr[None], pre, 1e-5).all()
    # assign_oov rewrites the tables: Gp and the cached item part are rebuilt
    uid = torch.arange(nu + 1, device=model.device)
    gp_before = model.Gp.clone()
    before = model.score_all_items(uid).cpu().numpy()
    oov = sorted({int(spec["user_sparse_unique"][nu, j]) for j in range(spec["user_sparse_unique"].shape[1])}
                 | {int(spec["item_sparse_unique"][N, j]) for j in range(spec["item_sparse_unique"].shape[1])})
    model.assign_oov(oov)
    assert (model.Gp[N] - gp_before[N]).abs().max().item() > 1e-6
    after = model.score_all_items(uid).cpu().numpy()
    assert np.abs(after - before).max() > 1e-6
    w2 = assign_oov_rows(w, nu, N, oov)
    uu, ii = np.repeat(np.arange(nu + 1), N), np.tile(np.arange(N), nu + 1)
    _, pos = model.attention_rows(uu, ii)
    to.close(after.reshape(-1), _oracle(w2, spec, uu, ii, seqs, sel=pos.cpu().numpy())[0])
