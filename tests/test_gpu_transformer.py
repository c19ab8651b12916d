"""GPU: the Transformer engine (csrc/transformer.cu through feat_models.Transformer) against the float64
restatement of the reference graph in tests/_transformer_oracle.py (parity unpinned, see its header).

Rows-mode logits are held to the bound of test_gpu_feat_models._close (1e-5 relative); test_transformer_cpu.py shows
float32 meets it with 4x to spare on the same cases.  Grid mode (all-items scoring through the pair kernel) re-associates
the first MLP layer, so it is held to rows mode by the same bound, and each mode repeats bit for bit."""
import os
import sys
import types

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _transformer_oracle as to  # noqa: E402

from oracle import tf_models as tm  # noqa: E402

pytestmark = pytest.mark.gpu


def _engine(spec, w, seqs, lens, consumed=None):
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import Transformer

    return Transformer(spec, wio.transformer_weights(w), seqs, lens, consumed)


def _grid_rows(model, user_ids):
    N = model.n_items
    return model.logits(np.repeat(user_ids, N), np.tile(np.arange(N), len(user_ids))).cpu().numpy().reshape(-1, N)


def _oracle_grid(w, spec, seqs, lens, user_ids, N):
    uu, ii = np.repeat(user_ids, N), np.tile(np.arange(N), len(user_ids))
    sparse, dense = tm.row_features(spec, uu, ii)
    return to.transformer_forward(w, spec, uu, ii, seqs, lens, sparse, dense).reshape(len(user_ids), N)


@pytest.mark.parametrize("c", to.CASES, ids=to.case_id)
def test_logits_match_fp64(c):
    import torch

    rng, spec, w, seqs, lens = to.make_case(c)
    model = _engine(spec, w, seqs, lens)
    users, items, sparse, dense = to.case_rows(rng, spec, R=333)
    z = model.logits(users, items)
    got = z.cpu().numpy()
    to.close(got, to.transformer_forward(w, spec, users, items, seqs, lens, sparse, dense))
    if c[0] != "multi":      # explicit feature rows (a predict feed) give the same bits
        np.testing.assert_array_equal(got, model.logits(users, items, sparse_rows=sparse, dense_rows=dense).cpu().numpy())
    np.testing.assert_array_equal(model.predict(users, items), torch.sigmoid(z).cpu().numpy())


@pytest.mark.parametrize("c", to.CASES, ids=to.case_id)
def test_grid_matches_rows_and_repeats_bit_for_bit(c):
    import torch

    rng, spec, w, seqs, lens = to.make_case(c)
    model = _engine(spec, w, seqs, lens)
    assert model._hoistable()
    uid = np.array([0, 1, 2, spec["n_users"], 17, 5])
    u = torch.as_tensor(uid, device=model.device)
    a = model.score_all_items(u).cpu().numpy()
    np.testing.assert_array_equal(a, model.score_all_items(u).cpu().numpy())
    rows = _grid_rows(model, uid)
    np.testing.assert_array_equal(rows, _grid_rows(model, uid))
    to.close(a.reshape(-1), rows.reshape(-1).astype(np.float64))
    to.close(a.reshape(-1), _oracle_grid(w, spec, seqs, lens, uid, spec["n_items"]).reshape(-1))


@pytest.mark.parametrize("c", [to.CASES[0], to.CASES[1], to.CASES[4]], ids=to.case_id)
def test_recommend_matches_oracle_and_excludes_consumed(c):
    from oracle import ranking as orc

    rng, spec, w, seqs, lens = to.make_case(c, n_users=50, n_items=300)
    N = spec["n_items"]
    consumed = {u: rng.choice(N, size=int(rng.integers(1, 30)), replace=False).tolist() for u in range(50)}
    model = _engine(spec, w, seqs, lens, consumed)
    user_ids = rng.choice(50, size=17, replace=False)
    got = model.recommend(user_ids, 10, True)
    preds = _oracle_grid(w, spec, seqs, lens, user_ids, N).astype(np.float32)
    ref = orc.rank_recommendations("ranking", user_ids.tolist(), preds.reshape(-1), 10, N, consumed, True)
    assert orc.near_tie_mask(ref, got, preds, 1e-5).all()
    assert (got == ref).mean() > 0.98
    for r, u in enumerate(user_ids.tolist()):
        assert not set(got[r].tolist()) & set(consumed[u])


def test_large_attention_logits():
    """Target-attention logits around +-100 (item table scaled up): the softmax max subtraction."""
    c = to.CASES[0]
    rng, spec, w, seqs, lens = to.make_case(c)
    w["rms_item"] = (w["rms_item"] * 40).astype(np.float32)
    G = to.item_table(w, spec, "concat", np.float64)
    S = to.encode(w, G, seqs, lens, np.float64)
    q = to.rms_norm(G, w["rms_item"].astype(np.float64))
    assert np.abs(np.einsum("nd,btd->bnt", q, S[:, :, :q.shape[1]])).max() > 80
    model = _engine(spec, w, seqs, lens)
    users, items, sparse, dense = to.case_rows(rng, spec)
    got = model.logits(users, items).cpu().numpy()
    assert np.isfinite(got).all()
    to.close(got, to.transformer_forward(w, spec, users, items, seqs, lens, sparse, dense))
    import torch
    uid = np.array([3, 4])
    # logits near 100 carry ~1e-5 of float32 rounding each, which the grid's re-associated first layer does not
    # cancel the way rows mode happens to: three times the bound here
    to.close(model.score_all_items(torch.as_tensor(uid, device=model.device)).cpu().numpy().reshape(-1),
             _oracle_grid(w, spec, seqs, lens, uid, spec["n_items"]).reshape(-1), tol=3e-5)


def test_envelope_edge_T64_D128_L4():
    import torch

    from librecommender_b200 import synthetic as syn

    _, _, _, seqs, lens = to.make_case(to.CASES[0], n_users=12, n_items=40, T=64)
    rng = np.random.default_rng(12)
    spec = syn.make_spec(rng, 12, 40, [5], [6], 1, 1)       # K' = 32 * 3, D = 128
    w = syn.make_transformer_weights(rng, spec, 32, 4, 4, 64, (64, 32), True, "trainable", True, "concat", "keras")
    model = _engine(spec, w, seqs, lens)
    assert model.D == 128 and model.T == 64 and model.n_layers == 4
    users, items, sparse, dense = to.case_rows(rng, spec, R=50)
    to.close(model.logits(users, items).cpu().numpy(),
             to.transformer_forward(w, spec, users, items, seqs, lens, sparse, dense))
    uid = np.array([0, 1, 2, 12])
    a = model.score_all_items(torch.as_tensor(uid, device=model.device)).cpu().numpy()
    to.close(a.reshape(-1), _oracle_grid(w, spec, seqs, lens, uid, 40).reshape(-1))


def test_non_hoistable_mlp_falls_back_to_rows_with_swish():
    import torch

    c = ("feat", 16, "concat", 2, 1, False, "trainable", True, "keras")
    rng, spec, w, seqs, lens = to.make_case(c, hidden=(32, 80, 16, 8))   # 4 layers, H2 = 80: outside the pair kernel
    model = _engine(spec, w, seqs, lens)
    assert not model._hoistable()
    assert [a for _, _, a in model.mlp] == [2, 2, 2, 0]
    uid = np.array([0, 7, spec["n_users"]])
    got = model.score_all_items(torch.as_tensor(uid, device=model.device)).cpu().numpy()
    to.close(got.reshape(-1), _oracle_grid(w, spec, seqs, lens, uid, spec["n_items"]).reshape(-1))


@pytest.mark.parametrize("what", ["T", "width", "layers", "heads", "mlp_in"])
def test_unsupported_shapes_raise_before_launch(what):
    from librecommender_b200 import _lib
    from librecommender_b200 import synthetic as syn
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import Transformer

    rng = np.random.default_rng(9)
    spec = syn.make_spec(rng, 20, 30, [3], [4], 1, 1)
    K, H, L, T = 16, 1, 1, 10
    if what == "T":
        T = 65
    elif what == "width":
        K = 40                               # D = 40 * 3 + 40 = 160
    elif what == "layers":
        L = 5
    w = syn.make_transformer_weights(rng, spec, K, H, L, T, (32, 16))
    w = wio.transformer_weights(w)
    if what == "heads":
        w["num_heads"] = 3                   # D = 64
    elif what == "mlp_in":
        w["mlp"] = dict(w["mlp"], kernels=[w["mlp"]["kernels"][0][:-1]] + w["mlp"]["kernels"][1:],
                        bn_in={k: v[:-1] for k, v in w["mlp"]["bn_in"].items()})
    seqs = np.full((21, T), 30, dtype=np.int32)
    lens = np.ones(21, dtype=np.int32)
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        Transformer(spec, w, seqs, lens)
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

    from librecommender_b200 import _lib
    from librecommender_b200.dynamic_feats import assign_oov_rows
    from oracle import ranking as orc

    c = ("feat", 16, "concat", 2, 1, True, "trainable", True, "keras")
    rng, spec, w, seqs, lens = to.make_case(c, n_users=40, n_items=200)
    N, nu = spec["n_items"], spec["n_users"]
    spec["item_sparse_unique"][0, 0] = spec["item_sparse_unique"][N, 0]      # item 0 reads an OOV slot
    consumed = {u: rng.choice(N, size=int(rng.integers(1, 20)), replace=False).tolist() for u in range(nu)}
    model = _engine(spec, w, seqs, lens, consumed)
    u = 7
    # a behaviour sequence supplied for the call (grid mode); the cached sequence is restored afterwards
    seq = [5, 9, 33, 2]
    got = model.recommend_dynamic(u, 12, _data_info(spec, {}), seq=seq, inner_id=True)
    s2, l2 = seqs.copy(), lens.copy()
    s2[u] = N
    s2[u, :4], l2[u] = seq, 4
    preds = _oracle_grid(w, spec, s2, l2, np.array([u]), N).astype(np.float32)
    ref = orc.rank_recommendations("ranking", [u], preds.reshape(-1), 12, N, consumed, True)
    assert orc.near_tie_mask(ref, got, preds, 1e-5).all()
    assert model.lens[u].item() == lens[u]
    # a user dense feature supplied for the call: rows mode over the flat grid, one encoder pass
    g = spec["user_dense_col_index"][0]
    n0 = _lib.launch_count()
    got = model.recommend_dynamic(u, 12, _data_info(spec, {"age": g}), user_feats={"age": 3.5})
    launches = _lib.launch_count() - n0
    uu, ii = np.repeat(u, N), np.arange(N)
    sparse, dense = tm.row_features(spec, uu, ii)
    dense[:, g] = 3.5
    preds = to.transformer_forward(w, spec, uu, ii, seqs, lens, sparse, dense).astype(np.float32)
    ref = orc.rank_recommendations("ranking", [u], preds, 12, N, consumed, True)
    assert orc.near_tie_mask(ref, got, preds.reshape(1, N), 1e-5).all()
    assert launches < 20
    # default_recs: the OOV user, no consumed filter
    dr = model.default_recs(30)
    pre = _oracle_grid(w, spec, seqs, lens, np.array([nu]), N).astype(np.float32)
    ref = orc.rank_recommendations("ranking", [nu], pre.reshape(-1), 30, N, {}, False)
    assert orc.near_tie_mask(ref, dr[None], pre, 1e-5).all()
    # assign_oov rewrites the tables: the cached Qi / Pi are rebuilt
    uid = torch.arange(nu + 1, device=model.device)
    before = model.score_all_items(uid).cpu().numpy()
    oov = sorted({int(spec["user_sparse_unique"][nu, j]) for j in range(spec["user_sparse_unique"].shape[1])}
                 | {int(spec["item_sparse_unique"][N, j]) for j in range(spec["item_sparse_unique"].shape[1])})
    model.assign_oov(oov)
    after = model.score_all_items(uid).cpu().numpy()
    assert np.abs(after[:, 0] - before[:, 0]).max() > 1e-6
    w2 = assign_oov_rows(w, nu, N, oov)
    to.close(after.reshape(-1), _oracle_grid(w2, spec, seqs, lens, np.arange(nu + 1), N).reshape(-1))
