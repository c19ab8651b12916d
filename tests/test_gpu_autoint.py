"""GPU: the AutoInt engine (csrc/autoint.cu through feat_models.AutoInt) against the float64 restatement of the
reference graph in tests/_autoint_oracle.py (parity unpinned, see its header).

Logits are held to the bound of test_gpu_feat_models._close (1e-5 relative); test_autoint_cpu.py shows float32
meets it with 4x to spare on the same cases.  The rows mode (materialised concat) and the grid mode (all-items
scoring from a user-side and an item-side block) must agree bit for bit."""
import os
import sys
import types

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _autoint_oracle as ao  # noqa: E402

pytestmark = pytest.mark.gpu


def _engine(spec, w, consumed=None):
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import AutoInt

    return AutoInt(spec, wio.autoint_weights(w), consumed)


def _grid_rows(model, user_ids):
    """Rows-mode logits of the explicit (user, item) grid, [b, N]."""
    N = model.n_items
    return model.logits(np.repeat(user_ids, N), np.tile(np.arange(N), len(user_ids))).cpu().numpy().reshape(-1, N)


@pytest.mark.parametrize("c", ao.CASES, ids=ao.case_id)
def test_logits_match_fp64(c):
    import torch

    rng, spec, w = ao.make_case(c)
    model = _engine(spec, w)
    users, items, sparse, dense = ao.case_rows(rng, spec, R=777)         # OOV rows included, 777 % 8 != 0
    z = model.logits(users, items)
    got = z.cpu().numpy()
    ao.close(got, ao.autoint_forward(w, users, items, sparse, dense, np.float64))
    if c[0] != "multi":      # explicit feature rows (a predict feed) give the same bits
        got2 = model.logits(users, items, sparse_rows=sparse, dense_rows=dense).cpu().numpy()
        np.testing.assert_array_equal(got, got2)
    np.testing.assert_array_equal(model.predict(users, items), torch.sigmoid(z).cpu().numpy())


@pytest.mark.parametrize("c", ao.CASES, ids=ao.case_id)
def test_grid_equals_rows_bit_for_bit(c):
    import torch

    rng, spec, w = ao.make_case(c)
    model = _engine(spec, w)
    uid = np.array([0, 5, spec["n_users"], 17, 3])
    u = torch.as_tensor(uid, device=model.device)
    a = model.score_all_items(u).cpu().numpy()
    b = model.score_all_items(u).cpu().numpy()
    np.testing.assert_array_equal(a, b)
    np.testing.assert_array_equal(a, _grid_rows(model, uid))


@pytest.mark.parametrize("c", [ao.CASES[0], ao.CASES[1], ao.CASES[8]], ids=ao.case_id)
def test_recommend_all_items_matches_oracle(c):
    from oracle import ranking as orc
    from oracle import tf_models as tm

    rng, spec, w = ao.make_case(c, n_users=80, n_items=400)
    N = spec["n_items"]
    consumed = {u: rng.choice(N, size=int(rng.integers(1, 40)), replace=False).tolist() for u in range(80)}
    model = _engine(spec, w, consumed)
    user_ids = rng.choice(80, size=23, replace=False)
    got = model.recommend(user_ids, 10, True)
    uu, ii = np.repeat(user_ids, N), np.tile(np.arange(N), len(user_ids))
    sparse, dense = tm.row_features(spec, uu, ii)
    preds = ao.autoint_forward(w, uu, ii, sparse, dense, np.float64).astype(np.float32)
    ref = orc.rank_recommendations("ranking", user_ids.tolist(), preds, 10, N, consumed, True)
    assert orc.near_tie_mask(ref, got, preds.reshape(len(user_ids), N), 1e-5).all()
    assert (got == ref).mean() > 0.98
    for r, u in enumerate(user_ids.tolist()):
        assert not set(got[r].tolist()) & set(consumed[u])


def test_max_fields_and_max_widths():
    """F = 2 + 128 fields, K = 64, D = 64, four layers: one pair fills ~150 KB of shared memory."""
    from librecommender_b200 import synthetic as syn

    rng = np.random.default_rng(4)
    spec = syn.make_spec(rng, 20, 30, [3] * 64, [3] * 63, 1, 0)
    w = syn.make_autoint_weights(rng, spec, 64, (32, 16, 1, 32), 2, True, "keras")
    model = _engine(spec, w)
    assert model.F == 130
    users, items, sparse, dense = ao.case_rows(rng, spec, R=45)
    ao.close(model.logits(users, items).cpu().numpy(), ao.autoint_forward(w, users, items, sparse, dense))
    uid = np.array([1, 20])
    import torch
    np.testing.assert_array_equal(model.score_all_items(torch.as_tensor(uid, device=model.device)).cpu().numpy(),
                                  _grid_rows(model, uid))


def test_single_item_catalogue():
    import torch

    rng, spec, w = ao.make_case(("feat", 16, None, 2, True, "keras"), n_users=40, n_items=1)
    model = _engine(spec, w)
    uid = np.arange(41)
    got = model.score_all_items(torch.as_tensor(uid, device=model.device)).cpu().numpy()
    np.testing.assert_array_equal(got, _grid_rows(model, uid))
    users, items = uid, np.zeros(41, dtype=np.int64)
    from oracle import tf_models as tm
    sparse, dense = tm.row_features(spec, users, items)
    ao.close(got[:, 0], ao.autoint_forward(w, users, items, sparse, dense))
    assert model.recommend(uid[:5], 1, False).tolist() == [[0]] * 5


def test_large_attention_logits():
    rng, spec, w = ao.make_case(ao.LARGE_LOGIT_CASE)
    rows = ao.case_rows(rng, spec)
    ao.scale_to_large_logits(w, rows)
    assert np.abs(ao.attention_logits_first_layer(w, *rows)).max() > 80
    got = _engine(spec, w).logits(rows[0], rows[1]).cpu().numpy()
    assert np.isfinite(got).all()
    ao.close(got, ao.autoint_forward(w, *rows))


@pytest.mark.parametrize("what", ["K", "layers", "width", "heads", "out_kernel", "fields"])
def test_unsupported_shapes_raise_before_launch(what):
    from librecommender_b200 import _lib
    from librecommender_b200 import synthetic as syn
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import AutoInt

    rng = np.random.default_rng(8)
    spec = syn.make_spec(rng, 20, 30, [3], [4], 1, 1)
    K, att, H = 16, (8, 8), 2
    if what == "K":
        K = 65
    elif what == "layers":
        att = (4, 4, 4, 4, 4)
    elif what == "width":
        att = (40,)                      # D = 80
    elif what == "fields":
        spec = syn.make_spec(rng, 20, 30, [3] * 64, [3] * 64, 1, 0)      # F = 131
    w = wio.autoint_weights(syn.make_autoint_weights(rng, spec, K, att, H, True, "keras"))
    if what == "heads":
        w["num_heads"] = 3               # D = 16 is not a multiple of 3
    elif what == "out_kernel":
        w["out_kernel"] = w["out_kernel"][:-1]
    n0 = _lib.launch_count()
    with pytest.raises(ValueError):
        AutoInt(spec, w)
    assert _lib.launch_count() == n0


def _data_info(spec, names_dense):
    """The DataInfo attributes dynamic_feature_rows reads, for a layout without sparse overrides."""
    col = lambda idx: types.SimpleNamespace(index=list(idx))      # noqa: E731
    return types.SimpleNamespace(
        n_items=spec["n_items"], user_sparse_unique=spec["user_sparse_unique"],
        item_sparse_unique=spec["item_sparse_unique"], user_sparse_col=col(spec["user_sparse_col_index"]),
        item_sparse_col=col(spec["item_sparse_col_index"]), user_dense_unique=spec["user_dense_unique"],
        item_dense_unique=spec["item_dense_unique"], user_dense_col=col(spec["user_dense_col_index"]),
        item_dense_col=col(spec["item_dense_col_index"]),
        col_name_mapping={"dense_col": names_dense, "sparse_col": {}}, sparse_idx_mapping={}, sparse_offset=[])


def test_recommend_dynamic_default_recs_assign_oov_and_shim():
    import torch

    from librecommender_b200.dynamic_feats import assign_oov_rows
    from librecommender_b200.recommendation import recommend_tf_feat
    from oracle import ranking as orc
    from oracle import tf_models as tm

    rng, spec, w = ao.make_case(ao.CASES[2], n_users=60, n_items=300)
    N, nu = spec["n_items"], spec["n_users"]
    # item 0 reads its first sparse field's OOV slot, so assign_oov changes an item-side block row
    spec["item_sparse_unique"][0, 0] = spec["item_sparse_unique"][N, 0]
    consumed = {u: rng.choice(N, size=int(rng.integers(1, 30)), replace=False).tolist() for u in range(nu)}
    model = _engine(spec, w, consumed)
    allu, alli = np.repeat(np.arange(nu + 1), N), np.tile(np.arange(N), nu + 1)

    def oracle_scores(wts, users, items, dense_override=None):
        sparse, dense = tm.row_features(spec, users, items)
        if dense_override is not None:
            dense[:, dense_override[0]] = dense_override[1]
        return ao.autoint_forward(wts, users, items, sparse, dense).astype(np.float32)

    # recommend_dynamic with a user dense feature supplied for the call (rows mode over the explicit grid)
    g = spec["user_dense_col_index"][0]
    di = _data_info(spec, {"age": g})
    u = 7
    preds = oracle_scores(w, np.repeat(u, N), np.arange(N), (g, 3.5))
    got = model.recommend_dynamic(u, 12, di, user_feats={"age": 3.5})
    ref = orc.rank_recommendations("ranking", [u], preds, 12, N, consumed, True)
    assert orc.near_tie_mask(ref, got, preds.reshape(1, N), 1e-5).all()
    base = oracle_scores(w, np.repeat(u, N), np.arange(N))
    assert np.abs(base - preds).max() > 1e-4
    # the shim hands a single-user call with features to the engine, and a batch to recommend
    shim_model = types.SimpleNamespace(b200_engine=model, n_items=N, n_users=nu, task="ranking", data_info=di,
                                       user_consumed=consumed, model_name="AutoInt")
    np.testing.assert_array_equal(recommend_tf_feat(shim_model, [u], 12, {"age": 3.5}, None, True, False,
                                                    inner_id=True), got)
    users = rng.choice(nu, size=9, replace=False).tolist()
    np.testing.assert_array_equal(recommend_tf_feat(shim_model, users, 10, None, None, True, False),
                                  model.recommend(users, 10, True))
    # default_recs: the OOV user, no consumed filter
    dr = model.default_recs(50)
    pre = oracle_scores(w, np.repeat(nu, N), np.arange(N))
    ref = orc.rank_recommendations("ranking", [nu], pre, 50, N, {}, False)
    assert orc.near_tie_mask(ref, dr[None], pre.reshape(1, N), 1e-5).all()
    # assign_oov rewrites the tables and invalidates the cached item-side block
    uid = torch.arange(nu + 1, device=model.device)
    before = model.score_all_items(uid).cpu().numpy()
    oov = sorted({int(spec["user_sparse_unique"][nu, j]) for j in range(spec["user_sparse_unique"].shape[1])}
                 | {int(spec["item_sparse_unique"][N, j]) for j in range(spec["item_sparse_unique"].shape[1])})
    model.assign_oov(oov)
    after = model.score_all_items(uid).cpu().numpy()
    np.testing.assert_array_equal(after, _grid_rows(model, np.arange(nu + 1)))
    assert np.abs(after[:, 0] - before[:, 0]).max() > 1e-6
    w2 = assign_oov_rows(w, nu, N, oov)
    ao.close(after.reshape(-1), ao.autoint_forward(w2, allu, alli, *tm.row_features(spec, allu, alli)))
