"""GPU parity of the FM / DeepFM inference engines against the numpy restatement of the
reference graphs (oracle/tf_models.py — parity unpinned, see its header): logits within 1e-5
relative (the tolerance BASELINE.json's north_star states), top-K ids equal to the oracle's
ranking of the oracle's own scores outside near-ties."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _case(seed, n_users=300, n_items=500, K=16, us=(7, 30), its=(11, 5, 40), ud=1, idn=2):
    from oracle import tf_models as tm

    rng = np.random.default_rng(seed)
    spec = tm.make_spec(rng, n_users, n_items, list(us), list(its), ud, idn)
    return rng, spec


def _close(got, ref, tol=1e-5):
    scale = np.maximum(np.abs(ref), np.abs(ref).mean())
    assert (np.abs(got - ref) <= tol * scale + 1e-6).all(), float(np.abs(got - ref).max())


@pytest.mark.parametrize("use_bn", [True, False])
@pytest.mark.parametrize("K", [16, 8, 64, 20])
def test_fm_logits_and_predict(use_bn, K):
    from librecommender_b200.feat_models import FM
    from oracle import tf_models as tm

    rng, spec = _case(K + int(use_bn), K=K)
    w = tm.make_fm_weights(rng, spec, K, use_bn)
    model = FM(spec, w)
    users = rng.integers(0, spec["n_users"] + 1, size=777)      # includes the OOV row
    items = rng.integers(0, spec["n_items"] + 1, size=777)
    sparse, dense = tm.row_features(spec, users, items)
    ref = tm.fm_forward(w, users, items, sparse, dense)
    ref64 = tm.fm_forward(w, users, items, sparse, dense, dtype=np.float64)
    got = model.logits(users, items).cpu().numpy()
    _close(got, ref64, 1e-5)
    _close(ref, ref64, 1e-5)
    # explicit feature rows (predict with a feed) give the same numbers
    got2 = model.logits(users, items, sparse_rows=sparse, dense_rows=dense).cpu().numpy()
    np.testing.assert_array_equal(got, got2)
    p = model.predict(users, items)
    np.testing.assert_allclose(p, 1 / (1 + np.exp(-ref64)), rtol=1e-5, atol=1e-6)


def test_fm_only_ids_no_features():
    from librecommender_b200.feat_models import FM
    from oracle import tf_models as tm

    rng = np.random.default_rng(0)
    spec = tm.make_spec(rng, 100, 80, [], [], 0, 0)          # DatasetPure: user / item ids only
    w = tm.make_fm_weights(rng, spec, 16, True)
    model = FM(spec, w)
    users, items = rng.integers(0, 100, 300), rng.integers(0, 80, 300)
    _close(model.logits(users, items).cpu().numpy(), tm.fm_forward(w, users, items, dtype=np.float64))


@pytest.mark.parametrize("use_bn", [True, False])
def test_deepfm_logits(use_bn):
    from librecommender_b200.feat_models import DeepFM
    from oracle import tf_models as tm

    rng, spec = _case(5 + int(use_bn), K=16)
    w = tm.make_deepfm_weights(rng, spec, 16, (128, 64, 32), use_bn)
    model = DeepFM(spec, w)
    users = rng.integers(0, spec["n_users"], size=1000)
    items = rng.integers(0, spec["n_items"], size=1000)
    sparse, dense = tm.row_features(spec, users, items)
    ref64 = tm.deepfm_forward(w, users, items, sparse, dense, dtype=np.float64)
    _close(model.logits(users, items).cpu().numpy(), ref64, 1e-5)


@pytest.mark.parametrize("cls_name", ["FM", "DeepFM"])
def test_recommend_all_items_matches_oracle(cls_name):
    from librecommender_b200 import feat_models as fmods
    from oracle import ranking as orc
    from oracle import tf_models as tm

    rng, spec = _case(11, n_users=120, n_items=700, K=16)
    N = spec["n_items"]
    if cls_name == "FM":
        w = tm.make_fm_weights(rng, spec, 16, True)
        fwd = tm.fm_forward
    else:
        w = tm.make_deepfm_weights(rng, spec, 16, (64, 32), True)
        fwd = tm.deepfm_forward
    consumed = {u: rng.choice(N, size=int(rng.integers(1, 40)), replace=False).tolist() for u in range(120)}
    model = getattr(fmods, cls_name)(spec, w, consumed)
    user_ids = rng.choice(120, size=37, replace=False)
    got = model.recommend(user_ids, 10, True)
    # oracle: the reference's own B*N-row feed (process_tf_feat), then rank_recommendations
    uu = np.repeat(user_ids, N)
    ii = np.tile(np.arange(N), len(user_ids))
    sparse, dense = tm.row_features(spec, uu, ii)
    preds = fwd(w, uu, ii, sparse, dense, dtype=np.float64).astype(np.float32)
    ref = orc.rank_recommendations("ranking", user_ids.tolist(), preds, 10, N, consumed, True)
    full = preds.reshape(len(user_ids), N)
    assert orc.near_tie_mask(ref, got, full, 1e-5).all()
    assert (got == ref).mean() > 0.98
    for r, u in enumerate(user_ids.tolist()):
        assert not set(got[r].tolist()) & set(consumed[u])


def _seq_case(seed, T=12):
    from librecommender_b200.feat_models import recent_sequences
    from oracle import tf_models as tm

    rng = np.random.default_rng(seed)
    spec = tm.make_spec(rng, 150, 400, [9], [6, 13, 21], 1, 1)
    consumed = {u: rng.choice(400, size=int(rng.integers(1, 30)), replace=False).tolist() for u in range(149)}
    seqs, lens = recent_sequences(consumed, 150, 400, T)       # user 149 has no history
    return rng, spec, consumed, seqs, lens


def test_recent_sequences_matches_reference_rule():
    from librecommender_b200.feat_models import recent_sequences

    consumed = {0: [5, 6, 7, 8, 9], 1: [3], 2: []}
    seqs, lens = recent_sequences(consumed, 3, 50, 3)
    np.testing.assert_array_equal(seqs, [[7, 8, 9], [3, 50, 50], [50, 50, 50], [50, 50, 50]])
    np.testing.assert_array_equal(lens, [3, 1, 0, 1])


@pytest.mark.parametrize("use_bn", [True, False])
def test_din_logits(use_bn):
    from librecommender_b200.feat_models import DIN
    from oracle import tf_models as tm

    rng, spec, consumed, seqs, lens = _seq_case(21)
    w = tm.make_seq_weights(rng, spec, 16, (64, 32), use_bn, din=True)
    model = DIN(spec, w, seqs, lens)
    users = rng.integers(0, 151, size=600)
    items = rng.integers(0, 400, size=600)
    sparse, dense = tm.row_features(spec, users, items)
    ref64 = tm.din_forward(w, spec, users, items, seqs[users], np.maximum(lens[users], 0), sparse, dense,
                           dtype=np.float64)
    ok = lens[users] > 0                                     # len 0 rows: reference divides 0/0 (never built)
    _close(model.logits(users, items).cpu().numpy()[ok], ref64[ok], 1e-5)


def test_din_use_tf_attention():
    """use_tf_attention=True (din.py:247-248): weight-free dot-product attention; predict rows and the
    all-items grid agree with the restatement of tf.keras.layers.Attention(use_scale=False)."""
    from librecommender_b200.feat_models import DIN
    from oracle import ranking as orc
    from oracle import tf_models as tm

    rng, spec, consumed, seqs, lens = _seq_case(23)
    w = tm.make_seq_weights(rng, spec, 16, (64, 32), True, din=True)
    w["use_tf_attention"] = True
    model = DIN(spec, w, seqs, lens, consumed)
    assert model.use_tf_attention
    users = rng.integers(0, 151, size=500)
    items = rng.integers(0, 400, size=500)
    sparse, dense = tm.row_features(spec, users, items)
    ref64 = tm.din_forward(w, spec, users, items, seqs[users], np.maximum(lens[users], 0), sparse, dense,
                           dtype=np.float64)
    ok = lens[users] > 0
    _close(model.logits(users, items).cpu().numpy()[ok], ref64[ok], 1e-5)
    us = np.array([u for u in range(0, 150, 13) if lens[u] > 0])
    N = spec["n_items"]
    uu, ii = np.repeat(us, N), np.tile(np.arange(N), len(us))
    sp, de = tm.row_features(spec, uu, ii)
    preds = tm.din_forward(w, spec, uu, ii, seqs[uu], lens[uu], sp, de, dtype=np.float64).astype(np.float32)
    got = model.recommend(us, 10, True)
    ref = orc.rank_recommendations("ranking", us.tolist(), preds, 10, N, consumed, True)
    assert orc.near_tie_mask(ref, got, preds.reshape(len(us), N), 1e-5).all()


@pytest.mark.parametrize("hidden,hoisted", [((64, 32), True), ((128, 64, 32), True), ((300, 64, 32), False)])
def test_youtube_ranking_logits_and_recommend(hidden, hoisted):
    """recommend goes through the hoisted all-items scorer when the MLP fits the pair kernel, else
    through the flat (user, item) grid — both against the oracle's B*N-row evaluation."""
    from librecommender_b200.feat_models import YouTubeRanking
    from oracle import ranking as orc
    from oracle import tf_models as tm

    rng, spec, consumed, seqs, lens = _seq_case(22)
    w = tm.make_seq_weights(rng, spec, 16, hidden, True, din=False)
    model = YouTubeRanking(spec, w, seqs, lens, consumed)
    assert model._hoistable() == hoisted
    users = rng.integers(0, 151, size=500)
    items = rng.integers(0, 400, size=500)
    sparse, dense = tm.row_features(spec, users, items)
    ref64 = tm.youtube_ranking_forward(w, users, items, seqs[users], lens[users], 400, sparse, dense,
                                       dtype=np.float64)
    _close(model.logits(users, items).cpu().numpy(), ref64, 1e-5)
    uid = np.arange(0, 40)
    got = model.recommend(uid, 7, True)
    uu, ii = np.repeat(uid, 400), np.tile(np.arange(400), len(uid))
    sp, de = tm.row_features(spec, uu, ii)
    preds = tm.youtube_ranking_forward(w, uu, ii, seqs[uu], lens[uu], 400, sp, de, dtype=np.float64).astype(np.float32)
    ref = orc.rank_recommendations("ranking", uid.tolist(), preds, 7, 400, consumed, True)
    assert orc.near_tie_mask(ref, got, preds.reshape(len(uid), 400), 1e-5).all()


def test_din_recommend_all_items():
    from librecommender_b200.feat_models import DIN
    from oracle import ranking as orc
    from oracle import tf_models as tm

    rng, spec, consumed, seqs, lens = _seq_case(23, T=20)
    w = tm.make_seq_weights(rng, spec, 16, (32, 16), True, din=True)
    model = DIN(spec, w, seqs, lens, consumed)
    uid = np.arange(3, 25)
    got = model.recommend(uid, 10, True)
    uu, ii = np.repeat(uid, 400), np.tile(np.arange(400), len(uid))
    sp, de = tm.row_features(spec, uu, ii)
    preds = tm.din_forward(w, spec, uu, ii, seqs[uu], lens[uu], sp, de, dtype=np.float64).astype(np.float32)
    ref = orc.rank_recommendations("ranking", uid.tolist(), preds, 10, 400, consumed, True)
    assert orc.near_tie_mask(ref, got, preds.reshape(len(uid), 400), 1e-5).all()
    assert (got == ref).mean() > 0.97


@pytest.mark.parametrize("hidden", [(32, 16), (128, 64, 32)])
def test_din_hoisted_scores_equal_flat_grid(hidden):
    """Per-user GEMM formulation of the attention vs the per-row kernel, incl. a user without history
    (len 0 -> zero attention output) and the OOV user row (len 1, pad key)."""
    import torch

    from librecommender_b200 import feat_models as fmods
    from librecommender_b200.feat_models import DIN

    rng, spec, consumed, seqs, lens = _seq_case(31, T=20)
    from oracle import tf_models as tm

    w = tm.make_seq_weights(rng, spec, 16, hidden, True, din=True)
    model = DIN(spec, w, seqs, lens, consumed)
    assert model._hoistable()
    uid = torch.tensor([0, 7, 149, 150, 33], device="cuda")          # 149: no history, 150: OOV row
    hoisted = model.score_all_items(uid).cpu().numpy()
    flat = fmods._FeatModelBase.score_all_items(model, uid).cpu().numpy()
    scale = np.maximum(np.abs(flat), np.abs(flat).mean())
    assert (np.abs(hoisted - flat) <= 1e-5 * scale + 1e-6).all(), float(np.abs(hoisted - flat).max())


@pytest.mark.parametrize("norm", [True, False])
def test_two_tower_embeddings_and_retrieval(norm):
    from librecommender_b200.engine import EmbedScorer
    from librecommender_b200.feat_models import TwoTower
    from oracle import ranking as orc
    from oracle import tf_models as tm

    rng = np.random.default_rng(31)
    spec = tm.make_spec(rng, 200, 300, [8, 17], [5, 9], 1, 2)
    w = tm.make_two_tower_weights(rng, spec, 16, (64, 32), True)
    tt = TwoTower(spec, w, norm_embed=norm)
    U, I = tt.set_embeddings()
    uids, iids = np.arange(200), np.arange(300)
    us = spec["user_sparse_unique"][uids]
    ud = spec["user_dense_unique"][uids]
    is_ = spec["item_sparse_unique"][iids]
    idn = spec["item_dense_unique"][iids]
    ru = tm.tower_forward(w, uids, us, ud, "user", norm, dtype=np.float64)
    ri = tm.tower_forward(w, iids, is_, idn, "item", norm, dtype=np.float64)
    _close(U[:200].cpu().numpy(), ru, 2e-5)
    _close(I[:300].cpu().numpy(), ri, 2e-5)
    np.testing.assert_allclose(U[200].cpu().numpy(), ru.mean(axis=0), rtol=1e-4, atol=1e-6)   # OOV row
    # the tower outputs feed the embed scorer directly (no host round trip)
    consumed = {u: rng.choice(300, size=5, replace=False).tolist() for u in range(200)}
    sc = EmbedScorer(U, I, 300, consumed, n_users=200)
    got = sc.recommend(np.arange(50), 10, True)
    Uh, Ih = U.cpu().numpy(), I.cpu().numpy()
    ref = orc.recommend_from_embedding("ranking", list(range(50)), 10, Uh, Ih, 300, consumed, True)
    assert orc.near_tie_mask(ref, got, orc.embed_scores(Uh, Ih, list(range(50)), 300), 1e-6).all()


def test_recommend_tf_feat_shim():
    """libreco/recommendation/recommend.py:81-105 seam: same arguments, engine underneath."""
    import types

    from librecommender_b200 import feat_models as fmods
    from librecommender_b200.recommendation import recommend_tf_feat
    from oracle import tf_models as tm

    rng, spec = _case(21, n_users=90, n_items=400, K=16)
    N = spec["n_items"]
    w = tm.make_fm_weights(rng, spec, 16, True)
    consumed = {u: rng.choice(N, size=int(rng.integers(1, 30)), replace=False).tolist() for u in range(90)}
    engine = fmods.FM(spec, w, consumed)
    model = types.SimpleNamespace(n_items=N, task="ranking", user_consumed=consumed, model_name="FM",
                                  b200_engine=engine)
    users = rng.choice(90, size=20, replace=False).tolist()
    ids = recommend_tf_feat(model, users, 10, None, None, True, False)
    np.testing.assert_array_equal(ids, engine.recommend(users, 10, True))
    assert ids.shape == (20, 10) and ids.dtype == np.int64
    rnd = recommend_tf_feat(model, users, 10, None, None, True, True)          # random_rec branch
    assert rnd.shape == (20, 10) and (rnd >= 0).all() and (rnd < N).all()
    for r, u in enumerate(users):
        assert not set(ids[r].tolist()) & set(consumed[u])
        assert not set(rnd[r].tolist()) & set(consumed[u])
        assert len(set(rnd[r].tolist())) == 10


@pytest.mark.parametrize("T", [20, 50])
def test_din_fused_attention_epilogue_equals_unfused_and_flat(T):
    """Catalogue large enough for the tensor-core path (N >= 4096): the fused GEMM epilogue
    (b200_linear_tf32x3_sigmoid_dot + b200_din_attention_from_logits) against the two-kernel hoisted form
    ([N, 16 len] pre-activations + b200_din_attention_hoisted) and the per-row kernel on the flat grid."""
    import torch

    from librecommender_b200 import feat_models as fmods
    from librecommender_b200.feat_models import DIN, recent_sequences
    from oracle import tf_models as tm

    rng = np.random.default_rng(41 + T)
    n_users, n_items = 60, 5003
    spec = tm.make_spec(rng, n_users, n_items, [9], [6, 13, 21], 1, 0)
    consumed = {u: rng.choice(n_items, size=int(rng.integers(1, 70)), replace=False).tolist() for u in range(n_users - 1)}
    seqs, lens = recent_sequences(consumed, n_users, n_items, T)       # the last user has no history
    w = tm.make_seq_weights(rng, spec, 16, (128, 64, 32), True, din=True)
    model = DIN(spec, w, seqs, lens, consumed)
    assert model._hoistable() and model.Kp == 64
    uid = torch.tensor([0, 7, n_users - 1, n_users, 33], device="cuda")
    try:
        fmods.DIN_FUSED_ATTENTION = True
        fused = model.score_all_items(uid).cpu().numpy()
        fmods.DIN_FUSED_ATTENTION = False
        unfused = model.score_all_items(uid).cpu().numpy()
    finally:
        fmods.DIN_FUSED_ATTENTION = False
    flat = fmods._FeatModelBase.score_all_items(model, uid).cpu().numpy()
    scale = np.maximum(np.abs(flat), np.abs(flat).mean())
    assert (np.abs(unfused - flat) <= 1e-5 * scale + 1e-6).all(), float(np.abs(unfused - flat).max())
    assert (np.abs(fused - flat) <= 1e-5 * scale + 1e-6).all(), float(np.abs(fused - flat).max())


def test_din_attention_kernel_versions_agree():
    """b200_din_attention: the lane-owns-position kernel (default) against the first version on explicit pairs and
    on the all-items grid, incl. the user without history and T = 50."""
    import torch

    from librecommender_b200 import _lib
    from librecommender_b200.feat_models import DIN, recent_sequences
    from oracle import tf_models as tm

    rng = np.random.default_rng(77)
    n_users, n_items, T = 80, 700, 50
    spec = tm.make_spec(rng, n_users, n_items, [9], [6, 13, 21], 1, 0)
    consumed = {u: rng.choice(n_items, size=int(rng.integers(1, 90)), replace=False).tolist() for u in range(n_users - 1)}
    seqs, lens = recent_sequences(consumed, n_users, n_items, T)
    w = tm.make_seq_weights(rng, spec, 16, (64, 32), True, din=True)
    model = DIN(spec, w, seqs, lens, consumed)
    users, items = rng.integers(0, n_users + 1, 3000), rng.integers(0, n_items, 3000)
    out = {}
    try:
        for v in (1, 0):
            _lib.check(_lib.lib.b200_din_attention_tune(v))
            out[v] = model.logits(users, items).cpu().numpy()
    finally:
        _lib.check(_lib.lib.b200_din_attention_tune(1))
    sparse, dense = tm.row_features(spec, users, items)
    ref = tm.din_forward(w, spec, users, items, seqs[users], lens[users], sparse, dense, dtype=np.float64)
    ok = lens[users] > 0                                   # length 0: documented divergence (zeros vs uniform softmax)
    scale = max(1.0, np.abs(ref).max())
    assert np.abs(out[1] - out[0]).max() <= 1e-5 * scale
    assert np.abs(out[1][ok] - ref[ok]).max() <= 1e-4 * scale


def test_wide_deep_runs_on_the_deepfm_engine():
    """SURVEY 8f-4 adjacent model: WideDeep's variables mapped onto the DeepFM engine (feat_models.wide_deep_weights):
    logits and the hoisted all-items recommend against the numpy restatement of wide_deep.py."""
    from librecommender_b200.feat_models import DeepFM, wide_deep_weights
    from oracle import ranking as orc
    from oracle import tf_models as tm

    rng = np.random.default_rng(17)
    spec = tm.make_spec(rng, 120, 260, [7, 30], [11, 5, 40], 1, 2)
    base = tm.make_deepfm_weights(rng, spec, 16, (64, 32), True)          # tables / MLP of the right shapes
    H = 32
    wd = dict(user_wide=base["user_linear"], item_wide=base["item_linear"], sparse_wide=base["sparse_linear"],
              dense_wide=base["dense_linear"], wide_kernel=base["lin_kernel"], wide_bias=np.float32(0.03),
              user_deep=base["user_embeds"], item_deep=base["item_embeds"], sparse_deep=base["sparse_embeds"],
              dense_deep=base["dense_embeds"], mlp=base["mlp"],
              deep_kernel=rng.standard_normal(H).astype(np.float32) * 0.3, deep_bias=np.float32(-0.02))
    w = wide_deep_weights(**wd)
    consumed = {u: rng.choice(260, size=6, replace=False).tolist() for u in range(120)}
    model = DeepFM(spec, w, consumed)
    users, items = rng.integers(0, 120, 700), rng.integers(0, 260, 700)
    sparse, dense = tm.row_features(spec, users, items)
    ref = tm.wide_deep_forward(wd, users, items, sparse, dense, dtype=np.float64)
    got = model.logits(users, items).cpu().numpy()
    _close(got, ref, 3e-5)
    uid = np.arange(0, 120, 5)
    got_ids = model.recommend(uid, 10, True)
    all_u, all_i = np.repeat(uid, 260), np.tile(np.arange(260), len(uid))
    sp, dn = tm.row_features(spec, all_u, all_i)
    full = tm.wide_deep_forward(wd, all_u, all_i, sp, dn, dtype=np.float64).reshape(len(uid), 260)
    ref_ids = orc.rank_recommendations("ranking", uid.tolist(), full.astype(np.float32).copy(), 10, 260, consumed, True)
    assert orc.near_tie_mask(ref_ids, got_ids, full.astype(np.float32), 1e-5).all()


@pytest.mark.parametrize("norm,n_rows", [(False, 300), (True, 5000)])
def test_youtube_retrieval_user_vectors_and_retrieval(norm, n_rows):
    """SURVEY 8f-4 adjacent model: YouTubeRetrieval's user tower (sqrtn-pooled history + user features, K1 without an
    id field, both the small-batch and the pipelined large-batch kernels) against the numpy restatement, then all-items
    retrieval through the embed scorer with the reference's pseudo-bias column."""
    from librecommender_b200 import _lib
    from librecommender_b200.engine import EmbedScorer
    from librecommender_b200.feat_models import YouTubeRetrieval, recent_sequences
    from librecommender_b200.synthetic import _glorot, make_embeddings, make_mlp
    from oracle import ranking as orc
    from oracle import tf_models as tm

    rng = np.random.default_rng(23 + n_rows)
    n_users, n_items, K, H, T = n_rows, 900, 16, 32, 10
    spec = tm.make_spec(rng, n_users, n_items, [8, 17], [5], 1, 0)
    emb = make_embeddings(rng, spec, K, linear=False)
    w = dict(seq_embeds=_glorot(rng, (n_items, K)), sparse_embeds=emb["sparse_embeds"], dense_embeds=emb["dense_embeds"],
             mlp=make_mlp(rng, (1 + 2 + 1) * K, (64, H), True), item_embeds=_glorot(rng, (n_items, H)),
             item_biases=(rng.standard_normal(n_items) * 0.1).astype(np.float32))
    consumed = {u: rng.choice(n_items, size=int(rng.integers(1, 25)), replace=False).tolist() for u in range(n_users - 1)}
    seqs, lens = recent_sequences(consumed, n_users, n_items, T)          # the last user has no history
    model = YouTubeRetrieval(spec, w, seqs, lens, norm_embed=norm)
    n0 = _lib.launch_count()
    for bad in ([n_users + 1], [-1], [0, n_users + 7]):
        with pytest.raises(ValueError, match="user ids"):
            model.user_vectors(bad)
    assert _lib.launch_count() == n0
    ids = np.arange(n_users)
    got = model.user_vectors(ids).cpu().numpy()
    ref = tm.youtube_retrieval_user_vectors(w, spec, ids, seqs, lens, norm, dtype=np.float64)
    _close(got, ref, 3e-5)
    U, I = model.set_embeddings()
    assert U.shape == (n_users + 1, H + 1) and I.shape == (n_items + 1, H + 1)
    assert float(U[:n_users, H].min()) == 1.0 and float(U[:n_users, H].max()) == 1.0
    sc = EmbedScorer(U, I, n_items, consumed, n_users=n_users)
    users = rng.integers(0, n_users, 64)
    got_ids = sc.recommend(users, 10, True)
    Ih = w["item_embeds"].astype(np.float64)
    if norm:
        Ih = Ih / np.linalg.norm(Ih, axis=1, keepdims=True)
    full = ref[users] @ Ih.T + w["item_biases"].astype(np.float64)[None, :]
    ref_ids = orc.rank_recommendations("ranking", users.tolist(), full.astype(np.float32).copy(), 10, n_items, consumed, True)
    assert orc.near_tie_mask(ref_ids, got_ids, full.astype(np.float32), 2e-5).all()
