"""The serving path the dynamic-embedding sequence models share (RNN4Rec, Caser, WaveNet): bit-identity of
``set_embeddings`` / ``user_vectors`` / ``recommend_dynamic``, the serving tables, all-items retrieval against the
float64 oracle, ``recommend_dynamic`` with a supplied sequence, and the ``ValueError`` checks of ``user_vectors``."""
from types import SimpleNamespace

import numpy as np
import pytest

import _conv_encoder_oracle as co
import _rnn4rec_oracle as ro
from _dyn_embed_data import GPU_ATOL, K, N_ITEMS, close, conv_model, conv_raw, data, rnn4rec_model

pytestmark = pytest.mark.gpu

MODELS = ["RNN4Rec", "Caser", "WaveNet"]


@pytest.fixture(scope="module", params=MODELS)
def served(request):
    """One model of 3001 users at T = 10; ``vectors(raw, ids, seqs, lens)`` is its float64 oracle and ``d`` the
    width of its user vectors."""
    from librecommender_b200.synthetic import make_rnn4rec_weights

    name = request.param
    rng = np.random.default_rng(2024)
    n_users, T = 3001, 10
    if name == "RNN4Rec":
        raw = make_rnn4rec_weights(rng, N_ITEMS, K, (32, 24), "gru", True, "keras")
        consumed, seqs, lens = data(rng, n_users, T)
        m = rnn4rec_model(raw, n_users, seqs, lens, False)
        vectors, d = (lambda r, ids, s, ln: ro.user_vectors(r, s, ln)), K
    else:
        raw = conv_raw(rng, name, n_users, T, (2, 4) if name == "Caser" else (16, 1, 4))
        consumed, seqs, lens = data(rng, n_users, T)
        m = conv_model(raw, n_users, seqs, lens, False)
        vectors, d = (lambda r, ids, s, ln: co.user_vectors(r, ids, s)), 2 * K
    return SimpleNamespace(name=name, raw=raw, consumed=consumed, seqs=seqs, lens=lens, model=m, n_users=n_users,
                           T=T, vectors=vectors, d=d)


def test_bit_identity(served):
    import torch

    from librecommender_b200 import _lib

    m = served.model
    U, I = m.set_embeddings()
    U7, I7 = m.set_embeddings(chunk=7)
    assert U.shape == U7.shape and bool((U == U7).all()) and bool((I == I7).all())
    U2, _ = m.set_embeddings()
    assert bool((U == U2).all())
    rng = np.random.default_rng(1)
    ids = np.concatenate([rng.permutation(served.n_users)[:999], [5, 5, 0, 0, 17]])
    got = m.user_vectors(ids)
    assert bool((got == U[ids][:, :served.d]).all())
    # the same rows supplied as seqs / lens give the same bits
    assert bool((m.user_vectors(ids, served.seqs[ids], served.lens[ids]) == got).all())
    if served.name != "RNN4Rec":
        # the length is never read: other lens give the same bits
        assert bool((m.user_vectors(ids, served.seqs[ids], np.zeros(len(ids))) == got).all())
    # recommend_dynamic with the user's own cached sequence scores exactly like its U row
    info = SimpleNamespace(item2id=None, user_consumed=served.consumed)
    u = 4
    seq = served.seqs[u, :served.lens[u]].tolist()
    ids_d, sc_d = m.recommend_dynamic(u, 20, info, seq=seq, inner_id=True, filter_consumed=False, return_scores=True)
    ids_c, sc_c = m.recommend_dynamic(u, 20, info, inner_id=True, filter_consumed=False, return_scores=True)
    np.testing.assert_array_equal(ids_d, ids_c)
    np.testing.assert_array_equal(sc_d, sc_c)
    exact = torch.empty((1, N_ITEMS), dtype=torch.float32, device=U.device)
    zero = torch.zeros(1, dtype=torch.int64, device=U.device)
    _lib.check(_lib.lib.b200_score_rows_f32(_lib.ptr(U[u:u + 1].contiguous()), U.shape[1], _lib.ptr(zero), 1,
                                            _lib.ptr(I), I.stride(0), N_ITEMS, U.shape[1], _lib.ptr(exact), N_ITEMS,
                                            _lib.current_stream()))
    np.testing.assert_array_equal(sc_d[0], exact.cpu().numpy()[0][ids_d[0]])
    full = (U[u:u + 1] @ I[:N_ITEMS].T).cpu().numpy()
    assert np.abs(sc_d[0] - full[0][ids_d[0]]).max() < 1e-4


@pytest.mark.parametrize("filter_consumed", [True, False])
def test_set_embeddings_layout_and_retrieval(served, filter_consumed):
    from librecommender_b200.engine import EmbedScorer
    from oracle import ranking as orc

    m, n_users, d = served.model, served.n_users, served.d
    U, I = m.set_embeddings()
    assert U.shape == (n_users + 1, d + 1) and I.shape == (N_ITEMS + 1, d + 1)
    assert float(U[:n_users, d].min()) == 1.0 and float(U[:n_users, d].max()) == 1.0
    raw = served.raw
    if served.name != "RNN4Rec":
        # the OOV user row of the device table is the mean of the known rows
        ue = m.user_embeds.double().cpu().numpy()
        np.testing.assert_allclose(ue[n_users], ue[:n_users].mean(0), atol=1e-6)
        raw = co.assign_user_oov(raw)
    ref_u = served.vectors(raw, np.arange(n_users), served.seqs[:n_users], served.lens[:n_users])
    Uo, Io = ro.serving_tables(raw, ref_u)
    close(U.cpu().numpy(), Uo, GPU_ATOL)
    close(I.cpu().numpy(), Io, 1e-6)
    np.testing.assert_allclose(U[n_users].cpu().numpy(), U[:n_users].double().mean(0).cpu().numpy(), atol=1e-6)
    np.testing.assert_allclose(I[N_ITEMS].cpu().numpy(), I[:N_ITEMS].double().mean(0).cpu().numpy(), atol=1e-6)
    sc = EmbedScorer(U, I, N_ITEMS, served.consumed, n_users=n_users)
    users = np.random.default_rng(3).integers(0, n_users, 64)
    got = sc.recommend(users, 10, filter_consumed)
    ref_ids, full = ro.recommend(raw, ref_u, users, 10, served.consumed, filter_consumed)
    assert orc.near_tie_mask(ref_ids, got, full.astype(np.float32), 2e-5).all()
    if filter_consumed:
        for r, u in enumerate(users):
            assert not set(got[r]) & set(served.consumed.get(int(u), []))


def test_recommend_dynamic(served):
    import torch

    m, T, n_users = served.model, served.T, served.n_users
    m.set_embeddings()
    before = {k: getattr(m, k).clone() for k in ("seqs", "lens", "user_embeds") if hasattr(m, k)}
    item2id = {f"i{j}": j for j in range(N_ITEMS)}
    info = SimpleNamespace(item2id=item2id, user_consumed=served.consumed)
    rng = np.random.default_rng(8)
    long = [f"i{j}" for j in rng.integers(0, N_ITEMS, 3 * T)]
    got = m.recommend_dynamic(3, 15, info, seq=long, return_scores=True)
    tail = m.recommend_dynamic(3, 15, info, seq=long[-T:], return_scores=True)
    np.testing.assert_array_equal(got[0], tail[0])          # longer than T: only the last T items count
    np.testing.assert_array_equal(got[1], tail[1])
    row, ln = np.array([[item2id[i] for i in long[-T:]]], np.int32), np.array([T])
    ref_raw = served.raw if served.name == "RNN4Rec" else co.assign_user_oov(served.raw)
    close(m.user_vectors([3], row, ln).cpu().numpy(), served.vectors(ref_raw, [3], row, ln), GPU_ATOL)
    assert not set(got[0][0]) & set(served.consumed.get(3, []))
    # unknown original ids become the pad id n_items
    unk = m.recommend_dynamic(3, 15, info, seq=["nope", "i5", "zzz"], return_scores=True)
    pad = m.recommend_dynamic(3, 15, info, seq=[N_ITEMS, 5, N_ITEMS], inner_id=True, return_scores=True)
    np.testing.assert_array_equal(unk[0], pad[0])
    np.testing.assert_array_equal(unk[1], pad[1])
    # the unknown user (id n_users) gets no consumed filter; user_feats is ignored
    cold = m.recommend_dynamic(n_users, 15, info, user_feats={"x": 1}, seq=long, return_scores=True)
    warm = m.recommend_dynamic(3, 15, info, seq=long, filter_consumed=False, return_scores=True)
    if served.name == "RNN4Rec":
        # no user table: the sequence alone makes the vector
        np.testing.assert_array_equal(cold[0], warm[0])
        np.testing.assert_array_equal(cold[1], warm[1])
    else:
        # the mean user row goes beside the sequence: not the warm user's vector
        cold_v = m.user_vectors([n_users], row).cpu().numpy()
        warm_v = m.user_vectors([3], row).cpu().numpy()
        ue = m.user_embeds.cpu().numpy()
        np.testing.assert_array_equal(cold_v[0, :K], ue[n_users])
        np.testing.assert_array_equal(cold_v[0, K:], warm_v[0, K:])
        assert np.abs(cold_v[0, :K] - warm_v[0, :K]).max() > 1e-3
        close(cold_v, co.user_vectors(ref_raw, [n_users], row), GPU_ATOL)
        assert not np.array_equal(cold[1], warm[1])
    for k, t in before.items():
        assert bool(torch.equal(getattr(m, k), t)), k
    with pytest.raises(ValueError):
        m.recommend_dynamic(3, N_ITEMS + 1, info)


def test_value_errors_launch_nothing():
    """Out-of-envelope constructors and malformed ``user_vectors`` / ``recommend_dynamic`` calls raise before any
    launch, for every model: the kernels cannot tell how many rows a table has."""
    from librecommender_b200 import _lib
    from librecommender_b200.synthetic import make_rnn4rec_weights

    rng = np.random.default_rng(0)
    n0 = _lib.launch_count()
    seqs, lens = np.full((5, 10), 50, np.int32), np.ones(5, np.int32)
    with pytest.raises(ValueError, match="max_seq_len"):
        conv_model(conv_raw(rng, "Caser", 4, 65, (2, 4), n_items=50), 4, np.full((5, 65), 50, np.int32), lens, False)
    with pytest.raises(ValueError, match="nv_filters"):
        conv_model(conv_raw(rng, "Caser", 4, 10, (2, 33), n_items=50), 4, seqs, lens, False)
    with pytest.raises(ValueError, match="embed_size"):
        conv_model(conv_raw(rng, "WaveNet", 4, 10, (8, 1, 2), k=129, n_items=50), 4, seqs, lens, False)
    with pytest.raises(ValueError, match="n_filters"):
        conv_model(conv_raw(rng, "WaveNet", 4, 10, (129, 1, 2), n_items=50), 4, seqs, lens, False)
    with pytest.raises(ValueError, match="dilations"):
        conv_model(conv_raw(rng, "WaveNet", 4, 10, (8, 17, 1), n_items=50), 4, seqs, lens, False)
    # RNN4Rec: 4 users, but sequence rows for users 0..2 only
    rnn = rnn4rec_model(make_rnn4rec_weights(rng, 50, K, (16,), "gru", False, "keras"), 4, seqs[:3], lens[:3], False)
    with pytest.raises(ValueError, match="cached sequence"):
        rnn.user_vectors([3])
    with pytest.raises(ValueError, match="cached sequence"):
        rnn.recommend_dynamic(4, 5, SimpleNamespace(item2id=None, user_consumed=None))
    with pytest.raises(ValueError, match="lens"):
        rnn.user_vectors([1, 2], seqs[:2], lens[:1])
    with pytest.raises(ValueError, match="both"):
        rnn.user_vectors([1, 2], seqs[:2])
    models = [rnn, conv_model(conv_raw(rng, "Caser", 4, 10, (2, 4), n_items=50), 4, seqs, lens, False),
              conv_model(conv_raw(rng, "WaveNet", 4, 10, (8, 1, 2), n_items=50), 4, seqs, lens, False)]
    for m in models:
        with pytest.raises(ValueError, match="user ids"):
            m.user_vectors([5])
        with pytest.raises(ValueError, match="user ids"):
            m.user_vectors([-1])
        with pytest.raises(ValueError, match="user ids"):
            m.user_vectors([0, 5], seqs[:2], lens[:2])
        with pytest.raises(ValueError, match="shape"):
            m.user_vectors([1, 2], seqs[:1], lens[:1])
        with pytest.raises(ValueError, match="n_rec"):
            m.recommend_dynamic(1, 51, SimpleNamespace(item2id=None, user_consumed=None))
        assert tuple(m.user_vectors([]).shape) == (0, m.item_embeds.shape[1])
    assert _lib.launch_count() == n0
