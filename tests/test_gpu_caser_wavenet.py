"""Caser / WaveNet on the GPU: ``b200_caser_encode`` / ``b200_wavenet_encode`` + the Dense head beside the user
table against the float64 oracle, bit-identity of a user's vector across calls and batches, the serving tables with
the OOV user row, all-items retrieval and ``recommend_dynamic``."""
from types import SimpleNamespace

import numpy as np
import pytest

from _conv_encoder_oracle import assign_user_oov, recommend as oracle_recommend
from _conv_encoder_oracle import serving_tables, user_vectors as oracle_vectors

pytestmark = pytest.mark.gpu

N_ITEMS, K = 700, 16
GPU_ATOL = 2e-5       # the float32 restatement of the same shapes stays under a quarter of this (test_caser_wavenet_cpu)


def _close(got, ref, atol):
    err = np.abs(np.asarray(got, np.float64) - ref).max() / max(1.0, np.abs(ref).max())
    assert err < atol, err


def _data(rng, n_users, T, n_items=N_ITEMS):
    """Consumed lists with an empty history (all pad), one item and long ones, as recent_sequences."""
    from librecommender_b200.feat_models import recent_sequences

    sizes = rng.integers(0, 2 * T, size=n_users)
    sizes[:3] = [0, 1, 3 * T]
    consumed = {u: rng.choice(n_items, size=int(s), replace=False).tolist() for u, s in enumerate(sizes) if s}
    seqs, lens = recent_sequences(consumed, n_users, n_items, T)
    return consumed, seqs, lens


def _raw(rng, model, n_users, T, widths, dilated=True, k=K, n_items=N_ITEMS):
    from librecommender_b200.synthetic import make_caser_weights, make_wavenet_weights

    if model == "Caser":
        return make_caser_weights(rng, n_users, n_items, k, T, *widths)
    return make_wavenet_weights(rng, n_users, n_items, k, *widths, dilated=dilated)


def _model(raw, n_users, seqs, lens, norm):
    from librecommender_b200.feat_models import Caser, WaveNet

    cls = Caser if "vertical" in raw else WaveNet
    return cls({"n_users": n_users, "n_items": raw["item_embeds"].shape[0]}, raw, seqs, lens, norm_embed=norm)


CASES = ([("Caser", w, True) for w in ((2, 4), (8, 1), (3, 16))] +
         [("WaveNet", w, dil) for w in ((16, 1, 4), (32, 2, 3), (5, 1, 1)) for dil in (True, False)])


@pytest.mark.parametrize("T", [10, 50])
@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("model,widths,dilated", CASES)
def test_user_vectors_match_oracle(model, widths, dilated, norm, T):
    rng = np.random.default_rng(CASES.index((model, widths, dilated)) * 4 + T + norm)
    n_users = 1003                                    # not a multiple of any tile
    raw = _raw(rng, model, n_users, T, widths, dilated)
    _, seqs, lens = _data(rng, n_users, T)
    m = _model(raw, n_users, seqs, lens, norm)
    ids = np.arange(n_users + 1)                      # the OOV user with the all-pad OOV sequence row included
    got = m.user_vectors(ids).cpu().numpy()
    _close(got, oracle_vectors(raw, ids, seqs, norm), GPU_ATOL)
    one = m.user_vectors([2]).cpu().numpy()           # n = 1: the same bits as in the big batch
    np.testing.assert_array_equal(one[0], got[2])


@pytest.mark.parametrize("model,widths", [("Caser", (32, 32)), ("WaveNet", (128, 4, 4))])
def test_envelope_maximum(model, widths):
    """T = 64, K = 128 and the widest filters (WaveNet: 16 causal layers): the longest chains the kernels run."""
    rng = np.random.default_rng(77)
    n_users, T = 37, 64
    raw = _raw(rng, model, n_users, T, widths, k=128, n_items=300)
    _, seqs, lens = _data(rng, n_users, T, 300)
    m = _model(raw, n_users, seqs, lens, False)
    ids = np.arange(n_users + 1)
    _close(m.user_vectors(ids).cpu().numpy(), oracle_vectors(raw, ids, seqs), 1e-4)


@pytest.fixture(scope="module", params=["Caser", "WaveNet"])
def served(request):
    rng = np.random.default_rng(2024)
    n_users, T = 3001, 10
    raw = _raw(rng, request.param, n_users, T, (2, 4) if request.param == "Caser" else (16, 1, 4))
    consumed, seqs, lens = _data(rng, n_users, T)
    m = _model(raw, n_users, seqs, lens, False)
    return SimpleNamespace(raw=raw, consumed=consumed, seqs=seqs, lens=lens, model=m, n_users=n_users, T=T)


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
    d = U.shape[1] - 1
    assert bool((got == U[ids][:, :d]).all())
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


@pytest.mark.parametrize("filter_consumed", [True, False])
def test_set_embeddings_layout_and_retrieval(served, filter_consumed):
    from librecommender_b200.engine import EmbedScorer
    from oracle import ranking as orc

    m, n_users = served.model, served.n_users
    U, I = m.set_embeddings()
    assert U.shape == (n_users + 1, 2 * K + 1) and I.shape == (N_ITEMS + 1, 2 * K + 1)
    assert float(U[:n_users, 2 * K].min()) == 1.0 and float(U[:n_users, 2 * K].max()) == 1.0
    # the OOV user row of the device table is the mean of the known rows
    ue = m.user_embeds.double().cpu().numpy()
    np.testing.assert_allclose(ue[n_users], ue[:n_users].mean(0), atol=1e-6)
    raw = assign_user_oov(served.raw)
    ref_u = oracle_vectors(raw, np.arange(n_users), served.seqs[:n_users])
    Uo, Io = serving_tables(raw, ref_u)
    _close(U.cpu().numpy(), Uo, GPU_ATOL)
    _close(I.cpu().numpy(), Io, 1e-6)
    np.testing.assert_allclose(U[n_users].cpu().numpy(), U[:n_users].double().mean(0).cpu().numpy(), atol=1e-6)
    np.testing.assert_allclose(I[N_ITEMS].cpu().numpy(), I[:N_ITEMS].double().mean(0).cpu().numpy(), atol=1e-6)
    sc = EmbedScorer(U, I, N_ITEMS, served.consumed, n_users=n_users)
    users = np.random.default_rng(3).integers(0, n_users, 64)
    got = sc.recommend(users, 10, filter_consumed)
    ref_ids, full = oracle_recommend(raw, ref_u, users, 10, served.consumed, filter_consumed)
    assert orc.near_tie_mask(ref_ids, got, full.astype(np.float32), 2e-5).all()
    if filter_consumed:
        for r, u in enumerate(users):
            assert not set(got[r]) & set(served.consumed.get(int(u), []))


def test_recommend_dynamic(served):
    import torch

    m, T, n_users = served.model, served.T, served.n_users
    m.set_embeddings()
    seqs_before, lens_before, ue_before = m.seqs.clone(), m.lens.clone(), m.user_embeds.clone()
    item2id = {f"i{j}": j for j in range(N_ITEMS)}
    info = SimpleNamespace(item2id=item2id, user_consumed=served.consumed)
    rng = np.random.default_rng(8)
    long = [f"i{j}" for j in rng.integers(0, N_ITEMS, 3 * T)]
    got = m.recommend_dynamic(3, 15, info, seq=long, return_scores=True)
    tail = m.recommend_dynamic(3, 15, info, seq=long[-T:], return_scores=True)
    np.testing.assert_array_equal(got[0], tail[0])          # longer than T: only the last T items count
    np.testing.assert_array_equal(got[1], tail[1])
    row = np.array([[item2id[i] for i in long[-T:]]], np.int32)
    _close(m.user_vectors([3], row).cpu().numpy(), oracle_vectors(served.raw, [3], row), GPU_ATOL)
    assert not set(got[0][0]) & set(served.consumed.get(3, []))
    # unknown original ids become the pad id n_items
    unk = m.recommend_dynamic(3, 15, info, seq=["nope", "i5", "zzz"], return_scores=True)
    pad = m.recommend_dynamic(3, 15, info, seq=[N_ITEMS, 5, N_ITEMS], inner_id=True, return_scores=True)
    np.testing.assert_array_equal(unk[0], pad[0])
    np.testing.assert_array_equal(unk[1], pad[1])
    # the unknown user (id n_users) uses the mean user row beside the sequence: not the warm user's vector
    cold_v = m.user_vectors([n_users], row).cpu().numpy()
    warm_v = m.user_vectors([3], row).cpu().numpy()
    ue = m.user_embeds.cpu().numpy()
    np.testing.assert_array_equal(cold_v[0, :K], ue[n_users])
    np.testing.assert_array_equal(cold_v[0, K:], warm_v[0, K:])
    assert np.abs(cold_v[0, :K] - warm_v[0, :K]).max() > 1e-3
    _close(cold_v, oracle_vectors(assign_user_oov(served.raw), [n_users], row), GPU_ATOL)
    cold = m.recommend_dynamic(n_users, 15, info, user_feats={"x": 1}, seq=long, return_scores=True)
    warm = m.recommend_dynamic(3, 15, info, seq=long, filter_consumed=False, return_scores=True)
    assert not np.array_equal(cold[1], warm[1])
    assert bool(torch.equal(m.seqs, seqs_before)) and bool(torch.equal(m.lens, lens_before))
    assert bool(torch.equal(m.user_embeds, ue_before))
    with pytest.raises(ValueError):
        m.recommend_dynamic(3, N_ITEMS + 1, info)


def test_value_errors_launch_nothing():
    from librecommender_b200 import _lib

    rng = np.random.default_rng(0)
    n0 = _lib.launch_count()
    seqs, lens = np.full((5, 10), 50, np.int32), np.ones(5, np.int32)
    with pytest.raises(ValueError, match="max_seq_len"):
        _model(_raw(rng, "Caser", 4, 65, (2, 4), n_items=50), 4, np.full((5, 65), 50, np.int32), lens, False)
    with pytest.raises(ValueError, match="nv_filters"):
        _model(_raw(rng, "Caser", 4, 10, (2, 33), n_items=50), 4, seqs, lens, False)
    with pytest.raises(ValueError, match="embed_size"):
        _model(_raw(rng, "WaveNet", 4, 10, (8, 1, 2), k=129, n_items=50), 4, seqs, lens, False)
    with pytest.raises(ValueError, match="n_filters"):
        _model(_raw(rng, "WaveNet", 4, 10, (129, 1, 2), n_items=50), 4, seqs, lens, False)
    with pytest.raises(ValueError, match="dilations"):
        _model(_raw(rng, "WaveNet", 4, 10, (8, 17, 1), n_items=50), 4, seqs, lens, False)
    m = _model(_raw(rng, "WaveNet", 4, 10, (8, 1, 2), n_items=50), 4, seqs, lens, False)
    with pytest.raises(ValueError, match="user ids"):
        m.user_vectors([5])
    with pytest.raises(ValueError, match="user ids"):
        m.user_vectors([-1])
    with pytest.raises(ValueError, match="shape"):
        m.user_vectors([1, 2], seqs[:1])
    with pytest.raises(ValueError, match="n_rec"):
        m.recommend_dynamic(1, 51, SimpleNamespace(item2id=None, user_consumed=None))
    assert _lib.launch_count() == n0
