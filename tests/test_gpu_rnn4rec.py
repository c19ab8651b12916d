"""RNN4Rec on the GPU: ``b200_rnn_encode`` + the Dense head against the float64 oracle of both TensorFlow graphs,
bit-identity of a user's vector across calls and batches, the serving tables, all-items retrieval and
``recommend_dynamic``."""
from types import SimpleNamespace

import numpy as np
import pytest

from _rnn4rec_oracle import recommend as oracle_recommend
from _rnn4rec_oracle import serving_tables, user_vectors as oracle_vectors

pytestmark = pytest.mark.gpu

N_ITEMS, K = 700, 16
GPU_ATOL = 2e-5       # float32 restatement of the same shapes stays under a quarter of this (test_rnn4rec_cpu)


def _close(got, ref, atol):
    err = np.abs(np.asarray(got, np.float64) - ref).max() / max(1.0, np.abs(ref).max())
    assert err < atol, err


def _data(rng, n_users, T, n_items=N_ITEMS):
    """Consumed lists with an empty history (len 0), one item (len 1) and long ones (len T), as recent_sequences."""
    from librecommender_b200.feat_models import recent_sequences

    sizes = rng.integers(0, 2 * T, size=n_users)
    sizes[:3] = [0, 1, 3 * T]
    consumed = {u: rng.choice(n_items, size=int(s), replace=False).tolist() for u, s in enumerate(sizes) if s}
    seqs, lens = recent_sequences(consumed, n_users, n_items, T)
    return consumed, seqs, lens


def _model(raw, n_users, seqs, lens, norm):
    from librecommender_b200.feat_models import RNN4Rec

    return RNN4Rec({"n_users": n_users, "n_items": raw["item_embeds"].shape[0]}, raw, seqs, lens, norm_embed=norm)


CASES = [(typ, scheme, hu, ln) for typ in ("gru", "lstm") for scheme in ("keras", "legacy")
         for hu in ((16,), (32, 64)) for ln in ((False, True) if scheme == "keras" else (False,))]


@pytest.mark.parametrize("T", [10, 50])
@pytest.mark.parametrize("norm", [False, True])
@pytest.mark.parametrize("typ,scheme,hu,ln", CASES)
def test_user_vectors_match_oracle(typ, scheme, hu, ln, norm, T):
    from librecommender_b200.synthetic import make_rnn4rec_weights

    rng = np.random.default_rng(CASES.index((typ, scheme, hu, ln)) * 4 + T + norm)
    n_users = 5003                                    # not a multiple of any tile
    raw = make_rnn4rec_weights(rng, N_ITEMS, K, hu, typ, ln, scheme)
    _, seqs, lens = _data(rng, n_users, T)
    model = _model(raw, n_users, seqs, lens, norm)
    ids = np.arange(n_users + 1)                      # the OOV row (all pad, len 1) included
    got = model.user_vectors(ids).cpu().numpy()
    ref = oracle_vectors(raw, seqs, lens, norm)
    _close(got, ref, GPU_ATOL)
    one = model.user_vectors([2]).cpu().numpy()       # n = 1: the same bits as in the big batch
    np.testing.assert_array_equal(one[0], got[2])


@pytest.mark.parametrize("typ,scheme,hu,ln", [("gru", "keras", (256, 256), True), ("lstm", "legacy", (256,) * 4, False),
                                              ("gru", "legacy", (256,), False)])
def test_envelope_maximum(typ, scheme, hu, ln):
    """T = 128, in_dim = hidden = 256 (and 4 layers): the longest chains the kernel runs."""
    from librecommender_b200.synthetic import make_rnn4rec_weights

    rng = np.random.default_rng(77)
    n_users, T = 67, 128
    raw = make_rnn4rec_weights(rng, 500, K, hu, typ, ln, scheme)
    _, seqs, lens = _data(rng, n_users, T, 500)
    model = _model(raw, n_users, seqs, lens, False)
    got = model.user_vectors(np.arange(n_users + 1)).cpu().numpy()
    _close(got, oracle_vectors(raw, seqs, lens), 1e-4)


@pytest.fixture(scope="module")
def served():
    from librecommender_b200.synthetic import make_rnn4rec_weights

    rng = np.random.default_rng(2024)
    n_users, T = 3001, 10
    raw = make_rnn4rec_weights(rng, N_ITEMS, K, (32, 24), "gru", True, "keras")
    consumed, seqs, lens = _data(rng, n_users, T)
    model = _model(raw, n_users, seqs, lens, False)
    return SimpleNamespace(raw=raw, consumed=consumed, seqs=seqs, lens=lens, model=model, n_users=n_users, T=T)


def test_bit_identity(served):
    m = served.model
    U, I = m.set_embeddings()
    U7, I7 = m.set_embeddings(chunk=7)
    assert U.shape == U7.shape and bool((U == U7).all()) and bool((I == I7).all())
    U2, _ = m.set_embeddings()
    assert bool((U == U2).all())
    rng = np.random.default_rng(1)
    ids = np.concatenate([rng.permutation(served.n_users)[:999], [5, 5, 0, 0, 17]])
    got = m.user_vectors(ids)
    Kd = U.shape[1] - 1
    assert bool((got == U[ids][:, :Kd]).all())
    # recommend_dynamic with the user's own cached sequence scores exactly like its U row
    info = SimpleNamespace(item2id=None, user_consumed=served.consumed)
    u = 4
    seq = served.seqs[u, :served.lens[u]].tolist()
    ids_d, sc_d = m.recommend_dynamic(u, 20, info, seq=seq, inner_id=True, filter_consumed=False, return_scores=True)
    ids_c, sc_c = m.recommend_dynamic(u, 20, info, inner_id=True, filter_consumed=False, return_scores=True)
    full = (U[u:u + 1] @ I[:N_ITEMS].T).cpu().numpy()
    np.testing.assert_array_equal(ids_d, ids_c)
    np.testing.assert_array_equal(sc_d, sc_c)
    from librecommender_b200 import _lib
    import torch

    exact = torch.empty((1, N_ITEMS), dtype=torch.float32, device=U.device)
    zero = torch.zeros(1, dtype=torch.int64, device=U.device)
    _lib.check(_lib.lib.b200_score_rows_f32(_lib.ptr(U[u:u + 1].contiguous()), U.shape[1], _lib.ptr(zero), 1,
                                            _lib.ptr(I), I.stride(0), N_ITEMS, U.shape[1], _lib.ptr(exact), N_ITEMS,
                                            _lib.current_stream()))
    np.testing.assert_array_equal(sc_d[0], exact.cpu().numpy()[0][ids_d[0]])
    assert np.abs(sc_d[0] - full[0][ids_d[0]]).max() < 1e-4


@pytest.mark.parametrize("filter_consumed", [True, False])
def test_set_embeddings_layout_and_retrieval(served, filter_consumed):
    from librecommender_b200.engine import EmbedScorer
    from oracle import ranking as orc

    m, n_users = served.model, served.n_users
    U, I = m.set_embeddings()
    assert U.shape == (n_users + 1, K + 1) and I.shape == (N_ITEMS + 1, K + 1)
    assert float(U[:n_users, K].min()) == 1.0 and float(U[:n_users, K].max()) == 1.0
    ref_u = oracle_vectors(served.raw, served.seqs[:n_users], served.lens[:n_users])
    Uo, Io = serving_tables(served.raw, ref_u)
    _close(U.cpu().numpy(), Uo, GPU_ATOL)
    _close(I.cpu().numpy(), Io, 1e-6)
    np.testing.assert_allclose(U[n_users].cpu().numpy(), U[:n_users].double().mean(0).cpu().numpy(), atol=1e-6)
    np.testing.assert_allclose(I[N_ITEMS].cpu().numpy(), I[:N_ITEMS].double().mean(0).cpu().numpy(), atol=1e-6)
    sc = EmbedScorer(U, I, N_ITEMS, served.consumed, n_users=n_users)
    users = np.random.default_rng(3).integers(0, n_users, 64)
    got = sc.recommend(users, 10, filter_consumed)
    ref_ids, full = oracle_recommend(served.raw, ref_u, users, 10, served.consumed, filter_consumed)
    assert orc.near_tie_mask(ref_ids, got, full.astype(np.float32), 2e-5).all()
    if filter_consumed:
        for r, u in enumerate(users):
            assert not set(got[r]) & set(served.consumed.get(int(u), []))


def test_recommend_dynamic(served):
    import torch

    m, T = served.model, served.T
    seqs_before, lens_before = m.seqs.clone(), m.lens.clone()
    item2id = {f"i{j}": j for j in range(N_ITEMS)}
    info = SimpleNamespace(item2id=item2id, user_consumed=served.consumed)
    rng = np.random.default_rng(8)
    long = [f"i{j}" for j in rng.integers(0, N_ITEMS, 3 * T)]
    got = m.recommend_dynamic(3, 15, info, seq=long, return_scores=True)
    tail = m.recommend_dynamic(3, 15, info, seq=long[-T:], return_scores=True)
    np.testing.assert_array_equal(got[0], tail[0])          # longer than T: only the last T items count
    np.testing.assert_array_equal(got[1], tail[1])
    v = m.user_vectors([0], np.array([[item2id[i] for i in long[-T:]]], np.int32), np.array([T]))
    ref = oracle_vectors(served.raw, np.array([[item2id[i] for i in long[-T:]]]), np.array([T]))
    _close(v.cpu().numpy(), ref, GPU_ATOL)
    assert not set(got[0][0]) & set(served.consumed.get(3, []))
    # unknown original ids become the pad id n_items
    unk = m.recommend_dynamic(3, 15, info, seq=["nope", "i5", "zzz"], return_scores=True)
    pad = m.recommend_dynamic(3, 15, info, seq=[N_ITEMS, 5, N_ITEMS], inner_id=True, return_scores=True)
    np.testing.assert_array_equal(unk[0], pad[0])
    np.testing.assert_array_equal(unk[1], pad[1])
    # the unknown user (id n_users) gets no consumed filter; user_feats is ignored
    cold = m.recommend_dynamic(served.n_users, 15, info, user_feats={"x": 1}, seq=long, return_scores=True)
    warm = m.recommend_dynamic(3, 15, info, seq=long, filter_consumed=False, return_scores=True)
    np.testing.assert_array_equal(cold[0], warm[0])
    assert bool(torch.equal(m.seqs, seqs_before)) and bool(torch.equal(m.lens, lens_before))
    with pytest.raises(ValueError):
        m.recommend_dynamic(3, N_ITEMS + 1, info)


def test_out_of_envelope_raises_before_launch():
    from librecommender_b200 import _lib
    from librecommender_b200.synthetic import make_rnn4rec_weights

    rng = np.random.default_rng(0)
    n0 = _lib.launch_count()
    raw = make_rnn4rec_weights(rng, 50, K, (16,) * 5, "gru", False, "keras")
    with pytest.raises(ValueError, match="layers"):
        _model(raw, 4, np.zeros((5, 10), np.int32), np.ones(5, np.int32), False)
    raw = make_rnn4rec_weights(rng, 50, K, (16,), "lstm", False, "legacy")
    with pytest.raises(ValueError, match="max_seq_len"):
        _model(raw, 4, np.zeros((5, 129), np.int32), np.ones(5, np.int32), False)
    assert _lib.launch_count() == n0
