"""RNN4Rec on the GPU: ``b200_rnn_encode`` + the Dense head against the float64 oracle of both TensorFlow graphs,
bit-identity of a user's vector across batches, and the encoder envelope.  The serving path (``set_embeddings``,
retrieval, ``recommend_dynamic``, the ``user_vectors`` checks) is tested for all three sequence models in
test_gpu_dyn_embed_serving."""
import numpy as np
import pytest

from _dyn_embed_data import GPU_ATOL, K, N_ITEMS, close as _close, data as _data, rnn4rec_model as _model
from _rnn4rec_oracle import user_vectors as oracle_vectors

pytestmark = pytest.mark.gpu


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
