"""Caser / WaveNet on the GPU: ``b200_caser_encode`` / ``b200_wavenet_encode`` + the Dense head beside the user
table against the float64 oracle, bit-identity of a user's vector across batches, and the encoder envelope.  The
serving path (``set_embeddings`` with the OOV user row, retrieval, ``recommend_dynamic``, the ``ValueError`` checks)
is tested for all three sequence models in test_gpu_dyn_embed_serving."""
import numpy as np
import pytest

from _conv_encoder_oracle import user_vectors as oracle_vectors
from _dyn_embed_data import GPU_ATOL, close as _close, conv_model as _model, conv_raw as _raw, data as _data

pytestmark = pytest.mark.gpu


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
