"""Seeded data and model builders of the GPU tests of the dynamic-embedding sequence models: RNN4Rec, Caser and
WaveNet."""
import numpy as np

N_ITEMS, K = 700, 16
GPU_ATOL = 2e-5       # the float32 restatements of the same shapes stay under a quarter of this (test_rnn4rec_cpu,
#                       test_caser_wavenet_cpu)


def close(got, ref, atol):
    err = np.abs(np.asarray(got, np.float64) - ref).max() / max(1.0, np.abs(ref).max())
    assert err < atol, err


def data(rng, n_users, T, n_items=N_ITEMS):
    """Consumed lists with an empty history (len 0, all pad), one item (len 1) and long ones (len T), as
    recent_sequences."""
    from librecommender_b200.feat_models import recent_sequences

    sizes = rng.integers(0, 2 * T, size=n_users)
    sizes[:3] = [0, 1, 3 * T]
    consumed = {u: rng.choice(n_items, size=int(s), replace=False).tolist() for u, s in enumerate(sizes) if s}
    seqs, lens = recent_sequences(consumed, n_users, n_items, T)
    return consumed, seqs, lens


def rnn4rec_model(raw, n_users, seqs, lens, norm):
    from librecommender_b200.feat_models import RNN4Rec

    return RNN4Rec({"n_users": n_users, "n_items": raw["item_embeds"].shape[0]}, raw, seqs, lens, norm_embed=norm)


def conv_raw(rng, model, n_users, T, widths, dilated=True, k=K, n_items=N_ITEMS):
    from librecommender_b200.synthetic import make_caser_weights, make_wavenet_weights

    if model == "Caser":
        return make_caser_weights(rng, n_users, n_items, k, T, *widths)
    return make_wavenet_weights(rng, n_users, n_items, k, *widths, dilated=dilated)


def conv_model(raw, n_users, seqs, lens, norm):
    from librecommender_b200.feat_models import Caser, WaveNet

    cls = Caser if "vertical" in raw else WaveNet
    return cls({"n_users": n_users, "n_items": raw["item_embeds"].shape[0]}, raw, seqs, lens, norm_embed=norm)
