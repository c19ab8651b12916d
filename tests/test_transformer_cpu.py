"""CPU: the Transformer oracle (tests/_transformer_oracle.py) against itself and per-head loops, the reference's
positional table, the OR-ed causal mask, weight interchange for both TensorFlow graphs, the float32 margin under
the GPU bound, and the C-ABI's shape checks (no device compute)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _transformer_oracle as to  # noqa: E402

from oracle import tf_models as tm  # noqa: E402


def _as_legacy(w):
    """The keras-scheme variables restated as the legacy graph's: flattened kernels, and a value Dense that maps the
    projected keys onto the keras values (Wv' = Wk^-1 Wv)."""
    out = dict(w, tfm_scheme="legacy", tfm_layers=[])
    for lw in w["tfm_layers"]:
        D = lw["query"].shape[0]
        wk = lw["key"].reshape(D, D).astype(np.float64)
        out["tfm_layers"].append(dict(
            query=lw["query"].reshape(D, D), key=lw["key"].reshape(D, D),
            value=np.linalg.solve(wk, lw["value"].reshape(D, D).astype(np.float64)),
            output=lw["attention_output"].reshape(D, D), rms_att=lw["rms_att"], rms_ffn=lw["rms_ffn"],
            ffn1=lw["ffn1"], ffn2=lw["ffn2"]))
    return out


def _head_loop_encode(w, G, seqs, lens):
    """The encoder with one explicit loop per (row, head, query, key), float64."""
    T = seqs.shape[1]
    K = w["user_embeds"].shape[1]
    pos = w.get("positional_encoding")
    pos = to.sinusoidal(T, K) if pos is None else pos.astype(np.float64)
    H = int(w["num_heads"])
    out = []
    for b in range(len(seqs)):
        x = np.concatenate([G[seqs[b]], pos], axis=1)
        for lw in w["tfm_layers"]:
            D = x.shape[1]
            hd = D // H
            h = to.rms_norm(x, lw["rms_att"].astype(np.float64))
            q = h @ lw["query"].reshape(D, D)
            k = h @ lw["key"].reshape(D, D)
            v = h @ lw["value"].reshape(D, D)
            o = np.zeros_like(q)
            for hh in range(H):
                c = slice(hh * hd, (hh + 1) * hd)
                for i in range(T):
                    sc = np.array([q[i, c] @ k[j, c] / np.sqrt(hd) for j in range(T)])
                    vis = np.array([j < lens[b] or (w["use_causal_mask"] and j <= i) for j in range(T)])
                    sc = np.where(vis, sc, (sc.astype(np.float32) - np.float32(1e9)).astype(np.float64))
                    p = np.exp(sc - sc.max())
                    p /= p.sum()
                    o[i, c] = p @ v[:, c]
            a = o @ lw["attention_output"].reshape(D, D) + x
            x = a + to.gelu(to.rms_norm(a, lw["rms_ffn"].astype(np.float64)) @ lw["ffn1"]) @ lw["ffn2"]
        out.append(to.rms_norm(x, w["rms_last"].astype(np.float64)))
    return np.stack(out)


@pytest.mark.parametrize("c", [to.CASES[0], to.CASES[2], to.CASES[4]], ids=to.case_id)
def test_oracle_versions_agree_and_match_loops(c):
    rng, spec, w, seqs, lens = to.make_case(c)
    users, items, sparse, dense = to.case_rows(rng, spec, R=60)
    a = to.transformer_forward(w, spec, users, items, seqs, lens, sparse, dense, np.float64, "keras")
    b = to.transformer_forward(_as_legacy(w), spec, users, items, seqs, lens, sparse, dense, np.float64, "legacy")
    np.testing.assert_allclose(a, b, rtol=1e-9, atol=1e-9)
    G = to.item_table(w, spec, c[2], np.float64)
    uid = np.array([0, 1, 2, spec["n_users"], 9])
    np.testing.assert_allclose(to.encode(w, G, seqs[uid], lens[uid], np.float64),
                               _head_loop_encode(w, G, seqs[uid], lens[uid]), rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("d", [16, 7, 1, 32])
def test_sinusoidal_table_matches_reference_formula(d):
    from librecommender_b200.feat_models import sinusoidal_positions

    T = 12
    ref = np.zeros((T, d))
    for t in range(T):
        for i in range(d):
            e = (i - i % 2) / d                    # dim[2i+1] = dim[2i], for odd d as well
            ref[t, i] = np.sin(t / 10000 ** e) if i % 2 == 0 else np.cos(t / 10000 ** e)
    np.testing.assert_allclose(to.sinusoidal(T, d), ref, rtol=1e-12, atol=1e-12)
    np.testing.assert_allclose(sinusoidal_positions(T, d), ref.astype(np.float32), rtol=1e-6, atol=1e-7)


def test_causal_flag_changes_only_empty_sequences():
    c = ("feat", 16, "concat", 2, 2, False, "trainable", True, "keras")
    rng, spec, w, seqs, lens = to.make_case(c)
    G = to.item_table(w, spec, "concat", np.float64)
    users = np.arange(spec["n_users"] + 1)
    items = rng.integers(0, spec["n_items"], size=len(users))
    sparse, dense = tm.row_features(spec, users, items)
    off = to.transformer_forward(w, spec, users, items, seqs, lens, sparse, dense, causal=False)
    on = to.transformer_forward(w, spec, users, items, seqs, lens, sparse, dense, causal=True)
    empty = lens[users] == 0
    assert empty.sum() >= 1 and (~empty).sum() > 10
    np.testing.assert_allclose(on[~empty], off[~empty], rtol=1e-12, atol=1e-12)
    assert np.abs(on[empty] - off[empty]).min() > 1e-6
    S_on = to.encode(w, G, seqs[:3], lens[:3], np.float64, causal=True)
    S_off = to.encode(w, G, seqs[:3], lens[:3], np.float64, causal=False)
    assert np.abs(S_on[0] - S_off[0]).max() > 1e-6      # len 0: every row differs


def test_empty_sequence_scores_are_formed_in_float32():
    """With len = 0 every key is hidden: fl32(score - 1e9) = -1e9 for |score| < 32, uniform weights."""
    S = np.random.default_rng(0).standard_normal((1, 5, 4))
    q = np.ones((1, 4))
    got = to.target_attention(q, S, [0], np.float64)
    np.testing.assert_allclose(got, S.mean(axis=1), rtol=1e-12)


@pytest.mark.parametrize("scheme", ["keras", "legacy"])
@pytest.mark.parametrize("pos", ["trainable", "sinusoidal"])
def test_weights_io_round_trip(tmp_path, scheme, pos):
    from librecommender_b200 import synthetic as syn
    from librecommender_b200 import weights_io as wio

    rng = np.random.default_rng(5)
    spec = syn.make_spec(rng, 20, 30, [4], [5, 6], 1, 1)
    raw = syn.make_transformer_weights(rng, spec, 8, 2, 2, 10, (32, 16), True, pos, True, "elementwise", scheme)
    np.savez(tmp_path / "m_tf_variables.npz", **wio.transformer_tf_variables(raw))
    got = wio.load_reference_tf_model(str(tmp_path), "m", "Transformer", 2, True, num_heads=2, num_tfm_layers=2,
                                      positional_embedding=pos, use_causal_mask=True, feat_agg_mode="elementwise")
    ref = wio.transformer_weights(raw)
    for lg, lr in zip(got["tfm_layers"], ref["tfm_layers"]):
        for k in lr:
            np.testing.assert_array_equal(lg[k], lr[k])
    for k in ("rms_last", "rms_item", "out_kernel", "out_bias"):
        np.testing.assert_array_equal(got[k], ref[k])
    assert ("positional_encoding" in got) == (pos == "trainable")
    np.testing.assert_array_equal(got["ln_sparse"]["scale"], ref["ln_sparse"]["scale"])
    for i in range(2):
        np.testing.assert_array_equal(got["mlp"]["kernels"][i], raw["mlp"]["kernels"][i])
    assert got["num_heads"] == 2 and got["use_causal_mask"] and got["feat_agg_mode"] == "elementwise"
    if scheme == "legacy":
        lw = raw["tfm_layers"][0]
        np.testing.assert_array_equal(got["tfm_layers"][0]["wv"], (lw["key"].astype(np.float64)
                                                                     @ lw["value"].astype(np.float64)).astype(np.float32))


def test_loader_reports_missing_or_misshaped_variable(tmp_path):
    from librecommender_b200 import synthetic as syn
    from librecommender_b200 import weights_io as wio

    rng = np.random.default_rng(6)
    spec = syn.make_spec(rng, 20, 30, [], [], 0, 0)
    raw = syn.make_transformer_weights(rng, spec, 8, 1, 1, 10, (32, 16), False)
    v = wio.transformer_tf_variables(raw)
    name = "transformer_layer1/rms_norm_ffn/scale:0"
    np.savez(tmp_path / "a_tf_variables.npz", **{k: a for k, a in v.items() if k != name})
    with pytest.raises(KeyError, match="rms_norm_ffn"):
        wio.load_reference_tf_model(str(tmp_path), "a", "Transformer", 2, False)
    bad = dict(v)
    bad["transformer_layer1/dense_1/kernel:0"] = bad["transformer_layer1/dense_1/kernel:0"][:-1]
    np.savez(tmp_path / "b_tf_variables.npz", **bad)
    with pytest.raises(KeyError, match="has shape"):
        wio.load_reference_tf_model(str(tmp_path), "b", "Transformer", 2, False)
    np.savez(tmp_path / "c_tf_variables.npz", **{k: a for k, a in v.items() if k != "transformer/positional_encoding:0"})
    with pytest.raises(KeyError, match="positional_encoding"):
        wio.load_reference_tf_model(str(tmp_path), "c", "Transformer", 2, False)
    got = wio.load_reference_tf_model(str(tmp_path), "c", "Transformer", 2, False, positional_embedding="sinusoidal")
    assert "positional_encoding" not in got


def test_default_names_follow_the_uniquifying_rule():
    from librecommender_b200 import weights_io as wio

    k = wio.default_tf_names("Transformer", 3, True, n_layers=2, scheme="keras")
    assert k["tfm_layers"][1]["query"] == "transformer_layer2/multi_head_attention_1/query/kernel:0"
    assert k["tfm_layers"][1]["ffn2"] == "transformer_layer2/dense_3/kernel:0"
    assert k["out_kernel"] == "dense_4/kernel:0"
    g = wio.default_tf_names("Transformer", 3, True, n_layers=2, scheme="legacy")
    assert g["tfm_layers"][1]["output"] == "transformer_layer2/dense_9/kernel:0"
    assert g["out_bias"] == "dense_12/bias:0"


@pytest.mark.parametrize("c", to.CASES, ids=to.case_id)
def test_float32_meets_gpu_bound_with_margin(c):
    rng, spec, w, seqs, lens = to.make_case(c)
    users, items, sparse, dense = to.case_rows(rng, spec, R=200)
    ref = to.transformer_forward(w, spec, users, items, seqs, lens, sparse, dense, np.float64)
    got = to.transformer_forward(w, spec, users, items, seqs, lens, sparse, dense, np.float32)
    to.close(got.astype(np.float64), ref, tol=2.5e-6)


def test_cabi_rejects_out_of_envelope_shapes_before_launch():
    from librecommender_b200 import _lib

    lib = _lib.lib
    x = np.zeros(64, dtype=np.float32)
    ix = np.zeros(64, dtype=np.int64)
    n0 = _lib.launch_count()
    # (T, Kp, Kpos, heads, layers)
    for T, Kp, Kpos, H, L in [(65, 16, 16, 1, 1), (10, 120, 16, 1, 1), (10, 16, 16, 3, 1), (10, 16, 16, 1, 5),
                              (10, 16, 16, 1, 0), (0, 16, 16, 1, 1)]:
        rc = lib.b200_transformer_encode(_lib.ptr(ix), 2, _lib.ptr(x), _lib.ptr(x), 64, _lib.ptr(x), 64, Kp, _lib.ptr(x),
                                         Kpos, T, H, L, 0, _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), None)
        assert rc == -2, (T, Kp, Kpos, H, L)
    for T, D, H1, H2, H3 in [(65, 32, 64, 32, 0), (10, 129, 64, 32, 0), (10, 32, 257, 32, 0), (10, 32, 64, 65, 0),
                             (10, 32, 64, 32, 33)]:
        rc = lib.b200_transformer_pair_scores(_lib.ptr(x), 200, 5, _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), 1,
                                              _lib.ptr(x), 300, T, D, H1, H2, H3, _lib.ptr(x), _lib.ptr(x), _lib.ptr(x),
                                              _lib.ptr(x), _lib.ptr(x), 0.0, _lib.ptr(x), 5, None)
        assert rc == -2, (T, D, H1, H2, H3)
    rc = lib.b200_transformer_target_attention(_lib.ptr(x), 200, _lib.ptr(x), 10, 129, _lib.ptr(x), None, None, 5, 3, 0,
                                               _lib.ptr(x), 200, None)
    assert rc == -2
    rc = lib.b200_linear_f32(_lib.ptr(x), 4, 1, _lib.ptr(x), 4, None, 4, 4, 3, _lib.ptr(x), 4, None)
    assert rc == -2 and b"activation code" in lib.b200_last_error()
    assert _lib.launch_count() == n0
    assert lib.b200_transformer_pair_smem_bytes(64, 128, 256) > 227 * 1024 >= lib.b200_transformer_pair_smem_bytes(50, 80, 128)
