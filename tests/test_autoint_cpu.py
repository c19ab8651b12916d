"""CPU: the AutoInt restatement (tests/_autoint_oracle.py) and its weight interchange.

* the two graphs ``multi_head_attention`` builds (keras for TF >= 2.10, legacy before) agree in float64 when the
  keras value kernel equals the legacy ``Wk Wv'``, and each matches a per-head loop restatement;
* ``weights_io`` reads both naming schemes back from ``.npz`` files, folds the legacy value map, and reports a
  missing or misshaped variable with what the file does contain;
* the stacked field block follows ``concat_embed`` (autoint.py:152-158), multi-sparse fields included;
* float32 meets the GPU tests' bound with 4x to spare, so that bound is not one float32 only just meets;
* the C-ABI rejects unsupported shapes before launching anything."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _autoint_oracle as ao  # noqa: E402


def _loop_forward(x, layers, H, residual, out_kernel, out_bias):
    """Per-row, per-head, per-field loops over the engine's weight layout (float64)."""
    R, F, K = x.shape
    out = np.empty(R)
    for r in range(R):
        X = x[r].copy()
        for lw in layers:
            wq, wk, wv, wo = (np.asarray(lw[k], dtype=np.float64) for k in ("wq", "wk", "wv", "wo"))
            D = wq.shape[1]
            hd = D // H
            Q, Kt, V = X @ wq, X @ wk, X @ wv
            O = np.zeros((F, D))
            for h in range(H):
                c = slice(h * hd, (h + 1) * hd)
                for f in range(F):
                    s = np.array([Q[f, c] @ Kt[g, c] for g in range(F)]) / np.sqrt(hd)
                    p = np.exp(s - s.max())
                    p /= p.sum()
                    O[f, c] = sum(p[g] * V[g, c] for g in range(F))
            X = X + O @ wo if residual else O @ wo
        out[r] = X.reshape(-1) @ np.asarray(out_kernel, dtype=np.float64).reshape(-1) + float(out_bias)
    return out


def _legacy_twin(w, rng):
    """Legacy variables with the same q / k / out maps as keras `w` and a random Wv'; the keras twin whose value
    kernel is Wk Wv' (float64) computes the same function."""
    leg, ker = dict(w), dict(w)
    leg["autoint_scheme"], leg["autoint_mha"], ker["autoint_mha"] = "legacy", [], []
    for lw in w["autoint_mha"]:
        K, H, hd = lw["query"].shape
        D = H * hd
        vp = rng.uniform(-0.4, 0.4, (D, D))
        leg["autoint_mha"].append(dict(query=lw["query"].reshape(K, D).astype(np.float64),
                                       key=lw["key"].reshape(K, D).astype(np.float64), value=vp,
                                       output=lw["attention_output"].reshape(D, K).astype(np.float64)))
        ker["autoint_mha"].append(dict(lw, value=(lw["key"].reshape(K, D).astype(np.float64) @ vp).reshape(K, H, hd)))
    return ker, leg


@pytest.mark.parametrize("c", [c for c in ao.CASES if c[5] == "keras"], ids=ao.case_id)
def test_oracle_versions_agree_and_match_loops(c):
    from librecommender_b200 import weights_io as wio

    rng, spec, w = ao.make_case(c)
    ker, leg = _legacy_twin(w, rng)
    users, items, sparse, dense = ao.case_rows(rng, spec, R=40)
    zk = ao.autoint_forward(ker, users, items, sparse, dense, np.float64)
    zl = ao.autoint_forward(leg, users, items, sparse, dense, np.float64)
    np.testing.assert_allclose(zl, zk, rtol=1e-12, atol=1e-12)
    x = ao.field_block(w, users, items, sparse, dense, np.float64)
    H, res = w["num_heads"], w["use_residual"]
    # keras: the [K, H, hd] / [H, hd, K] kernels reshaped head-major (kept in float64 here, Wk Wv' included)
    kl = [dict(wq=m["query"].reshape(m["query"].shape[0], -1), wk=m["key"].reshape(m["key"].shape[0], -1),
               wv=m["value"].reshape(m["value"].shape[0], -1),
               wo=m["attention_output"].reshape(-1, m["attention_output"].shape[2])) for m in ker["autoint_mha"]]
    np.testing.assert_allclose(_loop_forward(x, kl, H, res, w["out_kernel"], w["out_bias"][0]), zk, rtol=1e-12,
                               atol=1e-12)
    # legacy through the product conversion, which folds Wk Wv' in float64 and rounds it to float32
    ll = wio.autoint_layers(leg["autoint_mha"], "legacy")
    np.testing.assert_allclose(_loop_forward(x, ll, H, res, w["out_kernel"], w["out_bias"][0]), zl, rtol=2e-6,
                               atol=1e-7)


def _npz_vars(w, scheme, L):
    """{TF variable name: array} of raw weights `w`, named by weights_io.default_tf_names."""
    from librecommender_b200 import weights_io as wio

    names = wio.default_tf_names("AutoInt", None, False, n_layers=L, scheme=scheme)
    out = wio.to_tf_variables({k: w[k] for k in wio.EMBEDDING_SCOPE if k in w})
    for lw, ln in zip(w["autoint_mha"], names["autoint_mha"]):
        for k, n in ln.items():
            out[n] = np.asarray(lw[k], dtype=np.float32)
    out[names["out_kernel"]] = np.asarray(w["out_kernel"], dtype=np.float32)
    out[names["out_bias"]] = np.asarray(w["out_bias"], dtype=np.float32).reshape(1)
    return out


@pytest.mark.parametrize("scheme", ["keras", "legacy"])
@pytest.mark.parametrize("att", [None, (4, 8)])
def test_weights_io_round_trip(tmp_path, scheme, att):
    from librecommender_b200 import synthetic as syn
    from librecommender_b200 import weights_io as wio

    rng = np.random.default_rng(3)
    spec = syn.make_spec(rng, 30, 40, [5], [7, 3], 1, 1)
    H, K = 2, 8
    w = syn.make_autoint_weights(rng, spec, K, att, H, False, scheme)
    hds = wio.autoint_head_dims(att)
    L = len(hds)
    v = _npz_vars(w, scheme, L)
    # the names TensorFlow gives the variables of each graph
    if scheme == "keras":
        assert f"multi_head_attention_{L - 1}/attention_output/kernel:0" in v and "dense/kernel:0" in v
        assert v["multi_head_attention/query/kernel:0"].shape == (K, H, hds[0])
    else:
        assert f"dense_{4 * L - 1}/kernel:0" in v and f"dense_{4 * L}/bias:0" in v
        assert v["dense_2/kernel:0"].shape == (H * hds[0], H * hds[0])
    np.savez(tmp_path / "m_tf_variables.npz", **v)
    got = wio.load_reference_tf_model(str(tmp_path), "m", "AutoInt", None, False, num_heads=H, att_embed_size=att,
                                      use_residual=False)
    ref = wio.autoint_weights(w)
    assert got["num_heads"] == H and got["use_residual"] is False and len(got["autoint_layers"]) == L
    for a, b in zip(got["autoint_layers"], ref["autoint_layers"]):
        for k in ("wq", "wk", "wv", "wo"):
            np.testing.assert_array_equal(a[k], b[k])
    for lw, raw in zip(got["autoint_layers"], w["autoint_mha"]):
        if scheme == "legacy":      # the value map folded: Wk Wv' in float64, then cast
            fold = (raw["key"].astype(np.float64) @ raw["value"].astype(np.float64)).astype(np.float32)
            np.testing.assert_array_equal(lw["wv"], fold)
            assert not np.array_equal(lw["wv"], raw["key"])
        else:                       # head-major columns h * hd + j
            hd = raw["query"].shape[2]
            np.testing.assert_array_equal(lw["wq"][:, hd:2 * hd], raw["query"][:, 1, :])
            np.testing.assert_array_equal(lw["wo"][hd:2 * hd], raw["attention_output"][1])
    np.testing.assert_array_equal(got["out_kernel"], np.asarray(w["out_kernel"]).reshape(-1))
    np.testing.assert_array_equal(got["user_embeds"], w["user_embeds"])
    # a missing and a misshaped variable: KeyError naming it and listing what the file holds
    names = wio.default_tf_names("AutoInt", None, False, n_layers=L, scheme=scheme)
    victim = names["autoint_mha"][L - 1]["value"]
    bad = dict(v)
    del bad[victim]
    np.savez(tmp_path / "b_tf_variables.npz", **bad)
    with pytest.raises(KeyError, match="not in the file") as e:
        wio.load_reference_tf_model(str(tmp_path), "b", "AutoInt", None, False, num_heads=H, att_embed_size=att)
    assert victim in str(e.value) and names["out_kernel"] in str(e.value)
    bad = dict(v)
    bad[victim] = np.zeros((3, 3), np.float32)
    np.savez(tmp_path / "s_tf_variables.npz", **bad)
    with pytest.raises(KeyError, match="has shape") as e:
        wio.load_reference_tf_model(str(tmp_path), "s", "AutoInt", None, False, num_heads=H, att_embed_size=att)
    assert victim in str(e.value)
    # wrong head count for the file: every kernel is checked against the given shape
    with pytest.raises(KeyError, match="has shape"):
        wio.load_reference_tf_model(str(tmp_path), "m", "AutoInt", None, False, num_heads=1, att_embed_size=att)


def test_scheme_from_version_and_head_dims():
    from librecommender_b200 import weights_io as wio

    assert [wio.autoint_scheme(v) for v in ("2.10.0", "2.15.1", "2.9.3", "1.15", "keras", "legacy")] == \
        ["keras", "keras", "legacy", "legacy", "keras", "legacy"]
    assert wio.autoint_head_dims(None) == [8, 8, 8] and wio.autoint_head_dims(16) == [16]
    assert wio.autoint_head_dims((4, 8)) == [4, 8]


@pytest.mark.parametrize("combiner", ["sqrtn", "normal", None])
def test_field_block_follows_concat_embed(combiner):
    """autoint.py:152-158: [user, item, sparse fields (multi-sparse pooled per field unless "normal"), dense]."""
    rng, spec, w = ao.make_case(("multi" if combiner else "feat", 8, None, 2, True, "keras"))
    if combiner:
        w["multi_sparse"]["combiner"] = combiner
    users, items, sparse, dense = ao.case_rows(rng, spec, R=30)
    x = ao.field_block(w, users, items, sparse, dense, np.float64)
    E = w["sparse_embeds"].astype(np.float64)
    fields = [w["user_embeds"][users], w["item_embeds"][items]]
    info = spec.get("multi_sparse_combine_info")
    if combiner == "sqrtn":
        s0 = info["field_offset"][0]
        fields += [E[sparse[:, j]] for j in range(s0)]
        for off, ln, oov in zip(info["field_offset"], info["field_len"], info["feat_oov"]):
            idx = sparse[:, off:off + ln]
            keep = (idx != oov).astype(np.float64)
            n = keep.sum(axis=1, keepdims=True)
            fields.append(np.divide((E[idx] * keep[:, :, None]).sum(axis=1), np.sqrt(n), out=np.zeros((len(idx), 8)),
                                    where=n > 0))
    else:
        fields += [E[sparse[:, j]] for j in range(spec["n_sparse"])]
    fields += [dense[:, j:j + 1].astype(np.float64) * w["dense_embeds"][j] for j in range(spec["n_dense"])]
    ref = np.stack([np.asarray(f, dtype=np.float64) for f in fields], axis=1)
    np.testing.assert_allclose(x, ref, rtol=1e-15, atol=1e-15)
    F = 2 + (info["field_offset"][0] + len(info["field_offset"]) if combiner == "sqrtn" else spec["n_sparse"]) + \
        spec["n_dense"]
    assert x.shape[1] == F


@pytest.mark.parametrize("c", ao.CASES, ids=ao.case_id)
def test_float32_meets_gpu_bound_with_4x_spare(c):
    rng, spec, w = ao.make_case(c)
    users, items, sparse, dense = ao.case_rows(rng, spec)
    z64 = ao.autoint_forward(w, users, items, sparse, dense, np.float64)
    z32 = ao.autoint_forward(w, users, items, sparse, dense, np.float32).astype(np.float64)
    ao.close(z32, z64, 1e-5 / 4)


def test_float32_large_logits_meets_bound_with_4x_spare():
    rng, spec, w = ao.make_case(ao.LARGE_LOGIT_CASE)
    users, items, sparse, dense = ao.case_rows(rng, spec)
    ao.scale_to_large_logits(w, (users, items, sparse, dense))
    s = ao.attention_logits_first_layer(w, users, items, sparse, dense)
    assert np.abs(s).max() > 80
    z64 = ao.autoint_forward(w, users, items, sparse, dense, np.float64)
    z32 = ao.autoint_forward(w, users, items, sparse, dense, np.float32).astype(np.float64)
    assert np.isfinite(z64).all()
    ao.close(z32, z64, 1e-5 / 4)


def test_cabi_rejects_unsupported_shapes_before_launch():
    from librecommender_b200 import _lib

    lib = _lib.lib
    x = np.zeros(64, np.float32)
    hd = np.array([8, 8, 8, 8, 8], np.int32)
    n0 = _lib.launch_count()
    # (F, K, H, L, head dims)
    for F, K, H, L, hds in ((8, 65, 2, 3, hd), (8, 16, 2, 5, hd), (8, 16, 9, 3, hd), (131, 16, 2, 3, hd),
                            (1, 16, 2, 3, hd), (8, 16, 2, 2, np.array([8, 0], np.int32)), (8, 16, 0, 1, hd)):
        rc = lib.b200_autoint_rows(_lib.ptr(x), F * K, 10, F, K, H, L, _lib.ptr(hds), _lib.ptr(x), _lib.ptr(x),
                                   0.0, 1, _lib.ptr(x), None)
        assert rc == -2, (F, K, H, L)
        assert b"b200_autoint_rows" in lib.b200_last_error()
        rc = lib.b200_autoint_grid(_lib.ptr(x), K, 2, _lib.ptr(x), K, 5, _lib.ptr(hds), F, K, H, L, _lib.ptr(hds),
                                   _lib.ptr(x), _lib.ptr(x), 0.0, 1, _lib.ptr(x), 5, None)
        assert rc == -2
    assert _lib.launch_count() == n0
