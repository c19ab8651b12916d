"""CPU: the SIM oracle (tests/_sim_oracle.py) across both attention graphs, the dual-sequence builders against the
reference's algorithm, weight interchange for both TensorFlow graphs, the float32 margin under the GPU bound, and the
C-ABI's shape checks (no device compute)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import _sim_oracle as so  # noqa: E402
import _transformer_oracle as to  # noqa: E402

from librecommender_b200 import weights_io as wio  # noqa: E402
from librecommender_b200.consumed import ConsumedCSR  # noqa: E402
from librecommender_b200.dynamic_feats import build_dual_seq  # noqa: E402
from librecommender_b200.feat_models import recent_dual_sequences, recent_dual_sequences_csr  # noqa: E402
from oracle import tf_models as tm  # noqa: E402


def _ref_dual_seqs(n_users, user_consumed, pad_index, long_max_len, short_max_len):
    """get_recent_dual_seqs (libreco/batch/sequence.py:150-188), transcribed with its own loop and branches."""
    long_seqs = np.full((n_users, long_max_len), pad_index, dtype=np.int32)
    short_seqs = np.full((n_users, short_max_len), pad_index, dtype=np.int32)
    long_seq_lens, short_seq_lens = [], []
    total_max_len = long_max_len + short_max_len
    for u in range(n_users):
        consumed_items = user_consumed[u]
        items_len = len(consumed_items)
        if items_len <= short_max_len:
            long_seq_lens.append(1)
            short_seqs[u, :items_len] = consumed_items[:items_len]
            short_seq_lens.append(items_len)
        else:
            if items_len < total_max_len:
                long_size = items_len - short_max_len
                long_seqs[u, :long_size] = consumed_items[:long_size]
                long_seq_lens.append(long_size)
            else:
                long_start = items_len - total_max_len
                long_seqs[u] = consumed_items[long_start:long_start + long_max_len]
                long_seq_lens.append(long_max_len)
            short_seqs[u] = consumed_items[items_len - short_max_len:]
            short_seq_lens.append(short_max_len)
    long_seqs = np.vstack([long_seqs, np.full(long_max_len, pad_index, dtype=np.int32)])
    short_seqs = np.vstack([short_seqs, np.full(short_max_len, pad_index, dtype=np.int32)])
    return (long_seqs, np.append(long_seq_lens, [1]).astype(np.int32), short_seqs,
            np.append(short_seq_lens, [1]).astype(np.int32))


def _ref_build_dual_seq(seq, n_items, long_max_len, short_max_len):
    """build_dual_seq (recommendation/preprocess.py:49-76) on inner ids, transcribed."""
    total_max_len = long_max_len + short_max_len
    long_seq = np.full((1, long_max_len), n_items, dtype=np.int32)
    if len(seq) >= total_max_len:
        long_len = long_max_len
        start_index = len(seq) - total_max_len
        long_seq[0] = seq[start_index:start_index + long_len]
    elif len(seq) > short_max_len:
        long_len = len(seq) - short_max_len
        long_seq[0, :long_len] = seq[:long_len]
    else:
        long_len = 1
    short_seq = np.full((1, short_max_len), n_items, dtype=np.int32)
    short_len = min(short_max_len, len(seq))
    short_seq[0, :short_len] = seq[-short_len:]
    return long_seq, np.array([long_len], dtype=np.int32), short_seq, np.array([short_len], dtype=np.int32)


def _as_legacy(w):
    """The keras-scheme attention restated as the legacy graph's: flattened kernels and a value Dense that maps the
    projected keys onto the keras values (Wv' = Wk^-1 Wv)."""
    m = w["sim_mha"]
    K = m["query"].shape[0]
    wk = m["key"].reshape(K, K).astype(np.float64)
    return dict(w, sim_scheme="legacy", sim_mha=dict(
        query=m["query"].reshape(K, K), key=m["key"].reshape(K, K),
        value=np.linalg.solve(wk, m["value"].reshape(K, K).astype(np.float64)),
        output=m["attention_output"].reshape(K, K)))


@pytest.mark.parametrize("c", [c for c in so.CASES if c[4] == "keras"], ids=so.case_id)
def test_oracle_keras_equals_legacy(c):
    rng, spec, w, _, seqs = so.make_case(c)
    users, items, sparse, dense = so.case_rows(rng, spec, R=200)
    ref, sel, _, _ = so.sim_forward(w, spec, users, items, *seqs, so.TOPK_DEFAULT, sparse, dense)
    got, sel2, _, _ = so.sim_forward(_as_legacy(w), spec, users, items, *seqs, so.TOPK_DEFAULT, sparse, dense)
    assert (sel == sel2).all()
    np.testing.assert_allclose(got, ref, rtol=1e-9, atol=1e-9)


def test_oracle_selection_rule_and_margin():
    """Equal scores resolve to the lower position; masked positions fill up a short window from position len on;
    the margin is infinite exactly when at most k positions are valid."""
    s = np.array([[1.0, 3.0, 3.0, 2.0, 3.0, -so.NEG, -so.NEG]])
    assert so.gsu_select(s, 2).tolist() == [[1, 2]]
    assert so.gsu_select(s, 4).tolist() == [[1, 2, 3, 4]]
    assert so.gsu_select(s, 6).tolist() == [[0, 1, 2, 3, 4, 5]]
    m, sk = so.gsu_margin(s, [5], 2)
    assert m[0] == 1.0 and sk[0] == 3.0              # the tie at 3 is exact: the gap is to the next value, 2
    m, _ = so.gsu_margin(s, [5], 5)
    assert np.isinf(m[0])
    # long_len 0: every position masked, the selection is 0..k-1
    assert so.gsu_select(np.full((1, 8), -so.NEG), 3).tolist() == [[0, 1, 2]]


def test_oracle_forced_selection_changes_only_the_long_block():
    rng, spec, w, _, seqs = so.make_case(so.CASES[0])
    users, items, _, _ = so.case_rows(rng, spec, R=50)
    z, sel, _, _ = so.sim_forward(w, spec, users, items, *seqs, so.TOPK_DEFAULT)
    z2, sel2, _, _ = so.sim_forward(w, spec, users, items, *seqs, so.TOPK_DEFAULT, sel=sel)
    assert (sel2 == sel).all() and (z2 == z).all()
    shifted = np.sort((sel + 1) % so.L_DEFAULT, axis=1)
    z3, _, _, _ = so.sim_forward(w, spec, users, items, *seqs, so.TOPK_DEFAULT, sel=shifted)
    assert not np.allclose(z3, z)


def test_dual_sequences_match_the_reference_algorithm():
    rng = np.random.default_rng(3)
    n_users, n_items, L, S = 40, 50, 12, 4
    consumed = {u: [int(i) for i in rng.integers(0, n_items, size=int(rng.integers(0, L + S + 6)))]
                for u in range(n_users)}
    consumed[0], consumed[1], consumed[2] = [], list(range(S)), list(range(L + S))
    ref = _ref_dual_seqs(n_users, consumed, n_items, L, S)
    got = recent_dual_sequences(consumed, n_users, n_items, L, S)
    indptr = np.concatenate([[0], np.cumsum([len(consumed[u]) for u in range(n_users)])]).astype(np.int64)
    idx = np.array([i for u in range(n_users) for i in consumed[u]], dtype=np.int32)
    got_csr = recent_dual_sequences_csr(ConsumedCSR(indptr, idx), n_items, L, S)
    for a, b, c in zip(ref, got, got_csr):
        assert a.dtype == b.dtype == c.dtype == np.int32
        assert (a == b).all() and (a == c).all()
    assert got[1][n_users] == 1 and got[3][n_users] == 1 and (got[0][n_users] == n_items).all()


def test_build_dual_seq_matches_the_reference_algorithm():
    rng = np.random.default_rng(4)
    n_items, L, S = 30, 9, 3
    item2id = {100 + i: i for i in range(n_items)}
    for n in list(range(1, L + S + 4)):
        seq = [int(i) for i in rng.integers(0, n_items, size=n)]
        ref = _ref_build_dual_seq(seq, n_items, L, S)
        got = build_dual_seq(seq, n_items, L, S, inner_id=True)
        for a, b in zip(ref, got):
            assert a.dtype == b.dtype and (a == b).all(), n
        raw = [100 + i for i in seq] + [7]                     # 7: unknown -> n_items
        got = build_dual_seq(raw, n_items, L, S, item2id=item2id)
        ref = _ref_build_dual_seq(seq + [n_items], n_items, L, S)
        for a, b in zip(ref, got):
            assert (a == b).all(), n


@pytest.mark.parametrize("version", ["keras", "legacy"])
@pytest.mark.parametrize("use_bn", [True, False])
def test_tf_variables_round_trip(tmp_path, version, use_bn):
    from librecommender_b200 import synthetic as syn

    rng = np.random.default_rng(5)
    spec = syn.make_spec(rng, 20, 30, [5], [7, 4], 1, 1)
    raw = syn.make_sim_weights(rng, spec, 16, 2, (24, 8), use_bn, version)
    tv = wio.sim_tf_variables(raw)
    names = wio.default_tf_names("SIM", 2, use_bn, scheme=version)
    assert names["seq_proj"] in tv and names["out_kernel"] in tv and names["first_stage_out_kernel"] in tv
    assert names["out_kernel"] == ("dense_2/kernel:0" if version == "keras" else "dense_6/kernel:0")
    np.savez(tmp_path / "m_tf_variables.npz", **tv)
    w = wio.load_reference_tf_model(str(tmp_path), "m", "SIM", 2, use_bn, num_heads=2)
    ref = wio.sim_weights(raw)
    assert w["sim_scheme"] == version and w["num_heads"] == 2
    for k in ("wq", "wk", "wv", "wo"):
        assert (w["sim_attention"][k] == ref["sim_attention"][k]).all()
    for k in ("seq_proj", "out_kernel", "user_embeds", "item_embeds", "sparse_embeds", "dense_embeds"):
        assert (np.asarray(w[k]) == np.asarray(ref[k])).all(), k
    for a, b in zip(w["mlp"]["kernels"] + w["first_stage_mlp"]["kernels"],
                    raw["mlp"]["kernels"] + raw["first_stage_mlp"]["kernels"]):
        assert (a == b).all()
    assert (w["first_stage_out_kernel"] == raw["first_stage_out_kernel"]).all()
    # lossless: writing the loaded variables again gives the same file
    tv2 = wio.sim_tf_variables(w)
    assert sorted(tv2) == sorted(tv) and all((tv2[k] == tv[k]).all() for k in tv)


def test_loader_reports_missing_and_misshaped_variables(tmp_path):
    from librecommender_b200 import synthetic as syn

    rng = np.random.default_rng(6)
    spec = syn.make_spec(rng, 20, 30, [], [], 0, 0)
    raw = syn.make_sim_weights(rng, spec, 16, 2, (24, 8), False, "keras")
    tv = wio.sim_tf_variables(raw)
    bad = dict(tv)
    del bad["multi_head_attention/key/kernel:0"]
    np.savez(tmp_path / "a_tf_variables.npz", **bad)
    with pytest.raises(KeyError, match="multi_head_attention/key/kernel:0"):
        wio.load_reference_tf_model(str(tmp_path), "a", "SIM", 2, False, num_heads=2)
    bad = dict(tv)
    bad["dense/kernel:0"] = np.zeros((16, 8), dtype=np.float32)
    np.savez(tmp_path / "b_tf_variables.npz", **bad)
    with pytest.raises(KeyError, match="dense/kernel:0.*shape"):
        wio.load_reference_tf_model(str(tmp_path), "b", "SIM", 2, False, num_heads=2)
    np.savez(tmp_path / "c_tf_variables.npz", **tv)
    with pytest.raises(KeyError, match="query/kernel:0.*shape"):      # heads read off the file: 4 heads of 4 != 2 of 8
        wio.load_reference_tf_model(str(tmp_path), "c", "SIM", 2, False, num_heads=4)


@pytest.mark.parametrize("c", so.CASES, ids=so.case_id)
def test_float32_meets_the_gpu_bound_with_margin(c):
    """The float32 graph on float64's own selection stays within a quarter of the 1e-5 bound the GPU tests use."""
    rng, spec, w, _, seqs = so.make_case(c)
    users, items, sparse, dense = so.case_rows(rng, spec, R=200)
    ref, sel, _, _ = so.sim_forward(w, spec, users, items, *seqs, so.TOPK_DEFAULT, sparse, dense, np.float64)
    got, _, _, _ = so.sim_forward(w, spec, users, items, *seqs, so.TOPK_DEFAULT, sparse, dense, np.float32, sel=sel)
    to.close(got.astype(np.float64), ref, tol=2.5e-6)


def test_cabi_rejects_out_of_envelope_shapes_before_launch():
    from librecommender_b200 import _lib

    lib = _lib.lib
    x = np.zeros(64, dtype=np.float32)
    n0 = _lib.launch_count()
    # (K, H, L, S, topk)
    bad = [(65, 1, 100, 10, 10), (16, 3, 100, 10, 10), (16, 2, 257, 10, 10), (16, 2, 100, 65, 10),
           (16, 2, 100, 10, 33), (16, 2, 8, 10, 9), (16, 2, 100, 10, 0), (16, 2, 0, 10, 1), (16, 2, 100, 0, 10)]
    for K, H, L, S, k in bad:
        rc = lib.b200_sim_attention(_lib.ptr(x), 64, _lib.ptr(x), 64, K, H, _lib.ptr(x), 300, _lib.ptr(x), _lib.ptr(x),
                                    _lib.ptr(x), L, _lib.ptr(x), 300, _lib.ptr(x), S, k, _lib.ptr(x), None, None, 5, 3, 0,
                                    _lib.ptr(x), 200, None, None)
        assert rc == -2, (K, H, L, S, k)
        rc = lib.b200_sim_pair_scores(_lib.ptr(x), _lib.ptr(x), 10, 5, _lib.ptr(x), 64, _lib.ptr(x), 300, _lib.ptr(x),
                                      _lib.ptr(x), 300, _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), 1, _lib.ptr(x),
                                      10, K, H, L, S, k, 64, 32, 0, _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), None, None,
                                      _lib.ptr(x), 0.0, _lib.ptr(x), 5, None)
        assert rc == -2, (K, H, L, S, k)
    for H1, H2, H3 in [(257, 32, 0), (64, 129, 0), (64, 32, 65), (0, 32, 0)]:
        rc = lib.b200_sim_pair_scores(_lib.ptr(x), _lib.ptr(x), 10, 5, _lib.ptr(x), 64, _lib.ptr(x), 300, _lib.ptr(x),
                                      _lib.ptr(x), 300, _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), 1, _lib.ptr(x),
                                      10, 16, 2, 100, 10, 10, H1, H2, H3, _lib.ptr(x), _lib.ptr(x), _lib.ptr(x),
                                      _lib.ptr(x), _lib.ptr(x), _lib.ptr(x), 0.0, _lib.ptr(x), 5, None)
        assert rc == -2, (H1, H2, H3)
        assert lib.b200_sim_pair_smem_bytes(16, 100, 10, 10, H1, H2, H3) == -2
    assert _lib.launch_count() == n0
    # the reference defaults fit the shared-memory opt-in of an H100 (227 KB); the whole envelope does not
    assert lib.b200_sim_pair_smem_bytes(16, 100, 10, 10, 200, 80, 0) <= 227 * 1024
    assert lib.b200_sim_pair_smem_bytes(64, 256, 64, 32, 256, 128, 64) > 227 * 1024


def test_default_names_table():
    k = wio.default_tf_names("SIM", 2, True, scheme="keras")
    assert k["sim_mha"]["attention_output"] == "multi_head_attention/attention_output/kernel:0"
    assert k["mlp"]["kernels"][0] == "second_stage_mlp/second_stage_mlp_layer1/kernel:0"
    assert k["first_stage_mlp"]["bn_in"]["mean"] == "first_stage_mlp/batch_normalization/moving_mean:0"
    g = wio.default_tf_names("SIM", 2, False, scheme="legacy")
    assert [g["sim_mha"][n] for n in ("query", "key", "value", "output")] == [
        f"dense_{i}/kernel:0" for i in range(2, 6)]
    assert g["out_bias"] == "dense_6/bias:0" and g["first_stage_out_bias"] == "dense_1/bias:0"
    with pytest.raises(ValueError):
        wio.default_tf_names("SIM", 2, False, scheme="other")
    assert tm.BN_EPS == 1e-3
