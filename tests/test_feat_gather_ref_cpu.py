"""The float64 reference of K1 (tests/_feat_gather_ref.py) and its per-element bounds, without a GPU:
* the reference agrees with the FM / DeepFM oracle (oracle.tf_models) on the concatenated fields, the FM logit and
  DeepFM's pairwise / linear inputs;
* every bound holds with at least 4x to spare for float32 restatements of the gather in three summation orders
  (field order, reversed, field groups + an xor-shuffle tree), on the layouts and values of
  tests/test_gpu_feat_gather.py (dense values around +-1e3, heavy cancellation in pw, both sides of elu);
* every bound is broken by seeded wrong kernels that differ by one field or one constant;
* the dispatch restatement names the family the host code picks at its thresholds."""
import numpy as np
import pytest

import _feat_gather_ref as fr

OUTS = ("ssum", "sqsum", "pw", "lin", "fm_out")
ORDERS = ("field", "reversed", "group")


@pytest.mark.parametrize("model,K,us,its,nud,nid", [
    ("fm", 16, [7, 30, 12], [11, 5, 40, 8], 1, 2),
    ("fm", 8, [5] * 20, [9] * 25, 3, 3),
    ("deepfm", 32, [50, 9, 14], [8, 300, 21], 2, 1),
    ("deepfm", 4, [13], [7], 0, 0),
])
def test_reference_matches_oracle(model, K, us, its, nud, nid):
    from oracle import tf_models as tm

    rng = np.random.default_rng(K + len(us))
    spec = tm.make_spec(rng, 90, 70, us, its, nud, nid)
    w = tm.make_fm_weights(rng, spec, K, True) if model == "fm" else tm.make_deepfm_weights(rng, spec, K, (32, 16), True)
    users, items = rng.integers(0, 91, 300), rng.integers(0, 71, 300)
    sparse, dense = tm.row_features(spec, users, items)
    w64 = tm._cast(w, np.float64)
    P, Lf = tm._stacked_embeds(w64, users, items, sparse, dense, np.float64)
    if model == "deepfm":
        w = dict(w, pw_kernel=np.ones(K, np.float32), pw_bias=np.float32(0))
    r = fr.ref(fr.case_from_spec(spec, w, K, fold_dtype=np.float64), users, items)
    np.testing.assert_array_equal(r["concat"], P.astype(np.float32).reshape(len(users), -1))
    pw = 0.5 * (np.square(P.sum(axis=1)) - np.square(P).sum(axis=1))
    np.testing.assert_allclose(r["pw"], pw, rtol=1e-12, atol=1e-12)
    lin = Lf @ w64["lin_kernel"].reshape(-1) + w64["lin_bias"]
    np.testing.assert_allclose(r["lin"], lin, rtol=1e-12, atol=1e-12)
    if model == "fm":
        want = tm.fm_forward(w, users, items, sparse, dense, dtype=np.float64)
        np.testing.assert_allclose(r["fm_out"], want, rtol=1e-11, atol=1e-12)


def _cases():
    """(name, case, users, items, kwargs) on the value ranges of the GPU tests."""
    rng = np.random.default_rng(2024)
    out = []
    c = fr.make_case(rng, 16, 5, 7, 2, 3)
    out.append(("mixed", c, rng.integers(0, 301, 700), rng.integers(0, 401, 700), {}))
    c = fr.make_case(rng, 32, 128, 128, 0, 0)
    out.append(("wide", c, rng.integers(0, 301, 200), rng.integers(0, 401, 200), {}))
    c = fr.make_case(rng, 8, 2, 2, 3, 4, dense_scale=1e3, dense_row_perm=True)
    out.append(("dense_1e3", c, rng.integers(0, 301, 700), rng.integers(0, 401, 700), {}))
    c = fr.make_case(rng, 7, 0, 0, 60, 68, id_mask=0)
    out.append(("dense_only", c, rng.integers(0, 301, 400), rng.integers(0, 401, 400), {}))
    # heavy cancellation: every field paired with its negation, so ssum ~ 0 and pw ~ -sqsum / 2
    c = fr.make_case(rng, 12, 6, 6, 0, 0, vocab=64)
    c["sparse_embeds"] = np.concatenate([c["sparse_embeds"][:32], -c["sparse_embeds"][:32]])
    c["user_sparse_unique"] = np.concatenate([c["user_sparse_unique"][:, :3] % 32, c["user_sparse_unique"][:, :3] % 32 + 32], 1)
    c["item_sparse_unique"] = np.concatenate([c["item_sparse_unique"][:, :3] % 32, c["item_sparse_unique"][:, :3] % 32 + 32], 1)
    c["sparse_col"] = np.array([0, 1, 2, 3, 4, 5] * 2, np.int32)
    c["sparse_side"] = np.array([0] * 6 + [1] * 6, np.int32)
    c["id_mask"] = 0
    c["lin_kernel"] = c["lin_kernel"][:12]
    out.append(("cancel", c, rng.integers(0, 301, 500), rng.integers(0, 401, 500), {}))
    c = fr.make_case(rng, 4, 3, 3, 1, 1, n_users=40, n_items=30)
    out.append(("grid", c, rng.integers(0, 41, 12), None, dict(R=229, grid_items=31, row_offset=57)))
    c = fr.make_case(rng, 16, 5, 4, 2, 2)
    sr = rng.integers(0, 500, (600, 9)).astype(np.int32)
    dr = (rng.standard_normal((600, 4)) * 30).astype(np.float32)
    out.append(("explicit", c, rng.integers(0, 301, 600), rng.integers(0, 401, 600),
                dict(sparse_rows=sr, dense_rows=dr)))
    return out


CASES = _cases()


@pytest.mark.parametrize("bn", [True, False])
@pytest.mark.parametrize("name", [c[0] for c in CASES])
def test_bounds_hold_with_margin(name, bn):
    _, case, users, items, kw = next(c for c in CASES if c[0] == name)
    r = fr.ref(case, users, items, bn=bn, **kw)
    if name == "cancel":
        assert np.abs(r["ssum"]).max() < 1e-12 * np.abs(r["sqsum"]).max() + 1e-30
    if name in ("mixed", "dense_1e3"):
        assert (r["z"] < 0).mean() > 0.2 and (r["z"] > 0).mean() > 0.2      # both sides of elu
    for order in ORDERS:
        got = fr.restate32(case, users, items, bn=bn, order=order, **kw)
        np.testing.assert_array_equal(got["concat"], r["concat"])
        for o in OUTS:
            ratio = fr.worst(got[o], r[o], r["bound"][o])
            assert ratio <= 0.25, (name, order, o, ratio)


MUTANTS = {
    "drop_field": OUTS,
    "no_bn_shift": ("fm_out",),
    "relu": ("fm_out",),
    "ignore_row_offset": OUTS,
    "dense_twice": ("ssum", "sqsum", "pw", "fm_out"),
}


@pytest.mark.parametrize("mutant", list(MUTANTS))
def test_bounds_catch_one_field_errors(mutant):
    by_name = {c[0]: c for c in CASES}
    name = {"ignore_row_offset": "grid", "dense_twice": "dense_1e3"}.get(mutant, "mixed")
    _, case, users, items, kw = by_name[name]
    r = fr.ref(case, users, items, **kw)
    bad = fr.restate32(case, users, items, mutate=mutant, **kw)
    for o in MUTANTS[mutant]:
        assert fr.worst(bad[o], r[o], r["bound"][o]) > 1.0, (mutant, o)


def test_bounds_catch_dense_twice_in_lin():
    """The dense feature's linear term: a mutated x * x * dense_linear breaks the lin bound."""
    _, case, users, items, kw = next(c for c in CASES if c[0] == "dense_1e3")
    r = fr.ref(case, users, items)
    u, it = fr.row_ids(users, items, len(users))
    _, Lf, dense = fr.fields(case, u, it)
    x = np.stack([case["user_dense_unique"][u, c] if s == 0 else case["item_dense_unique"][it, c]
                  for s, c in zip(case["dense_side"], case["dense_col"])], 1).astype(np.float64)
    Lf[:, dense] *= x
    bad = Lf @ case["lin_kernel"].astype(np.float64)[: Lf.shape[1]] + float(case["lin_bias"])
    assert fr.worst(bad, r["lin"], r["bound"]["lin"]) > 1.0


@pytest.mark.parametrize("args,want", [
    ((16, 0, 10), ("none", None)),
    ((7, 5000, 10), ("generic", None)),
    ((64, 5000, 10), ("generic", None)),
    ((16, 5000, 10, False), ("generic", None)),
    ((12, 5000, 10), ("lanefield", 3)),
    ((16, 4095, 10), ("fieldgroup", 4)),
    ((16, 4096, 10), ("pipe", 4)),
    ((32, 4096, 64), ("pipe", 8)),
    ((32, 4096, 65), ("fieldgroup", 8)),
    ((32, 4096, 64, True, False, 8), ("async", 8)),
    ((32, 4096, 65, True, False, 8), ("fieldgroup", 8)),
    ((16, 4096, 10, True, True), ("fieldgroup", 4)),
    ((16, 4096, 10, True, False, 4), ("fieldgroup", 4)),
    ((16, 4096, 10, True, False, 2), ("lanefield", 4)),
    ((16, 2047, 10, True, False, 1), ("fieldgroup", 4)),
    ((16, 2048, 10, True, False, 1), ("tma", 4)),
    ((16, 2048, 10, True, True, 1), ("tma", 4)),
    ((12, 2048, 10, True, False, 1), ("lanefield", 3)),
    ((32, 2048, 258, True, False, 1), ("tma", 8)),
])
def test_expected_kernel(args, want):
    assert fr.expected_kernel(*args) == want


@pytest.mark.parametrize("name,want", [
    ("void b200::feat::feat_forward_pipe_kernel<4>(b200_feat_layout, b200_feat_tables, long const*)", ("pipe", 4)),
    ("void b200::feat::feat_forward_kernel(b200_feat_layout, b200_feat_tables, long const*)", ("generic", None)),
    ("_ZN4b2004feat23feat_forward_tma_kernelILi8EEEv16b200_feat_layout", ("tma", 8)),
    ("_ZN4b2004feat19feat_forward_kernelE16b200_feat_layout", ("generic", None)),
    ("void b200::feat::feat_backward_kernel(b200_feat_layout)", None),
])
def test_kernel_name_parser(name, want):
    assert fr.kernel_of(name) == want
