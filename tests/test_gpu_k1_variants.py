"""K1 (b200_feat_forward) kernel variants against the oracle's field embeddings: the software-pipelined field-group
kernel (default for >= 4096 rows), its cp.async staged variant, the plain field-group kernel and the lane-per-field
kernel (K = 12 takes the lane-per-field kernel under every switch setting; the generic kernel and the bulk-copy kernel
are covered by tests/test_gpu_feat_gather.py).  Concatenated rows must be bit-exact (pure copies / one multiply), the
FM sums agree to fp32 summation order; the three fast variants must agree with each other bit-for-bit on the copies.
Covers K in {4, 8, 16, 32, 12}, row counts that are no multiple of anything, tower layouts (one id field),
the all-items grid mode and more fields than one 8-step batch."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

TUNES = {"pipe": 0, "async": 8, "fieldgroup": 4, "lanefield": 2}


def _run(model, layout, users_d, items_d, R, K, F, grid_items=0, want_concat=True):
    import torch

    concat = torch.full((R, F * K), float("nan"), dtype=torch.float32, device="cuda") if want_concat else None
    pw = torch.empty((R, K), dtype=torch.float32, device="cuda")
    lin = torch.empty(R, dtype=torch.float32, device="cuda")
    ss = torch.empty((R, K), dtype=torch.float32, device="cuda")
    sq = torch.empty((R, K), dtype=torch.float32, device="cuda")
    model._feat_forward(layout, users_d, items_d, R, grid_items, concat=concat, pw=pw, lin=lin, ssum=ss, sqsum=sq)
    torch.cuda.synchronize()
    return (concat.cpu().numpy() if want_concat else None), pw.cpu().numpy(), lin.cpu().numpy(), ss.cpu().numpy(), sq.cpu().numpy()


@pytest.mark.parametrize("K,us,its,nud,nid,R", [
    (16, [7, 30, 12, 5, 9, 11, 200, 3, 17, 40], [11, 5, 40, 8, 21, 6, 90, 13, 4], 2, 3, 6007),   # F = 26
    (8, [7, 30], [11, 5, 40], 1, 0, 4099),
    (32, [50, 9, 14], [8, 300, 21, 5], 1, 2, 5001),
    (4, [6] * 20, [9] * 25, 3, 3, 8191),                                                      # F = 53, K4 = 1
    (16, [13] * 60, [7] * 55, 4, 5, 4500),                                                    # F = 126: 16 steps
    (12, [7, 30, 12], [11, 5], 1, 1, 4200),                                                   # lane-per-field only
    (32, [13] * 40, [7] * 38, 1, 1, 4100),                                                    # F = 82, K = 32: 21 steps > 16
    (4, [6] * 60, [9] * 60, 5, 5, 4300),                                                      # F = 132 fields of 16 bytes
    (8, [5] * 60, [4] * 60, 4, 4, 4097),                                                      # F = 130
    (16, [9], [4], 0, 0, 5000),                                                               # F = 4: one ragged step
])
def test_variants_match_oracle_and_each_other(K, us, its, nud, nid, R):
    import torch

    from librecommender_b200 import _lib
    from librecommender_b200.feat_models import FM
    from oracle import tf_models as tm

    rng = np.random.default_rng(K * 1000 + R)
    spec = tm.make_spec(rng, 900, 700, us, its, nud, nid)
    w = tm.make_fm_weights(rng, spec, K, True)
    model = FM(spec, w)
    users, items = rng.integers(0, 900, R), rng.integers(0, 700, R)
    sparse, dense = tm.row_features(spec, users, items)
    P, Lf = tm._stacked_embeds(tm._cast(w, np.float32), users, items, sparse, dense, np.float32)
    F = P.shape[1]
    ref_concat = P.reshape(R, F * K)
    P64 = P.astype(np.float64)
    ref_s, ref_q = P64.sum(axis=1), np.square(P64).sum(axis=1)
    ref_pw = 0.5 * (ref_s ** 2 - ref_q)
    ref_lin = Lf.astype(np.float64) @ np.asarray(w["lin_kernel"], dtype=np.float64).reshape(-1) + float(w["lin_bias"])
    u_d, i_d = torch.as_tensor(users).cuda(), torch.as_tensor(items).cuda()
    outs = {}
    try:
        for name, code in TUNES.items():
            _lib.check(_lib.lib.b200_feat_forward_tune(code))
            outs[name] = _run(model, model.spec.layout, u_d, i_d, R, K, F)
    finally:
        _lib.check(_lib.lib.b200_feat_forward_tune(0))
    scale = np.abs(ref_s).max()
    for name, (concat, pw, lin, ss, sq) in outs.items():
        np.testing.assert_array_equal(concat, ref_concat, err_msg=name)
        assert np.abs(ss - ref_s).max() <= 2e-6 * max(1.0, scale), name
        assert np.abs(sq - ref_q).max() <= 2e-6 * max(1.0, np.abs(ref_q).max()), name
        assert np.abs(pw - ref_pw).max() <= 1e-5 * max(1.0, np.abs(ref_pw).max()), name
        assert np.abs(lin - ref_lin).max() <= 1e-5 * max(1.0, np.abs(ref_lin).max()), name


@pytest.mark.parametrize("which", ["user", "item"])
def test_tower_layout_and_grid_mode(which):
    """One id field only (TwoTower towers) and the implicit all-items grid (users x every item)."""
    import torch

    from librecommender_b200 import _lib
    from librecommender_b200.feat_models import FM, TwoTower
    from oracle import tf_models as tm

    rng = np.random.default_rng(77)
    spec = tm.make_spec(rng, 5000, 4500, [8, 17, 40], [5, 9], 1, 2)
    wt = tm.make_two_tower_weights(rng, spec, 16, (32, 16), False)
    n = 5000 if which == "user" else 4500
    ids = np.arange(n)
    got = {}
    try:
        for name, code in TUNES.items():
            _lib.check(_lib.lib.b200_feat_forward_tune(code))
            got[name] = TwoTower(spec, wt, norm_embed=False).tower(which, ids).cpu().numpy()
    finally:
        _lib.check(_lib.lib.b200_feat_forward_tune(0))
    sp = spec[f"{which}_sparse_unique"][ids]
    dn = spec[f"{which}_dense_unique"][ids]
    ref = tm.tower_forward(wt, ids, sp, dn, which, False, dtype=np.float64)
    for name, v in got.items():
        assert np.abs(v - ref).max() <= 3e-5 * max(1.0, np.abs(ref).max()), name
    np.testing.assert_array_equal(got["async"], got["fieldgroup"])
    np.testing.assert_array_equal(got["pipe"], got["fieldgroup"])
    if which == "user":
        return
    # grid mode: 3 users x all 700 items of a smaller FM (rows = 3 * 700 < 4096 -> register kernel) and
    # 9 users x 700 items (6300 rows -> staged kernel) must agree with explicit pairs
    spec2 = tm.make_spec(rng, 300, 700, [7, 30], [11, 5, 40], 1, 1)
    w = tm.make_fm_weights(rng, spec2, 16, True)
    model = FM(spec2, w)
    users = rng.integers(0, 300, 9)
    u_d = torch.as_tensor(users).cuda()
    R = 9 * 700
    F = 2 + spec2["n_sparse"] + spec2["n_dense"]
    grid = _run(model, model.spec.layout, u_d, u_d, R, 16, F, grid_items=700)
    pairs_u = torch.as_tensor(np.repeat(users, 700)).cuda()
    pairs_i = torch.as_tensor(np.tile(np.arange(700), 9)).cuda()
    flat = _run(model, model.spec.layout, pairs_u, pairs_i, R, 16, F)
    for a, b in zip(grid, flat):
        np.testing.assert_array_equal(a, b)
