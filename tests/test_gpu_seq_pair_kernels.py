"""The all-items scorers of the sequence models, each C-ABI entry point called directly and compared with its float64
definition (tests/_seq_pair_kernels_ref.py):

* ``b200_transformer_pair_scores`` past its grid cap (min(tiles, 2 * SMs / B) blocks per user row, so each block runs
  several 256-item tiles and its cp.async chunk stream crosses tiles), at D and H1 giving partial, exact and maximal
  32-column chunk counts, H3 = 0 / 1 / 32, T = 1 / 10 / 64, every length class (-3, 0, 1, T, T + 5), the largest
  shape that fits, and NaN padding past D / H1 that must never be read; ``b200_transformer_target_attention`` in both
  addressing modes.
* ``b200_sim_pair_scores`` on each of its KP = 16 / 32 / 48 / 64 templates (K off a multiple of 16 included), past
  its grid cap, at L = 256 / topk = 32 / S = 64, with exact GSU ties at the cut and a NaN item in the long sequences;
  ``b200_sim_attention``'s ``gsu_pos`` against the float64 selection, and its two addressing modes.
* ``b200_autoint_grid`` past the item stride and the user stride, on a ``field_map`` that interleaves user and item
  fields out of order, against float64 and against ``b200_autoint_rows`` bit for bit.

Every call writes into NaN-filled outputs with a leading dimension past N (no column >= N may change) and repeats
bit for bit, and a pair's score does not depend on where the pair sits: rerun through offset pointers with N = 1
and B = 1 it gives the same bits.  Bounds per element: C * u * mag with mag from the reference module, C calibrated in
tests/test_seq_pair_kernels_cpu.py."""
from __future__ import annotations

import numpy as np
import pytest

import _seq_pair_kernels_ref as sp
from test_gpu_rank_kernels import _dev, _lib, _sample_items, _sync

pytestmark = pytest.mark.gpu

F32, F64 = np.float32, np.float64
C_TFM = 2.0          # Transformer pair scores and rows (tests/test_seq_pair_kernels_cpu.py)
C_SIM_ROWS = 2.0     # SIM rows
C_SIM_PAIR = 0.5     # SIM pair scores: mag's worst-case chain factors over three layers sit ~1000x above float32
C_AI = 2.0           # AutoInt
TP_ITEMS = 256       # items per Transformer pair tile
SP_THREADS = 256     # items per SIM pair block iteration


def _sms():
    import torch

    return torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count


def _nan(shape):
    import torch

    return torch.full(shape, float("nan"), dtype=torch.float32, device="cuda")


def _bits(x):
    return np.ascontiguousarray(x, dtype=F32).view(np.uint32)


def _check(got, ref, mag, C, what):
    err = np.abs(got.astype(F64) - ref)
    bound = C * sp.U * mag
    assert np.isfinite(got).all(), f"{what}: non-finite output"
    worst = np.unravel_index(np.argmax(err / bound), err.shape)
    assert (err <= bound).all(), f"{what}: err {err[worst]:.3g} > bound {bound[worst]:.3g} at {worst}"


def _pass_items(N, per_pass, tile, rng, n_mid=1500):
    """The first and the last tile of every pass of a grid-stride loop, plus ``_sample_items``."""
    parts = [_sample_items(N, per_pass, rng, n_mid)]
    for s in range(0, N, per_pass):
        e = min(s + per_pass, N)
        parts += [np.arange(s, min(s + tile, e)), np.arange(max(e - tile, s), e)]
    return np.unique(np.concatenate(parts))


def _upload(c):
    return {k: _dev(v) for k, v in c.items() if isinstance(v, np.ndarray)}


# =====================================================================================================================
# Transformer
# =====================================================================================================================
def _tfm_call(c, dv, B, N, out, lds, n0=0, b0=0, **over):
    L = _lib()
    T, D, H1, H2, H3 = (over.get(k, c[k]) for k in ("T", "D", "H1", "H2", "H3"))
    Qi, Pi = dv["Qi"], dv["Pi"]
    return L.lib.b200_transformer_pair_scores(
        L.ptr(Qi[n0:]), over.get("ldq", Qi.stride(0)), N, L.ptr(dv["S"][b0:]), L.ptr(dv["Vp"][b0:]),
        L.ptr(dv["Pu"][b0:]), L.ptr(dv["lens"][b0:]), B, L.ptr(Pi[n0:]), over.get("ldpi", Pi.stride(0)), T, D, H1,
        H2, H3, L.ptr(dv["W2"]), L.ptr(dv["b2"]), L.ptr(dv.get("W3")), L.ptr(dv.get("b3")), L.ptr(dv["w_out"]),
        c["b_out"], L.ptr(out), lds, L.current_stream())


def _tfm_run(c, dv, B, N, lds, **kw):
    out = _nan((B, lds))
    rc = _tfm_call(c, dv, B, N, out, lds, **kw)
    assert rc == 0, _lib().lib.b200_last_error()
    _sync()
    got = out.cpu().numpy()
    assert np.isnan(got[:, N:]).all(), "wrote past N"
    return got[:, :N]


TFM_CASES = [  # (B, N, T, D, H1, H2, H3)
    (8, 3 * 33 * 256 + 101, 10, 33, 33, 64, 1),     # past the grid cap: 33 blocks per row on 132 SMs, 100 tiles
    (5, 1000, 1, 7, 1, 1, 0),                       # one key, one partial chunk each
    (5, 700, 64, 128, 64, 64, 32),                  # the largest shape that fits: 208 128 B
    (5, 600, 10, 32, 256, 64, 32),                  # exact chunks, the maximal Pi chunk count
    (5, 513, 64, 33, 31, 1, 1),
    (6, 300, 10, 128, 32, 64, 0),
]


@pytest.mark.parametrize("B,N,T,D,H1,H2,H3", TFM_CASES)
def test_transformer_pair_scores(B, N, T, D, H1, H2, H3):
    L = _lib()
    assert L.lib.b200_transformer_pair_smem_bytes(T, D, H1) > 0
    c = sp.make_tfm_case(B, N, T, D, H1, H2, H3, seed=N + D + H1, ldq_pad=3, ldpi_pad=5)
    dv = _upload(c)
    lds = N + 7
    got = _tfm_run(c, dv, B, N, lds)
    np.testing.assert_array_equal(_bits(got), _bits(_tfm_run(c, dv, B, N, lds)), err_msg="repeat")
    tiles = -(-N // TP_ITEMS)
    gx = min(tiles, max(1, 2 * _sms() // B))
    if N > 20_000:
        assert -(-tiles // gx) >= 3, "the case must run at least three passes"
    rng = np.random.default_rng(H1)
    items = _pass_items(N, gx * TP_ITEMS, TP_ITEMS, rng)
    for b in range(B):
        ref, mag = sp.tfm_pair_ref(c, b, items)
        _check(got[b, items], ref, mag, C_TFM, f"transformer pair b={b} len={c['lens'][b]}")
    # the same pairs alone: one item through offset Qi / Pi, then one user through offset S / Vp / Pu / lens
    for n in np.unique(np.r_[0, N - 1, rng.integers(0, N, 6), min(N - 1, TP_ITEMS * gx), min(N - 1, TP_ITEMS - 1)]):
        one = _tfm_run(c, dv, B, 1, 2, n0=n)
        np.testing.assert_array_equal(_bits(one[:, 0]), _bits(got[:, n]), err_msg=f"item {n} alone")
        for b in (0, B - 1):
            one = _tfm_run(c, dv, 1, 1, 1, n0=n, b0=b)
            np.testing.assert_array_equal(_bits(one[0]), _bits(got[b, n:n + 1]), err_msg=f"pair ({b}, {n}) alone")


def test_transformer_pair_rejections_write_nothing():
    L = _lib()
    c = sp.make_tfm_case(2, 40, 10, 32, 64, 32, 8, seed=1)
    dv = _upload(c)
    assert L.lib.b200_transformer_pair_smem_bytes(64, 128, 128) == 241_152
    big = sp.make_tfm_case(1, 8, 64, 128, 128, 8, 0, seed=2)
    dvb = _upload(big)
    out = _nan((2, 48))
    assert _tfm_call(big, dvb, 1, 8, out, 48) == -2, "over the shared-memory opt-in"
    assert b"shared memory" in L.lib.b200_last_error()
    for B, kw in ((65536, {}), (2, dict(H1=257)), (2, dict(H2=65)), (2, dict(H2=129)), (2, dict(H3=33)),
                  (2, dict(H3=65)), (2, dict(ldq=31)), (2, dict(ldpi=63))):
        assert _tfm_call(c, dv, B, 40, out, 48, **kw) == -2, (B, kw)
    assert _tfm_call(c, dv, 2, 40, out, 39) == -2, "lds < N"
    rc = L.lib.b200_transformer_pair_scores(
        L.ptr(dv["Qi"]), dv["Qi"].stride(0), 40, L.ptr(dv["S"]), L.ptr(dv["Vp"]), L.ptr(dv["Pu"]), L.ptr(dv["lens"]),
        2, L.ptr(dv["Pi"]), dv["Pi"].stride(0), 10, 32, 64, 32, 8, L.ptr(dv["W2"]), L.ptr(dv["b2"]), None, None,
        L.ptr(dv["w_out"]), 0.0, L.ptr(out), 48, L.current_stream())
    assert rc == -2, "third layer weights missing"
    _sync()
    assert np.isnan(out.cpu().numpy()).all(), "a rejected call wrote"


def _tfm_rows(dv, T, D, slot, items, n, grid_items, row_offset, ldo):
    L = _lib()
    out = _nan((n, ldo))
    rc = L.lib.b200_transformer_target_attention(
        L.ptr(dv["Qi"]), dv["Qi"].stride(0), L.ptr(dv["S"]), T, D, L.ptr(dv["lens"]), L.ptr(slot), L.ptr(items), n,
        grid_items, row_offset, L.ptr(out), ldo, L.current_stream())
    assert rc == 0, L.lib.b200_last_error()
    _sync()
    got = out.cpu().numpy()
    assert np.isnan(got[:, D:]).all(), "wrote past D"
    return got[:, :D]


@pytest.mark.parametrize("T,D", [(1, 7), (10, 33), (64, 128), (40, 32)])
def test_transformer_target_attention_rows(T, D):
    """Both addressing modes: grid_items + row_offset (mid-slot, n over several slots) equals the explicit
    slot_of_row / items form bit for bit, and both are within the float64 bound."""
    B, G = 7, 97
    c = sp.make_tfm_case(B, G, T, D, 8, 8, 0, seed=T * D, ldq_pad=3)
    dv = _upload(c)
    row_offset, n = G + 41, 4 * G + 13                 # slot 1 from item 41 to slot 5 item 53
    r = np.arange(n) + row_offset
    slots, items = (r // G).astype(np.int32), (r % G).astype(np.int64)
    grid = _tfm_rows(dv, T, D, None, None, n, G, row_offset, D + 3)
    expl = _tfm_rows(dv, T, D, _dev(slots), _dev(items), n, 0, 0, D + 3)
    np.testing.assert_array_equal(_bits(grid), _bits(expl))
    np.testing.assert_array_equal(_bits(grid), _bits(_tfm_rows(dv, T, D, None, None, n, G, row_offset, D + 3)))
    ref, mag = sp.tfm_rows_ref(c["Qi"], c["S"], c["lens"], slots, items)
    _check(grid, ref, mag, C_TFM, f"transformer rows T={T} D={D}")
    # explicit rows in any order, repeated slots
    rng = np.random.default_rng(D)
    slots2 = rng.integers(0, B, 300).astype(np.int32)
    items2 = rng.integers(0, G, 300).astype(np.int64)
    got = _tfm_rows(dv, T, D, _dev(slots2), _dev(items2), 300, 0, 0, D)
    ref, mag = sp.tfm_rows_ref(c["Qi"], c["S"], c["lens"], slots2, items2)
    _check(got, ref, mag, C_TFM, f"transformer explicit rows T={T} D={D}")


# =====================================================================================================================
# SIM
# =====================================================================================================================
def _sim_call(c, dv, B, N, out, lds, n0=0, b0=0, **over):
    L = _lib()
    H1, H2, H3 = (over.get(k, c[k]) for k in ("H1", "H2", "H3"))
    return L.lib.b200_sim_pair_scores(
        L.ptr(dv["GpT"][:, n0:]), L.ptr(dv["QpT"][:, n0:]), over.get("ldt", dv["GpT"].stride(0)), N, L.ptr(dv["Gp"]),
        dv["Gp"].stride(0), L.ptr(dv["long_seqs"][b0:]), over.get("ld_long", dv["long_seqs"].stride(0)),
        L.ptr(dv["long_lens"][b0:]), L.ptr(dv["short_seqs"][b0:]), dv["short_seqs"].stride(0),
        L.ptr(dv["short_lens"][b0:]), L.ptr(dv["Kl"][b0:]), L.ptr(dv["Vl"][b0:]), L.ptr(dv["Pu"][b0:]), B,
        L.ptr(dv["PiT"][:, n0:]), over.get("ldpi", dv["PiT"].stride(0)), c["K"], c["H"], c["L"], c["S"], c["topk"],
        H1, H2, H3, L.ptr(dv["W_att"]), L.ptr(dv["W2"]), L.ptr(dv["b2"]),
        None if over.get("no_w3") else L.ptr(dv.get("W3")), None if over.get("no_w3") else L.ptr(dv.get("b3")),
        L.ptr(dv["w_out"]), c["b_out"], L.ptr(out), lds, L.current_stream())


def _sim_run(c, dv, B, N, lds, **kw):
    out = _nan((B, lds))
    rc = _sim_call(c, dv, B, N, out, lds, **kw)
    assert rc == 0, _lib().lib.b200_last_error()
    _sync()
    got = out.cpu().numpy()
    assert np.isnan(got[:, N:]).all(), "wrote past N"
    return got[:, :N]


SIM_CASES = [  # (B, N, K, H, L, S, topk, H1, H2, H3)
    (6, 3 * 33 * 256 + 77, 20, 4, 48, 12, 10, 40, 24, 8),   # past the grid cap: SMs / B blocks per row; KP = 32
    (6, 600, 16, 2, 256, 64, 32, 33, 17, 5),                # the longest sequences and selection: 170 880 B
    (6, 700, 33, 3, 40, 10, 12, 64, 32, 0),                 # KP = 48 from K = 33
    (6, 500, 48, 4, 64, 8, 8, 64, 32, 8),                   # K = 48: 187 648 B
    (6, 400, 64, 2, 32, 8, 8, 32, 16, 0),                   # KP = 64
    (9, 300, 8, 1, 24, 5, 6, 128, 128, 64),                 # the widest H2 / H3
]


@pytest.mark.parametrize("B,N,K,H,L,S,topk,H1,H2,H3", SIM_CASES)
def test_sim_pair_scores(B, N, K, H, L, S, topk, H1, H2, H3):
    import torch

    lib = _lib().lib
    smem = lib.b200_sim_pair_smem_bytes(K, L, S, topk, H1, H2, H3)
    assert 0 < smem <= torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    c = sp.make_sim_case(B, N, K, H, L, S, topk, H1, H2, H3, seed=N + K)
    dv = _upload(c)
    lds = N + 5
    got = _sim_run(c, dv, B, N, lds)
    np.testing.assert_array_equal(_bits(got), _bits(_sim_run(c, dv, B, N, lds)), err_msg="repeat")
    blocks = -(-N // SP_THREADS)
    gx = min(blocks, max(1, _sms() // B))
    if N > 20_000:
        assert -(-blocks // gx) >= 3, "the case must run at least three passes"
    rng = np.random.default_rng(K)
    items = _pass_items(N, gx * SP_THREADS, SP_THREADS, rng)
    assert sp.gsu_ties_at_cut(c, 3, items).any(), "user 3 must have exact GSU ties at the cut"
    for b in range(B):
        ref, mag = sp.sim_pair_ref(c, b, items)
        _check(got[b, items], ref, mag, C_SIM_PAIR, f"sim pair b={b} llen={c['long_lens'][b]} slen={c['short_lens'][b]}")
    for n in np.unique(np.r_[0, N - 1, rng.integers(0, N, 6), min(N - 1, SP_THREADS * gx)]):
        one = _sim_run(c, dv, B, 1, 1, n0=n)
        np.testing.assert_array_equal(_bits(one[:, 0]), _bits(got[:, n]), err_msg=f"item {n} alone")
        for b in (0, 1, B - 1):
            one = _sim_run(c, dv, 1, 1, 1, n0=n, b0=b)
            np.testing.assert_array_equal(_bits(one[0]), _bits(got[b, n:n + 1]), err_msg=f"pair ({b}, {n}) alone")


def test_sim_pair_rejections_write_nothing():
    L = _lib()
    c = sp.make_sim_case(2, 40, 16, 2, 32, 8, 8, 64, 32, 8, seed=3)
    dv = _upload(c)
    out = _nan((2, 48))
    for B, kw in ((65536, {}), (2, dict(H1=257)), (2, dict(H2=129)), (2, dict(H3=65)), (2, dict(ldt=39)),
                  (2, dict(ldpi=39)), (2, dict(ld_long=31)), (2, dict(no_w3=True))):
        assert _sim_call(c, dv, B, 40, out, 48, **kw) == -2, (B, kw)
    assert _sim_call(c, dv, 2, 40, out, 39) == -2, "lds < N"
    _sync()
    assert np.isnan(out.cpu().numpy()).all(), "a rejected call wrote"


def _sim_rows(c, dv, slot, items, n, grid_items, row_offset, ldo):
    import torch

    L = _lib()
    K, k = c["K"], c["topk"]
    out = _nan((n, ldo))
    pos = torch.full((n * k + 5,), -7, dtype=torch.int32, device="cuda")
    rc = L.lib.b200_sim_attention(
        L.ptr(dv["Gp"]), dv["Gp"].stride(0), L.ptr(dv["Qp"]), dv["Qp"].stride(0), K, c["H"], L.ptr(dv["long_seqs"]),
        dv["long_seqs"].stride(0), L.ptr(dv["long_lens"]), L.ptr(dv["Kl"]), L.ptr(dv["Vl"]), c["L"],
        L.ptr(dv["short_seqs"]), dv["short_seqs"].stride(0), L.ptr(dv["short_lens"]), c["S"], k, L.ptr(dv["Wo"]),
        L.ptr(slot), L.ptr(items), n, grid_items, row_offset, L.ptr(out), ldo, L.ptr(pos), L.current_stream())
    assert rc == 0, L.lib.b200_last_error()
    _sync()
    got, pos = out.cpu().numpy(), pos.cpu().numpy()
    assert np.isnan(got[:, 2 * K:]).all(), "wrote past 2K"
    assert (pos[n * k:] == -7).all(), "wrote past the selections"
    return got[:, :2 * K], pos[:n * k].reshape(n, k)


@pytest.mark.parametrize("case", [1, 2, 3, 4], ids=lambda i: "K{}-L{}".format(SIM_CASES[i][2], SIM_CASES[i][4]))
def test_sim_attention_rows(case):
    """gsu_pos equals the float64 selection on every row, [o Wo || s] is within the bound, and the grid addressing
    (row_offset mid-slot, rows over several slots) equals the explicit rows bit for bit."""
    B, _, K, H, L, S, topk, H1, H2, H3 = SIM_CASES[case]
    G = 150
    c = sp.make_sim_case(B, G, K, H, L, S, topk, H1, H2, H3, seed=G + K)
    dv = _upload(c)
    row_offset, n = G + 77, 4 * G + 5                  # slot 1 item 77 .. slot 5 item 81
    r = np.arange(n) + row_offset
    slots, items = (r // G).astype(np.int32), (r % G).astype(np.int64)
    grid, gpos = _sim_rows(c, dv, None, None, n, G, row_offset, 2 * K + 3)
    expl, epos = _sim_rows(c, dv, _dev(slots), _dev(items), n, 0, 0, 2 * K)
    np.testing.assert_array_equal(_bits(grid), _bits(expl))
    np.testing.assert_array_equal(gpos, epos)
    ref, mag, sel = sp.sim_rows_ref(c, slots, items)
    np.testing.assert_array_equal(gpos, sel)
    _check(grid, ref, mag, C_SIM_ROWS, f"sim rows K={K} L={L}")
    nan_item = c["Gp"].shape[0] - 1
    assert not (c["long_seqs"][slots[:, None], gpos] == nan_item).any(), "the NaN item was selected"
    assert sp.gsu_ties_at_cut(c, 3, items[slots == 3]).any(), "user 3 must have exact GSU ties at the cut"


# =====================================================================================================================
# AutoInt
# =====================================================================================================================
def _ai_setup(B, N, K, H, hds, field_map, n_user_slots, n_item_slots, seed, pad=5):
    rng = np.random.default_rng(seed)
    Xu = np.full((B, n_user_slots * K + pad), np.nan, F32)
    Xu[:, :n_user_slots * K] = rng.normal(0.0, 0.7, (B, n_user_slots * K))
    Xi = np.full((N, n_item_slots * K + pad), np.nan, F32)
    Xi[:, :n_item_slots * K] = rng.normal(0.0, 0.7, (N, n_item_slots * K))
    w, layers = sp.autoint_weights(rng, K, H, hds)
    F = len(field_map)
    w_out = rng.normal(0.0, 1.0 / np.sqrt(F * K), F * K).astype(F32)
    return Xu, Xi, w, layers, w_out, float(F32(0.0625))


def _ai_grid(Xu_d, Xi_d, B, N, fm_d, F, K, H, hds, w_d, wo_d, b_out, res, lds):
    L = _lib()
    out = _nan((B, lds))
    hd = np.asarray(hds, np.int32)           # host array: kept alive across the call
    rc = L.lib.b200_autoint_grid(L.ptr(Xu_d), Xu_d.stride(0), B, L.ptr(Xi_d), Xi_d.stride(0), N, L.ptr(fm_d), F, K, H,
                                 len(hds), L.ptr(hd), L.ptr(w_d), L.ptr(wo_d), b_out, int(res), L.ptr(out), lds,
                                 L.current_stream())
    assert rc == 0, L.lib.b200_last_error()
    _sync()
    got = out.cpu().numpy()
    assert np.isnan(got[:, N:]).all(), "wrote past N"
    return got[:, :N]


def _ai_passes(N, B, F, K, H, hds):
    ld = lambda n: n | 1  # noqa: E731
    warp_bytes = 4 * (F * ld(K) + 3 * F * ld(max(H * h for h in hds)) + 32 * ld(F))
    warps = max(1, min(8, 96 * 1024 // warp_bytes))
    cap = _sms() * 32
    gx = min(-(-N // warps), cap)
    gy = min(B, max(1, cap // gx), 65535)
    return warps, gx, gy


AI_CASES = [  # (B, N, K, H, hds, residual, field_map, user slots, item slots)
    (2, None, 8, 2, (4,), True, [-2, 1, -1, 0, -3, 2], 3, 3),                       # items past the item stride
    (9000, 3, 8, 2, (4, 3), False, [1, -1, 0], 2, 1),                               # users past cap / gx
    (5, 400, 16, 2, (8, 4), True, [-1, 3, -4, 0, 2, -2, -3, 1], 4, 4),
]


@pytest.mark.parametrize("B,N,K,H,hds,res,field_map,nu,ni", AI_CASES)
def test_autoint_grid(B, N, K, H, hds, res, field_map, nu, ni):
    import torch

    L = _lib()
    F = len(field_map)
    if N is None:
        N = 3 * _sms() * 32 * 8 + 37
    Xu, Xi, w, layers, w_out, b_out = _ai_setup(B, N, K, H, hds, field_map, nu, ni, seed=B + N)
    Xu_d, Xi_d, fm_d, w_d, wo_d = _dev(Xu), _dev(Xi), _dev(np.asarray(field_map, np.int32)), _dev(w), _dev(w_out)
    lds = N + 3
    got = _ai_grid(Xu_d, Xi_d, B, N, fm_d, F, K, H, hds, w_d, wo_d, b_out, res, lds)
    np.testing.assert_array_equal(_bits(got), _bits(_ai_grid(Xu_d, Xi_d, B, N, fm_d, F, K, H, hds, w_d, wo_d, b_out,
                                                             res, lds)), err_msg="repeat")
    warps, gx, gy = _ai_passes(N, B, F, K, H, hds)
    item_passes, user_passes = -(-N // (gx * warps)), -(-B // gy)
    rng = np.random.default_rng(F)
    if B > 1000:
        assert user_passes >= 3, "the case must stride over users at least three times"
        users = _pass_items(B, gy, 8, rng, n_mid=300)
        items = np.arange(N)
    else:
        if N > 20_000:
            assert item_passes >= 3, "the case must stride over items at least three times"
        users = np.arange(B)
        items = _pass_items(N, gx * warps, 64, rng, n_mid=1500)
    uu, ii = np.repeat(users, len(items)), np.tile(items, len(users))
    X = sp.autoint_block(Xu, Xi, field_map, K, uu, ii)
    ref, mag = sp.autoint_ref(X, layers, w_out, b_out, res)
    _check(got[uu, ii], ref, mag, C_AI, f"autoint F={F} K={K}")
    # the same pairs through b200_autoint_rows on the materialised block: bit for bit
    pick = rng.choice(len(uu), size=min(len(uu), 4000), replace=False)
    Xr = X[pick].reshape(len(pick), F * K)
    Xr_d = _dev(Xr)
    out = torch.empty(len(pick), dtype=torch.float32, device="cuda")
    hd = np.asarray(hds, np.int32)
    rc = L.lib.b200_autoint_rows(L.ptr(Xr_d), F * K, len(pick), F, K, H, len(hds), L.ptr(hd),
                                 L.ptr(w_d), L.ptr(wo_d), b_out, int(res), L.ptr(out), L.current_stream())
    assert rc == 0, L.lib.b200_last_error()
    _sync()
    np.testing.assert_array_equal(_bits(out.cpu().numpy()), _bits(got[uu[pick], ii[pick]]))
    # one pair alone through offset Xu / Xi pointers
    for p in pick[:4]:
        one = _ai_grid(Xu_d[int(uu[p]):], Xi_d[int(ii[p]):], 1, 1, fm_d, F, K, H, hds, w_d, wo_d, b_out, res, 1)
        np.testing.assert_array_equal(_bits(one[0]), _bits(got[uu[p], ii[p]:ii[p] + 1]))


# =====================================================================================================================
# the models' 65 535-user chunks
# =====================================================================================================================
def _chunk_check(model, n_users, seed):
    import torch

    rng = np.random.default_rng(seed)
    ids = rng.integers(0, n_users + 1, 65535 + 6)
    ids[65535:] = [n_users, 0, 1, 2, ids[7], ids[65534]]
    u = torch.as_tensor(ids, device=model.device)
    scores = model.score_all_items(u).cpu().numpy()
    assert np.isfinite(scores).all()
    for r in range(65535, len(ids)):
        one = model.score_all_items(u[r:r + 1]).cpu().numpy()
        np.testing.assert_array_equal(_bits(scores[r]), _bits(one[0]), err_msg=f"row {r} (user {ids[r]})")


def test_transformer_score_all_items_past_65535_users():
    import _transformer_oracle as to
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import Transformer

    _, spec, w, seqs, lens = to.make_case(to.CASES[0], n_users=40, n_items=5, T=8)
    model = Transformer(spec, wio.transformer_weights(w), seqs, lens)
    assert model._hoistable()
    _chunk_check(model, 40, 1)


def test_sim_score_all_items_past_65535_users():
    import _sim_oracle as so
    from librecommender_b200 import weights_io as wio
    from librecommender_b200.feat_models import SIM

    _, spec, w, _, seqs = so.make_case(so.CASES[0], n_users=40, n_items=5, L=16, S=4, k=4)
    model = SIM(spec, wio.sim_weights(w), *seqs, search_topk=4)
    assert model._hoistable()
    _chunk_check(model, 40, 2)
