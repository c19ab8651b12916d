"""GraphSage / PinSage inference without a GPU: the float64 oracle of ``tests/_sage_oracle.py`` against the reference's
recorded outputs (``tests/golden/sage.npz``), the oracle's walker rules against the reference's own sampling on the
same Python ``random`` streams, the engines' validation errors, the C-ABI rejections and symbols, and the ``sage=True``
drop-in wiring."""
import ctypes
import os
import random
import types

import numpy as np
import pytest

import _sage_oracle as orc

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "sage.npz")
CASES = [(data, kind, paradigm) for data in ("pure", "feat") for kind in ("graphsage", "pinsage")
         for paradigm in ("i2i", "u2i")]


def golden():
    return np.load(GOLDEN)


def consumed_dict(indptr, idx):
    return {k: idx[indptr[k]:indptr[k + 1]].tolist() for k in range(len(indptr) - 1)}


def data_info(z, data):
    """The data-info pieces the engines read, as a dict, from the golden."""
    n_u, n_i = (int(x) for x in z[f"{data}_shape"])
    di = dict(n_users=n_u, n_items=n_i,
              user_consumed=consumed_dict(z[f"{data}_uc_indptr"], z[f"{data}_uc_items"]),
              item_consumed=consumed_dict(z[f"{data}_ic_indptr"], z[f"{data}_ic_users"]))
    for side in ("user", "item"):
        for kind in ("sparse", "dense"):
            di[f"{side}_{kind}_col_index"] = z[f"{data}_{side}_{kind}_col_index"].tolist()
            key = f"{data}_{side}_{kind}_unique"
            di[f"{side}_{kind}_unique"] = z[key] if key in z.files else None
    return di


def state_dict(z, case):
    """The case's state dict; a table stored by rows (``sd_rows__``) is rebuilt at full size, zeros elsewhere."""
    pre = f"{case}_sd__"
    sd = {k[len(pre):]: z[k] for k in z.files if k.startswith(pre)}
    n_u, n_i = (int(x) for x in z[f"{case.split('_')[0]}_shape"])
    for key, n in (("item_embeds.weight", n_i), ("user_embeds.weight", n_u)):
        rows_key = f"{case}_sd_rows__{key}"
        if rows_key in z.files:
            full = np.zeros((n, sd[key].shape[1]), dtype=sd[key].dtype)
            full[z[rows_key]] = sd[key]
            sd[key] = full
    return sd


def message(z, case, kind, num_layers=2):
    items = z[f"{case}_msg_items"]
    nbs = [z[f"{case}_msg_nbs_{k}"].astype(np.int64) for k in range(num_layers)]
    offs = [z[f"{case}_msg_offsets_{k}"] for k in range(num_layers)]
    wts = [z[f"{case}_msg_weights_{k}"] for k in range(num_layers)] if kind == "pinsage" else None
    return items, nbs, offs, wts


def feats(di, side="item"):
    return (di[f"{side}_sparse_unique"], di[f"{side}_dense_unique"], di[f"{side}_dense_col_index"])


@pytest.mark.parametrize("data,kind,paradigm", CASES)
def test_oracle_encoder_matches_the_reference_outputs(data, kind, paradigm):
    z = golden()
    case = f"{data}_{kind}_{paradigm}"
    di, sd = data_info(z, data), state_dict(z, case)
    items, nbs, offs, wts = message(z, case, kind)
    got = orc.encode(kind, sd, items, nbs, offs, wts, 2, feats(di))
    ref = z[f"{case}_msg_out"]
    # the reference runs in float32: a few ulps of its largest intermediate per layer
    np.testing.assert_allclose(got, ref, rtol=1e-5, atol=1e-5 * max(1.0, np.abs(ref).max()))
    if paradigm == "u2i":
        users = z[f"{case}_users"]
        ref_u = z[f"{case}_user_rows"]
        np.testing.assert_allclose(orc.user_rows(kind, sd, users, feats(di, "user")), ref_u, rtol=1e-5,
                                   atol=1e-5 * max(1.0, np.abs(ref_u).max()))


def test_padded_message_round_trips_the_recorded_layout():
    """The oracle's padded levels, flattened the reference's way, give offsets of the reference's form."""
    z = golden()
    di = data_info(z, "pure")
    g = orc.Graph(di["user_consumed"], di["item_consumed"], di["n_users"], di["n_items"])
    items = z["pure_graphsage_i2i_msg_items"][:6]
    for kind in ("graphsage", "pinsage"):
        levels = orc.sample(kind, g, 5, items, 2, 3, 10, 2, 0.5)
        nbs, offs, _ = orc.padded_to_message(kind, items, levels)
        assert len(offs[0]) == len(items) and len(offs[1]) == len(nbs[0])
        assert all(np.all(np.diff(o) >= 0) for o in offs)


def test_walker_rules_reproduce_the_recorded_weight_cases():
    """compute_weights with ties, recorded from the reference under random.seed: the oracle's rules on the same
    Python stream give the same ids (in the same order), weights and lengths."""
    z = golden()
    uc = consumed_dict(z["cw_uc_indptr"], z["cw_uc_items"])
    ic = consumed_dict(z["cw_ic_indptr"], z["cw_ic_users"])
    g = orc.Graph(uc, ic, len(uc), len(ic))
    nodes = z["cw_nodes"].tolist()
    s = 0
    while f"cw_params_{s}" in z.files:
        nn, walks, wl, seed = (int(x) for x in z[f"cw_params_{s}"])
        random.seed(seed)
        draws = orc.PythonDraws(g, 0.5)
        ids, wts, lens = [], [], []
        for v in nodes:
            n, w = orc.pinsage_node(g, v, nn, walks, wl, draws.for_node(v))
            ids += n
            wts += w
            lens.append(len(n))
        assert ids == z[f"cw_ids_{s}"].tolist()
        assert lens == z[f"cw_lens_{s}"].tolist()
        np.testing.assert_array_equal(np.asarray(wts), z[f"cw_weights_{s}"])
        s += 1
    assert s >= 6


@pytest.mark.parametrize("kind", ["graphsage", "pinsage"])
def test_walker_rules_match_the_reference_functions(kind):
    from oracle.ref_loader import load_reference, reference_available

    if not reference_available():
        pytest.skip("reference tree not present")
    load_reference()
    from libreco.sampling.random_walks import bipartite_neighbors, bipartite_neighbors_with_weights

    z = golden()
    di = data_info(z, "pure")
    uc, ic = di["user_consumed"], di["item_consumed"]
    g = orc.Graph(uc, ic, di["n_users"], di["n_items"])
    nodes = list(range(0, di["n_items"], 7)) + [0, 0, 3]
    for seed, nn in ((1, 3), (2, 8), (3, 1)):
        random.seed(seed)
        if kind == "graphsage":
            ref, _ = bipartite_neighbors(nodes, uc, ic, nn)
        else:
            ref, ref_w, _, _ = bipartite_neighbors_with_weights(nodes, uc, ic, nn, 10, 3, termination_prob=0.4)
        random.seed(seed)
        draws = orc.PythonDraws(g, 0.4)
        got, got_w = [], []
        for v in nodes:
            if kind == "graphsage":
                got += orc.sage_node(v, nn, draws.for_node(v))
            else:
                n, w = orc.pinsage_node(g, v, nn, 10, 3, draws.for_node(v))
                got += n
                got_w += w
        assert got == list(ref)
        if kind == "pinsage":
            assert got_w == list(ref_w)


def test_keyed_streams_do_not_depend_on_the_batch():
    z = golden()
    di = data_info(z, "pure")
    g = orc.Graph(di["user_consumed"], di["item_consumed"], di["n_users"], di["n_items"])
    items = np.arange(0, 40)
    for kind in ("graphsage", "pinsage"):
        whole = orc.sample(kind, g, 9, items, 2, 3, 4, 2, 0.5)
        part = orc.sample(kind, g, 9, items[10:20], 2, 3, 4, 2, 0.5)
        for lw, lp in zip(whole, part):
            a = lw if kind == "graphsage" else lw[0]
            b = lp if kind == "graphsage" else lp[0]
            per = a.shape[0] // len(items)
            np.testing.assert_array_equal(a[10 * per:20 * per], b)


def test_cont_threshold_matches_random_random():
    from librecommender_b200.sage import cont_threshold

    for p in (0.0, 0.5, 0.3, 1.0, 1e-9, 0.999999):
        t = cont_threshold(p)
        assert t == orc.cont_threshold(p)
        for w in (t - 1, t):
            if 0 <= w < 1 << 32:
                assert (w * 2.0 ** -32 >= p) == (w >= t)


# ---- validation ------------------------------------------------------------------------------------------------------
def _engine(kind="graphsage", paradigm="i2i", sd=None, **kw):
    from librecommender_b200 import sage

    z = golden()
    case = f"pure_{kind}_{paradigm}"
    di = data_info(z, "pure")
    sd = state_dict(z, case) if sd is None else sd
    cls = sage.GraphSage if kind == "graphsage" else sage.PinSage
    return cls(di, sd, paradigm=paradigm, device="cpu", **kw), di, sd


def test_state_dict_keys_and_shapes_are_checked():
    _, di, sd = _engine()
    with pytest.raises(ValueError, match="missing"):
        _engine(sd={k: v for k, v in sd.items() if k != "w_linears.1.bias"})
    with pytest.raises(ValueError, match="unexpected"):
        _engine(sd={**sd, "G1.weight": np.zeros((8, 8), np.float32)})
    with pytest.raises(ValueError, match="shape"):
        _engine(sd={**sd, "w_linears.0.weight": np.zeros((8, 8), np.float32)})
    with pytest.raises(ValueError, match="missing"):           # the u2i paradigm needs the user tower
        _engine(paradigm="u2i", sd=sd)
    with pytest.raises(ValueError, match="missing"):           # a third layer the weights do not have
        _engine(sd=sd, num_layers=3)
    _, _, psd = _engine("pinsage")
    with pytest.raises(ValueError, match="unexpected"):
        _engine("graphsage", sd=psd)
    with pytest.raises(ValueError, match="missing"):
        _engine("pinsage", sd=sd)


def test_parameters_outside_the_envelope_raise():
    for kw in (dict(num_layers=0), dict(num_layers=4), dict(num_neighbors=0), dict(num_neighbors=33),
               dict(paradigm="x2y")):
        with pytest.raises(ValueError):
            _engine(**kw)
    for kw in (dict(num_walks=0), dict(neighbor_walk_len=0), dict(num_walks=65, neighbor_walk_len=4),
               dict(termination_prob=1.5)):
        with pytest.raises(ValueError):
            _engine("pinsage", **kw)


def test_item_ids_and_items_without_consumers_raise_before_launch():
    eng, di, sd = _engine()
    for bad in ([-1], [di["n_items"]], [0.5]):
        with pytest.raises(ValueError, match="outside"):
            eng.neighbors(bad)
    di2 = dict(di, n_items=di["n_items"] + 1, item_consumed={**di["item_consumed"], di["n_items"]: []})
    sd2 = dict(sd, **{"item_embeds.weight": np.zeros((di["n_items"] + 1, 8), np.float32)})
    from librecommender_b200 import sage

    eng2 = sage.GraphSage(di2, sd2, device="cpu")
    with pytest.raises(ValueError, match="no consumer"):
        eng2.neighbors([di["n_items"]])
    with pytest.raises(ValueError, match="no consumer"):
        eng2.item_embeddings()
    with pytest.raises(ValueError, match="levels"):
        eng.encode_message([0], [[1, 2, 3]], [[0]])
    with pytest.raises(ValueError, match="offsets"):
        eng.encode_message([0], [[1, 2, 3], [1]], [[0, 5], [0]])


def test_consumed_lists_with_foreign_ids_raise():
    from librecommender_b200 import sage

    _, di, sd = _engine()
    bad = dict(di, user_consumed={**di["user_consumed"], 0: [di["n_items"]]})
    with pytest.raises(ValueError, match="outside"):
        sage.GraphSage(bad, sd, device="cpu")


# ---- C-ABI -------------------------------------------------------------------------------------------------------
def test_cabi_symbols_are_declared_and_bound():
    from librecommender_b200 import _lib

    header = open(os.path.join(ROOT, "include", "b200reco.h")).read()
    for name in ("b200_sage_neighbors", "b200_pinsage_neighbors", "b200_sage_aggregate"):
        assert f"int {name}(" in header
        assert name in _lib.SIGNATURES
        assert getattr(_lib.lib, name).restype is not None


def test_cabi_rejections_return_minus_two():
    from librecommender_b200 import _lib

    lib, P = _lib.lib, ctypes.c_void_p
    nz = P(16)
    sn = lambda nn=3, n=4, per=1, level=0, p=nz: lib.b200_sage_neighbors(  # noqa: E731
        p, nz, nz, nz, nz, nz, n, per, level, nn, 1, nz, None)
    for rc in (sn(nn=0), sn(nn=33), sn(p=None), sn(n=5, per=2), sn(level=-1), sn(per=0)):
        assert rc == -2
    pn = lambda nn=3, walks=10, wl=2, thr=1 << 31, out=nz: lib.b200_pinsage_neighbors(  # noqa: E731
        nz, nz, nz, nz, nz, nz, 4, 1, 0, nn, walks, wl, thr, 1, out, nz, nz, None)
    for rc in (pn(nn=0), pn(nn=33), pn(walks=0), pn(wl=0), pn(walks=65, wl=4), pn(thr=(1 << 32) + 1), pn(out=None)):
        assert rc == -2
    ag = lambda d=8, lds=8, ldo=16, off=None, stride=3, S=nz: lib.b200_sage_aggregate(  # noqa: E731
        S, lds, None, 4, nz, 8, None, off, None, stride, None, d, nz, ldo, None)
    for rc in (ag(d=0), ag(d=129, lds=129, ldo=258), ag(ldo=15), ag(lds=7), ag(stride=-1), ag(S=None)):
        assert rc == -2


# ---- drop-in -----------------------------------------------------------------------------------------------------
def test_dropin_patches_and_restores_set_embeddings():
    from oracle.ref_loader import load_reference, reference_available

    if not reference_available():
        pytest.skip("reference tree not present")
    load_reference()
    import importlib

    from librecommender_b200 import dropin

    sb = importlib.import_module("libreco.bases.sage_base")
    before = sb.SageBase.set_embeddings
    dropin.install(sage=True)
    try:
        patched = sb.SageBase.set_embeddings
        assert patched is not before
        # the DGL classes keep the reference's method (which asserts a walker)
        with pytest.raises(AssertionError):
            patched(types.SimpleNamespace(use_dgl=True, neighbor_walker=None))
    finally:
        dropin.uninstall()
    assert sb.SageBase.set_embeddings is before
