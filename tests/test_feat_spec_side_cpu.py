"""FeatSpec.side: the one-sided layouts and field positions that hoisted all-items scoring, AutoInt's field map,
the towers and the first-layer column slices rely on — host logic only, on a CPU device."""
import numpy as np
import pytest


def _spec(ucols, icols, udcols, idcols, n_users=3, n_items=4):
    from librecommender_b200.feat_models import FeatSpec
    import torch

    d = dict(n_users=n_users, n_items=n_items, user_sparse_col_index=ucols, item_sparse_col_index=icols,
             user_dense_col_index=udcols, item_dense_col_index=idcols,
             user_sparse_unique=np.zeros((n_users + 1, len(ucols)), np.int32) if ucols else None,
             item_sparse_unique=np.zeros((n_items + 1, len(icols)), np.int32) if icols else None,
             user_dense_unique=np.zeros((n_users + 1, len(udcols)), np.float32) if udcols else None,
             item_dense_unique=np.zeros((n_items + 1, len(idcols)), np.float32) if idcols else None)
    return FeatSpec(d, 8, torch.device("cpu"))


def _fields(L):
    return (L.id_mask, L.n_sparse, L.n_dense, list(L.sparse_side[:L.n_sparse]), list(L.sparse_col[:L.n_sparse]),
            list(L.dense_side[:L.n_dense]), list(L.dense_col[:L.n_dense]), list(L.dense_embed_row[:L.n_dense]))


def test_interleaved_columns():
    # sparse fields 0..4: user 1, 3 / item 0, 2, 4; dense fields 0..2: user 2 / item 0, 1
    sp = _spec([1, 3], [0, 2, 4], [2], [0, 1])
    F = 2 + 5 + 3
    Lu, pu = sp.side("user")
    Li, pi = sp.side("item")
    assert pu == [0, 2 + 1, 2 + 3, 7 + 2]
    assert pi == [1, 2 + 0, 2 + 2, 2 + 4, 7 + 0, 7 + 1]
    assert sorted(pu + pi) == list(range(F))
    assert _fields(Lu) == (1, 2, 1, [0, 0], [0, 1], [0], [0], [2])
    assert _fields(Li) == (2, 3, 2, [1, 1, 1], [0, 1, 2], [1, 1], [0, 1], [0, 1])
    assert sp.side("user") is sp.side("user")                     # built once
    assert sp.layout.id_mask == 3 and sp.layout.n_sparse == 5    # the global layout is left alone


def test_empty_side():
    sp = _spec([], [0, 1], [], [0])
    Lu, pu = sp.side("user")
    Li, pi = sp.side("item")
    assert pu == [0]
    assert pi == [1, 2, 3, 4]
    assert sorted(pu + pi) == list(range(5))
    assert _fields(Lu) == (1, 0, 0, [], [], [], [], [])
    assert _fields(Li) == (2, 2, 1, [1, 1], [0, 1], [1], [0], [0])


@pytest.mark.parametrize("which", ["user", "item"])
def test_without_id(which):
    sp = _spec([0, 2], [1], [1], [0])
    L, pos = sp.side(which, with_id=False)
    Lid, pos_id = sp.side(which)
    assert L.id_mask == 0
    assert pos == pos_id[1:]
    assert _fields(L)[1:] == _fields(Lid)[1:]
    assert (L.ld_us, L.ld_is, L.ld_ud, L.ld_id) == (Lid.ld_us, Lid.ld_is, Lid.ld_ud, Lid.ld_id)
