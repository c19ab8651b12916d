"""CPU test of the fused scorer's organisation codes (b200_recommend_embed_tune) and of what the plan
reports for them (b200_recommend_embed_plan works without a device: the plan of a 132-SM H100)."""
import ctypes

import pytest


def _plan_groups(B, N, d, K):
    from librecommender_b200 import _lib

    out = (ctypes.c_int32 * 8)()
    _lib.check(_lib.lib.b200_recommend_embed_plan(B, N, d, K, out, 8))
    return int(out[6])


@pytest.fixture
def lib():
    from librecommender_b200 import _lib

    yield _lib
    _lib.check(_lib.lib.b200_recommend_embed_tune(215, 0.0))


@pytest.mark.parametrize("code", [235, 233, 135, 133])
def test_pipelined_codes_accepted_and_planned(lib, code):
    assert lib.lib.b200_recommend_embed_tune(code, 0.0) == 0
    cl = code // 100
    assert _plan_groups(32768, 1_000_000, 64, 100) == 10 * cl + 3
    # d_pad > 128 (one k-block per ring stage) cannot hold two whole tiles: one N=256 group instead
    assert _plan_groups(32768, 1_000_000, 192, 100) == 10 * cl + 1


@pytest.mark.parametrize("code", [245, 205, 234, 315])
def test_bad_codes_rejected(lib, code):
    assert lib.lib.b200_recommend_embed_tune(235, 0.0) == 0
    assert lib.lib.b200_recommend_embed_tune(code, 0.0) != 0
    assert b"b200_recommend_embed_tune" in lib.lib.b200_last_error()
    assert _plan_groups(32768, 1_000_000, 64, 100) == 23     # a rejected code changes nothing


def test_two_group_code_keeps_its_width_limit(lib):
    assert lib.lib.b200_recommend_embed_tune(225, 0.0) == 0
    assert _plan_groups(32768, 1_000_000, 128, 100) == 22
    out = (ctypes.c_int32 * 8)()
    assert lib.lib.b200_recommend_embed_plan(32768, 1_000_000, 192, 100, out, 8) != 0
