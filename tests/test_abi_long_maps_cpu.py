"""CPU checks of the long-map head entry points (mgp_head_select_long, mgp_head_select_top1_long, mgp_head_bwd_long_x):
argument validation runs before any CUDA call and refuses null pointers, bad sizes, an unknown feature format,
HW > 4096, T > 32, T > HW, K > 64 and too small a workspace."""
import ctypes

import pytest

C, K, D, B, HW, T = 4, 3, 64, 2, 1089, 20


def _lib():
    from mgproto_b200 import _lib
    return _lib.load()


@pytest.fixture
def ptrs():
    """16-byte aligned host memory (never dereferenced: validation fails before any launch)."""
    keep, p = [], {}
    for name in ("logp", "best", "xhat", "mu", "sigma", "weight", "gt", "logits", "vals", "idx", "gl", "inv", "ws", "gx"):
        raw = ctypes.create_string_buffer(64 + 16)
        keep.append(raw)
        p[name] = (ctypes.addressof(raw) + 15) & ~15
    p["_keep"] = keep
    return p


def _select(p, **o):
    a = dict(p, **o)
    return _lib().mgp_head_select_long(a["logp"], a["weight"], a["gt"], a["logits"], a["vals"], a["idx"], a.get("B", B),
                                       a.get("HW", HW), a.get("C", C), a.get("K", K), a.get("T", T), None)


def _top1(p, **o):
    a = dict(p, **o)
    return _lib().mgp_head_select_top1_long(a["best"], a["xhat"], a["mu"], a["sigma"], a["weight"], a["gt"], a["logits"],
                                            a["vals"], a["idx"], a.get("B", B), a.get("HW", HW), a.get("C", C),
                                            a.get("K", K), a.get("D", D), a.get("T", T), None)


def _ws(hw=HW):
    return _lib().mgp_head_bwd_long_ws_bytes(B, hw, C * K, D)


def _bwd(p, **o):
    a = dict(p, **o)
    hw = a.get("HW", HW)
    return _lib().mgp_head_bwd_long_x(a["gl"], a["logits"], a["vals"], a["idx"], a["weight"], a["gt"], a["xhat"],
                                      a["inv"], a["mu"], a["sigma"], a["ws"], a.get("ws_bytes", _ws(hw)), a["gx"],
                                      a.get("x_fmt", 0), a.get("B", B), hw, a.get("C", C), a.get("K", K),
                                      a.get("D", D), a.get("T", T), None)


@pytest.mark.parametrize("name", ["logp", "weight", "logits", "vals", "idx"])
def test_select_long_refuses_null(ptrs, name):
    assert _select(ptrs, **{name: None}) == -1


@pytest.mark.parametrize("name", ["best", "xhat", "mu", "sigma", "weight", "gt", "logits", "vals", "idx"])
def test_select_top1_long_refuses_null(ptrs, name):
    assert _top1(ptrs, **{name: None}) == -1


@pytest.mark.parametrize("name", ["gl", "logits", "vals", "idx", "weight", "xhat", "inv", "mu", "sigma", "ws", "gx"])
def test_bwd_long_refuses_null(ptrs, name):
    assert _bwd(ptrs, **{name: None}) == -1


@pytest.mark.parametrize("call", [_select, _top1, _bwd])
def test_long_entry_points_refuse_unsupported_shapes(ptrs, call):
    assert call(ptrs, HW=4097) == -2                           # above the 12-bit patch index
    assert call(ptrs, T=33) == -2
    assert call(ptrs, HW=16, T=20) == -2                      # T > HW


@pytest.mark.parametrize("call", [_select, _top1, _bwd])
def test_long_entry_points_refuse_bad_sizes(ptrs, call):
    for k in ("B", "HW", "C", "K", "T"):
        assert call(ptrs, **{k: 0}) == -1, k
        assert call(ptrs, **{k: -3}) == -1, k


def test_long_entry_points_specific_checks(ptrs):
    assert _select(ptrs, K=65) == -2 and _top1(ptrs, K=65) == -2     # [CT*K][T] winners: at most 64 rows per block
    assert _top1(ptrs, D=0) == -1 and _top1(ptrs, D=66) == -1          # rows are read as float4
    assert _top1(ptrs, C=4000, K=64, D=256) == -2                      # no room for a 32-patch slice in 200 KB
    assert _bwd(ptrs, D=0) == -1
    assert _bwd(ptrs, x_fmt=3) == -1 and _bwd(ptrs, x_fmt=-1) == -1
    assert _bwd(ptrs, ws_bytes=_ws() - 4) == -3
    assert _bwd(ptrs, C=1 << 18, K=4, ws_bytes=1 << 40) == -2          # P = 2^20: the 32-bit entry key overflows
