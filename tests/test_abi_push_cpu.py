"""CPU checks of the push store entry points (mgp_push_records, mgp_push_merge, mgp_push_assign): argument validation
runs before any CUDA call and refuses null pointers, K > 64, bad sizes, strides and misalignment."""
import ctypes

import pytest

C, K, D, B, HW = 4, 3, 128, 2, 9


def _lib():
    from mgproto_b200 import _lib
    return _lib.load()


def _rs(k=K, d=D):
    from mgproto_b200 import ops
    return ops._push_rec_stride(k, d)


@pytest.fixture
def ptrs():
    """16-byte aligned host memory (never dereferenced: validation fails before any launch)."""
    keep, p = [], {}
    for name in ("arg", "val", "xhat", "labels", "rows", "rval", "rpatch", "rlabel", "key", "patch", "row", "mu", "cid",
                 "cpatch", "cval"):
        raw = ctypes.create_string_buffer(64 + 16)
        keep.append(raw)
        p[name] = (ctypes.addressof(raw) + 15) & ~15
    p["_keep"] = keep
    return p


def _records(p, **o):
    a = dict(p, **o)
    return _lib().mgp_push_records(a["arg"], a["val"], a["xhat"], a["labels"], a["rows"], a["rval"], a["rpatch"],
                                   a["rlabel"], a.get("rs", _rs()), a.get("B", B), a.get("HW", HW), a.get("C", C),
                                   a.get("K", K), a.get("D", D), None)


def _merge(p, **o):
    a = dict(p, **o)
    return _lib().mgp_push_merge(a["rows"], a["rval"], a["rpatch"], a["rlabel"], a.get("rs", _rs()), a.get("n", B),
                                 a.get("id0", 0), a["key"], a["patch"], a["row"], a.get("C", C), a.get("K", K),
                                 a.get("D", D), None)


def _assign(p, **o):
    a = dict(p, **o)
    return _lib().mgp_push_assign(a["key"], a["patch"], a["row"], a["mu"], a["cid"], a["cpatch"], a["cval"],
                                  a.get("C", C), a.get("K", K), a.get("D", D), None)


@pytest.mark.parametrize("name", ["arg", "val", "xhat", "labels", "rows", "rval", "rpatch", "rlabel"])
def test_push_records_refuses_null(ptrs, name):
    assert _records(ptrs, **{name: None}) == -1


@pytest.mark.parametrize("name", ["rows", "rval", "rpatch", "rlabel", "key", "patch", "row"])
def test_push_merge_refuses_null(ptrs, name):
    assert _merge(ptrs, **{name: None}) == -1


@pytest.mark.parametrize("name", ["key", "patch", "row", "mu", "cid", "cpatch", "cval"])
def test_push_assign_refuses_null(ptrs, name):
    assert _assign(ptrs, **{name: None}) == -1


@pytest.mark.parametrize("call", [_records, _merge, _assign])
def test_push_entry_points_refuse_k_above_64_and_bad_sizes(ptrs, call):
    assert call(ptrs, K=65, rs=_rs(65)) == -2                    # a store slot per lane pair: at most 64 candidates
    assert call(ptrs, D=130, rs=_rs(K, 132)) == -2               # D % 4 != 0: the rows are copied as float4
    assert call(ptrs, C=0) == -1
    assert call(ptrs, K=0) == -1
    assert call(ptrs, D=0) == -1


def test_push_records_and_merge_refuse_bad_record_layouts(ptrs):
    p = ptrs
    for call in (_records, _merge):
        assert call(p, rs=K * D + 2 * K) == -1                   # too short for rows, values, patches and the label
        assert call(p, rs=_rs() + 2) == -1                       # not a multiple of 4 words: rows lose 16-byte alignment
        assert call(p, rows=p["rows"] + 4) == -1
        assert call(p, rlabel=p["rlabel"] + 4) == -1
    assert _records(p, B=0) == -1
    assert _records(p, HW=0) == -1
    assert _records(p, xhat=p["xhat"] + 4) == -1
    assert _merge(p, n=0) == -1
    assert _merge(p, id0=0xffffffff - B + 1) == -1                # the last id would be the empty slot's
    assert _merge(p, row=p["row"] + 4) == -1
    assert _assign(p, mu=p["mu"] + 4) == -1
    assert _assign(p, row=p["row"] + 8) == -1


def test_push_record_layout_extends_the_mined_record():
    """The push record is the mined record (ops._rec_views) whose row block carries K more words: the values."""
    import torch
    from mgproto_b200 import ops
    rec = torch.zeros((3, ops._push_rec_stride(K, D)))
    rows, val, patch, label = ops._push_rec_views(rec, K, D)
    assert rows.shape == (3, K * D) and val.shape == (3, K) and patch.shape == (3, K) and label.shape == (3,)
    assert rec.shape[1] % 4 == 0 and rec.shape[1] >= K * D + 2 * K + 2
    rows.fill_(1.0)
    val.fill_(2.0)
    patch.fill_(3)
    label.fill_(-1)
    w = rec.view(torch.int32)
    assert (rec[:, :K * D] == 1.0).all() and (rec[:, K * D:K * D + K] == 2.0).all()
    assert (w[:, K * D + K:K * D + 2 * K] == 3).all()
    assert (rec.view(torch.int64)[:, (K * D + 2 * K + 1) // 2] == -1).all()
    # the padding records every merge ignores
    pad = ops._push_rec_views(ops.push_padding_records(2, K, D, "cpu"), K, D)[3]
    assert (pad == -1).all()
