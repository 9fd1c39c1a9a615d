"""CPU checks of the feature-format decision (ops._feature_format): which MGP_X_* code the add-on features' dtype and
memory format map to, the fall-back to contiguous NCHW, the error on other dtypes, and the C ABI's handling of x_fmt."""
import os
import re

import pytest
import torch

from mgproto_b200 import _lib, ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

DTYPES = [(torch.float32, _lib.MGP_X_F32), (torch.bfloat16, _lib.MGP_X_BF16), (torch.float16, _lib.MGP_X_F16)]


@pytest.mark.parametrize("dtype,code", DTYPES)
def test_nchw_and_channels_last(dtype, code):
    x = torch.randn(3, 16, 5, 7).to(dtype)
    y, fmt = ops._feature_format(x)
    assert fmt == code and y is x
    xl = x.to(memory_format=torch.channels_last)
    y, fmt = ops._feature_format(xl)
    assert fmt == code | _lib.MGP_X_NHWC and y is xl
    assert y.permute(0, 2, 3, 1).is_contiguous()          # [B,H,W,D] rows: the [N,D] layout the kernels read


@pytest.mark.parametrize("dtype,code", DTYPES)
def test_other_strides_become_contiguous_nchw(dtype, code):
    base = torch.randn(3, 16, 5, 14).to(dtype)
    for x in (base[..., ::2],                               # strided view
              base.permute(0, 1, 3, 2),                     # H and W swapped
              torch.randn(3, 5, 7, 16).to(dtype).permute(0, 3, 2, 1)):
        assert not x.is_contiguous() and not x.is_contiguous(memory_format=torch.channels_last)
        y, fmt = ops._feature_format(x)
        assert fmt == code and y.is_contiguous() and torch.equal(y, x)


def test_ambiguous_strides_are_nchw():
    """H = W = 1 (or a size-1 channel dim) is contiguous in both formats: it stays NCHW."""
    x = torch.randn(4, 16, 1, 1).to(memory_format=torch.channels_last)
    assert ops._feature_format(x)[1] == _lib.MGP_X_F32


@pytest.mark.parametrize("dtype", [torch.float64, torch.int32, torch.int64, torch.uint8, torch.bool])
def test_other_dtypes_raise(dtype):
    x = torch.zeros(2, 8, 3, 3, dtype=dtype)
    with pytest.raises(RuntimeError, match="torch.float32, torch.bfloat16 or torch.float16"):
        ops._feature_format(x)
    with pytest.raises(RuntimeError, match="torch.float32, torch.bfloat16 or torch.float16"):
        ops._feature_format(x.to(memory_format=torch.channels_last))


def test_format_constants_match_header():
    hdr = open(os.path.join(ROOT, "include", "mgproto_b200.h")).read()
    defs = {m.group(1): int(m.group(2)) for m in re.finditer(r"#define\s+(MGP_X_[A-Z0-9_]+)\s+(-?\d+)\b", hdr)}
    assert defs == {"MGP_X_F32": _lib.MGP_X_F32, "MGP_X_BF16": _lib.MGP_X_BF16, "MGP_X_F16": _lib.MGP_X_F16,
                    "MGP_X_NHWC": _lib.MGP_X_NHWC}


def test_unknown_format_is_invalid():
    """Argument validation runs before any CUDA call: an unknown x_fmt returns MGP_ERR_INVALID (-1)."""
    import ctypes
    lib = _lib.load()
    p = ctypes.c_void_p(16)                                  # never dereferenced: validation rejects first
    for bad in (3, 7, 8, -1, 0x100):
        assert lib.mgp_normalize_fwd_x(p, bad, p, p, None, None, 0, 1, 4, 1, 0, 0, None) == -1
        assert lib.mgp_normalize_bwd_x(p, p, p, p, bad, 1, 4, 1, None) == -1
        assert lib.mgp_head_bwd_x(p, p, p, p, p, None, p, p, p, p, p, 1 << 20, p, bad, 1, 1, 1, 1, 4, 1, None) == -1
    assert lib.mgp_normalize_fwd_x(None, 0, p, p, None, None, 0, 1, 4, 1, 0, 0, None) == -1
    assert lib.mgp_normalize_fwd_x(p, 0, p, p, None, p, 1 << 20, 1, 4, 1, 0, 0, None) == -1   # staging needs P > 0
