"""Labelled head, image-tile top-1 kernel (logprob_top1_wide_kernel, -m gpu): the packed per (image, prototype)
max / arg-max of log p for isotropic sigma at every instantiated image width, against the max and first arg-max of
the materialised [B,P,HW] map (same operand split, same epilogue formula: bit for bit) and against float64."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

SHAPES = [(14, 14), (7, 7), (16, 16), (10, 10), (3, 11), (4, 8), (8, 8), (7, 9)]   # HW = 196, 49, 256, 100, 33, 32, 64, 63
B, P = 37, 2000        # 37 images do not divide into the teams of the schedule; the last prototype tile is partial


def _dev():
    return torch.device("cuda:0")


def _pack_first_max(lp):
    """[B,P,HW] float32 -> int64 [B,P]: top1_pack(max, first arg-max) as in include/mgproto_b200.h."""
    a = lp.cpu().numpy()
    idx = a.argmax(axis=2).astype(np.uint64)                         # numpy: first occurrence of the maximum
    val = np.take_along_axis(a, idx.astype(np.int64)[..., None], axis=2)[..., 0]
    u = val.astype(np.float32).view(np.uint32).astype(np.uint64)
    key = np.where(u & np.uint64(0x80000000), ~u & np.uint64(0xffffffff), u | np.uint64(0x80000000))
    return ((key << np.uint64(32)) | (np.uint64(0xffffffff) - idx)).view(np.int64)


def _unpack(best):
    bv = best.cpu().numpy().view(np.uint64)
    key = (bv >> np.uint64(32)).astype(np.uint32)
    u = np.where(key & np.uint32(0x80000000), key & np.uint32(0x7fffffff), ~key).astype(np.uint32)
    arg = (np.uint32(0xffffffff) - (bv & np.uint64(0xffffffff)).astype(np.uint32)).astype(np.int64)
    return u.view(np.float32), arg


@pytest.mark.parametrize("D", [128, 64])
@pytest.mark.parametrize("H,W", SHAPES)
def test_top1_image_tiles_vs_materialised(request, H, W, D):
    from mgproto_b200 import _lib, ops
    from test_gpu_shape_edges import assert_reached, trace
    HW = H * W
    g = torch.Generator().manual_seed(1000 * HW + D)
    x = torch.randn(B, D, H, W, generator=g).to(_dev())
    mu = F.normalize(torch.rand(P, D, generator=g), dim=1).to(_dev())
    sg = torch.full((P, D), 1 / np.sqrt(2 * np.pi), device=_dev())
    xhat, _, _ = ops.normalize_fwd(x)

    # unstaged route: operands prepared by the kernel's own pre-passes (the trace proves the launch of the image-tile
    # instantiation for this width; the 128-patch-tile kernel is launched behind it and returns at once)
    with trace() as tr:
        best = ops.logprob_top1(xhat, mu, sg, B, HW, "tc")
    assert_reached(request, tr)
    assert best is not None
    lp = ops.logprob(xhat, mu, sg, 1, B=B, HW=HW, math="tc")
    np.testing.assert_array_equal(best.cpu().numpy(), _pack_first_max(lp))

    # every entry is written (there is no zeroing pass any more): fill the output with a sentinel first
    lib = _lib.load()
    nbytes = lib.mgp_logprob_ws_bytes(B, HW, P, D, ops.MGP_MATH_TC)
    ws = torch.empty((nbytes,), device=_dev(), dtype=torch.uint8)
    out = torch.full((B, P), -1, device=_dev(), dtype=torch.int64)
    ops.check(lib.mgp_logprob_fwd(xhat.data_ptr(), mu.data_ptr(), sg.data_ptr(), 0.0, 0.0, out.data_ptr(),
                                  ops.MGP_OUT_TOP1_BP, B, HW, P, D, ops.MGP_MATH_TC, ws.data_ptr(), nbytes,
                                  ops._stream()), "mgp_logprob_fwd(top1)")
    assert (out != -1).all() and (out != 0).all()
    assert torch.equal(out, best)

    # staged route (what HeadFunction runs): against the map computed from the same staged operands
    stage = ops._stage_for_top1(B, HW, P, D, sg, "tc")
    assert stage == (P, False)
    xh2, _, _, ws2 = ops.normalize_fwd(x, stage=stage)
    best2 = ops.logprob_top1(xh2, mu, sg, B, HW, "tc", ws=ws2, staged=stage)
    assert (best2 != 0).all()
    lp2 = ops.logprob(xh2, mu, sg, 1, B=B, HW=HW, math="tc_reuse", ws=ws2)
    np.testing.assert_array_equal(best2.cpu().numpy(), _pack_first_max(lp2))

    # float64: log p = const - |x - mu|^2 / (2 sigma^2), sigma isotropic
    xd = xhat.double()
    md = mu.double()
    s2 = float(sg[0, 0]) ** 2
    q = (xd * xd).sum(1)[:, None] - 2.0 * xd @ md.t() + (md * md).sum(1)[None, :]
    lp64 = (-0.5 * D * np.log(2 * np.pi) - D * np.log(float(sg[0, 0])) - 0.5 * q / s2)
    lp64 = lp64.view(B, HW, P).permute(0, 2, 1)                                  # [B,P,HW]
    m64, a64 = lp64.max(dim=2)
    srt = torch.sort(lp64, dim=2, descending=True).values
    sep = ((srt[:, :, 0] - srt[:, :, 1]) > 1e-3).cpu().numpy()
    for b in (best, best2):
        val, arg = _unpack(b)
        np.testing.assert_allclose(val, m64.cpu().numpy(), rtol=1e-4, atol=1e-4)
        assert (arg >= 0).all() and (arg < HW).all()
        assert (arg[sep] == a64.cpu().numpy()[sep]).all()
