"""The head on long feature maps (1024 < HW <= 4096, -m gpu): head_select_long_kernel, head_top1_long_kernel and
head_bwd_long_v{2,4}_kernel against the float64 oracle, at the suite's tolerances (test_gpu_shape_edges.py).

HW = 1089 (33x33), 1156, 1600, 2115 (45x47) and 4096 (64x64): labelled and unlabelled head forward + backward with one
image without a class (gt = -1), head_level0 and push_search; T = 1, T = 32, C = 100 unlabelled at 4096 (many backward
drains), K = 40 (the labelled kernel's patch slice shrinks below 1024) and the materialised labelled route.  The long
backward must be bit-identical run to run; HW > 4096, T > 32 and T > HW are refused before any launch.
At HW = 1024 the long entry points reproduce the existing kernels bit for bit (the one torch.profiler window here shows
which kernel each op launches).  test_gpu_training_long_maps.py holds the model-level checks: the reference's
training body and GraphedStep."""
import numpy as np
import pytest
import torch

import headline_case as HC
from test_gpu_headline import TOL, _dev, _net, _t, normwise
from test_gpu_shape_edges import _check_head, _check_logprob, _f64, trace

pytestmark = pytest.mark.gpu

OLD = ("head_select_kernel", "head_top1_kernel", "head_bwd_kernel")
LONG_SEL, LONG_TOP1 = "head_select_long_kernel", "head_top1_long_kernel"
LONG_BWD = ("head_bwd_long_v2_kernel", "head_bwd_long_v4_kernel")


# op -> the kernel it launches (test_long_entry_points_reproduce_the_existing_kernels_at_1024 proves each pairing
# under the profiler)
_OPS = {"head_select_long": LONG_SEL, "head_select_top1_long": LONG_TOP1, "head_backward_long": "head_bwd_long",
        "head_select": "head_select_kernel", "head_select_top1": "head_top1_kernel", "head_backward": "head_bwd_kernel"}


class trace_ops:
    """The head selection / backward kernels a block of work reached, recorded at the ops layer (HeadFunction and
    head_level0 call them through the module).  torch.profiler drops device records late in a long run, and every
    window makes that more likely for the windows after it: this file opens one."""

    def __enter__(self):
        from mgproto_b200 import ops
        self.kernels, self._saved = set(), {}
        for name, kern in _OPS.items():
            fn = getattr(ops, name)
            self._saved[name] = fn

            def spy(*a, _fn=fn, _k=kern, **kw):
                out = _fn(*a, **kw)
                self.kernels.add(_k)
                return out
            setattr(ops, name, spy)
        return self

    def __exit__(self, *exc):
        from mgproto_b200 import ops
        for name, fn in self._saved.items():
            setattr(ops, name, fn)
        return False


def _no_old(tr):
    hit = sorted(k for k in tr.kernels if k.split("<")[0] in OLD)
    assert not hit, "a long map reached the <= 1024-patch kernels: %s" % hit


def _long_hits(tr):
    return sorted(k for k in tr.kernels if k.startswith((LONG_SEL, LONG_TOP1, "head_bwd_long")))


def _bwd_kernel(D):
    return "head_bwd_long"


# ------------------------------------------------------------------------------------ every size, D = 64 or 128 (+256)
SIZES = [(33, 33, 64), (34, 34, 128), (40, 40, 64), (45, 47, 128), (64, 64, 64), (64, 64, 128), (40, 40, 256)]


@pytest.mark.parametrize("H,W,D", SIZES, ids=["%dx%d-d%d" % s for s in SIZES])
def test_long_map_head(H, W, D):
    """Labelled and unlabelled head forward + backward, head_level0 and push_search; one labelled image has gt = -1."""
    from mgproto_b200 import ops
    from mgproto_b200._lib import MGP_OUT_LOGP_BPHW
    C, K, T, B = 8, 10, 20, 3
    HW = H * W
    mu, sg, wt = HC.mixture(C, K, D, seed=700 + HW + D)
    x, gt = HC.head_batch(B, C, K, D, H, W, mu, seed=701 + HW + D, gt_fixed=(C - 1, -1, 0))
    with trace_ops() as tl:
        _check_head(x, mu, sg, wt, gt, T)
    assert LONG_TOP1 in tl.kernels and _bwd_kernel(D) in tl.kernels, sorted(tl.kernels)
    with trace_ops() as tu:
        fw0, _ = _check_head(x, mu, sg, wt, None, T, seed=6)
    assert LONG_SEL in tu.kernels and _bwd_kernel(D) in tu.kernels, sorted(tu.kernels)
    with trace_ops() as t0:
        lv0 = ops.head_level0(_t(x), _t(mu), _t(sg), _t(wt))
    assert LONG_TOP1 in t0.kernels
    np.testing.assert_allclose(lv0.cpu().numpy(), fw0["logits"][:, :, 0], rtol=TOL, atol=1e-5)
    # push search (max / arg-max epilogue) against the argmin over the fp32 [B,P,HW] map and the oracle
    net = _net(C, K, D, T, 8, mu, sg, wt, "auto")
    labels = np.abs(gt)
    with trace_ops() as tp:
        arg, val, xh = net.push_search(_t(x), _t(labels, torch.int64))
    for tr in (tl, tu, t0, tp):
        _no_old(tr)
    lp = ops.logprob(xh, _t(mu).reshape(-1, D), _t(sg).reshape(-1, D), MGP_OUT_LOGP_BPHW, B=B, HW=HW)
    arg2, val2 = ops.push_argmin(lp, _t(labels, torch.int64), C, K)
    lp64 = fw0["logp"].reshape(B, HW, C * K).transpose(0, 2, 1)
    own = np.stack([lp64[b, labels[b] * K:(labels[b] + 1) * K] for b in range(B)])       # [B,K,HW]
    srt = -np.sort(-own, axis=2)
    sep = (srt[:, :, 0] - srt[:, :, 1]) > 1e-3
    a, a2 = arg.cpu().numpy(), arg2.cpu().numpy()
    assert sep.mean() > 0.5
    assert (a[sep] == own.argmax(2)[sep]).all() and (a2[sep] == a[sep]).all()
    np.testing.assert_allclose(val.cpu().numpy(), -np.exp(srt[:, :, 0]), rtol=TOL, atol=1e-9)
    np.testing.assert_allclose(val2.cpu().numpy(), val.cpu().numpy(), rtol=TOL, atol=1e-9)
    if D == 128 and HW == 4096:
        print("HW%d D%d: log p worst relative error %.2e" % (HW, D, _check_logprob(xh, mu, sg, B, HW)))


# ------------------------------------------------------------------------------------ T, drain and slice edges
EDGES = [  # id, C, K, H, W, T, labelled, B
    ("t1-hw1089-lab", 8, 10, 33, 33, 1, True, 3),
    ("t1-hw1089-unl", 8, 10, 33, 33, 1, False, 3),
    ("t32-hw1089-lab", 8, 10, 33, 33, 32, True, 3),
    ("t32-hw1089-unl", 8, 10, 33, 33, 32, False, 3),
    ("t32-c100-hw4096-unl", 100, 10, 64, 64, 32, False, 1),   # P*T = 32 000 backward entries: ~16 drains
    ("k40-hw1156-lab", 25, 40, 34, 34, 20, True, 2),           # head_top1_long_kernel's slice: 896 patches
]


@pytest.mark.parametrize("C,K,H,W,T,labelled,B", [e[1:] for e in EDGES], ids=[e[0] for e in EDGES])
def test_long_map_edges(C, K, H, W, T, labelled, B):
    D = 128
    HW = H * W
    mu, sg, wt = HC.mixture(C, K, D, seed=800 + HW + T + K)
    x, gt = HC.head_batch(B, C, K, D, H, W, mu, seed=801 + HW + T, gt_fixed=(C - 1, -1))
    with trace_ops() as tr:
        _check_head(x, mu, sg, wt, gt if labelled else None, T)
    assert (LONG_TOP1 if labelled else LONG_SEL) in tr.kernels and "head_bwd_long" in tr.kernels, sorted(tr.kernels)
    _no_old(tr)


def test_long_map_materialised_labelled_route():
    """math = "fp32" has no max / arg-max epilogue: the labelled head materialises [B,P,HW] and mines it with
    head_select_long_kernel; anisotropic sigma at D = 256 takes the same route under "auto"."""
    from mgproto_b200 import ops
    from oracle import mgproto_oracle as O
    C, K, T, B, H, W = 8, 10, 20, 2, 34, 34
    for D, math, mode in ((128, "fp32", "init"), (256, "auto", "diag")):
        mu, sg, wt = HC.mixture(C, K, D, seed=900 + D, sigma_mode=mode)
        x, gt = HC.head_batch(B, C, K, D, H, W, mu, seed=901 + D, gt_fixed=(C - 1, -1))
        fw = O.head_forward(_f64(x), _f64(mu), _f64(sg), _f64(wt), gt, T)
        gl = np.random.default_rng(7).standard_normal(fw["logits"].shape) / B
        xd = _t(x).requires_grad_(True)
        with trace_ops() as tr:
            logits, _, idx = ops.head_forward(xd, _t(mu), _t(sg), _t(wt), _t(gt, torch.int64), T, math)
            logits.backward(_t(gl))
        assert LONG_SEL in tr.kernels and LONG_TOP1 not in tr.kernels
        _no_old(tr)
        np.testing.assert_allclose(logits.detach().cpu().numpy(), fw["logits"], rtol=TOL, atol=1e-5)
        gx_ref, dev = O.head_backward(_f64(x), _f64(mu), _f64(sg), _f64(wt), gt, T, gl, idx=idx.cpu().numpy())
        assert dev < TOL, dev
        assert normwise(xd.grad.cpu().numpy(), gx_ref) < TOL


def test_no_long_kernel_at_1024_patches_or_fewer():
    from mgproto_b200 import ops
    C, K, D, T, B = 8, 10, 128, 20, 2
    mu, sg, wt = HC.mixture(C, K, D, seed=950)
    for H, W in ((32, 32), (14, 14)):
        x, gt = HC.head_batch(B, C, K, D, H, W, mu, seed=951)
        with trace_ops() as tr:
            for g in (_t(gt, torch.int64), None):
                xd = _t(x).requires_grad_(True)
                logits, _, _ = ops.head_forward(xd, _t(mu), _t(sg), _t(wt), g, T)
                logits.sum().backward()
            ops.head_level0(_t(x), _t(mu), _t(sg), _t(wt))
        assert not _long_hits(tr), _long_hits(tr)


# ------------------------------------------------------------------------------------ HW = 1024: long == existing
def test_long_entry_points_reproduce_the_existing_kernels_at_1024():
    from mgproto_b200 import ops
    from mgproto_b200._lib import MGP_OUT_LOGP_BPHW
    C, K, D, T, B, H, W = 8, 10, 128, 20, 3, 32, 32
    HW, P = H * W, C * K
    mu, sg, wt = HC.mixture(C, K, D, seed=960)
    x, gt = HC.head_batch(B, C, K, D, H, W, mu, seed=961, gt_fixed=(C - 1, -1, 0))
    mu2, sg2, w = _t(mu).reshape(P, D), _t(sg).reshape(P, D), _t(wt)
    g = _t(gt, torch.int64)
    xhat, inv, _ = ops.normalize_fwd(_t(x))
    lp = ops.logprob(xhat, mu2, sg2, MGP_OUT_LOGP_BPHW, B=B, HW=HW)
    best = ops.logprob_top1(xhat, mu2, sg2, B, HW)
    assert best is not None
    gl = _t(np.random.default_rng(3).standard_normal((B, C, T)) / B)
    dims = (B, HW, C, K, D, T, H, W)
    # written entries of head_select_top1: level 0 everywhere, every level of the own class
    written = np.zeros((B, P, T), bool)
    written[:, :, 0] = True
    for b in range(B):
        if gt[b] >= 0:
            written[b, gt[b] * K:(gt[b] + 1) * K] = True
    # the D = 64 lane width of the long backward (head_bwd_long_v2_kernel), unlabelled
    mu64, sg64, wt64 = HC.mixture(C, K, 64, seed=962)
    x64, _ = HC.head_batch(B, C, K, 64, H, W, mu64, seed=963)
    m64, s64, w64 = _t(mu64).reshape(P, 64), _t(sg64).reshape(P, 64), _t(wt64)
    xh64, inv64, _ = ops.normalize_fwd(_t(x64))
    lp64 = ops.logprob(xh64, m64, s64, MGP_OUT_LOGP_BPHW, B=B, HW=HW)
    dims64 = (B, HW, C, K, 64, T, H, W)
    # the one profiler window of this file: every new kernel and its <= 1024-patch counterpart
    with trace() as tr:
        a = ops.head_select(lp64, w64, None, T, C, K)
        b_ = ops.head_select_long(lp64, w64, None, T, C, K)
        ga = ops.head_backward(gl, a[0], a[1], a[2], w64, None, xh64, inv64, m64, s64, dims64)
        gb = ops.head_backward_long(gl, b_[0], b_[1], b_[2], w64, None, xh64, inv64, m64, s64, dims64)
        assert torch.equal(ga, gb)
        for gg in (g, None):
            a = ops.head_select(lp, w, gg, T, C, K)
            b_ = ops.head_select_long(lp, w, gg, T, C, K)
            for u, v in zip(a, b_):
                assert torch.equal(u, v)
            ga = ops.head_backward(gl, a[0], a[1], a[2], w, gg, xhat, inv, mu2, sg2, dims)
            gb = ops.head_backward_long(gl, b_[0], b_[1], b_[2], w, gg, xhat, inv, mu2, sg2, dims)
            assert torch.equal(ga, gb)
        a = ops.head_select_top1(best, xhat, mu2, sg2, w, g, T, C, K, HW)
        b_ = ops.head_select_top1_long(best, xhat, mu2, sg2, w, g, T, C, K, HW)
        assert torch.equal(a[0], b_[0])
        for u, v in zip(a[1:], b_[1:]):
            assert np.array_equal(u.cpu().numpy()[written], v.cpu().numpy()[written])
        ga = ops.head_backward(gl, a[0], a[1], a[2], w, g, xhat, inv, mu2, sg2, dims)
        gb = ops.head_backward_long(gl, b_[0], b_[1], b_[2], w, g, xhat, inv, mu2, sg2, dims)
        assert torch.equal(ga, gb)
    old = ("head_select_kernel<32, 1, false>", "head_top1_kernel<32, 1, 256>", "head_bwd_kernel<2>",
           "head_bwd_kernel<4>")
    for k in (LONG_SEL, LONG_TOP1) + LONG_BWD + old:
        assert k in tr.kernels, (k, sorted(tr.kernels))



def test_long_backward_is_deterministic_at_4096():
    from mgproto_b200 import ops
    C, K, D, T, B, H, W = 20, 10, 64, 20, 2, 64, 64
    mu, sg, wt = HC.mixture(C, K, D, seed=970)
    x, _ = HC.head_batch(B, C, K, D, H, W, mu, seed=971)
    grads = []
    with trace_ops() as tr:
        for _ in range(2):
            xd = _t(x).requires_grad_(True)
            logits, _, _ = ops.head_forward(xd, _t(mu), _t(sg), _t(wt), None, T)
            logits.backward(torch.ones_like(logits) / B)
            grads.append(xd.grad)
    assert LONG_SEL in tr.kernels and "head_bwd_long" in tr.kernels, sorted(tr.kernels)
    assert torch.equal(grads[0], grads[1])


# ------------------------------------------------------------------------------------ refusals
def test_long_map_refusals():
    """HW > 4096, T > 32 and T > HW raise "not supported" from the new ops and from head_forward (the entry points
    validate before any CUDA call: tests/test_abi_long_maps_cpu.py)."""
    from mgproto_b200 import ops
    C, K, D, B = 4, 3, 64, 2
    P = C * K
    mu, sg, wt = HC.mixture(C, K, D, seed=980)
    w, g = _t(wt), _t(np.array([0, 1]), torch.int64)
    mu2, sg2 = _t(mu).reshape(P, D), _t(sg).reshape(P, D)
    dev = _dev()
    with trace_ops() as tr:
        for HW, T in ((4097, 20), (1089, 33), (16, 20)):
            with pytest.raises(RuntimeError, match="not supported"):
                ops.head_select_long(torch.zeros((B, P, HW), device=dev), w, g, T, C, K)
            xh = torch.zeros((B * HW, D), device=dev)
            with pytest.raises(RuntimeError, match="not supported"):
                ops.head_select_top1_long(torch.zeros((B, P), dtype=torch.int64, device=dev), xh, mu2, sg2, w, g, T, C,
                                          K, HW)
            z = torch.zeros((B, C, T), device=dev)
            vi = torch.zeros((B, P, T), device=dev)
            with pytest.raises(RuntimeError, match="not supported"):
                ops.head_backward_long(z, z, vi, vi.int(), w, g, xh, torch.ones(B * HW, device=dev), mu2, sg2,
                                       (B, HW, C, K, D, T, 1, HW))
    assert not _long_hits(tr), _long_hits(tr)
    x, gt = HC.head_batch(B, C, K, D, 17, 241, mu, seed=981)                   # HW = 4097
    for gg in (_t(gt, torch.int64), None):
        with pytest.raises(RuntimeError, match="not supported"):
            ops.head_forward(_t(x), _t(mu), _t(sg), w, gg, 20)
    x, gt = HC.head_batch(B, C, K, D, 33, 33, mu, seed=982)
    for gg in (_t(gt, torch.int64), None):
        with pytest.raises(RuntimeError, match="not supported"):
            ops.head_forward(_t(x), _t(mu), _t(sg), w, gg, 33)
    with pytest.raises(RuntimeError, match="not supported"):
        ops.head_level0(_t(HC.head_batch(B, C, K, D, 17, 241, mu, seed=983)[0]), _t(mu), _t(sg), w)
