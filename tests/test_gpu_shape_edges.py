"""Every kernel instantiation the launchers pick by shape, against float64 (-m gpu).

The headline tests run the bench shapes (HW = 196, T = 20, K = 10, 800-row banks).  The launchers choose among template
instantiations by shape -- head_select_kernel / head_top1_kernel by R = ceil(HW / 32), logprob_top1_wide_kernel by the
image width, logprob_tc_kernel by output layout and HW, em_tc_kernel / em_fused_kernel by K and D -- and this file
runs each instantiation at least once, at the edges where an index, a mask or a padding assumption can go wrong:
feature maps of 417..1024 patches (128-patch tiles crossing several image ends), T = 1, T = HW = 32, the head
backward's two-drain and unlabelled many-drain entry lists, K < KT padding rows and banks below / at / just past one
64-row tile in the EM.

Reference: the float64 oracle (oracle/mgproto_oracle.py) or a float64 torch restatement, with the suite's tolerances:
1e-4 element-wise relative on logits, log p and pi; 1e-4 norm-wise on the feature gradient, mu and the Adam moments;
1e-3 norm-wise on the mu movement; indices exact where the reference's neighbouring log p are more than 1e-3 apart;
the gradient is routed through the kernel's own picks (O.head_backward(..., idx=...), pick deviation < 1e-4).

Each case runs under torch.profiler (CUDA activity) and asserts that the instantiations COVERS assigns to it were
launched.  One choice is made on the device, and there a trace entry proves only the launch: the image-tile vs the
128-patch-tile top-1 kernel when the host does not know sigma is isotropic.  Those cases select the kernel that does
the work with staging, as the existing tests do.

tests/test_kernel_coverage_cpu.py checks, without a GPU, that every template instantiation in the built library is a
key of COVERS or is listed in its EXEMPT."""
import functools
import re

import numpy as np
import pytest
import torch

import headline_case as HC
from test_gpu_headline import TOL, _fill_bank, _net, _seed_adam, _t, em_path, normwise

pytestmark = pytest.mark.gpu

_E = "test_gpu_shape_edges::"
_W = "test_gpu_top1_wide::test_top1_image_tiles_vs_materialised"
# demangled instantiation (kernel_key) -> the test that launches it and checks its result against float64
COVERS = {
    "normalize_fwd_kernel<float, false>": _E + "test_head_large_maps[21x21-d128]",
    "normalize_bwd_kernel<float, false>": _E + "test_head_large_maps[21x21-d128]",
    "head_bwd_kernel<2>": _E + "test_head_large_maps[21x21-d64]",
    "head_bwd_kernel<4>": _E + "test_head_T_edges[t32-c200-lab]",
    "head_top1_kernel<4, 2, 256>": _E + "test_head_T_edges[t32-hw32-lab]",
    "head_top1_kernel<7, 2, 256>": _E + "test_head_T_edges[t32-c200-lab]",
    "head_top1_kernel<13, 1, 256>": _E + "test_head_T_edges[t1-hw300-lab]",
    "head_top1_kernel<25, 1, 256>": _E + "test_head_large_maps[28x28-d128]",
    "head_top1_kernel<32, 1, 256>": _E + "test_head_large_maps[32x32-d128]",
    "head_select_kernel<2, 4, false>": _E + "test_head_T_edges[t32-hw32-unl]",
    "head_select_kernel<2, 4, true>": _E + "test_head_T_edges[t32-hw32-unl]",
    "head_select_kernel<4, 4, false>": _E + "test_head_T_edges[t1-hw100-unl]",
    "head_select_kernel<4, 4, true>": _E + "test_head_T_edges[t1-hw100-unl]",
    "head_select_kernel<7, 4, false>": _E + "test_unlabelled_backward_c200",
    "head_select_kernel<7, 4, true>": _E + "test_unlabelled_backward_c200",
    "head_select_kernel<13, 2, false>": _E + "test_head_T_edges[t1-hw300-unl]",
    "head_select_kernel<13, 2, true>": _E + "test_head_T_edges[t1-hw300-unl]",
    "head_select_kernel<25, 1, false>": _E + "test_head_large_maps[28x28-d128]",
    "head_select_kernel<25, 1, true>": _E + "test_head_large_maps[21x21-d128]",
    "head_select_kernel<32, 1, false>": _E + "test_head_large_maps[32x32-d128]",
    "head_select_kernel<32, 1, true>": _E + "test_labelled_fallback_k40",
    "logprob_tc_kernel<0>": _E + "test_head_large_maps[29x29-d128]",    # [N,P], P % 4 != 0: plain stores
    "logprob_tc_kernel<1>": _E + "test_head_large_maps[29x29-d128]",    # [B,P,HW] log p, HW > 256: plain stores
    "logprob_tc_kernel<2>": _E + "test_head_large_maps[29x29-d128]",    # [B,P,HW] -p, HW > 256
    "logprob_tc_kernel<3>": _E + "test_head_large_maps[29x29-d128]",    # [N,P] through TMA stores
    "logprob_tc_kernel<4>": _E + "test_head_T_edges[t1-hw100-unl]",     # [B,P,HW] log p through the 3-D tensor map
    "logprob_tc_kernel<5>": _E + "test_head_T_edges[t1-hw100-lab]",     # [B,P,HW] -p through the 3-D tensor map
    "logprob_tc_kernel<6>": _E + "test_head_large_maps[29x29-d128]",    # top-1, 128-patch tiles across image ends
    "logprob_top1_wide_kernel<32, 32>": _E + "test_head_T_edges[t32-hw32-lab]",
    "logprob_top1_wide_kernel<56, 33>": _W + "[3-11-128]",
    "logprob_top1_wide_kernel<64, 57>": _W + "[8-8-128]",
    "logprob_top1_wide_kernel<128, 65>": _E + "test_head_T_edges[t1-hw100-lab]",
    "logprob_top1_wide_kernel<200, 129>": _E + "test_head_T_edges[t32-c200-lab]",
    "logprob_top1_wide_kernel<256, 201>": _W + "[16-16-128]",
    "logprob_z_kernel<64>": _E + "test_head_large_maps[21x21-d64]",
    "logprob_z_kernel<128>": _E + "test_head_large_maps[21x21-d128]",
    "logprob_simt_kernel<0>": _E + "test_head_large_maps[21x21-d128]",
    "logprob_simt_kernel<1>": _E + "test_head_large_maps[21x21-d128]",
    "logprob_simt_kernel<2>": _E + "test_head_large_maps[21x21-d128]",
    "em_tc_kernel<128, 5>": _E + "test_em_instantiations[k2-d128-cap37-tc]",
    "em_tc_kernel<128, 10>": _E + "test_em_instantiations[k7-d128-cap65-tc]",
    "em_tc_kernel<128, 16>": _E + "test_em_instantiations[k11-d128-cap200-tc]",
    "em_tc_kernel<256, 5>": _E + "test_em_instantiations[k3-d256-cap50-tc]",
    "em_tc_kernel<256, 10>": _E + "test_em_instantiations[k10-d256-cap64-tc]",
    "em_tc_kernel<256, 16>": _E + "test_em_instantiations[k16-d256-cap129-tc]",
    "em_fused_kernel<128, 3>": _E + "test_em_instantiations[k2-d128-cap37-fused]",
    "em_fused_kernel<128, 5>": _E + "test_em_instantiations[k7-d128-cap65-fused]",
    "em_fused_kernel<128, 8>": _E + "test_em_instantiations[k16-d128-cap8-fused]",
    "em_fused_kernel<64, 3>": _E + "test_em_instantiations[k2-d64-cap37-fused]",
    "em_fused_kernel<64, 5>": _E + "test_em_instantiations[k10-d64-cap65-fused]",
    "em_fused_kernel<64, 8>": _E + "test_em_instantiations[k16-d64-cap200-fused]",
}

# instantiations (or whole kernels, by name) that no case here targets, and why
EXEMPT = {
    "normalize_fwd_kernel": "one instantiation per feature dtype and layout, not per shape: "
                            "test_gpu_feature_formats.py checks each bit for bit against the fp32 NCHW pass",
    "normalize_bwd_kernel": "as normalize_fwd_kernel",
    "em_stats_kernel": "statistics pass of the multi-launch and the row-sharded multi-GPU EM (48 instantiations over "
                       "D / 128, the K bucket and the s2 flag); its K bucket is chosen the same way at every cap",
    "em_stats_fast_kernel": "statistics pass of the multi-launch EM at D = 64 / 128, as em_stats_kernel",
    "em_estep_kernel": "E-step of the OoD scoring API (ops.em_estep), one instantiation per 128 dims; "
                       "not on the training step",
}


def kernel_key(name):
    """A demangled kernel name, as cu++filt or torch.profiler prints it -> 'kernel<args>' (or 'kernel'): the
    namespace, the parameter list and cu++filt's '(int)' / '(bool)' casts are dropped."""
    s = name.replace("(bool)0", "false").replace("(bool)1", "true")
    s = re.sub(r"\((?:unsigned )?(?:int|long|short|char)\)", "", s)
    m = re.search(r"([A-Za-z_]\w*)(<[^()]*>)?\(", s)
    return m.group(1) + (m.group(2) or "") if m else s


class trace:
    """The kernels a block of work launched (torch.profiler, CUDA activity), as kernel_key()s."""

    def __enter__(self):
        from torch.profiler import ProfilerActivity, profile
        torch.cuda.synchronize()
        self._prof = profile(activities=[ProfilerActivity.CUDA])
        self._prof.__enter__()
        return self

    def __exit__(self, *exc):
        torch.cuda.synchronize()
        self._prof.__exit__(*exc)
        self.kernels = {kernel_key(e.key) for e in self._prof.key_averages()}
        return False


def assert_reached(request, tr, absent=()):
    """Every instantiation COVERS assigns to the running test was launched; no kernel named in `absent` was."""
    me = "%s::%s" % (request.module.__name__, request.node.name)
    missing = sorted(k for k, v in COVERS.items() if v == me and k not in tr.kernels)
    assert not missing, "not launched: %s; launched: %s" % (missing, sorted(tr.kernels))
    hit = sorted(k for k in tr.kernels if k.split("<")[0] in absent)
    assert not hit, "launched, but this shape must not reach them: %s" % hit


def _f64(a):
    return np.asarray(a, np.float64)


def _lp64(xhat, mu, sg):
    """float64 log p [N,P] (model.py:256-275) from the kernel's own normalised features."""
    x, m = xhat.double(), torch.as_tensor(mu, device=xhat.device).double().reshape(-1, xhat.shape[1])
    s = torch.as_tensor(sg, device=xhat.device).double().reshape(m.shape)
    w = 1.0 / (s * s)
    q = (x * x) @ w.t() - 2.0 * x @ (m * w).t() + (m * m * w).sum(1)[None]
    return -0.5 * x.shape[1] * np.log(2 * np.pi) - torch.log(s).sum(1)[None] - 0.5 * q


def _check_logprob(xhat, mu, sg, B, HW):
    """ops.logprob in the three layouts, under the automatic choice, the tensor-core kernel's own stores (TMA and, with
    P % 4 != 0, plain) and the fp32 SIMT kernel, against float64."""
    from mgproto_b200 import ops
    from mgproto_b200._lib import MGP_OUT_LOGP_BPHW, MGP_OUT_LOGP_NP, MGP_OUT_NEGP_BPHW
    D = xhat.shape[1]
    mu_t, sg_t = _t(mu).reshape(-1, D), _t(sg).reshape(-1, D)
    P = mu_t.shape[0]
    ref = _lp64(xhat, mu, sg)
    bphw = ref.view(B, HW, P).permute(0, 2, 1)
    worst = 0.0

    def close(got, want):                        # worst: relative error where |log p| > 0.1
        nonlocal worst
        rel = (got.double() - want).abs() / want.abs()
        worst = max(worst, float(rel[want.abs() > 0.1].max()))
        np.testing.assert_allclose(got.cpu().numpy(), want.cpu().numpy(), rtol=TOL, atol=3e-5)

    for math in ("auto", "fp32"):
        close(ops.logprob(xhat, mu_t, sg_t, MGP_OUT_LOGP_NP, math=math), ref)
        close(ops.logprob(xhat, mu_t, sg_t, MGP_OUT_LOGP_BPHW, B=B, HW=HW, math=math), bphw)
        got = ops.logprob(xhat, mu_t, sg_t, MGP_OUT_NEGP_BPHW, B=B, HW=HW, math=math)
        np.testing.assert_allclose(got.cpu().numpy(), -torch.exp(bphw).cpu().numpy(), rtol=TOL, atol=1e-9)
    tc = "tc" if D <= 128 else "tc_iso"               # (D = 256 runs on the tensor cores with isotropic sigma only)
    close(ops.logprob(xhat, mu_t, sg_t, MGP_OUT_LOGP_NP, math=tc), ref)
    close(ops.logprob(xhat, mu_t[:P - 2].contiguous(), sg_t[:P - 2].contiguous(), MGP_OUT_LOGP_NP, math=tc), ref[:, :P - 2])
    return worst


def _np_select_fits(HW, C, K, T):
    """head_select on an [N,P] log p stages a transposed tile: mgp_head_select_np takes the shape when it fits."""
    ct = min(max(64 // K, 1), C)
    return (ct * K * T + HW * (ct * K + 1)) * 4 <= 200 * 1024


def _check_head(x, mu, sg, wt, gt, T, seed=5):
    """head_forward + backward (gt None: unlabelled) against the float64 oracle.  -> (oracle forward, kernel xhat)."""
    from mgproto_b200 import ops
    from oracle import mgproto_oracle as O
    B, D, H, W = x.shape
    C, K, _ = mu.shape
    HW, P = H * W, C * K
    fw = O.head_forward(_f64(x), _f64(mu), _f64(sg), _f64(wt), gt, T)
    gl = np.random.default_rng(seed).standard_normal(fw["logits"].shape) / B
    xd = _t(x).requires_grad_(True)
    logits, xhat, idx = ops.head_forward(xd, _t(mu), _t(sg), _t(wt), None if gt is None else _t(gt, torch.int64), T)
    logits.backward(_t(gl))
    lg = logits.detach().cpu().numpy()
    np.testing.assert_allclose(lg, fw["logits"], rtol=TOL, atol=1e-5)
    ix = idx.cpu().numpy()
    gx_ref, dev = O.head_backward(_f64(x), _f64(mu), _f64(sg), _f64(wt), gt, T, gl, idx=ix)
    assert dev < TOL, dev
    err = normwise(xd.grad.cpu().numpy(), gx_ref)
    print("head B%d C%d K%d D%d HW%d T%d %s: logits %.2e, grad_x %.2e (pick deviation %.1e)"
          % (B, C, K, D, HW, T, "unlabelled" if gt is None else "labelled",
             np.abs(lg - fw["logits"]).max() / np.abs(fw["logits"]).max(), err, dev))
    assert err < TOL, err
    # the entries the kernel writes: every level without labels; with labels level 0 and the own class's levels
    written = np.zeros((B, P, T), bool)
    written[:, :, 0] = True
    for b in range(B):
        if gt is None:
            written[b] = True
        elif gt[b] >= 0:
            written[b, gt[b] * K:(gt[b] + 1) * K] = True
    lp = fw["logp"].reshape(B, HW, P).transpose(0, 2, 1)
    srt = -np.sort(-lp, axis=2)[:, :, :T + 1]
    gaps = srt[:, :, :-1] - srt[:, :, 1:] if HW > T else np.concatenate(
        [srt[:, :, :-1] - srt[:, :, 1:], np.full((B, P, 1), np.inf)], axis=2)
    gap_hi = np.concatenate([np.full((B, P, 1), np.inf), gaps[:, :, :T - 1]], axis=2)
    ok = written & (gap_hi > 1e-3) & (gaps[:, :, :T] > 1e-3)
    assert ok[:, :, 0].mean() > 0.5
    assert (ix[ok] == fw["idx"][ok]).all()
    if T == HW:                                      # every patch picked once
        full = written.all(axis=2)
        assert (np.sort(ix[full], axis=1) == np.arange(HW)).all()
    return fw, xhat


def _check_np_select(xhat, mu, sg, wt, gt, T, B, HW, fw):
    """head_select from an [N,P] log p (mgp_head_select_np) against the oracle's logits."""
    from mgproto_b200 import ops
    from mgproto_b200._lib import MGP_OUT_LOGP_NP
    C, K, D = mu.shape
    lp = ops.logprob(xhat, _t(mu).reshape(-1, D), _t(sg).reshape(-1, D), MGP_OUT_LOGP_NP)
    lg = ops.head_select(lp, _t(wt), None if gt is None else _t(gt, torch.int64), T, C, K, B=B, HW=HW)[0]
    np.testing.assert_allclose(lg.cpu().numpy(), fw["logits"], rtol=TOL, atol=1e-5)


# ------------------------------------------------------------------------------------ head at 417..1024 patches
LARGE = [(21, 21, 64), (21, 21, 128), (28, 28, 64), (28, 28, 128), (29, 29, 64), (29, 29, 128), (32, 32, 64),
         (32, 32, 128), (28, 28, 256)]


@pytest.mark.parametrize("H,W,D", LARGE, ids=["%dx%d-d%d" % s for s in LARGE])
def test_head_large_maps(request, H, W, D):
    """HW = 441 / 784 / 841 / 1024 (R = 14, 25, 27, 32): labelled and unlabelled head forward + backward, head_level0,
    push_search and the three log p layouts; one labelled image has no class (gt = -1)."""
    from mgproto_b200 import ops
    from mgproto_b200._lib import MGP_OUT_LOGP_BPHW
    C, K, T, B = 8, 10, 20, 3
    HW = H * W
    mu, sg, wt = HC.mixture(C, K, D, seed=100 + HW + D)
    x, gt = HC.head_batch(B, C, K, D, H, W, mu, seed=101 + HW + D, gt_fixed=(C - 1, -1, 0))
    with trace() as tr:
        fw, xhat = _check_head(x, mu, sg, wt, gt, T)
        fw0, _ = _check_head(x, mu, sg, wt, None, T, seed=6)
        if _np_select_fits(HW, C, K, T):
            _check_np_select(xhat, mu, sg, wt, None, T, B, HW, fw0)
        lv0 = ops.head_level0(_t(x), _t(mu), _t(sg), _t(wt))
        np.testing.assert_allclose(lv0.cpu().numpy(), fw0["logits"][:, :, 0], rtol=TOL, atol=1e-5)
        # push search (max / arg-max epilogue) against the argmin over the fp32 [B,P,HW] map and the oracle
        net = _net(C, K, D, T, 8, mu, sg, wt, "auto")
        labels = np.abs(gt)
        arg, val, xh = net.push_search(_t(x), _t(labels, torch.int64))
        lp = ops.logprob(xh, _t(mu).reshape(-1, D), _t(sg).reshape(-1, D), MGP_OUT_LOGP_BPHW, B=B, HW=HW)
        arg2, val2 = ops.push_argmin(lp, _t(labels, torch.int64), C, K)
        worst = _check_logprob(xh, mu, sg, B, HW)
    lp64 = fw0["logp"].reshape(B, HW, C * K).transpose(0, 2, 1)
    own = np.stack([lp64[b, labels[b] * K:(labels[b] + 1) * K] for b in range(B)])       # [B,K,HW]
    srt = -np.sort(-own, axis=2)
    sep = (srt[:, :, 0] - srt[:, :, 1]) > 1e-3
    a, a2 = arg.cpu().numpy(), arg2.cpu().numpy()
    assert sep.mean() > 0.5
    assert (a[sep] == own.argmax(2)[sep]).all() and (a2[sep] == a[sep]).all()
    np.testing.assert_allclose(val.cpu().numpy(), -np.exp(srt[:, :, 0]), rtol=TOL, atol=1e-9)
    np.testing.assert_allclose(val2.cpu().numpy(), val.cpu().numpy(), rtol=TOL, atol=1e-9)
    print("HW%d D%d: log p worst relative error %.2e" % (HW, D, worst))
    assert_reached(request, tr)


# ------------------------------------------------------------------------------------ T and drain edges
EDGES = [  # id, C, K, H, W, T, labelled, B
    ("t1-hw100-lab", 8, 10, 10, 10, 1, True, 3),
    ("t1-hw100-unl", 8, 10, 10, 10, 1, False, 3),
    ("t1-hw300-lab", 8, 10, 15, 20, 1, True, 3),
    ("t1-hw300-unl", 8, 10, 15, 20, 1, False, 3),
    ("t32-hw32-lab", 8, 10, 4, 8, 32, True, 3),     # T = HW: the picks are a permutation of the patches
    ("t32-hw32-unl", 8, 10, 4, 8, 32, False, 3),
    ("t32-c200-lab", 200, 10, 14, 14, 32, True, 2),  # C*T > 2*LCAP, and P + K(T-1) = 2310 > LCAP: two drains
]


@pytest.mark.parametrize("C,K,H,W,T,labelled,B", [e[1:] for e in EDGES], ids=[e[0] for e in EDGES])
def test_head_T_edges(request, C, K, H, W, T, labelled, B):
    D = 128
    HW = H * W
    mu, sg, wt = HC.mixture(C, K, D, seed=200 + HW + T)
    x, gt = HC.head_batch(B, C, K, D, H, W, mu, seed=201 + HW + T, gt_fixed=(C - 1, 0, C // 2))
    with trace() as tr:
        fw, xhat = _check_head(x, mu, sg, wt, gt if labelled else None, T)
        if not labelled and _np_select_fits(HW, C, K, T):
            _check_np_select(xhat, mu, sg, wt, None, T, B, HW, fw)
        worst = _check_logprob(xhat, mu, sg, B, HW)
    print("log p worst relative error %.2e" % worst)
    assert_reached(request, tr)


def test_unlabelled_backward_c200(request):
    """head(x, None) under autograd at the bench mixture: all P*T = 40 000 entries carry gradient (18 drains of the
    backward's entry list per image)."""
    C, K, D, H, W, T, B = 200, 10, 128, 14, 14, 20, 2
    mu, sg, wt = HC.mixture(C, K, D, seed=300)
    x, _ = HC.head_batch(B, C, K, D, H, W, mu, seed=301)
    with trace() as tr:
        fw, xhat = _check_head(x, mu, sg, wt, None, T)
        _check_np_select(xhat, mu, sg, wt, None, T, B, H * W, fw)
    assert_reached(request, tr)


def test_labelled_fallback_k40(request):
    """K = 40, C = 50, HW = 1024: head_top1_kernel's shared-memory layout would need > 200 KB, so the labelled head
    materialises log p and selects from it."""
    C, K, D, H, W, T, B = 50, 40, 128, 32, 32, 20, 2
    mu, sg, wt = HC.mixture(C, K, D, seed=400)
    x, gt = HC.head_batch(B, C, K, D, H, W, mu, seed=401, gt_fixed=(C - 1, 3))
    assert (2 * C * K + K * T + K * (H * W + 1) + 2 * K * D + 2 * K + 4) * 4 > 200 * 1024
    with trace() as tr:
        fw, xhat = _check_head(x, mu, sg, wt, gt, T)
        _check_np_select(xhat, mu, sg, wt, gt, T, B, H * W, fw)
    assert "head_select_kernel<32, 1, false>" in tr.kernels
    assert_reached(request, tr, absent=("head_top1_kernel",))


def test_out_of_range_shapes_are_refused():
    """T > 32, T > HW and HW > 1024 are refused by the host checks (RuntimeError), before any selection kernel runs."""
    from mgproto_b200 import ops
    C, K, D, B = 4, 3, 64, 2
    mu, sg, wt = HC.mixture(C, K, D, seed=500)
    x, gt = HC.head_batch(B, C, K, D, 4, 8, mu, seed=501)
    args = (_t(mu), _t(sg), _t(wt))
    for g in (_t(gt, torch.int64), None):
        with pytest.raises(RuntimeError, match="not supported"):
            ops.head_forward(_t(x), *args, g, 33)                           # T = 33
        with pytest.raises(RuntimeError, match="not supported"):
            ops.head_forward(_t(x[:, :, :2]), *args, g, 20)                  # T = 20 > HW = 16
    # HW = 1025: every kernel that indexes patches with 10 bits refuses the shape
    HW, P, T = 1025, C * K, 1
    g = _t(gt, torch.int64)
    with pytest.raises(RuntimeError, match="not supported"):
        ops.head_select(torch.zeros((B, P, HW), device="cuda:0"), _t(wt), g, T, C, K)
    xh = torch.zeros((B * HW, D), device="cuda:0")
    with pytest.raises(RuntimeError, match="not supported"):
        ops.head_select_top1(torch.zeros((B, P), dtype=torch.int64, device="cuda:0"), xh, _t(mu).reshape(P, D),
                             _t(sg).reshape(P, D), _t(wt), g, T, C, K, HW)
    z = torch.zeros((B, C, T), device="cuda:0")
    vi = torch.zeros((B, P, T), device="cuda:0")
    with pytest.raises(RuntimeError, match="not supported"):
        ops.head_backward(z, z, vi, vi.int(), _t(wt), g, xh, torch.ones(B * HW, device="cuda:0"), _t(mu).reshape(P, D),
                          _t(sg).reshape(P, D), (B, HW, C, K, D, T, 25, 41))


# ------------------------------------------------------------------------------------ EM at every instantiation
EM_CASES = [(2, 128, 37), (5, 128, 64), (5, 128, 1000), (7, 128, 65), (11, 128, 200), (16, 128, 8), (16, 128, 1000),
            (3, 256, 50), (5, 256, 200), (10, 256, 64), (16, 256, 129), (1, 128, 50),
            (2, 64, 37), (10, 64, 65), (16, 64, 200)]
# every case also runs sparse: a random quarter, then half, of the classes flagged, so that most blocks only replay
# the others' Adam steps and, in the tensor-core kernel at D = 128 (active classes first), run classes far from their
# own index
EM_RUNS = [(K, D, cap, path, sparse) for K, D, cap in EM_CASES
           for path in {64: ("fused",), 128: ("tc", "fused"), 256: ("tc",)}[D] for sparse in (False, True)]


@functools.lru_cache(maxsize=None)
def _em_case(K, D, cap, sparse=False):
    """Seeded inputs and the float64 oracle's two successive update_GMM calls (ref model.py:277-301)."""
    from oracle import mgproto_oracle as O
    C = 40 if cap < 1000 else 12
    mu, sg, wt = HC.mixture(C, K, D, seed=600 + K + D + cap)
    rows = HC.bank_rows(C, K, D, cap, mu, seed=601 + cap)
    n_active = (C // 4, C // 2) if sparse else (C, C - 7)
    am, av, flags, short, step0 = HC.em_state(C, K, D, seed=602 + K, n_active=n_active, n_short=2, step0=500)
    short_len = cap // 2
    bank = O.MemoryBankOracle(C, D, cap, dtype=np.float64)
    bank.data[:] = rows
    bank.mem_len[:] = cap
    bank.mem_len[short] = short_len
    adam = O.AdamOracle((C, K, D), lr=3e-3)
    adam.m, adam.v, adam.t = _f64(am), _f64(av), step0
    ref, m, w = [], _f64(mu), _f64(wt)
    for f in flags:
        m, w, _ = O.update_gmm(bank, f, m, _f64(sg), w, adam)
        ref.append((m, w))
    return dict(C=C, mu=mu, sg=sg, wt=wt, rows=rows, am=am, av=av, flags=flags, short=short, short_len=short_len,
                step0=step0, ref=ref, adam=(adam.m, adam.v, adam.t))


@pytest.mark.parametrize("K,D,cap,path,sparse", EM_RUNS,
                         ids=["k%d-d%d-cap%d-%s" % r[:4] + ("-sparse" if r[4] else "") for r in EM_RUNS])
def test_em_instantiations(request, K, D, cap, path, sparse):
    """Two update_GMM calls (all classes flagged, then all but 7, or sparse: a quarter, then half; two classes short;
    Adam at step 500): mu (whole and per class), the movement, pi, both Adam moments and the step count against the
    float64 oracle."""
    g = _em_case(K, D, cap, sparse)
    C = g["C"]
    net = _net(C, K, D, 20, cap, g["mu"], g["sg"], g["wt"], "auto")
    _fill_bank(net, g["rows"], g["short"], g["short_len"])
    _seed_adam(net, g["am"], g["av"], g["step0"])
    outs = []
    with em_path(path), trace() as tr:
        for f in g["flags"]:
            net.queue.updated |= _t(f, torch.uint8)
            net.update_GMM()
            outs.append((net.prototype_means.detach().cpu().numpy().copy(), net.last_layer.weight.cpu().numpy().copy()))
        net.sync_optimizer_state()
    mu0 = _f64(g["mu"])
    for i, ((mu_got, wt_got), (mu_ref, wt_ref)) in enumerate(zip(outs, g["ref"])):
        e_mu = normwise(mu_got, mu_ref)
        e_mv = normwise(_f64(mu_got) - mu0, mu_ref - mu0)
        d = np.abs(_f64(mu_got) - mu_ref).reshape(C, -1).max(1) / np.abs(mu_ref).reshape(C, -1).max(1)
        e_pi = float((np.abs(wt_got - wt_ref) / np.maximum(np.abs(wt_ref), 1e-30))[wt_ref != 0].max())
        print("EM K%d D%d cap%d [%s] call %d: mu %.2e, per class %.2e, movement %.2e, pi %.2e"
              % (K, D, cap, path, i, e_mu, d.max(), e_mv, e_pi))
        assert e_mu < TOL and d.max() < TOL and e_mv < 1e-3, (i, e_mu, d.max(), e_mv)
        np.testing.assert_allclose(wt_got, wt_ref, rtol=TOL, atol=1e-9)
    m_ref, v_ref, t_ref = g["adam"]
    st = net.prototype_optimizer.state[net.prototype_means]
    assert int(st["step"]) == t_ref
    e_m, e_v = normwise(st["exp_avg"].cpu().numpy(), m_ref), normwise(st["exp_avg_sq"].cpu().numpy(), v_ref)
    print("EM K%d D%d cap%d [%s]: Adam moments %.2e / %.2e" % (K, D, cap, path, e_m, e_v))
    assert e_m < TOL and e_v < TOL
    # K = 1: neither the tensor-core nor the fused kernel takes it (multi-launch path); the fused switch never runs em_tc
    absent = ("em_tc_kernel", "em_fused_kernel") if K == 1 else (("em_tc_kernel",) if path == "fused" else ())
    assert_reached(request, tr, absent=absent)
