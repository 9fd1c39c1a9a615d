"""Per-patch class log-densities (ops.log_density / MGProto.log_density_maps, -m gpu) against the float64 oracle
(tests/log_density_oracle.py, pinned to the reference's _score by tests/test_oracle_log_density.py): 1e-4 element-wise
relative on logp_c [B,C,H,W] and logp_all [B,H,W].  Every case asserts under torch.profiler which of the new kernels
ran: the tensor-core kernel for isotropic sigma, D in {64, 128}, K <= 64, the chunked fallback otherwise."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import log_density_oracle as LD
from test_gpu_shape_edges import trace

pytestmark = pytest.mark.gpu

RTOL, ATOL = 1e-4, 1e-5
TC = {64: "log_density_tc_d64_kernel", 128: "log_density_tc_d128_kernel"}
FALLBACK = "log_density_lse_kernel"
# classes per K: C*K is never a multiple of the 128-column tile, and the last class-aligned tile is partial
CLASSES = {1: 300, 10: 29, 16: 19, 40: 7, 64: 5, 80: 3}


def _dev():
    return torch.device("cuda:0")


def _problem(B, H, W, C, K, D, iso=True, seed=0):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, D, H, W, generator=g)
    mu = F.normalize(torch.randn(C, K, D, generator=g), dim=2)
    if iso:      # sigma constant over d inside a prototype, different between prototypes
        sg = (0.25 + 0.2 * torch.rand(C, K, 1, generator=g)).expand(C, K, D).contiguous()
    else:
        sg = 0.25 + 0.2 * torch.rand(C, K, D, generator=g)
    pi = torch.softmax(torch.randn(C, K, generator=g), dim=1)
    if K > 1:
        pi[::3, K - 1] = 0.0                          # pruned prototypes: log(0 + 1e-10)
    wt = torch.zeros(C, C * K)
    for c in range(C):
        wt[c, c * K:(c + 1) * K] = pi[c]
    return x, mu, sg, wt


def _oracle(x, mu, sg, wt):
    return LD.log_density_maps(*(t.double().numpy() for t in (x, mu, sg, wt)))


def _run(x, mu, sg, wt, math):
    from mgproto_b200 import ops
    B, D, H, W = x.shape
    C, K, _ = mu.shape
    xhat, _, _ = ops.normalize_fwd(x.to(_dev()))
    lc, la = ops.log_density(xhat, mu.reshape(C * K, D).to(_dev()), sg.reshape(C * K, D).to(_dev()), wt.to(_dev()),
                             B, H * W, C, K, math=math)
    return lc.view(B, C, H, W), la.view(B, H, W)


def _close(got, want):
    np.testing.assert_allclose(got.cpu().numpy(), want, rtol=RTOL, atol=ATOL)


def _expect(tr, kernel):
    new = {FALLBACK} | set(TC.values())
    assert kernel in tr.kernels, (kernel, sorted(tr.kernels))
    assert not (new - {kernel}) & tr.kernels, sorted(tr.kernels)


@pytest.mark.parametrize("HW", [32, 196, 784, 1024, 1600])
@pytest.mark.parametrize("K", [1, 10, 16, 40, 64])
def test_tensor_core_d128(K, HW):
    H = {32: 4, 196: 14, 784: 28, 1024: 32, 1600: 40}[HW]
    x, mu, sg, wt = _problem(2, H, HW // H, CLASSES[K], K, 128, seed=K * 7919 + HW)
    with trace() as tr:
        lc, la = _run(x, mu, sg, wt, "auto")
    _expect(tr, TC[128])
    want_c, want_a = _oracle(x, mu, sg, wt)
    _close(lc, want_c)
    _close(la, want_a)


@pytest.mark.parametrize("K,HW", [(1, 196), (10, 1024), (16, 32), (40, 784), (64, 1600)])
def test_tensor_core_d64(K, HW):
    H = {32: 4, 196: 14, 784: 28, 1024: 32, 1600: 40}[HW]
    x, mu, sg, wt = _problem(3, H, HW // H, CLASSES[K], K, 64, seed=K + HW)
    with trace() as tr:
        lc, la = _run(x, mu, sg, wt, "tc")
    _expect(tr, TC[64])
    want_c, want_a = _oracle(x, mu, sg, wt)
    _close(lc, want_c)
    _close(la, want_a)


@pytest.mark.parametrize("math", ["auto", "tc", "tc_iso", "fp32"])
def test_math_modes(math):
    """Isotropic D = 128, K = 10: 'fp32' takes the fallback (SIMT log-likelihood), the others the tensor cores."""
    x, mu, sg, wt = _problem(3, 14, 14, 29, 10, 128, seed=5)
    with trace() as tr:
        lc, la = _run(x, mu, sg, wt, math)
    _expect(tr, FALLBACK if math == "fp32" else TC[128])
    want_c, want_a = _oracle(x, mu, sg, wt)
    _close(lc, want_c)
    _close(la, want_a)


@pytest.mark.parametrize("D,K,iso,math", [
    (128, 10, False, "auto"), (128, 10, False, "tc"), (128, 10, False, "fp32"),   # anisotropic sigma
    (128, 80, True, "auto"),                                                      # K > 64
    (256, 10, True, "auto"), (256, 10, False, "auto"), (256, 10, False, "fp32"),
    (512, 5, True, "auto"), (512, 5, False, "fp32"),
])
def test_fallback(D, K, iso, math):
    x, mu, sg, wt = _problem(2, 14, 14, CLASSES.get(K, 7) if D <= 128 else 7, K, D, iso=iso, seed=D + K)
    with trace() as tr:
        lc, la = _run(x, mu, sg, wt, math)
    _expect(tr, FALLBACK)
    want_c, want_a = _oracle(x, mu, sg, wt)
    _close(lc, want_c)
    _close(la, want_a)


def test_fallback_row_chunks():
    """More [n, P] rows than one fallback chunk holds (16 Mi floats): the chunk loop and its row offsets, against the
    tensor-core kernel (both are checked against float64 above)."""
    x, mu, sg, wt = _problem(2, 50, 60, 700, 10, 64, seed=3)      # N = 6000, P = 7000: 2396 rows per chunk, 3 chunks
    with trace() as tr:
        lc, la = _run(x, mu, sg, wt, "fp32")
    _expect(tr, FALLBACK)
    with trace() as tr:
        tc_c, tc_a = _run(x, mu, sg, wt, "auto")
    _expect(tr, TC[64])
    np.testing.assert_allclose(lc.cpu().numpy(), tc_c.cpu().numpy(), rtol=RTOL, atol=ATOL)
    np.testing.assert_allclose(la.cpu().numpy(), tc_a.cpu().numpy(), rtol=RTOL, atol=ATOL)


def _net(C, K, D):
    import mgproto_b200 as M
    torch.manual_seed(0)
    return M.MGProto(features=nn.Sequential(nn.Conv2d(3, 8, 1)), img_size=14, prototype_shape=(C * K, D, 1, 1),
                     proto_layer_rf_info=None, num_classes=C, add_on_layers_type="regular", sz_embedding=8,
                     mem_capacity=10, mine_K=4).to(_dev())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("channels_last", [False, True])
def test_model_feature_formats(dtype, channels_last):
    """MGProto.log_density_maps on every feature format the head accepts, against the oracle on x.float()."""
    C, K, D = 20, 10, 128
    net = _net(C, K, D)
    with torch.no_grad():
        net.last_layer.weight[3, 3 * K:3 * K + 4] = 0.0            # pruned prototypes
    x = torch.randn(4, D, 14, 14, device=_dev()).to(dtype)
    if channels_last:
        x = x.to(memory_format=torch.channels_last)
    with trace() as tr:
        lc, la = net.log_density_maps(x)
    _expect(tr, TC[128])
    assert lc.shape == (4, C, 14, 14) and la.shape == (4, 14, 14) and lc.dtype == torch.float32
    want_c, want_a = _oracle(x.float().cpu(), net.prototype_means.detach().cpu(), net.prototype_covs.cpu(),
                             net.last_layer.weight.detach().cpu())
    _close(lc, want_c)
    _close(la, want_a)


def test_equals_score_class_by_class():
    """logp_c equals MGProto._score(..., as_average=False) run class by class on the same normalised rows."""
    from mgproto_b200 import ops
    C, K, D = 12, 10, 128
    net = _net(C, K, D)
    x = torch.randn(3, D, 14, 14, device=_dev())
    lc, _ = net.log_density_maps(x)
    xhat, _, _ = ops.normalize_fwd(x)
    for c in range(C):
        pi = net.last_layer.weight[c, c * K:(c + 1) * K].view(1, K, 1)
        s = net._score(xhat.unsqueeze(1), net.prototype_means[c].unsqueeze(0), net.prototype_covs[c].unsqueeze(0), pi,
                       as_average=False)
        got = lc[:, c].reshape(-1)                                  # rows n = b HW + hw, as xhat
        np.testing.assert_allclose(got.cpu().numpy(), s.cpu().numpy(), rtol=RTOL, atol=ATOL)


def test_operand_cache_follows_mu():
    """Unchanged mu / sigma: the second call skips the prototype pre-pass; after an in-place change of mu it runs
    again and the result follows the new mu."""
    C, K, D = 20, 10, 128
    net = _net(C, K, D)
    x = torch.randn(2, D, 14, 14, device=_dev())
    with trace() as tr1:
        first, _ = net.log_density_maps(x)
    with trace() as tr2:
        again, _ = net.log_density_maps(x)
    assert "tc_proto_prep_kernel" in tr1.kernels and TC[128] in tr1.kernels
    assert "tc_proto_prep_kernel" not in tr2.kernels and TC[128] in tr2.kernels
    assert torch.equal(first, again)
    with torch.no_grad():
        net.prototype_means.mul_(0.9)
    with trace() as tr3:
        lc, la = net.log_density_maps(x)
    assert "tc_proto_prep_kernel" in tr3.kernels
    want_c, want_a = _oracle(x.cpu(), net.prototype_means.detach().cpu(), net.prototype_covs.cpu(),
                             net.last_layer.weight.detach().cpu())
    _close(lc, want_c)
    _close(la, want_a)


def test_without_marginal_and_deterministic():
    """out_bhw = NULL writes logp_c alone; two runs give the same bits (one writer per element, fixed sum order)."""
    from mgproto_b200 import ops
    x, mu, sg, wt = _problem(2, 14, 14, 29, 10, 128, seed=9)
    a_c, a_a = _run(x, mu, sg, wt, "auto")
    b_c, b_a = _run(x, mu, sg, wt, "auto")
    assert torch.equal(a_c, b_c) and torch.equal(a_a, b_a)
    xhat, _, _ = ops.normalize_fwd(x.to(_dev()))
    c, none = ops.log_density(xhat, mu.reshape(-1, 128).to(_dev()), sg.reshape(-1, 128).to(_dev()), wt.to(_dev()),
                              2, 196, 29, 10, want_all=False)
    assert none is None and torch.equal(c, a_c.view(2, 29, 196))
