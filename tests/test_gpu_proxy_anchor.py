"""The Proxy-Anchor auxiliary loss on the GPU (mgproto_b200.losses.Proxy_Anchor / ops.proxy_anchor, -m gpu) against
the float64 oracle (tests/proxy_anchor_oracle.py, pinned to the reference by tests/test_oracle_proxy_anchor.py): loss
1e-5 relative, both gradients 1e-5 norm-wise (max |err| / max |ref|).  Which of the three kernels (one per embedding
dtype) runs for which input, and that nothing is copied to the host, is asserted under torch.profiler in a process of
its own (test_each_dtype_runs_its_own_kernel).  Nothing here tries to make the device fault: the refused shapes are
refused by the host checks."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import proxy_anchor_oracle as PA

pytestmark = pytest.mark.gpu

KERNELS = {torch.float32: "proxy_anchor_f32_kernel", torch.bfloat16: "proxy_anchor_bf16_kernel",
           torch.float16: "proxy_anchor_f16_kernel"}
TOL = 1e-5


def _dev():
    return torch.device("cuda:0")


def _collinear():
    """Embeddings that are positive or negative multiples of proxies: cosines of +1 and -1, the largest exponents."""
    X, P, t = PA.problem(64, 20, 32, seed=11)
    for b in range(64):
        X[b] = (1.0 + 0.25 * b) * P[(b * 7) % 20] * (-1.0 if b % 3 == 0 else 1.0)
    return X, P, t


def _zero_proxy():
    X, P, t = PA.problem(64, 20, 32, seed=12)
    P[3] = 0.0                                          # the 1e-12 inside the root keeps 0 / |0| finite
    t[5] = 3
    return X, P, t


def _some_unlabelled():
    X, P, t = PA.problem(256, 200, 32, seed=13)
    t[::4] = -1
    t[2] = 200                                          # C itself is outside [0, C) too
    return X, P, t


def _far_positive():
    """Every present class has one positive, and one of them sits on its proxy: S+ = e^-28.8, where log(1 + S) needs log1p."""
    X, P, t = PA.problem(32, 40, 32, seed=14, rule="all")
    X[4] = 3.0 * P[t[4]]
    return X, P, t


CASES = {
    "golden-repeat": lambda: PA.case("repeat"),
    "golden-batch80": lambda: PA.case("batch80"),
    "golden-oneclass": lambda: PA.case("oneclass"),
    "b256-c200-e32": lambda: PA.problem(256, 200, 32, seed=1),
    "b1": lambda: PA.problem(1, 200, 32, seed=2),
    "b4096": lambda: PA.problem(4096, 200, 32, seed=3),                 # 7 image tiles
    "c2": lambda: PA.problem(64, 2, 32, seed=4),
    "c4096": lambda: PA.problem(256, 4096, 32, seed=5),                 # 7 proxy tiles, 512 classes per CTA
    "e4": lambda: PA.problem(256, 200, 4, seed=6),
    "e512": lambda: PA.problem(256, 200, 512, seed=7),                  # 16 accumulators per lane, tiles of 32 rows
    "e100-two-tiles": lambda: PA.problem(300, 150, 100, seed=8),        # 4 accumulators per lane, the last one partial
    "b1000-c777-e260": lambda: PA.problem(1000, 777, 260, seed=9),      # ragged everything, 16 and 13 tiles
    "one-class": lambda: PA.problem(256, 200, 32, seed=10, rule="one"),
    "every-class": lambda: PA.problem(400, 200, 32, seed=15, rule="all"),
    "quarter-unlabelled": _some_unlabelled,
    "collinear": _collinear,
    "zero-proxy": _zero_proxy,
    "far-positive": _far_positive,
}


def _run(X, P, t, dtype=torch.float32, mrg=0.1, beta=32.0):
    """-> (loss, grad_x, grad_p) tensors through autograd."""
    from mgproto_b200 import ops
    x = torch.from_numpy(X).to(_dev()).to(dtype).requires_grad_(True)
    p = torch.from_numpy(P).to(_dev()).requires_grad_(True)
    loss = ops.proxy_anchor(x, p, torch.from_numpy(t).to(_dev()), mrg, beta)
    gx, gp = torch.autograd.grad(loss, [x, p])
    assert loss.dim() == 0 and loss.dtype == torch.float32 and gx.dtype == dtype and gp.dtype == torch.float32
    return loss.detach(), gx, gp


# Runs in a fresh interpreter: forward + backward of one call per (dtype, width class) inside a torch.profiler window
# each, printing the window's event names.
_PROFILE_SCRIPT = """
import json, sys, torch
from torch.profiler import ProfilerActivity, profile
from mgproto_b200 import losses
dev = torch.device("cuda:0")
out = {}
for name, dtype in (("f32", torch.float32), ("bf16", torch.bfloat16), ("f16", torch.float16)):
    for E in (32, 100, 512):
        crit = losses.Proxy_Anchor(40, E).to(dev)
        x = torch.randn(64, E, device=dev).to(dtype).requires_grad_(True)
        t = torch.randint(0, 40, (64,), device=dev)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            crit(x, t).backward()
            torch.cuda.synchronize()
        out["%s-e%d" % (name, E)] = sorted({e.key for e in prof.key_averages()})
print("KEYS " + json.dumps(out))
"""


def test_each_dtype_runs_its_own_kernel():
    """Under torch.profiler, for fp32 / bf16 / fp16 embeddings at one width of each accumulator class: the window holds
    the dtype's kernel, neither of the other two, and no copy to or from the host.

    The windows are taken in a process of their own.  Late in a long pytest session that has opened many profiler
    windows, the device records of this library's kernels go missing from a window now and then (the runtime record of
    the launch and the ATen kernels around it are kept), and every further window moves where that happens for the
    modules that run later; a young process returns complete windows and leaves the session's profiler alone."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _PROFILE_SCRIPT], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    line = [ln for ln in r.stdout.splitlines() if ln.startswith("KEYS ")][-1]
    windows = json.loads(line[5:])
    assert len(windows) == 9
    names = {"f32": "proxy_anchor_f32_kernel", "bf16": "proxy_anchor_bf16_kernel", "f16": "proxy_anchor_f16_kernel"}
    for case, keys in windows.items():
        ran = {n for n in names.values() if any(n in k for k in keys)}
        assert ran == {names[case.split("-")[0]]}, (case, keys)
        assert not any("Memcpy DtoH" in k or "Memcpy HtoD" in k for k in keys), (case, keys)


def _check(X, P, t, loss, gx, gp, tol=TOL):
    want_l, want_x, want_p = PA.proxy_anchor(X, P, t)
    assert torch.isfinite(loss) and torch.isfinite(gx).all() and torch.isfinite(gp).all()
    assert abs(float(loss) - want_l) <= tol * abs(want_l), (float(loss), want_l)
    ex, ep = PA.normwise(gx.double().cpu().numpy(), want_x), PA.normwise(gp.double().cpu().numpy(), want_p)
    assert ex < tol and ep < tol, (ex, ep)


@pytest.mark.parametrize("name", sorted(CASES))
def test_against_float64(name):
    X, P, t = CASES[name]()
    _check(X, P, t, *_run(X, P, t))


def test_golden_cases_match_the_reference_outputs():
    import os
    z = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "proxy_anchor.npz"))
    for name in PA.GOLDEN_CASES:
        X, P, t = PA.case(name)
        loss, gx, gp = _run(X, P, t, mrg=float(z["mrg"]), beta=float(z["beta"]))
        assert abs(float(loss) - float(z[name + "_loss"])) < 1e-5 * float(z[name + "_loss"])
        assert PA.normwise(gx.cpu().numpy(), z[name + "_grad_x"]) < 1e-5
        assert PA.normwise(gp.cpu().numpy(), z[name + "_grad_p"]) < 1e-5


def test_margin_and_scale_are_arguments():
    X, P, t = PA.problem(96, 30, 64, seed=21)
    loss, gx, gp = _run(X, P, t, mrg=0.3, beta=8.0)
    want_l, want_x, want_p = PA.proxy_anchor(X, P, t, 0.3, 8.0)
    assert abs(float(loss) - want_l) < TOL * abs(want_l)
    assert PA.normwise(gx.cpu().numpy(), want_x) < TOL and PA.normwise(gp.cpu().numpy(), want_p) < TOL


def test_no_class_present():
    """All labels -1: the loss is the negative term over no image = sum of log 1 = 0, the gradients are 0, nothing NaN."""
    from mgproto_b200 import ops
    X, P, t = PA.problem(64, 20, 32, seed=22)
    t[:] = -1
    loss, gx, gp = _run(X, P, t)
    assert float(loss) == 0.0 and not gx.any() and not gp.any()
    _, _, _, nv = ops._proxy_anchor(torch.from_numpy(X).to(_dev()), torch.from_numpy(P).to(_dev()),
                                    torch.from_numpy(t).to(_dev()), 0.1, 32.0, False, False)
    assert int(nv) == 0


def test_n_valid_counts_the_classes_present():
    from mgproto_b200 import ops
    X, P, t = _some_unlabelled()
    _, _, _, nv = ops._proxy_anchor(torch.from_numpy(X).to(_dev()), torch.from_numpy(P).to(_dev()),
                                    torch.from_numpy(t).to(_dev()), 0.1, 32.0, False, False)
    assert int(nv) == len(set(t[(t >= 0) & (t < 200)].tolist()))


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("shape", [(256, 200, 32), (300, 150, 100), (64, 40, 512)])
def test_16bit_embeddings_equal_the_fp32_path(dtype, shape):
    """bf16 / fp16 embeddings: loss and grad_p bit for bit what the fp32 kernel gives for X.float(); grad_x the same
    values rounded to X's dtype."""
    X, P, t = PA.problem(*shape, seed=31)
    X16 = torch.from_numpy(X).to(dtype)
    Xf = X16.float().numpy()
    l16, gx16, gp16 = _run(Xf, P, t, dtype=dtype)             # Xf is exactly representable: .to(dtype) is lossless
    l32, gx32, gp32 = _run(Xf, P, t)
    assert torch.equal(l16, l32) and torch.equal(gp16, gp32)
    assert torch.equal(gx16, gx32.to(dtype))
    _check(Xf, P, t, l16, gx32, gp16)


def test_through_autograd_with_a_cross_entropy_term():
    """coefs['aux'] * criterion(x_embed, t) added to a CE term (ref train_and_test.py:42, :55): gradients of the proxies
    and of the tensor that feeds the embedding layer."""
    from mgproto_b200 import losses
    torch.manual_seed(0)
    B, C, E, F = 80, 200, 32, 48
    crit = losses.Proxy_Anchor(C, E).to(_dev())
    lin = torch.nn.Linear(F, E).to(_dev())
    feat = torch.randn(B, F, device=_dev(), requires_grad=True)
    logits = torch.randn(B, C, device=_dev(), requires_grad=True)
    t = torch.randint(0, C, (B,), device=_dev())
    x_embed = lin(feat)
    loss = torch.nn.functional.cross_entropy(logits, t) + 0.5 * crit(x_embed, t)
    loss.backward()
    Xn, Pn = x_embed.detach().cpu().numpy(), crit.proxies.detach().cpu().numpy()
    want_l, want_x, want_p = PA.proxy_anchor(Xn, Pn, t.cpu().numpy())
    assert PA.normwise(crit.proxies.grad.cpu().numpy(), 0.5 * want_p) < TOL
    want_feat = (0.5 * want_x) @ lin.weight.detach().double().cpu().numpy()
    assert PA.normwise(feat.grad.cpu().numpy(), want_feat) < 1e-4          # through an fp32 ATen GEMM
    ce = torch.nn.functional.cross_entropy(logits.detach(), t)
    assert abs(float(loss.detach()) - float(ce) - 0.5 * want_l) < 1e-5 * abs(want_l)


def test_null_gradient_pointers_without_grad(monkeypatch):
    """Under torch.no_grad() (evaluation) both gradient pointers are null; with only the proxies requiring a gradient,
    grad_x is null."""
    from mgproto_b200 import _lib, losses
    lib = _lib.load()
    seen = []

    class Spy:
        def __getattr__(self, name):
            fn = getattr(lib, name)
            if name != "mgp_proxy_anchor":
                return fn

            def wrapped(*a):
                seen.append((a[10], a[11]))
                return fn(*a)
            return wrapped

    monkeypatch.setattr(_lib, "load", lambda: Spy())
    crit = losses.Proxy_Anchor(20, 32).to(_dev())
    X, _, t = PA.problem(64, 20, 32, seed=41)
    x, tt = torch.from_numpy(X).to(_dev()), torch.from_numpy(t).to(_dev())
    with torch.no_grad():
        l0 = crit(x, tt)
    assert seen[-1] == (0, 0) and not l0.requires_grad
    l1 = crit(x, tt)
    assert seen[-1][0] == 0 and seen[-1][1] != 0 and l1.requires_grad
    l1.backward()
    l2 = crit(x.clone().requires_grad_(True), tt)
    assert seen[-1][0] != 0 and seen[-1][1] != 0
    assert torch.equal(l0, l1.detach()) and torch.equal(l0, l2.detach())       # the loss does not depend on the skipped passes
    want = PA.proxy_anchor(X, crit.proxies.detach().cpu().numpy(), t)
    assert PA.normwise(crit.proxies.grad.cpu().numpy(), want[2]) < TOL


def test_no_host_synchronisation_and_one_launch():
    from mgproto_b200 import losses, ops
    crit = losses.Proxy_Anchor(200, 32).to(_dev())
    x = torch.randn(256, 32, device=_dev(), requires_grad=True)
    t = torch.randint(0, 200, (256,), device=_dev())
    crit(x, t).backward()                                                      # first call: module load, allocator warm-up
    torch.cuda.synchronize()
    before = ops.launch_count()
    prev = torch.cuda.get_sync_debug_mode()
    torch.cuda.set_sync_debug_mode("error")
    try:
        loss = crit(x, t)
        assert ops.launch_count() == before + 1
        (0.5 * loss).backward()
        assert ops.launch_count() == before + 1
    finally:
        torch.cuda.set_sync_debug_mode(prev)

def test_capture_and_determinism():
    """Forward + backward + an SGD update of the proxies captured into a CUDA graph and replayed on three batches (the
    number of classes present changes between them): bit-identical to the eager run.  Two eager runs agree bit for bit."""
    from mgproto_b200 import losses
    B, C, E = 80, 200, 32
    torch.manual_seed(1)
    batches = []
    for i, rule in enumerate(("random", "one", "all")):
        X, _, t = PA.problem(B, C, E, seed=50 + i, rule=rule)
        batches.append((torch.from_numpy(X).to(_dev()), torch.from_numpy(t).to(_dev())))
    batches[1][1][::5] = -1

    def train(crit, step):
        out = []
        for x, t in batches:
            out.append(step(crit, x, t))
        return out, crit.proxies.detach().clone()

    def eager_step(crit, x, t):
        x = x.clone().requires_grad_(True)
        crit.proxies.grad = None
        loss = crit(x, t)
        loss.backward()
        with torch.no_grad():
            crit.proxies.add_(crit.proxies.grad, alpha=-0.1)
        return loss.detach().clone(), x.grad.clone()

    crit0 = losses.Proxy_Anchor(C, E).to(_dev())
    init = crit0.proxies.detach().clone()
    eager, p_eager = train(crit0, eager_step)
    with torch.no_grad():
        crit0.proxies.copy_(init)
    again, p_again = train(crit0, eager_step)
    for (l0, g0), (l1, g1) in zip(eager, again):
        assert torch.equal(l0, l1) and torch.equal(g0, g1)
    assert torch.equal(p_eager, p_again)
    assert len({float(l) for l, _ in eager}) == 3

    crit = losses.Proxy_Anchor(C, E).to(_dev())
    with torch.no_grad():
        crit.proxies.copy_(init)
    sx = torch.zeros(B, E, device=_dev(), requires_grad=True)
    st = torch.zeros(B, dtype=torch.int64, device=_dev())
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):                                              # warm-up outside the capture
        (gx0, gp0) = torch.autograd.grad(crit(sx, st), [sx, crit.proxies])
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        s_loss = crit(sx, st)
        s_gx, s_gp = torch.autograd.grad(s_loss, [sx, crit.proxies])
        with torch.no_grad():
            crit.proxies.add_(s_gp, alpha=-0.1)
    with torch.no_grad():
        crit.proxies.copy_(init)
    for (x, t), (l0, g0) in zip(batches, eager):
        sx.data.copy_(x)
        st.copy_(t)
        graph.replay()
        assert torch.equal(s_loss.detach(), l0) and torch.equal(s_gx, g0)
    assert torch.equal(crit.proxies.detach(), p_eager)


@pytest.mark.parametrize("B,C,E", [(8, 5, 6), (8, 5, 516), (8, 1, 16), (0, 5, 16), (8, 4097, 16), (4097, 5, 16)])
def test_shapes_outside_the_envelope_raise(B, C, E):
    from mgproto_b200 import ops
    before = ops.launch_count()
    x = torch.zeros(B, E, device=_dev())
    p = torch.zeros(C, E, device=_dev())
    t = torch.zeros(B, dtype=torch.int64, device=_dev())
    with pytest.raises(RuntimeError, match="mgp_proxy_anchor"):
        ops.proxy_anchor(x, p, t)
    assert ops.launch_count() == before
    with pytest.raises(RuntimeError):
        ops.proxy_anchor(x.double(), p, t)
