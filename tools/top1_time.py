#!/usr/bin/env python
"""Time the labelled step's max / arg-max log-likelihood kernel (logprob_top1_wide_kernel at cfg2) with the ablation
switches of MGP_TC_DEBUG: 1 no global results, 4 no MMAs, 8 no epilogue work, 16 no prototype loads.
The operands are pre-staged without telling the host that sigma is isotropic, so each launch also includes the
zeroing of the output and the 128-patch-tile kernel, which returns at once (the anisotropic fallback)."""
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mgproto_b200 import _lib, ops                 # noqa: E402

dev = torch.device("cuda:0")
torch.cuda.set_device(0)
lib = _lib.load()
B, HW, P, D = 256, 196, 2000, int(os.environ.get("KA_D", "128"))
N = B * HW
g = torch.Generator().manual_seed(0)
xs = [F.normalize(torch.randn(N, D, generator=g), dim=1).to(dev) for _ in range(6)]
mu = F.normalize(torch.rand(P, D, generator=g), dim=1).to(dev)
sg = torch.full((P, D), 0.3989, device=dev)
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
flops = 2.0 * 3 * N * P * D
for dbg in os.environ.get("KA_DEBUGS", "0,2,4,8,16,6,12,10").split(","):
    os.environ["MGP_TC_DEBUG"] = dbg
    wss = [ops.logprob_top1(xs[i], mu, sg, B, HW, "tc", return_ws=True)[1] for i in range(6)]
    for i in range(3):
        ops.logprob_top1(xs[i % 6], mu, sg, B, HW, "tc_reuse", ws=wss[i % 6])
    torch.cuda.synchronize()
    torch.cuda._sleep(10_000_000)
    e0.record()
    for i in range(20):
        ops.logprob_top1(xs[i % 6], mu, sg, B, HW, "tc_reuse", ws=wss[i % 6])
    e1.record()
    torch.cuda.synchronize()
    t = e0.elapsed_time(e1) / 20 * 1e-3
    print("debug=%-3s %.1f us per launch (memset + kernels, operands pre-staged)  %.0f TFLOP/s equivalent" % (dbg, t * 1e6, flops / t / 1e12))
os.environ["MGP_TC_DEBUG"] = "0"
