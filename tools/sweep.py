#!/usr/bin/env python
"""BASELINE.json configs[3]: prototype sweep on 1 GPU, K in {5,10,20,40} x D in {64,128,256,512}, B=256, C=200:
achieved algorithmic HBM GB/s of the [N,P] log-likelihood op against the measured roof.  Prints a markdown table."""
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mgproto_b200 import ops  # noqa: E402

peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"] if os.path.exists(
    os.path.join(ROOT, "MEASURED_PEAKS.json")) else 3350.0
dev = torch.device("cuda:0")
B, HW, C = 256, 196, 200
N = B * HW
print("| K | D | P | path | us / launch | algorithmic GB/s | frac of %.0f GB/s | pairs/s |" % peak)
print("|---|---|---|---|---|---|---|---|")
for D in (64, 128, 256, 512):
    g = torch.Generator().manual_seed(D)
    x = F.normalize(torch.randn(N, D, generator=g), dim=1).to(dev)
    for K in (5, 10, 20, 40):
        P = C * K
        mu = F.normalize(torch.rand(P, D, generator=g), dim=1).to(dev)
        sg = torch.full((P, D), 0.3989422804, device=dev)
        out = torch.empty(N, P, device=dev)
        path = "wgmma fp16x3" if D in (64, 128, 256) else "fp32 SIMT"
        for _ in range(3):
            ops.logprob(x, mu, sg, 0, math="auto", out=out)
        torch.cuda.synchronize()
        reps = 10 if D < 512 else 3
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(reps):
            ops.logprob(x, mu, sg, 0, math="auto", out=out)
        e1.record()
        torch.cuda.synchronize()
        t = e0.elapsed_time(e1) / reps / 1e3
        by = 4.0 * (N * D + 2 * P * D + N * P)
        print("| %d | %d | %d | %s | %.1f | %.0f | %.3f | %.3g |" % (K, D, P, path, t * 1e6, by / t / 1e9, by / t / 1e9 / peak,
                                                                    N * P / t))
        del out, mu, sg
    del x
