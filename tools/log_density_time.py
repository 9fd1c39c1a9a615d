#!/usr/bin/env python
"""Time ops.log_density (per-patch class log-densities, one tensor-core kernel) at cfg2 against the composed route that
produces the same two outputs: compute_log_prob's [N,P] log-likelihood (ops.logprob, _estimate_log_prob's eps) +
torch logsumexp over each class's K prototypes and over the classes.

    python tools/log_density_time.py [--blocks 7] [--iters 20]

CUDA events around blocks of `iters` calls after a warm-up; the median block is reported per route, the routes
alternated block by block.  Prints the card name and power limit read in the same run, the achieved TFLOP/s of the
three fp16 passes (3 x 2 N P D over the op's time), and the largest element-wise difference of the two routes."""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mgproto_b200 import ops                       # noqa: E402
from mgproto_b200._lib import MGP_OUT_LOGP_NP      # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    B, HW, C, K, D = 256, 196, 200, 10, 128
    N, P = B * HW, C * K
    g = torch.Generator().manual_seed(0)
    xhat = F.normalize(torch.randn(N, D, generator=g), dim=1).to(dev)
    mu = F.normalize(torch.randn(P, D, generator=g), dim=1).to(dev)
    sg = torch.full((P, D), 0.3989422804014327, device=dev)          # the shipped sigma = 1/sqrt(2 pi)
    wt = torch.zeros(C, P)
    pi = torch.softmax(torch.randn(C, K, generator=g), dim=1)
    for c in range(C):
        wt[c, c * K:(c + 1) * K] = pi[c]
    wt = wt.to(dev)
    lpi = torch.log(pi.to(dev).reshape(1, C, K) + 1e-10)

    def fused():
        return ops.log_density(xhat, mu, sg, wt, B, HW, C, K, math="auto")

    def composed():
        lp = ops.logprob(xhat, mu, sg, MGP_OUT_LOGP_NP, eps=1e-10, eps_log=1e-10, math="auto")   # [N,P], 401 MB
        lc = torch.logsumexp(lp.view(N, C, K) + lpi, dim=2)                                      # [N,C]
        return lc.view(B, HW, C).permute(0, 2, 1).contiguous(), torch.logsumexp(lc, dim=1).view(B, HW)

    routes = {"log_density": fused, "composed": composed}
    for f in routes.values():                                           # warm-up (modules, operand caches)
        for _ in range(3):
            f()
    torch.cuda.synchronize()
    times = {k: [] for k in routes}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(a.blocks):
        for name, f in routes.items():
            e0.record()
            for _ in range(a.iters):
                f()
            e1.record()
            torch.cuda.synchronize()
            times[name].append(e0.elapsed_time(e1) / a.iters * 1e3)     # us per call
    fc, fa = fused()
    cc, ca = composed()
    diff = max(float((fc - cc).abs().max()), float((fa - ca).abs().max()))
    flops = 3 * 2.0 * N * P * D
    res = {"card": card(), "shape": dict(B=B, HW=HW, C=C, K=K, D=D)}
    for name, ts in times.items():
        med = sorted(ts)[len(ts) // 2]
        res[name] = {"median_us": round(med, 1), "blocks_us": [round(t, 1) for t in ts],
                     "tflops_fp16x3": round(flops / (med * 1e-6) / 1e12, 1)}
    res["speedup"] = round(res["composed"]["median_us"] / res["log_density"]["median_us"], 2)
    res["max_abs_diff"] = diff
    print(json.dumps(res))


if __name__ == "__main__":
    main()
