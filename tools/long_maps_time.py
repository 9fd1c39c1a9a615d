#!/usr/bin/env python
"""Time the head on long feature maps at about 50 000 patches per call (B * HW ~ 256 x 196), bench mixture
(C = 200, K = 10, D = 128, T = 20, isotropic sigma):

  labelled head forward + backward (HeadFunction: max / arg-max epilogue, top-T, pi mix, feature gradient), and
  head_level0 (the test / OoD head),

for HW = 1024 on the existing kernels, HW = 1024 routed through the long-map entry points (ops.LONG_MAP_HW lowered:
the cost of the long path itself), HW = 1600 and HW = 4096; and the reference's chain on the same GPU and shapes in
torch -- log p, exp, topk over h*w, gather, wrong-class rule, pi mix, log, autograd backward.  The reference's
compute_log_prob broadcasts [N,P,D] (model.py:256-275): under autograd that keeps N*P*D*4 = 51 GB per saved tensor
here, so the torch chain evaluates the same log p as |x|^2 w - 2 x.(w mu) + w |mu|^2 with one matmul.

CUDA events, median over blocks of calls; the card's name and power limit are read in the same run.
    python tools/long_maps_time.py [--blocks 7] [--calls 5]"""
import argparse
import json
import math
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mgproto_b200 import ops                 # noqa: E402

C, K, D, T = 200, 10, 128, 20
P = C * K


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        q = "nvidia-smi unavailable (%s)" % e
    return "%s | %s" % (torch.cuda.get_device_name(0), q)


def median_ms(fn, blocks, calls):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = []
    for _ in range(blocks):
        e0.record()
        for _ in range(calls):
            fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1) / calls)
    return statistics.median(out)


def torch_reference(x, mu, sg, wt, gt):
    """model.py:208-222, :254 in torch (log p through one matmul, see the module docstring)."""
    B, _, H, W = x.shape
    xn = x / x.norm(dim=1, keepdim=True).clamp_min(1e-12)
    f = xn.permute(0, 2, 3, 1).reshape(-1, D)
    m, s = mu.reshape(P, D), sg.reshape(P, D)
    w = 1.0 / (s * s)
    q = (f * f) @ w.t() - 2.0 * f @ (m * w).t() + (m * m * w).sum(1)[None]
    lp = -0.5 * D * math.log(2 * math.pi) - s.log().sum(1)[None] - 0.5 * q                  # [N,P]
    prob = lp.exp().view(B, H * W, P).transpose(1, 2)                                         # [B,P,HW]
    val, ind = torch.topk(prob, T, dim=2)
    feat = torch.gather(xn.reshape(B, D, H * W), 2, ind[:, :, :1].transpose(1, 2).expand(B, D, P))  # enqueue gather
    if gt is not None:
        wrong = (torch.arange(P, device=x.device)[None, :] // K) != gt[:, None]
        val = torch.where(wrong[:, :, None], val[:, :, :1].expand_as(val), val)
    out = torch.log(torch.einsum("bpt,cp->bct", val, wt))
    return out, feat


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=7)
    ap.add_argument("--calls", type=int, default=5)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(0)
    mu = torch.nn.functional.normalize(torch.rand(C, K, D, generator=g), dim=2).to(dev)
    sg = torch.full((C, K, D), 1.0 / math.sqrt(2 * math.pi), device=dev)
    pi = torch.softmax(torch.randn(C, K, generator=g), 1)
    wt = torch.zeros(C, P)
    for c in range(C):
        wt[c, c * K:(c + 1) * K] = pi[c]
    wt = wt.to(dev)
    print("card: %s" % card())
    rows = []
    for name, HW, side, thr in (("1024 existing", 1024, (32, 32), ops.LONG_MAP_HW), ("1024 long", 1024, (32, 32), 1023),
                                ("1600 long", 1600, (40, 40), ops.LONG_MAP_HW), ("4096 long", 4096, (64, 64), ops.LONG_MAP_HW)):
        B = round(256 * 196 / HW)
        x = torch.randn(B, D, *side, generator=g).to(dev)
        gt = torch.randint(0, C, (B,), generator=g).to(dev)
        gl = torch.randn(B, C, T, generator=g).to(dev) / B
        xd = x.clone().requires_grad_(True)
        saved = ops.LONG_MAP_HW
        ops.LONG_MAP_HW = thr
        try:
            def step():
                xd.grad = None
                logits, _, _ = ops.head_forward(xd, mu, sg, wt, gt, T)
                logits.backward(gl)

            def level0():
                ops.head_level0(x, mu, sg, wt)
            t_step = median_ms(step, a.blocks, a.calls)
            t_l0 = median_ms(level0, a.blocks, a.calls)
        finally:
            ops.LONG_MAP_HW = saved

        def ref_step():
            xd.grad = None
            out, _ = torch_reference(xd, mu, sg, wt, gt)
            out.backward(gl)

        def ref_l0():
            with torch.no_grad():
                torch_reference(x, mu, sg, wt, None)
        t_rs = median_ms(ref_step, a.blocks, a.calls)
        t_rl = median_ms(ref_l0, a.blocks, a.calls)
        r = dict(case=name, B=B, HW=HW, patches=B * HW, head_fwd_bwd_ms=round(t_step, 3), head_level0_ms=round(t_l0, 3),
                 torch_fwd_bwd_ms=round(t_rs, 3), torch_level0_ms=round(t_rl, 3))
        rows.append(r)
        print(json.dumps(r))
        del x, xd, gt, gl
        torch.cuda.empty_cache()
    print("%-14s %5s %6s %8s | %12s %12s | %12s %12s" % ("case", "B", "HW", "patches", "head f+b ms", "level0 ms",
                                                           "torch f+b ms", "torch l0 ms"))
    for r in rows:
        print("%-14s %5d %6d %8d | %12.3f %12.3f | %12.3f %12.3f" % (r["case"], r["B"], r["HW"], r["patches"],
                                                                   r["head_fwd_bwd_ms"], r["head_level0_ms"],
                                                                   r["torch_fwd_bwd_ms"], r["torch_level0_ms"]))


if __name__ == "__main__":
    main()
