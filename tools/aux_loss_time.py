#!/usr/bin/env python
"""Time the Proxy-Anchor auxiliary loss, forward + backward to the embeddings and the proxies: ops.proxy_anchor (one
cluster kernel, csrc/aux_loss.cu) against a torch restatement of the same formula written here WITHOUT the reference's
host round trips (one-hot by comparison on the device, the number of positive proxies kept on the device), i.e. the
best ATen can do, at the reference's embedding width and class count for batches of 256 and 80.

    python tools/aux_loss_time.py [--blocks 9] [--iters 200]

CUDA events around blocks of `iters` calls after a warm-up, the routes alternated block by block, the median block
reported: once issued eagerly (host launch cost included, as a training loop pays it) and once replayed from a CUDA
graph (device time alone).  Also ops.launch_count() and torch.profiler's kernel count per call for each route, the
card name, power limit and clocks as read in the same run (no setting is changed), and the largest difference of the
two routes' results."""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mgproto_b200 import ops                       # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def torch_proxy_anchor(X, P, T, mrg=0.1, beta=32.0):
    """The criterion's formula in ATen, nothing read back by the host."""
    xh = X / torch.sqrt((X * X).sum(1, keepdim=True) + 1e-12)
    ph = P / torch.sqrt((P * P).sum(1, keepdim=True) + 1e-12)
    cos = xh @ ph.t()
    pos = T.view(-1, 1) == torch.arange(P.shape[0], device=X.device).view(1, -1)
    zero = torch.zeros((), device=X.device)
    sp = torch.where(pos, torch.exp(-beta * (cos - mrg)), zero).sum(0)
    sn = torch.where(pos, zero, torch.exp(beta * (cos + mrg))).sum(0)
    nv = pos.any(0).sum().clamp(min=1)
    return torch.log1p(sp).sum() / nv + torch.log1p(sn).sum() / P.shape[0]


def kernels_per_call(f):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        f()
        torch.cuda.synchronize()
    return int(sum(e.count for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=9)
    ap.add_argument("--iters", type=int, default=200)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    res = {"card_power_limit_max_sm_clock_sm_clock": card(), "iters_per_block": a.iters, "blocks": a.blocks}
    for B in (256, 80):
        C, E = 200, 32
        g = torch.Generator().manual_seed(B)
        X = torch.randn(B, E, generator=g).to(dev).requires_grad_(True)
        P = (torch.randn(C, E, generator=g) * (2.0 / C) ** 0.5).to(dev).requires_grad_(True)
        T = torch.randint(0, C, (B,), generator=g).to(dev)

        def ours():
            return torch.autograd.grad(ops.proxy_anchor(X, P, T), [X, P])

        def aten():
            return torch.autograd.grad(torch_proxy_anchor(X, P, T), [X, P])

        routes = {"proxy_anchor_kernel": ours, "torch_restatement": aten}
        graphs = {}
        side = torch.cuda.Stream()
        for name, f in routes.items():
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(5):                                       # warm-up (modules, allocator)
                    f()
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize()
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                f()
            graphs[name] = gr
            for _ in range(5):
                gr.replay()
        torch.cuda.synchronize()
        times = {(k, m): [] for k in routes for m in ("eager", "graph")}
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(a.blocks):
            for name, f in routes.items():
                for mode, call in (("eager", f), ("graph", graphs[name].replay)):
                    e0.record()
                    for _ in range(a.iters):
                        call()
                    e1.record()
                    torch.cuda.synchronize()
                    times[(name, mode)].append(e0.elapsed_time(e1) / a.iters * 1e3)     # us per call
        out = {}
        for name, f in routes.items():
            n0 = ops.launch_count()
            f()
            out[name] = {"library_launches": ops.launch_count() - n0, "profiler_kernels": kernels_per_call(f)}
            for mode in ("eager", "graph"):
                ts = sorted(times[(name, mode)])
                out[name][mode + "_median_us"] = round(ts[len(ts) // 2], 2)
                out[name][mode + "_min_max_us"] = [round(ts[0], 2), round(ts[-1], 2)]
        (gx, gp), (hx, hp) = ours(), aten()
        out["max_rel_diff_grad_x_grad_p"] = [float((gx - hx).abs().max() / hx.abs().max()),
                                             float((gp - hp).abs().max() / hp.abs().max())]
        for mode in ("eager", "graph"):
            out["speedup_" + mode] = round(out["torch_restatement"][mode + "_median_us"] /
                                           out["proxy_anchor_kernel"][mode + "_median_us"], 2)
        res["B%d_C%d_E%d" % (B, C, E)] = out
    print(json.dumps(res, indent=1))


if __name__ == "__main__":
    main()
