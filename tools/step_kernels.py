#!/usr/bin/env python
"""Per-kernel device times of one eager hot-path step at the bench workload (torch.profiler, CUDA activities).

  python tools/step_kernels.py [--steps N] [--json OUT]

Warms up, then profiles N eager steps (head forward + backward + update_GMM) and prints each kernel's calls, device
time per step and share of the step's summed kernel time, largest first, with the card's name and power limit.
Run it on its own: the profiler slows the host, so end-to-end numbers come from bench.py."""
import argparse
import json
import os
import subprocess
import sys

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:                                           # noqa: BLE001
        return torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3, help="profiled steps (times are per step)")
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--json", default=None, help="also write the table as JSON to this path")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(0)
    net = bench.build_model(dev)
    c = bench.CFG
    g = torch.Generator().manual_seed(1)
    x = torch.randn(c["B"], c["D"], c["H"], c["W"], generator=g).to(dev)
    gt = torch.randint(0, c["C"], (c["B"],), generator=g).to(dev)

    def step():
        xr = x.clone().requires_grad_(True)
        out = net.head(xr, gt)
        bench.loss_fn(out, gt).backward()
        net.update_GMM()

    for _ in range(a.warmup):
        step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(a.steps):
            step()
        torch.cuda.synchronize()
    rows = []
    for e in prof.key_averages():
        t = getattr(e, "device_time_total", None)
        if t is None:
            t = getattr(e, "cuda_time_total", 0.0)
        if t > 0:
            rows.append({"kernel": e.key, "calls_per_step": e.count / a.steps, "us_per_step": t / a.steps})
    rows.sort(key=lambda r: -r["us_per_step"])
    total = sum(r["us_per_step"] for r in rows)
    print("card: %s" % card())
    print("summed device time per step: %.1f us over %d profiled steps" % (total, a.steps))
    print("%9s %6s %6s  %s" % ("us/step", "share", "calls", "kernel"))
    for r in rows:
        r["share"] = r["us_per_step"] / total if total else 0.0
        print("%9.1f %5.1f%% %6.1f  %s" % (r["us_per_step"], 100 * r["share"], r["calls_per_step"], r["kernel"][:110]))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump({"card": card(), "steps": a.steps, "us_per_step": total, "kernels": rows}, f, indent=1)


if __name__ == "__main__":
    main()
