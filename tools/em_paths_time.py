#!/usr/bin/env python
"""Time update_GMM (cfg2 / cfg3 mixture shapes) through each implementation: tensor-core kernel, fp32 cluster kernel,
multi-launch path, at 1 .. 200 active classes.  The active classes are a seeded random set (the seed is their count,
as in tests/test_gpu_em_waves.py), as in training, where any class can be flagged.  CUDA events, 20 calls after 3
warm-ups; prints the card and its power limit.

    python tools/em_paths_time.py [--paths tc,fused,multilaunch] [--dims 128,256]"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                   # noqa: E402
from mgproto_b200 import _lib                  # noqa: E402

PATHS = {"tc": (1, 1), "fused": (0, 1), "multilaunch": (0, 0)}    # (em_tc, em_fused) switches of mgp_set_option
COUNTS = (1, 8, 40, 80, 100, 132, 133, 146, 200)

ap = argparse.ArgumentParser()
ap.add_argument("--paths", default="tc,fused,multilaunch")
ap.add_argument("--dims", default="128,256")
args = ap.parse_args()
dev = torch.device("cuda:0")
torch.cuda.set_device(0)
lib = _lib.load()
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      stdout=subprocess.PIPE, text=True).stdout.strip()
print("card: %s, %d SMs" % (card, torch.cuda.get_device_properties(0).multi_processor_count))
for D in (int(d) for d in args.dims.split(",")):
    bench.CFG["D"] = D
    net = bench.build_model(dev)
    C = net.queue.updated.numel()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name in args.paths.split(","):
        tc, fused = PATHS[name]
        lib.mgp_set_option(b"em_tc", tc)
        lib.mgp_set_option(b"em_fused", fused)
        for n_act in COUNTS:
            flags = torch.zeros(C, dtype=torch.uint8)
            flags[np.random.default_rng(n_act).permutation(C)[:n_act]] = 1
            flags = flags.to(dev)

            def run():
                net.queue.updated.copy_(flags)
                net.update_GMM()
            for _ in range(3):
                run()
            torch.cuda.synchronize()
            torch.cuda._sleep(20_000_000)          # ~10 ms of GPU spin: the host enqueues the 20 calls behind it, so the events see GPU time only
            e0.record()
            for _ in range(20):
                run()
            e1.record()
            torch.cuda.synchronize()
            print("D=%d %-12s active=%3d  %.1f us per update_GMM (incl. 1 tiny copy)" % (D, name, n_act, e0.elapsed_time(e1) / 20 * 1e3))
    lib.mgp_set_option(b"em_tc", 1)
    lib.mgp_set_option(b"em_fused", 1)
    net.sync_optimizer_state()
