#!/usr/bin/env python
"""Time update_GMM (cfg2 / cfg3 mixture shapes) through each implementation: tensor-core kernel, fp32 cluster kernel,
multi-launch path, at 80 .. 200 active classes.  At D = 128 the tensor-core kernel takes its pipelined variant while
the active classes fit one CTA per SM (132 on an H100 SXM) and its one-warpgroup variant (two CTAs per SM) beyond;
tc_serial always takes the latter.  CUDA events, 20 calls after 3 warm-ups; prints the card and its power limit."""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                   # noqa: E402
from mgproto_b200 import _lib                  # noqa: E402

dev = torch.device("cuda:0")
torch.cuda.set_device(0)
lib = _lib.load()
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      stdout=subprocess.PIPE, text=True).stdout.strip()
print("card: %s, %d SMs" % (card, torch.cuda.get_device_properties(0).multi_processor_count))
for D in (128, 256):
    bench.CFG["D"] = D
    net = bench.build_model(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for name, (tc, fused, pipe) in (("tc", (1, 1, 1)), ("tc_serial", (1, 1, 0)), ("fused", (0, 1, 1)), ("multilaunch", (0, 0, 1))):
        if D == 256 and name == "tc_serial":
            continue
        lib.mgp_set_option(b"em_tc", tc)
        lib.mgp_set_option(b"em_fused", fused)
        lib.mgp_set_option(b"em_pipe", pipe)
        for n_act in (80, 132, 133, 146, 200):
            def run():
                net.queue.updated.zero_()
                net.queue.updated[:n_act] = 1
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
            print("D=%d %-12s active=%3d  %.1f us per update_GMM (incl. 2 tiny fills)" % (D, name, n_act, e0.elapsed_time(e1) / 20 * 1e3))
    lib.mgp_set_option(b"em_tc", 1)
    lib.mgp_set_option(b"em_fused", 1)
    net.sync_optimizer_state()
