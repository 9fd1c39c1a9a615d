#!/usr/bin/env python
"""Step time with update_GMM's EM overlapped with the loss and backward (MGProto.overlap_em) and without, at the bench
workload, from CUDA-graph replays (mgproto_b200.pipeline.GraphedStep), plus the kernel timeline of one replay.

  python tools/em_overlap_time.py [--steps N] [--rounds R] [--json OUT]

Two models with the same state, one per setting, each captured as a GraphedStep.  The R rounds alternate the two
settings (N timed replays each, bracketed by CUDA events, rotating bench's feature batches), so that clock drift hits
both alike; the medians over the rounds are reported with the card's name and power limit.  Then one replay of each
setting runs under torch.profiler and every kernel's start and end (us from the replay's first kernel) is printed: with
the overlap, em_tc_kernel must start before head_bwd_kernel and the two must run at the same time."""
import argparse
import json
import os
import statistics
import sys
import tempfile

import torch
from torch.profiler import ProfilerActivity, profile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from step_kernels import card  # noqa: E402


def timeline(gs, x, gt):
    """Kernels of one replay: [(name, start_us, end_us)] from the replay's first kernel, in start order."""
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        gs(x, gt)
        torch.cuda.synchronize()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "trace.json")
        prof.export_chrome_trace(path)
        ev = json.load(open(path))["traceEvents"]
    ks = sorted((e["ts"], e["ts"] + e.get("dur", 0), e["name"]) for e in ev
                if e.get("ph") == "X" and e.get("cat") == "kernel")
    t0 = ks[0][0] if ks else 0.0
    return [(n, s - t0, e - t0) for s, e, n in ks]


def first(tl, name):
    return next(((s, e) for n, s, e in tl if name in n), None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50, help="timed replays per round and setting")
    ap.add_argument("--rounds", type=int, default=7)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    torch.cuda.set_device(0)
    from mgproto_b200.pipeline import GraphedStep
    c = bench.CFG
    g = torch.Generator().manual_seed(1)
    feats = [torch.randn(c["B"], c["D"], c["H"], c["W"], generator=g).to(dev) for _ in range(bench.N_ROT)]
    gts = [torch.randint(0, c["C"], (c["B"],), generator=g).to(dev) for _ in range(bench.N_ROT)]
    steps = {}
    for ov in (True, False):
        torch.manual_seed(0)
        net = bench.build_model(dev)
        net.overlap_em = ov
        steps[ov] = GraphedStep(net, bench.loss_fn, feats[0], gts[0], warmup=3)
    for ov in (True, False):
        for i in range(5):
            steps[ov](feats[i % bench.N_ROT], gts[i % bench.N_ROT])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    per = {True: [], False: []}
    for r in range(a.rounds):
        for ov in ((True, False) if r % 2 == 0 else (False, True)):
            torch.cuda.synchronize()
            e0.record()
            for i in range(a.steps):
                steps[ov](feats[i % bench.N_ROT], gts[i % bench.N_ROT])
            e1.record()
            torch.cuda.synchronize()
            per[ov].append(e0.elapsed_time(e1) * 1e3 / a.steps)
    med = {ov: statistics.median(v) for ov, v in per.items()}
    print("card: %s" % card())
    print("GraphedStep replay, bench shapes (B=%d, C=%d, K=%d, D=%d, cap=%d), %d rounds x %d replays, alternating"
          % (c["B"], c["C"], c["K"], c["D"], c["cap"], a.rounds, a.steps))
    for ov in (False, True):
        print("  overlap_em=%-5s median %.1f us/step  (rounds: %s)" % (ov, med[ov], " ".join("%.1f" % t for t in per[ov])))
    print("  speed-up %.3fx, %.0f -> %.0f images/s" % (med[False] / med[True], c["B"] / med[False] * 1e6,
                                                     c["B"] / med[True] * 1e6))
    tls = {}
    for ov in (True, False):
        tl = tls[ov] = timeline(steps[ov], feats[0], gts[0])
        print("\nkernels of one replay, overlap_em=%s (start / end in us from the first kernel):" % ov)
        for n, s, e in tl:
            print("  %8.1f %8.1f %7.1f  %s" % (s, e, e - s, n[:100]))
    em, bwd = first(tls[True], "em_tc_kernel"), first(tls[True], "head_bwd_kernel")
    if em and bwd:
        print("\noverlap_em=True: em_tc_kernel %.1f-%.1f us, head_bwd_kernel %.1f-%.1f us: EM %s, overlapping %.1f us"
              % (em[0], em[1], bwd[0], bwd[1], "first" if em[0] <= bwd[0] else "SECOND",
                 max(0.0, min(em[1], bwd[1]) - max(em[0], bwd[0]))))
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump({"card": card(), "rounds_us": {str(k): v for k, v in per.items()},
                       "median_us": {str(k): v for k, v in med.items()},
                       "timeline": {str(k): v for k, v in tls.items()}}, f, indent=1)
    for s in steps.values():
        s.close()


if __name__ == "__main__":
    main()
