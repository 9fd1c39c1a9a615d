#!/usr/bin/env python
"""Where the tensor-core EM kernel (csrc/em_tc.cu) spends a class's timeline: clock64 stamps of its pipeline phases for
one class, printed per row tile (64 rows at D = 128, 128 at D = 256) in microseconds at the SM clock read from
nvidia-smi."""
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
net = bench.build_model(dev)
buf = torch.zeros(64 * 8, dtype=torch.int64, device=dev)
# classes [:N_ACT] are active; the kernel stamps the CTA that runs class `cls` (the first and the last active class)
N_ACT = int(os.environ.get("N_ACT", "120"))
for cls in (0, N_ACT - 1):
    for _ in range(3):
        net.queue.updated.fill_(1)
        net.queue.updated[N_ACT:] = 0
        net.update_GMM()
    buf.zero_()
    lib.mgp_debug_set_ptr(b"em_tc_prof", buf.data_ptr(), cls)
    net.queue.updated.fill_(1)
    net.queue.updated[N_ACT:] = 0
    net.update_GMM()
    torch.cuda.synchronize()
    lib.mgp_debug_set_ptr(b"em_tc_prof", None, 0)
    mhz = float(subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm", "--format=csv,noheader,nounits", "-i", "0"],
                               stdout=subprocess.PIPE, text=True).stdout.split()[0])
    t = buf.cpu().view(64, 8).double() / mhz          # microseconds
    t0 = t[0, 0]
    print("class %d (SM clock %.0f MHz): tile: TMA-wait E-issue E-done epilogue S-issue | tile total; * = loop tail" % (cls, mhz))
    for i in range(63):
        if t[i, 0] == 0:
            break
        r = t[i]
        nxt = t[i + 1, 0] if i + 1 < 64 and t[i + 1, 0] > 0 else r[5]
        tail = "  * tail %.2f us (gather S0/S1 + update)" % (r[7] - r[6]) if r[6] > 0 else ""
        print("%2d @%7.2f: %5.2f %5.2f %5.2f %5.2f %5.2f | %5.2f%s" % (i, r[0] - t0, r[1] - r[0], r[2] - r[1], r[3] - r[2],
                                                                     r[4] - r[3], r[5] - r[4], nxt - r[0], tail))
    if "--raw" in sys.argv:
        print("raw stamps relative to tile 0 (us): iter-start X-landed E-issued E-seen R-written S-issued tail-in tail-out")
        for i in range(63):
            if t[i, 0] == 0:
                break
            print("%2d: " % i + " ".join("%7.2f" % (v - t0) if v > 0 else "      -" for v in t[i]))
    m = t[63]
    print("   entry->state loaded %.2f | set-up %.2f | lead replay %.2f | EM loops %.2f | trail replay %.2f | write-back+dealloc %.2f | total %.2f us"
          % (m[1] - m[0], m[2] - m[1], m[3] - m[2], m[4] - m[3], m[5] - m[4], m[6] - m[5], m[6] - m[0]))
net.sync_optimizer_state()
st = net.prototype_optimizer.state[net.prototype_means]
a = st["exp_avg_sq"].float().sqrt().flatten()
q = torch.quantile(a[:1_000_000], torch.tensor([0.0, 0.001, 0.01, 0.5], device=a.device))
print("Adam step %d; sqrt(exp_avg_sq): min %.3e  0.1%% %.3e  1%% %.3e  median %.3e  (the replay's series form needs > ~1e-5)"
      % (int(st["step"]), q[0], q[1], q[2], q[3]))
