#!/usr/bin/env python
"""Generate tests/golden/proxy_anchor.npz: loss and autograd gradients of the UNMODIFIED reference's Proxy_Anchor
(utils/losses.py:29-61) on the CPU in fp32, for the seeded cases of tests/proxy_anchor_oracle.py.  The fixture holds
the seeds and the reference's outputs only; the tests rebuild the inputs from the seeds.

Run from the repo root in the dev container:  python tests/golden/make_golden_proxy_anchor.py
It touches no reference file.  Two shims: ``Tensor.cuda`` is a no-op (utils/losses.py:15, :33 hard-code ``.cuda()``),
and ``pytorch_metric_learning`` -- imported at :6 for the other criteria, which are not used here -- is an empty
stub module with ``losses`` and ``miners``.
"""
import os
import sys
import types

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = os.environ.get("MGPROTO_REFERENCE", "/root/reference")
sys.path.insert(0, REF)
sys.path.insert(0, os.path.dirname(HERE))
torch.Tensor.cuda = lambda self, *a, **k: self
pml = types.ModuleType("pytorch_metric_learning")
pml.losses, pml.miners = types.ModuleType("pytorch_metric_learning.losses"), types.ModuleType("pytorch_metric_learning.miners")
sys.modules.update({"pytorch_metric_learning": pml, "pytorch_metric_learning.losses": pml.losses,
                    "pytorch_metric_learning.miners": pml.miners})
from utils import losses as ref_losses                  # noqa: E402  (the reference's utils/losses.py)
import proxy_anchor_oracle as PA                        # noqa: E402

if __name__ == "__main__":
    torch.set_num_threads(4)
    rec = {"cases": np.array(sorted(PA.GOLDEN_CASES)), "mrg": np.float32(0.1), "beta": np.float32(32)}
    for name in sorted(PA.GOLDEN_CASES):
        B, C, E, seed, _ = PA.GOLDEN_CASES[name]
        X, P, t = PA.case(name)
        crit = ref_losses.Proxy_Anchor(nb_classes=C, sz_embed=E, mrg=0.1, beta=32)
        with torch.no_grad():
            crit.proxies.copy_(torch.from_numpy(P))
        x = torch.from_numpy(X).requires_grad_(True)
        loss = crit(x, torch.from_numpy(t))
        loss.backward()
        rec[name + "_dims"] = np.array([B, C, E, seed])
        rec[name + "_loss"] = loss.detach().numpy().copy()
        rec[name + "_grad_x"] = x.grad.numpy().copy()
        rec[name + "_grad_p"] = crit.proxies.grad.numpy().copy()
        print(name, float(loss.detach()))
    np.savez_compressed(os.path.join(HERE, "proxy_anchor.npz"), **rec)
    print("proxy_anchor.npz written")
