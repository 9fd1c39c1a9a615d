#!/usr/bin/env python
"""Generate tests/golden/log_density.npz: the per-patch class log-densities of two small feature maps, recorded from
the UNMODIFIED reference's own _score (model.py:403-421, as_average=False) run class by class on the features
normalised as its head does (model.py:210-211), and the log-sum-exp of those scores over the classes (the per-patch
log sum_c p(x|c) of train_and_test.py:199).

Run from the repo root in the dev container:  python tests/golden/make_golden_log_density.py
Only this script (and make_golden.py, whose model builder and shims it reuses) imports the reference.
"""
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import make_golden as MG                                # noqa: E402  (imports the reference's model.py, CPU shims)

OUT = os.path.dirname(os.path.abspath(__file__))


def make_case(rec, name, C, K, D, B, H, W, sigma_mode, seed):
    g = torch.Generator().manual_seed(seed)
    m = MG.build(C, K, D, cap=4, T=2, seed=seed)
    if sigma_mode == 'rand':                            # anisotropic sigma
        m.prototype_covs.data.copy_(0.2 + 0.6 * torch.rand(C, K, D, generator=g))
    pi = torch.softmax(torch.randn(C, K, generator=g), dim=1)
    pi[0, K - 1] = 0.0                                  # a pruned prototype (prune_prototypes_topM zeroes weights)
    wt = torch.zeros(C, C * K)
    for c in range(C):
        wt[c, c * K:(c + 1) * K] = pi[c]
    x = torch.randn(B, D, H, W, generator=g)
    with torch.no_grad():
        feat = F.normalize(x, p=2, dim=1).permute(0, 2, 3, 1).reshape(-1, D)      # model.py:210-211
        cols = []
        for c in range(C):
            mu = m.prototype_means[c].detach().unsqueeze(0)                         # [1,K,D]
            sg = m.prototype_covs[c].detach().unsqueeze(0)
            p = wt[c, c * K:(c + 1) * K].view(1, K, 1)
            cols.append(m._score(feat.unsqueeze(1), mu, sg, p, as_average=False))   # [N]
        lp = torch.stack(cols, 1)                                                   # [N,C]
        logp_c = lp.reshape(B, H, W, C).permute(0, 3, 1, 2).contiguous()
        logp_all = torch.logsumexp(logp_c, dim=1)
    pre = name + '_'
    rec[pre + 'x_add'] = x.numpy().copy()
    rec[pre + 'mu'] = m.prototype_means.detach().numpy().copy()
    rec[pre + 'sigma'] = m.prototype_covs.detach().numpy().copy()
    rec[pre + 'weight'] = wt.numpy().copy()
    rec[pre + 'logp_c'] = logp_c.numpy().copy()
    rec[pre + 'logp_all'] = logp_all.numpy().copy()


if __name__ == '__main__':
    torch.set_num_threads(4)
    rec = {}
    make_case(rec, 'init', C=5, K=3, D=16, B=2, H=3, W=4, sigma_mode='init', seed=21)
    make_case(rec, 'aniso', C=4, K=5, D=8, B=2, H=2, W=5, sigma_mode='rand', seed=22)
    rec['cases'] = np.array(['init', 'aniso'])
    np.savez_compressed(os.path.join(OUT, 'log_density.npz'), **rec)
    print('log_density.npz written')
