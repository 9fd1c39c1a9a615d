"""update_GMM through the tensor-core EM kernel (csrc/em_tc.cu) at the headline EM shapes (200 classes x 10
prototypes, D = 128, 800-row banks, Adam pre-seeded at step 1000) with a seeded random set of 1 .. 200 active classes,
against the fp32 cluster kernel.  At D = 128 the kernel runs two one-warpgroup CTAs per SM, one per class, with the
active classes on the lowest block indices (the planner's order): the counts cover a single class, fewer active
classes than SMs, one wave of CTAs on an H100 (132 SMs) and one class past it, and more classes than SMs.

Tolerance: 1e-4 norm-wise (max |err| over max |ref|), as in tests/test_gpu_headline.py."""
import numpy as np
import pytest
import torch
import torch.nn as nn

import headline_case as HC

pytestmark = pytest.mark.gpu
C, K, D, T, CAP = 200, 10, 128, 20, 800
TOL = 1e-4
# (em_tc, em_fused) switches of mgp_set_option
PATHS = {"tc": (1, 1), "fused": (0, 1)}


def _t(a, dtype=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=dtype, device=torch.device("cuda:0"))


def normwise(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


def _update(path, n_active):
    """One update_GMM with n_active classes flagged (a seeded random choice); returns mu before and after, pi, the
    Adam moments and step."""
    import mgproto_b200 as M
    from mgproto_b200 import _lib
    mu, sg, wt = HC.mixture(C, K, D)
    net = M.MGProto(features=nn.Sequential(nn.Conv2d(3, 8, 1)), img_size=224, prototype_shape=(C * K, D, 1, 1),
                    proto_layer_rf_info=None, num_classes=C, add_on_layers_type="regular", sz_embedding=8,
                    mem_capacity=CAP, mine_K=T).to(torch.device("cuda:0"))
    net.prototype_means.data.copy_(_t(mu))
    net.prototype_covs.data.copy_(_t(sg))
    net.last_layer.weight.data.copy_(_t(wt))
    net.prototype_optimizer = torch.optim.Adam([{"params": net.prototype_means, "lr": 3e-3}])
    net.train()
    q = net.queue
    q.bank.copy_(_t(HC.bank_rows(C, K, D, CAP, mu)))
    q.mem_len.fill_(q.cap_cls)
    q.head.zero_()
    am, av, _, _, step0 = HC.em_state(C, K, D)
    net.prototype_optimizer.state[net.prototype_means] = {"step": torch.tensor(float(step0)), "exp_avg": _t(am).clone(),
                                                          "exp_avg_sq": _t(av).clone()}
    flags = np.zeros(C, np.uint8)
    flags[np.random.default_rng(n_active).permutation(C)[:n_active]] = 1
    lib = _lib.load()
    want = PATHS[path]
    prev = (lib.mgp_set_option(b"em_tc", want[0]), lib.mgp_set_option(b"em_fused", want[1]))
    try:
        q.updated |= _t(flags, torch.uint8)
        net.update_GMM()
        net.sync_optimizer_state()
    finally:
        lib.mgp_set_option(b"em_tc", prev[0])
        lib.mgp_set_option(b"em_fused", prev[1])
    assert int(net.memory_updated_cls.sum()) == 0
    w = net.last_layer.weight.detach().cpu().numpy()
    st = net.prototype_optimizer.state[net.prototype_means]
    return {"mu0": mu, "mu": net.prototype_means.detach().cpu().numpy(), "pi": np.stack([w[i, i * K:(i + 1) * K] for i in range(C)]),
            "exp_avg": st["exp_avg"].cpu().numpy(), "exp_avg_sq": st["exp_avg_sq"].cpu().numpy(), "step": int(st["step"])}


@pytest.mark.parametrize("n_active", [1, 8, 40, 100, 132, 133, 150, 200])
def test_em_tc_vs_fused(n_active):
    ref = _update("fused", n_active)
    got = _update("tc", n_active)
    assert got["step"] == ref["step"]
    for k in ("mu", "pi", "exp_avg", "exp_avg_sq"):
        err = normwise(got[k], ref[k])
        print("%d active: %s norm-wise %.2e" % (n_active, k, err))
        assert err < TOL, (k, err)
    mv = normwise(got["mu"].astype(np.float64) - got["mu0"], ref["mu"].astype(np.float64) - ref["mu0"])
    print("%d active: mu movement norm-wise %.2e" % (n_active, mv))
    assert mv < 1e-3, mv
