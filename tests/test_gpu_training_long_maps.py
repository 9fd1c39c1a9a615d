"""Training on long feature maps (-m gpu): the reference's training-loop body on construct_MGProto('resnet18') with
34 x 34 = 1156-patch add-on maps, and GraphedStep at the same size, through the long-map head kernels
(test_gpu_long_maps.py checks the kernels themselves against float64 and under torch.profiler)."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

from test_gpu_headline import TOL, _dev
from test_gpu_long_maps import LONG_TOP1, _no_old, trace_ops

pytestmark = pytest.mark.gpu


def test_reference_training_body_at_1156_patches():
    """construct_MGProto('resnet18', img_size=544) (the backbone's output stride is 16): 34 x 34 = 1156 patches through
    the reference's training-loop body (train_and_test.py:26-63) for two iterations: forward(image, target), CE +
    mining loss, backward into the backbone, update_GMM once the banks fill.  Logits and the enqueue against the float64
    oracle on the add-on features."""
    import mgproto_b200 as M
    from oracle import mgproto_oracle as O
    torch.manual_seed(0)
    C, K, D, T, cap, B, S = 6, 4, 64, 4, 8, 6, 544
    net = M.construct_MGProto("resnet18", pretrained=False, img_size=S, prototype_shape=(C * K, D, 1, 1), num_classes=C,
                              add_on_layers_type="regular", sz_embedding=16, mem_capacity=cap, mine_K=T).to(_dev())
    net.prototype_optimizer = torch.optim.Adam([{"params": net.prototype_means, "lr": 3e-3}])
    joint = torch.optim.Adam([{"params": net.features.parameters(), "lr": 1e-4},
                              {"params": net.add_on_layers.parameters(), "lr": 3e-3}])
    net.train()
    g = torch.Generator().manual_seed(1)
    bank = O.MemoryBankOracle(C, D, cap)
    for it in range(2):
        image = torch.randn(B, 3, S, S, generator=g).to(_dev())
        target = torch.randint(0, C, (B,), generator=g).to(_dev())
        with trace_ops() as tr:
            output, x_aux = net(image, target)
            mine_loss = sum(F.cross_entropy(output[:, :, k], target) for k in range(1, T)) / (T - 1)
            loss = F.cross_entropy(output[:, :, 0], target) + 0.2 * mine_loss
            joint.zero_grad()
            loss.backward()
        assert LONG_TOP1 in tr.kernels and "head_bwd_long" in tr.kernels, sorted(tr.kernels)
        _no_old(tr)
        gn = sum(float(p.grad.abs().sum()) for p in net.features.parameters() if p.grad is not None)
        assert np.isfinite(gn) and gn > 0
        with torch.no_grad():
            x_add, _ = net.conv_features(image)
        assert x_add.shape[2] * x_add.shape[3] == 1156
        fw = O.head_forward(x_add.double().cpu().numpy(), net.prototype_means.detach().double().cpu().numpy(),
                            net.prototype_covs.double().cpu().numpy(), net.last_layer.weight.double().cpu().numpy(),
                            target.cpu().numpy(), T)
        np.testing.assert_allclose(output.detach().cpu().numpy(), fw["logits"], rtol=TOL, atol=1e-5)
        for c, rows in O.enqueue_rows(fw["xhat"].astype(np.float32), fw["idx"], target.cpu().numpy(), C, K, 1156):
            bank.push(c, rows)
        np.testing.assert_array_equal(net.queue.mem_len.cpu().numpy(), bank.mem_len)
        lin = net.queue.linear().cpu().numpy()
        for c in range(C):
            n = int(bank.mem_len[c])
            np.testing.assert_allclose(lin[c, :n], bank.data[c, :n], rtol=1e-5, atol=1e-6)
        joint.step()
        if net.queue.mem_len.sum() > 0 and net.iteration_counter % net.update_interval == 0:
            net.update_GMM()
    net.sync_optimizer_state()
    assert torch.isfinite(net.prototype_means).all() and torch.isfinite(net.last_layer.weight).all()


def test_graphed_step_replays_the_eager_step_at_1156_patches():
    """GraphedStep on 34 x 34 add-on maps (head_top1_long_kernel and head_bwd_long_v4_kernel inside the graph) against
    the same eager steps on a twin model: bit for bit."""
    import mgproto_b200 as M
    from mgproto_b200 import ops
    from mgproto_b200.pipeline import GraphedStep
    torch.manual_seed(3)
    C, K, D, T, cap, B, H = 6, 4, 128, 4, 8, 8, 34
    net_a = M.MGProto(features=nn.Sequential(nn.Conv2d(3, 8, 1)), img_size=H, prototype_shape=(C * K, D, 1, 1),
                      proto_layer_rf_info=None, num_classes=C, add_on_layers_type="regular", sz_embedding=8,
                      mem_capacity=cap, mine_K=T).to(_dev())
    net_b = copy.deepcopy(net_a)
    for n in (net_a, net_b):
        n.prototype_optimizer = torch.optim.Adam([{"params": n.prototype_means, "lr": 3e-3}])
        n.train()
    g = torch.Generator().manual_seed(4)
    xs = [torch.randn(B, D, H, H, generator=g).to(_dev()) for _ in range(4)]
    gts = [torch.randint(0, C, (B,), generator=g).to(_dev()) for _ in range(4)]

    def loss_fn(out, gt):
        return ops.mine_cross_entropy(out, gt, 0.2)

    seq = [0, 0, 0, 1, 2, 3, 1]
    with trace_ops() as tr:
        for i in seq:
            x = xs[i].clone().requires_grad_(True)
            out_a = net_a.head(x, gts[i])
            loss_a = loss_fn(out_a, gts[i])
            loss_a.backward()
            net_a.update_GMM()
            grad_a = x.grad
    assert LONG_TOP1 in tr.kernels and "head_bwd_long" in tr.kernels
    _no_old(tr)
    step = GraphedStep(net_b, loss_fn, xs[0], gts[0], warmup=2)
    for i in seq[2:]:
        out_b, loss_b = step(xs[i], gts[i])
    torch.cuda.synchronize()
    assert torch.equal(out_b, out_a) and torch.equal(loss_b, loss_a) and torch.equal(step.x_grad, grad_a)
    assert torch.equal(net_b.prototype_means, net_a.prototype_means)
    assert torch.equal(net_b.last_layer.weight, net_a.last_layer.weight)
    assert torch.equal(net_b.queue.bank, net_a.queue.bank) and torch.equal(net_b.queue.mem_len, net_a.queue.mem_len)
