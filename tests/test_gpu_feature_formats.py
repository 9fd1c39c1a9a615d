"""Add-on features in bf16 / fp16 and channels_last (-m gpu): what torch.autocast hands the head.

Every feature format must give bit-identical results to the fp32 NCHW path fed x.float().contiguous(): logits, the
mined values and indices, xhat, the bank after an enqueue, head_level0, push_search and push_forward_features; the
feature gradient comes back in x's dtype and memory format and equals the fp32 gradient rounded to that dtype.
The shapes cover every route after the normalise pass: the staged image-tile max / arg-max kernel (HW = 196, 49),
the 128-patch-tile kernel and the materialised [B,P,HW] map (HW = 300) and the D = 256 tensor-core kernel."""
import copy

import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

FORMATS = [(torch.bfloat16, False), (torch.bfloat16, True), (torch.float16, False), (torch.float16, True),
           (torch.float32, True)]
FORMAT_IDS = ["bf16", "bf16-cl", "fp16", "fp16-cl", "fp32-cl"]
# (B, H, W, D, C, K, T): P = C * K = 2000
SHAPES = [(37, 14, 14, 128, 200, 10, 20), (37, 7, 7, 64, 200, 10, 20), (37, 15, 20, 128, 200, 10, 20),
          (37, 14, 14, 256, 200, 10, 20)]
SHAPE_IDS = ["hw196-d128", "hw49-d64", "hw300-d128", "hw196-d256"]


def _dev():
    return torch.device("cuda:0")


def _net(C, K, D, H, T, seed):
    import mgproto_b200 as M
    torch.manual_seed(seed)
    net = M.MGProto(features=nn.Sequential(nn.Conv2d(3, 8, 1)), img_size=H, prototype_shape=(C * K, D, 1, 1),
                    proto_layer_rf_info=None, num_classes=C, add_on_layers_type="regular", sz_embedding=8,
                    mem_capacity=8, mine_K=T).to(_dev())
    net.prototype_optimizer = torch.optim.Adam([{"params": net.prototype_means, "lr": 3e-3}])
    net.train()
    return net


def _features(B, D, H, W, dtype, cl, seed):
    """x built in its own dtype (and memory format) first; the reference input is x.float().contiguous()."""
    g = torch.Generator(device=_dev()).manual_seed(seed)
    x = torch.randn(B, D, H, W, generator=g, device=_dev(), dtype=dtype)
    if cl:
        x = x.to(memory_format=torch.channels_last)
        assert not x.is_contiguous()
    return x


def _saved(out):
    """(logits, vals, idx, xhat, inv) that HeadFunction saved for the backward."""
    logits, vals, idx, _, _, xhat, inv, _, _ = out.grad_fn.saved_tensors
    return logits, vals, idx, xhat, inv


def _written(t, gt, K):
    """The entries of vals / idx [B,P,T] the labelled head writes: level 0 of every prototype, all levels of the
    image's own class."""
    B, P, T = t.shape
    parts = [t[:, :, 0]]
    if gt is not None:
        for b in range(B):
            c = int(gt[b])
            parts.append(t[b, c * K:(c + 1) * K].reshape(1, -1))
    return [p.contiguous() for p in parts]


def _check_format(t, dtype, cl):
    assert t.dtype == dtype
    if cl:
        assert t.is_contiguous(memory_format=torch.channels_last) and not t.is_contiguous()
    else:
        assert t.is_contiguous()


@pytest.mark.parametrize("B,H,W,D,C,K,T", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("dtype,cl", FORMATS, ids=FORMAT_IDS)
def test_head_forward_and_gradient_bitwise(dtype, cl, B, H, W, D, C, K, T):
    from mgproto_b200 import ops
    net = _net(C, K, D, H, T, seed=D + H)
    mu, sg, wt = net.prototype_means, net.prototype_covs, net.last_layer.weight
    x = _features(B, D, H, W, dtype, cl, seed=1000 * H + D)
    x32 = x.float().contiguous()
    gen = torch.Generator().manual_seed(7)
    gt = torch.randint(0, C, (B,), generator=gen).to(_dev())
    for labels in (gt, None):
        def run(inp):
            xa = inp.detach().clone().requires_grad_(True)
            out, xhat, idx = ops.head_forward(xa, mu, sg, wt, labels, T, "auto")
            gl = torch.randn(out.shape, generator=torch.Generator().manual_seed(11)).to(_dev())
            (gx,) = torch.autograd.grad(out, xa, gl, retain_graph=True)
            return out, gx

        ref, gref = run(x32)
        ref2, gref2 = run(x32)
        assert torch.equal(ref, ref2) and torch.equal(gref, gref2)      # the reference is deterministic
        out, gx = run(x)
        assert out.dtype == torch.float32
        assert torch.equal(out, ref)
        r, n = _saved(ref), _saved(out)
        assert torch.equal(n[3], r[3]) and torch.equal(n[4], r[4])        # xhat, inv_norm
        assert n[3].dtype == torch.float32 and n[3].shape == (B * H * W, D)
        for a, b in zip(_written(n[1], labels, K) + _written(n[2], labels, K),
                        _written(r[1], labels, K) + _written(r[2], labels, K)):
            assert torch.equal(a, b)                                      # vals, idx
        _check_format(gx, dtype, cl)
        assert torch.equal(gx, gref.to(dtype))
        assert torch.isfinite(gx.float()).all() and bool((gx != 0).any())


@pytest.mark.parametrize("B,H,W,D,C,K,T", SHAPES, ids=SHAPE_IDS)
@pytest.mark.parametrize("dtype,cl", FORMATS, ids=FORMAT_IDS)
def test_bank_and_entry_points_bitwise(dtype, cl, B, H, W, D, C, K, T):
    net_a = _net(C, K, D, H, T, seed=3 * D + H)
    net_b = copy.deepcopy(net_a)
    x = _features(B, D, H, W, dtype, cl, seed=77 * H + D)
    x32 = x.float().contiguous()
    gt = torch.randint(0, C, (B,), generator=torch.Generator().manual_seed(5)).to(_dev())
    gt[1] = gt[0]                                                        # two images of one class share a FIFO
    for n in (net_a, net_b):
        n.queue.ensure_shadow()
    out_a = net_a.head(x32, gt)
    out_b = net_b.head(x, gt)
    assert torch.equal(out_a, out_b)
    qa, qb = net_a.queue, net_b.queue
    assert int(qa.mem_len.sum()) > 0
    assert torch.equal(qa.mem_len, qb.mem_len) and torch.equal(qa.head, qb.head)
    assert torch.equal(qa.bank, qb.bank)
    sa, sb = qa.shadow_if_valid(), qb.shadow_if_valid()
    assert sa is not None and sb is not None
    for a, b in zip(sa, sb):
        assert torch.equal(a, b)

    with torch.no_grad():
        assert torch.equal(net_b.head_level0(x), net_a.head_level0(x32))
        arg_a, val_a, xh_a = net_a.push_search(x32, gt)
        arg_b, val_b, xh_b = net_b.push_search(x, gt)
        assert torch.equal(arg_a, arg_b) and torch.equal(val_a, val_b) and torch.equal(xh_a, xh_b)
        f_a, d_a = net_a.push_forward_features(x32)
        f_b, d_b = net_b.push_forward_features(x)
        assert f_b.dtype == torch.float32 and f_b.is_contiguous()
        assert torch.equal(f_a, f_b) and torch.equal(d_a, d_b)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16], ids=["bf16", "fp16"])
@pytest.mark.parametrize("cl", [False, True], ids=["nchw", "channels_last"])
def test_autocast_training_body(dtype, cl):
    """construct_MGProto('resnet18') trained under torch.autocast as a user would: the reference's training body
    (train_and_test.py:26-63: forward with labels, level-0 + mining CE, backward, joint optimiser step, update_GMM once
    the banks fill); fp16 with a GradScaler.  The head must receive 16-bit features and the gradient must reach the
    backbone."""
    import mgproto_b200 as M
    torch.manual_seed(0)
    C, K, D, T, cap, B = 6, 4, 64, 4, 8, 12
    net = M.construct_MGProto("resnet18", pretrained=False, img_size=64, prototype_shape=(C * K, D, 1, 1), num_classes=C,
                              add_on_layers_type="regular", sz_embedding=16, mem_capacity=cap, mine_K=T).to(_dev())
    if cl:
        net = net.to(memory_format=torch.channels_last)
    net.prototype_optimizer = torch.optim.Adam([{"params": net.prototype_means, "lr": 3e-3}])
    joint = torch.optim.Adam([{"params": net.features.parameters(), "lr": 1e-4},
                              {"params": net.add_on_layers.parameters(), "lr": 3e-3}])
    scaler = torch.amp.GradScaler("cuda", init_scale=256.0) if dtype == torch.float16 else None
    seen = []
    hook = net.add_on_layers.register_forward_hook(lambda m, i, o: seen.append((o.dtype, o.is_contiguous(),
                                                                                o.is_contiguous(memory_format=torch.channels_last))))
    first_conv = next(m for m in net.features.modules() if isinstance(m, nn.Conv2d))
    net.train()
    g = torch.Generator().manual_seed(1)
    updates = 0
    for it in range(4):
        image = torch.randn(B, 3, 64, 64, generator=g).to(_dev())
        if cl:
            image = image.to(memory_format=torch.channels_last)
        target = torch.randint(0, C, (B,), generator=g).to(_dev())
        with torch.autocast("cuda", dtype=dtype):
            output, _ = net(image, target)
            mine_loss = sum(F.cross_entropy(output[:, :, k], target) for k in range(1, T)) / (T - 1)
            loss = F.cross_entropy(output[:, :, 0], target) + 0.2 * mine_loss
        assert seen[-1][0] == dtype
        if cl:
            assert seen[-1][2] and not seen[-1][1]
        assert output.dtype == torch.float32 and torch.isfinite(output).all() and torch.isfinite(loss)
        joint.zero_grad()
        if scaler is not None:
            scaler.scale(loss).backward()
            scaler.unscale_(joint)
        else:
            loss.backward()
        gw = first_conv.weight.grad
        assert gw is not None and torch.isfinite(gw).all() and float(gw.abs().sum()) > 0
        if scaler is not None:
            scaler.step(joint)
            scaler.update()
        else:
            joint.step()
        if net.queue.mem_len.sum() > 0 and net.iteration_counter % net.update_interval == 0:
            net.update_GMM()
            updates += int((net.queue.mem_len == cap).any())
    hook.remove()
    assert updates > 0
    net.sync_optimizer_state()
    assert torch.isfinite(net.prototype_means).all() and torch.isfinite(net.last_layer.weight).all()


def test_graphed_step_bf16_channels_last_replays_eager_bitwise():
    """GraphedStep built from bf16 channels_last features: its static input and x_grad keep that dtype and format,
    and its replays equal the eager steps of a twin model bit for bit."""
    from mgproto_b200 import ops
    from mgproto_b200.pipeline import GraphedStep
    C, K, D, T, H, B = 6, 4, 128, 4, 6, 16
    net_a = _net(C, K, D, H, T, seed=3)
    net_b = copy.deepcopy(net_a)
    net_b.prototype_optimizer = torch.optim.Adam([{"params": net_b.prototype_means, "lr": 3e-3}])
    xs = [_features(B, D, H, H, torch.bfloat16, True, seed=40 + i) for i in range(4)]
    gts = [torch.randint(0, C, (B,), generator=torch.Generator().manual_seed(4 + i)).to(_dev()) for i in range(4)]

    def loss_fn(out, gt):
        return ops.mine_cross_entropy(out, gt, 0.2)

    seq = [0, 0, 0, 1, 2, 3, 1]                      # warm-up (2) + 5 replays
    for i in seq:
        x = xs[i].clone().requires_grad_(True)
        out_a = net_a.head(x, gts[i])
        loss_a = loss_fn(out_a, gts[i])
        loss_a.backward()
        net_a.update_GMM()
        grad_a = x.grad
    _check_format(grad_a, torch.bfloat16, True)
    step = GraphedStep(net_b, loss_fn, xs[0], gts[0], warmup=2)
    _check_format(step.x, torch.bfloat16, True)
    for i in seq[2:]:
        out_b, loss_b = step(xs[i], gts[i])
    torch.cuda.synchronize()
    _check_format(step.x_grad, torch.bfloat16, True)
    assert torch.equal(out_b, out_a) and torch.equal(loss_b, loss_a) and torch.equal(step.x_grad, grad_a)
    assert torch.equal(net_b.prototype_means, net_a.prototype_means)
    assert torch.equal(net_b.last_layer.weight, net_a.last_layer.weight)
    assert torch.equal(net_b.queue.bank, net_a.queue.bank) and torch.equal(net_b.queue.mem_len, net_a.queue.mem_len)
