"""update_GMM's EM on a side stream beside the loss and the backward (MGProto.overlap_em, the default), against the same
steps with overlap_em = False (the EM in place on the caller's stream), at the bench shapes (200 classes x 10
prototypes, D = 128, full 800-row banks, T = 20) with a smaller batch.

The overlapped EM computes exactly what the in-place one does -- the same kernel, writing staged copies of the means
and the class-diagonal mixture weights that a commit kernel copies over -- so everything is compared bit for bit:
logits, feature gradients, means, mixture weights, both Adam moments, the Adam step, the bank and its cursors."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
C, K, D, T, CAP, B, H, W = 200, 10, 128, 20, 800, 64, 14, 14


def _dev():
    return torch.device("cuda:0")


def _net(overlap):
    import mgproto_b200 as M
    g = torch.Generator().manual_seed(2)
    mu = F.normalize(torch.rand(C, K, D, generator=g), dim=2)
    kk = torch.randint(0, K, (C, CAP), generator=g)
    rows = F.normalize(mu[torch.arange(C)[:, None], kk] + 0.3 * torch.randn(C, CAP, D, generator=g), dim=2)
    torch.manual_seed(0)
    net = M.MGProto(features=nn.Sequential(nn.Conv2d(3, 8, 1)), img_size=224, prototype_shape=(C * K, D, 1, 1),
                    proto_layer_rf_info=None, num_classes=C, add_on_layers_type="regular", sz_embedding=8,
                    mem_capacity=CAP, mine_K=T).to(_dev())
    net.prototype_means.data.copy_(mu)
    net.queue.bank.copy_(rows)
    net.queue.mem_len.fill_(CAP)
    net.prototype_optimizer = torch.optim.Adam([{"params": net.prototype_means, "lr": 3e-3}])
    net.overlap_em = overlap
    net.train()
    return net


def _batches(n, dtype=torch.float32, channels_last=False):
    g = torch.Generator().manual_seed(1)
    out = []
    for _ in range(n):
        x = torch.randn(B, D, H, W, generator=g).to(_dev(), dtype)
        if channels_last:
            x = x.contiguous(memory_format=torch.channels_last)
        out.append((x, torch.randint(0, C, (B,), generator=g).to(_dev())))
    return out


def _loss(out, gt):
    from mgproto_b200 import ops
    return ops.mine_cross_entropy(out, gt, 0.2)


def _step(net, x, gt, between=None):
    """-> (logits, feature gradient, library launches of update_GMM: the overlapped EM adds em_commit_kernel's)."""
    from mgproto_b200 import ops
    x = x.detach().clone().requires_grad_(True)
    out = net.head(x, gt)
    _loss(out, gt).backward()
    if between is not None:
        between(net)
    n0 = ops.launch_count()
    net.update_GMM()
    return out.detach().clone(), x.grad.clone(), ops.launch_count() - n0


def _state(net):
    net.sync_optimizer_state()
    q = net.queue
    st = net.prototype_optimizer.state[net.prototype_means]
    return {"mu": net.prototype_means.detach().clone(), "weight": net.last_layer.weight.detach().clone(),
            "exp_avg": st["exp_avg"].clone(), "exp_avg_sq": st["exp_avg_sq"].clone(), "step": int(st["step"]),
            "bank": q.bank.clone(), "mem_len": q.mem_len.clone(), "head": q.head.clone(),
            "updated": q.updated.clone()}


def _assert_same(a, b, what):
    for k in a:
        if torch.is_tensor(a[k]):
            assert torch.equal(a[k], b[k]), "%s: %s differs" % (what, k)
        else:
            assert a[k] == b[k], "%s: %s %r != %r" % (what, k, a[k], b[k])


SERIAL_LAUNCHES = 2              # em_plan + em_tc_kernel in place
OVERLAP_LAUNCHES = 3             # em_plan + em_tc_kernel on the side stream, em_commit_kernel on the caller's


@pytest.mark.parametrize("dtype,channels_last", [(torch.float32, False), (torch.bfloat16, True)],
                         ids=["f32-nchw", "bf16-nhwc"])
def test_eager_steps_bit_identical(dtype, channels_last):
    steps = 6 if dtype == torch.float32 else 3
    nets = {ov: _net(ov) for ov in (True, False)}
    for i, (x, gt) in enumerate(_batches(steps, dtype, channels_last)):
        res = {ov: _step(net, x, gt) for ov, net in nets.items()}
        if i > 0:            # (the first call seeds the device Adam counter: in place)
            assert res[True][2] == OVERLAP_LAUNCHES and res[False][2] == SERIAL_LAUNCHES, (res[True][2], res[False][2])
        assert torch.equal(res[True][0], res[False][0]), "step %d: logits" % i
        assert torch.equal(res[True][1], res[False][1]), "step %d: feature gradient" % i
        _assert_same(_state(nets[True]), _state(nets[False]), "step %d" % i)


def test_graphed_replays_bit_identical():
    from mgproto_b200.pipeline import GraphedStep
    batches = _batches(6)
    res = {}
    for ov in (True, False):
        net = _net(ov)
        gs = GraphedStep(net, _loss, batches[0][0], batches[0][1], warmup=3)
        outs = []
        for x, gt in batches[1:]:
            out, _ = gs(x, gt)
            outs.append((out.clone(), gs.x_grad.clone()))
        torch.cuda.synchronize()
        res[ov] = (outs, _state(net))
        gs.close()
    for i, (a, b) in enumerate(zip(res[True][0], res[False][0])):
        assert torch.equal(a[0], b[0]), "replay %d: logits" % i
        assert torch.equal(a[1], b[1]), "replay %d: feature gradient" % i
    _assert_same(res[True][1], res[False][1], "after the replays")


def _bump_means(net):
    with torch.no_grad():
        net.prototype_means.add_(1e-3)


def _flag_all(net):
    net.queue.updated.fill_(1)


@pytest.mark.parametrize("between", [_bump_means, _flag_all], ids=["means-add", "updated-fill"])
def test_guard_takes_the_serial_order(between):
    """A write between head() and update_GMM() to something the EM reads: the EM must see it, as in the serial order."""
    nets = {ov: _net(ov) for ov in (True, False)}
    batches = _batches(3)
    for ov, net in nets.items():
        for x, gt in batches[:2]:
            _step(net, x, gt)
    res = {}
    for ov, net in nets.items():
        x, gt = batches[2]
        res[ov] = _step(net, x, gt, between=between)
        assert res[ov][2] == SERIAL_LAUNCHES, "the guard must fall back to the in-place EM"
    assert torch.equal(res[True][0], res[False][0]) and torch.equal(res[True][1], res[False][1])
    _assert_same(_state(nets[True]), _state(nets[False]), "guarded step")


def test_means_read_before_update_gmm_are_pre_step():
    """Reads of mu and pi enqueued between head() and update_GMM() run beside the EM and must see the pre-step values;
    after update_GMM() the caller's stream sees the committed ones."""
    net = _net(True)
    ref = _net(False)
    batches = _batches(3)
    for x, gt in batches[:2]:
        _step(net, x, gt)
        _step(ref, x, gt)
    x, gt = batches[2]
    mu0 = net.prototype_means.detach().clone()
    wt0 = net.last_layer.weight.detach().clone()
    seen = {}

    def read(n):
        seen["mu"] = n.prototype_means.detach().clone()
        seen["wt"] = n.last_layer.weight.detach().clone()
        seen["sum"] = n.prototype_means.detach().sum()

    assert _step(net, x, gt, between=read)[2] == OVERLAP_LAUNCHES
    _step(ref, x, gt)
    assert torch.equal(seen["mu"], mu0) and torch.equal(seen["wt"], wt0)
    assert torch.equal(seen["sum"], mu0.sum())
    assert not torch.equal(net.prototype_means.detach(), mu0)
    _assert_same(_state(net), _state(ref), "after the step")
