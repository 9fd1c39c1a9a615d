"""GPU tests of prototype projection from the device-side candidate store (push.py, csrc/push.cu): the picks against
the float64 push_forward map and the oracle's greedy, bit-identical rows, invariance to the batch size, to the order of
the merges and to an image-sharded ("two rank") delivery, ties to the smaller image id, the operand cache after a
push, and the three kernels under the profiler."""
import numpy as np
import pytest
import torch
import torch.nn as nn

pytestmark = pytest.mark.gpu

C, K, D, H, W = 20, 10, 128, 14, 14
HW = H * W
SIGMA = 0.4          # isotropic: log p of unit-norm rows stays near -6 at D = 128, so -p = -exp(log p) is a normal fp32


def _dev():
    return torch.device("cuda:0")


def _net(c=C, k=K, d=D, h=H, seed=0):
    """A model whose conv_features returns its input: the push set is fed as add-on features (no backbone)."""
    import mgproto_b200 as M
    torch.manual_seed(seed)
    net = M.MGProto(features=nn.Sequential(nn.Conv2d(3, 16, 1)), img_size=h, prototype_shape=(c * k, d, 1, 1),
                    proto_layer_rf_info=None, num_classes=c, add_on_layers_type="regular", sz_embedding=8,
                    mem_capacity=8, mine_K=4).to(_dev())
    net.conv_features = lambda x: (x, None)
    return net


def _bench_like_data():
    """292 images [n, D, H, W] of add-on features: class 0 has 4 images (fewer than K), class 1 none, the others 16.
    Each image carries a scaled copy of a few of its class's prototype directions at random patches, so the per-image
    best values spread out and the greedy's decisions are separated."""
    g = torch.Generator().manual_seed(11)
    mu = torch.nn.functional.normalize(torch.randn(C, K, D, generator=g), dim=-1)
    labs = torch.cat([torch.zeros(4, dtype=torch.int64)] + [torch.full((16,), c, dtype=torch.int64) for c in range(2, C)])
    labs = labs[torch.randperm(labs.numel(), generator=g)]
    n = labs.numel()
    x = torch.randn(n, D, H, W, generator=g)
    for i in range(n):
        c = int(labs[i])
        for k in torch.randperm(K, generator=g)[:4].tolist():
            p = int(torch.randint(0, HW, (1,), generator=g))
            a = 4.0 + 12.0 * float(torch.rand(1, generator=g))
            x[i, :, p // W, p % W] += a * mu[c, k]
    sg = torch.full((C, K, D), SIGMA)
    return x, labs, mu, sg


def _oracle_own_class(x, labs, mu, sg):
    """float64 push_forward map of every image against its own class's K prototypes -> oracle push_argmin
    (idx [n,K], val [n,K] = min -p)."""
    from oracle import mgproto_oracle as O
    x64, mu64, sg64 = x.double().numpy(), mu.double().numpy(), sg.double().numpy()
    n = x.shape[0]
    idx = np.zeros((n, K), np.int64)
    val = np.zeros((n, K), np.float64)
    for c in np.unique(labs.numpy()):
        sel = np.nonzero(labs.numpy() == c)[0]
        _, dist = O.push_forward(x64[sel], mu64[c:c + 1], sg64[c:c + 1])
        idx[sel], val[sel] = O.push_argmin(dist, np.zeros(sel.size, np.int64), K)
    return idx, val


def _decision_margin(val, labs, chosen, c_, k_):
    """Smallest relative gap, over the greedy's decisions, between the picked image's -p and the best other image
    still available to that prototype: the picks are exact wherever this is above the kernels' error."""
    m = np.inf
    for c in range(c_):
        used = set()
        cand = np.nonzero(labs == c)[0]
        for k in range(k_):
            i = chosen[c * k_ + k]
            if i < 0:
                continue
            rest = [val[j, k] for j in cand if j != i and j not in used]
            if rest:
                m = min(m, (min(rest) - val[i, k]) / abs(val[i, k]))
            used.add(int(i))
    return m


def _loader(x, labs, bs):
    return [(x[i:i + bs], labs[i:i + bs]) for i in range(0, x.shape[0], bs)]


def _push(net, loader):
    import mgproto_b200 as M
    return M.push_prototypes(loader, net, log=lambda *_: None)


def _setup(net, mu, sg):
    with torch.no_grad():
        net.prototype_means.copy_(mu.to(_dev()))
        net.prototype_covs.copy_(sg.to(_dev()))


def test_push_store_matches_oracle_at_bench_like_shapes():
    from oracle import mgproto_oracle as O
    from mgproto_b200 import ops
    x, labs, mu, sg = _bench_like_data()
    idx, val = _oracle_own_class(x, labs, mu, sg)
    want = O.push_assign(val, labs.numpy(), C, K)
    assert _decision_margin(val, labs.numpy(), want, C, K) > 1e-4       # the data keeps every decision separated
    net = _net()
    _setup(net, mu, sg)
    mu0 = net.prototype_means.detach().clone()
    res = _push(net, _loader(x, labs, 64))
    assert res["image"].dtype == np.int64 and res["patch"].dtype == np.int64 and res["distance"].dtype == np.float32
    assert res["image"].shape == res["patch"].shape == res["distance"].shape == (C * K,)
    np.testing.assert_array_equal(res["image"], want)
    xhat = ops.normalize_fwd(x.to(_dev()))[0]                            # [n*HW, D], the rows push copies from
    x64 = x.double().numpy()
    for j in range(C * K):
        c, k = divmod(j, K)
        i = int(want[j])
        if i < 0:                                                        # class 1 (no image), class 0 beyond 4 images
            assert c == 1 or (c == 0 and k >= 4), j
            assert res["patch"][j] == -1 and np.isinf(res["distance"][j])
            assert torch.equal(net.prototype_means[c, k], mu0[c, k])
            continue
        p = int(res["patch"][j])
        if p != idx[i, k]:                                               # only a near tie in the float64 map
            from oracle import mgproto_oracle as Oc
            _, dist = Oc.push_forward(x64[i:i + 1], mu.double().numpy()[c:c + 1], sg.double().numpy()[c:c + 1])
            row = dist[0, k].reshape(-1)
            assert row[p] <= row.min() + 1e-5 * abs(row.min()), (j, p, idx[i, k])
        np.testing.assert_allclose(res["distance"][j], val[i, k], rtol=1e-4)
        assert torch.equal(net.prototype_means[c, k], xhat[i * HW + p]), j
    assert (want[C:] >= 0).all() and (want[:4] >= 0).all() and (want[4:C] == -1).all()


def test_push_store_invariant_to_batch_size_merge_order_and_sharding():
    """Push batch sizes 7 and 64 give bit-identical means and results; so do the records of the push set merged in
    reverse batch order, and each global batch delivered as two rank shards (padded with ignored records, gathered in
    rank order) -- what keeps image-sharded replicas identical."""
    from mgproto_b200 import ops
    x, labs, mu, sg = _bench_like_data()
    net = _net()
    _setup(net, mu, sg)
    r7 = _push(net, _loader(x, labs, 7))
    m7 = net.prototype_means.detach().clone()
    _setup(net, mu, sg)
    r64 = _push(net, _loader(x, labs, 64))
    assert torch.equal(net.prototype_means, m7)
    for f in ("image", "patch", "distance"):
        np.testing.assert_array_equal(r7[f], r64[f])

    def records(bs):
        out = []
        for i0 in range(0, x.shape[0], bs):
            xb, yb = x[i0:i0 + bs].to(_dev()), labs[i0:i0 + bs].to(_dev())
            arg, val, xhat = net.push_search(xb, yb)
            out.append((i0, xb.shape[0], arg, val, xhat, yb))
        return out

    # reverse order of the merges, same ids
    _setup(net, mu, sg)
    store = ops.push_store(C, K, D, _dev())
    for i0, b, arg, val, xhat, yb in reversed(records(32)):
        ops.push_merge(ops.push_records(arg, val, xhat, yb, C, HW), store, i0)
    out = ops.push_assign(store, net.prototype_means.detach()).cpu()
    assert torch.equal(net.prototype_means, m7)
    np.testing.assert_array_equal(out[0].numpy(), r7["image"])
    np.testing.assert_array_equal(out[1].numpy(), r7["patch"])

    # two "ranks": every global batch of 40 split 23 / 17, both padded to 23 records, gathered in rank order
    _setup(net, mu, sg)
    store = ops.push_store(C, K, D, _dev())
    pos = []                                                              # gathered position -> global image id
    id0 = 0
    for i0, b, arg, val, xhat, yb in records(40):
        s = min(23, b)
        shards = [(0, s), (s, b)]
        n = max(e - a for a, e in shards)
        parts = []
        for a, e in shards:
            if e > a:
                hw0, hw1 = a * HW, e * HW
                parts.append(ops.push_records(arg[a:e].contiguous(), val[a:e].contiguous(), xhat[hw0:hw1], yb[a:e],
                                              C, HW, n_out=n))
            else:
                parts.append(ops.push_padding_records(n, K, D, _dev()))
            pos += list(range(i0 + a, i0 + e)) + [-1] * (n - (e - a))
        gathered = torch.cat(parts)
        ops.push_merge(gathered, store, id0)
        id0 += gathered.shape[0]
    out = ops.push_assign(store, net.prototype_means.detach()).cpu()
    assert torch.equal(net.prototype_means, m7)
    ids = out[0].numpy()
    pos = np.asarray(pos)
    np.testing.assert_array_equal(np.where(ids >= 0, pos[np.maximum(ids, 0)], -1), r7["image"])
    np.testing.assert_array_equal(out[1].numpy(), r7["patch"])
    np.testing.assert_array_equal(out[2].view(torch.float32)[:C * K].numpy(), r7["distance"])


def test_push_ties_go_to_the_smaller_image_id():
    """Exact duplicates of images in one class tie in -p bit for bit: the earlier image id wins, whichever batch
    each copy arrives in; the greedy matches a host (-p, id) lexicographic greedy on the device's own values."""
    c_, k_, d_, h_ = 3, 4, 64, 5
    g = torch.Generator().manual_seed(3)
    base = torch.randn(3, d_, h_, h_, generator=g)
    # class 0: images 1, 4, 6 are copies of base[0]; 3 and 7 copies of base[1]; class 1 / 2 fill the rest
    x = torch.randn(9, d_, h_, h_, generator=g)
    labs = torch.tensor([1, 0, 2, 0, 0, 1, 0, 0, 2])
    for i in (1, 4, 6):
        x[i] = base[0]
    for i in (3, 7):
        x[i] = base[1]
    net = _net(c_, k_, d_, h_, seed=5)
    with torch.no_grad():
        net.prototype_covs.fill_(0.35)
    mu0 = net.prototype_means.detach().clone()
    _, val, _ = net.push_search(x.to(_dev()), labs.to(_dev()))
    val = val.cpu().numpy()
    assert val[1].tolist() == val[4].tolist() == val[6].tolist() and val[3].tolist() == val[7].tolist()
    want = np.full(c_ * k_, -1)
    for c in range(c_):
        used = set()
        cand = np.nonzero(labs.numpy() == c)[0]
        for k in range(k_):
            for i in cand[np.lexsort((cand, val[cand, k]))]:
                if int(i) not in used:
                    want[c * k_ + k] = i
                    used.add(int(i))
                    break
    for bs in (1, 4, 9):
        with torch.no_grad():
            net.prototype_means.copy_(mu0)
        res = _push(net, _loader(x, labs, bs))
        np.testing.assert_array_equal(res["image"], want)
    for k in range(k_):                                                  # a copy is only taken after its earlier twin
        i = want[k]
        assert i not in (4, 6) or 1 in want[:k]
        assert i != 7 or 3 in want[:k]


def test_compute_log_prob_after_push_sees_the_pushed_means():
    """The prototype operands cached on (data_ptr, version) of the means are rebuilt after a push: compute_log_prob
    before the push, the push, then compute_log_prob again matches float64 with the pushed means."""
    from oracle import mgproto_oracle as O
    x, labs, mu, sg = _bench_like_data()
    x, labs = x[:96], labs[:96]
    net = _net()
    _setup(net, mu, sg)
    feat = torch.nn.functional.normalize(torch.randn(300, D, generator=torch.Generator().manual_seed(2)), dim=1)
    before = net.compute_log_prob(feat.to(_dev()))
    np.testing.assert_allclose(before.cpu().numpy(), O.compute_log_prob(feat.double().numpy(), mu.double().numpy(),
                                                                        sg.double().numpy()), rtol=1e-4, atol=1e-4)
    res = _push(net, _loader(x, labs, 32))
    assert (res["image"] >= 0).sum() > C
    after = net.compute_log_prob(feat.to(_dev()))
    want = O.compute_log_prob(feat.double().numpy(), net.prototype_means.detach().double().cpu().numpy(),
                              sg.double().numpy())
    np.testing.assert_allclose(after.cpu().numpy(), want, rtol=1e-4, atol=1e-4)


def test_push_store_kernels_run():
    """All three store kernels run in a push (the profiler sees them by name)."""
    from torch.profiler import ProfilerActivity, profile
    x, labs, mu, sg = _bench_like_data()
    net = _net()
    _setup(net, mu, sg)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _push(net, _loader(x[:40], labs[:40], 20))
        torch.cuda.synchronize()
    names = " ".join(e.name for e in prof.events())
    for k in ("push_records_kernel", "push_merge_kernel", "push_assign_kernel"):
        assert k in names, k
