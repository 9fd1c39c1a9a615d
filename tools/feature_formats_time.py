#!/usr/bin/env python
"""Time the feature formats of the head (bf16 / fp16, channels_last add-on features, as torch.autocast produces them).

1. The labelled head step at the bench shapes (cfg2: B = 256, HW = 196, D = 128, P = 2000, T = 20): net.head + loss +
   backward, no update_GMM, replayed from CUDA graphs.  Routes: fp32 NCHW; bf16 NCHW read natively vs the x.float() workaround; bf16
   channels_last read natively vs the x.contiguous().float() workaround (autograd then casts the gradient back).
2. The normalise forward / backward kernels alone, per format, with the bytes each must move (computed from shapes).
3. With --backbone: the whole training step with a ResNet-50 backbone (224 x 224 images, 7 x 7 features) at B = 256,
   fp32 vs bf16 autocast + channels_last.

CUDA events; every route is warmed up, then timed in blocks that alternate between the routes; the median block is
reported.  Prints the card and its power limit."""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                   # noqa: E402
from mgproto_b200 import _lib, ops             # noqa: E402


def timed_blocks(routes, steps, blocks, warmup):
    """routes: name -> fn(i) (one step on input i).  -> name -> median ms per step over the blocks."""
    for fn in routes.values():
        for i in range(warmup):
            fn(i)
    torch.cuda.synchronize()
    res = {k: [] for k in routes}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(blocks):
        for name, fn in routes.items():
            torch.cuda.synchronize()
            e0.record()
            for i in range(steps):
                fn(i)
            e1.record()
            torch.cuda.synchronize()
            res[name].append(e0.elapsed_time(e1) / steps)
    return {k: statistics.median(v) for k, v in res.items()}


def head_step_times(dev, args):
    c = bench.CFG
    B, D, H, W = c["B"], c["D"], c["H"], c["W"]
    net = bench.build_model(dev)
    gen = torch.Generator().manual_seed(1)
    n_in = 4
    x32 = [torch.randn(B, D, H, W, generator=gen).to(dev) for _ in range(n_in)]
    gts = [torch.randint(0, c["C"], (B,), generator=gen).to(dev) for _ in range(n_in)]
    inputs = {"fp32": x32,
              "bf16": [x.to(torch.bfloat16) for x in x32],
              "bf16_cl": [x.to(torch.bfloat16).to(memory_format=torch.channels_last) for x in x32]}
    for xs in inputs.values():
        for x in xs:
            x.requires_grad_(True)

    def route(key, prep):
        def fn(i):
            x = inputs[key][i % n_in]
            x.grad = None
            out = net.head(prep(x), gts[i % n_in])
            bench.loss_fn(out, gts[i % n_in]).backward()
        return fn

    routes = {"fp32 NCHW": route("fp32", lambda x: x),
              "bf16 NCHW native": route("bf16", lambda x: x),
              "bf16 NCHW x.float()": route("bf16", lambda x: x.float()),
              "bf16 channels_last native": route("bf16_cl", lambda x: x),
              "bf16 channels_last x.contiguous().float()": route("bf16_cl", lambda x: x.contiguous().float())}
    # Eagerly the step is bound by the host's ~0.5 ms of Python / ctypes work, which hides the device-side difference:
    # each (route, input) is captured once in a CUDA graph and the replays are timed.
    graphs = {}
    for name, fn in routes.items():
        graphs[name] = []
        for i in range(n_in):
            side = torch.cuda.Stream()
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    fn(i)
            torch.cuda.current_stream().wait_stream(side)
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr):
                fn(i)
            graphs[name].append(gr)
    t = timed_blocks({k: (lambda i, g=g: g[i % n_in].replay()) for k, g in graphs.items()}, args.steps, args.blocks,
                     args.warmup)
    print("\nlabelled head step (net.head + loss + backward, CUDA-graph replay), B=%d HW=%d D=%d P=%d T=%d:"
          % (B, H * W, D, c["C"] * c["K"], c["T"]))
    for k, v in t.items():
        print("  %-44s %8.1f us" % (k, v * 1e3))


def kernel_times(dev, args):
    c = bench.CFG
    B, D, H, W = c["B"], c["D"], c["H"], c["W"]
    HW, N = H * W, c["B"] * c["H"] * c["W"]
    lib = _lib.load()
    gen = torch.Generator().manual_seed(2)
    base = torch.randn(B, D, H, W, generator=gen).to(dev)
    fmts = {"fp32 NCHW": base,
            "bf16 NCHW": base.to(torch.bfloat16), "fp16 NCHW": base.to(torch.float16),
            "fp32 channels_last": base.to(memory_format=torch.channels_last),
            "bf16 channels_last": base.to(torch.bfloat16).to(memory_format=torch.channels_last),
            "fp16 channels_last": base.to(torch.float16).to(memory_format=torch.channels_last)}
    xhat, inv, _ = ops.normalize_fwd(base)
    g = torch.randn(N, D, generator=gen).to(dev)
    st = torch.cuda.current_stream().cuda_stream
    routes, nbytes = {}, {}
    for name, x in fmts.items():
        x, fmt = ops._feature_format(x)
        es = x.element_size()
        gx = torch.empty_like(x)
        xh, iv = torch.empty_like(xhat), torch.empty_like(inv)
        routes["fwd " + name] = (lambda i, x=x, fmt=fmt, xh=xh, iv=iv: lib.mgp_normalize_fwd_x(
            x.data_ptr(), fmt, xh.data_ptr(), iv.data_ptr(), None, None, 0, B, D, HW, 0, 0, st))
        nbytes["fwd " + name] = N * D * es + N * D * 4 + N * 4                 # read x; write xhat, inv_norm
        routes["bwd " + name] = (lambda i, fmt=fmt, gx=gx: lib.mgp_normalize_bwd_x(
            g.data_ptr(), xhat.data_ptr(), inv.data_ptr(), gx.data_ptr(), fmt, B, D, HW, st))
        nbytes["bwd " + name] = 2 * N * D * 4 + N * 4 + N * D * es             # read g, xhat, inv_norm; write g_x
    for fn in routes.values():
        _lib.check(fn(0), "normalize")
    t = timed_blocks(routes, args.kernel_steps, args.blocks, args.warmup)
    print("\nnormalise kernels alone, N=%d D=%d (bytes from shapes):" % (N, D))
    for k, v in t.items():
        print("  %-26s %8.1f us  %6.1f MB  %7.0f GB/s" % (k, v * 1e3, nbytes[k] / 1e6, nbytes[k] / (v * 1e-3) / 1e9))


def backbone_times(dev, args):
    import mgproto_b200 as M
    c = bench.CFG
    B = 256
    torch.manual_seed(0)
    res = {}
    for name in ("fp32 NCHW", "bf16 autocast + channels_last"):
        amp = name != "fp32 NCHW"
        net = M.construct_MGProto("resnet50", pretrained=False, img_size=224, prototype_shape=(c["C"] * c["K"], c["D"], 1, 1),
                                  num_classes=c["C"], add_on_layers_type="regular", sz_embedding=32,
                                  mem_capacity=c["cap"], mine_K=c["T"]).to(dev)
        if amp:
            net = net.to(memory_format=torch.channels_last)
        net.prototype_optimizer = torch.optim.Adam([{"params": net.prototype_means, "lr": 3e-3}])
        joint = torch.optim.Adam([{"params": net.features.parameters(), "lr": 1e-4},
                                  {"params": net.add_on_layers.parameters(), "lr": 3e-3}])
        net.train()
        gen = torch.Generator().manual_seed(3)
        imgs = [torch.randn(B, 3, 224, 224, generator=gen).to(dev) for _ in range(2)]
        if amp:
            imgs = [x.to(memory_format=torch.channels_last) for x in imgs]
        gts = [torch.randint(0, c["C"], (B,), generator=gen).to(dev) for _ in range(2)]

        def step(i, net=net, joint=joint, imgs=imgs, amp=amp):
            with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
                out, _ = net(imgs[i % 2], gts[i % 2])
                loss = bench.loss_fn(out, gts[i % 2])
            joint.zero_grad(set_to_none=True)
            loss.backward()
            joint.step()
            net.update_GMM()
        res[name] = timed_blocks({name: step}, args.backbone_steps, args.blocks, 3)[name]
        del net, joint, imgs
        torch.cuda.empty_cache()
    print("\nwhole training step, ResNet-50 backbone, B=%d, 224 x 224 images (7 x 7 features):" % B)
    for k, v in res.items():
        print("  %-32s %8.1f ms  %7.0f images/s" % (k, v, B / (v * 1e-3)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20, help="head steps per block")
    ap.add_argument("--kernel-steps", type=int, default=50, help="kernel launches per block")
    ap.add_argument("--blocks", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--backbone", action="store_true", help="also time the ResNet-50 training step")
    ap.add_argument("--backbone-steps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.set_device(0)
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                          stdout=subprocess.PIPE, text=True).stdout.strip()
    print("card: %s" % card)
    head_step_times(dev, args)
    kernel_times(dev, args)
    if args.backbone:
        backbone_times(dev, args)


if __name__ == "__main__":
    main()
