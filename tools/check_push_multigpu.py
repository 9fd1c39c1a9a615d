#!/usr/bin/env python
"""Push under image sharding: every rank pushes its DistributedSampler shard of one synthetic push set, and the
replicas must end with bit-identical prototype means, equal to a one-process push over the same images in the order
the ranks gathered them.

  torchrun --nproc_per_node 2 tools/check_push_multigpu.py [--backend gloo]

NCCL, one GPU per rank.  With --backend gloo the ranks may share a GPU (rank r uses GPU r % #GPUs), which runs the
same exchange on a one-GPU machine.  The push set (101 images of add-on features, fed without a backbone) does not divide evenly,
and the last rank drops its last batch, so the ranks run different numbers of batches with a smaller last batch: the
push's count exchange and padding are exercised.  Exits non-zero on a mismatch."""
import argparse
import os
import sys

import torch
import torch.distributed as dist
import torch.nn as nn
from torch.utils.data import DistributedSampler

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import mgproto_b200 as M  # noqa: E402
from mgproto_b200 import parallel  # noqa: E402

C, K, D, H, W, N, BS = 12, 6, 128, 14, 14, 101, 8


def _net(dev):
    torch.manual_seed(0)
    net = M.MGProto(features=nn.Sequential(nn.Conv2d(3, 16, 1)), img_size=H, prototype_shape=(C * K, D, 1, 1),
                    proto_layer_rf_info=None, num_classes=C, add_on_layers_type="regular", sz_embedding=8,
                    mem_capacity=8, mine_K=4).to(dev)
    net.conv_features = lambda x: (x, None)
    with torch.no_grad():
        net.prototype_covs.fill_(0.4)
    return net


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--backend", default="nccl", choices=("nccl", "gloo"))
    dist.init_process_group(ap.parse_args().backend)
    rank, world = dist.get_rank(), dist.get_world_size()
    dev = torch.device("cuda", int(os.environ.get("LOCAL_RANK", rank)) % torch.cuda.device_count())
    torch.cuda.set_device(dev)
    g = torch.Generator().manual_seed(1)
    x = torch.randn(N, D, H, W, generator=g)
    labs = torch.randint(0, C, (N,), generator=g)

    def shard(r):
        idx = list(DistributedSampler(range(N), num_replicas=world, rank=r, shuffle=False))
        batches = [idx[i:i + BS] for i in range(0, len(idx), BS)]
        return batches[:-1] if r == world - 1 and world > 1 else batches

    net = parallel.attach(_net(dev))
    res = M.push_prototypes([(x[b], labs[b]) for b in shard(rank)], net, log=lambda *_: None)
    mu = net.prototype_means.detach().contiguous()
    every = torch.empty((world * mu.numel(),), device=dev, dtype=mu.dtype)
    dist.all_gather_into_tensor(every, mu.reshape(-1))
    every = every.view((world,) + tuple(mu.shape))
    same = all(torch.equal(every[r], mu) for r in range(world))

    # one process over the same images in gathered order: step s = rank 0's batch s, rank 1's batch s, ...
    shards = [shard(r) for r in range(world)]
    order = [i for s in range(max(len(b) for b in shards)) for r in range(world) if s < len(shards[r])
             for i in shards[r][s]]
    ref = _net(dev)
    ref_res = M.push_prototypes([(x[order], labs[order])], ref, log=lambda *_: None)
    single = torch.equal(ref.prototype_means.detach(), mu)
    pushed = int((res["image"] >= 0).sum())
    ok = same and single and pushed == int((ref_res["image"] >= 0).sum())
    print("rank %d/%d: replicas identical %s, equal to one process %s, %d prototypes pushed" %
          (rank, world, same, single, pushed), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
