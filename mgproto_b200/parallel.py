"""Multi-GPU plumbing for the hot path (SURVEY.md section 8e): one process per GPU,
``torch.distributed`` (NCCL on GPUs, gloo in CPU tests).

The path shards by image: the head (log-likelihood, top-T, logits, backward) touches one
image's patches against replicated prototypes -- no communication.  Two exchanges keep every
rank's memory bank and prototypes identical to a single-GPU run on the concatenated batch:

* ``all_gather_records``: the per-image mined rows (top1 [B,K], rows [B,K,D], gt [B]; ~1.3 MB at
  B=256, K=10, D=128), packed into one fp32 record per image BY the gather kernel, are all-gathered in rank
  (= global image) order before the enqueue and read in place by the enqueue kernels, so every replica of the bank
  receives the whole global batch in the reference's order;
* ``update_GMM`` needs no exchange: the bank is replicated, the EM kernels are deterministic, so every rank runs
  the whole (single-launch) update on its replica and all replicas stay bit-identical.  With
  ``model.em_shard = True`` the rows are sharded instead (``shard_rows``) and the packed statistics
  [C, 1, K + K*D + 1] are all-reduced once per EM loop -- the layout for banks too large to re-reduce per rank.
"""
from __future__ import annotations

import torch
import torch.distributed as dist


def shard_rows(cap: int, world: int, rank: int):
    """Contiguous bank-slot range [r0, r1) reduced by ``rank`` (the last ranks may be empty)."""
    per = (cap + world - 1) // world
    return min(cap, rank * per), min(cap, (rank + 1) * per)


def shard_batch(global_batch: int, world: int, rank: int):
    """Image range [b0, b1) of ``rank`` for an evenly divisible global batch."""
    if global_batch % world != 0:
        raise ValueError("global batch %d not divisible by world size %d" % (global_batch, world))
    per = global_batch // world
    return rank * per, (rank + 1) * per


def all_gather_records(rec, group=None):
    """All-gather the packed per-image records ``ops.mined_gather(..., packed=True)`` wrote ([b, stride] fp32: rows,
    top-1 indices and label of every local image) in rank (= global image) order: ONE collective, no packing or
    unpacking copies -- the gather kernel writes the send buffer and the enqueue kernels read the receive buffer in
    place through strided views (ops._rec_views).  Every rank must contribute the same number of images (the
    reference's loaders use a fixed batch size; use drop_last=True): the collective's buffers are sized from it."""
    world = dist.get_world_size(group)
    if world == 1:
        return rec
    buf = torch.empty((world * rec.shape[0], rec.shape[1]), dtype=rec.dtype, device=rec.device)
    dist.all_gather_into_tensor(buf, rec, group=group)
    return buf


def all_gather_mined(top1, rows, gt, group=None):
    """(top1 [b,K] int32, rows [b,K,D] fp32, gt [b] int64) of every rank concatenated in rank order -- the tensor-level
    form of the exchange (the model's step uses ``all_gather_records``, which skips the packing below)."""
    from . import ops
    world = dist.get_world_size(group)
    if world == 1:
        return top1, rows, gt
    b, K, D = rows.shape
    if top1.dtype != torch.int32 or gt.dtype != torch.int64 or rows.dtype != torch.float32:
        raise TypeError("all_gather_mined expects int32 top1, fp32 rows, int64 gt")
    rec = torch.empty((b, ops._rec_stride(K, D)), dtype=torch.float32, device=rows.device)
    r, t, g = ops._rec_views(rec, K, D)
    r.copy_(rows.reshape(b, K * D))
    t.copy_(top1)
    g.copy_(gt)
    buf = all_gather_records(rec, group)
    r, t, g = ops._rec_views(buf, K, D)
    return t.contiguous(), r.reshape(world * b, K, D).contiguous(), g.contiguous()


def attach(model, group=None):
    """Turn on the sharded enqueue / EM for ``model`` (an ``MGProto``) on this process group."""
    model.em_group = group if group is not None else dist.group.WORLD
    return model
