"""Prototype projection ("push"), numeric half of the reference's push.py:82-200 (SURVEY.md section 8f-1).

For every prototype, find over the push set the image of the prototype's class whose best patch is closest
(highest p), greedily keeping images unique across prototypes (push.py:165-200), and copy that patch's normalised
feature vector into ``prototype_means``.  The reference copies the whole [B,P,H,W] distance map (401 MB at
B=256) to the host per batch and searches it with Python loops.  Here everything stays on the device:

* per batch, the per-(image, own-class prototype) arg-min (``push_search``) and one packed record per image with the
  K candidate rows, values, patches and the label (``ops.push_records``);
* the records are merged into a candidate store that keeps, per prototype, its K best candidates (``ops.push_merge``).
  Prototype k of a class picks after prototypes 0..k-1 of the same class, so its pick is always among its own k + 1
  best candidates: the store gives the reference's greedy exactly, in C*K*K*(D+4)*4 bytes (10.6 MB at 200 x 10 x 128)
  whatever the number of images;
* after the last batch the greedy runs from the store and writes the picks into ``prototype_means``
  (``ops.push_assign``), and one copy brings the result to the host.

Candidates are ordered by (-p ascending, image id ascending): exact ties in distance go to the smaller image id, where
the reference's ``np.argsort`` order is undefined.  The store is then a set that does not depend on the order in which
batches arrive.

Image-sharded replicas (``parallel.attach(net)``): every rank calls ``push_prototypes`` on its own shard of the push
set (e.g. under a ``DistributedSampler``).  Each step all-gathers the ranks' batch sizes, every rank pads its records
to the largest with ignored records, and one all-gather of the records gives every rank the same global batch, merged
into identical stores: every replica ends with the same ``prototype_means``.  The loop ends when no rank has images
left, so ranks may have different numbers of batches.  Image ids are positions in the gathered stream (padding
included); with one process they are positions in the loader's order.

The image dumping half of push.py (heat maps, bounding boxes, JPEGs) is out of scope.
"""
from __future__ import annotations

import time

import torch
import torch.distributed as dist

from . import ops
from .parallel import all_gather_records


def _unpack(item):
    """Reference loader items are ((images, labels), (paths, labels)) (utils/helpers.py MyImageFolder);
    plain (images, labels) batches are accepted too."""
    if isinstance(item[0], (tuple, list)):
        names = item[1][0] if len(item) > 1 else None
        return item[0][0], item[0][1], names
    return item[0], item[1], None


@torch.no_grad()
def push_prototypes(dataloader, prototype_network_parallel, class_specific=True, preprocess_input_function=None,
                    prototype_layer_stride=1, root_dir_for_saving_prototypes=None, epoch_number=None,
                    prototype_img_filename_prefix=None, prototype_self_act_filename_prefix=None,
                    proto_bound_boxes_filename_prefix=None, save_prototype_class_identity=True, log=print,
                    prototype_activation_function_in_numpy=None):
    """Same signature as the reference's push_prototypes (push.py:14-26); returns a dict of numpy arrays with, per
    prototype, the chosen image id (int64; -1: no image of the class was left, the prototype is unchanged), the flat
    patch index (int64, -1) and the distance -p (float32, inf)."""
    net = getattr(prototype_network_parallel, "module", prototype_network_parallel)
    net.eval()
    log("\tpush")
    start = time.time()
    C, K, D = net.prototype_means.shape
    dev = net.prototype_means.device
    group = getattr(net, "em_group", None)
    world = 1 if group is None else dist.get_world_size(group)
    store = ops.push_store(C, K, D, dev)
    batches = iter(dataloader)
    id0 = 0
    while True:
        item = next(batches, None)
        B = 0
        if item is not None:
            x, y, _ = _unpack(item)
            B = int(x.shape[0])
        n = B
        if world > 1:
            # every rank must agree on the record count of this step and on when the push ends
            mine = torch.tensor([B, item is not None], device=dev, dtype=torch.int64)
            every = torch.empty((world * 2,), device=dev, dtype=torch.int64)
            dist.all_gather_into_tensor(every, mine, group=group)
            n, alive = (int(v) for v in every.view(world, 2).max(0).values.tolist())
            if not alive:
                break
        elif item is None:
            break
        if n == 0:
            continue
        if B > 0:
            if preprocess_input_function is not None:
                x = preprocess_input_function(x)
            x = x.to(dev)
            y = torch.as_tensor(y).to(dev).long()
            x_add, _ = net.conv_features(x)                                    # push.py:107 (push_forward)
            arg, val, xhat = net.push_search(x_add, y)                         # push.py:125-158 on the device
            rec = ops.push_records(arg, val, xhat, y, C, x_add.shape[2] * x_add.shape[3], n_out=n)
        else:
            rec = ops.push_padding_records(n, K, D, dev)
        if world > 1:
            rec = all_gather_records(rec, group)
        ops.push_merge(rec, store, id0)
        id0 += rec.shape[0]

    log("\tExecuting push ...")
    mu = net.prototype_means
    out = ops.push_assign(store, mu.detach())                                  # push.py:165-200, writes mu in place
    torch.autograd.graph.increment_version(mu)       # the operand caches keyed on mu's version must see the new means
    host = out.cpu()
    log("\tpush time: \t{0}".format(time.time() - start))
    return {"image": host[0].numpy(), "patch": host[1].numpy(),
            "distance": host[2].view(torch.float32)[:C * K].numpy()}
