"""Drop-in for the reference's ``utils/losses.py`` criterion that ``main.py:187-198`` constructs: ``Proxy_Anchor``.

``from mgproto_b200 import losses`` replaces ``from utils import losses``.  The reference's forward copies the labels
to the host to one-hot encode them (utils/losses.py:9-16) and reads the number of positive proxies back (:51-52): two
device synchronisations per training step.  Here the loss and both gradients come from one CUDA launch
(csrc/aux_loss.cu) that reads nothing back, so the criterion can also be captured into a CUDA graph.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import ops

__all__ = ["Proxy_Anchor"]


class Proxy_Anchor(nn.Module):
    """ref utils/losses.py:29-61: same constructor, attributes, parameter name (``proxies``) and initialisation.  The
    parameter is created on the default device; move the module with ``.cuda()`` / ``.to()`` like any other.

    Beyond the reference: a label outside ``[0, nb_classes)`` (the head's ``gt = -1``) takes the image out of every
    sum; a batch with no labelled image gives the negative term alone instead of 0 / 0; ``nb_classes = 2`` works.
    """

    def __init__(self, nb_classes, sz_embed, mrg=0.1, beta=32):
        super().__init__()
        self.proxies = nn.Parameter(torch.randn(nb_classes, sz_embed))
        nn.init.kaiming_normal_(self.proxies, mode='fan_out')
        self.nb_classes = nb_classes
        self.sz_embed = sz_embed
        self.mrg = mrg
        self.beta = beta

    def forward(self, X, T):
        """X [B, sz_embed] fp32 / bf16 / fp16 embeddings, T [B] int64 labels -> 0-dim fp32 loss."""
        return ops.proxy_anchor(X, self.proxies, T, self.mrg, self.beta)
