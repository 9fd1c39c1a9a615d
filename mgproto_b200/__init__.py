"""mgproto_b200 -- CUDA-native (H100, sm_90a) implementation of MGProto's Gaussian-prototype hot path.

Drop-in for the reference's ``model`` module on that path: ``construct_MGProto``, ``MGProto``
(forward / push_forward / update_GMM / compute_log_prob / _e_step / ...), ``MemoryBank``.
The compute lives in ``libmgproto_b200.so`` (hand-written sm_90a CUDA behind the C ABI in
``include/mgproto_b200.h``); importing the package requires the built library.
"""
from . import _lib

_lib.load()   # fail loudly at import if the CUDA library is missing -- there is no fallback

from . import losses, ops  # noqa: E402
from .memory import MemoryBank  # noqa: E402
from .model import (MGProto, NonNegLinear, construct_MGProto, l2_normalize, momentum_update)  # noqa: E402
from .push import push_prototypes  # noqa: E402

__all__ = ["MGProto", "NonNegLinear", "MemoryBank", "construct_MGProto", "l2_normalize", "momentum_update", "ops",
           "push_prototypes", "losses"]
__version__ = "0.1.0"
