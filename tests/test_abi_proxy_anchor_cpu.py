"""CPU checks of the auxiliary-loss boundary: mgp_proxy_anchor is declared in the header and bound with matching
types, its argument checks answer before any CUDA call, and mgproto_b200.losses.Proxy_Anchor has the surface the
reference's callers rely on (utils/losses.py:29-40, main.py:187-218)."""
import inspect
import os
import re

import pytest
import torch

from test_abi_cpu import ROOT, _declared


def test_symbol_declared_bound_and_exported():
    import ctypes as C
    from mgproto_b200 import _lib
    assert "mgp_proxy_anchor" in _declared()
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "mgproto_b200.h")).read(), flags=re.S)
    args = re.search(r"\bint\s+mgp_proxy_anchor\s*\(([^)]*)\)\s*;", src).group(1).split(",")
    want = []
    for a in args:
        want.append(C.c_void_p if "*" in a else C.c_float if re.search(r"\bfloat\b", a) else C.c_int)
    res, got = _lib.SIGNATURES["mgp_proxy_anchor"]
    assert res is C.c_int and got == want
    assert [a.split()[-1].lstrip("*") for a in args] == ["x", "x_dtype", "proxies", "labels", "B", "C", "E", "margin",
                                                          "beta", "loss", "grad_x", "grad_p", "n_valid", "stream"]
    assert hasattr(_lib.load(), "mgp_proxy_anchor")


def test_argument_checks_precede_any_launch():
    from mgproto_b200 import _lib
    lib = _lib.load()
    p = 4096                                                       # an aligned, never dereferenced address

    def call(B=8, C=5, E=16, x=p, dtype=_lib.MGP_X_F32, loss=p):
        return lib.mgp_proxy_anchor(x, dtype, p, p, B, C, E, 0.1, 32.0, loss, None, None, None, None)

    assert call(x=None) == -1 and call(loss=None) == -1 and call(B=0) == -1 and call(dtype=3) == -1
    assert call(dtype=_lib.MGP_X_BF16 | _lib.MGP_X_NHWC) == -1     # an element type, not a layout
    assert call(x=p + 4) == -1                                     # misaligned
    for bad in (dict(E=6), dict(E=516), dict(C=1), dict(C=4097), dict(B=4097)):
        assert call(**bad) == -2, bad


def test_module_surface_matches_reference():
    from mgproto_b200 import losses
    sig = inspect.signature(losses.Proxy_Anchor.__init__)
    assert [(n, p.default) for n, p in list(sig.parameters.items())[1:]] == [
        ("nb_classes", inspect.Parameter.empty), ("sz_embed", inspect.Parameter.empty), ("mrg", 0.1), ("beta", 32)]
    torch.manual_seed(0)
    crit = losses.Proxy_Anchor(nb_classes=200, sz_embed=32)
    assert (crit.nb_classes, crit.sz_embed, crit.mrg, crit.beta) == (200, 32, 0.1, 32)
    assert [n for n, _ in crit.named_parameters()] == ["proxies"] and list(crit.state_dict()) == ["proxies"]
    assert crit.proxies.shape == (200, 32) and crit.proxies.requires_grad and crit.proxies.device.type == "cpu"
    # kaiming_normal_(mode='fan_out') on [200, 32]: std = sqrt(2 / 200)
    assert abs(float(crit.proxies.detach().std()) - (2.0 / 200) ** 0.5) < 0.01
    other = losses.Proxy_Anchor(200, 32)
    other.load_state_dict(crit.state_dict())
    assert torch.equal(other.proxies, crit.proxies)
    import mgproto_b200
    assert mgproto_b200.losses is losses and "proxy_anchor" in mgproto_b200.ops.__all__


def test_no_cpu_path():
    from mgproto_b200 import losses
    crit = losses.Proxy_Anchor(5, 16)
    with pytest.raises(RuntimeError, match="CUDA"):
        crit(torch.randn(4, 16), torch.tensor([0, 1, 2, 3]))


def test_losses_does_not_import_the_oracle():
    src = open(os.path.join(ROOT, "mgproto_b200", "losses.py")).read()
    assert "oracle" not in src and "numpy" not in src and "sklearn" not in src
