"""CPU: the numpy oracle of the Proxy-Anchor auxiliary loss (tests/proxy_anchor_oracle.py) against the reference's own
fp32 forward and autograd (tests/golden/proxy_anchor.npz, made by tests/golden/make_golden_proxy_anchor.py from the
unmodified utils/losses.py), and records how far the reference's fp32 sits from the fp64 oracle: the yardstick for the
GPU tolerances.  The three cases the reference cannot express (a label outside [0, C), no class present, C = 2) are
checked against central differences of the oracle's own loss."""
import os

import numpy as np
import pytest

import proxy_anchor_oracle as PA

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "proxy_anchor.npz")


@pytest.mark.parametrize("name", sorted(PA.GOLDEN_CASES))
def test_oracle_vs_reference(name):
    z = np.load(GOLD)
    assert sorted(z["cases"].tolist()) == sorted(PA.GOLDEN_CASES)
    B, C, E, seed, _ = PA.GOLDEN_CASES[name]
    assert z[name + "_dims"].tolist() == [B, C, E, seed]
    X, P, t = PA.case(name)
    loss, dx, dp = PA.proxy_anchor(X, P, t, float(z["mrg"]), float(z["beta"]), np.float64)
    e = (abs(float(z[name + "_loss"]) - loss) / abs(loss), PA.normwise(z[name + "_grad_x"], dx),
         PA.normwise(z[name + "_grad_p"], dp))
    print("reference fp32 vs fp64 oracle (%s): loss %.2e, grad_x %.2e, grad_p %.2e" % ((name,) + e))
    assert max(e) < 1e-5
    l32, dx32, dp32 = PA.proxy_anchor(X, P, t, float(z["mrg"]), float(z["beta"]), np.float32)
    assert l32.dtype == np.float32 and dx32.dtype == np.float32
    assert abs(float(l32) - loss) / abs(loss) < 1e-5 and PA.normwise(dx32, dx) < 1e-4 and PA.normwise(dp32, dp) < 1e-4


def _finite_difference(X, P, t, h=1e-6):
    f = lambda x, p: float(PA.proxy_anchor(x, p, t)[0])                          # noqa: E731
    X, P = X.astype(np.float64), P.astype(np.float64)
    dx, dp = np.zeros_like(X), np.zeros_like(P)
    for a, d in ((X, dx), (P, dp)):
        for i in np.ndindex(a.shape):
            keep = a[i]
            a[i] = keep + h
            up = f(X, P)
            a[i] = keep - h
            d[i] = (up - f(X, P)) / (2 * h)
            a[i] = keep
    return dx, dp


@pytest.mark.parametrize("what", ["label_minus_one", "no_class_present", "two_classes", "plain"])
def test_extensions_against_finite_differences(what):
    C = 2 if what == "two_classes" else 4
    X, P, t = PA.problem(6, C, 8, seed=7, rule="random")
    if what == "label_minus_one":
        t[1] = -1
        t[4] = C                                                   # C is outside [0, C) too
    elif what == "no_class_present":
        t[:] = -1
    loss, dx, dp = PA.proxy_anchor(X, P, t)
    fx, fp = _finite_difference(X, P, t)
    assert np.isfinite(loss) and PA.normwise(dx, fx) < 1e-6 and PA.normwise(dp, fp) < 1e-6
    if what == "label_minus_one":
        assert not dx[1].any() and not dx[4].any() and dx[0].any()
        keep = np.array([0, 2, 3, 5])                              # the same batch without the two images
        l2, dx2, dp2 = PA.proxy_anchor(X[keep], P, t[keep])
        assert abs(l2 - loss) < 1e-12 and np.abs(dx2 - dx[keep]).max() < 1e-12 and np.abs(dp2 - dp).max() < 1e-12
    if what == "no_class_present":
        assert loss == 0.0 and not dx.any() and not dp.any()       # log(1 + 0) over every proxy
