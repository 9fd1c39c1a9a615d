"""Pins the per-patch class log-density oracle (tests/log_density_oracle.py) against the reference's own _score
(tests/golden/log_density.npz, written by tests/golden/make_golden_log_density.py).  CPU only."""
import os

import numpy as np
import pytest

import log_density_oracle as LD

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "log_density.npz")


@pytest.mark.parametrize("case", ["init", "aniso"])
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_log_density_oracle_vs_reference(case, dtype):
    g = np.load(GOLDEN)
    pre = case + "_"
    lc, la = LD.log_density_maps(*(g[pre + k].astype(dtype) for k in ("x_add", "mu", "sigma", "weight")))
    assert lc.shape == g[pre + "logp_c"].shape and la.shape == g[pre + "logp_all"].shape
    np.testing.assert_allclose(lc, g[pre + "logp_c"], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(la, g[pre + "logp_all"], rtol=1e-5, atol=1e-5)
    # the pruned prototype (pi = 0) still enters through log(0 + 1e-10), as in the reference
    assert g[pre + "weight"][0, 2 if case == "init" else 4] == 0.0
