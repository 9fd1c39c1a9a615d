"""Numpy oracle of the Proxy-Anchor auxiliary loss and the seeded cases its golden fixture was recorded on  --  TEST
INFRASTRUCTURE ONLY (the product package never imports it).

``proxy_anchor`` restates utils/losses.py:19-61 of the reference (cwangrun/MGProto @ 02a3042) in closed form, value and
both gradients; tests/test_oracle_proxy_anchor.py pins it to the reference's own fp32 autograd
(tests/golden/proxy_anchor.npz, written by tests/golden/make_golden_proxy_anchor.py).  Arithmetic is done in ``dtype``
(float64 for an error-attribution oracle, float32 for a like-for-like one).
"""
import numpy as np

GOLDEN_CASES = {                       # name -> (B, C, E, seed, label rule)
    "repeat": (8, 5, 16, 101, "repeat"),          # one class three times, another twice
    "batch80": (80, 200, 32, 102, "random"),      # the reference's batch size: most classes absent
    "oneclass": (64, 37, 128, 103, "one"),        # every image in one class
}


def case(name):
    """Inputs of a golden case, from its seed: X [B,E] fp32, P [C,E] fp32, t [B] int64."""
    B, C, E, seed, rule = GOLDEN_CASES[name]
    return problem(B, C, E, seed, rule)


def problem(B, C, E, seed, rule="random"):
    r = np.random.RandomState(seed)
    X = r.standard_normal((B, E)).astype(np.float32)
    P = (r.standard_normal((C, E)) * np.sqrt(2.0 / C)).astype(np.float32)      # the scale kaiming_normal_(fan_out) gives
    if rule == "random":
        t = r.randint(0, C, size=B)
    elif rule == "one":
        t = np.full(B, C // 3)
    elif rule == "all":                                                        # every class present
        t = np.arange(B) % C
    else:
        t = r.randint(0, C, size=B)
        t[:3] = 1
        t[3:5] = C - 1
    return X, P, t.astype(np.int64)


def proxy_anchor(X, P, t, mrg=0.1, beta=32.0, dtype=np.float64):
    """utils/losses.py:41-61 and its gradients -> (loss, dL/dX [B,E], dL/dP [C,E]).

    :19-26 l2_norm (1e-12 inside the root) on both sides, :44 cosines, :48-49 the two exponentials, :54-55 their sums
    over the positive / negative images of every proxy, :57-59 log(1 + .) averaged over the proxies that have a positive
    (:51-52) and over all proxies.  Beyond the reference: a label outside [0, C) takes the image out of every sum, and
    without any positive proxy the first term is 0."""
    X, P = np.asarray(X).astype(dtype), np.asarray(P).astype(dtype)
    t = np.asarray(t)
    B, C = X.shape[0], P.shape[0]
    mrg, beta = dtype(mrg), dtype(beta)
    nx = np.sqrt((X * X).sum(1) + dtype(1e-12))[:, None]
    npr = np.sqrt((P * P).sum(1) + dtype(1e-12))[:, None]
    xh, ph = X / nx, P / npr
    s = xh @ ph.T
    valid = (t >= 0) & (t < C)
    pos = np.zeros((B, C), bool)
    pos[np.nonzero(valid)[0], t[valid]] = True
    neg = valid[:, None] & ~pos
    ep = np.where(pos, np.exp(-beta * (s - mrg)), dtype(0))
    en = np.where(neg, np.exp(beta * (s + mrg)), dtype(0))
    sp, sn = ep.sum(0), en.sum(0)
    nv = int(pos.any(0).sum())
    loss = np.log1p(sn).sum() / dtype(C)
    a = beta * en / ((1 + sn) * dtype(C))
    if nv > 0:
        loss = loss + np.log1p(sp).sum() / dtype(nv)
        a = a - beta * ep / ((1 + sp) * dtype(nv))
    gx, gp = a @ ph, a.T @ xh
    dx = (gx - xh * (xh * gx).sum(1, keepdims=True)) / nx
    dp = (gp - ph * (ph * gp).sum(1, keepdims=True)) / npr
    return dtype(loss), dx.astype(dtype), dp.astype(dtype)


def normwise(a, b):
    """max |a - b| / max |b| (0 when both vanish)."""
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    den = np.abs(b).max()
    err = np.abs(a - b).max()
    return 0.0 if err == 0.0 else float(err / den) if den > 0 else float("inf")
