"""float64-capable numpy oracle of the per-patch class log-densities (MGProto.log_density_maps), built on the
oracle's score() / estimate_log_prob() (oracle/mgproto_oracle.py).  Test infrastructure only."""
import numpy as np

from oracle import mgproto_oracle as O


def log_density_maps(x_bdhw, mu_ckd, sigma_ckd, weight_cp):
    """model.py:403-421 (_score(..., as_average=False), eps = 1e-10 as in _estimate_log_prob :323-336) for every patch
    of a feature map and every class, on the features normalised as model.py:210-211 does; pi_c = the class-diagonal
    block of last_layer.weight.  Returns (logp_c [B,C,H,W], logp_all [B,H,W] = logsumexp over the classes: the
    per-patch form of the OoD statistic log sum_c p(x|c), train_and_test.py:199)."""
    b, d, h, w = x_bdhw.shape
    c, k, _ = mu_ckd.shape
    rows = O.features_to_rows(O.l2_normalize(x_bdhw, axis=1))
    step = max(1, (1 << 22) // max(1, k * d))          # bounds the [n, K, D] temporaries of estimate_log_prob
    out = np.empty((rows.shape[0], c), dtype=rows.dtype)
    for ci in range(c):
        pi = weight_cp[ci, ci * k:(ci + 1) * k]
        for n0 in range(0, rows.shape[0], step):
            out[n0:n0 + step, ci] = O.score(rows[n0:n0 + step], mu_ckd[ci], sigma_ckd[ci], pi, as_average=False)
    logp_c = np.ascontiguousarray(out.reshape(b, h, w, c).transpose(0, 3, 1, 2))
    return logp_c, O.logsumexp(logp_c, axis=1)
