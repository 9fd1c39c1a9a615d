"""CPU checks of the staged update_GMM entry points (mgp_update_gmm_staged, mgp_em_commit): argument validation runs
before any CUDA call and refuses null pointers, bad sizes, misalignment and staging that aliases the parameters."""
import ctypes

import pytest

C, K, D, CAP, L, NS = 4, 3, 128, 8, 3, 2


def _lib():
    from mgproto_b200 import _lib
    return _lib.load()


def _buf(nbytes):
    """16-byte aligned host memory (never dereferenced: validation fails before any launch)."""
    raw = ctypes.create_string_buffer(nbytes + 16)
    addr = (ctypes.addressof(raw) + 15) & ~15
    return raw, addr


@pytest.fixture
def ptrs():
    keep, p = [], {}
    for name in ("sh", "sl", "sxx", "status", "updated", "mem_len", "mu", "sigma", "weight", "m", "v", "step", "order",
                 "sched", "stats", "mu_stage", "pi_stage"):
        raw, addr = _buf(64)
        keep.append(raw)
        p[name] = addr
    p["_keep"] = keep
    return p


def _staged(p, **over):
    a = dict(p, **over)
    return _lib().mgp_update_gmm_staged(a["sh"], a["sl"], a["sxx"], a["status"], a["updated"], a["mem_len"], a["mu"],
                                        a["sigma"], a["weight"], a["m"], a["v"], a["step"], a["order"], a["sched"],
                                        a["stats"], a.get("n_split", NS), a.get("L", L), 0.1, 3e-3, 0.9, 0.999, 1e-8,
                                        0.99, 1.0, a["mu_stage"], a["pi_stage"], a.get("C", C), K, a.get("D", D), CAP,
                                        None)


@pytest.mark.parametrize("name", ["sh", "sl", "sxx", "status", "updated", "mem_len", "mu", "sigma", "weight", "m", "v",
                                  "step", "order", "sched", "stats", "mu_stage", "pi_stage"])
def test_update_gmm_staged_refuses_null(ptrs, name):
    assert _staged(ptrs, **{name: None}) == -1


def test_update_gmm_staged_refuses_bad_sizes_and_aliasing(ptrs):
    assert _staged(ptrs, C=0) == -1
    assert _staged(ptrs, L=0) == -1
    assert _staged(ptrs, n_split=0) == -1
    assert _staged(ptrs, D=130) == -2                          # D % 4 != 0: no kernel takes it
    assert _staged(ptrs, mu_stage=ptrs["mu"]) == -1            # the staging must not alias what the kernel reads
    assert _staged(ptrs, pi_stage=ptrs["weight"]) == -1


def test_em_commit_validation(ptrs):
    lib = _lib()
    p = ptrs
    assert lib.mgp_em_commit(None, p["pi_stage"], p["mu"], p["weight"], C, K, D, None) == -1
    assert lib.mgp_em_commit(p["mu_stage"], None, p["mu"], p["weight"], C, K, D, None) == -1
    assert lib.mgp_em_commit(p["mu_stage"], p["pi_stage"], None, p["weight"], C, K, D, None) == -1
    assert lib.mgp_em_commit(p["mu_stage"], p["pi_stage"], p["mu"], None, C, K, D, None) == -1
    assert lib.mgp_em_commit(p["mu_stage"], p["pi_stage"], p["mu"], p["weight"], 0, K, D, None) == -1
    assert lib.mgp_em_commit(p["mu_stage"], p["pi_stage"], p["mu"], p["weight"], C, K, 126, None) == -1
    assert lib.mgp_em_commit(p["mu_stage"] + 4, p["pi_stage"], p["mu"], p["weight"], C, K, D, None) == -1
    assert lib.mgp_em_commit(p["mu_stage"], p["pi_stage"], p["mu"] + 4, p["weight"], C, K, D, None) == -1


def test_overlap_em_is_on_by_default_and_single_replica_only():
    import mgproto_b200 as M
    net = M.construct_MGProto("resnet18", pretrained=False, prototype_shape=(12, 16, 1, 1), num_classes=4,
                              add_on_layers_type="regular", sz_embedding=8, mem_capacity=8, mine_K=3)
    assert net.overlap_em is True
    assert net._em_fork is None
    assert not net._em_fork_holds(None)
