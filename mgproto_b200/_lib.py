"""ctypes binding of libmgproto_b200.so (the C ABI declared in include/mgproto_b200.h).

The library is the product: there is no CPU or PyTorch fallback.  Importing this module
without the built library raises; calling an op without a CUDA device raises.
"""
from __future__ import annotations

import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libmgproto_b200.so")

MGP_MATH_FP32, MGP_MATH_TC, MGP_MATH_AUTO, MGP_MATH_TC_REUSE, MGP_MATH_TC_ISO, MGP_MATH_TC_ISO_REUSE = 0, 1, 2, 3, 4, 5
MGP_MATH_X_STAGED, MGP_MATH_X_STAGED_ISO = 0x100, 0x200
MGP_OUT_LOGP_NP, MGP_OUT_LOGP_BPHW, MGP_OUT_NEGP_BPHW, MGP_OUT_TOP1_BP = 0, 1, 2, 3
MGP_X_F32, MGP_X_BF16, MGP_X_F16, MGP_X_NHWC = 0, 1, 2, 4

_vp, _i, _f, _sz, _d = C.c_void_p, C.c_int, C.c_float, C.c_size_t, C.c_double

# name -> (restype, argtypes); mirrors include/mgproto_b200.h one to one
SIGNATURES = {
    "mgp_abi_version": (_i, []),
    "mgp_error_string": (C.c_char_p, [_i]),
    "mgp_has_tensor_core_path": (_i, []),
    "mgp_set_option": (_i, [C.c_char_p, _i]),
    "mgp_debug_set_ptr": (_i, [C.c_char_p, _vp, _i]),
    "mgp_normalize_fwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "mgp_normalize_bwd": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "mgp_logprob_ws_bytes": (_sz, [_i, _i, _i, _i, _i]),
    "mgp_normalize_fwd_stage": (_i, [_vp, _vp, _vp, _vp, _vp, _sz, _i, _i, _i, _i, _i, _vp]),
    "mgp_normalize_fwd_x": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _sz, _i, _i, _i, _i, _i, _vp]),
    "mgp_normalize_bwd_x": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "mgp_logprob_ws_is_prototype_only": (_i, [_i, _i, _i, _i]),
    "mgp_logprob_fwd": (_i, [_vp, _vp, _vp, _f, _f, _vp, _i, _i, _i, _i, _i, _i, _vp, _sz, _vp]),
    "mgp_log_density_ws_bytes": (_sz, [_i] * 6),
    "mgp_log_density": (_i, [_vp] * 6 + [_i] * 6 + [_vp, _sz, _vp]),
    "mgp_head_select": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "mgp_head_select_np": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "mgp_head_select_top1": (_i, [_vp] * 9 + [_i] * 6 + [_vp]),
    "mgp_head_bwd_ws_bytes": (_sz, [_i, _i, _i, _i]),
    "mgp_head_bwd": (_i, [_vp] * 11 + [_sz, _vp] + [_i] * 6 + [_vp]),
    "mgp_head_bwd_x": (_i, [_vp] * 11 + [_sz, _vp] + [_i] * 7 + [_vp]),
    "mgp_head_select_long": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "mgp_head_select_top1_long": (_i, [_vp] * 9 + [_i] * 6 + [_vp]),
    "mgp_head_bwd_long_ws_bytes": (_sz, [_i, _i, _i, _i]),
    "mgp_head_bwd_long_x": (_i, [_vp] * 11 + [_sz, _vp] + [_i] * 7 + [_vp]),
    "mgp_mined_gather": (_i, [_vp] * 5 + [_i] * 8 + [_vp]),
    "mgp_bank_enqueue": (_i, [_vp] * 7 + [_i] * 3 + [_vp] * 4 + [_i] * 5 + [_vp]),
    "mgp_bank_enqueue_plan_ints": (_sz, [_i, _i, _i]),
    "mgp_bank_shadow_sync": (_i, [_vp] * 4 + [_i] * 3 + [_vp]),
    "mgp_bank_linearize": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "mgp_em_stat_stride": (_sz, [_i, _i, _i]),
    "mgp_update_gmm_launches": (_i, [_i, _i, _i, _i, _i]),
    "mgp_update_gmm": (_i, [_vp] * 4 + [_i] + [_vp] * 12 + [_i, _i] + [_f] + [_d] * 5 + [_f] + [_i] * 4 + [_vp]),
    "mgp_update_gmm_staged": (_i, [_vp] * 15 + [_i, _i, _f] + [_d] * 5 + [_f, _vp, _vp] + [_i] * 4 + [_vp]),
    "mgp_em_commit": (_i, [_vp] * 4 + [_i] * 3 + [_vp]),
    "mgp_em_plan": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "mgp_em_stats": (_i, [_vp, _vp, _vp, _vp, _vp, _f, _i, _i, _i, _i, _vp, _i, _i, _i, _i, _vp]),
    "mgp_em_update": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i,
                           _d, _d, _d, _d, _d, _f, _vp, _i, _i, _i, _i, _vp]),
    "mgp_em_estep": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "mgp_em_mstep_closed": (_i, [_vp, _vp, _f, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "mgp_em_mstep_div": (_i, [_vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "mgp_ood_score": (_i, [_vp, _i, _i, _vp, _vp, _vp, _i, _i, _vp]),
    "mgp_topt_pool": (_i, [_vp] * 5 + [_i] * 6 + [_vp]),
    "mgp_mine_ce": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _f, _vp]),
    "mgp_proxy_anchor": (_i, [_vp, _i, _vp, _vp, _i, _i, _i, _f, _f, _vp, _vp, _vp, _vp, _vp]),
    "mgp_push_argmin": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _vp]),
    "mgp_push_argmin_top1": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _vp]),
    "mgp_push_records": (_i, [_vp] * 8 + [_i] * 6 + [_vp]),
    "mgp_push_merge": (_i, [_vp] * 4 + [_i, _i, _sz] + [_vp] * 3 + [_i] * 3 + [_vp]),
    "mgp_push_assign": (_i, [_vp] * 7 + [_i] * 3 + [_vp]),
}

_lib = None


class MGProtoLibraryError(RuntimeError):
    pass


def load():
    """Load (once) and return the ctypes handle.  Raises if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    try:
        if not os.path.exists(LIB_PATH):
            raise OSError("not built")
        lib = C.CDLL(LIB_PATH)
        for name in SIGNATURES:
            getattr(lib, name)
    except (OSError, AttributeError) as first:
        # missing or stale library: rebuild it in-tree with nvcc (a build step, not a fallback)
        try:
            from .build import build
            build(force=True)
            lib = C.CDLL(LIB_PATH)
        except Exception as e:  # noqa: BLE001
            raise MGProtoLibraryError(
                "libmgproto_b200.so could not be loaded (%s) or rebuilt (%s). Run `python -m "
                "mgproto_b200.build` (needs nvcc, sm_90a). There is no CPU fallback." % (first, e)) from e
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is missing: fail loudly
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(code: int, what: str):
    if code != 0:
        msg = load().mgp_error_string(int(code))
        raise MGProtoLibraryError("%s failed (%d): %s" % (what, code, msg.decode() if msg else "?"))
