// C-ABI glue: version / error strings and the log-likelihood dispatcher.
#include "mgp_common.cuh"
#include <stdlib.h>
#include <string.h>

int mgp_logprob_simt_launch(const float* xhat, const float* mu, const float* sigma, float eps, float eps_log,
                            float* out, int layout, int B, int HW, int P, int D, float* ws, cudaStream_t st);
// logprob_tc.cu
bool mgp_logprob_tc_supported(int layout, int B, int HW, int P, int D, int assume_iso);
size_t mgp_logprob_tc_ws_bytes(long long N, int P, int D);
int mgp_logprob_tc_launch(const float* xhat, const float* mu, const float* sigma, float eps, float eps_log,
                          float* out, int layout, int B, int HW, int P, int D, void* ws, size_t ws_bytes,
                          int reuse_operands, int assume_iso, int x_staged, cudaStream_t st);

extern "C" int mgp_abi_version(void) { return MGP_ABI_VERSION; }

extern "C" const char* mgp_error_string(int code) {
    switch (code) {
        case MGP_OK: return "ok";
        case MGP_ERR_INVALID: return "mgproto_b200: invalid argument (null pointer, non-positive size or misalignment)";
        case MGP_ERR_UNSUPPORTED: return "mgproto_b200: shape not supported by the sm_90a kernels";
        case MGP_ERR_WORKSPACE: return "mgproto_b200: workspace too small";
        default: break;
    }
    if (code > 0) return cudaGetErrorString((cudaError_t)code);
    return "mgproto_b200: unknown error";
}

int g_mgp_em_fused = -1;   // -1: not decided yet (environment), see mgp_opt_em_fused()
int mgp_opt_em_fused() {
    if (g_mgp_em_fused < 0) g_mgp_em_fused = getenv("MGP_EM_UNFUSED") ? 0 : 1;
    return g_mgp_em_fused;
}
void mgp_em_tc_set_prof(void* p, int cls);   // em_tc.cu
extern "C" int mgp_debug_set_ptr(const char* key, void* p, int arg) {
    if (!key) return MGP_ERR_INVALID;
#ifdef MGP_WITH_TC
    if (strcmp(key, "em_tc_prof") == 0) { mgp_em_tc_set_prof(p, arg); return MGP_OK; }
#endif
    return MGP_ERR_INVALID;
}
int g_mgp_tc_z = -1;
int mgp_opt_tc_z() {
    if (g_mgp_tc_z < 0) g_mgp_tc_z = getenv("MGP_TC_NO_Z") ? 0 : 1;
    return g_mgp_tc_z;
}
int g_mgp_em_tc = -1;
int mgp_opt_em_tc() {
    if (g_mgp_em_tc < 0) g_mgp_em_tc = getenv("MGP_EM_NO_TC") ? 0 : 1;
    return g_mgp_em_tc;
}
extern "C" int mgp_set_option(const char* key, int value) {
    if (!key) return MGP_ERR_INVALID;
    if (strcmp(key, "tc_z") == 0) {
        const int prev = mgp_opt_tc_z();
        g_mgp_tc_z = value ? 1 : 0;
        return prev;
    }
    if (strcmp(key, "em_tc") == 0) {
        const int prev = mgp_opt_em_tc();
        g_mgp_em_tc = value ? 1 : 0;
        return prev;
    }
    if (strcmp(key, "em_fused") == 0) {
        const int prev = mgp_opt_em_fused();
        g_mgp_em_fused = value ? 1 : 0;
        return prev;
    }
    return MGP_ERR_INVALID;
}

extern "C" int mgp_has_tensor_core_path(void) {
#ifdef MGP_WITH_TC
    return 1;
#else
    return 0;
#endif
}

extern "C" size_t mgp_logprob_ws_bytes(int B, int HW, int P, int D, int math) {
    size_t simt = ((size_t)P * D + P) * sizeof(float);
#ifdef MGP_WITH_TC
    if (math != MGP_MATH_FP32 && mgp_logprob_tc_supported(0, B, HW, P, D, math == MGP_MATH_TC_ISO || math == MGP_MATH_TC_ISO_REUSE)) {
        size_t tc = mgp_logprob_tc_ws_bytes((long long)B * HW, P, D);
        return tc > simt ? tc : simt;
    }
#endif
    (void)math; (void)B; (void)HW;
    return simt;
}

bool mgp_logprob_tcz_supported(int P, int D);   // logprob_tcz.cu
extern "C" int mgp_logprob_ws_is_prototype_only(int out_layout, int P, int D, int math) {
#ifdef MGP_WITH_TC
    return (out_layout == MGP_OUT_LOGP_NP && (math == MGP_MATH_TC_ISO || math == MGP_MATH_TC_ISO_REUSE) && mgp_opt_tc_z() &&
            P > 0 && mgp_logprob_tcz_supported(P, D)) ? 1 : 0;
#else
    (void)out_layout; (void)P; (void)D; (void)math;
    return 0;
#endif
}

extern "C" int mgp_logprob_fwd(const float* xhat_nd, const float* mu, const float* sigma, float eps, float eps_log,
                               float* out, int out_layout, int B, int HW, int P, int D, int math, void* ws,
                               size_t ws_bytes, void* stream) {
    // MGP_MATH_X_STAGED / MGP_MATH_X_STAGED_ISO: the patch-side operands of `ws` were written by mgp_normalize_fwd_stage
    const int x_staged = (math & MGP_MATH_X_STAGED_ISO) ? 1 : ((math & MGP_MATH_X_STAGED) ? 2 : 0);
    math &= 0xff;
    if (!xhat_nd || !mu || !sigma || !out || !ws) return MGP_ERR_INVALID;
    if (B <= 0 || HW <= 0 || P <= 0 || D <= 0 || (D & 3)) return MGP_ERR_INVALID;
    if (out_layout < MGP_OUT_LOGP_NP || out_layout > MGP_OUT_TOP1_BP) return MGP_ERR_INVALID;
    if (!mgp_aligned16(xhat_nd) || !mgp_aligned16(mu) || !mgp_aligned16(sigma) || !mgp_aligned16(out) ||
        !mgp_aligned16(ws))
        return MGP_ERR_INVALID;
    if ((long long)B * HW > 0x7fffffffLL) return MGP_ERR_UNSUPPORTED;
    if (ws_bytes < mgp_logprob_ws_bytes(B, HW, P, D, math)) return MGP_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
#ifdef MGP_WITH_TC
    const bool iso_mode = (math == MGP_MATH_TC_ISO || math == MGP_MATH_TC_ISO_REUSE);
    if (math == MGP_MATH_TC || math == MGP_MATH_AUTO || math == MGP_MATH_TC_REUSE || iso_mode) {
        if (mgp_logprob_tc_supported(out_layout, B, HW, P, D, iso_mode))
            return mgp_logprob_tc_launch(xhat_nd, mu, sigma, eps, eps_log, out, out_layout, B, HW, P, D, ws, ws_bytes,
                                         math == MGP_MATH_TC_REUSE ? 2 : (math == MGP_MATH_TC_ISO_REUSE ? 1 : 0), iso_mode,
                                         x_staged, st);
        if (math != MGP_MATH_AUTO) return MGP_ERR_UNSUPPORTED;
    }
#else
    if (math == MGP_MATH_TC || math == MGP_MATH_TC_REUSE || math == MGP_MATH_TC_ISO || math == MGP_MATH_TC_ISO_REUSE)
        return MGP_ERR_UNSUPPORTED;
#endif
    if (out_layout == MGP_OUT_TOP1_BP) return MGP_ERR_UNSUPPORTED;   // fused max/arg-max exists on the tensor-core path only
    return mgp_logprob_simt_launch(xhat_nd, mu, sigma, eps, eps_log, out, out_layout, B, HW, P, D,
                                   reinterpret_cast<float*>(ws), st);
}
