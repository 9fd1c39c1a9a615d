// a1: channel L2-normalisation fused with the NCHW -> [N, D] rearrangement, and its backward.
// ref: model.py:40-41, :210-211 (F.normalize(p=2, dim=1) then 'b c h w -> (b h w) c').
//
// HBM-bound: reads x once, writes xhat once (+ optional NCHW copy).  A CTA owns NT consecutive patches of one image
// and transposes them through a shared tile [D][NT+1] (pitch NT+1: conflict-free both ways); each patch row is then
// written with D contiguous floats.
//
// Feature formats (MGP_X_*): x may be fp32, bf16 or fp16, NCHW or NHWC (channels_last, i.e. [N, D] rows).  16-bit
// values are widened on load; everything after the load is fp32, and xhat, inv_norm, the staged operands and the
// NCHW copy are fp32 in every format.  The tile fill is the only format-dependent part of the forward:
//   - NCHW: warp w reads channels d = w, w+8, ...; lanes run over hw.  NT = 32 patches for fp32 and 64 for 16-bit
//     values, so that a warp reads whole 128 B lines (two 64 B halves, lanes at hw and hw + 32);
//   - NHWC: warp w reads patch rows w, w+8, ... (lanes run over d, coalesced) and stores them transposed into the tile.
// Every format sums each patch's squares in the same order (eight partials, warp w over d = w, w+8, ..., then
// w = 0..7), so xhat / inv_norm / the staged operands are bit-identical to the fp32 NCHW pass on x.float().
// The backward writes g_x in the feature format: the fp32 value is the same in every format and rounded once
// (round-to-nearest-even) for 16-bit; NCHW goes through the transposing tile, NHWC rows are written directly.
#include "mgp_common.cuh"
#include "tc_ptx.cuh"
#include <cuda_bf16.h>
#include <cuda_fp16.h>

// logprob_tc.cu: where the tensor-core log-likelihood kernels expect the patch-side operands inside their workspace
bool mgp_logprob_tc_stage_ptrs(void* ws, size_t ws_bytes, long long N, int P, int D, __half** ah, __half** al, float** sn);

namespace {

// patches per CTA
template <typename T, bool NHWC>
__host__ __device__ constexpr int tile_patches() { return (!NHWC && sizeof(T) == 2) ? 64 : 32; }

__device__ __forceinline__ float load_f32(const float* p) { return __ldg(p); }
__device__ __forceinline__ float load_f32(const __nv_bfloat16* p) { return __bfloat162float(__ldg(p)); }
__device__ __forceinline__ float load_f32(const __half* p) { return __half2float(__ldg(p)); }

template <typename T> __device__ __forceinline__ T store_as(float v);
template <> __device__ __forceinline__ float store_as<float>(float v) { return v; }
template <> __device__ __forceinline__ __nv_bfloat16 store_as<__nv_bfloat16>(float v) { return __float2bfloat16_rn(v); }
template <> __device__ __forceinline__ __half store_as<__half>(float v) { return __float2half_rn(v); }

template <typename T, bool NHWC>
__global__ void __launch_bounds__(256) normalize_fwd_kernel(const T* __restrict__ x, float* __restrict__ xhat,
                                                            float* __restrict__ inv_norm,
                                                            float* __restrict__ xhat_nchw, int D, int HW,
                                                            __half* __restrict__ ah, __half* __restrict__ al,
                                                            float* __restrict__ sn, int stage_aniso) {
    constexpr int NT = tile_patches<T, NHWC>();
    constexpr int PL = NT / 32;      // patches per lane: lane + 32 * j
    extern __shared__ float tile[];  // [D][NT+1]
    __shared__ float red[8][NT];
    __shared__ float s_inv[NT];
    const int b = blockIdx.y;
    const int hw0 = blockIdx.x * NT;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float ss[PL];
#pragma unroll
    for (int j = 0; j < PL; ++j) ss[j] = 0.f;
    if constexpr (NHWC) {
        const T* xb = x + ((size_t)b * HW + hw0) * D;
        for (int r = warp; r < NT; r += 8) {
            const bool okr = hw0 + r < HW;
            for (int d = lane; d < D; d += 32) tile[d * (NT + 1) + r] = okr ? load_f32(xb + (size_t)r * D + d) : 0.f;
        }
        __syncthreads();
        for (int d = warp; d < D; d += 8) {
            const float v = tile[d * (NT + 1) + lane];
            ss[0] += v * v;
        }
    } else if constexpr (PL == 1) {
        // (the j loop below computes the same, but ptxas schedules this form's loads ~10 % faster at D = 128)
        const T* xb = x + (size_t)b * D * HW;
        const int hw = hw0 + lane;
        const bool ok = hw < HW;
        for (int d = warp; d < D; d += 8) {
            float v = ok ? load_f32(xb + (size_t)d * HW + hw) : 0.f;
            tile[d * (NT + 1) + lane] = v;
            ss[0] += v * v;
        }
    } else {
        const T* xb = x + (size_t)b * D * HW;
        for (int d = warp; d < D; d += 8) {
#pragma unroll
            for (int j = 0; j < PL; ++j) {
                const int hw = hw0 + lane + 32 * j;
                float v = hw < HW ? load_f32(xb + (size_t)d * HW + hw) : 0.f;
                tile[d * (NT + 1) + lane + 32 * j] = v;
                ss[j] += v * v;
            }
        }
    }
#pragma unroll
    for (int j = 0; j < PL; ++j) red[warp][lane + 32 * j] = ss[j];
    __syncthreads();
    if (warp == 0) {
#pragma unroll
        for (int j = 0; j < PL; ++j) {
            const int hw = hw0 + lane + 32 * j;
            float t = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) t += red[w][lane + 32 * j];
            float inv = 1.0f / fmaxf(sqrtf(t), 1e-12f);
            s_inv[lane + 32 * j] = inv;
            if (hw < HW) inv_norm[(size_t)b * HW + hw] = inv;
        }
    }
    __syncthreads();
    // [N, D] rows: warp w writes patches w, w+8, ...; lanes run over d (conflict-free: pitch NT+1)
    for (int r = warp; r < NT; r += 8) {
        if (hw0 + r >= HW) break;
        const float inv = s_inv[r];
        const size_t n = (size_t)b * HW + hw0 + r;
        float* dst = xhat + n * D;
        if (ah == nullptr) {
            for (int d = lane; d < D; d += 32) dst[d] = tile[d * (NT + 1) + r] * inv;
        } else {
            // ... and the operands the tensor-core log-likelihood kernels read (csrc/logprob_tc.cu tc_x_prep_kernel: rows
            // of [N, 2D] fp16, hi / lo split of X_SCALE * [ x^2 | x ], the x^2 half only on request; sn = |xhat|^2)
            __half* hr = ah + n * 2 * D;
            __half* lr = al + n * 2 * D;
            float ss = 0.f;
            for (int d = lane; d < D; d += 32) {
                const float a = tile[d * (NT + 1) + r] * inv;
                dst[d] = a;
                ss = fmaf(a, a, ss);
                mgp_tc::split_f16(a * mgp_tc::X_SCALE, hr[D + d], lr[D + d]);
                if (stage_aniso) mgp_tc::split_f16(a * a * mgp_tc::X_SCALE, hr[d], lr[d]);
            }
            ss = warp_sum(ss);
            if (lane == 0) sn[n] = ss;
        }
    }
    if (xhat_nchw != nullptr) {
#pragma unroll
        for (int j = 0; j < PL; ++j) {
            const int hw = hw0 + lane + 32 * j;
            if (hw >= HW) break;
            const float inv = s_inv[lane + 32 * j];
            float* dst = xhat_nchw + (size_t)b * D * HW + hw;
            for (int d = warp; d < D; d += 8) dst[(size_t)d * HW] = tile[d * (NT + 1) + lane + 32 * j] * inv;
        }
    }
}

// g_x = (g - xhat <xhat, g>) * inv_norm, written back in the feature format.
template <typename T, bool NHWC>
__global__ void __launch_bounds__(256) normalize_bwd_kernel(const float* __restrict__ g, const float* __restrict__ xhat,
                                                            const float* __restrict__ inv_norm,
                                                            T* __restrict__ gx, int D, int HW) {
    constexpr int NT = tile_patches<T, NHWC>();
    extern __shared__ float tile[];  // NCHW: [D][NT+1] holds g_x rows
    const int b = blockIdx.y;
    const int hw0 = blockIdx.x * NT;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int r = warp; r < NT; r += 8) {
        if (hw0 + r >= HW) break;
        const size_t n = (size_t)b * HW + hw0 + r;
        const float* gr = g + n * D;
        const float* xr = xhat + n * D;
        float dot = 0.f;
        for (int d = lane; d < D; d += 32) dot += gr[d] * xr[d];
        dot = warp_sum(dot);
        const float inv = inv_norm[n];
        if constexpr (NHWC) {
            for (int d = lane; d < D; d += 32) gx[n * D + d] = store_as<T>((gr[d] - xr[d] * dot) * inv);
        } else {
            for (int d = lane; d < D; d += 32) tile[d * (NT + 1) + r] = (gr[d] - xr[d] * dot) * inv;
        }
    }
    if constexpr (!NHWC) {
        __syncthreads();
#pragma unroll
        for (int j = 0; j < NT / 32; ++j) {
            const int hw = hw0 + lane + 32 * j;
            if (hw < HW) {
                T* dst = gx + (size_t)b * D * HW + hw;
                for (int d = warp; d < D; d += 8) dst[(size_t)d * HW] = store_as<T>(tile[d * (NT + 1) + lane + 32 * j]);
            }
        }
    }
}

template <typename T, bool NHWC>
int launch_fwd(const void* x, float* xhat_nd, float* inv_norm, float* xhat_nchw, int B, int D, int HW, __half* ah,
               __half* al, float* sn, int stage_aniso, cudaStream_t st) {
    constexpr int NT = tile_patches<T, NHWC>();
    const size_t smem = (size_t)D * (NT + 1) * sizeof(float);
    if (smem > 200 * 1024) return MGP_ERR_UNSUPPORTED;
    MGP_CUDA(cudaFuncSetAttribute(normalize_fwd_kernel<T, NHWC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((HW + NT - 1) / NT, B);
    normalize_fwd_kernel<T, NHWC><<<grid, 256, smem, st>>>(static_cast<const T*>(x), xhat_nd, inv_norm, xhat_nchw, D, HW,
                                                            ah, al, sn, stage_aniso);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

template <typename T, bool NHWC>
int launch_bwd(const float* g_xhat_nd, const float* xhat_nd, const float* inv_norm, void* g_x, int B, int D, int HW,
               cudaStream_t st) {
    constexpr int NT = tile_patches<T, NHWC>();
    const size_t smem = NHWC ? 0 : (size_t)D * (NT + 1) * sizeof(float);
    if (smem > 200 * 1024) return MGP_ERR_UNSUPPORTED;
    MGP_CUDA(cudaFuncSetAttribute(normalize_bwd_kernel<T, NHWC>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    dim3 grid((HW + NT - 1) / NT, B);
    normalize_bwd_kernel<T, NHWC><<<grid, 256, smem, st>>>(g_xhat_nd, xhat_nd, inv_norm, static_cast<T*>(g_x), D, HW);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

}  // namespace

// one instantiation per feature format (mgp_x_fmt_valid() has been checked)
#define MGP_X_DISPATCH(fmt, FN, ...)                                              \
    switch (fmt) {                                                                \
        case MGP_X_F32: return FN<float, false>(__VA_ARGS__);                     \
        case MGP_X_BF16: return FN<__nv_bfloat16, false>(__VA_ARGS__);            \
        case MGP_X_F16: return FN<__half, false>(__VA_ARGS__);                    \
        case MGP_X_F32 | MGP_X_NHWC: return FN<float, true>(__VA_ARGS__);         \
        case MGP_X_BF16 | MGP_X_NHWC: return FN<__nv_bfloat16, true>(__VA_ARGS__); \
        case MGP_X_F16 | MGP_X_NHWC: return FN<__half, true>(__VA_ARGS__);        \
        default: return MGP_ERR_INVALID;                                          \
    }

extern "C" int mgp_normalize_fwd_x(const void* x, int x_fmt, float* xhat_nd, float* inv_norm, float* xhat_nchw,
                                   void* ws, size_t ws_bytes, int B, int D, int HW, int P, int stage_aniso,
                                   void* stream) {
    if (!x || !mgp_x_fmt_valid(x_fmt) || !xhat_nd || !inv_norm || B <= 0 || D <= 0 || HW <= 0) return MGP_ERR_INVALID;
    __half *ah = nullptr, *al = nullptr;
    float* sn = nullptr;
    if (ws != nullptr) {
        if (P <= 0) return MGP_ERR_INVALID;
#ifdef MGP_WITH_TC
        if (!mgp_logprob_tc_stage_ptrs(ws, ws_bytes, (long long)B * HW, P, D, &ah, &al, &sn)) return MGP_ERR_WORKSPACE;
#else
        (void)ws_bytes;
        return MGP_ERR_UNSUPPORTED;
#endif
    }
    MGP_X_DISPATCH(x_fmt, launch_fwd, x, xhat_nd, inv_norm, xhat_nchw, B, D, HW, ah, al, sn, stage_aniso ? 1 : 0,
                   (cudaStream_t)stream)
}

extern "C" int mgp_normalize_fwd(const float* x_nchw, float* xhat_nd, float* inv_norm, float* xhat_nchw, int B,
                                 int D, int HW, void* stream) {
    return mgp_normalize_fwd_x(x_nchw, MGP_X_F32, xhat_nd, inv_norm, xhat_nchw, nullptr, 0, B, D, HW, 0, 0, stream);
}

extern "C" int mgp_normalize_fwd_stage(const float* x_nchw, float* xhat_nd, float* inv_norm, float* xhat_nchw, void* ws,
                                       size_t ws_bytes, int B, int D, int HW, int P, int stage_aniso, void* stream) {
    if (!ws) return MGP_ERR_INVALID;
    return mgp_normalize_fwd_x(x_nchw, MGP_X_F32, xhat_nd, inv_norm, xhat_nchw, ws, ws_bytes, B, D, HW, P, stage_aniso,
                               stream);
}

extern "C" int mgp_normalize_bwd_x(const float* g_xhat_nd, const float* xhat_nd, const float* inv_norm, void* g_x,
                                   int x_fmt, int B, int D, int HW, void* stream) {
    if (!g_xhat_nd || !xhat_nd || !inv_norm || !g_x || !mgp_x_fmt_valid(x_fmt) || B <= 0 || D <= 0 || HW <= 0)
        return MGP_ERR_INVALID;
    MGP_X_DISPATCH(x_fmt, launch_bwd, g_xhat_nd, xhat_nd, inv_norm, g_x, B, D, HW, (cudaStream_t)stream)
}

extern "C" int mgp_normalize_bwd(const float* g_xhat_nd, const float* xhat_nd, const float* inv_norm,
                                 float* g_x_nchw, int B, int D, int HW, void* stream) {
    return mgp_normalize_bwd_x(g_xhat_nd, xhat_nd, inv_norm, g_x_nchw, MGP_X_F32, B, D, HW, stream);
}
