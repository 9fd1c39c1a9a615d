// Shared helpers for the mgproto_b200 kernels (sm_90a).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>

#include "../../include/mgproto_b200.h"

#define MGP_LOG_2PI 1.8378770664093453f

#define MGP_CHECK_LAUNCH()                               \
    do {                                                 \
        cudaError_t e__ = cudaGetLastError();            \
        if (e__ != cudaSuccess) return (int)e__;         \
    } while (0)

#define MGP_CUDA(call)                                   \
    do {                                                 \
        cudaError_t e__ = (call);                        \
        if (e__ != cudaSuccess) return (int)e__;         \
    } while (0)

static inline bool mgp_aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }
static inline size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }
// streaming multiprocessors of the current device
static inline cudaError_t mgp_sm_count(int* sms) {
    int dev = 0;
    cudaError_t e = cudaGetDevice(&dev);
    return e != cudaSuccess ? e : cudaDeviceGetAttribute(sms, cudaDevAttrMultiProcessorCount, dev);
}
// MGP_X_F32 / _BF16 / _F16, optionally | MGP_X_NHWC
static inline bool mgp_x_fmt_valid(int f) { return f >= 0 && (f & ~MGP_X_NHWC) <= MGP_X_F16; }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// monotone float <-> uint keys (larger float = larger key; 0 sorts below every float incl. -inf)
__device__ __forceinline__ unsigned f2key(float f) {
    unsigned u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key2f(unsigned k) {
    unsigned u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
    return __uint_as_float(u);
}
// (value, patch) packed so that a 64-bit max picks the larger value and, among equal values, the smaller patch
__device__ __forceinline__ unsigned long long top1_pack(float v, int hw) {
    return ((unsigned long long)f2key(v) << 32) | (unsigned long long)(0xffffffffu - (unsigned)hw);
}

// d = a * b + c lane-wise, each lane an IEEE fma (two FFMA on sm_90a)
__device__ __forceinline__ float2 ffma2(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}
