// a8/a9: enqueue of the mined top-1 patches into the per-class FIFO memory bank.
// ref: model.py:225-250 (dedupe per image, class-ascending, image order), utils/memory.py:31-73
// (FIFO with eviction of the oldest rows).
//
// The reference keeps each class buffer physically ordered oldest->newest by shifting it on
// every push and runs ~B*K host-synchronising torch.unique / torch.where calls; here the bank
// is one [C, cap, D] ring (head[c], mem_len[c]) and an iteration's enqueue is three small fully
// parallel launches with no host synchronisation: per-image dedupe, per-class offsets / ring
// arithmetic, row scatter.  Row order inside a class does not change any EM result except through
// fp32 summation order; mgp_bank_linearize reproduces the reference layout on demand.
#include <cuda_fp16.h>

#include "mgp_common.cuh"
#include "tc_ptx.cuh"

namespace {

// fp16 hi / lo split of X_SCALE x (tc_ptx.cuh) + |x|^2: the tensor-core EM kernel (em_tc.cu) TMA-loads these tiles instead of converting fp32 rows on chip.
__device__ __forceinline__ void shadow_store_row(const float* __restrict__ src, __half* __restrict__ xh,
                                                 __half* __restrict__ xl, float* __restrict__ xx, size_t row, int D,
                                                 int lane) {
    float ss = 0.f;
    for (int d4 = lane; d4 < D / 4; d4 += 32) {
        const float4 v = *reinterpret_cast<const float4*>(src + 4 * d4);
        const float a[4] = {v.x, v.y, v.z, v.w};
        __align__(8) __half h[4], l[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            ss = fmaf(a[i], a[i], ss);
            mgp_tc::split_f16(a[i] * mgp_tc::X_SCALE, h[i], l[i]);
        }
        *reinterpret_cast<uint2*>(xh + row * D + 4 * d4) = *reinterpret_cast<uint2*>(h);
        *reinterpret_cast<uint2*>(xl + row * D + 4 * d4) = *reinterpret_cast<uint2*>(l);
    }
    ss = warp_sum(ss);
    if (lane == 0) xx[row] = ss;
}

__global__ void bank_shadow_kernel(const float* __restrict__ bank, __half* __restrict__ xh, __half* __restrict__ xl,
                                   float* __restrict__ xx, long long rows, int D) {
    const long long wg = (long long)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (wg >= rows) return;
    shadow_store_row(bank + (size_t)wg * D, xh, xl, xx, (size_t)wg, D, threadIdx.x & 31);
}

// ---------------------------------------------------------------------------------------------------------------
// Planner, three small fully parallel launches (the single-CTA planner they replace took 27 us for 256 images and
// ~200 us for the 2048-image global batch of an 8-GPU run):
//   1. enqueue_dedupe_kernel   warp per image: rank of each of its K top-1 indices among the image's distinct values
//                              (ascending, torch.unique's order; -1 for duplicates), number of distinct values, class
//   2. enqueue_offsets_kernel  warp per class: running row offsets of the class's images in batch order (prefix scan
//                              over the batch), the class's ring base and accepted row count, new mem_len / head / flag
//   3. enqueue_scatter_kernel  warp per (image, prototype): slot = (base[c] + offs[b] + rank) % cap, row copy
// scratch (int32): plan [B*K] ranks | cls [B] | ucount [B] | offs [B] | base [C] | macc [C]
__global__ void __launch_bounds__(256)
enqueue_dedupe_kernel(const int32_t* __restrict__ top1_bk, const int64_t* __restrict__ gt, int32_t* __restrict__ plan,
                      int32_t* __restrict__ cls, int32_t* __restrict__ ucount, int B, int C, int K, int top1_stride,
                      int gt_stride) {
    const int lane = threadIdx.x & 31;
    const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (b >= B) return;
    const long long c = gt[(size_t)b * gt_stride];
    const bool okc = (c >= 0 && c < C);
    const int32_t* top1 = top1_bk + (size_t)b * top1_stride;
    if (K <= 32) {
        // lane per prototype: duplicates by MATCH.ANY, rank among the distinct values by K shuffles
        const int v = (okc && lane < K) ? top1[lane] : (-1 - lane);
        const unsigned m = __match_any_sync(0xffffffffu, v);
        const bool first = okc && lane < K && (__ffs(m) - 1 == lane);
        const unsigned fm = __ballot_sync(0xffffffffu, first);
        int rank = 0;
        for (int j = 0; j < K; ++j) {
            const int vj = __shfl_sync(0xffffffffu, v, j);
            rank += (((fm >> j) & 1u) && vj < v) ? 1 : 0;
        }
        if (lane < K) plan[(size_t)b * K + lane] = first ? rank : -1;
        if (lane == 0) { cls[b] = okc ? (int)c : -1; ucount[b] = __popc(fm); }
    } else {
        int u = 0;
        for (int k = lane; k < K; k += 32) {
            int rank = -1;
            if (okc) {
                const int v = top1[k];
                bool first = true;
                for (int k2 = 0; k2 < k; ++k2) first = first && (top1[k2] != v);
                if (first) {
                    rank = 0;
                    for (int k2 = 0; k2 < K; ++k2) {
                        const int v2 = top1[k2];
                        if (v2 < v) {
                            bool f2 = true;
                            for (int k3 = 0; k3 < k2; ++k3) f2 = f2 && (top1[k3] != v2);
                            rank += f2 ? 1 : 0;
                        }
                    }
                    ++u;
                }
            }
            plan[(size_t)b * K + k] = rank;
        }
        u = __reduce_add_sync(0xffffffffu, u);
        if (lane == 0) { cls[b] = okc ? (int)c : -1; ucount[b] = u; }
    }
}

__global__ void __launch_bounds__(128)
enqueue_offsets_kernel(int64_t* __restrict__ mem_len, int32_t* __restrict__ head, uint8_t* __restrict__ updated,
                       const int32_t* __restrict__ cls, const int32_t* __restrict__ ucount, int32_t* __restrict__ offs,
                       int32_t* __restrict__ base, int32_t* __restrict__ macc, int B, int C, int cap) {
    const int lane = threadIdx.x & 31;
    const int c = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (c >= C) return;
    int off = 0;
    for (int b0 = 0; b0 < B; b0 += 32) {                    // rows of class c accepted before each of its images (image order)
        const int b = b0 + lane;
        const bool mine = (b < B) && (__ldg(cls + b) == c);
        const int u = mine ? __ldg(ucount + b) : 0;
        int incl = u;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const int y = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += y;
        }
        if (mine) offs[b] = off + incl - u;
        off += __shfl_sync(0xffffffffu, incl, 31);
    }
    if (lane == 0) {
        const int m = min(off, cap);                        // a push larger than the capacity keeps its first cap rows
        const int len = (int)mem_len[c];
        const int hd = head[c];
        base[c] = (hd + len) % cap;
        macc[c] = m;
        if (m > 0) {
            if (len + m <= cap) {
                mem_len[c] = len + m;
            } else {
                head[c] = (hd + (len + m - cap)) % cap;
                mem_len[c] = cap;
            }
            updated[c] = 1;                                  // ref model.py:250
        }
    }
}

// top-1 patch of each of the GT class's K prototypes: spatial index and feature row
__global__ void mined_gather_kernel(const float* __restrict__ xhat, const int32_t* __restrict__ idx,
                                    const int64_t* __restrict__ gt, int32_t* __restrict__ top1,
                                    float* __restrict__ rows, int B, int HW, int C, int K, int D, int T, int rows_stride,
                                    int top1_stride) {
    const int wg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (wg >= B * K) return;
    const int b = wg / K, k = wg - b * K;
    const long long c = gt[b];
    float4* dst = reinterpret_cast<float4*>(rows + (size_t)b * rows_stride + (size_t)k * D);
    if (c < 0 || c >= C) {
        if (lane == 0) top1[(size_t)b * top1_stride + k] = -1;
        for (int d = lane; d < D / 4; d += 32) dst[d] = make_float4(0.f, 0.f, 0.f, 0.f);
        return;
    }
    const int n = idx[((size_t)b * C * K + (size_t)c * K + k) * T];     // level 0 (ref model.py:225-226)
    if (lane == 0) top1[(size_t)b * top1_stride + k] = n;
    const float4* src = reinterpret_cast<const float4*>(xhat + ((size_t)b * HW + n) * D);
    for (int d = lane; d < D / 4; d += 32) dst[d] = src[d];
}

__global__ void enqueue_scatter_kernel(float* __restrict__ bank, const float* __restrict__ rows,
                                       const int32_t* __restrict__ plan, const int32_t* __restrict__ cls,
                                       const int32_t* __restrict__ offs, const int32_t* __restrict__ base,
                                       const int32_t* __restrict__ macc, __half* __restrict__ xh, __half* __restrict__ xl,
                                       float* __restrict__ xx, int B, int K, int D, int cap, int rows_stride) {
    const int wg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (wg >= B * K) return;
    const int r = plan[wg];
    if (r < 0) return;                                       // duplicate index of this image, or image without a class
    const int sb = wg / K, sk = wg - sb * K;
    const int c = cls[sb];
    const int o = offs[sb] + r;
    if (o >= macc[c]) return;                                // beyond the capacity of one push
    const int slot = (base[c] + o) % cap;
    const float* srow = rows + (size_t)sb * rows_stride + (size_t)sk * D;
    const float4* src = reinterpret_cast<const float4*>(srow);
    float4* dst = reinterpret_cast<float4*>(bank + ((size_t)c * cap + slot) * D);
    for (int d = lane; d < D / 4; d += 32) dst[d] = src[d];
    if (xh) shadow_store_row(srow, xh, xl, xx, (size_t)c * cap + slot, D, lane);   // keep the shadow in step
}

__global__ void bank_linearize_kernel(const float* __restrict__ bank, const int64_t* __restrict__ mem_len,
                                      const int32_t* __restrict__ head, float* __restrict__ lin, int C, int cap,
                                      int D) {
    const int wg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (wg >= C * cap) return;
    const int c = wg / cap, r = wg - c * cap;
    float* dst = lin + (size_t)wg * D;
    if (r < (int)mem_len[c]) {
        const float* src = bank + ((size_t)c * cap + (head[c] + r) % cap) * D;
        for (int d = lane; d < D; d += 32) dst[d] = src[d];
    } else {
        for (int d = lane; d < D; d += 32) dst[d] = 0.f;
    }
}

}  // namespace

extern "C" int mgp_mined_gather(const float* xhat_nd, const int32_t* idx, const int64_t* gt, int32_t* top1,
                               float* rows, int rows_stride, int top1_stride, int B, int HW, int C, int K, int D, int T,
                               void* stream) {
    if (!xhat_nd || !idx || !gt || !top1 || !rows) return MGP_ERR_INVALID;
    if (B <= 0 || HW <= 0 || C <= 0 || K <= 0 || D <= 0 || T <= 0 || (D & 3)) return MGP_ERR_INVALID;
    if (rows_stride == 0) rows_stride = K * D;
    if (top1_stride == 0) top1_stride = K;
    if (rows_stride < K * D || (rows_stride & 3) || top1_stride < K || !mgp_aligned16(rows)) return MGP_ERR_INVALID;
    const int warps = B * K;
    mined_gather_kernel<<<(warps + 7) / 8, 256, 0, (cudaStream_t)stream>>>(xhat_nd, idx, gt, top1, rows, B, HW, C, K, D, T,
                                                                          rows_stride, top1_stride);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" int mgp_bank_enqueue(float* bank, int64_t* mem_len, int32_t* head, uint8_t* updated, const float* rows,
                                const int32_t* top1, const int64_t* gt, int rows_stride, int top1_stride, int gt_stride,
                                int32_t* plan, void* shadow_h, void* shadow_l, float* shadow_xx, int B, int C, int K, int D,
                                int cap, void* stream) {
    if (!bank || !mem_len || !head || !updated || !rows || !top1 || !gt || !plan) return MGP_ERR_INVALID;
    if ((shadow_h != nullptr) != (shadow_l != nullptr) || (shadow_h != nullptr) != (shadow_xx != nullptr)) return MGP_ERR_INVALID;
    if (B <= 0 || C <= 0 || K <= 0 || D <= 0 || cap <= 0 || (D & 3)) return MGP_ERR_INVALID;
    if (K > 1024) return MGP_ERR_UNSUPPORTED;
    if (rows_stride == 0) rows_stride = K * D;
    if (top1_stride == 0) top1_stride = K;
    if (gt_stride == 0) gt_stride = 1;
    if (rows_stride < K * D || (rows_stride & 3) || top1_stride < K || gt_stride < 1 || !mgp_aligned16(rows)) return MGP_ERR_INVALID;
    cudaStream_t st = (cudaStream_t)stream;
    int32_t* cls = plan + (size_t)B * K;
    int32_t* ucount = cls + B;
    int32_t* offs = ucount + B;
    int32_t* base = offs + B;
    int32_t* macc = base + C;
    enqueue_dedupe_kernel<<<(B + 7) / 8, 256, 0, st>>>(top1, gt, plan, cls, ucount, B, C, K, top1_stride, gt_stride);
    MGP_CHECK_LAUNCH();
    enqueue_offsets_kernel<<<(C + 3) / 4, 128, 0, st>>>(mem_len, head, updated, cls, ucount, offs, base, macc, B, C, cap);
    MGP_CHECK_LAUNCH();
    const int warps = B * K;
    enqueue_scatter_kernel<<<(warps + 7) / 8, 256, 0, st>>>(bank, rows, plan, cls, offs, base, macc,
                                                            reinterpret_cast<__half*>(shadow_h),
                                                            reinterpret_cast<__half*>(shadow_l), shadow_xx, B, K, D, cap,
                                                            rows_stride);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" size_t mgp_bank_enqueue_plan_ints(int B, int C, int K) { return (size_t)B * K + 3 * (size_t)B + 2 * (size_t)C; }

extern "C" int mgp_bank_shadow_sync(const float* bank, void* shadow_h, void* shadow_l, float* shadow_xx, int C, int cap,
                                    int D, void* stream) {
    if (!bank || !shadow_h || !shadow_l || !shadow_xx || C <= 0 || cap <= 0 || D <= 0 || (D & 3)) return MGP_ERR_INVALID;
    const long long rows = (long long)C * cap;
    bank_shadow_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(
        bank, reinterpret_cast<__half*>(shadow_h), reinterpret_cast<__half*>(shadow_l), shadow_xx, rows, D);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" int mgp_bank_linearize(const float* bank, const int64_t* mem_len, const int32_t* head, float* lin, int C,
                                  int cap, int D, void* stream) {
    if (!bank || !mem_len || !head || !lin || C <= 0 || cap <= 0 || D <= 0) return MGP_ERR_INVALID;
    const int warps = C * cap;
    bank_linearize_kernel<<<(warps + 7) / 8, 256, 0, (cudaStream_t)stream>>>(bank, mem_len, head, lin, C, cap, D);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}
