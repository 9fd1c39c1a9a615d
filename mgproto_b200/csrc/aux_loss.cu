// Auxiliary loss: the Proxy-Anchor criterion on the embedding (ref: utils/losses.py:19-61, called at
// train_and_test.py:42), value and both gradients from ONE launch of one thread-block cluster.
//
//   xh_b = X_b / sqrt(|X_b|^2 + 1e-12)    ph_c = P_c / sqrt(|P_c|^2 + 1e-12)    s_bc = xh_b . ph_c
//   S+_c = sum_{b: t_b = c} exp(-beta (s_bc - mrg))      S-_c = sum_{b: t_b != c} exp(beta (s_bc + mrg))
//   L = (1/|C+|) sum_c log(1 + S+_c) + (1/C) sum_c log(1 + S-_c)
//   a_bc = dL/ds_bc = -beta e+_bc / ((1 + S+_c) |C+|)  for t_b = c,   beta e-_bc / ((1 + S-_c) C)  otherwise
//   dL/dph_c = sum_b a_bc xh_b,  dL/dxh_b = sum_c a_bc ph_c,  then the normalisation backward (g - v (v . g)) / |.|
//
// Layout.  A cluster of 8 CTAs x 16 warps.  Every output has exactly one writer and every sum a fixed order (lane-local
// sequence, xor-shuffle tree, rank-0 block tree): no atomics, bit-identical from run to run.
//   phase A  CTA r owns a contiguous slice of the classes, one class per warp at a time.  The warp keeps ph_c in shared
//            memory (broadcast reads) and streams the normalised embeddings through a shared-memory tile, a lane per
//            image: sweep 1 gives S+_c and S-_c, which it writes into EVERY CTA's [C] arrays through distributed shared
//            memory; sweep 2 recomputes s_bc, forms a_bc and accumulates dL/dph_c (lane = embedding dim, a_bc
//            broadcast by shuffle), and finishes dP_c in registers.
//   sync     cluster barrier; rank 0 sums log1p(S+-) over the classes into the loss; every CTA turns its copy of S+- into
//            the per-class coefficients -beta / ((1 + S+) |C+|) and beta / ((1 + S-) C).
//   phase B  CTA r owns a contiguous slice of the IMAGES, one image per warp at a time, and streams the normalised
//            proxies through the tile, a lane per class: s_bc a third time, a_bc from the coefficient arrays, dL/dxh_b
//            in registers, dX_b finished and rounded to X's dtype.
// dX is summed where the image lives instead of being reduced over the class slices: that costs one more pass over
// s_bc (B C E = 1.6 M FMAs at 256 x 200 x 32) and removes a [8, B, E] exchange, whose 8 MB at the largest shape
// would fit neither shared memory nor an ABI without workspaces.  |C+| is counted by every CTA from the labels, so the
// only cluster traffic is 2 C floats per CTA.
// Three passes are 10 MFLOP at the default shape: latency, not throughput, so the math is fp32 FMAs, not wgmma.
#include "mgp_common.cuh"

#include <cooperative_groups.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>

namespace cg = cooperative_groups;

namespace {

constexpr int PA_CLUSTER = 8;
constexpr int PA_WARPS = 16;
constexpr int PA_THREADS = PA_WARPS * 32;
constexpr int PA_MAX_B = 4096, PA_MAX_C = 4096, PA_MAX_E = 512;
constexpr int PA_TILE_FLOATS = 24576;      // streamed tile: at most 96 KB of rows of E + 4 floats

struct PaParams {
    const void* x;
    const float* p;
    const int64_t* labels;
    float* loss;
    void* grad_x;
    float* grad_p;
    int32_t* n_valid;
    int B, C, E, tj;                       // tj: rows of the streamed tile, a multiple of 32
    float margin, beta;
};

extern __shared__ float4 pa_smem[];

template <class T> __device__ __forceinline__ float4 pa_ld4(const T* row, int q);
template <> __device__ __forceinline__ float4 pa_ld4<float>(const float* row, int q) {
    return __ldg(reinterpret_cast<const float4*>(row) + q);
}
template <> __device__ __forceinline__ float4 pa_ld4<__nv_bfloat16>(const __nv_bfloat16* row, int q) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(row) + q);
    const float2 a = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.x));
    const float2 b = __bfloat1622float2(*reinterpret_cast<const __nv_bfloat162*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
template <> __device__ __forceinline__ float4 pa_ld4<__half>(const __half* row, int q) {
    const uint2 u = __ldg(reinterpret_cast<const uint2*>(row) + q);
    const float2 a = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
    const float2 b = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
    return make_float4(a.x, a.y, b.x, b.y);
}
__device__ __forceinline__ void pa_st(float* p, float v) { *p = v; }
__device__ __forceinline__ void pa_st(__nv_bfloat16* p, float v) { *p = __float2bfloat16_rn(v); }
__device__ __forceinline__ void pa_st(__half* p, float v) { *p = __float2half_rn(v); }

// One warp: dst[0..E) = v / sqrt(|v|^2 + 1e-12) (ref utils/losses.py:19-26: the 1e-12 is inside the root); returns
// the factor.  Every lane rereads only what it wrote itself.
template <class T>
__device__ __forceinline__ float pa_load_unit(const T* src, float* dst, int E, int lane) {
    float4* d4 = reinterpret_cast<float4*>(dst);
    float ss = 0.f;
    for (int q = lane; q < (E >> 2); q += 32) {
        const float4 v = pa_ld4<T>(src, q);
        d4[q] = v;
        ss = fmaf(v.x, v.x, ss); ss = fmaf(v.y, v.y, ss); ss = fmaf(v.z, v.z, ss); ss = fmaf(v.w, v.w, ss);
    }
    ss = warp_sum(ss);
    const float r = 1.0f / sqrtf(ss + 1e-12f);
    for (int q = lane; q < (E >> 2); q += 32) {
        float4 v = d4[q];
        v.x *= r; v.y *= r; v.z *= r; v.w *= r;
        d4[q] = v;
    }
    return r;
}

// All warps: rows j0 .. j0 + tj of src [n, E], normalised, into the tile (rows past n: zeros, label -1).
template <class T>
__device__ __forceinline__ void pa_load_tile(const T* src, int n, int j0, int tj, int E, float* s_tile, int* s_lab,
                                             const int64_t* labels, int C, int warp, int lane) {
    const int stride = E + 4;
    for (int j = warp; j < tj; j += PA_WARPS) {
        const int jj = j0 + j;
        float* dst = s_tile + j * stride;
        if (jj < n) {
            pa_load_unit<T>(src + (size_t)jj * E, dst, E, lane);
        } else {
            for (int q = lane; q < (E >> 2); q += 32) reinterpret_cast<float4*>(dst)[q] = make_float4(0.f, 0.f, 0.f, 0.f);
        }
        if (labels != nullptr && lane == 0) {
            int lab = -1;
            if (jj < n) {
                const long long t = labels[jj];
                if (t >= 0 && t < C) lab = (int)t;
            }
            s_lab[j] = lab;
        }
    }
}

// One warp, one own vector u (a class in modes 0 / 1, an image in mode 2) against the nrows valid rows of the tile,
// a lane per row.  MODE 0: sp / sn += e+ / e- of the pairs;  MODE 1 / 2: acc[k] (dim lane + 32 k) += a_bc * row.
//   modes 0 / 1: own = class c, the rows are images with labels s_lab, coefficients wpos / wneg;
//   mode 2:      own = label of the image, the rows are classes j0 + j with coefficients s_wp / s_wn.
template <int KE, int MODE>
__device__ __forceinline__ void pa_sweep(const float* s_tile, int E, int nrows, int j0, const float* u, int lane, int own,
                                         const int* s_lab, float wpos, float wneg, const float* s_wp, const float* s_wn,
                                         float margin, float beta, float& sp, float& sn, float (&acc)[KE]) {
    const int stride = E + 4;
    const float4* u4 = reinterpret_cast<const float4*>(u);
    const int ngroups = (nrows + 31) >> 5;
#pragma unroll 1
    for (int g = 0; g < ngroups; ++g) {
        const int j = g * 32 + lane;
        const float4* row = reinterpret_cast<const float4*>(s_tile + j * stride);
        float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll 2
        for (int q = 0; q < (E >> 2); ++q) {
            const float4 a = row[q], b = u4[q];
            s0 = fmaf(a.x, b.x, s0); s1 = fmaf(a.y, b.y, s1); s2 = fmaf(a.z, b.z, s2); s3 = fmaf(a.w, b.w, s3);
        }
        const float s = (s0 + s1) + (s2 + s3);
        bool ok, pos;
        float wp, wn;
        if (MODE == 2) {
            const int jj = j0 + j;
            ok = j < nrows;
            pos = jj == own;
            wp = ok ? s_wp[jj] : 0.f;
            wn = ok ? s_wn[jj] : 0.f;
        } else {
            const int lab = s_lab[j];
            ok = lab >= 0;
            pos = lab == own;
            wp = wpos;
            wn = wneg;
        }
        const float e = pos ? expf(-beta * (s - margin)) : expf(beta * (s + margin));
        if (MODE == 0) {
            if (ok) {
                if (pos) sp += e; else sn += e;
            }
        } else {
            const float a = ok ? (pos ? wp : wn) * e : 0.f;
            const float* base = s_tile + g * 32 * stride + lane;
#pragma unroll(KE >= 16 ? 1 : 4)
            for (int jl = 0; jl < 32; ++jl) {
                const float aj = __shfl_sync(0xffffffffu, a, jl);
                const float* r = base + jl * stride;
#pragma unroll
                for (int k = 0; k < KE; ++k)
                    if (lane + 32 * k < E) acc[k] = fmaf(aj, r[32 * k], acc[k]);
            }
        }
    }
}

// (g - u (u . g)) * r for the warp's vector u, written to out[0..E) in out's type
template <int KE, class TO>
__device__ __forceinline__ void pa_finish(const float (&acc)[KE], const float* u, float r, TO* out, int E, int lane) {
    float dot = 0.f;
#pragma unroll
    for (int k = 0; k < KE; ++k)
        if (lane + 32 * k < E) dot = fmaf(acc[k], u[lane + 32 * k], dot);
    dot = warp_sum(dot);
#pragma unroll
    for (int k = 0; k < KE; ++k)
        if (lane + 32 * k < E) pa_st(out + lane + 32 * k, (acc[k] - u[lane + 32 * k] * dot) * r);
}

template <class T, int KE>
__device__ __forceinline__ void pa_body(const PaParams& p) {
    cg::cluster_group cluster = cg::this_cluster();
    const int rank = (int)cluster.block_rank();
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int B = p.B, C = p.C, E = p.E, tj = p.tj, stride = E + 4;
    const int C4 = (C + 3) & ~3;
    const float margin = p.margin, beta = p.beta;

    float* s_tile = reinterpret_cast<float*>(pa_smem);       // [tj][E + 4]
    float* s_u = s_tile + tj * stride;               // [PA_WARPS][E]: the warp's own unit vector
    float* s_sp = s_u + PA_WARPS * E;                        // [C]: S+ of every class, later its coefficient
    float* s_sn = s_sp + C4;                                 // [C]: S-
    int* s_lab = reinterpret_cast<int*>(s_sn + C4);          // [tj]: labels of the images in the tile, -1 = none
    float* s_red = reinterpret_cast<float*>(s_lab + tj);     // [2 PA_WARPS]
    float* u = s_u + warp * E;

    // |C+|: every CTA counts the classes present in the batch (s_sp holds the flags until the cluster starts)
    int* s_flag = reinterpret_cast<int*>(s_sp);
    for (int c = tid; c < C; c += PA_THREADS) s_flag[c] = 0;
    __syncthreads();
    for (int b = tid; b < B; b += PA_THREADS) {
        const long long t = p.labels[b];
        if (t >= 0 && t < C) s_flag[t] = 1;
    }
    __syncthreads();
    int cnt = 0;
    for (int c = tid; c < C; c += PA_THREADS) cnt += s_flag[c];
    cnt = __reduce_add_sync(0xffffffffu, cnt);
    if (lane == 0) reinterpret_cast<int*>(s_red)[warp] = cnt;
    __syncthreads();
    int nv = 0;
    for (int w = 0; w < PA_WARPS; ++w) nv += reinterpret_cast<const int*>(s_red)[w];
    const float wpos0 = nv > 0 ? -beta / (float)nv : 0.f;    // no class present: the positive term and its gradient are 0
    const float wneg0 = beta / (float)C;
    cluster.sync();                                          // every CTA runs and is done with its flags: S+- may arrive

    int cur = -1;                                            // tile resident in s_tile
    // ---- phase A: classes [c_begin, c_end), images streamed
    {
        const int Cs = (C + PA_CLUSTER - 1) / PA_CLUSTER;
        const int c_begin = rank * Cs, c_end = min(C, c_begin + Cs);
        const int ntiles = (B + tj - 1) / tj, rounds = (Cs + PA_WARPS - 1) / PA_WARPS;
        const T* x = reinterpret_cast<const T*>(p.x);
        for (int round = 0; round < rounds; ++round) {
            const int c = c_begin + round * PA_WARPS + warp;
            const bool have = c < c_end;
            float rp = 0.f;
            __syncwarp();
            if (have) rp = pa_load_unit<float>(p.p + (size_t)c * E, u, E, lane);
            __syncwarp();
            float sp = 0.f, sn = 0.f, acc[KE];
#pragma unroll
            for (int k = 0; k < KE; ++k) acc[k] = 0.f;
            for (int t = 0; t < ntiles; ++t) {
                if (cur != t) {
                    __syncthreads();
                    pa_load_tile<T>(x, B, t * tj, tj, E, s_tile, s_lab, p.labels, C, warp, lane);
                    __syncthreads();
                    cur = t;
                }
                if (have)
                    pa_sweep<KE, 0>(s_tile, E, min(tj, B - t * tj), t * tj, u, lane, c, s_lab, 0.f, 0.f, nullptr, nullptr,
                                    margin, beta, sp, sn, acc);
            }
            sp = warp_sum(sp);
            sn = warp_sum(sn);
            if (have && lane < PA_CLUSTER) {
                cluster.map_shared_rank(s_sp, lane)[c] = sp;
                cluster.map_shared_rank(s_sn, lane)[c] = sn;
            }
            if (p.grad_p != nullptr) {
                const float wpos = wpos0 / (1.0f + sp), wneg = wneg0 / (1.0f + sn);
                for (int t = 0; t < ntiles; ++t) {
                    if (cur != t) {
                        __syncthreads();
                        pa_load_tile<T>(x, B, t * tj, tj, E, s_tile, s_lab, p.labels, C, warp, lane);
                        __syncthreads();
                        cur = t;
                    }
                    if (have)
                        pa_sweep<KE, 1>(s_tile, E, min(tj, B - t * tj), t * tj, u, lane, c, s_lab, wpos, wneg, nullptr,
                                        nullptr, margin, beta, sp, sn, acc);
                }
                if (have) pa_finish<KE, float>(acc, u, rp, p.grad_p + (size_t)c * E, E, lane);
            }
        }
    }
    cluster.sync();                                          // S+ and S- of every class are in every CTA

    if (rank == 0) {
        float lp = 0.f, ln = 0.f;
        for (int c = tid; c < C; c += PA_THREADS) {
            lp += log1pf(s_sp[c]);
            ln += log1pf(s_sn[c]);
        }
        lp = warp_sum(lp);
        ln = warp_sum(ln);
        if (lane == 0) {
            s_red[warp] = lp;
            s_red[PA_WARPS + warp] = ln;
        }
        __syncthreads();
        if (tid == 0) {
            float a = 0.f, b = 0.f;
            for (int w = 0; w < PA_WARPS; ++w) {
                a += s_red[w];
                b += s_red[PA_WARPS + w];
            }
            p.loss[0] = (nv > 0 ? a / (float)nv : 0.f) + b / (float)C;
            if (p.n_valid != nullptr) p.n_valid[0] = nv;
        }
    }
    if (p.grad_x == nullptr) return;
    __syncthreads();
    for (int c = tid; c < C; c += PA_THREADS) {
        s_sp[c] = wpos0 / (1.0f + s_sp[c]);
        s_sn[c] = wneg0 / (1.0f + s_sn[c]);
    }
    cur = -1;                                                // the tile holds images; phase B streams proxies
    __syncthreads();

    // ---- phase B: images [b_begin, b_end), proxies streamed
    {
        const int Bs = (B + PA_CLUSTER - 1) / PA_CLUSTER;
        const int b_begin = rank * Bs, b_end = min(B, b_begin + Bs);
        const int ntiles = (C + tj - 1) / tj, rounds = (Bs + PA_WARPS - 1) / PA_WARPS;
        const T* x = reinterpret_cast<const T*>(p.x);
        T* gx = reinterpret_cast<T*>(p.grad_x);
        for (int round = 0; round < rounds; ++round) {
            const int b = b_begin + round * PA_WARPS + warp;
            const bool have = b < b_end;
            float rx = 0.f;
            int lab = -1;
            __syncwarp();
            if (have) {
                rx = pa_load_unit<T>(x + (size_t)b * E, u, E, lane);
                const long long t = p.labels[b];
                if (t >= 0 && t < C) lab = (int)t;
            }
            __syncwarp();
            float sp = 0.f, sn = 0.f, acc[KE];
#pragma unroll
            for (int k = 0; k < KE; ++k) acc[k] = 0.f;               // an image without a class keeps a zero gradient
            for (int t = 0; t < ntiles; ++t) {
                if (cur != t) {
                    __syncthreads();
                    pa_load_tile<float>(p.p, C, t * tj, tj, E, s_tile, s_lab, nullptr, C, warp, lane);
                    __syncthreads();
                    cur = t;
                }
                if (have && lab >= 0)
                    pa_sweep<KE, 2>(s_tile, E, min(tj, C - t * tj), t * tj, u, lane, lab, s_lab, 0.f, 0.f, s_sp, s_sn,
                                    margin, beta, sp, sn, acc);
            }
            if (have) pa_finish<KE, T>(acc, u, rx, gx + (size_t)b * E, E, lane);
        }
    }
}

// accumulators per lane: E <= 32 -> 1, <= 128 -> 4, <= 512 -> 16
template <class T>
__device__ __forceinline__ void pa_by_width(const PaParams& p) {
    if (p.E <= 32) pa_body<T, 1>(p);
    else if (p.E <= 128) pa_body<T, 4>(p);
    else pa_body<T, 16>(p);
}

// one plain kernel per embedding dtype (proxies, sums, loss and dP are fp32 in all three)
__global__ void __cluster_dims__(PA_CLUSTER, 1, 1) __launch_bounds__(PA_THREADS, 1)
proxy_anchor_f32_kernel(const PaParams p) { pa_by_width<float>(p); }
__global__ void __cluster_dims__(PA_CLUSTER, 1, 1) __launch_bounds__(PA_THREADS, 1)
proxy_anchor_bf16_kernel(const PaParams p) { pa_by_width<__nv_bfloat16>(p); }
__global__ void __cluster_dims__(PA_CLUSTER, 1, 1) __launch_bounds__(PA_THREADS, 1)
proxy_anchor_f16_kernel(const PaParams p) { pa_by_width<__half>(p); }

}  // namespace

extern "C" int mgp_proxy_anchor(const void* x, int x_dtype, const float* proxies, const int64_t* labels, int B, int C,
                                int E, float margin, float beta, float* loss, void* grad_x, float* grad_p,
                                int32_t* n_valid, void* stream) {
    if (x == nullptr || proxies == nullptr || labels == nullptr || loss == nullptr || B <= 0 || C <= 0 || E <= 0)
        return MGP_ERR_INVALID;
    if (x_dtype != MGP_X_F32 && x_dtype != MGP_X_BF16 && x_dtype != MGP_X_F16) return MGP_ERR_INVALID;
    if (!mgp_aligned16(x) || !mgp_aligned16(proxies) || !mgp_aligned16(grad_x) || !mgp_aligned16(grad_p))
        return MGP_ERR_INVALID;
    if (B > PA_MAX_B || C < 2 || C > PA_MAX_C || E > PA_MAX_E || (E & 3) != 0) return MGP_ERR_UNSUPPORTED;

    PaParams prm;
    prm.x = x; prm.p = proxies; prm.labels = labels; prm.loss = loss; prm.grad_x = grad_x; prm.grad_p = grad_p;
    prm.n_valid = n_valid; prm.B = B; prm.C = C; prm.E = E; prm.margin = margin; prm.beta = beta;
    const int want = ((B > C ? B : C) + 31) & ~31, fit = (PA_TILE_FLOATS / (E + 4)) & ~31;
    prm.tj = want < fit ? want : fit;
    const int C4 = (C + 3) & ~3;
    const size_t smem = sizeof(float) * ((size_t)prm.tj * (E + 4) + (size_t)PA_WARPS * E + 2 * (size_t)C4 + prm.tj +
                                         2 * PA_WARPS);
    void (*kernel)(const PaParams) = x_dtype == MGP_X_F32 ? proxy_anchor_f32_kernel
                                     : x_dtype == MGP_X_BF16 ? proxy_anchor_bf16_kernel : proxy_anchor_f16_kernel;
    MGP_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kernel<<<PA_CLUSTER, PA_THREADS, smem, (cudaStream_t)stream>>>(prm);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}
