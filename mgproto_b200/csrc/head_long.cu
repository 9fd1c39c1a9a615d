// a4-a7 on long feature maps (1024 < HW <= 4096; callable at any HW <= 4096): top-T mining over the patches of each
// image, wrong-class rule, block-diagonal pi mix and log, and its backward -- the same quantities as head.cu's
// head_select_kernel / head_top1_kernel / head_bwd_kernel, whose 10-bit patch keys and [HW]-sized shared-memory
// tiles stop at 1024 patches.  Shared memory per CTA does not grow with HW.
// ref: model.py:188-206 (global_max_pooling_gmm_topT: a torch.topk over h*w of any size), :214-222, :254.
#include "mgp_common.cuh"

#include "head_bwd.cuh"
#include "head_topt.cuh"

namespace {

constexpr int LSLICE = 1024;      // patches per register-resident slice (warp_topT<32, .>: 32 keys per lane)
constexpr int LMAX_HW = 4096;     // 12-bit patch index in the backward's entry key
constexpr int LMAX_K = 64;
constexpr unsigned FULL = 0xffffffffu;

// Merge a slice's top-T into a running top-T (one entry per lane, levels 0..T-1 in lanes 0..T-1, all T valid):
// a warp top-T over 64 positions, the running list at `lane`, the slice's (ns valid entries, patch indices already
// absolute) at 32 + lane.  Every running index is smaller than every slice index, so among equal values position
// order is patch order and the merge keeps "ties -> smaller index".  scr: 64 floats of this warp's shared memory.
__device__ __forceinline__ void long_merge(float* scr, float& rv, int& ri, float sv, int si, int ns, int T, int lane) {
    const float none = __uint_as_float(0xffffffffu);      // f2key() == 0: sorts below every real value
    scr[lane] = (lane < T) ? rv : none;
    scr[32 + lane] = (lane < ns) ? sv : none;
    __syncwarp();
    const float* rows[1] = {scr};
    float v[1];
    int pos[1];
    warp_topT<2, 1>(rows, 1, 64, T, lane, v, pos);
    const int from_run = __shfl_sync(FULL, ri, pos[0] & 31);
    const int from_slice = __shfl_sync(FULL, si, pos[0] & 31);
    __syncwarp();
    if (lane < T) {
        rv = v[0];
        ri = (pos[0] < 32) ? from_run : from_slice;
    }
}

// Top-T of one [HW] row in global memory (descending, ties -> smaller index): slices of LSLICE patches, each
// selected in registers and merged into the running list.  The first slice holds min(HW, LSLICE) >= T patches.
__device__ __forceinline__ void long_row_topT(const float* row, int HW, int T, int lane, float* scr, float& rv, int& ri) {
    for (int s0 = 0; s0 < HW; s0 += LSLICE) {
        const int n = min(LSLICE, HW - s0);
        const float* rows[1] = {row + s0};
        float v[1];
        int ix[1];
        warp_topT<32, 1>(rows, 1, n, T, lane, v, ix);
        if (s0 == 0) {
            rv = v[0];
            ri = ix[0];
        } else {
            long_merge(scr, rv, ri, v[0], ix[0] + s0, min(T, n), T, lane);
        }
    }
}

// Level 0 (max, ties -> smaller index) of one [HW] row: a streaming scan, any HW.
__device__ __forceinline__ void long_row_top1(const float* row, int HW, int lane, float& v, int& i) {
    unsigned best = 0u;
    int bi = 0x7fffffff;
#pragma unroll 4
    for (int j = lane; j < HW; j += 32) {
        const unsigned k = f2key(row[j]);
        if (k > best) { best = k; bi = j; }
    }
    const unsigned wb = __reduce_max_sync(FULL, best);
    i = __reduce_min_sync(FULL, (best == wb) ? bi : 0x7fffffff);
    v = key2f(wb);
}

// mgp_head_select_long: logp [B,P,HW] -> logits, vals, idx as head_select_kernel<R, NR, false>.  grid (C / CT, B),
// CT = 64 / K classes per CTA, 256 threads; a warp per row.  With labels wrong-class rows need level 0 only (its
// value and index fill all T levels, as in head_select_kernel; ref model.py:218-221).
__global__ void __launch_bounds__(256, 1)
head_select_long_kernel(const float* __restrict__ logp, const float* __restrict__ weight, const int64_t* __restrict__ gt,
                        float* __restrict__ logits, float* __restrict__ vals, int32_t* __restrict__ idx, int HW, int C,
                        int K, int T, int CT) {
    __shared__ float win[LMAX_K * 32];                      // [CT*K][T] exp(log p) of the winners
    __shared__ float scr[8][64];                            // per-warp merge buffer
    const int b = blockIdx.y;
    const int c0 = blockIdx.x * CT;
    const int nc = min(CT, C - c0);
    const int P = C * K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int npl = nc * K;
    const bool labelled = (gt != nullptr);
    const long long g = labelled ? (long long)gt[b] : -1;
    const int gl0 = (labelled && g >= c0 && g < c0 + nc) ? (int)(g - c0) * K : -1;
    for (int pl = warp; pl < npl; pl += 8) {
        const int p = c0 * K + pl;
        const float* row = logp + ((size_t)b * P + p) * HW;
        const bool all = !labelled || (gl0 >= 0 && pl >= gl0 && pl < gl0 + K);
        float v;
        int ix;
        if (all) long_row_topT(row, HW, T, lane, scr[warp], v, ix);
        else long_row_top1(row, HW, lane, v, ix);
        if (lane < T) {
            const float e = expf(v);                        // ref model.py:215
            win[pl * T + lane] = e;
            vals[((size_t)b * P + p) * T + lane] = e;
            idx[((size_t)b * P + p) * T + lane] = ix;
        }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < nc * T; e += blockDim.x) {
        const int cl = e / T, t = e - cl * T;
        const int c = c0 + cl;
        const bool fold = labelled && ((long long)c != g) && (t > 0);          // ref model.py:218-221
        const float* wrow = weight + (size_t)c * P + (size_t)c * K;            // class-diagonal block of last_layer.weight
        float s = 0.f;
        for (int k = 0; k < K; ++k) s = fmaf(__ldg(wrow + k), win[(cl * K + k) * T + (fold ? 0 : t)], s);
        logits[((size_t)b * C + c) * T + t] = logf(s);                         // ref model.py:222, :254
    }
}

// Shared-memory layout of head_top1_long_kernel, in floats: [P] exp(level 0), [P] pi, [K][T] winners, [K][T] running
// log p, [K][T] running indices, [K][S+1] the own class's log p over a slice of S patches, then (16-byte aligned)
// [K][D] mu, [K][D] 1/sigma, [K] sum log sigma, [K] |mu|^2.
struct Top1LongLayout {
    int S;            // patches per slice (a multiple of 32, 32..1024); 0: the shape does not fit
    size_t floats;
};
__host__ __device__ inline size_t top1_long_head(int P, int K, int T, int S) {
    return ((size_t)2 * P + (size_t)3 * K * T + (size_t)K * (S + 1) + 3) & ~(size_t)3;
}
inline Top1LongLayout top1_long_layout(int P, int K, int D, int T, size_t budget_floats) {
    const size_t fixed = top1_long_head(P, K, T, 0) + (size_t)2 * K * D + 2 * K;
    Top1LongLayout l{0, 0};
    if (fixed + (size_t)K * 33 > budget_floats) return l;
    size_t s = (budget_floats - fixed) / K - 1;
    s = s > (size_t)LSLICE ? (size_t)LSLICE : (s & ~(size_t)31);
    if (s < 32) return l;
    l.S = (int)s;
    l.floats = top1_long_head(P, K, T, l.S) + (size_t)2 * K * D + 2 * K;
    return l;
}

// mgp_head_select_top1_long: the labelled step without log p (head_top1_kernel on slices).  grid B, 256 threads.
//   1. level 0 of every prototype from the packed (max, arg max) in `best`
//   2. the image's own class: exact fp32 log p of its K prototypes over S patches at a time (the evaluation of
//      head_top1_kernel, operation for operation), each slice's top-T merged into the running top-T of its row
//   3. logits (wrong classes: every level = level 0, ref model.py:218-221)
// gt[b] outside [0, C) skips step 2: with gt = -1 everywhere this is the level-0 head.
__global__ void __launch_bounds__(256, 1)
head_top1_long_kernel(const unsigned long long* __restrict__ best, const float* __restrict__ xhat,
                      const float* __restrict__ mu, const float* __restrict__ sigma, const float* __restrict__ weight,
                      const int64_t* __restrict__ gt, float* __restrict__ logits, float* __restrict__ vals,
                      int32_t* __restrict__ idx, int HW, int C, int K, int D, int T, int S) {
    constexpr int NTHR = 256;
    extern __shared__ __align__(16) float sm[];
    __shared__ float scr[8][64];
    const int P = C * K;
    const int Sp = S + 1;
    float* win0 = sm;                    // [P]      exp(level-0 log p)
    float* s_wd = win0 + P;              // [P]      pi_p = last_layer.weight[c, c*K + k]
    float* winT = s_wd + P;              // [K][T]   own class, all levels
    float* runv = winT + K * T;          // [K][T]   running top-T log p of the own class's rows
    int* runi = reinterpret_cast<int*>(runv + K * T);   // [K][T] their patches
    float* lp = runv + 2 * K * T;        // [K][Sp]  own-class log p over the current slice
    float* s_mu = sm + top1_long_head(P, K, T, S);      // [K][D], 16-byte aligned
    float* s_ri = s_mu + K * D;          // [K][D]   1/sigma
    float* s_ls = s_ri + K * D;          // [K]      sum_d log sigma
    float* s_mm = s_ls + K;              // [K]      |mu_k|^2
    const int b = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long g = gt[b];
    const bool gok = (g >= 0 && g < C);

    for (int p0 = threadIdx.x; p0 < P; p0 += NTHR * 4) {
        unsigned long long pk[4];
        float wd[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int p = p0 + NTHR * u;
            pk[u] = (p < P) ? best[(size_t)b * P + p] : 0ull;
            wd[u] = (p < P) ? __ldg(weight + (size_t)(p / K) * P + p) : 0.f;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int p = p0 + NTHR * u;
            if (p < P) {
                const float e = expf(key2f((unsigned)(pk[u] >> 32)));            // ref model.py:215
                win0[p] = e;
                s_wd[p] = wd[u];
                vals[((size_t)b * P + p) * T] = e;
                idx[((size_t)b * P + p) * T] = (int)(0xffffffffu - (unsigned)(pk[u] & 0xffffffffull));
            }
        }
    }
    if (gok) {
        const float* mug = mu + (size_t)g * K * D;
        const float* sgg = sigma + (size_t)g * K * D;
        for (int i = threadIdx.x; i < K * D; i += NTHR) {
            s_mu[i] = mug[i];
            s_ri[i] = 1.0f / sgg[i];
        }
        for (int k = warp; k < K; k += NTHR / 32) {
            float ls = 0.f;
            for (int d = lane; d < D; d += 32) ls += logf(sgg[k * D + d]) + 0.5f * MGP_LOG_2PI;
            ls = warp_sum(ls);
            if (lane == 0) s_ls[k] = ls;
        }
        __syncthreads();
        // log p[n,k] = -D/2 log 2pi - sum log sigma - 1/2 sum ((x-mu)/sigma)^2   (ref model.py:256-275, exact form);
        // isotropic sigma: w (|x|^2 - 2 x.mu + |mu|^2), as head_top1_kernel
        bool same = true;
        for (int i = threadIdx.x; i < K * D; i += NTHR) same = same && (s_ri[i] == s_ri[(i / D) * D]);
        const bool iso = __syncthreads_and(same ? 1 : 0) != 0;
        for (int k = warp; k < K; k += NTHR / 32) {
            float mm = 0.f;
            for (int d = lane; d < D; d += 32) mm = fmaf(s_mu[k * D + d], s_mu[k * D + d], mm);
            mm = warp_sum(mm);
            if (lane == 0) s_mm[k] = mm;
        }
        __syncthreads();
        const int KHh = (K + 1) / 2;
        for (int s0 = 0; s0 < HW; s0 += S) {
            const int ns = min(S, HW - s0);
            // thread = (patch of the slice, half of the prototypes)
            for (int it = threadIdx.x; it < 2 * ns; it += NTHR) {
                const int j = it >> 1, kb = (it & 1) * KHh, ke = min(K, kb + KHh);
                const float4* xr = reinterpret_cast<const float4*>(xhat + ((size_t)b * HW + s0 + j) * D);
                for (int k0 = kb; k0 < ke; k0 += 5) {
                    float q[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
                    float2 q2[5], xx2 = make_float2(0.f, 0.f);
#pragma unroll
                    for (int i = 0; i < 5; ++i) q2[i] = make_float2(0.f, 0.f);
                    for (int d0 = 0; d0 < D / 4; d0 += 8) {
                        float4 xv[8];
#pragma unroll
                        for (int u = 0; u < 8; ++u) xv[u] = (d0 + u < D / 4) ? __ldg(xr + d0 + u) : make_float4(0.f, 0.f, 0.f, 0.f);
                        if (iso) {
#pragma unroll
                            for (int u = 0; u < 8; ++u) {
                                if (d0 + u >= D / 4) break;
                                const float2 x01 = make_float2(xv[u].x, xv[u].y), x23 = make_float2(xv[u].z, xv[u].w);
                                xx2 = ffma2(x01, x01, xx2);
                                xx2 = ffma2(x23, x23, xx2);
#pragma unroll
                                for (int i = 0; i < 5; ++i) {
                                    const int k = min(k0 + i, K - 1);
                                    const float4 m = *reinterpret_cast<const float4*>(s_mu + k * D + 4 * (d0 + u));
                                    q2[i] = ffma2(x01, make_float2(m.x, m.y), q2[i]);
                                    q2[i] = ffma2(x23, make_float2(m.z, m.w), q2[i]);
                                }
                            }
                        } else {
#pragma unroll
                            for (int u = 0; u < 8; ++u) {
                                if (d0 + u >= D / 4) break;
#pragma unroll
                                for (int i = 0; i < 5; ++i) {
                                    const int k = min(k0 + i, K - 1);
                                    const float4 m = *reinterpret_cast<const float4*>(s_mu + k * D + 4 * (d0 + u));
                                    const float4 r = *reinterpret_cast<const float4*>(s_ri + k * D + 4 * (d0 + u));
                                    float t;
                                    t = (xv[u].x - m.x) * r.x; q[i] = fmaf(t, t, q[i]);
                                    t = (xv[u].y - m.y) * r.y; q[i] = fmaf(t, t, q[i]);
                                    t = (xv[u].z - m.z) * r.z; q[i] = fmaf(t, t, q[i]);
                                    t = (xv[u].w - m.w) * r.w; q[i] = fmaf(t, t, q[i]);
                                }
                            }
                        }
                    }
                    if (iso) {
                        const float xx = xx2.x + xx2.y;
#pragma unroll
                        for (int i = 0; i < 5; ++i) {
                            const int k = min(k0 + i, K - 1);
                            const float ri = s_ri[k * D];
                            q[i] = ri * ri * (xx - 2.0f * (q2[i].x + q2[i].y) + s_mm[k]);
                        }
                    }
#pragma unroll
                    for (int i = 0; i < 5; ++i)
                        if (k0 + i < ke) lp[(k0 + i) * Sp + j] = -s_ls[k0 + i] - 0.5f * q[i];
                }
            }
            __syncthreads();
            for (int k = warp; k < K; k += NTHR / 32) {
                const float* rows[1] = {lp + k * Sp};
                float v[1];
                int ix[1];
                warp_topT<32, 1>(rows, 1, ns, T, lane, v, ix);
                float rv = v[0];
                int ri = ix[0];
                if (s0 > 0) {
                    rv = (lane < T) ? runv[k * T + lane] : 0.f;
                    ri = (lane < T) ? runi[k * T + lane] : 0;
                    long_merge(scr[warp], rv, ri, v[0], ix[0] + s0, min(T, ns), T, lane);
                }
                if (lane < T) {
                    runv[k * T + lane] = rv;
                    runi[k * T + lane] = ri;
                }
            }
            __syncthreads();
        }
        for (int k = warp; k < K; k += NTHR / 32)
            if (lane < T) {
                const int p = (int)g * K + k;
                const float e = expf(runv[k * T + lane]);                        // ref model.py:215
                winT[k * T + lane] = e;
                vals[((size_t)b * P + p) * T + lane] = e;
                idx[((size_t)b * P + p) * T + lane] = runi[k * T + lane];
            }
    }
    __syncthreads();
    for (int e = threadIdx.x; e < C * T; e += NTHR) {
        const int c = e / T, t = e - c * T;
        const bool own = gok && (long long)c == g;
        float s = 0.f;
        for (int k = 0; k < K; ++k) s = fmaf(s_wd[c * K + k], own ? winT[k * T + t] : win0[c * K + k], s);
        logits[((size_t)b * C + c) * T + t] = logf(s);                         // ref model.py:222, :254
    }
}

// Long-map backward: head_bwd_body with the 12-bit patch key and the two-pass row sort; one plain kernel per lane
// width.  (256, 3) rather than head_bwd_kernel<2>'s (256, 4): 80 registers, no spills.
__global__ void __launch_bounds__(256, 3) head_bwd_long_v2_kernel(MGP_HEAD_BWD_PARAMS) {
    head_bwd_body<2, true>(MGP_HEAD_BWD_ARGS);
}
__global__ void __launch_bounds__(256, 2) head_bwd_long_v4_kernel(MGP_HEAD_BWD_PARAMS) {
    head_bwd_body<4, true>(MGP_HEAD_BWD_ARGS);
}
#undef MGP_HEAD_BWD_PARAMS
#undef MGP_HEAD_BWD_ARGS

constexpr size_t SMEM_BUDGET = 200 * 1024;

}  // namespace

extern "C" int mgp_head_select_long(const float* logp_bphw, const float* weight_cp, const int64_t* gt, float* logits,
                                    float* vals, int32_t* idx, int B, int HW, int C, int K, int T, void* stream) {
    if (!logp_bphw || !weight_cp || !logits || !vals || !idx) return MGP_ERR_INVALID;
    if (B <= 0 || HW <= 0 || C <= 0 || K <= 0 || T <= 0) return MGP_ERR_INVALID;
    if (T > 32 || T > HW || HW > LMAX_HW || K > LMAX_K) return MGP_ERR_UNSUPPORTED;
    int CT = LMAX_K / K;
    if (CT > C) CT = C;
    dim3 grid((C + CT - 1) / CT, B);
    head_select_long_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(logp_bphw, weight_cp, gt, logits, vals, idx, HW, C,
                                                                    K, T, CT);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" int mgp_head_select_top1_long(const uint64_t* best, const float* xhat_nd, const float* mu, const float* sigma,
                                         const float* weight_cp, const int64_t* gt, float* logits, float* vals,
                                         int32_t* idx, int B, int HW, int C, int K, int D, int T, void* stream) {
    if (!best || !xhat_nd || !mu || !sigma || !weight_cp || !gt || !logits || !vals || !idx) return MGP_ERR_INVALID;
    if (B <= 0 || HW <= 0 || C <= 0 || K <= 0 || D <= 0 || T <= 0 || (D & 3)) return MGP_ERR_INVALID;
    if (T > 32 || T > HW || HW > LMAX_HW || K > LMAX_K) return MGP_ERR_UNSUPPORTED;
    const Top1LongLayout l = top1_long_layout(C * K, K, D, T, SMEM_BUDGET / sizeof(float));
    if (l.S == 0) return MGP_ERR_UNSUPPORTED;
    const size_t smem = l.floats * sizeof(float);
    MGP_CUDA(cudaFuncSetAttribute(head_top1_long_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    head_top1_long_kernel<<<B, 256, smem, (cudaStream_t)stream>>>(reinterpret_cast<const unsigned long long*>(best),
                                                                  xhat_nd, mu, sigma, weight_cp, gt, logits, vals, idx,
                                                                  HW, C, K, D, T, l.S);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" size_t mgp_head_bwd_long_ws_bytes(int B, int HW, int P, int D) {
    return ((size_t)2 * P * D + (size_t)B * HW * D + (size_t)P + 64) * sizeof(float);
}

extern "C" int mgp_head_bwd_long_x(const float* grad_logits, const float* logits, const float* vals, const int32_t* idx,
                                   const float* weight_cp, const int64_t* gt, const float* xhat_nd, const float* inv_norm,
                                   const float* mu, const float* sigma, void* ws, size_t ws_bytes, void* g_x, int x_fmt,
                                   int B, int HW, int C, int K, int D, int T, void* stream) {
    if (!grad_logits || !logits || !vals || !idx || !weight_cp || !xhat_nd || !inv_norm || !mu || !sigma || !ws ||
        !g_x || !mgp_x_fmt_valid(x_fmt))
        return MGP_ERR_INVALID;
    if (B <= 0 || HW <= 0 || C <= 0 || K <= 0 || D <= 0 || T <= 0) return MGP_ERR_INVALID;
    // entry key p*4096 + n in 32 bits
    if (T > 32 || T > HW || HW > LMAX_HW || (size_t)C * K >= (1u << 20)) return MGP_ERR_UNSUPPORTED;
    const int P = C * K;
    if (ws_bytes < mgp_head_bwd_long_ws_bytes(B, HW, P, D)) return MGP_ERR_WORKSPACE;
    const size_t smem = (size_t)LCAP * 16 + (size_t)(8 * 64 + C + T) * 4;
    if (smem > SMEM_BUDGET) return MGP_ERR_UNSUPPORTED;
    cudaStream_t st = (cudaStream_t)stream;
    float* w = reinterpret_cast<float*>(ws);
    float* wm = w + (size_t)P * D;
    float* g_xhat = wm + (size_t)P * D;
    float* wsc = g_xhat + (size_t)B * HW * D;
    int* noniso = reinterpret_cast<int*>(wsc + P);
    const int rc = head_bwd_proto_weights(mu, sigma, w, wm, wsc, noniso, P, D, st);
    if (rc != MGP_OK) return rc;
    // dims per CTA: 32 lanes x 4 when D is a multiple of 128 (one CTA per image at D = 128), else x 2
    const int DC = (D % 128) == 0 ? 128 : 64;
    MGP_CUDA(cudaFuncSetAttribute(head_bwd_long_v2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MGP_CUDA(cudaFuncSetAttribute(head_bwd_long_v4_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MGP_CUDA(cudaMemsetAsync(g_xhat, 0, (size_t)B * HW * D * sizeof(float), st));   // rows without mined patches stay zero
    dim3 grid(B, (D + DC - 1) / DC);
    if (DC == 128)
        head_bwd_long_v4_kernel<<<grid, 256, smem, st>>>(grad_logits, logits, vals, idx, weight_cp, gt, xhat_nd, w, wm, wsc,
                                                         noniso, g_xhat, HW, C, K, D, T);
    else
        head_bwd_long_v2_kernel<<<grid, 256, smem, st>>>(grad_logits, logits, vals, idx, weight_cp, gt, xhat_nd, w, wm, wsc,
                                                         noniso, g_xhat, HW, C, K, D, T);
    MGP_CHECK_LAUNCH();
    return mgp_normalize_bwd_x(g_xhat, xhat_nd, inv_norm, g_x, x_fmt, B, D, HW, stream);
}
