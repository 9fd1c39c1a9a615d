// a4-a7: top-T prototype mining over the patches of each image, wrong-class rule, block-diagonal
// pi mix and log (head_select_kernel: from a materialised log p; head_top1_kernel: labelled step, from the
// tensor-core epilogue's packed max/arg-max); its backward; the fused loss; the push-projection argmin (f1).
// ref: model.py:188-206, :214-222, :254, :54-74; push.py:125-158.
#include "mgp_common.cuh"
#include <type_traits>

#include "head_topt.cuh"

namespace {

// FROM_NP = false: logp is [B,P,HW] (one contiguous row per (image, prototype)).
// FROM_NP = true : logp is [N,P] (the compute_log_prob / tensor-core layout): the CTA first stages the
//                  [HW x CT*K] block of its image and classes in shared memory (each patch row is a contiguous
//                  CT*K*4-byte read), then selects along the columns (pitch CT*K+1: conflict-free).
template <int R, int NR, bool FROM_NP>
__global__ void __launch_bounds__(256, (R <= 8) ? 3 : 1)
head_select_kernel(const float* __restrict__ logp, const float* __restrict__ weight, const int64_t* __restrict__ gt,
                   float* __restrict__ logits, float* __restrict__ vals, int32_t* __restrict__ idx, int HW, int C,
                   int K, int T, int CT, int is_prob) {
    // is_prob: the input rows already hold p = exp(log p) (mgp_topt_pool: the reference's
    // global_max_pooling_gmm_topT takes probabilities); the order is the same, the values are passed through
    extern __shared__ float win[];  // [CT*K][T] exp(log p) of the winners  (+ [HW][CT*K+1] tile when FROM_NP)
    const int b = blockIdx.y;
    const int c0 = blockIdx.x * CT;
    const int nc = min(CT, C - c0);
    const int P = C * K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int npl = nc * K;
    const int pitch = CT * K + 1;
    float* tile = win + CT * K * T;
    if (FROM_NP) {
        const float* src = logp + (size_t)b * HW * P + (size_t)c0 * K;
        // asynchronous 4-byte copies (LDGSTS): every element of the block is in flight at once, no register
        // staging; rows are only 4-byte aligned in general (P need not be a multiple of 4)
        for (int hw = warp; hw < HW; hw += 8)
            for (int j = lane; j < npl; j += 32) {
                const uint32_t dst = (uint32_t)__cvta_generic_to_shared(tile + hw * pitch + j);
                asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(dst), "l"(src + (size_t)hw * P + j) : "memory");
            }
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();
    }
    const long long g = (gt != nullptr) ? (long long)gt[b] : -1;
    const bool labelled = (gt != nullptr);
    const int rs = FROM_NP ? pitch : 1;
    // rows [gl0, gl0 + K) of this CTA belong to the image's own class (-1: none here / no labels)
    const int gl0 = (labelled && g >= c0 && g < c0 + nc) ? (int)(g - c0) * K : -1;
    if (labelled) {
        for (int pl0 = warp * NR; pl0 < npl; pl0 += 8 * NR) {
            const float* rows[NR];
#pragma unroll
            for (int i = 0; i < NR; ++i) {
                const int pl = min(pl0 + i, npl - 1);
                rows[i] = FROM_NP ? (tile + pl) : (logp + ((size_t)b * P + c0 * K + pl) * HW);
            }
            float v[NR];
            int ix[NR];
            warp_top1<R, NR>(rows, rs, HW, lane, v, ix);
#pragma unroll
            for (int i = 0; i < NR; ++i) {
                const int pl = pl0 + i;
                const bool own = gl0 >= 0 && pl >= gl0 && pl < gl0 + K;     // done with all levels below
                if (pl < npl && !own && lane < T) {
                    const int p = c0 * K + pl;
                    const float e = is_prob ? v[i] : expf(v[i]);  // ref model.py:215; levels >= 1 alias level 0 (ref :218-221)
                    if (lane == 0) win[pl * T] = e;
                    vals[((size_t)b * P + p) * T + lane] = e;
                    idx[((size_t)b * P + p) * T + lane] = ix[i];
                }
            }
        }
    }
    const int fb = labelled ? gl0 : 0, fe = labelled ? (gl0 >= 0 ? gl0 + K : -1) : npl;   // rows needing all T levels
    for (int pl0 = fb + warp * NR; pl0 < fe; pl0 += 8 * NR) {
        const float* rows[NR];
#pragma unroll
        for (int i = 0; i < NR; ++i) {
            const int pl = min(pl0 + i, fe - 1);               // surplus slots recompute the last row, not stored
            rows[i] = FROM_NP ? (tile + pl) : (logp + ((size_t)b * P + c0 * K + pl) * HW);
        }
        float v[NR];
        int ix[NR];
        if (R <= 8) warp_topT_sorted<(R <= 8 ? R : 1), NR>(rows, rs, HW, T, lane, v, ix);
        else warp_topT<R, NR>(rows, rs, HW, T, lane, v, ix);
#pragma unroll
        for (int i = 0; i < NR; ++i) {
            const int pl = pl0 + i;
            if (pl < fe && lane < T) {
                const int p = c0 * K + pl;
                const float e = is_prob ? v[i] : expf(v[i]);  // ref model.py:215
                win[pl * T + lane] = e;
                vals[((size_t)b * P + p) * T + lane] = e;
                idx[((size_t)b * P + p) * T + lane] = ix[i];
            }
        }
    }
    __syncthreads();
    if (weight == nullptr) return;                                             // pooling only (mgp_topt_pool)
    for (int e = threadIdx.x; e < nc * T; e += blockDim.x) {
        const int cl = e / T, t = e - cl * T;
        const int c = c0 + cl;
        const bool fold = (gt != nullptr) && ((long long)c != g) && (t > 0);  // ref model.py:218-221
        const float* wrow = weight + (size_t)c * P + (size_t)c * K;            // class-diagonal block of last_layer.weight
        float s = 0.f;
        for (int k = 0; k < K; ++k) s = fmaf(__ldg(wrow + k), win[(cl * K + k) * T + (fold ? 0 : t)], s);
        logits[((size_t)b * C + c) * T + t] = logf(s);                         // ref model.py:222, :254
    }
}

// Labelled head without the log-likelihood matrix (mgp_head_select_top1).  grid B, block NTHR (256).
//   1. level 0 of every prototype from the packed (max, arg max) the tensor-core epilogue left in `best`
//   2. the image's own class: exact fp32 log p of its K prototypes over the HW patches (thread per patch,
//      prototype rows broadcast from shared memory), then the usual warp top-T on those K rows
//   3. logits (wrong classes: every level = level 0, ref model.py:218-221)
template <int R, int NR, int NTHR>
__global__ void __launch_bounds__(NTHR)
head_top1_kernel(const unsigned long long* __restrict__ best, const float* __restrict__ xhat,
                 const float* __restrict__ mu, const float* __restrict__ sigma, const float* __restrict__ weight,
                 const int64_t* __restrict__ gt, float* __restrict__ logits, float* __restrict__ vals,
                 int32_t* __restrict__ idx, int HW, int C, int K, int D, int T) {
    extern __shared__ __align__(16) float sm[];
    const int P = C * K;
    const int HWp = HW + 1;
    float* win0 = sm;                    // [P]      exp(level-0 log p)
    float* winT = win0 + P;              // [K][T]   own class, all levels
    float* lp = winT + K * T;            // [K][HWp] own-class log p rows
    float* s_mu = sm + ((P + K * T + K * HWp + 3) & ~3);   // [K][D], 16-byte aligned
    float* s_ri = s_mu + K * D;          // [K][D]   1/sigma
    float* s_ls = s_ri + K * D;          // [K]      sum_d log sigma
    float* s_mm = s_ls + K;              // [K]      |mu_k|^2
    float* s_wd = s_mm + K;              // [P]      pi_p = last_layer.weight[c, c*K + k]
    const int b = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const long long g = gt[b];
    const bool gok = (g >= 0 && g < C);

    // (all loads of a thread are issued before their first use: the kernel is a chain of L2 latencies otherwise)
    for (int p0 = threadIdx.x; p0 < P; p0 += NTHR * 4) {
        unsigned long long pk[4];
        float wd[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int p = p0 + NTHR * u;
            pk[u] = (p < P) ? best[(size_t)b * P + p] : 0ull;
            wd[u] = (p < P) ? __ldg(weight + (size_t)(p / K) * P + p) : 0.f;     // class-diagonal block of last_layer.weight
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
            for (int d = lane; d < D; d += 32) ls += logf(sgg[k * D + d]) + 0.5f * MGP_LOG_2PI;   // per-dim terms
            ls = warp_sum(ls);
            if (lane == 0) s_ls[k] = ls;
        }
        __syncthreads();
        // log p[n,k] = -D/2 log 2pi - sum log sigma - 1/2 sum ((x-mu)/sigma)^2   (ref model.py:256-275, exact form)
        // sigma constant over d inside each of the K prototypes (every state the shipped loop reaches)?  Then
        // sum ((x-mu)/sigma)^2 = w (|x|^2 - 2 x.mu + |mu|^2): one FMA per element instead of three operations
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
        // thread = (patch n, half of the prototypes): eight 16-byte loads of the patch row are in flight at a time
        // (the row is read once; prototype rows are shared-memory broadcasts)
        const int KHh = (K + 1) / 2;
        for (int it = threadIdx.x; it < 2 * HW; it += NTHR) {
            const int n = it >> 1, kb = (it & 1) * KHh, ke = min(K, kb + KHh);
            const float4* xr = reinterpret_cast<const float4*>(xhat + ((size_t)b * HW + n) * D);
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
                    if (k0 + i < ke) lp[(k0 + i) * HWp + n] = -s_ls[k0 + i] - 0.5f * q[i];
            }
        }
        __syncthreads();
        for (int k0 = warp * NR; k0 < K; k0 += (NTHR / 32) * NR) {
            const float* rows[NR];
#pragma unroll
            for (int i = 0; i < NR; ++i) rows[i] = lp + min(k0 + i, K - 1) * HWp;
            float v[NR];
            int ix[NR];
            if (R <= 8) warp_topT_sorted<(R <= 8 ? R : 1), NR>(rows, 1, HW, T, lane, v, ix);
            else warp_topT<R, NR>(rows, 1, HW, T, lane, v, ix);
#pragma unroll
            for (int i = 0; i < NR; ++i) {
                const int k = k0 + i;
                if (k < K && lane < T) {
                    const int p = (int)g * K + k;
                    const float e = expf(v[i]);
                    winT[k * T + lane] = e;
                    vals[((size_t)b * P + p) * T + lane] = e;
                    idx[((size_t)b * P + p) * T + lane] = ix[i];
                }
            }
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

// ------------------------------------------------------------------------------------------
// Backward: for image b accumulate  G[n,:] = sum_{(p,t)->n} a_bpt * (w_p*mu_p - w_p*xhat_n)
//   a_bpt = gl[b,c,t] * pi_p * v[b,p,t] / exp(logits[b,c,t])      (wrong-class levels fold onto t = 0)
// One CTA per (image, D-chunk); see head_bwd_kernel below for the schedule (compaction, stable sort by patch row,
// balanced walk, direct row writes) -- atomics-free and deterministic.
__global__ void proto_weight_kernel(const float* __restrict__ mu, const float* __restrict__ sigma,
                                    float* __restrict__ w, float* __restrict__ wm, float* __restrict__ wsc,
                                    int* __restrict__ noniso, size_t n, int D) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) {
        const float s = sigma[i];
        const float ww = 1.0f / (s * s);
        w[i] = ww;
        wm[i] = ww * mu[i];
        const size_t p = i / D;
        if (i == p * D) wsc[p] = ww;
        if (s != sigma[p * D]) atomicOr(noniso, 1);          // sigma varies over d inside a prototype
    }
}

}  // namespace

#include "head_bwd.cuh"

namespace {

template <int VEC>
__global__ void __launch_bounds__(256, VEC == 4 ? 2 : 4) head_bwd_kernel(MGP_HEAD_BWD_PARAMS) {
    head_bwd_body<VEC, false>(MGP_HEAD_BWD_ARGS);
}

#undef MGP_HEAD_BWD_PARAMS
#undef MGP_HEAD_BWD_ARGS

// a17 helper: the training loss on the head's output (ref train_and_test.py:37-41, :55)
//   loss = CE(out[:,:,0], gt) + mine_coef * mean_{t>=1} CE(out[:,:,t], gt),   CE = mean over the batch
// One CTA per image computes, for every level t, logsumexp_c out[b,c,t]; writes the image's loss share and
// d loss / d out[b,:,:] (softmax - onehot, weighted) in the same pass -- one launch instead of ~25 ATen ones.
__global__ void __launch_bounds__(256)
mine_ce_kernel(const float* __restrict__ out, const int64_t* __restrict__ gt, float* __restrict__ loss_b,
               float* __restrict__ grad, int B, int C, int T, float mine_coef) {
    extern __shared__ float sm[];
    float* lse = sm;            // [T]
    const int b = blockIdx.x;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const float* ob = out + (size_t)b * C * T;
    for (int t = warp; t < T; t += 8) {
        float m = -INFINITY;
        for (int c = lane; c < C; c += 32) m = fmaxf(m, ob[(size_t)c * T + t]);
        m = warp_max(m);
        float se = 0.f;
        for (int c = lane; c < C; c += 32) se += expf(ob[(size_t)c * T + t] - m);
        se = warp_sum(se);
        if (lane == 0) lse[t] = m + logf(se);
    }
    __syncthreads();
    const long long g = gt[b];
    const float wt0 = 1.0f / (float)B, wtm = (T > 1) ? mine_coef / ((float)(T - 1) * (float)B) : 0.f;
    if (threadIdx.x == 0) {
        float l = 0.f;
        for (int t = 0; t < T; ++t) l += (t == 0 ? wt0 : wtm) * (lse[t] - ob[(size_t)g * T + t]);
        loss_b[b] = l;
    }
    float* gb = grad + (size_t)b * C * T;
    for (int i = threadIdx.x; i < C * T; i += 256) {
        const int c = i / T, t = i - c * T;
        const float wv = (t == 0) ? wt0 : wtm;
        gb[i] = wv * (expf(ob[i] - lse[t]) - (((long long)c == g) ? 1.0f : 0.0f));
    }
}

// f1: per (image, prototype of the image's class): argmax_hw log p and -exp(log p) there.
__global__ void push_argmin_kernel(const float* __restrict__ logp, const int64_t* __restrict__ labels,
                                   int32_t* __restrict__ arg, float* __restrict__ val, int HW, int C, int K, int B) {
    const int wg = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (wg >= B * K) return;
    const int b = wg / K, k = wg - b * K;
    const long long c = labels[b];
    if (c < 0 || c >= C) {
        if (lane == 0) { arg[wg] = -1; val[wg] = 0.f; }
        return;
    }
    const float* row = logp + ((size_t)b * C * K + (size_t)c * K + k) * HW;
    unsigned best = 0;
    int bi = 0x7fffffff;
    for (int i = lane; i < HW; i += 32) {
        unsigned kk = f2key(row[i]);
        if (kk > best) { best = kk; bi = i; }
    }
    const unsigned wb = __reduce_max_sync(0xffffffffu, best);
    const int wi = __reduce_min_sync(0xffffffffu, (best == wb) ? bi : 0x7fffffff);
    if (lane == 0) {
        arg[wg] = wi;
        val[wg] = -expf(key2f(wb));
    }
}

// f1 without the log p matrix: the same (arg, val) from the packed per-(image, prototype) max / arg-max that the
// tensor-core epilogue leaves in `best` (MGP_OUT_TOP1_BP; ties already resolved towards the first patch).
__global__ void push_from_top1_kernel(const unsigned long long* __restrict__ best, const int64_t* __restrict__ labels,
                                      int32_t* __restrict__ arg, float* __restrict__ val, int B, int C, int K) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= B * K) return;
    const int b = i / K, k = i - b * K;
    const long long c = labels[b];
    if (c < 0 || c >= C) { arg[i] = -1; val[i] = 0.f; return; }
    const unsigned long long pk = best[(size_t)b * C * K + (size_t)c * K + k];
    arg[i] = (int)(0xffffffffu - (unsigned)(pk & 0xffffffffull));
    val[i] = -expf(key2f((unsigned)(pk >> 32)));
}

}  // namespace

static int head_select_launch(const float* logp, int from_np, const float* weight_cp, const int64_t* gt, float* logits,
                              float* vals, int32_t* idx, int B, int HW, int C, int K, int T, void* stream,
                              int is_prob = 0) {
    if (!logp || !vals || !idx || (!is_prob && (!weight_cp || !logits))) return MGP_ERR_INVALID;
    if (B <= 0 || HW <= 0 || C <= 0 || K <= 0 || T <= 0) return MGP_ERR_INVALID;
    if (T > 32 || T > HW || HW > 1024) return MGP_ERR_UNSUPPORTED;
    int CT = 64 / K;
    if (CT < 1) CT = 1;
    if (CT > C) CT = C;
    size_t smem = (size_t)CT * K * T * sizeof(float);
    if (from_np) smem += (size_t)HW * (CT * K + 1) * sizeof(float);
    if (smem > 200 * 1024) return MGP_ERR_UNSUPPORTED;
    dim3 grid((C + CT - 1) / CT, B);
    cudaStream_t st = (cudaStream_t)stream;
    const int R = (HW + 31) / 32;
#define MGP_LAUNCH_SEL2(RR, NRR, NP)                                                                                 \
    do {                                                                                                             \
        MGP_CUDA(cudaFuncSetAttribute(head_select_kernel<RR, NRR, NP>, cudaFuncAttributeMaxDynamicSharedMemorySize,  \
                                      (int)smem));                                                                   \
        MGP_CUDA(cudaFuncSetAttribute(head_select_kernel<RR, NRR, NP>,                                               \
                                      cudaFuncAttributePreferredSharedMemoryCarveout, NP ? 100 : 25));               \
        head_select_kernel<RR, NRR, NP><<<grid, 256, smem, st>>>(logp, weight_cp, gt, logits, vals, idx, HW, C, K,   \
                                                                 T, CT, is_prob);                                    \
    } while (0)
#define MGP_LAUNCH_SEL(RR, NRR)                                                                                      \
    do {                                                                                                             \
        if (from_np) MGP_LAUNCH_SEL2(RR, NRR, true);                                                                 \
        else MGP_LAUNCH_SEL2(RR, NRR, false);                                                                        \
    } while (0)
    if (R <= 2) MGP_LAUNCH_SEL(2, 4);
    else if (R <= 4) MGP_LAUNCH_SEL(4, 4);
    else if (R <= 7) MGP_LAUNCH_SEL(7, 4);
    else if (R <= 13) MGP_LAUNCH_SEL(13, 2);
    else if (R <= 25) MGP_LAUNCH_SEL(25, 1);
    else MGP_LAUNCH_SEL(32, 1);
#undef MGP_LAUNCH_SEL
#undef MGP_LAUNCH_SEL2
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" int mgp_head_select(const float* logp_bphw, const float* weight_cp, const int64_t* gt, float* logits,
                               float* vals, int32_t* idx, int B, int HW, int C, int K, int T, void* stream) {
    return head_select_launch(logp_bphw, 0, weight_cp, gt, logits, vals, idx, B, HW, C, K, T, stream);
}

extern "C" int mgp_head_select_np(const float* logp_np, const float* weight_cp, const int64_t* gt, float* logits,
                                  float* vals, int32_t* idx, int B, int HW, int C, int K, int T, void* stream) {
    return head_select_launch(logp_np, 1, weight_cp, gt, logits, vals, idx, B, HW, C, K, T, stream);
}

// feats[b, p, d, t] = x[b, d, idx[b, p, t]]  (ref model.py:197-206: the T gathers of global_max_pooling_gmm_topT)
namespace {
__global__ void topt_gather_kernel(const float* __restrict__ x, const int32_t* __restrict__ idx, float* __restrict__ feats,
                                   int HW, int P, int D, int T) {
    const int b = blockIdx.y, p = blockIdx.x;
    __shared__ int s_i[32];
    if (threadIdx.x < T) s_i[threadIdx.x] = idx[((size_t)b * P + p) * T + threadIdx.x];
    __syncthreads();
    float* dst = feats + ((size_t)b * P + p) * D * T;
    const float* src = x + (size_t)b * D * HW;
    for (int e = threadIdx.x; e < D * T; e += blockDim.x) {
        const int d = e / T, t = e - d * T;
        dst[e] = src[(size_t)d * HW + s_i[t]];
    }
}
}  // namespace

// f2 (ref train_and_test.py:184-199, :212-213): per image, from the level-0 log evidences out0 [B,C]:
//   p_sum = sum_c exp(out0), p_mean = p_sum / C (the reference thresholds on the sum and tests the mean), pred = argmax_c.
namespace {
__global__ void ood_score_kernel(const float* __restrict__ out0, int stride_b, int stride_c, float* __restrict__ p_sum,
                                 float* __restrict__ p_mean, int64_t* __restrict__ pred, int B, int C) {
    const int b = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (b >= B) return;
    float s = 0.f, best = -INFINITY;
    int bi = 0x7fffffff;
    for (int c = lane; c < C; c += 32) {
        const float v = out0[(size_t)b * stride_b + (size_t)c * stride_c];
        s += expf(v);
        if (v > best) { best = v; bi = c; }
    }
    s = warp_sum(s);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {                      // max value, smallest index among equals (torch.argmax on CUDA)
        const float ov = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ov > best || (ov == best && oi < bi)) { best = ov; bi = oi; }
    }
    if (lane == 0) {
        p_sum[b] = s;
        p_mean[b] = s / (float)C;
        pred[b] = bi;
    }
}
}  // namespace

extern "C" int mgp_ood_score(const float* out0, int stride_b, int stride_c, float* p_sum, float* p_mean, int64_t* pred,
                             int B, int C, void* stream) {
    if (!out0 || !p_sum || !p_mean || !pred || B <= 0 || C <= 0 || stride_b <= 0 || stride_c <= 0) return MGP_ERR_INVALID;
    ood_score_kernel<<<(B + 7) / 8, 256, 0, (cudaStream_t)stream>>>(out0, stride_b, stride_c, p_sum, p_mean, pred, B, C);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" int mgp_topt_pool(const float* sims_bphw, const float* x_nchw, float* vals, int32_t* idx, float* feats, int B,
                             int HW, int C, int K, int D, int T, void* stream) {
    if (!sims_bphw || !vals || !idx || (feats && !x_nchw) || D <= 0) return MGP_ERR_INVALID;
    int rc = head_select_launch(sims_bphw, 0, nullptr, nullptr, nullptr, vals, idx, B, HW, C, K, T, stream, 1);
    if (rc != MGP_OK || !feats) return rc;
    dim3 grid(C * K, B);
    topt_gather_kernel<<<grid, 128, 0, (cudaStream_t)stream>>>(x_nchw, idx, feats, HW, C * K, D, T);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" int mgp_head_select_top1(const uint64_t* best, const float* xhat_nd, const float* mu, const float* sigma,
                                    const float* weight_cp, const int64_t* gt, float* logits, float* vals, int32_t* idx,
                                    int B, int HW, int C, int K, int D, int T, void* stream) {
    if (!best || !xhat_nd || !mu || !sigma || !weight_cp || !gt || !logits || !vals || !idx) return MGP_ERR_INVALID;
    if (B <= 0 || HW <= 0 || C <= 0 || K <= 0 || D <= 0 || T <= 0 || (D & 3)) return MGP_ERR_INVALID;
    if (T > 32 || T > HW || HW > 1024) return MGP_ERR_UNSUPPORTED;
    const int P = C * K;
    const size_t smem = ((size_t)2 * P + (size_t)K * T + (size_t)K * (HW + 1) + (size_t)2 * K * D + 2 * K + 4) * sizeof(float);
    if (smem > 200 * 1024) return MGP_ERR_UNSUPPORTED;
    const int R = (HW + 31) / 32;
    cudaStream_t st = (cudaStream_t)stream;
#define MGP_LAUNCH_T1(RR, NRR)                                                                                       \
    do {                                                                                                             \
        MGP_CUDA(cudaFuncSetAttribute(head_top1_kernel<RR, NRR, 256>, cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                                      (int)smem));                                                                   \
        head_top1_kernel<RR, NRR, 256><<<B, 256, smem, st>>>(reinterpret_cast<const unsigned long long*>(best),      \
                                                             xhat_nd, mu, sigma, weight_cp, gt, logits, vals, idx,   \
                                                             HW, C, K, D, T);                                         \
    } while (0)
    // (8 warps per image: 16 warps were measured slower, 50.9 vs 45.5 us at cfg2 -- the phases are barrier-separated)
    if (R <= 4) MGP_LAUNCH_T1(4, 2);
    else if (R <= 7) MGP_LAUNCH_T1(7, 2);
    else if (R <= 13) MGP_LAUNCH_T1(13, 1);
    else if (R <= 25) MGP_LAUNCH_T1(25, 1);
    else MGP_LAUNCH_T1(32, 1);
#undef MGP_LAUNCH_T1
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

int head_bwd_proto_weights(const float* mu, const float* sigma, float* w, float* wm, float* wsc, int* noniso, int P,
                           int D, cudaStream_t st) {
    const size_t npd = (size_t)P * D;
    MGP_CUDA(cudaMemsetAsync(noniso, 0, sizeof(int), st));
    proto_weight_kernel<<<(unsigned)((npd + 255) / 256), 256, 0, st>>>(mu, sigma, w, wm, wsc, noniso, npd, D);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" size_t mgp_head_bwd_ws_bytes(int B, int HW, int P, int D) {
    return ((size_t)2 * P * D + (size_t)B * HW * D + (size_t)P + 64) * sizeof(float);
}

extern "C" int mgp_head_bwd_x(const float* grad_logits, const float* logits, const float* vals, const int32_t* idx,
                              const float* weight_cp, const int64_t* gt, const float* xhat_nd, const float* inv_norm,
                              const float* mu, const float* sigma, void* ws, size_t ws_bytes, void* g_x, int x_fmt,
                              int B, int HW, int C, int K, int D, int T, void* stream) {
    if (!grad_logits || !logits || !vals || !idx || !weight_cp || !xhat_nd || !inv_norm || !mu || !sigma || !ws ||
        !g_x || !mgp_x_fmt_valid(x_fmt))
        return MGP_ERR_INVALID;
    if (B <= 0 || HW <= 0 || C <= 0 || K <= 0 || D <= 0 || T <= 0) return MGP_ERR_INVALID;
    if (HW > 1024 || (size_t)C * K >= (1u << 22)) return MGP_ERR_UNSUPPORTED;
    const int P = C * K;
    if (ws_bytes < mgp_head_bwd_ws_bytes(B, HW, P, D)) return MGP_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    float* w = reinterpret_cast<float*>(ws);
    float* wm = w + (size_t)P * D;
    float* g_xhat = wm + (size_t)P * D;
    float* wsc = g_xhat + (size_t)B * HW * D;
    int* noniso = reinterpret_cast<int*>(wsc + P);
    const int rc = head_bwd_proto_weights(mu, sigma, w, wm, wsc, noniso, P, D, st);
    if (rc != MGP_OK) return rc;
    // dims per CTA: 32 lanes x 4 (one CTA per image at D = 128: the entry list is built and sorted once) or x 2
    static const bool vec2_forced = getenv("MGP_HEAD_BWD_VEC2") != nullptr;
    const int DC = ((D % 128) == 0 && !vec2_forced) ? 128 : 64;
    size_t smem = (size_t)LCAP * 16 + (size_t)(8 * HW + C + T) * 4;
    if (smem > 200 * 1024) return MGP_ERR_UNSUPPORTED;
    MGP_CUDA(cudaFuncSetAttribute(head_bwd_kernel<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MGP_CUDA(cudaFuncSetAttribute(head_bwd_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    MGP_CUDA(cudaMemsetAsync(g_xhat, 0, (size_t)B * HW * D * sizeof(float), st));   // rows without mined patches stay zero
    dim3 grid(B, (D + DC - 1) / DC);
    if (DC == 128)
        head_bwd_kernel<4><<<grid, 256, smem, st>>>(grad_logits, logits, vals, idx, weight_cp, gt, xhat_nd, w, wm, wsc, noniso,
                                                    g_xhat, HW, C, K, D, T);
    else
        head_bwd_kernel<2><<<grid, 256, smem, st>>>(grad_logits, logits, vals, idx, weight_cp, gt, xhat_nd, w, wm, wsc, noniso,
                                                    g_xhat, HW, C, K, D, T);
    MGP_CHECK_LAUNCH();
    return mgp_normalize_bwd_x(g_xhat, xhat_nd, inv_norm, g_x, x_fmt, B, D, HW, stream);
}

extern "C" int mgp_head_bwd(const float* grad_logits, const float* logits, const float* vals, const int32_t* idx,
                            const float* weight_cp, const int64_t* gt, const float* xhat_nd, const float* inv_norm,
                            const float* mu, const float* sigma, void* ws, size_t ws_bytes, float* g_x_nchw, int B,
                            int HW, int C, int K, int D, int T, void* stream) {
    return mgp_head_bwd_x(grad_logits, logits, vals, idx, weight_cp, gt, xhat_nd, inv_norm, mu, sigma, ws, ws_bytes,
                          g_x_nchw, MGP_X_F32, B, HW, C, K, D, T, stream);
}

extern "C" int mgp_mine_ce(const float* out, const int64_t* gt, float* loss_b, float* grad, int B, int C, int T,
                           float mine_coef, void* stream) {
    if (!out || !gt || !loss_b || !grad || B <= 0 || C <= 0 || T <= 0) return MGP_ERR_INVALID;
    mine_ce_kernel<<<B, 256, (size_t)T * sizeof(float), (cudaStream_t)stream>>>(out, gt, loss_b, grad, B, C, T, mine_coef);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" int mgp_push_argmin(const float* logp_bphw, const int64_t* labels, int32_t* arg, float* val, int B, int HW,
                               int C, int K, void* stream) {
    if (!logp_bphw || !labels || !arg || !val || B <= 0 || HW <= 0 || C <= 0 || K <= 0) return MGP_ERR_INVALID;
    const int warps = B * K;
    push_argmin_kernel<<<(warps + 7) / 8, 256, 0, (cudaStream_t)stream>>>(logp_bphw, labels, arg, val, HW, C, K, B);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" int mgp_push_argmin_top1(const unsigned long long* best_bp, const int64_t* labels, int32_t* arg, float* val, int B,
                                    int C, int K, void* stream) {
    if (!best_bp || !labels || !arg || !val || B <= 0 || C <= 0 || K <= 0) return MGP_ERR_INVALID;
    push_from_top1_kernel<<<(B * K + 255) / 256, 256, 0, (cudaStream_t)stream>>>(best_bp, labels, arg, val, B, C, K);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}
