// a10-a14: memory-bank EM.  ref: model.py:277-301 (update_GMM), :303-321 (_e_step),
// :338-365 (_m_step), :367-401 (_m_step_diversified), :403-421 (_score).
//
// The reference runs, per updated class and EM loop, ~100 small ATen launches plus an autograd
// backward and an Adam step over the whole [C,K,D] mean tensor (~40k launches per iteration at
// B=256).  Here one iteration's update_GMM is em_plan + ONE cluster kernel (em_fused_kernel: a class's whole
// timeline on chip; single replica, K <= 16, D in {64,128}), or -- row-sharded multi-GPU, other shapes,
// MGP_EM_UNFUSED=1 -- 2 + 2*num_em_loop + 1 launches, independent of the number of classes, with identical
// sequential semantics:
//
//   em_plan            active[c] = updated[c] && bank full; order[c] = rank among active
//   em_update phase 0  leading zero-gradient Adam steps of every class
//   per EM loop:       em_stats  (E-step + segmented weighted reduction over bank rows; HBM-bound)
//                      [multi-GPU: all-reduce of `stats` here]
//                      em_update phase 1 (gradient from S0/S1 + diversity term, Adam step, pi momentum)
//   em_update phase 2  trailing zero-gradient Adam steps
//
// Why the zero-gradient steps: the reference's optimiser owns the whole mean tensor, so every
// (class, loop) step also decays the momentum of -- and moves -- all other classes (SURVEY KA7).
// Classes only interact through the global step count, so each class replays its own timeline.
#include "mgp_common.cuh"
#include "em_common.cuh"
#include <cooperative_groups.h>
namespace cg = cooperative_groups;

int mgp_opt_em_fused();   // abi.cu
int mgp_opt_em_tc();      // abi.cu
// em_tc.cu
bool mgp_em_tc_supported(int K, int D, int cap);
int mgp_em_tc_launch(const void* shadow_h, const void* shadow_l, const float* shadow_xx, const float* bias_corr, const int32_t* order,
                     const int32_t* sched, float* mu, const float* sigma, float* weight, float* exp_avg, float* exp_avg_sq,
                     int* status, int num_em_loop, float alpha, double lr, double beta1, double beta2, double adam_eps,
                     double tau, float lamda, float* mu_stage, float* pi_stage, int C, int K, int D, int cap,
                     cudaStream_t st);

namespace {
using namespace mgp_em;

__global__ void __launch_bounds__(1024)
em_plan_kernel(uint8_t* __restrict__ updated, const int64_t* __restrict__ mem_len, int32_t* __restrict__ order,
               int32_t* __restrict__ sched, int32_t* __restrict__ adam_step, int step0, int C, int cap, int num_em_loop,
               AdamCfg adam, float* __restrict__ bias_corr, int32_t* __restrict__ clist = nullptr) {
    __shared__ int s_plan[2];
    __shared__ int s_wsum[32];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarp = blockDim.x >> 5;
    auto active = [&](int c) { return c < C && updated[c] != 0 && mem_len[c] >= (int64_t)cap; };   // ref model.py:283, :289
    // pass 1: how many classes are active
    int cnt = 0;
    for (int c = tid; c < C; c += blockDim.x) cnt += active(c) ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    if (lane == 0) s_wsum[warp] = cnt;
    __syncthreads();
    if (tid == 0) {
        int r = 0;
        for (int w = 0; w < nwarp; ++w) r += s_wsum[w];
        sched[0] = r;
        const int s0 = adam_step ? adam_step[0] : step0;
        sched[1] = s0;
        if (adam_step) adam_step[0] = s0 + r * num_em_loop;
        s_plan[0] = r; s_plan[1] = s0;
    }
    __syncthreads();
    // pass 2: order[c] = rank among the active (ascending id) or -1; clist = the classes in launch order, the active ones first
    const int r_total = s_plan[0];
    int base = 0;
    for (int c0 = 0; c0 < C; c0 += blockDim.x) {
        const int c = c0 + tid;
        const bool act = active(c);
        const unsigned bal = __ballot_sync(0xffffffffu, act);
        if (lane == 0) s_wsum[warp] = __popc(bal);
        __syncthreads();
        int before = 0, chunk = 0;
        for (int w = 0; w < nwarp; ++w) {
            const int v = s_wsum[w];
            before += (w < warp) ? v : 0;
            chunk += v;
        }
        const int rank = base + before + __popc(bal & ((1u << lane) - 1u));   // active classes with a smaller id
        if (c < C) {
            order[c] = act ? rank : -1;
            if (clist) clist[act ? rank : r_total + (c - rank)] = c;
        }
        base += chunk;
        __syncthreads();
    }
    for (int c = tid; c < C; c += blockDim.x) updated[c] = 0;             // ref model.py:287, :301
    if (bias_corr) {
        // Step-dependent factors of this call's Adam steps s0+1 .. s0+n (n = r*L), evaluated ONCE here in double (torch:
        // Python doubles, narrowed last) instead of per class in the EM kernel:
        //   [2i] = lr / (1 - b1^t), [2i+1] = sqrt(1 - b2^t), t = s0+1+i;  then b1^i, b2^(i/2), b2^i for i = 0..n
        const int n = s_plan[0] * num_em_loop, s0 = s_plan[1];
        float* t_b1 = bias_corr + 2 * n;
        float* t_b2h = t_b1 + (n + 1);
        float* t_b2 = t_b2h + (n + 1);
        for (int i = threadIdx.x; i <= n; i += blockDim.x) {
            if (i < n) {
                const double t = (double)(s0 + i + 1);
                bias_corr[2 * i] = (float)(adam.lr / (1.0 - exp(t * adam.ln_b1)));
                bias_corr[2 * i + 1] = (float)sqrt(1.0 - exp(t * adam.ln_b2));
            }
            const double b2h = exp(0.5 * (double)i * adam.ln_b2);
            t_b1[i] = (float)exp((double)i * adam.ln_b1);
            t_b2h[i] = (float)b2h;
            t_b2[i] = (float)(b2h * b2h);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// E-step for one row held by a warp: lane l owns elements d = 4*(l + 32 j) .. +3, j < VEC4.
// Returns the log-normaliser; lane k (and k+32) keeps the smoothed responsibility of component k.
template <int VEC4, int KBLK>
__device__ __forceinline__ float warp_estep_rowb(const float4 (&xv)[VEC4], const float* __restrict__ s_mu,
                                                const float* __restrict__ s_rinv, const float* __restrict__ s_cst,
                                                int K, int D, int lane, float alpha, float& r_lo, float& r_hi,
                                                float& lr_lo, float& lr_hi) {
    float w_lo = -INFINITY, w_hi = -INFINITY;
    for (int k0 = 0; k0 < K; k0 += KBLK) {
        float q[KBLK];
#pragma unroll
        for (int i = 0; i < KBLK; ++i) {
            q[i] = 0.f;
            const int k = k0 + i;
            if (k < K) {
#pragma unroll
                for (int j = 0; j < VEC4; ++j) {
                    const int d = 4 * (lane + 32 * j);
                    if (d >= D) continue;
                    const float4 m = *reinterpret_cast<const float4*>(s_mu + k * D + d);
                    const float4 r = *reinterpret_cast<const float4*>(s_rinv + k * D + d);
                    float t;
                    t = (xv[j].x - m.x) * r.x; q[i] = fmaf(t, t, q[i]);
                    t = (xv[j].y - m.y) * r.y; q[i] = fmaf(t, t, q[i]);
                    t = (xv[j].z - m.z) * r.z; q[i] = fmaf(t, t, q[i]);
                    t = (xv[j].w - m.w) * r.w; q[i] = fmaf(t, t, q[i]);
                }
            }
        }
        // KBLK independent butterflies: the shuffles of different components overlap
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
#pragma unroll
            for (int i = 0; i < KBLK; ++i) q[i] += __shfl_xor_sync(0xffffffffu, q[i], o);
#pragma unroll
        for (int i = 0; i < KBLK; ++i) {
            const int k = k0 + i;
            if (k < K) {
                const float wl = s_cst[k] - 0.5f * q[i];   // lp + log(pi + eps)   (ref :316)
                if (lane == (k & 31)) {
                    if (k < 32) w_lo = wl; else w_hi = wl;
                }
            }
        }
    }
    const float mx = warp_max(fmaxf(w_lo, w_hi));
    const float e_lo = (lane < K) ? expf(w_lo - mx) : 0.f;
    const float e_hi = (lane + 32 < K) ? expf(w_hi - mx) : 0.f;
    const float se = warp_sum(e_lo + e_hi);
    const float norm = mx + logf(se);               // logsumexp (ref :318)
    lr_lo = w_lo - norm;                            // log_resp (ref :319)
    lr_hi = w_hi - norm;
    // smoothed responsibility (ref :380-383): (resp + alpha) / sum_k(resp + alpha); resp sums to one
    // (up to an ulp), so the denominator is 1 + K alpha
    const float inv_se = 1.0f / se, inv_den = 1.0f / (1.0f + (float)K * alpha);
    r_lo = (lane < K) ? fmaf(e_lo, inv_se, alpha) * inv_den : 0.f;
    r_hi = (lane + 32 < K) ? fmaf(e_hi, inv_se, alpha) * inv_den : 0.f;
    return norm;
}

// E-step of one bank row for the statistics kernel, K <= 16.  Per-lane partial sums of all components are
// reduced with a recursive-halving butterfly (16 values: 8+4+2+1+1 = 16 shuffles instead of 5 per component);
// afterwards lane l holds the total of component kidx(l) (each component twice: lanes l and l^1).
//   iso  : sigma constant over d inside each component -> q_k = w_k (|x|^2 + |mu_k|^2) + x . a_k, a_k = -2 w_k mu_k
//          (s_mu holds a_k, s_rinv is unused, s_cst[k] folds -0.5*w_k*|mu_k|^2; s_w[k] = w_k)
//   !iso : exact form sum_d ((x - mu) rinv)^2
// Returns the log-normaliser; `r` = smoothed responsibility of component kidx(lane) (valid lanes only).
__device__ __forceinline__ int estep_kidx(int lane) {       // component (within a block of 8) a lane ends up holding
    return (((lane >> 4) & 1) << 2) | (((lane >> 3) & 1) << 1) | ((lane >> 2) & 1);
}
// partial sums of components k0 .. k0+7 of this lane, reduced over the warp: 4+2+1+1+1 = 9 shuffles;
// returns the total of component k0 + estep_kidx(lane) (each component ends up in 4 lanes)
template <int VEC4>
__device__ __forceinline__ float estep_block8(const float4 (&xv)[VEC4], float xx, const float* __restrict__ s_mu,
                                              const float* __restrict__ s_rinv, const float* __restrict__ s_w, bool iso,
                                              int k0, int K, int D, int lane) {
    float q[8];
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        q[i] = 0.f;
        const int k = k0 + i;
        if (k < K) {
#pragma unroll
            for (int j = 0; j < VEC4; ++j) {
                const int d = 4 * (lane + 32 * j);
                if (d >= D) continue;
                const float4 m = *reinterpret_cast<const float4*>(s_mu + k * D + d);
                if (iso) {
                    q[i] = fmaf(xv[j].x, m.x, q[i]); q[i] = fmaf(xv[j].y, m.y, q[i]);
                    q[i] = fmaf(xv[j].z, m.z, q[i]); q[i] = fmaf(xv[j].w, m.w, q[i]);
                } else {
                    const float4 rr = *reinterpret_cast<const float4*>(s_rinv + k * D + d);
                    float t;
                    t = (xv[j].x - m.x) * rr.x; q[i] = fmaf(t, t, q[i]);
                    t = (xv[j].y - m.y) * rr.y; q[i] = fmaf(t, t, q[i]);
                    t = (xv[j].z - m.z) * rr.z; q[i] = fmaf(t, t, q[i]);
                    t = (xv[j].w - m.w) * rr.w; q[i] = fmaf(t, t, q[i]);
                }
            }
            if (iso) q[i] = fmaf(s_w[k], xx, q[i]);          // every lane adds its share of w_k |x|^2
        }
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const bool up = (lane & 16) != 0;
        const float keep = up ? q[i + 4] : q[i], send = up ? q[i] : q[i + 4];
        q[i] = keep + __shfl_xor_sync(0xffffffffu, send, 16);
    }
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const bool up = (lane & 8) != 0;
        const float keep = up ? q[i + 2] : q[i], send = up ? q[i] : q[i + 2];
        q[i] = keep + __shfl_xor_sync(0xffffffffu, send, 8);
    }
    {
        const bool up = (lane & 4) != 0;
        const float keep = up ? q[1] : q[0], send = up ? q[0] : q[1];
        q[0] = keep + __shfl_xor_sync(0xffffffffu, send, 4);
    }
    q[0] += __shfl_xor_sync(0xffffffffu, q[0], 2);
    q[0] += __shfl_xor_sync(0xffffffffu, q[0], 1);
    return q[0];
}
template <int VEC4>
__device__ __forceinline__ float warp_estep_packed(const float4 (&xv)[VEC4], const float* __restrict__ s_mu,
                                                   const float* __restrict__ s_rinv, const float* __restrict__ s_cst,
                                                   const float* __restrict__ s_w, bool iso, int K, int D, int lane,
                                                   float alpha, float& r0, float& r1, int& kk) {
    float xx = 0.f;
    if (iso) {
#pragma unroll
        for (int j = 0; j < VEC4; ++j) {
            xx = fmaf(xv[j].x, xv[j].x, xx); xx = fmaf(xv[j].y, xv[j].y, xx);
            xx = fmaf(xv[j].z, xv[j].z, xx); xx = fmaf(xv[j].w, xv[j].w, xx);
        }
    }
    kk = estep_kidx(lane);
    const float q0 = estep_block8<VEC4>(xv, xx, s_mu, s_rinv, s_w, iso, 0, K, D, lane);
    const float q1 = (K > 8) ? estep_block8<VEC4>(xv, xx, s_mu, s_rinv, s_w, iso, 8, K, D, lane) : 0.f;
    const bool v0 = kk < K, v1 = kk + 8 < K;
    const float w0 = v0 ? s_cst[kk] - 0.5f * q0 : -INFINITY;            // lp + log(pi + eps)   (ref :316)
    const float w1 = v1 ? s_cst[kk + 8] - 0.5f * q1 : -INFINITY;
    const float mx = warp_max(fmaxf(w0, w1));
    const float e0 = v0 ? expf(w0 - mx) : 0.f, e1 = v1 ? expf(w1 - mx) : 0.f;
    const float se = 0.25f * warp_sum(e0 + e1);                         // every component sits in four lanes
    const float inv_se = 1.0f / se, inv_den = 1.0f / (1.0f + (float)K * alpha);
    r0 = v0 ? fmaf(e0, inv_se, alpha) * inv_den : 0.f;                  // ref :380-383
    r1 = v1 ? fmaf(e1, inv_se, alpha) * inv_den : 0.f;
    return mx + logf(se);                                               // logsumexp (ref :318)
}

template <int VEC4>
__device__ __forceinline__ float warp_estep_row(const float4 (&xv)[VEC4], const float* __restrict__ s_mu,
                                                const float* __restrict__ s_rinv, const float* __restrict__ s_cst,
                                                int K, int D, int lane, float alpha, float& r_lo, float& r_hi,
                                                float& lr_lo, float& lr_hi) {
    if (K % 5 == 0) return warp_estep_rowb<VEC4, 5>(xv, s_mu, s_rinv, s_cst, K, D, lane, alpha, r_lo, r_hi, lr_lo, lr_hi);
    return warp_estep_rowb<VEC4, 8>(xv, s_mu, s_rinv, s_cst, K, D, lane, alpha, r_lo, r_hi, lr_lo, lr_hi);
}

constexpr int RB = 32;  // rows per batch

// grid (C, n_split); CTA (c, s) reduces rows [seg_begin, seg_end) of class c.
// Thread t owns outputs o = t + 256 i (o = k*D + d) of S1 (and S2); threads t < K own S0[t].
template <int VEC4, int NOUT, bool WITH_S2>
__global__ void __launch_bounds__(256, (NOUT <= 10) ? 3 : 1)
em_stats_kernel(const float* __restrict__ bank, const int32_t* __restrict__ order, const float* __restrict__ mu,
                const float* __restrict__ sigma, const float* __restrict__ weight, float alpha, int row_begin,
                int row_end, int n_split, float* __restrict__ stats, size_t stat_stride, int C, int K, int D, int cap) {
    const int c = blockIdx.x;
    if (order[c] < 0) return;
    extern __shared__ __align__(16) float sm[];
    float* s_mu = sm;                    // [K][D]
    float* s_rinv = s_mu + K * D;        // [K][D]
    float* s_x = s_rinv + K * D;         // [RB][D]
    float* s_r = s_x + RB * D;           // [RB][K]
    float* s_cst = s_r + RB * K;         // [K]
    float* s_w = s_cst + K;              // [K]  w_k (isotropic classes)
    __shared__ float s_ll[8];
    __shared__ int s_iso;

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int P = C * K;
    const int split = blockIdx.y;
    const int rows = row_end - row_begin;
    const int per = (rows + n_split - 1) / n_split;
    const int seg_b = row_begin + split * per;
    const int seg_e = min(row_end, seg_b + per);

    // sigma constant over d inside every component of this class?  (every state the shipped loop reaches)
    if (tid == 0) s_iso = 1;
    __syncthreads();
    {
        bool same = true;
        for (int i = tid; i < K * D; i += 256) same = same && (sigma[(size_t)c * K * D + i] == sigma[(size_t)c * K * D + (i / D) * D]);
        if (!same) s_iso = 0;
    }
    __syncthreads();
    const bool packed = (K <= 16);
    const bool iso = packed && (s_iso != 0);
    for (int i = tid; i < K * D; i += 256) {
        const float rinv = 1.0f / (sigma[(size_t)c * K * D + i] + EM_EPS);           // ref :333
        const float m = mu[(size_t)c * K * D + i];
        s_rinv[i] = rinv;
        s_mu[i] = iso ? -2.0f * rinv * rinv * m : m;                                  // a_k = -2 w_k mu_k
    }
    __syncthreads();
    for (int k = warp; k < K; k += 8) {
        float ls = 0.f, mm = 0.f;
        for (int d = lane; d < D; d += 32) {
            ls += logf(sigma[(size_t)c * K * D + k * D + d] + EM_EPS);               // ref :334
            const float m = mu[(size_t)c * K * D + k * D + d];
            mm = fmaf(m, m, mm);
        }
        ls = warp_sum(ls);
        mm = warp_sum(mm);
        if (lane == 0) {
            const float rinv0 = s_rinv[k * D];
            const float wk = rinv0 * rinv0;
            s_w[k] = wk;
            s_cst[k] = -0.5f * (float)D * MGP_LOG_2PI - ls + logf(weight[(size_t)c * P + c * K + k] + EM_EPS) -
                       (iso ? 0.5f * wk * mm : 0.f);
        }
    }
    __syncthreads();

    float a1[NOUT], a2[NOUT];
    int ok_[NOUT], od_[NOUT];                 // component / dim of each owned output (-1: none)
    const int KD = K * D;
    // fast mapping when D divides 256 (D = 64/128/256): the thread keeps ONE dim d = tid % D and NOUT
    // consecutive components -> per bank row one x load, NOUT broadcast r loads, NOUT FMAs
    const bool fastmap = (256 % D == 0) && ((256 / D) * NOUT >= K);
    const int fd = tid % D, fk0 = (tid / D) * NOUT;
#pragma unroll
    for (int i = 0; i < NOUT; ++i) {
        a1[i] = 0.f;
        a2[i] = 0.f;
        const int o = tid + 256 * i;
        if (fastmap) {
            ok_[i] = (fk0 + i < K) ? fk0 + i : -1;
            od_[i] = fd;
        } else {
            ok_[i] = (o < KD) ? o / D : -1;
            od_[i] = (o < KD) ? o - (o / D) * D : 0;
        }
    }
    float a0 = 0.f, ll = 0.f;

    for (int r0 = seg_b; r0 < seg_e; r0 += RB) {
        const int nr = min(RB, seg_e - r0);
        // phase 1: E-step, warp per row
        for (int rl = warp; rl < nr; rl += 8) {
            const float* xr = bank + ((size_t)c * cap + r0 + rl) * D;
            float4 xv[VEC4];
#pragma unroll
            for (int j = 0; j < VEC4; ++j) {
                xv[j] = make_float4(0.f, 0.f, 0.f, 0.f);
                if (4 * (lane + 32 * j) < D) {
                    xv[j] = __ldg(reinterpret_cast<const float4*>(xr) + lane + 32 * j);
                    *reinterpret_cast<float4*>(s_x + rl * D + 4 * (lane + 32 * j)) = xv[j];
                }
            }
            if (packed) {
                float ra, rb;
                int kk;
                const float norm = warp_estep_packed<VEC4>(xv, s_mu, s_rinv, s_cst, s_w, iso, K, D, lane, alpha, ra, rb, kk);
                if ((lane & 3) == 0) {
                    if (kk < K) s_r[rl * K + kk] = ra;
                    if (kk + 8 < K) s_r[rl * K + kk + 8] = rb;
                }
                if (lane == 0) ll += norm;
            } else {
                float r_lo, r_hi, l_lo, l_hi;
                const float norm = warp_estep_row<VEC4>(xv, s_mu, s_rinv, s_cst, K, D, lane, alpha, r_lo, r_hi, l_lo, l_hi);
                if (lane < K) s_r[rl * K + lane] = r_lo;
                if (lane + 32 < K) s_r[rl * K + lane + 32] = r_hi;
                if (lane == 0) ll += norm;
            }
        }
        __syncthreads();
        // phase 2: rank-nr update of the statistics, thread per output
        if (fastmap) {
            const float* xp = s_x + fd;
            const float* rp = s_r + fk0;
#pragma unroll 4
            for (int rl = 0; rl < nr; ++rl) {
                const float xx = xp[rl * D];
#pragma unroll
                for (int i = 0; i < NOUT; ++i) {
                    const float rr = (fk0 + i < K) ? rp[rl * K + i] : 0.f;
                    a1[i] = fmaf(rr, xx, a1[i]);
                    if (WITH_S2) a2[i] = fmaf(rr * xx, xx, a2[i]);
                }
            }
            if (tid < K)
                for (int rl = 0; rl < nr; ++rl) a0 += s_r[rl * K + tid];
        } else {
            for (int rl = 0; rl < nr; ++rl) {
#pragma unroll
                for (int i = 0; i < NOUT; ++i) {
                    if (ok_[i] >= 0) {
                        const float xx = s_x[rl * D + od_[i]];
                        const float rx = s_r[rl * K + ok_[i]] * xx;
                        a1[i] += rx;
                        if (WITH_S2) a2[i] = fmaf(rx, xx, a2[i]);
                    }
                }
                if (tid < K) a0 += s_r[rl * K + tid];
            }
        }
        __syncthreads();
    }

    float* out = stats + ((size_t)c * n_split + split) * stat_stride;
    if (tid < K) out[tid] = a0;
#pragma unroll
    for (int i = 0; i < NOUT; ++i) {
        if (ok_[i] >= 0) {
            const int o = ok_[i] * D + od_[i];
            out[K + o] = a1[i];
            if (WITH_S2) out[K + KD + o] = a2[i];
        }
    }
    if (lane == 0) s_ll[warp] = ll;
    __syncthreads();
    if (tid == 0) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += s_ll[w];
        out[stat_stride - 1] = t;
    }
}

// ---------------------------------------------------------------------------------------------
// Specialised statistics kernel for the shipped shapes (K <= 16, D = 64 / 128 at compile time):
// the generic kernel above spends most of its issue slots on index arithmetic and predicates (ncu: FFMA
// is 18 % of its instructions).  Here a batch of up to `rbf` bank rows is staged once in shared memory
// (cp.async, row pitch D+4 so both access patterns below are conflict-free) and
//   phase 1 (E-step):   thread = (row, half of the components): one LDS.128 of x feeds KH*4 FMAs against
//                       LDS.128 broadcasts of the packed means; the two halves meet with one shuffle pair
//                       for the soft-max; no warp reductions over d.
//   phase 2 (S1 [,S2]): thread = (dim d, row group): x[row][d] (1 LDS) times the row's K responsibilities
//                       (RS/4 broadcast LDS.128) -> 2*KH FMAs, accumulators in registers.
// Same outputs and layout as em_stats_kernel; grid (C, n_split).
template <int D, int KH, bool WITH_S2>
__global__ void __launch_bounds__(256, 3)
em_stats_fast_kernel(const float* __restrict__ bank, const int32_t* __restrict__ order, const float* __restrict__ mu,
                     const float* __restrict__ sigma, const float* __restrict__ weight, float alpha, int row_begin,
                     int row_end, int n_split, int rbf, float* __restrict__ stats, size_t stat_stride, int C, int K,
                     int cap) {
    constexpr int DP = D + 4, K2 = 2 * KH, RS = (K2 + 3) & ~3, G = 256 / D, D4 = D / 4;
    const int c = blockIdx.x;
    if (order[c] < 0) return;
    extern __shared__ __align__(16) float sm[];
    const int xfl = max(rbf * DP, G * K2 * D);
    float* s_a = sm;                     // [K2][DP]  iso: -2 w_k mu_k, else mu_k   (rows >= K are zero)
    float* s_ri = s_a + K2 * DP;         // [K2][DP]  1/(sigma+eps)
    float* s_x = s_ri + K2 * DP;         // [rbf][DP] bank rows of the batch (reused for the group combine)
    float* s_r = s_x + xfl;              // [rbf][RS] smoothed responsibilities
    float* s_cst = s_r + rbf * RS;       // [K2]
    float* s_w = s_cst + K2;             // [K2]
    float* s_red = s_w + K2;             // [8][K2]
    __shared__ float s_ll[8];

    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int P = C * K;
    const int split = blockIdx.y;
    const int rows = row_end - row_begin;
    const int per = (rows + n_split - 1) / n_split;
    const int seg_b = row_begin + split * per;
    const int seg_e = min(row_end, seg_b + per);
    const float* sg_c = sigma + (size_t)c * K * D;
    const float* mu_c = mu + (size_t)c * K * D;

    bool same = true;
    for (int i = tid; i < K * D; i += 256) same = same && (sg_c[i] == sg_c[(i / D) * D]);
    const bool iso = __syncthreads_and(same ? 1 : 0) != 0;
    for (int i = tid; i < K2 * D; i += 256) {
        const int k = i / D, d = i - k * D;
        float av = 0.f, rv = 0.f;
        if (k < K) {
            rv = 1.0f / (sg_c[i] + EM_EPS);                                           // ref :333
            av = iso ? -2.0f * rv * rv * mu_c[i] : mu_c[i];
        }
        s_a[k * DP + d] = av;
        s_ri[k * DP + d] = rv;
    }
    for (int k = warp; k < K2; k += 8) {
        float ls = 0.f, mm = 0.f;
        if (k < K)
            for (int d = lane; d < D; d += 32) {
                ls += logf(sg_c[k * D + d] + EM_EPS);                                 // ref :334
                const float m = mu_c[k * D + d];
                mm = fmaf(m, m, mm);
            }
        ls = warp_sum(ls);
        mm = warp_sum(mm);
        if (lane == 0) {
            float wk = 0.f, cst = 0.f;
            if (k < K) {
                const float rinv0 = 1.0f / (sg_c[k * D] + EM_EPS);
                wk = rinv0 * rinv0;
                cst = -0.5f * (float)D * MGP_LOG_2PI - ls + logf(weight[(size_t)c * P + c * K + k] + EM_EPS) -
                      (iso ? 0.5f * wk * mm : 0.f);
            }
            s_w[k] = wk;
            s_cst[k] = cst;
        }
    }
    __syncthreads();

    float a1[K2], a2[WITH_S2 ? K2 : 1], s0[KH];
#pragma unroll
    for (int i = 0; i < K2; ++i) a1[i] = 0.f;
#pragma unroll
    for (int i = 0; i < (WITH_S2 ? K2 : 1); ++i) a2[i] = 0.f;
#pragma unroll
    for (int i = 0; i < KH; ++i) s0[i] = 0.f;
    float ll = 0.f;
    const int row = tid >> 1, half = tid & 1;
    const int pd = tid & (D - 1), pg = tid / D;
    const float inv_den = 1.0f / (1.0f + (float)K * alpha);
    const unsigned sx_addr = (unsigned)__cvta_generic_to_shared(s_x);

    for (int r0 = seg_b; r0 < seg_e; r0 += rbf) {
        const int nr = min(rbf, seg_e - r0);
        const float* src = bank + ((size_t)c * cap + r0) * D;
        for (int q = tid; q < nr * D4; q += 256) {
            const int rr = q / D4, c4 = q - rr * D4;
            asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sx_addr + (unsigned)(rr * DP + 4 * c4) * 4u),
                         "l"(src + (size_t)q * 4)
                         : "memory");
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
        asm volatile("cp.async.wait_group 0;" ::: "memory");
        __syncthreads();
        // phase 1
        if (warp * 16 < nr) {
            const float* xr = s_x + min(row, nr - 1) * DP;
            const float* ar = s_a + half * KH * DP;
            const float* rr_ = s_ri + half * KH * DP;
            float acc[KH], xx = 0.f;
#pragma unroll
            for (int i = 0; i < KH; ++i) acc[i] = 0.f;
            if (iso) {
                // paired FMAs (FFMA2): even / odd dims accumulate separately and are added at the end
                float2 acc2[KH], xx2 = make_float2(0.f, 0.f);
#pragma unroll
                for (int i = 0; i < KH; ++i) acc2[i] = make_float2(0.f, 0.f);
#pragma unroll 4
                for (int j = 0; j < D4; ++j) {
                    const float4 xv = *reinterpret_cast<const float4*>(xr + 4 * j);
                    const float2 x01 = make_float2(xv.x, xv.y), x23 = make_float2(xv.z, xv.w);
                    xx2 = ffma2(x01, x01, xx2);
                    xx2 = ffma2(x23, x23, xx2);
#pragma unroll
                    for (int i = 0; i < KH; ++i) {
                        const float4 m = *reinterpret_cast<const float4*>(ar + i * DP + 4 * j);
                        acc2[i] = ffma2(x01, make_float2(m.x, m.y), acc2[i]);
                        acc2[i] = ffma2(x23, make_float2(m.z, m.w), acc2[i]);
                    }
                }
                xx = xx2.x + xx2.y;
#pragma unroll
                for (int i = 0; i < KH; ++i) acc[i] = acc2[i].x + acc2[i].y;
            } else {
#pragma unroll 2
                for (int j = 0; j < D4; ++j) {
                    const float4 xv = *reinterpret_cast<const float4*>(xr + 4 * j);
#pragma unroll
                    for (int i = 0; i < KH; ++i) {
                        const float4 m = *reinterpret_cast<const float4*>(ar + i * DP + 4 * j);
                        const float4 ri = *reinterpret_cast<const float4*>(rr_ + i * DP + 4 * j);
                        float t;
                        t = (xv.x - m.x) * ri.x; acc[i] = fmaf(t, t, acc[i]);
                        t = (xv.y - m.y) * ri.y; acc[i] = fmaf(t, t, acc[i]);
                        t = (xv.z - m.z) * ri.z; acc[i] = fmaf(t, t, acc[i]);
                        t = (xv.w - m.w) * ri.w; acc[i] = fmaf(t, t, acc[i]);
                    }
                }
            }
            float wl[KH], mx = -INFINITY;
#pragma unroll
            for (int i = 0; i < KH; ++i) {
                const int k = half * KH + i;
                const float q = iso ? fmaf(s_w[k], xx, acc[i]) : acc[i];
                wl[i] = (k < K) ? s_cst[k] - 0.5f * q : -INFINITY;                    // lp + log(pi + eps)  (ref :316)
                mx = fmaxf(mx, wl[i]);
            }
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
            float se = 0.f;
#pragma unroll
            for (int i = 0; i < KH; ++i) {
                wl[i] = (half * KH + i < K) ? expf(wl[i] - mx) : 0.f;
                se += wl[i];
            }
            se += __shfl_xor_sync(0xffffffffu, se, 1);
            const float inv_se = 1.0f / se;
            const bool live = row < nr;
#pragma unroll
            for (int i = 0; i < KH; ++i) {
                const int k = half * KH + i;
                const float r = (k < K && live) ? fmaf(wl[i], inv_se, alpha) * inv_den : 0.f;   // ref :380-383
                s0[i] += r;
                if (live) s_r[row * RS + k] = r;
            }
            if (live && half == 0) ll += mx + logf(se);                               // logsumexp (ref :318)
        }
        __syncthreads();
        // phase 2
        {
            const int per_g = (nr + G - 1) / G;
            const int rb = pg * per_g, re = min(nr, rb + per_g);
#pragma unroll 2
            for (int rl = rb; rl < re; ++rl) {
                const float xv = s_x[rl * DP + pd];
                float rv[RS];
#pragma unroll
                for (int i = 0; i < RS / 4; ++i)
                    *reinterpret_cast<float4*>(rv + 4 * i) = *reinterpret_cast<const float4*>(s_r + rl * RS + 4 * i);
                const float2 xd = make_float2(xv, xv);
#pragma unroll
                for (int q = 0; q < K2 / 2; ++q) {              // FFMA2: two components per issue slot
                    const float2 t = ffma2(make_float2(rv[2 * q], rv[2 * q + 1]), xd, make_float2(a1[2 * q], a1[2 * q + 1]));
                    a1[2 * q] = t.x;
                    a1[2 * q + 1] = t.y;
                }
                if (WITH_S2) {
#pragma unroll
                    for (int i = 0; i < K2; ++i) a2[i] = fmaf(rv[i] * xv, xv, a2[i]);
                }
            }
        }
        __syncthreads();
    }

    float* out = stats + ((size_t)c * n_split + split) * stat_stride;
    // S0 and the score: lanes of equal half hold partial sums
#pragma unroll
    for (int i = 0; i < KH; ++i) {
#pragma unroll
        for (int o = 2; o < 32; o <<= 1) s0[i] += __shfl_xor_sync(0xffffffffu, s0[i], o);
        if (lane < 2) s_red[warp * K2 + lane * KH + i] = s0[i];
    }
    ll = warp_sum(ll);
    if (lane == 0) s_ll[warp] = ll;
    // combine the G row groups of S1 (and S2) through shared memory in a fixed order
#pragma unroll
    for (int i = 0; i < K2; ++i) s_x[(pg * K2 + i) * D + pd] = a1[i];
    __syncthreads();
    if (tid < K) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += s_red[w * K2 + tid];
        out[tid] = t;
    }
    if (tid == 0) {
        float t = 0.f;
#pragma unroll
        for (int w = 0; w < 8; ++w) t += s_ll[w];
        out[stat_stride - 1] = t;
    }
    const int KD = K * D;
    for (int o = tid; o < KD; o += 256) {
        const int k = o / D, d = o - k * D;
        float t = 0.f;
#pragma unroll
        for (int g = 0; g < G; ++g) t += s_x[(g * K2 + k) * D + d];
        out[K + o] = t;
    }
    if (WITH_S2) {
        __syncthreads();
#pragma unroll
        for (int i = 0; i < K2; ++i) s_x[(pg * K2 + i) * D + pd] = a2[i];
        __syncthreads();
        for (int o = tid; o < KD; o += 256) {
            const int k = o / D, d = o - k * D;
            float t = 0.f;
#pragma unroll
            for (int g = 0; g < G; ++g) t += s_x[(g * K2 + k) * D + d];
            out[K + KD + o] = t;
        }
    }
}

// ---------------------------------------------------------------------------------------------
// The whole update_GMM of a single replica in ONE launch (after em_plan): classes only interact through the global
// Adam step count (file header), so a cluster of two CTAs owns a class for all of its timeline --
//   leading zero-gradient steps, num_em_loop x [E-step + statistics over the class's bank rows (each CTA half of
//   them, partial sums exchanged through distributed shared memory), gradient + diversity + Adam step + pi
//   momentum], trailing zero-gradient steps --
// with the class's means, Adam moments and mixture weights held on chip in between.  Both CTAs carry identical
// copies of that state (the exchange sums the two partials in rank order), rank 0 writes it back.  Arithmetic and
// summation order are those of em_stats_fast_kernel (n_split = 2) + em_update_kernel.
template <int D, int KH>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(256, 3)
em_fused_kernel(const float* __restrict__ bank, const int32_t* __restrict__ order, const int32_t* __restrict__ sched,
                float* __restrict__ mu, const float* __restrict__ sigma, float* __restrict__ weight,
                float* __restrict__ exp_avg, float* __restrict__ exp_avg_sq, float alpha, int rbf, int num_em_loop,
                AdamCfg adam, float tau, float omtau, float lamda, int C, int K, int cap) {
    constexpr int DP = D + 4, K2 = 2 * KH, RS = (K2 + 3) & ~3, G = 256 / D, D4 = D / 4, TAB = 256;
    constexpr int NE = (K2 * D + 255) / 256;                     // elements of the class's [K,D] state owned by a thread
    cg::cluster_group cluster = cg::this_cluster();
    const int c = blockIdx.x >> 1, rank = blockIdx.x & 1;
    const int ord = order[c];
    const int n_active = sched[0], step0 = sched[1];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int P = C * K, KD = K * D, L = num_em_loop;
    extern __shared__ __align__(16) float sm[];
    const int xfl = max(rbf * DP, (K + KD + 3 + G * K2 * D + 3) & ~3);
    float* s_a = sm;                     // [K2][DP]  iso: -2 w_k mu_k, else mu_k (rows >= K zero)
    float* s_ri = s_a + K2 * DP;         // [K2][DP]  1/(sigma+eps)
    float* s_x = s_ri + K2 * DP;         // [rbf][DP] bank rows; afterwards group combine and the partials [K + KD]
    float* s_r = s_x + xfl;              // [rbf][RS]
    float* s_mu = s_r + rbf * RS;        // [K][D]    current means
    float* s_cst = s_mu + K2 * D;        // [K2]
    float* s_w = s_cst + K2;             // [K2]
    float* s_ls = s_w + K2;              // [K2]      sum_d log(sigma + eps)
    float* s_pi = s_ls + K2;             // [K2]
    float* s_s0 = s_pi + K2;             // [K2]      S0 of the whole class
    float* s_red = s_s0 + K2;            // [8][K2]
    float* s_e = s_red + 8 * K2;         // [K][K]
    float* s_c = s_e + K2 * K2;          // [TAB]
    float* s_d = s_c + TAB;              // [TAB]
    __shared__ float s_adam[2];
    __shared__ float s_tail[2];
    float* mu_c = mu + (size_t)c * KD;
    const float* sg_c = sigma + (size_t)c * KD;

    float p_[NE], m_[NE], v_[NE];
#pragma unroll
    for (int i = 0; i < NE; ++i) {
        const int o = tid + 256 * i;
        p_[i] = 0.f; m_[i] = 0.f; v_[i] = 1.f;
        if (o < KD) {
            p_[i] = mu_c[o];
            m_[i] = exp_avg[(size_t)c * KD + o];
            v_[i] = exp_avg_sq[(size_t)c * KD + o];
        }
    }
    // `count` zero-gradient Adam steps first+1 .. first+count on the registers (see em_update_kernel phase 0/2)
    auto replay = [&](int first, int count) {
        if (count <= 0) return;
        float a_[NE];
#pragma unroll
        for (int i = 0; i < NE; ++i) a_[i] = sqrtf(v_[i]);
        const int count_p = replay_explicit_steps(count, first, (float)adam.beta1);
        for (int s0 = 0; s0 < count_p; s0 += TAB) {
            const int ns = min(TAB, count_p - s0);
            __syncthreads();
            for (int s = tid; s < ns; s += 256) replay_coeffs(adam, first, s0 + s + 1, s_c[s], s_d[s]);
            if (tid == 255 && s0 + TAB >= count_p && count > count_p) replay_tail(adam, first, count_p, count, s_tail[0], s_tail[1]);
            __syncthreads();
            for (int s = 0; s < ns; ++s) {
                const float cs = -s_c[s], ds = s_d[s];
#pragma unroll
                for (int i = 0; i < NE; ++i) {
                    float rc;
                    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(fmaf(a_[i], ds, adam.epsf)));
                    p_[i] = fmaf(cs * m_[i], rc, p_[i]);
                }
            }
        }
        if (count > count_p) {                       // steps count_p+1 .. count in one term (see replay_tail)
            const float cs = -s_tail[0], ds = s_tail[1];
#pragma unroll
            for (int i = 0; i < NE; ++i) {
                float rc;
                asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(fmaf(a_[i], ds, adam.epsf)));
                p_[i] = fmaf(cs * m_[i], rc, p_[i]);
            }
        }
        const float mdec = (float)pow(adam.beta1, (double)count);
        const float vdec = (float)pow(adam.beta2, (double)count);
#pragma unroll
        for (int i = 0; i < NE; ++i) { m_[i] *= mdec; v_[i] *= vdec; }
    };
    auto write_back = [&]() {
#pragma unroll
        for (int i = 0; i < NE; ++i) {
            const int o = tid + 256 * i;
            if (o < KD) {
                mu_c[o] = p_[i];
                exp_avg[(size_t)c * KD + o] = m_[i];
                exp_avg_sq[(size_t)c * KD + o] = v_[i];
            }
        }
    };

    if (ord < 0) {                                   // inactive class: it only takes everybody's zero-gradient steps
        if (rank == 0) {
            replay(step0, L * n_active);
            write_back();
        }
        return;
    }
    replay(step0, L * ord);

    // sigma-derived constants (sigma does not change)
    bool same = true;
    for (int i = tid; i < KD; i += 256) same = same && (sg_c[i] == sg_c[(i / D) * D]);
    const bool iso = __syncthreads_and(same ? 1 : 0) != 0;
    for (int i = tid; i < K2 * D; i += 256) {
        const int k = i / D, d = i - k * D;
        s_ri[k * DP + d] = (k < K) ? 1.0f / (sg_c[i] + EM_EPS) : 0.f;                  // ref :333
    }
    for (int k = warp; k < K2; k += 8) {
        float ls = 0.f;
        if (k < K)
            for (int d = lane; d < D; d += 32) ls += logf(sg_c[k * D + d] + EM_EPS);  // ref :334
        ls = warp_sum(ls);
        if (lane == 0) {
            const float r0 = (k < K) ? 1.0f / (sg_c[k * D] + EM_EPS) : 0.f;
            s_ls[k] = ls;
            s_w[k] = r0 * r0;
            s_pi[k] = (k < K) ? weight[(size_t)c * P + c * K + k] : 0.f;
        }
    }
#pragma unroll
    for (int i = 0; i < NE; ++i) {
        const int o = tid + 256 * i;
        if (o < KD) s_mu[o] = p_[i];
    }
    __syncthreads();

    const int per = (cap + 1) / 2;
    const int seg_b = rank * per, seg_e = min(cap, seg_b + per);
    const int row = tid >> 1, half = tid & 1;
    const int pd = tid & (D - 1), pg = tid / D;
    const float inv_den = 1.0f / (1.0f + (float)K * alpha);
    const unsigned sx_addr = (unsigned)__cvta_generic_to_shared(s_x);
    const float n_rows = (float)cap;
    const float div_scale = -4.0f * lamda / ((float)K * (float)(K - 1));

    for (int loop = 0; loop < L; ++loop) {
        // packed means and per-component constants from the current state
        for (int i = tid; i < K2 * D; i += 256) {
            const int k = i / D, d = i - k * D;
            float av = 0.f;
            if (k < K) {
                const float rv = s_ri[k * DP + d];
                av = iso ? -2.0f * rv * rv * s_mu[i] : s_mu[i];
            }
            s_a[k * DP + d] = av;
        }
        for (int k = warp; k < K2; k += 8) {
            float mm = 0.f;
            if (k < K)
                for (int d = lane; d < D; d += 32) mm = fmaf(s_mu[k * D + d], s_mu[k * D + d], mm);
            mm = warp_sum(mm);
            if (lane == 0)
                s_cst[k] = (k < K) ? -0.5f * (float)D * MGP_LOG_2PI - s_ls[k] + logf(s_pi[k] + EM_EPS) -
                                         (iso ? 0.5f * s_w[k] * mm : 0.f)
                                   : 0.f;
        }
        __syncthreads();

        float a1[K2], s0[KH];
#pragma unroll
        for (int i = 0; i < K2; ++i) a1[i] = 0.f;
#pragma unroll
        for (int i = 0; i < KH; ++i) s0[i] = 0.f;
        for (int r0 = seg_b; r0 < seg_e; r0 += rbf) {
            const int nr = min(rbf, seg_e - r0);
            const float* src = bank + ((size_t)c * cap + r0) * D;
            for (int q = tid; q < nr * D4; q += 256) {
                const int rr = q / D4, c4 = q - rr * D4;
                asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sx_addr + (unsigned)(rr * DP + 4 * c4) * 4u),
                             "l"(src + (size_t)q * 4)
                             : "memory");
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
            asm volatile("cp.async.wait_group 0;" ::: "memory");
            __syncthreads();
            if (warp * 16 < nr) {
                const float* xr = s_x + min(row, nr - 1) * DP;
                const float* ar = s_a + half * KH * DP;
                const float* rr_ = s_ri + half * KH * DP;
                float acc[KH], xx = 0.f;
#pragma unroll
                for (int i = 0; i < KH; ++i) acc[i] = 0.f;
                if (iso) {
                    // paired FMAs (FFMA2): even / odd dims accumulate separately and are added at the end
                    float2 acc2[KH], xx2 = make_float2(0.f, 0.f);
#pragma unroll
                    for (int i = 0; i < KH; ++i) acc2[i] = make_float2(0.f, 0.f);
#pragma unroll 4
                    for (int j = 0; j < D4; ++j) {
                        const float4 xv = *reinterpret_cast<const float4*>(xr + 4 * j);
                        const float2 x01 = make_float2(xv.x, xv.y), x23 = make_float2(xv.z, xv.w);
                        xx2 = ffma2(x01, x01, xx2);
                        xx2 = ffma2(x23, x23, xx2);
#pragma unroll
                        for (int i = 0; i < KH; ++i) {
                            const float4 m = *reinterpret_cast<const float4*>(ar + i * DP + 4 * j);
                            acc2[i] = ffma2(x01, make_float2(m.x, m.y), acc2[i]);
                            acc2[i] = ffma2(x23, make_float2(m.z, m.w), acc2[i]);
                        }
                    }
                    xx = xx2.x + xx2.y;
#pragma unroll
                    for (int i = 0; i < KH; ++i) acc[i] = acc2[i].x + acc2[i].y;
                } else {
#pragma unroll 2
                    for (int j = 0; j < D4; ++j) {
                        const float4 xv = *reinterpret_cast<const float4*>(xr + 4 * j);
#pragma unroll
                        for (int i = 0; i < KH; ++i) {
                            const float4 m = *reinterpret_cast<const float4*>(ar + i * DP + 4 * j);
                            const float4 ri = *reinterpret_cast<const float4*>(rr_ + i * DP + 4 * j);
                            float t;
                            t = (xv.x - m.x) * ri.x; acc[i] = fmaf(t, t, acc[i]);
                            t = (xv.y - m.y) * ri.y; acc[i] = fmaf(t, t, acc[i]);
                            t = (xv.z - m.z) * ri.z; acc[i] = fmaf(t, t, acc[i]);
                            t = (xv.w - m.w) * ri.w; acc[i] = fmaf(t, t, acc[i]);
                        }
                    }
                }
                float wl[KH], mx = -INFINITY;
#pragma unroll
                for (int i = 0; i < KH; ++i) {
                    const int k = half * KH + i;
                    const float q = iso ? fmaf(s_w[k], xx, acc[i]) : acc[i];
                    wl[i] = (k < K) ? s_cst[k] - 0.5f * q : -INFINITY;                // ref :316
                    mx = fmaxf(mx, wl[i]);
                }
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                float se = 0.f;
#pragma unroll
                for (int i = 0; i < KH; ++i) {
                    wl[i] = (half * KH + i < K) ? expf(wl[i] - mx) : 0.f;
                    se += wl[i];
                }
                se += __shfl_xor_sync(0xffffffffu, se, 1);
                const float inv_se = 1.0f / se;
                const bool live = row < nr;
#pragma unroll
                for (int i = 0; i < KH; ++i) {
                    const int k = half * KH + i;
                    const float r = (k < K && live) ? fmaf(wl[i], inv_se, alpha) * inv_den : 0.f;   // ref :380-383
                    s0[i] += r;
                    if (live) s_r[row * RS + k] = r;
                }
            }
            __syncthreads();
            {
                const int per_g = (nr + G - 1) / G;
                const int rb = pg * per_g, re = min(nr, rb + per_g);
#pragma unroll 2
                for (int rl = rb; rl < re; ++rl) {
                    const float xv = s_x[rl * DP + pd];
                    float rv[RS];
#pragma unroll
                    for (int i = 0; i < RS / 4; ++i)
                        *reinterpret_cast<float4*>(rv + 4 * i) = *reinterpret_cast<const float4*>(s_r + rl * RS + 4 * i);
                    const float2 xd = make_float2(xv, xv);
#pragma unroll
                    for (int q = 0; q < K2 / 2; ++q) {          // FFMA2: two components per issue slot
                        const float2 t = ffma2(make_float2(rv[2 * q], rv[2 * q + 1]), xd, make_float2(a1[2 * q], a1[2 * q + 1]));
                        a1[2 * q] = t.x;
                        a1[2 * q + 1] = t.y;
                    }
                }
            }
            __syncthreads();
        }
        // this CTA's partial sums -> s_x: [0,K) S0, [K, K+KD) S1 (group combine staged behind them)
#pragma unroll
        for (int i = 0; i < KH; ++i) {
#pragma unroll
            for (int o = 2; o < 32; o <<= 1) s0[i] += __shfl_xor_sync(0xffffffffu, s0[i], o);
            if (lane < 2) s_red[warp * K2 + lane * KH + i] = s0[i];
        }
        float part1[NE];
        // group combine: each group writes its a1 to its own slice, then owners sum the slices
        float* gsl = s_x + ((K + KD + 3) & ~3);                   // [G][K2][D]
#pragma unroll
        for (int i = 0; i < K2; ++i) gsl[(pg * K2 + i) * D + pd] = a1[i];
        __syncthreads();
        if (tid < K) {
            float t = 0.f;
#pragma unroll
            for (int w = 0; w < 8; ++w) t += s_red[w * K2 + tid];
            s_x[tid] = t;
        }
#pragma unroll
        for (int i = 0; i < NE; ++i) {
            const int o = tid + 256 * i;
            part1[i] = 0.f;
            if (o < KD) {
                const int k = o / D, d = o - k * D;
                float t = 0.f;
#pragma unroll
                for (int g = 0; g < G; ++g) t += gsl[(g * K2 + k) * D + d];
                part1[i] = t;
                s_x[K + o] = t;
            }
        }
        cluster.sync();                                           // both partials are published
        const float* rem = cluster.map_shared_rank(s_x, rank ^ 1);
        float s1_[NE];
#pragma unroll
        for (int i = 0; i < NE; ++i) {
            const int o = tid + 256 * i;
            s1_[i] = 0.f;
            if (o < KD) {
                const float other = rem[K + o];
                s1_[i] = (rank == 0) ? part1[i] + other : other + part1[i];   // split 0 + split 1, as em_update_kernel sums them
            }
        }
        if (tid < K) {
            const float mine = s_x[tid], other = rem[tid];
            s_s0[tid] = (rank == 0) ? mine + other : other + mine;
        }
        // diversity kernel on the current means (ref utils/helpers.py:13-14, model.py:390-392)
        for (int pr = warp; pr < K * K; pr += 8) {
            const int i = pr / K, j = pr - i * K;
            float t = 0.f;
            for (int d = lane; d < D; d += 32) {
                const float df = s_mu[i * D + d] - s_mu[j * D + d];
                t = fmaf(df, df, t);
            }
            t = warp_sum(t);
            if (lane == 0) s_e[pr] = (i == j) ? 0.f : expf(-t);
        }
        if (tid == 0) {
            const double stp = (double)(step0 + L * ord + loop + 1);
            s_adam[0] = (float)(adam.lr / (1.0 - pow(adam.beta1, stp)));
            s_adam[1] = (float)sqrt(1.0 - pow(adam.beta2, stp));
        }
        cluster.sync();                                           // the partner has read my partials; s_s0 / s_e / s_adam visible
        // Adam's bias corrections of this step (torch: double), computed once per CTA
        const float step_size = s_adam[0], bc2_sqrt = s_adam[1];
        float newp[NE];
#pragma unroll
        for (int i = 0; i < NE; ++i) {
            const int o = tid + 256 * i;
            newp[i] = p_[i];
            if (o >= KD) continue;
            const int k = o / D, d = o - k * D;
            const float sg = sg_c[o] + EM_EPS;
            const float w = 1.0f / (sg * sg);
            const float muv = s_mu[o];
            float g = -(s1_[i] - muv * s_s0[k]) * w / n_rows;                 // SURVEY KA6
            float esum = 0.f, emu = 0.f;
            for (int j = 0; j < K; ++j) {
                const float e = s_e[k * K + j];
                esum += e;
                emu = fmaf(e, s_mu[j * D + d], emu);
            }
            g += div_scale * (esum * muv - emu);
            // torch.optim.Adam (_single_tensor_adam): lerp, mul/addcmul
            const float mm = m_[i] + (g - m_[i]) * adam.omb1;
            const float vv = v_[i] * adam.b2f + adam.omb2 * g * g;
            const float denom = sqrtf(vv) / bc2_sqrt + adam.epsf;
            newp[i] = muv - step_size * (mm / denom);
            m_[i] = mm; v_[i] = vv;
        }
        __syncthreads();                                          // every reader of the old means is done
#pragma unroll
        for (int i = 0; i < NE; ++i) {
            const int o = tid + 256 * i;
            p_[i] = newp[i];
            if (o < KD) s_mu[o] = newp[i];
        }
        if (tid < K) s_pi[tid] = tau * s_pi[tid] + omtau * ((s_s0[tid] + EM_EPS) / n_rows);   // ref :385, :399
        __syncthreads();
    }
    replay(step0 + L * (ord + 1), L * (n_active - ord - 1));
    if (rank == 0) {
        write_back();
        if (tid < K) weight[(size_t)c * P + (size_t)c * K + tid] = s_pi[tid];
    }
}

// grid C, block 256.  See the file header for the phases.
__global__ void __launch_bounds__(256)
em_update_kernel(const float* __restrict__ stats, int n_split, size_t stat_stride, int n_rows_total,
                 const int32_t* __restrict__ order, const int32_t* __restrict__ sched, float* __restrict__ mu,
                 const float* __restrict__ sigma, float* __restrict__ weight, float* __restrict__ exp_avg,
                 float* __restrict__ exp_avg_sq, int em_loop, int num_em_loop, int phase, AdamCfg adam, float tau,
                 float omtau, float lamda, float* __restrict__ grad_out, int only_class, int C, int K, int D) {
    const int c = blockIdx.x;
    const int ord = order[c];
    const int n_active = sched[0];
    const int step0 = sched[1];
    const int tid = threadIdx.x;
    const int KD = K * D;
    const int P = C * K;
    float* mu_c = mu + (size_t)c * KD;
    const bool do_adam = (exp_avg != nullptr);

    if (phase != 1) {
        if (!do_adam) return;
        int first, count;   // steps first+1 .. first+count are zero-gradient steps of this class
        if (phase == 0) {
            first = step0;
            count = (ord >= 0) ? num_em_loop * ord : num_em_loop * n_active;
        } else {
            if (ord < 0) return;
            first = step0 + num_em_loop * (ord + 1);
            count = num_em_loop * (n_active - ord - 1);
        }
        if (count <= 0) return;
        // With g = 0 Adam's moments just decay: m_s = b1^s m_0, v_s = b2^s v_0, and
        //   p <- p - [lr b1^s / (1 - b1^(first+s))] * m_0 / (sqrt(v_0) * b2^(s/2) / sqrt(1 - b2^(first+s)) + eps).
        // The bracketed scalars c_s, d_s are the same for every element: tabulate them in shared memory
        // (double precision pow once per step), then each element costs one FMA + one reciprocal per step.
        extern __shared__ float sm[];
        constexpr int TAB = 2048;
        float* s_c = sm;            // [TAB]
        float* s_d = sm + TAB;      // [TAB]
        float p_[8], a_[8], m0_[8];
        for (int ob = 0; ob < KD; ob += 256 * 8) {
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int o = ob + tid + 256 * i;
                p_[i] = 0.f; m0_[i] = 0.f; a_[i] = 1.f;
                if (o < KD) {
                    p_[i] = mu_c[o];
                    m0_[i] = exp_avg[(size_t)c * KD + o];
                    a_[i] = sqrtf(exp_avg_sq[(size_t)c * KD + o]);
                }
            }
            // explicit terms up to beta1^s < 1e-3, the rest as one geometric tail term (replay_explicit_steps /
            // replay_tail above); the moments decay by the full `count`
            const int count_p = replay_explicit_steps(count, first, (float)adam.beta1);
            __shared__ float s_tail[2];
            for (int s0 = 0; s0 < count_p; s0 += TAB) {
                const int ns = min(TAB, count_p - s0);
                __syncthreads();
                for (int s = tid; s < ns; s += 256) replay_coeffs(adam, first, s0 + s + 1, s_c[s], s_d[s]);
                if (tid == 255 && s0 + TAB >= count_p && count > count_p)
                    replay_tail(adam, first, count_p, count, s_tail[0], s_tail[1]);
                __syncthreads();
                const int nel = min(8, (KD - ob + 255) / 256);         // elements this thread row actually owns
                // one FMA + one MUFU.RCP + FMUL + FMA per (step, element); the element count is a compile-time
                // constant of each branch (padding slots have m0 = 0, a = 1)
#define MGP_REPLAY(NEL)                                                                                              \
    for (int s = 0; s < ns; ++s) {                                                                                  \
        const float cs = -s_c[s], ds = s_d[s];                                                                      \
        _Pragma("unroll") for (int i = 0; i < NEL; ++i) {                                                           \
            float rc;                                                                                               \
            asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(fmaf(a_[i], ds, adam.epsf)));                          \
            p_[i] = fmaf(cs * m0_[i], rc, p_[i]);                                                                   \
        }                                                                                                           \
    }
                if (nel <= 3) { MGP_REPLAY(3) }
                else if (nel <= 5) { MGP_REPLAY(5) }
                else { MGP_REPLAY(8) }
#undef MGP_REPLAY
            }
            if (count > count_p) {                   // steps count_p+1 .. count in one term (see replay_tail)
                const float cs = -s_tail[0], ds = s_tail[1];
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    float rc;
                    asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(rc) : "f"(fmaf(a_[i], ds, adam.epsf)));
                    p_[i] = fmaf(cs * m0_[i], rc, p_[i]);
                }
            }
            const float mdec = (float)pow(adam.beta1, (double)count);
            const float vdec = (float)pow(adam.beta2, (double)count);
#pragma unroll
            for (int i = 0; i < 8; ++i) {
                const int o = ob + tid + 256 * i;
                if (o < KD) {
                    mu_c[o] = p_[i];
                    exp_avg[(size_t)c * KD + o] = m0_[i] * mdec;
                    exp_avg_sq[(size_t)c * KD + o] *= vdec;
                }
            }
        }
        return;
    }

    // phase 1: one EM-loop step of an active class
    if (ord < 0) return;
    if (only_class >= 0 && c != only_class) return;
    extern __shared__ float sm1[];
    float* s_mu = sm1;              // [K][D]
    float* s_e = s_mu + KD;         // [K][K] exp(-|mu_i - mu_j|^2)
    float* s_s0 = s_e + K * K;      // [K]
    const int lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < KD; i += 256) s_mu[i] = mu_c[i];
    for (int k = tid; k < K; k += 256) {
        float t = 0.f;
        for (int s = 0; s < n_split; ++s) t += stats[((size_t)c * n_split + s) * stat_stride + k];
        s_s0[k] = t;
    }
    __syncthreads();
    for (int pr = warp; pr < K * K; pr += 8) {      // ref utils/helpers.py:13-14, model.py:390-392
        const int i = pr / K, j = pr - i * K;
        float t = 0.f;
        for (int d = lane; d < D; d += 32) {
            const float df = s_mu[i * D + d] - s_mu[j * D + d];
            t = fmaf(df, df, t);
        }
        t = warp_sum(t);
        if (lane == 0) s_e[pr] = (i == j) ? 0.f : expf(-t);
    }
    __syncthreads();
    const float n_rows = (float)n_rows_total;
    // K = 1 has no prototype pairs: no diversity term (the reference's mean over the empty pair set is 0/0, NaN)
    const float div_scale = (K > 1) ? -4.0f * lamda / ((float)K * (float)(K - 1)) : 0.f;
    const int step = step0 + num_em_loop * ord + em_loop + 1;
    const double b1p = pow(adam.beta1, (double)step), b2p = pow(adam.beta2, (double)step);
    // all global operands of up to 8 owned elements are fetched before any is used (the kernel is a chain of
    // cold-miss latencies otherwise: ncu long_scoreboard 5.6 per issue)
    for (int ob = 0; ob < KD; ob += 256 * 8) {
        float s1_[8], sg_[8], m_[8], v_[8];
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int o = ob + tid + 256 * i;
            s1_[i] = 0.f; sg_[i] = 1.f; m_[i] = 0.f; v_[i] = 0.f;
            if (o < KD) {
                for (int sp = 0; sp < n_split; ++sp) s1_[i] += stats[((size_t)c * n_split + sp) * stat_stride + K + o];
                sg_[i] = sigma[(size_t)c * KD + o];
                if (do_adam) {
                    m_[i] = exp_avg[(size_t)c * KD + o];
                    v_[i] = exp_avg_sq[(size_t)c * KD + o];
                }
            }
        }
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int o = ob + tid + 256 * i;
            if (o >= KD) continue;
            const int k = o / D, d = o - k * D;
            const float sg = sg_[i] + EM_EPS;
            const float w = 1.0f / (sg * sg);
            const float muv = s_mu[o];
            float g = -(s1_[i] - muv * s_s0[k]) * w / n_rows;                 // SURVEY KA6
            float esum = 0.f, emu = 0.f;
            for (int j = 0; j < K; ++j) {
                const float e = s_e[k * K + j];
                esum += e;
                emu = fmaf(e, s_mu[j * D + d], emu);
            }
            g += div_scale * (esum * muv - emu);
            if (grad_out) grad_out[(size_t)c * KD + o] = g;
            if (do_adam) {
                float p = muv, m = m_[i], v = v_[i];
                adam_apply(p, m, v, g, adam, b1p, b2p);
                mu_c[o] = p;
                exp_avg[(size_t)c * KD + o] = m;
                exp_avg_sq[(size_t)c * KD + o] = v;
            }
        }
    }
    // pi <- tau*pi + (1-tau)*(S0 + eps)/n   (ref :385, :399, :297-298)
    for (int k = tid; k < K; k += 256) {
        float* wp = weight + (size_t)c * P + (size_t)c * K + k;
        const float pi_new = (s_s0[k] + EM_EPS) / n_rows;
        *wp = tau * (*wp) + omtau * pi_new;
    }
}

// ---------------------------------------------------------------------------------------------
// E-step on explicit rows (API parity for _e_step / _score).  Warp per row.
template <int VEC4>
__global__ void __launch_bounds__(256)
em_estep_kernel(const float* __restrict__ x, const float* __restrict__ mu, const float* __restrict__ sigma,
                const float* __restrict__ pi, float* __restrict__ log_resp, float* __restrict__ score, int n, int K,
                int D) {
    extern __shared__ __align__(16) float sm[];
    float* s_mu = sm;
    float* s_rinv = s_mu + K * D;
    float* s_cst = s_rinv + K * D;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    for (int i = tid; i < K * D; i += 256) {
        s_mu[i] = mu[i];
        s_rinv[i] = 1.0f / (sigma[i] + EM_EPS);
    }
    __syncthreads();
    for (int k = warp; k < K; k += 8) {
        float ls = 0.f;
        for (int d = lane; d < D; d += 32) ls += logf(sigma[k * D + d] + EM_EPS);
        ls = warp_sum(ls);
        if (lane == 0) s_cst[k] = -0.5f * (float)D * MGP_LOG_2PI - ls + logf(pi[k] + EM_EPS);
    }
    __syncthreads();
    for (int row = blockIdx.x * 8 + warp; row < n; row += gridDim.x * 8) {
        float4 xv[VEC4];
#pragma unroll
        for (int j = 0; j < VEC4; ++j) {
            xv[j] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (4 * (lane + 32 * j) < D) xv[j] = __ldg(reinterpret_cast<const float4*>(x + (size_t)row * D) + lane + 32 * j);
        }
        float r_lo, r_hi, l_lo, l_hi;
        const float norm = warp_estep_row<VEC4>(xv, s_mu, s_rinv, s_cst, K, D, lane, 0.f, r_lo, r_hi, l_lo, l_hi);
        if (log_resp) {
            if (lane < K) log_resp[(size_t)row * K + lane] = l_lo;
            if (lane + 32 < K) log_resp[(size_t)row * K + lane + 32] = l_hi;
        }
        if (score && lane == 0) score[row] = norm;
    }
}

// closed-form M-step (ref :338-365): thread per (k,d), serial over rows.
__global__ void em_mstep_closed_kernel(const float* __restrict__ x, const float* __restrict__ log_resp, float alpha,
                                       float* __restrict__ pi_out, float* __restrict__ mu_out,
                                       float* __restrict__ sigma_out, int n, int K, int D) {
    const int o = blockIdx.x * blockDim.x + threadIdx.x;
    if (o >= K * D) return;
    const int k = o / D, d = o - k * D;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int r = 0; r < n; ++r) {
        float den = 0.f;
        for (int j = 0; j < K; ++j) den += expf(log_resp[(size_t)r * K + j]) + alpha;
        const float rr = (expf(log_resp[(size_t)r * K + k]) + alpha) / den;
        const float xx = x[(size_t)r * D + d];
        s0 += rr;
        s1 = fmaf(rr, xx, s1);
        s2 = fmaf(rr * xx, xx, s2);
    }
    const float pi = s0 + EM_EPS;
    const float m = s1 / pi;
    const float x2 = s2 / pi;
    const float xmu = m * s1 / pi;
    const float var = x2 - 2.0f * xmu + m * m + EM_EPS;
    mu_out[o] = m;
    sigma_out[o] = sqrtf(var);
    if (d == 0) pi_out[k] = pi / (float)n;
}

}  // namespace

extern "C" size_t mgp_em_stat_stride(int K, int D, int with_s2) {
    return (size_t)K + (size_t)K * D * (with_s2 ? 2 : 1) + 1;
}

extern "C" int mgp_em_plan(uint8_t* updated, const int64_t* mem_len, int32_t* order, int32_t* sched,
                           int32_t* adam_step, int step0, int C, int cap, int num_em_loop, void* stream) {
    if (!updated || !mem_len || !order || !sched || C <= 0 || cap <= 0 || num_em_loop <= 0) return MGP_ERR_INVALID;
    em_plan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(updated, mem_len, order, sched, adam_step, step0, C, cap,
                                                         num_em_loop, make_adam(1.0, 0.9, 0.999, 1e-8), nullptr);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

template <int VEC4, bool S2>
static int launch_stats(int nout, dim3 grid, size_t smem, cudaStream_t st, const float* bank, const int32_t* order,
                        const float* mu, const float* sigma, const float* weight, float alpha, int rb, int re,
                        int n_split, float* stats, size_t stride, int C, int K, int D, int cap) {
#define MGP_EM_CASE(NO)                                                                                             \
    if (nout <= NO) {                                                                                               \
        MGP_CUDA(cudaFuncSetAttribute(em_stats_kernel<VEC4, NO, S2>, cudaFuncAttributeMaxDynamicSharedMemorySize,   \
                                      (int)smem));                                                                  \
        em_stats_kernel<VEC4, NO, S2><<<grid, 256, smem, st>>>(bank, order, mu, sigma, weight, alpha, rb, re,       \
                                                               n_split, stats, stride, C, K, D, cap);               \
        MGP_CHECK_LAUNCH();                                                                                         \
        return MGP_OK;                                                                                              \
    }
    MGP_EM_CASE(2)
    MGP_EM_CASE(5)
    MGP_EM_CASE(10)
    MGP_EM_CASE(20)
    MGP_EM_CASE(40)
    MGP_EM_CASE(80)
#undef MGP_EM_CASE
    return MGP_ERR_UNSUPPORTED;
}

extern "C" int mgp_em_stats(const float* bank, const int32_t* order, const float* mu, const float* sigma,
                            const float* weight_cp, float alpha, int row_begin, int row_end, int n_split, int with_s2,
                            float* stats, int C, int K, int D, int cap, void* stream) {
    if (!bank || !order || !mu || !sigma || !weight_cp || !stats) return MGP_ERR_INVALID;
    if (C <= 0 || K <= 0 || D <= 0 || cap <= 0 || n_split <= 0 || row_begin < 0 || row_end > cap || row_begin >= row_end)
        return MGP_ERR_INVALID;
    if (K > 64 || (D % 4) != 0 || D > 512) return MGP_ERR_UNSUPPORTED;
    const size_t stride = mgp_em_stat_stride(K, D, with_s2);
    static const bool legacy = (getenv("MGP_EM_LEGACY") != nullptr);
    if (!legacy && K <= 16 && (D == 64 || D == 128)) {
        const int kh = (K + 1) / 2 <= 3 ? 3 : ((K + 1) / 2 <= 5 ? 5 : 8);
        const int per = (row_end - row_begin + n_split - 1) / n_split;
        const int nb = (per + 127) / 128;
        int rbf = (((per + nb - 1) / nb) + 3) & ~3;
        if (rbf < 32) rbf = 32;
        const int k2 = 2 * kh, rs = (k2 + 3) & ~3, g = 256 / D, dp = D + 4;
        const int xfl = rbf * dp > g * k2 * D ? rbf * dp : g * k2 * D;
        const size_t fsmem = ((size_t)2 * k2 * dp + xfl + (size_t)rbf * rs + 2 * k2 + 8 * k2) * sizeof(float);
        dim3 fgrid(C, n_split);
        cudaStream_t fst = (cudaStream_t)stream;
#define MGP_EM_FAST(DD, KK, SS)                                                                                     \
    if (D == DD && kh == KK && (with_s2 != 0) == SS) {                                                              \
        MGP_CUDA(cudaFuncSetAttribute(em_stats_fast_kernel<DD, KK, SS>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                      (int)fsmem));                                                                 \
        em_stats_fast_kernel<DD, KK, SS><<<fgrid, 256, fsmem, fst>>>(bank, order, mu, sigma, weight_cp, alpha,       \
                                                                     row_begin, row_end, n_split, rbf, stats,       \
                                                                     stride, C, K, cap);                            \
        MGP_CHECK_LAUNCH();                                                                                         \
        return MGP_OK;                                                                                              \
    }
        MGP_EM_FAST(128, 3, false) MGP_EM_FAST(128, 5, false) MGP_EM_FAST(128, 8, false)
        MGP_EM_FAST(64, 3, false) MGP_EM_FAST(64, 5, false) MGP_EM_FAST(64, 8, false)
        MGP_EM_FAST(128, 3, true) MGP_EM_FAST(128, 5, true) MGP_EM_FAST(128, 8, true)
        MGP_EM_FAST(64, 3, true) MGP_EM_FAST(64, 5, true) MGP_EM_FAST(64, 8, true)
#undef MGP_EM_FAST
    }
    const int nout = (K * D + 255) / 256;
    const size_t smem = ((size_t)2 * K * D + (size_t)RB * D + (size_t)RB * K + 2 * K) * sizeof(float);
    if (smem > 220 * 1024) return MGP_ERR_UNSUPPORTED;
    dim3 grid(C, n_split);
    cudaStream_t st = (cudaStream_t)stream;
    const int vec4 = (D + 127) / 128;
#define MGP_EM_V(V)                                                                                                 \
    if (vec4 == V)                                                                                                  \
        return with_s2 ? launch_stats<V, true>(nout, grid, smem, st, bank, order, mu, sigma, weight_cp, alpha,      \
                                               row_begin, row_end, n_split, stats, stride, C, K, D, cap)            \
                       : launch_stats<V, false>(nout, grid, smem, st, bank, order, mu, sigma, weight_cp, alpha,     \
                                                row_begin, row_end, n_split, stats, stride, C, K, D, cap);
    MGP_EM_V(1)
    MGP_EM_V(2)
    MGP_EM_V(3)
    MGP_EM_V(4)
#undef MGP_EM_V
    return MGP_ERR_UNSUPPORTED;
}

extern "C" int mgp_em_update(const float* stats, int n_split, int with_s2, int n_rows_total, const int32_t* order,
                             const int32_t* sched, float* mu, const float* sigma, float* weight_cp, float* exp_avg,
                             float* exp_avg_sq, int em_loop, int num_em_loop, int phase, double lr, double beta1,
                             double beta2, double adam_eps, double tau, float lamda, float* grad_out, int only_class,
                             int C, int K, int D, void* stream) {
    if (!order || !sched || !mu || !sigma || !weight_cp) return MGP_ERR_INVALID;
    if (phase < 0 || phase > 2 || C <= 0 || K <= 0 || D <= 0 || num_em_loop <= 0) return MGP_ERR_INVALID;
    if (phase == 1 && (!stats || n_split <= 0 || n_rows_total <= 0)) return MGP_ERR_INVALID;
    if ((exp_avg == nullptr) != (exp_avg_sq == nullptr)) return MGP_ERR_INVALID;
    const size_t stride = mgp_em_stat_stride(K, D, with_s2);
    size_t smem = ((size_t)K * D + (size_t)K * K + K) * sizeof(float);
    if (smem < 2 * 2048 * sizeof(float)) smem = 2 * 2048 * sizeof(float);
    if (smem > 220 * 1024) return MGP_ERR_UNSUPPORTED;
    MGP_CUDA(cudaFuncSetAttribute(em_update_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const AdamCfg a = make_adam(lr, beta1, beta2, adam_eps);
    em_update_kernel<<<C, 256, smem, (cudaStream_t)stream>>>(stats, n_split, stride, n_rows_total, order, sched, mu,
                                                             sigma, weight_cp, exp_avg, exp_avg_sq, em_loop,
                                                             num_em_loop, phase, a, (float)tau, (float)(1.0 - tau), lamda, grad_out, only_class,
                                                             C, K, D);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

static bool em_fused_applies(int K, int D, int cap) {
    return mgp_opt_em_fused() && K >= 2 && K <= 16 && (D == 64 || D == 128) && cap >= 2;
}

static bool em_tc_applies(int K, int D, int cap, int have_shadow_iso) {
#ifdef MGP_WITH_TC
    return have_shadow_iso && mgp_opt_em_tc() && mgp_em_tc_supported(K, D, cap);
#else
    (void)K; (void)D; (void)cap; (void)have_shadow_iso;
    return false;
#endif
}

extern "C" int mgp_update_gmm_launches(int K, int D, int cap, int num_em_loop, int have_shadow_iso) {
    if (em_tc_applies(K, D, cap, have_shadow_iso)) return 2;         // plan + kernel
    return em_fused_applies(K, D, cap) ? 2 : 3 + 2 * num_em_loop;
}

// shape / resource validation shared by the paths below: nothing is enqueued (and no flag cleared, no step counted)
// for a shape the kernels cannot take
static int em_validate(int C, int K, int D, int cap, int num_em_loop) {
    if (C <= 0 || K <= 0 || D <= 0 || cap <= 0 || num_em_loop <= 0) return MGP_ERR_INVALID;
    if (K > 64 || (D % 4) != 0 || D > 512) return MGP_ERR_UNSUPPORTED;
    if (((size_t)2 * K * D + (size_t)RB * D + (size_t)RB * K + 2 * K) * sizeof(float) > 220 * 1024) return MGP_ERR_UNSUPPORTED;
    return MGP_OK;
}

static bool em_tc_fits(const void* shadow_h, const void* shadow_l, const float* shadow_xx, const int32_t* status,
                       int sigma_iso, int n_split, int num_em_loop, int C, int K, int D, int cap) {
    return shadow_h && shadow_l && shadow_xx && status && em_tc_applies(K, D, cap, sigma_iso) &&
           (size_t)5 * num_em_loop * C + 4 + C <= (size_t)C * n_split * mgp_em_stat_stride(K, D, 0);
}

#ifdef MGP_WITH_TC
// planner + tensor-core kernel (em_tc.cu); mu_stage / pi_stage null: the new means and pi are written in place
static int em_tc_enqueue(const void* shadow_h, const void* shadow_l, const float* shadow_xx, int32_t* status,
                         uint8_t* updated, const int64_t* mem_len, float* mu, const float* sigma, float* weight_cp,
                         float* exp_avg, float* exp_avg_sq, int32_t* adam_step, int32_t* order, int32_t* sched, float* stats,
                         int num_em_loop, float alpha, double lr, double beta1, double beta2, double adam_eps, double tau,
                         float lamda, float* mu_stage, float* pi_stage, int C, int K, int D, int cap, void* stream) {
    // the planner also tabulates the steps' Adam bias corrections into the (otherwise unused) stats scratch
    em_plan_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(updated, mem_len, order, sched, adam_step, 0, C, cap, num_em_loop,
                                                         make_adam(lr, beta1, beta2, adam_eps), stats,
                                                         reinterpret_cast<int32_t*>(stats + (size_t)5 * num_em_loop * C + 4));
    MGP_CHECK_LAUNCH();
    return mgp_em_tc_launch(shadow_h, shadow_l, shadow_xx, stats, order, sched, mu, sigma, weight_cp, exp_avg, exp_avg_sq,
                            status, num_em_loop, alpha, lr, beta1, beta2, adam_eps, tau, lamda, mu_stage, pi_stage, C, K, D,
                            cap, (cudaStream_t)stream);
}
#endif

extern "C" int mgp_update_gmm(const float* bank, const void* shadow_h, const void* shadow_l, const float* shadow_xx,
                              int sigma_iso, int32_t* status, uint8_t* updated, const int64_t* mem_len, float* mu,
                              const float* sigma,
                              float* weight_cp, float* exp_avg, float* exp_avg_sq, int32_t* adam_step, int32_t* order,
                              int32_t* sched, float* stats, int n_split, int num_em_loop, float alpha, double lr,
                              double beta1, double beta2, double adam_eps, double tau, float lamda, int C, int K, int D,
                              int cap, void* stream) {
    if (!bank || !updated || !mem_len || !mu || !sigma || !weight_cp || !exp_avg || !exp_avg_sq || !adam_step ||
        !order || !sched || !stats)
        return MGP_ERR_INVALID;
    int rc = em_validate(C, K, D, cap, num_em_loop);                 // before the planner clears flags / counts steps
    if (rc != MGP_OK) return rc;
#ifdef MGP_WITH_TC
    if (em_tc_fits(shadow_h, shadow_l, shadow_xx, status, sigma_iso, n_split, num_em_loop, C, K, D, cap))
        return em_tc_enqueue(shadow_h, shadow_l, shadow_xx, status, updated, mem_len, mu, sigma, weight_cp, exp_avg,
                             exp_avg_sq, adam_step, order, sched, stats, num_em_loop, alpha, lr, beta1, beta2, adam_eps,
                             tau, lamda, nullptr, nullptr, C, K, D, cap, stream);
#endif
    rc = mgp_em_plan(updated, mem_len, order, sched, adam_step, 0, C, cap, num_em_loop, stream);
    if (rc != MGP_OK) return rc;
    if (em_fused_applies(K, D, cap)) {
        // one cluster of two CTAs per class runs the class's whole timeline (em_fused_kernel)
        const int kh = (K + 1) / 2 <= 3 ? 3 : ((K + 1) / 2 <= 5 ? 5 : 8);
        const int per = (cap + 1) / 2;
        const int nb = (per + 87) / 88;
        int rbf = (((per + nb - 1) / nb) + 3) & ~3;
        if (rbf < 32) rbf = 32;
        const int k2 = 2 * kh, rs = (k2 + 3) & ~3, g = 256 / D, dp = D + 4;
        int xfl = (K + K * D + 3 + g * k2 * D + 3) & ~3;
        if (rbf * dp > xfl) xfl = rbf * dp;
        const size_t fsmem = ((size_t)2 * k2 * dp + xfl + (size_t)rbf * rs + (size_t)k2 * D + 13 * k2 + (size_t)k2 * k2 + 512) *
                             sizeof(float);
        const AdamCfg a = make_adam(lr, beta1, beta2, adam_eps);
        cudaStream_t fst = (cudaStream_t)stream;
#define MGP_EM_FUSED(DD, KK)                                                                                        \
    if (D == DD && kh == KK) {                                                                                      \
        MGP_CUDA(cudaFuncSetAttribute(em_fused_kernel<DD, KK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fsmem)); \
        em_fused_kernel<DD, KK><<<2 * C, 256, fsmem, fst>>>(bank, order, sched, mu, sigma, weight_cp, exp_avg, exp_avg_sq, \
                                                            alpha, rbf, num_em_loop, a, (float)tau, (float)(1.0 - tau), lamda, C, K, cap);     \
        MGP_CHECK_LAUNCH();                                                                                         \
        return MGP_OK;                                                                                              \
    }
        MGP_EM_FUSED(128, 3) MGP_EM_FUSED(128, 5) MGP_EM_FUSED(128, 8)
        MGP_EM_FUSED(64, 3) MGP_EM_FUSED(64, 5) MGP_EM_FUSED(64, 8)
#undef MGP_EM_FUSED
    }
    rc = mgp_em_update(nullptr, n_split, 0, cap, order, sched, mu, sigma, weight_cp, exp_avg, exp_avg_sq, 0, num_em_loop,
                       0, lr, beta1, beta2, adam_eps, tau, lamda, nullptr, -1, C, K, D, stream);
    if (rc != MGP_OK) return rc;
    for (int i = 0; i < num_em_loop; ++i) {
        rc = mgp_em_stats(bank, order, mu, sigma, weight_cp, alpha, 0, cap, n_split, 0, stats, C, K, D, cap, stream);
        if (rc != MGP_OK) return rc;
        rc = mgp_em_update(stats, n_split, 0, cap, order, sched, mu, sigma, weight_cp, exp_avg, exp_avg_sq, i,
                           num_em_loop, 1, lr, beta1, beta2, adam_eps, tau, lamda, nullptr, -1, C, K, D, stream);
        if (rc != MGP_OK) return rc;
    }
    return mgp_em_update(nullptr, n_split, 0, cap, order, sched, mu, sigma, weight_cp, exp_avg, exp_avg_sq, 0,
                         num_em_loop, 2, lr, beta1, beta2, adam_eps, tau, lamda, nullptr, -1, C, K, D, stream);
}

extern "C" int mgp_update_gmm_staged(const void* shadow_h, const void* shadow_l, const float* shadow_xx, int32_t* status,
                                     uint8_t* updated, const int64_t* mem_len, const float* mu, const float* sigma,
                                     const float* weight_cp, float* exp_avg, float* exp_avg_sq, int32_t* adam_step,
                                     int32_t* order, int32_t* sched, float* stats, int n_split, int num_em_loop, float alpha,
                                     double lr, double beta1, double beta2, double adam_eps, double tau, float lamda,
                                     float* mu_stage, float* pi_stage, int C, int K, int D, int cap, void* stream) {
    if (!shadow_h || !shadow_l || !shadow_xx || !status || !updated || !mem_len || !mu || !sigma || !weight_cp ||
        !exp_avg || !exp_avg_sq || !adam_step || !order || !sched || !stats || !mu_stage || !pi_stage || n_split <= 0)
        return MGP_ERR_INVALID;
    const int rc = em_validate(C, K, D, cap, num_em_loop);
    if (rc != MGP_OK) return rc;
    if (mu_stage == mu || (const float*)pi_stage == weight_cp) return MGP_ERR_INVALID;
#ifdef MGP_WITH_TC
    if (em_tc_fits(shadow_h, shadow_l, shadow_xx, status, 1, n_split, num_em_loop, C, K, D, cap))
        // the kernel only reads mu and weight_cp (the staged outputs take the writes)
        return em_tc_enqueue(shadow_h, shadow_l, shadow_xx, status, updated, mem_len, const_cast<float*>(mu), sigma,
                             const_cast<float*>(weight_cp), exp_avg, exp_avg_sq, adam_step, order, sched, stats,
                             num_em_loop, alpha, lr, beta1, beta2, adam_eps, tau, lamda, mu_stage, pi_stage, C, K, D, cap,
                             stream);
#endif
    return MGP_ERR_UNSUPPORTED;                                      // nothing enqueued: no flag cleared, no step counted
}

namespace {
// mu <- mu_stage (float4), and pi_stage [C,K] into weight_cp's class-diagonal blocks
__global__ void __launch_bounds__(256)
em_commit_kernel(const float4* __restrict__ mu_stage, const float* __restrict__ pi_stage, float4* __restrict__ mu,
                 float* __restrict__ weight_cp, int n4, int C, int K) {
    const int stride = gridDim.x * blockDim.x;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += stride) mu[i] = mu_stage[i];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < C * K; i += stride) {
        const int c = i / K;
        weight_cp[(size_t)c * C * K + i] = pi_stage[i];             // row c, column c K + k
    }
}
}  // namespace

extern "C" int mgp_em_commit(const float* mu_stage, const float* pi_stage, float* mu, float* weight_cp, int C, int K, int D,
                             void* stream) {
    if (!mu_stage || !pi_stage || !mu || !weight_cp || C <= 0 || K <= 0 || D <= 0 || (D & 3)) return MGP_ERR_INVALID;
    if (!mgp_aligned16(mu_stage) || !mgp_aligned16(mu)) return MGP_ERR_INVALID;
    if ((long long)C * K * D > 0x7fffffffLL) return MGP_ERR_UNSUPPORTED;
    const int n4 = C * K * D / 4;
    int blocks = (n4 + 255) / 256;
    if (blocks > 1024) blocks = 1024;
    em_commit_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4*>(mu_stage), pi_stage,
                                                               reinterpret_cast<float4*>(mu), weight_cp, n4, C, K);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" int mgp_em_estep(const float* x, const float* mu, const float* sigma, const float* pi, float* log_resp,
                            float* score, int n, int K, int D, void* stream) {
    if (!x || !mu || !sigma || !pi || n <= 0 || K <= 0 || D <= 0) return MGP_ERR_INVALID;
    if (K > 64 || (D % 4) != 0 || D > 512) return MGP_ERR_UNSUPPORTED;
    const size_t smem = ((size_t)2 * K * D + K) * sizeof(float);
    if (smem > 220 * 1024) return MGP_ERR_UNSUPPORTED;
    int sms = 0;
    MGP_CUDA(mgp_sm_count(&sms));
    int grid = (n + 7) / 8;
    if (grid > sms * 8) grid = sms * 8;
    cudaStream_t st = (cudaStream_t)stream;
#define MGP_ES(V)                                                                                                   \
    if ((D + 127) / 128 == V) {                                                                                           \
        MGP_CUDA(cudaFuncSetAttribute(em_estep_kernel<V>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        em_estep_kernel<V><<<grid, 256, smem, st>>>(x, mu, sigma, pi, log_resp, score, n, K, D);                    \
        MGP_CHECK_LAUNCH();                                                                                         \
        return MGP_OK;                                                                                              \
    }
    MGP_ES(1)
    MGP_ES(2)
    MGP_ES(3)
    MGP_ES(4)
#undef MGP_ES
    return MGP_ERR_UNSUPPORTED;
}

extern "C" int mgp_em_mstep_closed(const float* x, const float* log_resp, float alpha, float* pi_out, float* mu_out,
                                   float* sigma_out, int n, int K, int D, void* stream) {
    if (!x || !log_resp || !pi_out || !mu_out || !sigma_out || n <= 0 || K <= 0 || D <= 0) return MGP_ERR_INVALID;
    const int tot = K * D;
    em_mstep_closed_kernel<<<(tot + 127) / 128, 128, 0, (cudaStream_t)stream>>>(x, log_resp, alpha, pi_out, mu_out,
                                                                                sigma_out, n, K, D);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}
