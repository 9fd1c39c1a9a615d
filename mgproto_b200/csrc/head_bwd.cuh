// The head backward's body (entry compaction, stable sort by patch row, balanced walk, direct row writes), shared by
// head_bwd_kernel (head.cu) and the long-map kernels (head_long.cu).
#pragma once
#include "mgp_common.cuh"
#include <type_traits>

namespace {

constexpr int LCAP = 2304;   // entries per drain (>= P + K(T-1) of the labelled cfg: one drain per image)

// grid (B, D/DC), DC = 32 VEC (VEC = 4 floats per lane when D is a multiple of 128: ONE CTA per image at D = 128, so the
// list is built and sorted once; VEC = 2 otherwise): CTA (b, j) produces dims [DC j, DC j + DC) of image b's rows of
// g_xhat (zeroed by the caller).  Entries with gradient are compacted in a fixed order, stably counting-sorted by patch row, then each
// warp walks one eighth of the sorted list with lanes owning two dims each (see the walk below) and adds every
// finished row straight into global memory (a row has exactly one writer per drain): balanced however the mined
// patches cluster, no atomics, fixed summation order, 48 KB of shared memory -> 4 CTAs per SM.
template <int VEC> struct LaneVec { float v[VEC]; };
template <int VEC>
__device__ __forceinline__ LaneVec<VEC> lv_ldg(const float* p) {
    LaneVec<VEC> r;
    if constexpr (VEC == 4) { const float4 t = __ldg(reinterpret_cast<const float4*>(p)); r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w; }
    else { const float2 t = __ldg(reinterpret_cast<const float2*>(p)); r.v[0] = t.x; r.v[1] = t.y; }
    return r;
}
template <int VEC>
__device__ __forceinline__ LaneVec<VEC> lv_ldcg(const float* p) {
    LaneVec<VEC> r;
    if constexpr (VEC == 4) { const float4 t = __ldcg(reinterpret_cast<const float4*>(p)); r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w; }
    else { const float2 t = __ldcg(reinterpret_cast<const float2*>(p)); r.v[0] = t.x; r.v[1] = t.y; }
    return r;
}
template <int VEC>
__device__ __forceinline__ LaneVec<VEC> lv_ld(const float* p) {
    LaneVec<VEC> r;
    if constexpr (VEC == 4) { const float4 t = *reinterpret_cast<const float4*>(p); r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w; }
    else { const float2 t = *reinterpret_cast<const float2*>(p); r.v[0] = t.x; r.v[1] = t.y; }
    return r;
}
template <int VEC>
__device__ __forceinline__ void lv_st(float* p, const LaneVec<VEC>& r) {
    if constexpr (VEC == 4) *reinterpret_cast<float4*>(p) = make_float4(r.v[0], r.v[1], r.v[2], r.v[3]);
    else *reinterpret_cast<float2*>(p) = make_float2(r.v[0], r.v[1]);
}
template <int VEC>
__device__ __forceinline__ LaneVec<VEC> lv_zero() {
    LaneVec<VEC> r;
#pragma unroll
    for (int i = 0; i < VEC; ++i) r.v[i] = 0.f;
    return r;
}

// LONG = false: head_bwd_kernel, HW <= 1024, entry key p*1024 + n, one counting-sort pass over [8][HW] row histograms.
// LONG = true : head_bwd_long_v{2,4}_kernel, HW <= 4096, entry key p*4096 + n, the 12-bit row sorted by two stable
//               64-bin counting passes (low 6 bits, then high 6 bits) over [8][64] histograms: shared memory does not
//               grow with HW, and the sorted list -- rows ascending, list order inside a row -- is the one the single
//               pass gives, so the walk below sums every row in the same order.
template <int VEC, bool LONG>
__device__ __forceinline__ void
head_bwd_body(const float* __restrict__ gl, const float* __restrict__ logits, const float* __restrict__ vals,
              const int32_t* __restrict__ idx, const float* __restrict__ weight, const int64_t* __restrict__ gt,
              const float* __restrict__ xhat, const float* __restrict__ w, const float* __restrict__ wm,
              const float* __restrict__ wsc, const int* __restrict__ noniso, float* __restrict__ g_xhat, int HW,
              int C, int K, int D, int T) {
    constexpr int DC = 32 * VEC;
    constexpr unsigned KS = LONG ? 12u : 10u;                // entry key = p << KS | n
    constexpr unsigned KM = (1u << KS) - 1u;
    using LV = LaneVec<VEC>;
    extern __shared__ float smem[];
    const bool aniso = (*noniso != 0);
    unsigned* lkey = reinterpret_cast<unsigned*>(smem);     // [LCAP] p*1024 + n
    float* lval = reinterpret_cast<float*>(lkey + LCAP);    // [LCAP]
    unsigned* skey = reinterpret_cast<unsigned*>(lval + LCAP);                // [LCAP] sorted by row
    float* sval = reinterpret_cast<float*>(skey + LCAP);    // [LCAP]
    int* bins = reinterpret_cast<int*>(sval + LCAP);        // [8][HW] per-warp row histograms / start offsets
    float* Qs = reinterpret_cast<float*>(bins + 8 * (LONG ? 64 : HW));    // [C]  sum_t gl/exp(logit)      (wrong-class fold)
    float* qg = Qs + C;                                     // [T]  gl/exp(logit) of the GT class
    __shared__ int wcount[8];
    __shared__ int lcount;
    __shared__ __align__(16) float part[16 * DC];           // boundary runs of the warps' list ranges (s1 vectors)
    __shared__ float part2[16];                             // ... their scalar sum_e a_e w_p (isotropic sigma)
    __shared__ int prow[16];
    __shared__ int mrow[16], mcount;                        // boundary runs merged by row

    const int b = blockIdx.x;
    const int d0 = blockIdx.y * DC;
    const int dc = min(DC, D - d0);
    const int P = C * K;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool has_gt = (gt != nullptr);
    const long long g = has_gt ? (long long)gt[b] : -1;

    if (has_gt) {
        if (C * T <= 2 * LCAP) {
            // q[c][t] = gl / exp(logit) for the whole image in one coalesced pass (staged in the sorted-list
            // area, free until the first drain), then one thread per class sums its T levels
            float* qtmp = reinterpret_cast<float*>(skey);
            const size_t lo = (size_t)b * C * T;
            for (int i = threadIdx.x; i < C * T; i += 256) qtmp[i] = gl[lo + i] / expf(logits[lo + i]);
            __syncthreads();
            for (int c = threadIdx.x; c < C; c += 256) {
                float q = 0.f;
                for (int t = 0; t < T; ++t) q += qtmp[c * T + t];
                Qs[c] = q;
            }
            if (g >= 0 && g < C)
                for (int t = threadIdx.x; t < T; t += 256) qg[t] = qtmp[(int)g * T + t];
        } else {
            for (int c = threadIdx.x; c < C; c += 256) {
                const size_t lo = ((size_t)b * C + c) * T;
                float q = 0.f;
                for (int t = 0; t < T; ++t) q += gl[lo + t] / expf(logits[lo + t]);
                Qs[c] = q;
            }
            if (g >= 0 && g < C)
                for (int t = threadIdx.x; t < T; t += 256) {
                    const size_t lo = ((size_t)b * C + (size_t)g) * T;
                    qg[t] = gl[lo + t] / expf(logits[lo + t]);
                }
        }
    }
    if (threadIdx.x == 0) lcount = 0;
    __syncthreads();

    // entry space: with labels only level 0 of every prototype plus levels 1..T-1 of the GT class carry
    // gradient (wrong-class levels alias level 0, ref model.py:221); without labels all P*T entries
    const bool gvalid = has_gt && g >= 0 && g < C;
    const int E = has_gt ? (P + (gvalid ? K * (T - 1) : 0)) : P * T;
    // entry e -> (coefficient a, key p*1024 + n); evaluated one iteration ahead so the gathers of the next
    // 256 entries are in flight while the current ones are compacted
    auto entry = [&](int e, float& a, unsigned& key) {
        a = 0.f;
        key = 0;
        if (e < E) {
            int p, t;
            float qv;
            if (has_gt) {
                if (e < P) {
                    p = e; t = 0;
                    const int c = p / K;
                    qv = ((long long)c == g) ? qg[0] : Qs[c];
                } else {
                    const int r = e - P;
                    const int k = r / (T - 1);
                    t = 1 + (r - k * (T - 1));
                    p = (int)g * K + k;
                    qv = qg[t];
                }
            } else {
                p = e / T; t = e - p * T;
                const size_t lo = ((size_t)b * C + p / K) * T + t;
                qv = gl[lo] / expf(logits[lo]);
            }
            const int c = p / K;
            const size_t vi = ((size_t)b * P + p) * T + t;
            a = qv * __ldg(weight + (size_t)c * P + p) * vals[vi];
            key = (unsigned)p * (KM + 1u) + (unsigned)idx[vi];
        }
    };
    float a_nx;
    unsigned key_nx;
    entry(threadIdx.x, a_nx, key_nx);
    for (int e0 = 0; e0 < E; e0 += 256) {
        const float a = a_nx;
        const unsigned key = key_nx;
        entry(e0 + 256 + threadIdx.x, a_nx, key_nx);
        const bool keep = (a != 0.f);
        const unsigned bal = __ballot_sync(0xffffffffu, keep);
        if (lane == 0) wcount[warp] = __popc(bal);
        __syncthreads();
        int base = lcount;
        for (int wv = 0; wv < warp; ++wv) base += wcount[wv];
        if (keep) {
            const int pos = base + __popc(bal & ((1u << lane) - 1u));
            lkey[pos] = key;
            lval[pos] = a;
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            int tot = 0;
            for (int wv = 0; wv < 8; ++wv) tot += wcount[wv];
            lcount += tot;
        }
        __syncthreads();
        const int cnt = lcount;
        const bool last = (e0 + 256 >= E);
        if (cnt + 256 > LCAP || last) {
            if constexpr (!LONG) {
                // Stable counting sort of the entries by patch row (deterministic): warp w owns the w-th contiguous
                // eighth of the list; per-warp row histograms (MATCH.ANY, leader adds) -> per-warp start offsets ->
                // in-order scatter.  Mined patches cluster on a few dozen rows, so after the sort a lane meets long
                // runs of one row.
                int* whist = bins;                                  // [8][HW] per-warp histograms, then start offsets
                for (int i = threadIdx.x; i < 8 * HW; i += 256) whist[i] = 0;
                __syncthreads();
                const int seg = (cnt + 7) / 8, sb = min(cnt, warp * seg), se = min(cnt, sb + seg);
                for (int i0 = sb; i0 < se; i0 += 32) {
                    const int i = i0 + lane;
                    const int n = (i < se) ? (int)(lkey[i] & 1023u) : (0x10000 + lane);
                    const unsigned m = __match_any_sync(0xffffffffu, n);
                    if (i < se && (m & ((1u << lane) - 1u)) == 0) whist[warp * HW + n] += __popc(m);
                    __syncwarp();
                }
                __syncthreads();
                // start offset of (warp, row): rows ascending, warps ascending inside a row
                if (warp == 0) {
                    int carry = 0;
                    for (int r0 = 0; r0 < HW; r0 += 32) {
                        const int r = r0 + lane;
                        int tot = 0;
                        if (r < HW)
                            for (int wv = 0; wv < 8; ++wv) tot += whist[wv * HW + r];
                        int x = tot;
    #pragma unroll
                        for (int o = 1; o < 32; o <<= 1) {
                            const int y = __shfl_up_sync(0xffffffffu, x, o);
                            if (lane >= o) x += y;
                        }
                        int start = carry + x - tot;                // exclusive prefix
                        if (r < HW)
                            for (int wv = 0; wv < 8; ++wv) {
                                const int c = whist[wv * HW + r];
                                whist[wv * HW + r] = start;
                                start += c;
                            }
                        carry += __shfl_sync(0xffffffffu, x, 31);
                    }
                }
                __syncthreads();
                for (int i0 = sb; i0 < se; i0 += 32) {
                    const int i = i0 + lane;
                    const unsigned kk = (i < se) ? lkey[i] : 0u;
                    const int n = (i < se) ? (int)(kk & 1023u) : (0x10000 + lane);
                    const unsigned m = __match_any_sync(0xffffffffu, n);
                    if (i < se) {
                        const int pos = whist[warp * HW + n] + __popc(m & ((1u << lane) - 1u));
                        skey[pos] = kk;
                        sval[pos] = lval[i];
                    }
                    __syncwarp();
                    if (i < se && (m & ((1u << lane) - 1u)) == 0) whist[warp * HW + n] += __popc(m);
                    __syncwarp();
                }
                __syncthreads();
            } else {
                // Two stable 64-bin counting passes on the 12-bit row, low 6 bits (lkey -> skey), then high 6 bits
                // (skey -> lkey), each exactly as the single pass above with [8][64] histograms: the sorted list ends
                // in lkey / lval.
                const int seg = (cnt + 7) / 8, sb = min(cnt, warp * seg), se = min(cnt, sb + seg);
                auto pass = [&](const unsigned* sk, const float* sv, unsigned* dk, float* dv, unsigned sh) {
                    int* whist = bins;                              // [8][64] per-warp histograms, then start offsets
                    for (int i = threadIdx.x; i < 8 * 64; i += 256) whist[i] = 0;
                    __syncthreads();
                    for (int i0 = sb; i0 < se; i0 += 32) {
                        const int i = i0 + lane;
                        const int n = (i < se) ? (int)((sk[i] >> sh) & 63u) : (0x10000 + lane);
                        const unsigned m = __match_any_sync(0xffffffffu, n);
                        if (i < se && (m & ((1u << lane) - 1u)) == 0) whist[warp * 64 + n] += __popc(m);
                        __syncwarp();
                    }
                    __syncthreads();
                    if (warp == 0) {                                // (digit, warp) start offsets, as above
                        int carry = 0;
#pragma unroll
                        for (int r0 = 0; r0 < 64; r0 += 32) {
                            const int r = r0 + lane;
                            int tot = 0;
                            for (int wv = 0; wv < 8; ++wv) tot += whist[wv * 64 + r];
                            int x = tot;
#pragma unroll
                            for (int o = 1; o < 32; o <<= 1) {
                                const int y = __shfl_up_sync(0xffffffffu, x, o);
                                if (lane >= o) x += y;
                            }
                            int start = carry + x - tot;
                            for (int wv = 0; wv < 8; ++wv) {
                                const int c = whist[wv * 64 + r];
                                whist[wv * 64 + r] = start;
                                start += c;
                            }
                            carry += __shfl_sync(0xffffffffu, x, 31);
                        }
                    }
                    __syncthreads();
                    for (int i0 = sb; i0 < se; i0 += 32) {
                        const int i = i0 + lane;
                        const unsigned kk = (i < se) ? sk[i] : 0u;
                        const int n = (i < se) ? (int)((kk >> sh) & 63u) : (0x10000 + lane);
                        const unsigned m = __match_any_sync(0xffffffffu, n);
                        if (i < se) {
                            const int pos = whist[warp * 64 + n] + __popc(m & ((1u << lane) - 1u));
                            dk[pos] = kk;
                            dv[pos] = sv[i];
                        }
                        __syncwarp();
                        if (i < se && (m & ((1u << lane) - 1u)) == 0) whist[warp * 64 + n] += __popc(m);
                        __syncwarp();
                    }
                    __syncthreads();
                };
                pass(lkey, lval, skey, sval, 0u);
                pass(skey, sval, lkey, lval, 6u);
            }
            // Walk: warp w owns the w-th eighth of the row-sorted list (balanced however the patches cluster),
            // lanes own two dims each, so one instruction handles one entry x 64 dims and the prototype rows
            // are read as coalesced 256-byte segments, eight in flight.  Per row n:
            //   g[n] += sum_e a_e * wm_p  -  xhat_n * sum_e a_e * w_p
            // (w_p is a per-prototype scalar when every sigma is isotropic).  xhat_n and the old g[n] are fetched
            // when a run starts and used when it ends.  Runs inside a warp's range are complete rows (single
            // writer); the first and last run of a range may continue in the neighbour's range: they are parked in
            // `part`, merged by row in a fixed order and added afterwards -> no atomics, deterministic.
            const unsigned* wkey = LONG ? lkey : skey;           // the row-sorted list
            const float* wval = LONG ? lval : sval;
            if (threadIdx.x < 16) prow[threadIdx.x] = -1;
            __syncthreads();
            const int dl = VEC * lane;
            const bool dok2 = dl < dc;
            const int dle = dok2 ? dl : 0;                       // lanes beyond dc shadow the first dims, never store
            const float* xcol2 = xhat + (size_t)b * HW * D + d0 + dle;
            float* gcol = g_xhat + (size_t)b * HW * D + d0 + dle;
            {
                const int wseg = (cnt + 7) / 8, wb = min(cnt, warp * wseg), we = min(cnt, wb + wseg);
                const float* wmcol_l = wm + d0 + dle;
                const float* wcol_l = w + d0 + dle;
                int cur_n = -1;
                bool first_run = true;
                LV s1 = lv_zero<VEC>(), s2v = lv_zero<VEC>(), xpre = lv_zero<VEC>(), gpre = lv_zero<VEC>();
                float s2 = 0.f;
                auto flush = [&](int slot) {
                    if (slot < 0) {
                        LV v = gpre;
#pragma unroll
                        for (int i = 0; i < VEC; ++i) v.v[i] += aniso ? fmaf(-xpre.v[i], s2v.v[i], s1.v[i]) : fmaf(-xpre.v[i], s2, s1.v[i]);
                        if (dok2) lv_st<VEC>(gcol + (size_t)cur_n * D, v);
                    } else {
                        LV v = s1;                                // isotropic: raw sums, xhat applied after the merge
                        if (aniso) {
#pragma unroll
                            for (int i = 0; i < VEC; ++i) v.v[i] = fmaf(-xpre.v[i], s2v.v[i], v.v[i]);
                        }
                        if (dok2) lv_st<VEC>(part + (warp * 2 + slot) * DC + dl, v);
                        if (lane == 0) { part2[warp * 2 + slot] = aniso ? 0.f : s2; prow[warp * 2 + slot] = cur_n; }
                    }
                };
                auto walk = [&](auto aniso_tag) {
                    constexpr bool AN = decltype(aniso_tag)::value;
                    constexpr int PF = (VEC == 4 && !AN) ? 16 : 8;    // prototype rows in flight per lane
                    for (int i0 = wb; i0 < we; i0 += 32) {
                        const int i = i0 + lane;
                        const bool ok = i < we;
                        const unsigned kk = wkey[ok ? i : we - 1];    // slots beyond the range: last entry, zero coefficient
                        const float av = ok ? wval[i] : 0.f;
                        const float v2 = (!AN && ok) ? av * __ldg(wsc + (kk >> KS)) : 0.f;
                        const int m = min(32, we - i0);
                        for (int j0 = 0; j0 < m; j0 += PF) {
                            LV fm[PF], fw[AN ? PF : 1];
#pragma unroll
                            for (int u = 0; u < PF; ++u) {
                                const unsigned ku = __shfl_sync(0xffffffffu, kk, j0 + u);
                                const unsigned po = (ku >> KS) * (unsigned)D;
                                fm[u] = lv_ldg<VEC>(wmcol_l + po);
                                if constexpr (AN) fw[u] = lv_ldg<VEC>(wcol_l + po);
                            }
#pragma unroll
                            for (int u = 0; u < PF; ++u) {
                                const int n = (int)(__shfl_sync(0xffffffffu, kk, j0 + u) & KM);
                                const float a = __shfl_sync(0xffffffffu, av, j0 + u);
                                if (n != cur_n) {
                                    if (cur_n >= 0) {
                                        flush(first_run ? 0 : -1);
                                        first_run = false;
                                    }
                                    cur_n = n;
                                    xpre = lv_ldg<VEC>(xcol2 + (size_t)n * D);
                                    gpre = lv_ldcg<VEC>(gcol + (size_t)n * D);
                                    s1 = lv_zero<VEC>();
                                    s2v = lv_zero<VEC>();
                                    s2 = 0.f;
                                }
#pragma unroll
                                for (int i = 0; i < VEC; ++i) s1.v[i] = fmaf(a, fm[u].v[i], s1.v[i]);
                                if constexpr (AN) {
#pragma unroll
                                    for (int i = 0; i < VEC; ++i) s2v.v[i] = fmaf(a, fw[u].v[i], s2v.v[i]);
                                } else {
                                    s2 += __shfl_sync(0xffffffffu, v2, j0 + u);
                                }
                            }
                        }
                    }
                };
                if (aniso) walk(std::true_type{}); else walk(std::false_type{});
                if (cur_n >= 0) flush(first_run ? 0 : 1);
            }
            __syncthreads();
            if (warp == 0) {                                      // merge the parked runs by row, in list order (in place)
                int j = -1, last = -1;
                LV acc = lv_zero<VEC>();
                float a2 = 0.f;
                for (int i = 0; i < 16; ++i) {
                    const int n = prow[i];
                    if (n < 0) continue;
                    const LV v = lv_ld<VEC>(part + i * DC + dl);
                    const float p2 = part2[i];
                    __syncwarp();
                    if (n != last) { ++j; last = n; acc = lv_zero<VEC>(); a2 = 0.f; }
#pragma unroll
                    for (int q = 0; q < VEC; ++q) acc.v[q] += v.v[q];
                    a2 += p2;
                    lv_st<VEC>(part + j * DC + dl, acc);
                    if (lane == 0) { part2[j] = a2; mrow[j] = n; }
                    __syncwarp();
                }
                if (lane == 0) mcount = j + 1;
            }
            __syncthreads();
            for (int j = warp; j < mcount; j += 8) {
                const int n = mrow[j];
                const LV xv = lv_ldg<VEC>(xcol2 + (size_t)n * D);
                LV gv = lv_ldcg<VEC>(gcol + (size_t)n * D);
                const LV v = lv_ld<VEC>(part + j * DC + dl);
                const float p2 = part2[j];
#pragma unroll
                for (int q = 0; q < VEC; ++q) gv.v[q] += fmaf(-xv.v[q], p2, v.v[q]);
                if (dok2) lv_st<VEC>(gcol + (size_t)n * D, gv);
            }
            __syncthreads();
            if (threadIdx.x == 0) lcount = 0;
            __syncthreads();
        }
    }
}

#define MGP_HEAD_BWD_PARAMS                                                                                           \
    const float* __restrict__ gl, const float* __restrict__ logits, const float* __restrict__ vals,                  \
        const int32_t* __restrict__ idx, const float* __restrict__ weight, const int64_t* __restrict__ gt,           \
        const float* __restrict__ xhat, const float* __restrict__ w, const float* __restrict__ wm,                   \
        const float* __restrict__ wsc, const int* __restrict__ noniso, float* __restrict__ g_xhat, int HW, int C,    \
        int K, int D, int T
#define MGP_HEAD_BWD_ARGS gl, logits, vals, idx, weight, gt, xhat, w, wm, wsc, noniso, g_xhat, HW, C, K, D, T

}  // namespace

// The per-prototype operands the walk reads, from mu / sigma [P,D] (proto_weight_kernel, head.cu): w = 1/sigma^2,
// wm = w*mu, wsc[p] = w[p,0] and *noniso = 1 if sigma varies over d inside a prototype.
int head_bwd_proto_weights(const float* mu, const float* sigma, float* w, float* wm, float* wsc, int* noniso, int P,
                           int D, cudaStream_t st);
