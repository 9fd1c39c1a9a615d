// a10-a12 on the Hopper tensor cores: the whole update_GMM (ref model.py:277-301, :303-321, :367-401) of a single
// replica in ONE launch after em_plan, one CTA per class, for the shapes the shipped loop produces
// (K <= 16 components, D = 128 or 256, sigma constant over d inside every component).
//
// Per class and EM loop the two inner products are GEMMs over the class's bank rows X [cap x D]:
//     E-step     Q  [cap x K]  = X . A^T        A_k = -2 w_k mu_k          (q_nk = w_k (|x_n|^2 + |mu_k|^2) + Q_nk)
//     statistics S1^T [D x K]  = X^T . R        R_nk = smoothed responsibility
// They run as wgmma.mma_async (fp16 operands from shared memory, fp32 accumulators in registers) on fp16 hi/lo
// splits -- hi*hi + lo*hi + hi*lo, 22 mantissa bits, the scheme of logprob_tc.cu -- of
//   * the bank rows: a SHADOW of the fp32 bank kept in HBM as fp16 hi / lo of 256 x (written by the enqueue scatter,
//     csrc/bank.cu), so a 128-row tile is four TMA boxes into 128B-swizzled shared memory with no conversion pass.
//     The same tile serves both GEMMs: as the K-major A operand of the E-step (rows x d) and as the MN-major
//     (transposed) A operand of the statistics GEMM (d x rows) -- one copy, two descriptors;
//   * the means operand A (rebuilt from the on-chip means after every Adam step) and the responsibilities R (written
//     by the E-step epilogue), both split in registers and stored in the K-major SWIZZLE_128B layout.
// Everything else (soft-max, S0, gradient, diversity term, Adam, pi momentum, the zero-gradient replay of the other
// classes' steps) is fp32 SIMT on the class's state, which stays in registers / shared memory for the whole timeline
// exactly as in em_fused_kernel (em.cu); thread d owns mean / moment elements (k, d) for all k.
//
// The E-step of a row tile (per m64 half: m64n32 with the X hi rows against [means hi ; means lo], m64n16 with the
// X lo rows against means hi) is followed by its soft-max straight from the accumulator fragments (the 16 components
// of a row sit in 4 lanes) and the statistics GEMM of the tile (D / 64 m64 blocks), which keeps S1 in registers across
// the tiles of a loop; at the end of a loop S1 goes to the owners through shared memory.  Two variants of the same
// kernel, by D:
//   * D = 128: ONE warpgroup of 128 threads runs E-step, soft-max and statistics of a tile in turn, so that two CTAs
//     share an SM and up to 2 x #SMs classes run in one wave.  64-row tiles -- tile t is the half t % 2 of a 128-row
//     tile, so the MMAs into S1 come in the same order -- stream through a two-slot ring: the TMA load of tile t+1
//     runs under tile t;
//   * D = 256: two warpgroups, 128-row tiles, one tile buffer.  Warpgroup 0 (warps 0-3) runs the E-step and soft-max,
//     then warpgroup 1 (warps 4-7) the statistics of the tile.
// At D = 128 block b runs class clist[b], the planner's order with the active classes first: they take the lowest
// block indices, so while they fit one CTA per SM none shares its SM with another active class.  At D = 256 (one CTA
// per SM in any case) block b runs class b.
// HBM/L2 traffic: num_em_loop x (4 D + 4) bytes per bank row -- the algorithmic bytes of SURVEY 8(d) K-D.
// Staged outputs (mgp_update_gmm_staged): the new means go to a [C,K,D] copy and the new class-diagonal pi to a [C,K]
// copy instead of the parameters, so that a backward still reading mu and pi can run beside the kernel; every class
// (inactive and skipped ones included) writes its slots, and mgp_em_commit copies them over afterwards.
#include <cuda.h>
#include <cuda_fp16.h>

#include "mgp_common.cuh"
#include "em_common.cuh"
#include "tc_ptx.cuh"

namespace {
using namespace mgp_em;
using namespace mgp_tc;

constexpr float SR = 1024.0f;     // responsibilities are stored as 1024 r
constexpr int S1_STRIDE = 17;     // S1 hand-over [D][17] fp32 (padded against bank conflicts)

// the kernel at D = 128 is the one-warpgroup variant (two CTAs per SM, 64-row tiles); at D = 256 it has two
// warpgroups and 128-row tiles (bank rows per tile = M of the E-step, K extent of the statistics GEMM)
__host__ __device__ constexpr bool em_one_wg(int D) { return D == 128; }
__host__ __device__ constexpr int em_threads(int D) { return em_one_wg(D) ? 128 : 256; }
__host__ __device__ constexpr int em_rows(int D) { return em_one_wg(D) ? 64 : 128; }

struct EmTcParams {
    const float* xx;              // [C*cap] |x|^2 of the bank rows (shadow)
    const float* bc;              // planner tables: [2 n] Adam bias corrections of steps step0+1.., then b1^i, b2^(i/2), b2^i for i <= n = L * n_active
    const int32_t* order;
    const int32_t* sched;
    const int32_t* clist;         // planner: classes in launch order, active first (stats scratch at 5 L C + 4)
    float* mu;
    const float* sigma;
    float* weight;
    float* exp_avg;
    float* exp_avg_sq;
    float* mu_out;                // where the new means go: mu itself, or a staging [C,K,D] copy (see mgp_update_gmm_staged)
    float* pi_out;                // staging [C,K] for the new class-diagonal pi, or nullptr: written into weight in place
    int* status;                  // set to 1 if a class turned out to have anisotropic sigma (its update is skipped)
    long long* prof;              // profiling (mgp_debug_set_ptr("em_tc_prof")): clock64 stamps of class `prof_class`
    AdamCfg adam;
    float alpha, tau, omtau, lamda;
    int num_em_loop, C, K, cap, prof_class;
};
// stamp layout: prof[(tile_ctr * 8 + phase)]; phases: 0 TMA issued, 1 TMA landed (seen by thread 0), 4 soft-max done,
// 5 statistics MMAs done, 6 loop tail entered, 7 loop tail done
#define MGP_PROF(ctr, ph)                                                                          \
    do {                                                                                           \
        if (prm.prof && c == prm.prof_class && (ctr) < 64) prm.prof[(ctr) * 8 + (ph)] = clock64();  \
    } while (0)

// Sum V = 32 R values per lane across the warp with V - R shuffles (a butterfly that halves the live set each round)
// instead of 5 V: afterwards a[i], i < R, holds the warp total of entry R * lane + i.
template <int V>
__device__ __forceinline__ void warp_multi_reduce(float (&a)[V], int lane) {
    static_assert(V % 32 == 0, "V must be a multiple of the warp size");
#pragma unroll
    for (int off = 16, n = V / 2; off >= 1; off >>= 1, n >>= 1) {
        const bool up = (lane & off) != 0;
#pragma unroll
        for (int i = 0; i < n; ++i) {
            const float send = up ? a[i] : a[i + n], keep = up ? a[i + n] : a[i];
            a[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
        }
    }
}

template <int D, int KT>
__global__ void __launch_bounds__(em_threads(D), em_one_wg(D) ? 2 : 1)
em_tc_kernel(const __grid_constant__ CUtensorMap map_h, const __grid_constant__ CUtensorMap map_l, const EmTcParams prm) {
    constexpr bool WG1 = em_one_wg(D);             // one warpgroup runs everything (D = 128)
    constexpr int NT = em_threads(D), NW = NT / 32;
    constexpr int TR = em_rows(D);                 // bank rows per tile
    constexpr int NCH = D / 64;                    // 64-element (128 B) chunks along d
    constexpr uint32_t CH_BYTES = TR * 128;        // one [TR rows x 64] fp16 block
    constexpr uint32_t X_BYTES = NCH * CH_BYTES;   // hi (lo follows)
    constexpr uint32_t R_BYTES = (TR / 64) * 4096; // one R buffer
    constexpr int OWN = D;                         // threads owning mean/moment elements: thread d <-> (k, d) for all k
    constexpr int MB = D / 64;                     // m64 blocks of the statistics GEMM
    constexpr int SW0 = NW - 4;                    // first warp of the warpgroup that runs the statistics GEMM
    // the TMA issuing thread: lane 0 of warp 4 (warps 0-3 run the E-step), or thread 0 of the single warpgroup
    constexpr int ISSUER = 32 * SW0;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* bp = smem_raw + (base - raw);
    // carve-up (bytes from `base`)
    constexpr int NXBUF = WG1 ? 2 : 1;
    const uint32_t o_xh = 0, o_xl = X_BYTES;                               // buffer b: + b * 2 * X_BYTES
    // means operand A and responsibilities R: per 64-wide K chunk one [32 rows x 128 B] block, rows 0-15 = hi,
    // rows 16-31 = lo, so ONE N = 32 MMA multiplies the row tile's hi half with both and an N = 16 MMA adds lo x hi
    const uint32_t o_a = NXBUF * 2 * X_BYTES;                             // [NCH][32][128 B]
    const uint32_t o_r = o_a + NCH * 4096;                                // [TR / 64 (64-row chunks)][32][128 B]
    const uint32_t o_s1 = o_r + R_BYTES;                                  // S1 hand-over [D][S1_STRIDE]
    const uint32_t o_misc = o_s1 + (uint32_t)((D * S1_STRIDE * 4 + 15) & ~15);
    // two warpgroups: tma, (unused), stats | one warpgroup: xfull[2]
    uint64_t* bars = reinterpret_cast<uint64_t*>(bp + o_misc);
    float* s_e = reinterpret_cast<float*>(bars + 12);                     // [KT][KT]
    float* s_red = s_e + KT * KT;                                         // [8] + [8][16]
    float* s_w = s_red + 136;                                             // [16] w_k
    float* s_ls = s_w + 16;                                               // [16] sum_d (log(sigma+eps) + log(2pi)/2)
    float* s_pi = s_ls + 16;                                              // [16]
    float* s_cst = s_pi + 16;                                             // [16]
    float* s_s0 = s_cst + 16;                                             // [16]
    float* s_misc = s_s0 + 16;                                            // [8]: replay sums T1..T3, min d; operand scale; moment decays
    constexpr int NPAIR = KT * (KT - 1) / 2;
    // per-warp partials of the loop top: |mu_i - mu_j|^2 for the NPAIR pairs, then |mu_k|^2 for the KT components
    constexpr bool MULTI = (NPAIR + KT) <= 64;                            // one transposing reduction (warp_multi_reduce)
    constexpr int PV = MULTI ? 32 * ((NPAIR + KT + 31) / 32) : NPAIR + KT;
    float* s_pair = s_misc + 8;                                           // [8 warps][PV]
    const uint32_t bar_tma = smem_u32(bars), bar_s = bar_tma + 16;

    const int n_active = prm.sched[0], step0 = prm.sched[1];
    // two CTAs per SM (D = 128): the active classes first (the planner's order), so that no two share an SM while
    // they fit one per SM.  D = 256 runs one CTA per SM and keeps class order: the planner's order measured up to 3 %
    // slower there at some active counts (DESIGN 8.3)
    const int c = WG1 ? prm.clist[blockIdx.x] : (int)blockIdx.x;
    const int ord = prm.order[c];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int K = prm.K, cap = prm.cap, L = prm.num_em_loop, P = prm.C * K, KD = K * D;
    const AdamCfg& adam = prm.adam;
    const bool own = tid < OWN;
    const float* sg_c = prm.sigma + (size_t)c * KD;

    if (tid == 0) MGP_PROF(63, 0);
    float p_[KT], m_[KT], v_[KT];
#pragma unroll
    for (int k = 0; k < KT; ++k) {
        p_[k] = 0.f; m_[k] = 0.f; v_[k] = 1.f;
        if (own && k < K) {
            const size_t o = (size_t)c * KD + k * D + tid;
            p_[k] = prm.mu[o]; m_[k] = prm.exp_avg[o]; v_[k] = prm.exp_avg_sq[o];
        }
    }
    // `count` zero-gradient Adam steps first+1 .. first+count on the registers (em_common.cuh).  The per-step sum
    //   p <- p - m0 * sum_s c_s / (a d_s + eps),   a = sqrt(v0),
    // is evaluated through its expansion in eps / (a d_s) (< 1e-3 whenever a d_min > 1e3 eps, i.e. v0 > ~1e-10):
    //   sum_s c_s / (a d_s + eps) = T1 / a - eps T2 / a^2 + eps^2 T3 / a^3 - ...,   Tj = sum_s c_s / d_s^j,
    // three block-wide scalars per replay (truncation < 1e-9) instead of one reciprocal per (step, element); elements
    // with a tiny second moment (a fresh optimiser) take the explicit loop.
    // The step-dependent factors come from tables the planner wrote once for the whole launch (em.cu em_plan_kernel):
    //   bc[2i] = lr / (1 - b1^t), bc[2i+1] = sqrt(1 - b2^t), t = step0 + 1 + i;   B1[n] = b1^n, B2H[n] = b2^(n/2), B2[n] = b2^n
    // so that c_s = bc0[t] B1[s], d_s = B2H[s] / bc1[t]: no transcendental is evaluated per class.
    const int n_steps = L * n_active;
    const float* t_b1 = prm.bc + 2 * n_steps;
    const float* t_b2h = t_b1 + (n_steps + 1);
    const float* t_b2 = t_b2h + (n_steps + 1);
    // (a) one warp: the replay's block-wide scalars T1..T3 and min d_s
    auto replay_sums = [&](int first, int count, int ns, bool tail, float& T1, float& T2, float& T3, float& dmin_out) {
        const int i0 = first - step0;                       // table index of step first+1
        double t1 = 0.0, t2 = 0.0, t3 = 0.0;
        float dmin = INFINITY;
        for (int s = lane + 1; s <= ns + (tail ? 1 : 0); s += 32) {
            float cs, ds;
            if (s <= ns) {
                cs = __ldg(prm.bc + 2 * (i0 + s - 1)) * __ldg(t_b1 + s);
                ds = __ldg(t_b2h + s) / __ldg(prm.bc + 2 * (i0 + s - 1) + 1);
            } else {                                    // steps ns+1 .. count as one geometric term (em_common.cuh)
                const float geo = __ldg(t_b1 + ns + 1) * (1.0f - __ldg(t_b1 + (count - ns))) / (float)(1.0 - adam.beta1);
                const int ss = min(count, ns + 1 + (int)(adam.beta1 / (1.0 - adam.beta1)));
                cs = __ldg(prm.bc + 2 * (i0 + ns)) * geo;
                ds = __ldg(t_b2h + ss) / __ldg(prm.bc + 2 * (i0 + ss - 1) + 1);
            }
            const double c = (double)cs, r = 1.0 / (double)ds;
            t1 += c * r; t2 += c * r * r; t3 += c * r * r * r;
            dmin = fminf(dmin, ds);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            t1 += __shfl_xor_sync(0xffffffffu, t1, o);
            t2 += __shfl_xor_sync(0xffffffffu, t2, o);
            t3 += __shfl_xor_sync(0xffffffffu, t3, o);
            dmin = fminf(dmin, __shfl_xor_sync(0xffffffffu, dmin, o));
        }
        T1 = (float)t1; T2 = (float)t2; T3 = (float)t3; dmin_out = dmin;
    };
    // (b) one element: p after the `count` zero-gradient steps (the moments decay separately)
    auto replay_elem = [&](float p, float m, float v, int first, int count, int ns, bool tail, float T1, float T2, float T3,
                           float dmin) -> float {
        const float a = sqrtf(v);
        if (a * dmin > 1000.0f * adam.epsf) {
            const float inv = 1.0f / a;
            const float e = adam.epsf * inv;
            return fmaf(-m * inv, fmaf(-e, fmaf(-e, T3, T2), T1), p);
        }
        if (m != 0.f) {                                     // tiny second moment (fresh optimiser): term by term
            const int i0 = first - step0;
            for (int s = 1; s <= ns; ++s) {
                const float cs = __ldg(prm.bc + 2 * (i0 + s - 1)) * __ldg(t_b1 + s);
                const float ds = __ldg(t_b2h + s) / __ldg(prm.bc + 2 * (i0 + s - 1) + 1);
                p = fmaf(-cs * m, 1.0f / fmaf(a, ds, adam.epsf), p);
            }
            if (tail) {
                const float geo = __ldg(t_b1 + ns + 1) * (1.0f - __ldg(t_b1 + (count - ns))) / (float)(1.0 - adam.beta1);
                const int ss = min(count, ns + 1 + (int)(adam.beta1 / (1.0 - adam.beta1)));
                const float cs = __ldg(prm.bc + 2 * (i0 + ns)) * geo;
                const float ds = __ldg(t_b2h + ss) / __ldg(prm.bc + 2 * (i0 + ss - 1) + 1);
                p = fmaf(-cs * m, 1.0f / fmaf(a, ds, adam.epsf), p);
            }
        }
        return p;
    };
    // the sums of a replay, by ONE warp, into sums[0..3] (shared memory; the caller's next block barrier publishes them)
    auto replay_prepare = [&](int first, int count, float* sums) {
        if (count <= 0) return;
        const int ns = replay_explicit_steps(count, first, (float)adam.beta1);
        float T1, T2, T3, dmin;
        replay_sums(first, count, ns, count > ns, T1, T2, T3, dmin);
        if (lane == 0) { sums[0] = T1; sums[1] = T2; sums[2] = T3; sums[3] = dmin; }
    };
    auto replay = [&](int first, int count, const float* sums) {
        if (count <= 0) return;
        const int ns = replay_explicit_steps(count, first, (float)adam.beta1);
        const bool tail = count > ns;
        if (own) {
            const float T1 = sums[0], T2 = sums[1], T3 = sums[2], dmin = sums[3];
#pragma unroll
            for (int k = 0; k < KT; ++k) p_[k] = replay_elem(p_[k], m_[k], v_[k], first, count, ns, tail, T1, T2, T3, dmin);
        }
        const float mdec = __ldg(t_b1 + count), vdec = __ldg(t_b2 + count);   // the moments decay by the full count
#pragma unroll
        for (int k = 0; k < KT; ++k) { m_[k] *= mdec; v_[k] *= vdec; }
    };
    auto write_back = [&]() {
        if (!own) return;
#pragma unroll
        for (int k = 0; k < KT; ++k)
            if (k < K) {
                const size_t o = (size_t)c * KD + k * D + tid;
                prm.mu_out[o] = p_[k]; prm.exp_avg[o] = m_[k]; prm.exp_avg_sq[o] = v_[k];
            }
    };

    if (ord < 0) {                                   // inactive class: it only takes everybody's zero-gradient steps
        if (warp == 0) replay_prepare(step0, L * n_active, s_misc);
        __syncthreads();
        replay(step0, L * n_active, s_misc);
        write_back();
        if (prm.pi_out && tid < K) prm.pi_out[(size_t)c * K + tid] = prm.weight[(size_t)c * P + (size_t)c * K + tid];
        return;
    }
    // the two replays' block-wide sums depend on the plan only: two otherwise idle warps evaluate them under the set-up
    if (warp == NW - 1) replay_prepare(step0, L * ord, s_misc);
    if (warp == NW - 2) replay_prepare(step0 + L * (ord + 1), L * (n_active - ord - 1), s_misc + 4);

    if (tid == 0) MGP_PROF(63, 1);
    // ---- set-up: barriers, sigma-derived constants, zeroed operand tiles
    if (tid == 0) {
        if (WG1) {
            for (int i = 0; i < 2; ++i) mbar_init(bar_tma + 8u * i, 1);
        } else {
            mbar_init(bar_tma, 1);
            mbar_init(bar_s, 4);
        }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    bool same = true;
    for (int i = tid; i < KD; i += NT) same = same && (sg_c[i] == sg_c[(i / D) * D]);
    for (uint32_t i = tid * 16u; i < NCH * 4096u + R_BYTES; i += NT * 16u)     // A and R blocks: rows >= K stay zero
        *reinterpret_cast<uint4*>(bp + o_a + i) = make_uint4(0u, 0u, 0u, 0u);
    for (int i = tid; i < KT * KT; i += NT) s_e[i] = 0.f;
    if (tid < 16) {
        float w = 0.f, ls = 0.f, pi = 0.f;
        if (tid < K) {
            const float sg = sg_c[tid * D] + EM_EPS;                                     // ref :333-334
            w = 1.0f / (sg * sg);
            ls = (float)D * (logf(sg) + 0.5f * MGP_LOG_2PI);                             // D equal terms
            pi = prm.weight[(size_t)c * P + (size_t)c * K + tid];
        }
        s_w[tid] = w; s_ls[tid] = ls; s_pi[tid] = pi;
    }
    const bool iso = __syncthreads_and(same ? 1 : 0) != 0;
    if (!iso) {                                      // the host promised isotropic sigma: flag it, leave the class untouched
        if (tid == 0) atomicExch(prm.status, 1);
        if (prm.pi_out) {                            // staged: the class's staging slots keep its current values
            if (own) {
#pragma unroll
                for (int k = 0; k < KT; ++k)
                    if (k < K) prm.mu_out[(size_t)c * KD + k * D + tid] = p_[k];
            }
            if (tid < K) prm.pi_out[(size_t)c * K + tid] = s_pi[tid];
        }
        return;
    }
    if (tid == 0) MGP_PROF(63, 2);
    replay(step0, L * ord, s_misc);
    if (tid == 0) MGP_PROF(63, 3);

    const int ntiles = (cap + TR - 1) / TR;
    const float n_rows = (float)cap;
    const float inv_den = 1.0f / (1.0f + (float)K * prm.alpha);
    const float div_scale = -4.0f * prm.lamda / ((float)K * (float)(K - 1));
    uint32_t tile_ctr = 0;                                           // tiles issued so far (mbarrier phases)
    const int t4 = lane & 3, g8 = lane >> 2;                         // accumulator fragment coordinates (tc_ptx.cuh)
    float s32[MB][16], s16[MB][8];                                   // statistics warpgroup: S1 of the current loop
#pragma unroll
    for (int mb = 0; mb < MB; ++mb) {
#pragma unroll
        for (int j = 0; j < 16; ++j) s32[mb][j] = 0.f;
#pragma unroll
        for (int j = 0; j < 8; ++j) s16[mb][j] = 0.f;
    }

    // E-step of one tile + soft-max + R (warps 0-3).  E-step: A = X (K-major), B = [means hi ; means lo] (K-major):
    // N = 32 with X hi, N = 16 (means hi only) with X lo; rows h * 64 + 16 warp + g8 + 8 rr of the tile (NH m64
    // halves), components k = 8 i + 2 t4 + j (columns k: hi.hi, 16 + k: hi.lo; the N = 16 accumulator: lo.hi).
    constexpr int NH = TR / 64;
    auto estep_tile = [&](uint32_t xb, int t, float inv_a, float (&s0v)[4]) {
        uint8_t* rbp = bp + o_r;
        float e32[NH][16], e16[NH][8];
#pragma unroll
        for (int h = 0; h < NH; ++h) {
#pragma unroll
            for (int j = 0; j < 16; ++j) e32[h][j] = 0.f;
#pragma unroll
            for (int j = 0; j < 8; ++j) e16[h][j] = 0.f;
        }
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < D / 16; ++ks) {
            const uint32_t xo = (uint32_t)(ks >> 2) * CH_BYTES + (uint32_t)(ks & 3) * 32u;
            const uint64_t bd = gmma_desc(base + o_a + (uint32_t)(ks >> 2) * 4096u + (uint32_t)(ks & 3) * 32u);
#pragma unroll
            for (int h = 0; h < NH; ++h) {                           // rows 64 h .. 64 h + 63 of the tile: + 8 KiB
                wg_mma_n32<0>(e32[h], gmma_desc(xb + o_xh + xo + (uint32_t)h * 8192u), bd, 1u);
                wg_mma_n16<0>(e16[h], gmma_desc(xb + o_xl + xo + (uint32_t)h * 8192u), bd, 1u);
            }
        }
        wg_commit();
        wg_wait0();
        float rr_v[NH][2][4];
#pragma unroll
        for (int h = 0; h < NH; ++h)
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const int row = t * TR + h * 64 + 16 * warp + g8 + 8 * rr;
                const bool valid = row < cap;
                const float xxv = valid ? __ldg(prm.xx + (size_t)c * cap + row) : 0.f;
                float wl[4], mx = -INFINITY;
#pragma unroll
                for (int i = 0; i < 2; ++i)
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const int k = 8 * i + 2 * t4 + j, idx = 4 * i + 2 * rr + j;
                        const float acc = (e32[h][idx] + e16[h][idx]) + e32[h][idx + 8];
                        const float qq = fmaf(s_w[k], xxv, acc * inv_a);
                        wl[2 * i + j] = (k < K) ? s_cst[k] - 0.5f * qq : -INFINITY;   // lp + log(pi + eps)  (ref :316)
                        mx = fmaxf(mx, wl[2 * i + j]);
                    }
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
                mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
                float se = 0.f;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int k = 8 * (q >> 1) + 2 * t4 + (q & 1);
                    wl[q] = (k < K) ? expf(wl[q] - mx) : 0.f;
                    se += wl[q];
                }
                se += __shfl_xor_sync(0xffffffffu, se, 1);
                se += __shfl_xor_sync(0xffffffffu, se, 2);
                const float inv_se = 1.0f / se;
#pragma unroll
                for (int q = 0; q < 4; ++q) rr_v[h][rr][q] = valid ? fmaf(wl[q], inv_se, prm.alpha) * inv_den : 0.f;   // ref :380-383
            }
#pragma unroll
        for (int h = 0; h < NH; ++h)
#pragma unroll
            for (int rr = 0; rr < 2; ++rr) {
                const int rt = h * 64 + 16 * warp + g8 + 8 * rr;     // row within the tile
                const uint32_t rbase = (uint32_t)(rt >> 6) * 4096u + (uint32_t)(rt & 7) * 2u;
                const int c16 = (rt & 63) >> 3;
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int k = 8 * (q >> 1) + 2 * t4 + (q & 1);
                    if (k < K) {
                        const float r = rr_v[h][rr][q];
                        s0v[q] += r;
                        const uint32_t off = rbase + (uint32_t)k * 128u + (uint32_t)(((c16 ^ (k & 7)) & 7) << 4);
                        split_f16(r * SR, *reinterpret_cast<__half*>(rbp + off),                  // row k
                                  *reinterpret_cast<__half*>(rbp + off + 2048u));                 // row 16 + k
                    }
                }
            }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // R stores -> visible to the MMA (async proxy)
    };
    // statistics of one tile (warps SW0 .. SW0 + 3): S1 += X^T . [R hi ; R lo] (m64n32, A = X hi MN-major) and X lo^T . R hi
    // (m64n16), one m64 block per 64 d
    auto stats_tile = [&](uint32_t xb, bool first) {
        const uint32_t rb = base + o_r;
        wg_fence();
#pragma unroll
        for (int ks = 0; ks < TR / 16; ++ks) {
            const uint64_t bd = gmma_desc(rb + (uint32_t)(ks >> 2) * 4096u + (uint32_t)(ks & 3) * 32u);
            const uint32_t acc = (first && ks == 0) ? 0u : 1u;
#pragma unroll
            for (int mb = 0; mb < MB; ++mb) {
                const uint32_t xo = (uint32_t)mb * CH_BYTES + (uint32_t)ks * 2048u;   // 16 rows x 128 B
                wg_mma_n32<1>(s32[mb], gmma_desc_mn(xb + o_xh + xo, CH_BYTES, 1024u), bd, acc);
                wg_mma_n16<1>(s16[mb], gmma_desc_mn(xb + o_xl + xo, CH_BYTES, 1024u), bd, acc);
            }
        }
        wg_commit();
        wg_wait0();
    };

    auto load_tile = [&](int t) {                                    // issuer only (D = 256): one tile, hi + lo, into the X buffer
        mbar_expect_tx(bar_tma, 2 * X_BYTES);
        const int row0 = c * cap + t * TR;
#pragma unroll
        for (int ch = 0; ch < NCH; ++ch) {
            tma_load_2d(base + o_xh + ch * CH_BYTES, &map_h, ch * 64, row0, bar_tma);
            tma_load_2d(base + o_xl + ch * CH_BYTES, &map_l, ch * 64, row0, bar_tma);
        }
    };
    for (int loop = 0; loop < L; ++loop) {
        // ---- means operand, |mu_k|^2, diversity kernel from the current means (all from the owners' registers)
        float amax = 0.f;
        if (own) {                                                   // (warp-uniform: OWN is a multiple of 32)
#pragma unroll
            for (int k = 0; k < KT; ++k)
                if (k < K) amax = fmaxf(amax, fabsf(2.0f * s_w[k] * p_[k]));
            amax = warp_max(amax);
            // this thread's dimension of |mu_i - mu_j|^2 (ref utils/helpers.py:13-14; i < j) and of |mu_k|^2, summed over the warp
            if constexpr (MULTI) {
                float a[PV];
                int pi = 0;
#pragma unroll
                for (int i = 0; i < KT; ++i)
#pragma unroll
                    for (int j = i + 1; j < KT; ++j, ++pi) {
                        const float df = (j < K) ? p_[i] - p_[j] : 0.f;
                        a[pi] = df * df;
                    }
#pragma unroll
                for (int k = 0; k < KT; ++k) a[NPAIR + k] = (k < K) ? p_[k] * p_[k] : 0.f;
#pragma unroll
                for (int i = NPAIR + KT; i < PV; ++i) a[i] = 0.f;
                warp_multi_reduce<PV>(a, lane);                      // lane l now holds entries (PV/32) l + i
#pragma unroll
                for (int i = 0; i < PV / 32; ++i) s_pair[warp * PV + (PV / 32) * lane + i] = a[i];
            } else {
                int pi = 0;
#pragma unroll
                for (int i = 0; i < KT; ++i)
#pragma unroll
                    for (int j = i + 1; j < KT; ++j, ++pi) {
                        const float df = (j < K) ? p_[i] - p_[j] : 0.f;
                        const float t = warp_sum(df * df);
                        if (lane == 0) s_pair[warp * PV + pi] = t;
                    }
#pragma unroll
                for (int k = 0; k < KT; ++k) {
                    const float t = warp_sum((k < K) ? p_[k] * p_[k] : 0.f);
                    if (lane == 0) s_pair[warp * PV + NPAIR + k] = t;
                }
            }
        }
        if (lane == 0) s_red[warp] = amax;
        __syncthreads();
        float a_scale;
        {
            float mx = 0.f;
#pragma unroll
            for (int w8 = 0; w8 < NW; ++w8) mx = fmaxf(mx, s_red[w8]);
            int ex = 0;
            if (mx > 0.f) frexpf(mx, &ex);
            a_scale = ldexpf(1.0f, 8 - ex);                          // max |a| * scale in [128, 256)
        }
        if (tid < K) {
            float mm = 0.f;
#pragma unroll
            for (int w8 = 0; w8 < OWN / 32; ++w8) mm += s_pair[w8 * PV + NPAIR + tid];
            s_cst[tid] = -s_ls[tid] + logf(s_pi[tid] + EM_EPS) - 0.5f * s_w[tid] * mm;   // ref :316, :323-336
        }
        // exp(-|mu_i - mu_j|^2), ref model.py:390-392: pair pr on thread 32 + pr (one warpgroup: (32 + pr) % 128)
        static_assert(NPAIR <= 128, "one thread per pair");
        if (const int pr = WG1 ? (tid + NT - 32) % NT : tid - 32; pr >= 0 && pr < NPAIR) {
            int i = 0, rem = pr;
            while (rem >= KT - 1 - i) { rem -= KT - 1 - i; ++i; }
            const int j = i + 1 + rem;
            float t = 0.f;
#pragma unroll
            for (int w8 = 0; w8 < OWN / 32; ++w8) t += s_pair[w8 * PV + pr];
            const float e = (j < K) ? expf(-t) : 0.f;
            s_e[i * KT + j] = e;
            s_e[j * KT + i] = e;
        }
#pragma unroll
        for (int k = 0; k < KT; ++k)
            if (own && k < K) {
                const uint32_t off = (uint32_t)(tid >> 6) * 4096u + (uint32_t)k * 128u +
                                     (uint32_t)(((((tid & 63) >> 3) ^ (k & 7)) & 7) << 4) + (uint32_t)(tid & 7) * 2u;
                split_f16(-2.0f * s_w[k] * p_[k] * a_scale, *reinterpret_cast<__half*>(bp + o_a + off),   // row k      (hi)
                          *reinterpret_cast<__half*>(bp + o_a + off + 2048u));   // row 16 + k (lo): same swizzle phase
            }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // operand stores -> visible to the MMA (async proxy)
        __syncthreads();

        float s0v[4] = {0.f, 0.f, 0.f, 0.f};                          // warps 0-3: S0 of components 8 (q / 2) + 2 t4 + q % 2
        const float inv_a = 1.0f / (a_scale * X_SCALE);

        if constexpr (WG1) {
            // xfull[s]: a tile landed in slot s.  Tile g of the class's timeline (row tile g % ntiles of loop
            // g / ntiles) goes to slot g & 1, so xfull[s] completes once per tile in slot s: phase parity (g / 2) & 1.
            // Slot g & 1 takes tile g + 2 as soon as the statistics MMAs of tile g have retired.
            const uint32_t n_total = (uint32_t)(L * ntiles);
            auto xslot = [&](uint32_t g) { return base + (g & 1u) * 2 * X_BYTES; };
            auto load_tile_r = [&](uint32_t g) {                     // issuer only
                const uint32_t bar = bar_tma + 8u * (g & 1u);
                mbar_expect_tx(bar, 2 * X_BYTES);
                const int row0 = c * cap + (int)(g % (uint32_t)ntiles) * TR;
#pragma unroll
                for (int ch = 0; ch < NCH; ++ch) {
                    tma_load_2d(xslot(g) + o_xh + ch * CH_BYTES, &map_h, ch * 64, row0, bar);
                    tma_load_2d(xslot(g) + o_xl + ch * CH_BYTES, &map_l, ch * 64, row0, bar);
                }
                MGP_PROF(g, 0);
            };
            if (tid == ISSUER && loop == 0) {
                load_tile_r(0);
                if (n_total > 1) load_tile_r(1);
            }
            for (int t = 0; t < ntiles; ++t, ++tile_ctr) {
                const uint32_t g = tile_ctr;
                mbar_wait(bar_tma + 8u * (g & 1u), (g >> 1) & 1u);
                if (tid == 0) MGP_PROF(g, 1);
                estep_tile(xslot(g), t, inv_a, s0v);
                if (tid == 0) MGP_PROF(g, 4);
                __syncthreads();                                     // every warp's R rows are stored and fenced
                stats_tile(xslot(g), t == 0);
                if (tid == 0) MGP_PROF(g, 5);
                __syncthreads();                                     // every warp's statistics MMAs retired: slot and R free
                if (tid == ISSUER && g + 2 < n_total) load_tile_r(g + 2);   // (a loop's last two: the next loop's first two)
            }
        } else {
            for (int t = 0; t < ntiles; ++t, ++tile_ctr) {
                const uint32_t par = tile_ctr & 1u;
                if (tid == ISSUER) {
                    if (!(t == 0 && loop > 0)) {                             // (a loop's first tile was prefetched by the previous loop)
                        if (tile_ctr > 0) mbar_wait(bar_s, (tile_ctr - 1) & 1u);   // previous statistics MMAs have read X and R
                        load_tile(t);
                        MGP_PROF(tile_ctr, 0);
                    }
                }
                if (warp < 4) {
                    mbar_wait(bar_tma, par);
                    if (tid == 0) MGP_PROF(tile_ctr, 1);
                    estep_tile(base, t, inv_a, s0v);
                    if (tid == 0) MGP_PROF(tile_ctr, 4);
                }
                __syncthreads();
                if (warp >= 4) {
                    mbar_wait(bar_tma, par);                                 // (the tile is visible to this warpgroup's MMAs)
                    stats_tile(base, t == 0);
                    if (tid == ISSUER) MGP_PROF(tile_ctr, 5);
                    __syncwarp();
                    if (lane == 0) mbar_arrive(bar_s);
                }
            }
            if (tid == ISSUER && loop + 1 < L) {      // the next loop starts on the same rows: fetch its first tile under the tail
                mbar_wait(bar_s, (tile_ctr - 1) & 1u);
                load_tile(0);
            }
            mbar_wait(bar_s, (tile_ctr - 1) & 1u);                    // all statistics MMAs of this loop have retired
        }
        if (tid == 0) MGP_PROF(tile_ctr - 1, 6);
        // ---- S0 over the class (warps 0-3: reduce over the 8 rows of a fragment column, then lanes 0-3 hold all 16)
        if (warp < 4) {
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                float v = s0v[q];
                v += __shfl_xor_sync(0xffffffffu, v, 4);
                v += __shfl_xor_sync(0xffffffffu, v, 8);
                v += __shfl_xor_sync(0xffffffffu, v, 16);
                if (g8 == 0) s_red[warp * 16 + 8 * (q >> 1) + 2 * t4 + (q & 1)] = v;
            }
        }
        // ---- S1 from the statistics warpgroup's registers to the owners: s1[d][k] = (hi.hi + lo.hi) + hi.lo
        float* s_s1 = reinterpret_cast<float*>(bp + o_s1);
        if (warp >= SW0) {
#pragma unroll
            for (int mb = 0; mb < MB; ++mb)
#pragma unroll
                for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        const int d = mb * 64 + 16 * (warp - SW0) + g8 + 8 * rr, k = 8 * (q >> 1) + 2 * t4 + (q & 1);
                        const int idx = 4 * (q >> 1) + 2 * rr + (q & 1);
                        s_s1[d * S1_STRIDE + k] = (s32[mb][idx] + s16[mb][idx]) + s32[mb][idx + 8];
                    }
        }
        __syncthreads();
        if (tid < K) s_s0[tid] = (s_red[tid] + s_red[16 + tid]) + (s_red[32 + tid] + s_red[48 + tid]);
        float sacc[KT];
        if (own) {
#pragma unroll
            for (int k = 0; k < KT; ++k) sacc[k] = s_s1[tid * S1_STRIDE + k];
        }
        __syncthreads();
        // ---- gradient + diversity + Adam on the owned elements (ref model.py:385-397; SURVEY KA6)
        if (own) {
            const int sidx = L * ord + loop;                                  // this Adam step's bias corrections
            const float step_size = __ldg(prm.bc + 2 * sidx), bc2_sqrt = __ldg(prm.bc + 2 * sidx + 1);
            float newp[KT];
#pragma unroll
            for (int k = 0; k < KT; ++k) {
                newp[k] = p_[k];
                if (k < K) {
                    const float muv = p_[k];
                    const float s1 = sacc[k] * (1.0f / (X_SCALE * SR));
                    float g = -(s1 - muv * s_s0[k]) * s_w[k] / n_rows;
                    float esum = 0.f, emu = 0.f;
#pragma unroll
                    for (int j = 0; j < KT; ++j)
                        if (j < K) {
                            const float e = s_e[k * KT + j];                  // broadcast
                            esum += e;
                            emu = fmaf(e, p_[j], emu);                        // mu_j[d] is this thread's own register
                        }
                    g += div_scale * (esum * muv - emu);
                    const float mm = m_[k] + (g - m_[k]) * adam.omb1;             // torch.optim.Adam (_single_tensor_adam)
                    const float vv = v_[k] * adam.b2f + adam.omb2 * g * g;
                    const float denom = sqrtf(vv) / bc2_sqrt + adam.epsf;
                    newp[k] = muv - step_size * (mm / denom);
                    m_[k] = mm; v_[k] = vv;
                }
            }
#pragma unroll
            for (int k = 0; k < KT; ++k) p_[k] = newp[k];
        }
        __syncthreads();                                              // every reader of s_mu / s_s0 is done
        if (tid < K) s_pi[tid] = prm.tau * s_pi[tid] + prm.omtau * ((s_s0[tid] + EM_EPS) / n_rows);   // ref :385, :399, :297
        if (tid == 0) MGP_PROF(tile_ctr - 1, 7);
    }
    if (tid == 0) MGP_PROF(63, 4);
    replay(step0 + L * (ord + 1), L * (n_active - ord - 1), s_misc + 4);
    if (tid == 0) MGP_PROF(63, 5);
    write_back();
    if (tid < K) {
        if (prm.pi_out) prm.pi_out[(size_t)c * K + tid] = s_pi[tid];
        else prm.weight[(size_t)c * P + (size_t)c * K + tid] = s_pi[tid];
    }
    if (tid == 0) MGP_PROF(63, 6);
}

template <int D>
size_t em_tc_smem(int kt) {
    const size_t tr = em_rows(D), nx = em_one_wg(D) ? 2 : 1;
    return 1024 + nx * 2 * (size_t)(D / 64) * tr * 128 + (size_t)(D / 64) * 4096 + (tr / 64) * 4096 +
           (size_t)((D * S1_STRIDE * 4 + 15) & ~15) +
           ((size_t)kt * kt + 136 + 6 * 16 + 8 + 8 * (size_t)(32 * ((kt * (kt - 1) / 2 + kt + 31) / 32))) * 4 + 128;
}

}  // namespace

static long long* g_em_tc_prof = nullptr;
static int g_em_tc_prof_class = 0;
void mgp_em_tc_set_prof(void* p, int cls) { g_em_tc_prof = reinterpret_cast<long long*>(p); g_em_tc_prof_class = cls; }

bool mgp_em_tc_supported(int K, int D, int cap) {
    return K >= 2 && K <= 16 && (D == 128 || D == 256) && cap >= 1 && get_encode() != nullptr;
}

int mgp_em_tc_launch(const void* shadow_h, const void* shadow_l, const float* shadow_xx, const float* bias_corr, const int32_t* order,
                     const int32_t* sched, float* mu, const float* sigma, float* weight, float* exp_avg, float* exp_avg_sq,
                     int* status, int num_em_loop, float alpha, double lr, double beta1, double beta2, double adam_eps,
                     double tau, float lamda, float* mu_stage, float* pi_stage, int C, int K, int D, int cap,
                     cudaStream_t st) {
    CUtensorMap mh, ml;                             // boxes of em_rows(D) rows: one tile, hi and lo
    const uint64_t rows = (uint64_t)C * cap;
    if (!make_map_f16(&mh, shadow_h, rows, D, em_rows(D)) || !make_map_f16(&ml, shadow_l, rows, D, em_rows(D)))
        return MGP_ERR_UNSUPPORTED;
    EmTcParams prm;
    prm.xx = shadow_xx; prm.bc = bias_corr; prm.order = order; prm.sched = sched; prm.mu = mu; prm.sigma = sigma; prm.weight = weight;
    prm.exp_avg = exp_avg; prm.exp_avg_sq = exp_avg_sq; prm.status = status;
    prm.mu_out = mu_stage ? mu_stage : mu; prm.pi_out = pi_stage;
    prm.adam = make_adam(lr, beta1, beta2, adam_eps);
    prm.alpha = alpha; prm.tau = (float)tau; prm.omtau = (float)(1.0 - tau); prm.lamda = lamda;
    prm.num_em_loop = num_em_loop; prm.C = C; prm.K = K; prm.cap = cap;
    prm.prof = g_em_tc_prof; prm.prof_class = g_em_tc_prof_class;
    prm.clist = reinterpret_cast<const int32_t*>(bias_corr + (size_t)5 * num_em_loop * C + 4);
#define MGP_EMTC(DD, KK)                                                                                            \
    do {                                                                                                            \
        const size_t smem = em_tc_smem<DD>(KK);                                                                     \
        MGP_CUDA(cudaFuncSetAttribute(em_tc_kernel<DD, KK>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        em_tc_kernel<DD, KK><<<C, em_threads(DD), smem, st>>>(mh, ml, prm);                                         \
    } while (0)
#define MGP_EMTC_K(DD)                                                                                              \
    do {                                                                                                            \
        if (K <= 5) MGP_EMTC(DD, 5);                                                                                \
        else if (K <= 10) MGP_EMTC(DD, 10);                                                                         \
        else MGP_EMTC(DD, 16);                                                                                      \
    } while (0)
    if (D == 128) MGP_EMTC_K(128);
    else MGP_EMTC_K(256);
#undef MGP_EMTC_K
#undef MGP_EMTC
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}
