// Per-patch class log-densities over a feature map (ref model.py:403-421 _score, :323-336 _estimate_log_prob):
//
//   logp_c[b,c,hw] = logsumexp_k( lp_ck(x_n) + log(pi_ck + 1e-10) ),   lp with eps = 1e-10 in (sigma + eps), log(sigma + eps)
//   logp_all[b,hw] = logsumexp_c logp_c[b,c,hw]                         (per-patch log sum_c p(x|c))
//
// Tensor-core path (isotropic sigma, D in {64, 128}, K <= 64): the log-likelihood GEMM of logprob_tcz.cu, from the same
// mainloop (tc_rs_gemm.cuh: fp32 patch tiles split in registers into the fp16 hi / lo A fragments of wgmma, prototype
// tiles from the cached pre-pass operands of logprob_tc.cu through a TMA / mbarrier ring) with its own schedule and
// epilogue: nothing of [N,P] leaves the SM.
//   * class-aligned prototype tiles: tile t holds classes [t cpt, (t+1) cpt), cpt = floor(128 / K), i.e. the first
//     cpt K of the 128 MMA columns; the columns behind them (the next tile's classes, or zero fill past P) are computed
//     and ignored, so a class never straddles two tiles;
//   * each warpgroup writes log p + log(pi + 1e-10) of its 64 patches x cpt K prototypes into a column-major shared
//     tile [128 prototypes][68 floats] (the pitch puts the fragment stores of a warp on 32 different banks), then
//     thread u reads patch u % 64 and classes u / 64, u / 64 + 2, ...: K consecutive prototypes of a class sit in one
//     thread, a warp reads 32 consecutive patches (conflict-free), max then sum of exp, one plain store per output
//     element ([B,C,HW]: a warp stores 32 consecutive patches of one class) -- one writer, no atomics;
//   * the marginal over the classes: x-stationary schedule.  A CTA owns whole x tiles (tile i, i + grid, ...) and runs
//     every prototype tile against each, so the running (max, sum) of a patch over all its classes stays in the two
//     threads that own the patch; they merge through shared memory after the last prototype tile and one of them stores
//     logp_all.  No partials in HBM, no combine kernel; the order of every sum is fixed, so results are deterministic.
//
// Fallback (every other shape and math mode): mgp_logprob_fwd into a row-chunked [n, P] workspace, then
// log_density_lse_kernel (warp per patch row).
#include <cuda.h>
#include <cuda_fp16.h>

#include "mgp_common.cuh"
#include "tc_ptx.cuh"
#include "tc_rs_gemm.cuh"

namespace {
using namespace mgp_tc;
using namespace mgp_rs;

constexpr int RP = 68;             // pitch (floats) of the reduction tile [PT prototypes][64 patches]: 2 t RP = 8 t mod 32
constexpr uint32_t RED_BYTES = PT * RP * 4;
constexpr float PI_EPS = 1e-10f;   // ref model.py:415 torch.log(pi + eps)
constexpr long long FALLBACK_CHUNK_FLOATS = 16ll << 20;   // [n, P] rows of the fallback: at most 64 MiB per chunk

struct LdParams {
    const float* c0;               // e0 + log(pi + 1e-10) per prototype
    const float* e1;
    const float* e2;
    const int* noniso;
    float* out_bchw;
    float* out_bhw;                // may be null
    int N, B, HW, C, K;
    int cpt;                       // classes per prototype tile
    int n_xtiles, n_ptiles;
    int stages;                    // prototype ring depth
};

// (M, S) stands for M + log S; merge the partial (m, s) into it
__device__ __forceinline__ void lse_merge(float& M, float& S, float m, float s) {
    if (m == -INFINITY) return;
    if (m > M) {
        S = S * expf(M - m) + s;
        M = m;
    } else {
        S += s * expf(m - M);
    }
}

__device__ __forceinline__ float lse_value(float m, float s) { return m == -INFINITY ? -INFINITY : m + logf(s); }

template <int D>
__device__ __forceinline__ void log_density_tc_body(const CUtensorMap* map_x, const CUtensorMap* map_ph,
                                                    const CUtensorMap* map_pl, const LdParams& prm) {
    const int S = prm.stages;
    const RsSmem<D> sm(S, 2 * RED_BYTES);                      // epilogue region: two reduction tiles, one per warpgroup
    // behind the barriers: the row partials [2 warpgroups][64 patches] (max, sum)
    float2* s_part = reinterpret_cast<float2*>(sm.epi() + 2 * RED_BYTES + 256);

    if (*reinterpret_cast<const volatile int*>(prm.noniso) != 0) {
        // the caller asserted isotropic sigma and the prototype pre-pass found otherwise: NaN outputs, no fault
        const long long nc = (long long)prm.B * prm.C * prm.HW;
        for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < nc; i += (long long)gridDim.x * blockDim.x) {
            prm.out_bchw[i] = __int_as_float(0x7fc00000);
            if (prm.out_bhw && i < prm.N) prm.out_bhw[i] = __int_as_float(0x7fc00000);
        }
        return;
    }

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    init_barriers(sm);

    // x-stationary schedule: x tiles blockIdx.x, blockIdx.x + grid, ...; every prototype tile against each
    const int n_my_x = blockIdx.x < prm.n_xtiles ? (prm.n_xtiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    const int n_ptiles = prm.n_ptiles, K = prm.K;
    const int tile_rows = prm.cpt * K;                         // prototype rows a tile uses

    if (n_my_x == 0) {
        // nothing to do for this CTA
    } else if (warp == 9 && lane == 0) {
        produce_x_tiles(sm, map_x, n_my_x, [](int c) { return (int)(blockIdx.x + c * gridDim.x); });
    } else if (warp == 8 && lane == 0) {
        // 128 rows from the first row of the tile's classes
        produce_proto_tiles(sm, map_ph, map_pl, S, n_my_x, [](int) { return 0; }, [&](int) { return n_ptiles; },
                            [&](int pt) { return pt * tile_rows; });
    } else if (warp < 8) {
        // =========================== consumers: split, MMA, class log-sum-exp ===========================
        const int wg = warp >> 2, wq = warp & 3, g = lane >> 2, t = lane & 3;
        const int rA = wg * 64 + wq * 16 + g;                    // this thread's fragment rows of the tile: rA, rA + 8
        const int u = threadIdx.x & 127, rr = u & 63, par = u >> 6;   // reduction role: patch rr of the slice, classes par + 2 j
        float* red = reinterpret_cast<float*>(sm.epi() + (uint32_t)wg * RED_BYTES);
        const uint32_t wg_bar = 2 + wg;
        auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(wg_bar) : "memory"); };
        const int C = prm.C, HW = prm.HW;
        int stage = 0;
        uint32_t phase = 0;
        for (int c = 0; c < n_my_x; ++c) {
            const int row0 = (blockIdx.x + c * gridDim.x) * XT;
            uint32_t ah[RsSmem<D>::NKS][4], al[RsSmem<D>::NKS][4];
            float ssA, ssB;
            split_x_tile(sm, c, rA, lane, ah, al, ssA, ssB);

            const int n = row0 + wg * 64 + rr;                   // the patch this thread reduces
            const bool nok = n < prm.N;
            const int b = nok ? n / HW : 0, hw = n - b * HW;
            float run_m = -INFINITY, run_s = 0.f;                // over the classes par, par + 2, ... of every tile
            for (int pt = 0; pt < n_ptiles; ++pt) {
                float acc[64];
                mma_proto_tile(sm, acc, ah, al, S, lane, stage, phase);
                const int cls0 = pt * prm.cpt;
                const int ncls = min(prm.cpt, C - cls0);
                const int ncol = ncls * K, p0 = cls0 * K;
                // ---- weighted log p = c0 + e1 acc + e2 |x|^2 of the tile's valid columns -> reduction tile
                wg_sync();                                       // the previous tile's reducers are done with it
#pragma unroll
                for (int i = 0; i < 16; ++i) {
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const int col = 8 * i + 2 * t + j;
                        if (col < ncol) {
                            const float c0 = __ldg(prm.c0 + p0 + col), c1 = __ldg(prm.e1 + p0 + col), c2 = __ldg(prm.e2 + p0 + col);
                            float* dst = red + col * RP + (rA - wg * 64);
                            dst[0] = fmaf(c1, acc[4 * i + j], fmaf(c2, ssA, c0));
                            dst[8] = fmaf(c1, acc[4 * i + 2 + j], fmaf(c2, ssB, c0));
                        }
                    }
                }
                wg_sync();
                // ---- per (patch, class) log-sum-exp over the class's K prototypes
                for (int cl = par; cl < ncls; cl += 2) {
                    const float* src = red + cl * K * RP + rr;
                    float m = -INFINITY;
                    for (int k = 0; k < K; ++k) m = fmaxf(m, src[k * RP]);
                    float s = 0.f;
                    if (m != -INFINITY)
                        for (int k = 0; k < K; ++k) s += expf(src[k * RP] - m);
                    if (nok) prm.out_bchw[((long long)b * C + cls0 + cl) * HW + hw] = lse_value(m, s);
                    lse_merge(run_m, run_s, m, s);
                }
            }
            // ---- the marginal: merge the two class-parity partials of each patch
            if (prm.out_bhw) {
                if (par == 1) s_part[wg * 64 + rr] = make_float2(run_m, run_s);
                wg_sync();
                if (par == 0) {
                    const float2 o = s_part[wg * 64 + rr];
                    lse_merge(run_m, run_s, o.x, o.y);
                    if (nok) prm.out_bhw[n] = lse_value(run_m, run_s);
                }
                // (the next write of s_part comes after the next x tile's wg_syncs)
            }
        }
    }
}

__global__ void __launch_bounds__(RS_THREADS, 1)
log_density_tc_d64_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_ph,
                          const __grid_constant__ CUtensorMap map_pl, const LdParams prm) {
    log_density_tc_body<64>(&map_x, &map_ph, &map_pl, prm);
}

__global__ void __launch_bounds__(RS_THREADS, 1)
log_density_tc_d128_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_ph,
                           const __grid_constant__ CUtensorMap map_pl, const LdParams prm) {
    log_density_tc_body<128>(&map_x, &map_ph, &map_pl, prm);
}

// out[p] = (e0 ? e0[p] : 0) + log(pi_p + 1e-10), pi_p = weight[p / K, p] (the class-diagonal block of last_layer.weight)
__global__ void log_density_prior_kernel(const float* __restrict__ weight, const float* __restrict__ e0,
                                         float* __restrict__ out, int C, int K) {
    const int P = C * K;
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= P) return;
    const float lp = logf(weight[(size_t)(p / K) * P + p] + PI_EPS);
    out[p] = e0 ? e0[p] + lp : lp;
}

// Fallback reduction, warp per patch row of a chunk lp [n_rows, P] (rows n0 ...): lane j takes classes j, j + 32, ...
__global__ void log_density_lse_kernel(const float* __restrict__ lp, const float* __restrict__ lpi, long long n0,
                                       int n_rows, int HW, int C, int K, float* __restrict__ out_bchw,
                                       float* __restrict__ out_bhw) {
    const int r = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (r >= n_rows) return;
    const float* row = lp + (size_t)r * C * K;
    const long long n = n0 + r, b = n / HW;
    const int hw = (int)(n - b * HW);
    float M = -INFINITY, S = 0.f;
    for (int c = lane; c < C; c += 32) {
        const float* v = row + (size_t)c * K;
        const float* w = lpi + (size_t)c * K;
        float m = -INFINITY;
        for (int k = 0; k < K; ++k) m = fmaxf(m, v[k] + w[k]);
        float s = 0.f;
        if (m != -INFINITY)
            for (int k = 0; k < K; ++k) s += expf(v[k] + w[k] - m);
        out_bchw[(b * C + c) * HW + hw] = lse_value(m, s);
        lse_merge(M, S, m, s);
    }
    if (out_bhw) {
#pragma unroll
        for (int o = 16; o >= 1; o >>= 1) {
            const float mo = __shfl_xor_sync(0xffffffffu, M, o), so = __shfl_xor_sync(0xffffffffu, S, o);
            lse_merge(M, S, mo, so);
        }
        if (lane == 0) out_bhw[n] = lse_value(M, S);
    }
}

bool tc_shape(int K, int D) { return (D == 64 || D == 128) && K >= 1 && K <= 64 && get_encode() != nullptr; }
bool tc_math(int math) { return math == MGP_MATH_TC_ISO || math == MGP_MATH_TC_ISO_REUSE; }

// fallback: rows per chunk, and the math mode handed to mgp_logprob_fwd.  No operand reuse across chunks, and no
// isotropy assertion: logprob_tc.cu decides on the device at D <= 128, AUTO takes the exact SIMT kernel beyond, so a
// wrong assertion cannot fault
long long chunk_rows(long long N, int P) {
    long long r = FALLBACK_CHUNK_FLOATS / P;
    if (r < 1) r = 1;
    return r < N ? r : N;
}
int fallback_math(int math, int D) {
    if (math == MGP_MATH_TC_REUSE) return MGP_MATH_TC;
    if (tc_math(math)) return D <= 128 ? MGP_MATH_TC : MGP_MATH_AUTO;
    return math;
}

}  // namespace

// logprob_tc.cu
size_t mgp_logprob_tc_ws_bytes(long long N, int P, int D);
int mgp_logprob_tc_proto_prep(const float* mu, const float* sigma, float eps, float eps_log, void* ws, int P, int D,
                              int run, void** bh, void** bl, float** e0, float** e1, float** e2, int** flag,
                              cudaStream_t st);

extern "C" size_t mgp_log_density_ws_bytes(int B, int HW, int C, int K, int D, int math) {
    const long long P = (long long)C * K, N = (long long)B * HW;
    if (B <= 0 || HW <= 0 || C <= 0 || K <= 0 || D <= 0 || P > 0x7fffffffLL) return 0;
    if (tc_math(math) && tc_shape(K, D)) return align256(mgp_logprob_tc_ws_bytes(0, (int)P, D)) + align256((size_t)P * 4);
    const long long n = chunk_rows(N, (int)P);
    return align256(mgp_logprob_ws_bytes((int)n, 1, (int)P, D, fallback_math(math, D))) + align256((size_t)(n * P) * 4) +
           align256((size_t)P * 4);
}

extern "C" int mgp_log_density(const float* xhat_nd, const float* mu, const float* sigma, const float* weight_cp,
                               float* out_bchw, float* out_bhw, int B, int HW, int C, int K, int D, int math, void* ws,
                               size_t ws_bytes, void* stream) {
    if (!xhat_nd || !mu || !sigma || !weight_cp || !out_bchw || !ws) return MGP_ERR_INVALID;
    if (B <= 0 || HW <= 0 || C <= 0 || K <= 0 || D <= 0 || (D & 3)) return MGP_ERR_INVALID;
    if (math < MGP_MATH_FP32 || math > MGP_MATH_TC_ISO_REUSE) return MGP_ERR_INVALID;
    if (!mgp_aligned16(xhat_nd) || !mgp_aligned16(mu) || !mgp_aligned16(sigma) || !mgp_aligned16(ws))
        return MGP_ERR_INVALID;
    const long long N = (long long)B * HW, P = (long long)C * K;
    if (N > 0x7fffffffLL || P > 0x7fffffffLL) return MGP_ERR_UNSUPPORTED;
    if (ws_bytes < mgp_log_density_ws_bytes(B, HW, C, K, D, math)) return MGP_ERR_WORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    uint8_t* wsb = reinterpret_cast<uint8_t*>(ws);

    if (tc_math(math) && tc_shape(K, D)) {
        void *bh, *bl;
        float *e0, *e1, *e2;
        int* flag;
        const size_t o_c0 = align256(mgp_logprob_tc_ws_bytes(0, (int)P, D));
        float* c0 = reinterpret_cast<float*>(wsb + o_c0);
        // the prototype pre-pass of logprob_tc.cu with _estimate_log_prob's eps (skipped for MGP_MATH_TC_ISO_REUSE)
        const int rc = mgp_logprob_tc_proto_prep(mu, sigma, 1e-10f, 1e-10f, ws, (int)P, D, math == MGP_MATH_TC_ISO,
                                                 &bh, &bl, &e0, &e1, &e2, &flag, st);
        if (rc != MGP_OK) return rc;
        log_density_prior_kernel<<<(unsigned)((P + 255) / 256), 256, 0, st>>>(weight_cp, e0, c0, C, K);
        MGP_CHECK_LAUNCH();
        CUtensorMap mx, mph, mpl;
        if (!make_map_x(&mx, xhat_nd, (uint64_t)N, (uint64_t)D) || !make_map_f16(&mph, bh, (uint64_t)P, 2 * (uint64_t)D, PT) ||
            !make_map_f16(&mpl, bl, (uint64_t)P, 2 * (uint64_t)D, PT))
            return MGP_ERR_UNSUPPORTED;
        LdParams prm;
        prm.c0 = c0; prm.e1 = e1; prm.e2 = e2; prm.noniso = flag;
        prm.out_bchw = out_bchw; prm.out_bhw = out_bhw;
        prm.N = (int)N; prm.B = B; prm.HW = HW; prm.C = C; prm.K = K;
        prm.cpt = PT / K;
        prm.n_xtiles = (int)((N + XT - 1) / XT);
        prm.n_ptiles = (C + prm.cpt - 1) / prm.cpt;
        int sms = 0;
        MGP_CUDA(mgp_sm_count(&sms));
        size_t smem;
        if (!rs_smem_plan(D, 2 * RED_BYTES + 2 * 64 * 8, &prm.stages, &smem)) return MGP_ERR_UNSUPPORTED;
        const int grid = prm.n_xtiles < sms ? prm.n_xtiles : sms;
        if (D == 64) {
            MGP_CUDA(cudaFuncSetAttribute(log_density_tc_d64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            log_density_tc_d64_kernel<<<grid, RS_THREADS, smem, st>>>(mx, mph, mpl, prm);
        } else {
            MGP_CUDA(cudaFuncSetAttribute(log_density_tc_d128_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            log_density_tc_d128_kernel<<<grid, RS_THREADS, smem, st>>>(mx, mph, mpl, prm);
        }
        MGP_CHECK_LAUNCH();
        return MGP_OK;
    }

    // fallback: the existing log-likelihood into bounded [n, P] chunks, then the log-sum-exp reduction
    const int fm = fallback_math(math, D);
    const long long n_chunk = chunk_rows(N, (int)P);
    const size_t lp_ws = align256(mgp_logprob_ws_bytes((int)n_chunk, 1, (int)P, D, fm));
    float* chunk = reinterpret_cast<float*>(wsb + lp_ws);
    float* lpi = reinterpret_cast<float*>(wsb + lp_ws + align256((size_t)(n_chunk * P) * 4));
    log_density_prior_kernel<<<(unsigned)((P + 255) / 256), 256, 0, st>>>(weight_cp, nullptr, lpi, C, K);
    MGP_CHECK_LAUNCH();
    for (long long n0 = 0; n0 < N; n0 += n_chunk) {
        const int rows = (int)(N - n0 < n_chunk ? N - n0 : n_chunk);
        const int rc = mgp_logprob_fwd(xhat_nd + n0 * D, mu, sigma, 1e-10f, 1e-10f, chunk, MGP_OUT_LOGP_NP, rows, 1,
                                       (int)P, D, fm, ws, lp_ws, stream);
        if (rc != MGP_OK) return rc;
        log_density_lse_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, st>>>(chunk, lpi, n0, rows, HW, C, K, out_bchw,
                                                                            out_bhw);
        MGP_CHECK_LAUNCH();
    }
    return MGP_OK;
}
