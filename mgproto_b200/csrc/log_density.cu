// Per-patch class log-densities over a feature map (ref model.py:403-421 _score, :323-336 _estimate_log_prob):
//
//   logp_c[b,c,hw] = logsumexp_k( lp_ck(x_n) + log(pi_ck + 1e-10) ),   lp with eps = 1e-10 in (sigma + eps), log(sigma + eps)
//   logp_all[b,hw] = logsumexp_c logp_c[b,c,hw]                         (per-patch log sum_c p(x|c))
//
// Tensor-core path (isotropic sigma, D in {64, 128}, K <= 64): the log-likelihood GEMM of logprob_tcz.cu -- fp32 patch
// tiles TMA-loaded and split in registers into the fp16 hi / lo A fragments of wgmma (RS form), prototype tiles from the
// cached pre-pass operands of logprob_tc.cu through a TMA / mbarrier ring, hi*hi + lo*hi + hi*lo in fp32 accumulators --
// with a new epilogue: nothing of [N,P] leaves the SM.
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

namespace {
using namespace mgp_tc;

constexpr int LT = 320;            // threads: warps 0-7 two consumer warpgroups, 8 prototype TMA, 9 patch-tile TMA
constexpr int PT = 128;            // MMA columns per prototype tile (wgmma N)
constexpr int XT = 128;            // patches per x tile (two warpgroups x m64)
constexpr int KB = 64;             // K elements per prototype smem block (128 B rows)
constexpr int PSUB = PT * KB * 2;  // one [128 x 64] fp16 block = 16 KiB
constexpr int RP = 68;             // pitch (floats) of the reduction tile [PT prototypes][64 patches]: 2 t RP = 8 t mod 32
constexpr uint32_t RED_BYTES = PT * RP * 4;
constexpr float X_SCALE = 256.0f;
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

__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
    return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

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
    constexpr int NKB = D / KB;                    // prototype K blocks per tile
    constexpr int NKS = D / 16;                    // k16 steps
    constexpr int NXB = D / 32;                    // fp32 landing blocks of [128 rows x 32 floats] (128 B rows, swizzled)
    constexpr uint32_t XB_BYTES = XT * 128;
    constexpr uint32_t X_BYTES = NXB * XB_BYTES;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* bp = smem_raw + (base - raw);
    const int S = prm.stages;
    const uint32_t o_x = 0;                                    // fp32 landing tile
    const uint32_t o_ring = X_BYTES;                           // S x (proto hi, proto lo)
    const uint32_t o_red = o_ring + (uint32_t)S * 2 * PSUB;    // two reduction tiles, one per warpgroup
    const uint32_t o_misc = o_red + 2 * RED_BYTES;             // barriers, then the row partials
    const uint32_t bar0 = base + o_misc;                       // full[8] empty[8] xfull xempty
    auto FULL = [&](int i) { return bar0 + 8u * i; };
    auto EMPTY = [&](int i) { return bar0 + 8u * (8 + i); };
    const uint32_t XFULL = bar0 + 8u * 16, XEMPTY = bar0 + 8u * 17;
    float2* s_part = reinterpret_cast<float2*>(bp + o_misc + 256);   // [2 warpgroups][64 patches] (max, sum)

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
    if (threadIdx.x == 0) {
        for (int i = 0; i < 8; ++i) { mbar_init(FULL(i), 1); mbar_init(EMPTY(i), 8); }   // empty: one arrive per consumer warp
        mbar_init(XFULL, 1);
        mbar_init(XEMPTY, 8);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // x-stationary schedule: x tiles blockIdx.x, blockIdx.x + grid, ...; every prototype tile against each
    const int n_my_x = blockIdx.x < prm.n_xtiles ? (prm.n_xtiles - 1 - blockIdx.x) / gridDim.x + 1 : 0;
    const int n_ptiles = prm.n_ptiles, K = prm.K;
    const int tile_rows = prm.cpt * K;                         // prototype rows a tile uses

    if (n_my_x == 0) {
        // nothing to do for this CTA
    } else if (warp == 9 && lane == 0) {
        // =========================== fp32 patch-tile producer (the next tile lands under the current one's MMAs) =====
        for (int c = 0; c < n_my_x; ++c) {
            if (c > 0) mbar_wait(XEMPTY, (uint32_t)((c - 1) & 1));   // the consumers converted the previous tile
            mbar_expect_tx(XFULL, X_BYTES);
            const int xt = blockIdx.x + c * gridDim.x;
#pragma unroll
            for (int b = 0; b < NXB; ++b) tma_load_2d(base + o_x + b * XB_BYTES, map_x, b * 32, xt * XT, XFULL);
        }
    } else if (warp == 8 && lane == 0) {
        // =========================== prototype TMA producer: 128 rows from the first row of the tile's classes =====
        int stage = 0;
        uint32_t phase = 0;
        for (int c = 0; c < n_my_x; ++c)
            for (int pt = 0; pt < n_ptiles; ++pt)
                for (int kb = 0; kb < NKB; ++kb) {
                    mbar_wait(EMPTY(stage), phase ^ 1u);
                    mbar_expect_tx(FULL(stage), 2 * PSUB);
                    const uint32_t dst = base + o_ring + (uint32_t)stage * 2 * PSUB;
                    tma_load_2d(dst, map_ph, D + kb * KB, pt * tile_rows, FULL(stage));   // the [-2 w mu] half of [P, 2D]
                    tma_load_2d(dst + PSUB, map_pl, D + kb * KB, pt * tile_rows, FULL(stage));
                    if (++stage == S) { stage = 0; phase ^= 1u; }
                }
    } else if (warp < 8) {
        // =========================== consumers: split, MMA, class log-sum-exp ===========================
        const int wg = warp >> 2, wq = warp & 3, g = lane >> 2, t = lane & 3;
        const int rA = wg * 64 + wq * 16 + g;                    // this thread's fragment rows of the tile: rA, rA + 8
        const int u = threadIdx.x & 127, rr = u & 63, par = u >> 6;   // reduction role: patch rr of the slice, classes par + 2 j
        float* red = reinterpret_cast<float*>(bp + o_red + (uint32_t)wg * RED_BYTES);
        const uint32_t wg_bar = 2 + wg;
        auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(wg_bar) : "memory"); };
        const int C = prm.C, HW = prm.HW;
        int stage = 0;
        uint32_t phase = 0;
        for (int c = 0; c < n_my_x; ++c) {
            const int row0 = (blockIdx.x + c * gridDim.x) * XT;
            // ---- fused operand split: fp32 landing tile -> A fragments (hi, lo of 256 x) + |x|^2 of rows rA, rA + 8
            uint32_t ah[NKS][4], al[NKS][4];
            float ssA = 0.f, ssB = 0.f;
            mbar_wait(XFULL, (uint32_t)(c & 1));
#pragma unroll
            for (int ks = 0; ks < NKS; ++ks) {
#pragma unroll
                for (int q = 0; q < 4; ++q) {                    // fragment register q: row rA + 8 (q & 1), k 16 ks + 2 t + 8 (q >> 1)
                    const int r = rA + 8 * (q & 1), col = 16 * ks + 2 * t + 8 * (q >> 1), w = col & 31;
                    const float2 v = *reinterpret_cast<const float2*>(
                        bp + o_x + (uint32_t)(col >> 5) * XB_BYTES + (uint32_t)r * 128u + ((((w >> 2) ^ (r & 7)) & 7) << 4) + (w & 3) * 4);
                    if (q & 1) ssB = fmaf(v.x, v.x, fmaf(v.y, v.y, ssB)); else ssA = fmaf(v.x, v.x, fmaf(v.y, v.y, ssA));
                    const float s0 = v.x * X_SCALE, s1 = v.y * X_SCALE;
                    const __half h0 = __float2half_rn(s0), h1 = __float2half_rn(s1);
                    ah[ks][q] = pack_h2(h0, h1);
                    al[ks][q] = pack_h2(__float2half_rn(s0 - __half2float(h0)), __float2half_rn(s1 - __half2float(h1)));
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(XEMPTY);                  // landing tile consumed: the next one may land
            ssA += __shfl_xor_sync(0xffffffffu, ssA, 1); ssA += __shfl_xor_sync(0xffffffffu, ssA, 2);
            ssB += __shfl_xor_sync(0xffffffffu, ssB, 1); ssB += __shfl_xor_sync(0xffffffffu, ssB, 2);

            const int n = row0 + wg * 64 + rr;                   // the patch this thread reduces
            const bool nok = n < prm.N;
            const int b = nok ? n / HW : 0, hw = n - b * HW;
            float run_m = -INFINITY, run_s = 0.f;                // over the classes par, par + 2, ... of every tile
            for (int pt = 0; pt < n_ptiles; ++pt) {
                float acc[64];
#pragma unroll
                for (int j = 0; j < 64; ++j) acc[j] = 0.f;
                for (int kb = 0; kb < NKB; ++kb) {
                    mbar_wait(FULL(stage), phase);
                    const uint32_t ph = base + o_ring + (uint32_t)stage * 2 * PSUB, pl = ph + PSUB;
                    wg_fence();
#pragma unroll
                    for (int k = 0; k < KB / 16; ++k) {
                        const int ks = (kb * KB) / 16 + k;
                        const uint64_t b_h = gmma_desc(ph + (uint32_t)k * 32u), b_l = gmma_desc(pl + (uint32_t)k * 32u);
                        wg_mma_rs_n128(acc, ah[ks], b_h);
                        wg_mma_rs_n128(acc, al[ks], b_h);
                        wg_mma_rs_n128(acc, ah[ks], b_l);
                    }
                    wg_commit();
                    wg_wait0();
                    __syncwarp();
                    if (lane == 0) mbar_arrive(EMPTY(stage));    // this warp no longer reads the stage
                    if (++stage == S) { stage = 0; phase ^= 1u; }
                }
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

__global__ void __launch_bounds__(LT, 1)
log_density_tc_d64_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_ph,
                          const __grid_constant__ CUtensorMap map_pl, const LdParams prm) {
    log_density_tc_body<64>(&map_x, &map_ph, &map_pl, prm);
}

__global__ void __launch_bounds__(LT, 1)
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

bool make_map_x(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {cols * 4};
    cuuint32_t box[2] = {32, XT};
    cuuint32_t es[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(ptr), dims, strides, box, es,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

size_t align256(size_t v) { return (v + 255) & ~(size_t)255; }

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
        int dev = 0, sms = 0;
        MGP_CUDA(cudaGetDevice(&dev));
        MGP_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
        const size_t x_bytes = (size_t)XT * D * 4, fixed = 1024 + x_bytes + 2 * RED_BYTES + 256 + 2 * 64 * 8;
        const size_t smem_max = 227 * 1024;
        int stages = (int)((smem_max - fixed) / (2 * PSUB));
        if (stages > 8) stages = 8;
        if (stages < 2) return MGP_ERR_UNSUPPORTED;
        prm.stages = stages;
        const size_t smem = fixed + (size_t)stages * 2 * PSUB;
        const int grid = prm.n_xtiles < sms ? prm.n_xtiles : sms;
        if (D == 64) {
            MGP_CUDA(cudaFuncSetAttribute(log_density_tc_d64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            log_density_tc_d64_kernel<<<grid, LT, smem, st>>>(mx, mph, mpl, prm);
        } else {
            MGP_CUDA(cudaFuncSetAttribute(log_density_tc_d128_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
            log_density_tc_d128_kernel<<<grid, LT, smem, st>>>(mx, mph, mpl, prm);
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
