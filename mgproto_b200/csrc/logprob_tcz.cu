// a2 (compute_log_prob, [N,P] output) on the tensor cores with the PATCH operands resident in registers.
//
// logprob_tc.cu feeds both operands of every MMA from shared memory and needs a separate pass that splits x into fp16
// hi/lo operands in HBM (25.7 MB read, 2 x 25.7 MB written and read back at cfg2).  Here:
//   * the fp32 patch tile [128 x D] is TMA-loaded as it is (no operand pre-pass over x: the split is fused); each of the
//     two consumer warpgroups converts its 64-patch slice in registers to fp16 hi / lo of 256 x, laid out as the A
//     fragments of wgmma.mma_async (RS form), where they stay for the 3 * D/16 MMAs of every prototype tile the CTA
//     visits with this x tile; |x|^2 of the rank-1 epilogue term is summed in the same pass;
//   * only the prototype tiles (B operand, the small side: 2 * P * D * 2 bytes in total, L2-resident) stream through a
//     TMA / mbarrier ring in shared memory; the next fp32 patch tile lands under the current one's MMAs;
//   * accumulator rows are patches and columns prototypes, so the fragments of a warp are 16 consecutive output rows:
//     they go, with the affine fix-up, into 128B-swizzled [16 rows x 32 floats] blocks (conflict-free float2 stores)
//     and out through asynchronous TMA bulk tensor stores (plain stores from the row owners if P % 4 != 0);
//   * balanced schedule: CTA i owns the pairs [i U / G, (i+1) U / G) of the x-major list of (x tile, prototype tile)
//     pairs, so every CTA gets U / G pairs +- 1 however the x tiles divide by the grid.
//
// Shapes: sigma constant over d inside every prototype (inner dimension K = D; the caller asserts it, the kernel traps
// if the prototype pre-pass says otherwise) and D in {64, 128}: the hi / lo fragments of a 64 x D slice take D / 2
// registers per thread next to the 64 of the accumulator.  Everything else takes logprob_tc.cu.
//
// Warps: 0-7 two consumer warpgroups (convert, MMA, epilogue) | 8 prototype TMA producer | 9 patch-tile TMA producer.
#include <cuda.h>
#include <cuda_fp16.h>

#include "mgp_common.cuh"
#include "tc_ptx.cuh"

namespace {
using namespace mgp_tc;

constexpr int ZT = 320;            // threads
constexpr int PT = 128;            // prototypes per tile (wgmma N)
constexpr int XT = 128;            // patches per tile (two warpgroups x m64)
constexpr int KB = 64;             // K elements per prototype smem block (128 B rows)
constexpr int PSUB = PT * KB * 2;  // one [128 x 64] fp16 block = 16 KiB
constexpr int STG = 2048;          // one [16 rows x 32 floats] output block; two per consumer warp
constexpr float X_SCALE = 256.0f;

struct ZParams {
    const float* e0;
    const float* e1;
    const float* e2;
    const int* noniso;
    float* out;
    int N, P;
    int n_xtiles, n_ptiles;
    int stages;                    // prototype ring depth
};

__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
    return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}

template <int D>
__global__ void __launch_bounds__(ZT, 1)
logprob_z_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_ph,
                 const __grid_constant__ CUtensorMap map_pl, const __grid_constant__ CUtensorMap map_out,
                 const ZParams prm) {
    constexpr int NKB = D / KB;                    // prototype K blocks per tile
    constexpr int NKS = D / 16;                    // k16 steps
    constexpr int NXB = D / 32;                    // fp32 landing blocks of [128 rows x 32 floats] (128 B rows, swizzled)
    constexpr uint32_t XB_BYTES = XT * 128;        // 16 KiB
    constexpr uint32_t X_BYTES = NXB * XB_BYTES;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;
    uint8_t* bp = smem_raw + (base - raw);
    const int S = prm.stages;
    const uint32_t o_x = 0;                                    // fp32 landing tile
    const uint32_t o_ring = X_BYTES;                           // S x (proto hi, proto lo)
    const uint32_t o_stg = o_ring + (uint32_t)S * 2 * PSUB;    // 8 warps x 2 output blocks
    const uint32_t o_misc = o_stg + 8 * 2 * STG;
    const uint32_t bar0 = base + o_misc;                       // full[8] empty[8] xfull xempty
    auto FULL = [&](int i) { return bar0 + 8u * i; };
    auto EMPTY = [&](int i) { return bar0 + 8u * (8 + i); };
    const uint32_t XFULL = bar0 + 8u * 16, XEMPTY = bar0 + 8u * 17;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int i = 0; i < 8; ++i) { mbar_init(FULL(i), 1); mbar_init(EMPTY(i), 8); }   // empty: one arrive per consumer warp
        mbar_init(XFULL, 1);
        mbar_init(XEMPTY, 8);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int n_ptiles = prm.n_ptiles;
    const long long n_pairs = (long long)prm.n_xtiles * n_ptiles;
    const long long u0 = n_pairs * blockIdx.x / gridDim.x, u1 = n_pairs * (blockIdx.x + 1) / gridDim.x;
    const int xt_first = (int)(u0 / n_ptiles), xt_last = (int)((u1 - 1) / n_ptiles);
    const int n_my_x = u1 > u0 ? xt_last - xt_first + 1 : 0;
    auto p_begin = [&](int c) { return c == 0 ? (int)(u0 - (long long)xt_first * n_ptiles) : 0; };
    auto p_end = [&](int c) { return (xt_first + c == xt_last) ? (int)(u1 - (long long)xt_last * n_ptiles) : n_ptiles; };

    if (n_my_x == 0) {
        // nothing to do for this CTA (tiny problems)
    } else if (warp == 9 && lane == 0) {
        // =========================== fp32 patch-tile producer (the next tile lands under the current one's MMAs) =====
        for (int c = 0; c < n_my_x; ++c) {
            if (c > 0) mbar_wait(XEMPTY, (uint32_t)((c - 1) & 1));   // the consumers converted the previous tile
            mbar_expect_tx(XFULL, X_BYTES);
#pragma unroll
            for (int b = 0; b < NXB; ++b) tma_load_2d(base + o_x + b * XB_BYTES, &map_x, b * 32, (xt_first + c) * XT, XFULL);
        }
    } else if (warp == 8 && lane == 0) {
        // =========================== prototype TMA producer ===========================
        int stage = 0;
        uint32_t phase = 0;
        for (int c = 0; c < n_my_x; ++c)
            for (int pt = p_begin(c); pt < p_end(c); ++pt)
                for (int kb = 0; kb < NKB; ++kb) {
                    mbar_wait(EMPTY(stage), phase ^ 1u);
                    mbar_expect_tx(FULL(stage), 2 * PSUB);
                    const uint32_t dst = base + o_ring + (uint32_t)stage * 2 * PSUB;
                    tma_load_2d(dst, &map_ph, D + kb * KB, pt * PT, FULL(stage));    // the [-2 w mu] half of [P, 2D]
                    tma_load_2d(dst + PSUB, &map_pl, D + kb * KB, pt * PT, FULL(stage));
                    if (++stage == S) { stage = 0; phase ^= 1u; }
                }
    } else if (warp < 8) {
        // =========================== consumers ===========================
        if (*reinterpret_cast<const volatile int*>(prm.noniso) != 0) __trap();   // the caller asserted isotropic sigma
        const int wg = warp >> 2, wq = warp & 3, g = lane >> 2, t = lane & 3;
        const int rA = wg * 64 + wq * 16 + g;                    // this thread's patch rows of the tile: rA, rA + 8
        const bool tma_out = (prm.P & 3) == 0;                   // row pitch must be a multiple of 16 B
        int stage = 0, sbuf = 0;
        uint32_t phase = 0;
        for (int c = 0; c < n_my_x; ++c) {
            const int row0 = (xt_first + c) * XT;
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
            for (int pt = p_begin(c); pt < p_end(c); ++pt) {
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
                // ---- epilogue: log p = e0 + e1 acc + e2 |x|^2, 4 blocks of [16 patches x 32 prototypes] per warp
#pragma unroll
                for (int ch = 0; ch < 4; ++ch) {
                    const int p0 = pt * PT + ch * 32;
                    // epilogue constants of prototype column p (read per n8 block: keeps them out of the live set)
                    auto ev = [&](int p, float& c0, float& c1, float& c2) {
                        const bool ok = p < prm.P;
                        c0 = ok ? __ldg(prm.e0 + p) : 0.f;
                        c1 = ok ? __ldg(prm.e1 + p) : 0.f;
                        c2 = ok ? __ldg(prm.e2 + p) : 0.f;
                    };
                    if (tma_out) {
                        uint8_t* stg = bp + o_stg + (uint32_t)(warp * 2 + sbuf) * STG;
                        if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 1;" ::: "memory");   // this block's previous store has read it
                        __syncwarp();
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int cc = 8 * i + 2 * t;
                            float a0, a1, a2, b0, b1, b2;
                            ev(p0 + cc, a0, a1, a2);
                            ev(p0 + cc + 1, b0, b1, b2);
#pragma unroll
                            for (int rr = 0; rr < 2; ++rr) {
                                const int idx = 4 * (4 * ch + i) + 2 * rr, r16 = g + 8 * rr;
                                const float sn = rr ? ssB : ssA;
                                const float v0 = fmaf(a1, acc[idx], fmaf(a2, sn, a0));
                                const float v1 = fmaf(b1, acc[idx + 1], fmaf(b2, sn, b0));
                                *reinterpret_cast<float2*>(stg + r16 * 128 + ((((cc >> 2) ^ (r16 & 7)) & 7) << 4) + (cc & 3) * 4) =
                                    make_float2(v0, v1);
                            }
                        }
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                        __syncwarp();
                        if (lane == 0) {
                            tma_store_2d(&map_out, smem_u32(stg), p0, row0 + wg * 64 + wq * 16);
                            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
                        }
                        sbuf ^= 1;
                    } else {
#pragma unroll
                        for (int i = 0; i < 4; ++i)
#pragma unroll
                            for (int rr = 0; rr < 2; ++rr)
#pragma unroll
                                for (int j = 0; j < 2; ++j) {
                                    const int n = row0 + rA + 8 * rr, p = p0 + 8 * i + 2 * t + j;
                                    const float sn = rr ? ssB : ssA;
                                    float c0, c1, c2;
                                    ev(p, c0, c1, c2);
                                    if (n < prm.N && p < prm.P)
                                        prm.out[(size_t)n * prm.P + p] = fmaf(c1, acc[4 * (4 * ch + i) + 2 * rr + j], fmaf(c2, sn, c0));
                                }
                    }
                }
            }
        }
        if (lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // my TMA stores have landed
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

// output [N, P] fp32, box = 32 prototypes x 16 patches, 128B swizzle (inner box = 128 B)
bool make_map_out(CUtensorMap* m, const void* ptr, uint64_t N, uint64_t P) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[2] = {P, N};
    cuuint64_t strides[1] = {P * 4};
    cuuint32_t box[2] = {32, 16};
    cuuint32_t es[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(ptr), dims, strides, box, es,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace

bool mgp_logprob_tcz_supported(int P, int D) { return (D == 64 || D == 128) && P >= 1 && get_encode() != nullptr; }

int mgp_logprob_tcz_launch(const float* xhat, const void* bh, const void* bl, const float* e0, const float* e1,
                           const float* e2, const int* noniso, float* out, long long N, int P, int D, cudaStream_t st) {
    CUtensorMap mx, mph, mpl, mout;
    if ((P & 3) == 0) {
        if (!make_map_out(&mout, out, (uint64_t)N, (uint64_t)P)) return MGP_ERR_UNSUPPORTED;
    } else if (!make_map_out(&mout, bh, 64, 64)) {             // (unused by the kernel: any valid map)
        return MGP_ERR_UNSUPPORTED;
    }
    if (!make_map_x(&mx, xhat, (uint64_t)N, (uint64_t)D) || !make_map_f16(&mph, bh, (uint64_t)P, 2 * (uint64_t)D, PT) ||
        !make_map_f16(&mpl, bl, (uint64_t)P, 2 * (uint64_t)D, PT))
        return MGP_ERR_UNSUPPORTED;
    ZParams prm;
    prm.e0 = e0; prm.e1 = e1; prm.e2 = e2; prm.noniso = noniso; prm.out = out;
    prm.N = (int)N; prm.P = P;
    prm.n_xtiles = (int)((N + XT - 1) / XT);
    prm.n_ptiles = (P + PT - 1) / PT;
    int dev = 0, sms = 0;
    MGP_CUDA(cudaGetDevice(&dev));
    MGP_CUDA(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const size_t x_bytes = (size_t)XT * D * 4;
    int stages = (int)((227 * 1024 - 1024 - 256 - 8 * 2 * STG - x_bytes) / (2 * PSUB));
    if (stages > 8) stages = 8;
    if (stages < 2) return MGP_ERR_UNSUPPORTED;
    prm.stages = stages;
    const long long n_pairs = (long long)prm.n_xtiles * prm.n_ptiles;
    const int grid = (int)(n_pairs < sms ? n_pairs : sms);
    const size_t smem = 1024 + x_bytes + (size_t)stages * 2 * PSUB + 8 * 2 * STG + 256;
#define MGP_Z_LAUNCH(DD)                                                                                           \
    do {                                                                                                           \
        MGP_CUDA(cudaFuncSetAttribute(logprob_z_kernel<DD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        logprob_z_kernel<DD><<<grid, ZT, smem, st>>>(mx, mph, mpl, mout, prm);                                     \
    } while (0)
    if (D == 64) MGP_Z_LAUNCH(64);
    else MGP_Z_LAUNCH(128);
#undef MGP_Z_LAUNCH
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}
