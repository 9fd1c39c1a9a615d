// a2 (compute_log_prob, [N,P] output) on the tensor cores with the PATCH operands resident in registers.
//
// logprob_tc.cu feeds both operands of every MMA from shared memory and needs a separate pass that splits x into fp16
// hi/lo operands in HBM (25.7 MB read, 2 x 25.7 MB written and read back at cfg2).  Here:
//   * the GEMM is the register-operand mainloop of tc_rs_gemm.cuh (shared with log_density.cu): the fp32 patch tile
//     [128 x D] is TMA-loaded as it is and split in registers into the fp16 hi / lo A fragments of wgmma (RS form), so
//     there is no operand pre-pass over x; they stay for the 3 * D/16 MMAs of every prototype tile the CTA visits with
//     this x tile; only the prototype tiles (B operand, the small side: 2 * P * D * 2 bytes in total, L2-resident)
//     stream through a TMA / mbarrier ring in shared memory;
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
#include "tc_rs_gemm.cuh"

namespace {
using namespace mgp_tc;
using namespace mgp_rs;

constexpr int STG = 2048;          // one [16 rows x 32 floats] output block; two per consumer warp

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

template <int D>
__global__ void __launch_bounds__(RS_THREADS, 1)
logprob_z_kernel(const __grid_constant__ CUtensorMap map_x, const __grid_constant__ CUtensorMap map_ph,
                 const __grid_constant__ CUtensorMap map_pl, const __grid_constant__ CUtensorMap map_out,
                 const ZParams prm) {
    const int S = prm.stages;
    const RsSmem<D> sm(S, 8 * 2 * STG);                       // epilogue region: 8 warps x 2 output blocks
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    init_barriers(sm);

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
        produce_x_tiles(sm, &map_x, n_my_x, [&](int c) { return xt_first + c; });
    } else if (warp == 8 && lane == 0) {
        produce_proto_tiles(sm, &map_ph, &map_pl, S, n_my_x, p_begin, p_end, [](int pt) { return pt * PT; });
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
            uint32_t ah[RsSmem<D>::NKS][4], al[RsSmem<D>::NKS][4];
            float ssA, ssB;
            split_x_tile(sm, c, rA, lane, ah, al, ssA, ssB);
            for (int pt = p_begin(c); pt < p_end(c); ++pt) {
                float acc[64];
                mma_proto_tile(sm, acc, ah, al, S, lane, stage, phase);
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
                        uint8_t* stg = sm.epi() + (uint32_t)(warp * 2 + sbuf) * STG;
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
    int sms = 0;
    MGP_CUDA(mgp_sm_count(&sms));
    size_t smem;
    if (!rs_smem_plan(D, 8 * 2 * STG, &prm.stages, &smem)) return MGP_ERR_UNSUPPORTED;
    const long long n_pairs = (long long)prm.n_xtiles * prm.n_ptiles;
    const int grid = (int)(n_pairs < sms ? n_pairs : sms);
#define MGP_Z_LAUNCH(DD)                                                                                           \
    do {                                                                                                           \
        MGP_CUDA(cudaFuncSetAttribute(logprob_z_kernel<DD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        logprob_z_kernel<DD><<<grid, RS_THREADS, smem, st>>>(mx, mph, mpl, mout, prm);                                     \
    } while (0)
    if (D == 64) MGP_Z_LAUNCH(64);
    else MGP_Z_LAUNCH(128);
#undef MGP_Z_LAUNCH
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}
