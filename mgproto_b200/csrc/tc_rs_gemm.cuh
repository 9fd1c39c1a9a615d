// The register-operand (RS) log-likelihood GEMM of logprob_tcz.cu ([N,P] output) and log_density.cu (class
// log-densities), which differ only in their schedule, their response to a false isotropy assertion and their epilogue.
//
//   * the fp32 patch tile [128 x D] is TMA-loaded as it is into a 128B-swizzled landing tile; each of the two consumer
//     warpgroups converts its 64-patch slice in registers to the fp16 hi / lo A fragments of X_SCALE x (RS form of
//     wgmma.mma_async), where they stay for every prototype tile the CTA runs against this x tile; |x|^2 of the
//     rank-1 epilogue term is summed in the same pass;
//   * the prototype tiles (B operand: the [-2 w mu] half of the [P, 2D] pre-pass operands of logprob_tc.cu, hi and lo)
//     stream through a TMA / mbarrier ring; the next fp32 patch tile lands under the current one's MMAs;
//   * per prototype tile, hi*hi + lo*hi + hi*lo into one m64n128 fp32 accumulator per warpgroup.
//
// Warps: 0-7 two consumer warpgroups | 8 prototype TMA producer | 9 patch-tile TMA producer.  Shared memory, from a
// 1024 B-aligned base: the landing tile, the ring, the kernel's own epilogue region, then the barriers
// full[8] empty[8] xfull xempty (256 B) and whatever the kernel keeps behind them.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>

#include "mgp_common.cuh"
#include "tc_ptx.cuh"

namespace mgp_rs {
using namespace mgp_tc;

constexpr int RS_THREADS = 320;    // warps 0-7 consumers, 8 prototype TMA, 9 patch-tile TMA
constexpr int PT = 128;            // MMA columns per prototype tile (wgmma N)
constexpr int XT = 128;            // patches per x tile (two warpgroups x m64)
constexpr int KB = 64;             // K elements per prototype smem block (128 B rows)
constexpr int PSUB = PT * KB * 2;  // one [128 x 64] fp16 block = 16 KiB

template <int D>
struct RsSmem {
    static constexpr int NKB = D / KB;                 // prototype K blocks per tile
    static constexpr int NKS = D / 16;                 // k16 steps
    static constexpr int NXB = D / 32;                 // fp32 landing blocks of [128 rows x 32 floats] (128 B rows, swizzled)
    static constexpr uint32_t XB_BYTES = XT * 128;     // 16 KiB
    static constexpr uint32_t X_BYTES = NXB * XB_BYTES;
    uint8_t* bp;                                       // the aligned base (generic) ...
    uint32_t base;                                     // ... and its shared-memory address; the landing tile is at 0
    uint32_t o_epi;                                    // the kernel's epilogue region, behind the ring
    uint32_t bar0, xfull, xempty;                      // shared addresses of the barriers
    __device__ __forceinline__ uint32_t ring(int stage) const { return base + X_BYTES + (uint32_t)stage * 2 * PSUB; }
    __device__ __forceinline__ uint32_t full(int i) const { return bar0 + 8u * i; }
    __device__ __forceinline__ uint32_t empty(int i) const { return bar0 + 8u * (8 + i); }
    __device__ __forceinline__ uint8_t* epi() const { return bp + o_epi; }

    // the layout of the dynamic shared memory for a ring of S stages and an epilogue region of epi_bytes
    __device__ __forceinline__ RsSmem(int S, uint32_t epi_bytes) {
        extern __shared__ uint8_t smem_raw[];
        const uint32_t raw = smem_u32(smem_raw);
        base = (raw + 1023u) & ~1023u;
        bp = smem_raw + (base - raw);
        o_epi = X_BYTES + (uint32_t)S * 2 * PSUB;
        bar0 = base + (o_epi + epi_bytes);
        xfull = bar0 + 8u * 16;
        xempty = bar0 + 8u * 17;
    }
};

template <int D>
__device__ __forceinline__ void init_barriers(const RsSmem<D>& sm) {
    if (threadIdx.x == 0) {
        for (int i = 0; i < 8; ++i) { mbar_init(sm.full(i), 1); mbar_init(sm.empty(i), 8); }   // empty: one arrive per consumer warp
        mbar_init(sm.xfull, 1);
        mbar_init(sm.xempty, 8);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();
}

// warp 9, lane 0: the CTA's x tiles x_tile(0), ..., x_tile(n_x - 1) into the landing tile, each one as soon as the
// consumers have converted the previous one (so it lands under that one's MMAs)
template <int D, typename XTile>
__device__ __forceinline__ void produce_x_tiles(const RsSmem<D>& sm, const CUtensorMap* map_x, int n_x, XTile x_tile) {
    for (int c = 0; c < n_x; ++c) {
        if (c > 0) mbar_wait(sm.xempty, (uint32_t)((c - 1) & 1));
        mbar_expect_tx(sm.xfull, RsSmem<D>::X_BYTES);
        const int row = x_tile(c) * XT;
#pragma unroll
        for (int b = 0; b < RsSmem<D>::NXB; ++b)
            tma_load_2d(sm.base + b * RsSmem<D>::XB_BYTES, map_x, b * 32, row, sm.xfull);
    }
}

// warp 8, lane 0: for x tile c, the prototype tiles [p_begin(c), p_end(c)); tile pt is the 128 rows from
// first_row(pt), in NKB blocks of KB columns of the [-2 w mu] half of [P, 2D], hi and lo into one ring stage each
template <int D, typename PBegin, typename PEnd, typename FirstRow>
__device__ __forceinline__ void produce_proto_tiles(const RsSmem<D>& sm, const CUtensorMap* map_ph,
                                                    const CUtensorMap* map_pl, int S, int n_x, PBegin p_begin,
                                                    PEnd p_end, FirstRow first_row) {
    int stage = 0;
    uint32_t phase = 0;
    for (int c = 0; c < n_x; ++c)
        for (int pt = p_begin(c); pt < p_end(c); ++pt)
            for (int kb = 0; kb < RsSmem<D>::NKB; ++kb) {
                mbar_wait(sm.empty(stage), phase ^ 1u);
                mbar_expect_tx(sm.full(stage), 2 * PSUB);
                const uint32_t dst = sm.ring(stage);
                tma_load_2d(dst, map_ph, D + kb * KB, first_row(pt), sm.full(stage));
                tma_load_2d(dst + PSUB, map_pl, D + kb * KB, first_row(pt), sm.full(stage));
                if (++stage == S) { stage = 0; phase ^= 1u; }
            }
}

// consumers: the c-th landing tile -> the A fragments (hi, lo of X_SCALE x) of this thread's rows rA, rA + 8 and their
// |x|^2 (ssA, ssB, summed over the quad); then the landing tile is released to the patch producer
template <int D>
__device__ __forceinline__ void split_x_tile(const RsSmem<D>& sm, int c, int rA, int lane,
                                             uint32_t (&ah)[RsSmem<D>::NKS][4], uint32_t (&al)[RsSmem<D>::NKS][4],
                                             float& ssA, float& ssB) {
    const int t = lane & 3;
    ssA = 0.f;
    ssB = 0.f;
    mbar_wait(sm.xfull, (uint32_t)(c & 1));
#pragma unroll
    for (int ks = 0; ks < RsSmem<D>::NKS; ++ks) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {                    // fragment register q: row rA + 8 (q & 1), k 16 ks + 2 t + 8 (q >> 1)
            const int r = rA + 8 * (q & 1), col = 16 * ks + 2 * t + 8 * (q >> 1), w = col & 31;
            const float2 v = *reinterpret_cast<const float2*>(
                sm.bp + (uint32_t)(col >> 5) * RsSmem<D>::XB_BYTES + (uint32_t)r * 128u + ((((w >> 2) ^ (r & 7)) & 7) << 4) + (w & 3) * 4);
            if (q & 1) ssB = fmaf(v.x, v.x, fmaf(v.y, v.y, ssB)); else ssA = fmaf(v.x, v.x, fmaf(v.y, v.y, ssA));
            split_f16x2(v.x * X_SCALE, v.y * X_SCALE, ah[ks][q], al[ks][q]);
        }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(sm.xempty);             // landing tile consumed: the next one may land
    ssA += __shfl_xor_sync(0xffffffffu, ssA, 1); ssA += __shfl_xor_sync(0xffffffffu, ssA, 2);
    ssB += __shfl_xor_sync(0xffffffffu, ssB, 1); ssB += __shfl_xor_sync(0xffffffffu, ssB, 2);
}

// consumers: one prototype tile from the ring into acc (zeroed first), stage by stage, each released after its MMAs
template <int D>
__device__ __forceinline__ void mma_proto_tile(const RsSmem<D>& sm, float (&acc)[64],
                                               const uint32_t (&ah)[RsSmem<D>::NKS][4],
                                               const uint32_t (&al)[RsSmem<D>::NKS][4], int S, int lane, int& stage,
                                               uint32_t& phase) {
#pragma unroll
    for (int j = 0; j < 64; ++j) acc[j] = 0.f;
    for (int kb = 0; kb < RsSmem<D>::NKB; ++kb) {
        mbar_wait(sm.full(stage), phase);
        const uint32_t ph = sm.ring(stage), pl = ph + PSUB;
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
        if (lane == 0) mbar_arrive(sm.empty(stage));    // this warp no longer reads the stage
        if (++stage == S) { stage = 0; phase ^= 1u; }
    }
}

// host: [rows, cols] fp32 row-major patch map, box = 32 cols (128 B) x XT rows, 128 B swizzle (the landing tile)
static inline bool make_map_x(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols) {
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

// host: the deepest ring (at most 8 stages) that fits beside a kernel's epi_bytes of own shared memory, and the
// dynamic shared memory to launch with; false if fewer than 2 stages fit
static inline bool rs_smem_plan(int D, size_t epi_bytes, int* stages, size_t* smem) {
    const size_t fixed = 1024 + (size_t)XT * D * 4 + epi_bytes + 256;   // alignment slack, landing tile, own, barriers
    int s = (int)((227 * 1024 - fixed) / (2 * PSUB));
    if (s > 8) s = 8;
    if (s < 2) return false;
    *stages = s;
    *smem = fixed + (size_t)s * 2 * PSUB;
    return true;
}

}  // namespace mgp_rs
