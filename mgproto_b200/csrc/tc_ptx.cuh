// Inline PTX for the sm_90a tensor-core / TMA / mbarrier path, shared by logprob_tc.cu and em_tc.cu.
// SASS: wgmma.mma_async -> HGMMA, cp.async.bulk.tensor -> UTMALDG / UTMASTG, mbarrier -> SYNCS.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace mgp_tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

// The fp16 operand format of every tensor-core GEMM here: v = hi + lo with hi = fp16(v), lo = fp16(v - hi) (22
// mantissa bits); products run as hi*hi + lo*hi + hi*lo with fp32 accumulation.  Patch and bank rows are split as
// X_SCALE x (the factor keeps lo in fp16's normal range for unit-norm rows); whoever consumes such a product divides
// X_SCALE out again.  Prototype-side operands carry their own power-of-two scales.
constexpr float X_SCALE = 256.0f;

__device__ __forceinline__ __half split_f16_lo(float v, __half hi) { return __float2half_rn(v - __half2float(hi)); }
__device__ __forceinline__ void split_f16(float v, __half& hi, __half& lo) {
    const __half h = __float2half_rn(v);
    hi = h;
    lo = split_f16_lo(v, h);
}
__device__ __forceinline__ uint32_t pack_h2(__half a, __half b) {
    return (uint32_t)__half_as_ushort(a) | ((uint32_t)__half_as_ushort(b) << 16);
}
// two consecutive k of an RS A fragment register (the lower k in the low half); both hi halves are packed before the
// lo halves are formed, which keeps fewer values live in the fully unrolled fragment loops
__device__ __forceinline__ void split_f16x2(float v0, float v1, uint32_t& hi, uint32_t& lo) {
    const __half h0 = __float2half_rn(v0), h1 = __float2half_rn(v1);
    hi = pack_h2(h0, h1);
    lo = pack_h2(split_f16_lo(v0, h0), split_f16_lo(v1, h1));
}

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0;
    long long t0 = 0;
    for (uint32_t it = 0; !ok; ++it) {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok)
            : "r"(bar), "r"(parity)
            : "memory");
        if (!ok && (it & 1023u) == 1023u) {              // a protocol bug must fault, not hang the device
            const long long now = clock64();
            if (t0 == 0) t0 = now;
            else if (now - t0 > 4000000000LL) __trap();
        }
    }
}
// Named barriers (bar.sync / bar.arrive, ids 1..15; 0 is __syncthreads): THREADS counts every participant, waiting
// or arriving, and is a multiple of 32.  A warpgroup that arrives does not wait, so a pair of them orders two
// warpgroups without making the signalling one block.  The id is an immediate, so ptxas reserves only the barriers a
// kernel names.
template <int ID, int THREADS>
__device__ __forceinline__ void named_bar_sync() {
    asm volatile("bar.sync %0, %1;" ::"n"(ID), "n"(THREADS) : "memory");
}
template <int ID, int THREADS>
__device__ __forceinline__ void named_bar_arrive() {
    asm volatile("bar.arrive %0, %1;" ::"n"(ID), "n"(THREADS) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
        ::"r"(dst), "l"(map), "r"(c0), "r"(c1), "r"(bar)
        : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(map), "r"(src), "r"(c0), "r"(c1)
                 : "memory");
}
__device__ __forceinline__ void tma_store_3d(const CUtensorMap* map, uint32_t src, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.global.shared::cta.bulk_group [%0, {%2, %3, %4}], [%1];"
                 ::"l"(map), "r"(src), "r"(c0), "r"(c1), "r"(c2)
                 : "memory");
}
// Warpgroup MMA (sm_90a wgmma.mma_async): fp16 x fp16 -> fp32, both operands from shared memory, the accumulator in
// the registers of the issuing warpgroup.  Fragment of an m64nN accumulator, warp w (of the warpgroup), lane l:
// d[4 i + 2 h + j] = D[16 w + l / 4 + 8 h][8 i + 2 (l % 4) + j].
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x 32] (+)= A[64 x 16] . B[16 x 32]; TA = 1: A is MN-major (transposed) in shared memory
template <int TA>
__device__ __forceinline__ void wg_mma_n32(float (&d)[16], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %18, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, %19, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]),
          "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TA));
}
// D[64 x 16] (+)= A[64 x 16] . B[16 x 16]
template <int TA>
__device__ __forceinline__ void wg_mma_n16(float (&d)[8], uint64_t a_desc, uint64_t b_desc, uint32_t accumulate) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %10, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, %11, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
        : "l"(a_desc), "l"(b_desc), "r"(accumulate), "n"(TA));
}

// D[64 x 128] (+)= A[64 x 16] (registers: the m64k16 fp16 fragment, 4 x 2 halves) . B[16 x 128] (shared memory)
__device__ __forceinline__ void wg_mma_rs_n128(float (&d)[64], const uint32_t (&a)[4], uint64_t b_desc) {
    asm volatile(
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, {%64, %65, %66, %67}, %68, 1, 1, 1, 0;"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b_desc));
}

// Image-wide MMAs: D[64 x NI] (+)= A[64 x 16] . B[16 x NI], both K-major in shared memory, accumulator d[NI / 2].
// wg_mma_ss<NI> exists for the widths MGP_WG_MMA_SS instantiates below.  The asm operand lists are generated:
// accumulator r is operand %r, so the placeholder "%r" and the constraint "+f"(d[r]) come from the same
// decimal-digit macros (X(p, u) stands for register pu; p is the leading digits, empty for r < 10).
template <int NI>
__device__ __forceinline__ void wg_mma_ss(float (&d)[NI / 2], uint64_t a_desc, uint64_t b_desc);

#define MGP_WG_S0 "%0"
#define MGP_WG_S(p, u) ", %" #p #u
#define MGP_WG_F0 "+f"(d[0])
#define MGP_WG_F(p, u) , "+f"(d[p##u])
#define MGP_WG_D2(X, p) X(p, 0) X(p, 1)
#define MGP_WG_D4(X, p) MGP_WG_D2(X, p) X(p, 2) X(p, 3)
#define MGP_WG_D6(X, p) MGP_WG_D4(X, p) X(p, 4) X(p, 5)
#define MGP_WG_D8(X, p) MGP_WG_D6(X, p) X(p, 6) X(p, 7)
#define MGP_WG_D10(X, p) MGP_WG_D8(X, p) X(p, 8) X(p, 9)
#define MGP_WG_R10(X, X0) X0 X(, 1) X(, 2) X(, 3) X(, 4) X(, 5) X(, 6) X(, 7) X(, 8) X(, 9)
#define MGP_WG_R50(X, X0) MGP_WG_R10(X, X0) MGP_WG_D10(X, 1) MGP_WG_D10(X, 2) MGP_WG_D10(X, 3) MGP_WG_D10(X, 4)
#define MGP_WG_R100(X, X0) MGP_WG_R50(X, X0) MGP_WG_D10(X, 5) MGP_WG_D10(X, 6) MGP_WG_D10(X, 7) MGP_WG_D10(X, 8) MGP_WG_D10(X, 9)
// accumulator registers per width: NI / 2
#define MGP_WG_ACC16(X, X0) MGP_WG_R10(X, X0) MGP_WG_D6(X, 1)
#define MGP_WG_ACC28(X, X0) MGP_WG_R10(X, X0) MGP_WG_D10(X, 1) MGP_WG_D8(X, 2)
#define MGP_WG_ACC32(X, X0) MGP_WG_R10(X, X0) MGP_WG_D10(X, 1) MGP_WG_D10(X, 2) MGP_WG_D2(X, 3)
#define MGP_WG_ACC64(X, X0) MGP_WG_R50(X, X0) MGP_WG_D10(X, 5) MGP_WG_D4(X, 6)
#define MGP_WG_ACC100(X, X0) MGP_WG_R100(X, X0)
#define MGP_WG_ACC128(X, X0) MGP_WG_R100(X, X0) MGP_WG_D10(X, 10) MGP_WG_D10(X, 11) MGP_WG_D8(X, 12)
// NI, then the operand numbers of the A descriptor, the B descriptor and the scale-d flag (NI / 2, + 1, + 2)
#define MGP_WG_MMA_SS(NI, OA, OB, OS)                                                                         \
    template <>                                                                                                \
    __device__ __forceinline__ void wg_mma_ss<NI>(float (&d)[NI / 2], uint64_t a_desc, uint64_t b_desc) {      \
        static_assert(OA == NI / 2 && OB == OA + 1 && OS == OA + 2, "operand numbering");                     \
        asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #OS ", 0;\n\t"                                  \
                     "wgmma.mma_async.sync.aligned.m64n" #NI "k16.f32.f16.f16 "                              \
                     "{" MGP_WG_ACC##OA(MGP_WG_S, MGP_WG_S0) "}, %" #OA ", %" #OB ", p, 1, 1, 0, 0;\n\t}"      \
                     : MGP_WG_ACC##OA(MGP_WG_F, MGP_WG_F0)                                                     \
                     : "l"(a_desc), "l"(b_desc), "r"(1u));                                                     \
    }
MGP_WG_MMA_SS(32, 16, 17, 18)
MGP_WG_MMA_SS(56, 28, 29, 30)
MGP_WG_MMA_SS(64, 32, 33, 34)
MGP_WG_MMA_SS(128, 64, 65, 66)
MGP_WG_MMA_SS(200, 100, 101, 102)
MGP_WG_MMA_SS(256, 128, 129, 130)
#undef MGP_WG_MMA_SS

// Ties the accumulator registers to this point of the program: the compiler may not move their reads or writes across it
// (after wg_wait, before the epilogue reads the results).
template <int R>
__device__ __forceinline__ void wg_fence_operands(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int N>
__device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// Shared-memory matrix descriptors (sm_90 GMMA): start>>4 at [0,14), LBO>>4 at [16,30), SBO>>4 at [32,46),
// layout SWIZZLE_128B (1) at [62,64).
//   K-major, SWIZZLE_128B : 8-row groups of 128 B rows (1024 B) -> SBO = 1024 B; LBO unused (1).  A K step of 16
//   fp16 inside the 128 B row advances the start address by 32 B.
__device__ __forceinline__ uint64_t gmma_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | (1ull << 16) | (64ull << 32) | (1ull << 62);
}
//   MN-major, SWIZZLE_128B (canonical ((8,n),(8,k)):((1,LBO),(8,SBO)) in 16-byte units): 64 MN-elements (128 B)
//   contiguous, the next 64 at +LBO; 8 k-rows at 128 B stride, the next 8 at +SBO
__device__ __forceinline__ uint64_t gmma_desc_mn(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFFu) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFFu) << 32) | (1ull << 62);
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static inline EncodeTiledFn get_encode() {
    static EncodeTiledFn fn = nullptr;
    static bool tried = false;
    if (!tried) {
        tried = true;
        void* sym = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &sym, cudaEnableDefault, &qr) == cudaSuccess &&
            qr == cudaDriverEntryPointSuccess)
            fn = reinterpret_cast<EncodeTiledFn>(sym);
    }
    return fn;
}

// [rows, cols] fp16 row-major, box = 64 cols x box_rows rows, 128 B swizzle; out-of-bounds rows read as zero
static inline bool make_map_f16(CUtensorMap* m, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[2] = {cols, rows};
    cuuint64_t strides[1] = {cols * 2};
    cuuint32_t box[2] = {64, box_rows};
    cuuint32_t es[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, es,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

}  // namespace mgp_tc
