// a2/a16 on the Hopper tensor cores (MGP_MATH_TC): the squared Mahalanobis distance as a GEMM
//
//   q[n,p] = sum_d w_pd x_nd^2 - 2 sum_d (w mu)_pd x_nd + sum_d w_pd mu_pd^2 ,   w = 1/(sigma+eps)^2
//          = [x^2 | x]_n . [w | -2 w mu]_p + c2_p                       (inner dim 2D, general diagonal)
//          = w_p |x_n|^2 + x_n . (-2 w mu)_p + c2_p                     (inner dim  D, sigma constant over d:
//                                                                        every state the shipped loop reaches)
//   log p = e0_p + e1_p * acc[n,p] + e2_p * |x_n|^2
//
// Precision: operands are split into fp16 hi + lo (22 mantissa bits) and accumulated as
// hi*hi + lo*hi + hi*lo in fp32 register accumulators -- three fp16 wgmma passes instead of one TF32
// pass at half rate; |error| on q ~1e-6, inside the 1e-4 bar on logits (a single bf16 or tf32
// pass is not).  Power-of-two scalings keep the lo parts in fp16's normal range and are undone
// exactly in the epilogue.
//
// Structure (one persistent CTA per SM, 10 warps):
//   warp 8   TMA producer: prototype (A) K-blocks through an S-stage mbarrier ring
//   warp 9   TMA producer of the x tile (B, 128 patches x Kg), resident per n-tile, double-buffered when
//            it fits so the next n-tile is prefetched under the current one's MMAs
//   warps 0-7  two consumer warpgroups: warpgroup g issues wgmma.mma_async m64n32k16 for prototypes
//            [64 g, 64 g + 64) of the 128-prototype tile x all patches of the x tile, then runs the epilogue:
//            the accumulator goes through a shared-memory transpose so that a thread holds 32 patches of ONE
//            prototype and the 32 lanes of a warp hold 32 consecutive prototypes (for the [N,P] layout: 32
//            consecutive floats of one output row), affine fix-up, stores.
// HBM traffic per launch: 4*N*P (output) + 8*N*Kg (fp16 hi/lo operand written by the prep pass and
// read once) + 4*N*D (x) -- the output dominates; the kernel is bound by the HBM write stream.
//
// The labelled step's per (image, prototype) max / arg-max (MGP_OUT_TOP1_BP) with isotropic sigma, 32 <= HW <= 256 and
// D in {64, 128} takes logprob_top1_wide_kernel instead: one x tile per image, one m64nNIk16 MMA per k16 step and pass
// (NI = HW rounded up to 32, 56, 64, 128, 200 or 256), the max / arg-max read straight from the accumulator fragments and
// written with plain stores; nothing is stored but B*P packed results, so it is bound by the tensor cores.  Its other
// cases (anisotropic sigma, other HW, D = 256) run logprob_tc_kernel<top1> on 128-patch tiles, into a zeroed output
// by 64-bit RED.MAX.
#include <cuda.h>
#include <cstdlib>
#include <cuda_fp16.h>

#include "mgp_common.cuh"
#include "tc_ptx.cuh"

namespace {

constexpr int LAYOUT_NP_TMA = 3; // internal: [N,P] output written by TMA bulk tensor stores from a shared-memory stage
constexpr int LAYOUT_BPHW_TMA = 4;   // internal: [B,P,HW] log p through a 3-D tensor map (boxes clipped at image ends)
constexpr int LAYOUT_NEGP_TMA = 5;   // internal: [B,P,HW] -exp(log p), same
constexpr int LAYOUT_TOP1 = 6;       // internal: no log p output at all -- per (image, prototype) max / arg-max (MGP_OUT_TOP1_BP)
constexpr int STAGING_BYTES = 8 * 32 * 32 * 4;   // one [32 x 32] fp32 block per consumer warp (transpose, TMA stores)
constexpr int PT = 128;          // prototypes per tile (two warpgroups x 64)
constexpr int KB = 64;           // K elements per smem block (128 B rows, SWIZZLE_128B)
constexpr int SUB_BYTES = 128 * KB * 2;   // one [128 x 64] fp16 block = 16 KiB

// ------------------------------------------------------------------------------------------ PTX (tc_ptx.cuh)
using namespace mgp_tc;

// ------------------------------------------------------------------------------------------ prep
// Prototype side: Bh/Bl [P, 2D] fp16 = split of scale_p * [ w | -2 w mu ]; e0,e1,e2 [P]; noniso flag.
__global__ void tc_proto_prep_kernel(const float* __restrict__ mu, const float* __restrict__ sigma, float eps,
                                     float eps_log, __half* __restrict__ bh, __half* __restrict__ bl,
                                     float* __restrict__ e0, float* __restrict__ e1, float* __restrict__ e2,
                                     int* __restrict__ noniso, int P, int D) {
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");   // a dependent launched programmatically may start its prologue
    const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (p >= P) return;
    const float* mr = mu + (size_t)p * D;
    const float* sr = sigma + (size_t)p * D;
    const float s0 = sr[0];
    float ls = 0.f, c2 = 0.f, mx = 0.f;
    bool same = true;
    for (int d = lane; d < D; d += 32) {
        const float s = sr[d];
        same = same && (s == s0);
        const float r = 1.0f / (s + eps);
        const float w = r * r;
        const float m = mr[d];
        ls += logf(s + eps_log) + 0.5f * MGP_LOG_2PI;   // per-dim terms (they cancel for sigma = 1/sqrt(2 pi))
        c2 = fmaf(w * m, m, c2);
        mx = fmaxf(mx, fmaxf(w, fabsf(2.0f * w * m)));
    }
    ls = warp_sum(ls);
    c2 = warp_sum(c2);
    mx = warp_max(mx);
    same = __all_sync(0xffffffffu, same);
    int ex = 0;
    if (mx > 0.f) frexpf(mx, &ex);                       // mx = f * 2^ex, f in [0.5, 1)
    const float scale = ldexpf(1.0f, 8 - ex);            // max |B'| * scale in [128, 256)
    for (int d = lane; d < D; d += 32) {
        const float r = 1.0f / (sr[d] + eps);
        const float w = r * r;
        const float v0 = w * scale, v1 = -2.0f * w * mr[d] * scale;
        split_f16(v0, bh[(size_t)p * 2 * D + d], bl[(size_t)p * 2 * D + d]);
        split_f16(v1, bh[(size_t)p * 2 * D + D + d], bl[(size_t)p * 2 * D + D + d]);
    }
    if (lane == 0) {
        const float r0 = 1.0f / (s0 + eps);
        e0[p] = -ls - 0.5f * c2;
        e1[p] = -0.5f / (scale * X_SCALE);
        e2[p] = -0.5f * r0 * r0;                          // used only when every prototype is isotropic
        if (!same) atomicOr(noniso, 1);
    }
}

// Patch side: Ah/Al [N, 2D] fp16 = split of 256 * [ x^2 | x ] (the x^2 half only if some prototype is
// anisotropic), sn [N] = |x|^2.  Warp per row.
__global__ void tc_x_prep_kernel(const float* __restrict__ x, __half* __restrict__ ah, __half* __restrict__ al,
                                 float* __restrict__ sn, const int* __restrict__ noniso, int N, int D) {
    const int n = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (n >= N) return;
    const bool gen = (*noniso != 0);
    const float4* xr = reinterpret_cast<const float4*>(x + (size_t)n * D);
    __half* hr = ah + (size_t)n * 2 * D;
    __half* lr = al + (size_t)n * 2 * D;
    float ss = 0.f;
    for (int d4 = lane; d4 < D / 4; d4 += 32) {
        const float4 v = __ldg(xr + d4);
        const float a[4] = {v.x, v.y, v.z, v.w};
        __align__(8) __half h[4], l[4], h2[4], l2[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            ss = fmaf(a[i], a[i], ss);
            split_f16(a[i] * X_SCALE, h[i], l[i]);
            split_f16(a[i] * a[i] * X_SCALE, h2[i], l2[i]);
        }
        *reinterpret_cast<uint2*>(hr + D + d4 * 4) = *reinterpret_cast<uint2*>(h);
        *reinterpret_cast<uint2*>(lr + D + d4 * 4) = *reinterpret_cast<uint2*>(l);
        if (gen) {
            *reinterpret_cast<uint2*>(hr + d4 * 4) = *reinterpret_cast<uint2*>(h2);
            *reinterpret_cast<uint2*>(lr + d4 * 4) = *reinterpret_cast<uint2*>(l2);
        }
    }
    ss = warp_sum(ss);
    if (lane == 0) sn[n] = ss;
}

// ------------------------------------------------------------------------------------------ main
struct TcParams {
    const float* e0;
    const float* e1;
    const float* e2;
    const float* sn;
    const int* noniso;
    float* out;
    int N, HW, P, D;
    int n_ntiles, n_ptiles;
    int xbox;              // rows of the x tensor-map box
    int B, nti;            // image-aligned tiling of the [B,P,HW] TMA path: one x tile = one image, nti = round_up(HW, 32) columns
    int team;              // CTAs per team: the CTAs of a team work on the SAME x tile at the same time, on
                           // adjacent prototype tiles, so each output row receives team*512 contiguous bytes at once
    uint32_t smem_bytes;   // dynamic shared memory of the launch
    int x_no_sq;           // the staged patch operands lack the x^2 half (isotropic sigma asserted by the producer)
    int iso_elsewhere;     // top-1 fallback: return at once when sigma turns out isotropic (the image-tile kernel ran)
    int debug;   // ablation switches for profiling (MGP_TC_DEBUG): 1 no global stores, 4 no MMAs,
                 // 8 no epilogue work, 16 no prototype TMA loads
};

constexpr int TC_THREADS = 320;   // warps: 0-7 two consumer warpgroups (MMA + epilogue), 8 proto TMA, 9 x-tile TMA

template <int LAYOUT>
__device__ __forceinline__ void epilogue_chunk(const uint32_t (&r)[32], const float* __restrict__ s_sn_c, float c0,
                                               float c1, float c2, int n0, int p, bool pok, const TcParams& prm,
                                               float* stg = nullptr, const CUtensorMap* map_out = nullptr, int img_b = 0,
                                               int img_hw0 = 0) {
    const int N = prm.N, P = prm.P, HW = prm.HW;
    float v[32];
    const float4* s4 = reinterpret_cast<const float4*>(s_sn_c);    // |x_n|^2 of the 32 columns (shared memory)
#pragma unroll
    for (int j4 = 0; j4 < 8; ++j4) {
        const float4 s = s4[j4];
        // two columns per FFMA2 (same rounding as two scalar fmaf: each half is an IEEE fused multiply-add)
        const float2 c00 = make_float2(c0, c0), c11 = make_float2(c1, c1), c22 = make_float2(c2, c2);
        const float2 v01 = ffma2(c11, make_float2(__uint_as_float(r[4 * j4 + 0]), __uint_as_float(r[4 * j4 + 1])),
                                 ffma2(c22, make_float2(s.x, s.y), c00));
        const float2 v23 = ffma2(c11, make_float2(__uint_as_float(r[4 * j4 + 2]), __uint_as_float(r[4 * j4 + 3])),
                                 ffma2(c22, make_float2(s.z, s.w), c00));
        v[4 * j4 + 0] = v01.x; v[4 * j4 + 1] = v01.y; v[4 * j4 + 2] = v23.x; v[4 * j4 + 3] = v23.y;
    }
    if (LAYOUT == LAYOUT_TOP1) {
        // only max_n log p[n, p] and its patch per image are wanted (labelled training step: the reference aliases
        // the other levels of wrong-class prototypes to level 0): nothing is stored, the log-likelihood matrix
        // never reaches HBM.  This is the 128-patch-tile fallback (anisotropic sigma, HW outside [32, 256], D = 256;
        // image tiles take logprob_top1_wide_kernel): a tile may cross image ends, so the chunk is reduced per image
        // segment and merged by a 64-bit RED.MAX into the zeroed `best`.
        if (!pok) return;
        unsigned long long* best = reinterpret_cast<unsigned long long*>(prm.out);
        int b = n0 / HW, hw = n0 - b * HW;
        float mv = -INFINITY;
        int mi = -1;
#pragma unroll
        for (int j = 0; j < 32; ++j) {
            if (n0 + j < N) {
                if (mi < 0 || v[j] > mv) { mv = v[j]; mi = hw; }
                if (++hw == HW) {
                    atomicMax(best + (size_t)b * P + p, top1_pack(mv, mi));
                    ++b; hw = 0; mi = -1;
                }
            }
        }
        if (mi >= 0) atomicMax(best + (size_t)b * P + p, top1_pack(mv, mi));
        return;
    }
    if (LAYOUT == LAYOUT_NP_TMA) {
        // stage the [32 patches x 32 prototypes] block in shared memory (row = patch, 128 B) and hand it to
        // the TMA engine: the global writes are issued asynchronously as whole row segments, the warp only
        // pays 32 conflict-free STS.  Out-of-range rows / columns are clipped by the tensor map.
        const int lane = threadIdx.x & 31;
        if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");   // previous block has been read
        __syncwarp();
#pragma unroll
        for (int j = 0; j < 32; ++j) stg[j * 32 + lane] = v[j];
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0 && !(prm.debug & 1)) {
            tma_store_2d(map_out, smem_u32(stg), p - lane, n0);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        return;
    }
    if (LAYOUT == LAYOUT_BPHW_TMA || LAYOUT == LAYOUT_NEGP_TMA) {
        // [B,P,HW]: this thread's 32 values are 128 contiguous bytes of row (b, p).  Stage [32 prototypes x 128 B]
        // with the tensor map's 128B swizzle (8 x STS.128 per thread, conflict-free) and let the TMA engine write
        // it.  Tiles are image-aligned here, so a chunk lies in ONE image; columns past HW are clipped by the map.
        const int lane = threadIdx.x & 31;
        if (LAYOUT == LAYOUT_NEGP_TMA) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = -expf(v[j]);
        }
        if (lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
        __syncwarp();
        uint8_t* rowp = reinterpret_cast<uint8_t*>(stg) + lane * 128;
#pragma unroll
        for (int c = 0; c < 8; ++c)
            *reinterpret_cast<float4*>(rowp + ((c ^ (lane & 7)) << 4)) = make_float4(v[4 * c], v[4 * c + 1], v[4 * c + 2], v[4 * c + 3]);
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncwarp();
        if (lane == 0 && !(prm.debug & 1)) {
            tma_store_3d(map_out, smem_u32(stg), img_hw0, p - lane, img_b);
            asm volatile("cp.async.bulk.commit_group;" ::: "memory");
        }
        return;
    }
    if (!pok) return;
    if (prm.debug & 1) {
        float acc = 0.f;
#pragma unroll
        for (int j = 0; j < 32; ++j) acc += v[j];
        if (acc == 123.456f) prm.out[0] = acc;
        return;
    }
    const bool full = (n0 + 32 <= N);
    if (LAYOUT == MGP_OUT_LOGP_NP) {
        float* dst = prm.out + (size_t)n0 * P + p;          // lanes = consecutive p: 128 B per warp store
        if (full) {
#pragma unroll
            for (int j = 0; j < 32; ++j) dst[(size_t)j * P] = v[j];
        } else {
            for (int j = 0; j < 32; ++j)
                if (n0 + j < N) dst[(size_t)j * P] = v[j];
        }
    } else {
        if (LAYOUT == MGP_OUT_NEGP_BPHW) {
#pragma unroll
            for (int j = 0; j < 32; ++j) v[j] = -expf(v[j]);
        }
        int b = n0 / HW, hw = n0 - b * HW;
        if (full && (HW & 3) == 0) {                         // 4 consecutive patches share an image, 16 B aligned
#pragma unroll
            for (int j = 0; j < 32; j += 4) {
                *reinterpret_cast<float4*>(prm.out + ((size_t)b * P + p) * HW + hw) =
                    make_float4(v[j], v[j + 1], v[j + 2], v[j + 3]);
                hw += 4;
                if (hw >= HW) { hw -= HW; ++b; }
            }
        } else {
            for (int j = 0; j < 32; ++j) {
                if (n0 + j < N) prm.out[((size_t)b * P + p) * HW + hw] = v[j];
                if (++hw == HW) { hw = 0; ++b; }
            }
        }
    }
}

template <int LAYOUT>
__global__ void __launch_bounds__(TC_THREADS, 1)
logprob_tc_kernel(const __grid_constant__ CUtensorMap map_xh, const __grid_constant__ CUtensorMap map_xl,
                  const __grid_constant__ CUtensorMap map_ph, const __grid_constant__ CUtensorMap map_pl,
                  const __grid_constant__ CUtensorMap map_out, const TcParams prm) {
    constexpr bool TMA_ST = (LAYOUT == LAYOUT_NP_TMA || LAYOUT == LAYOUT_BPHW_TMA || LAYOUT == LAYOUT_NEGP_TMA);
    constexpr bool BPHW_TMA = (LAYOUT == LAYOUT_BPHW_TMA || LAYOUT == LAYOUT_NEGP_TMA);
    // image tiles (up to 256 patches = 8 chunks) exist only for these layouts; 128-patch tiles have 4 chunks
    constexpr int NCH = BPHW_TMA ? 8 : 4;
    // the layout used by the non-TMA fallback of the same instantiation (anisotropic sigma: see `img` below)
    constexpr int STG_LAYOUT = (LAYOUT == LAYOUT_BPHW_TMA) ? MGP_OUT_LOGP_BPHW
                               : (LAYOUT == LAYOUT_NEGP_TMA) ? MGP_OUT_NEGP_BPHW : LAYOUT;
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;                 // SWIZZLE_128B tiles need 1024 B alignment
    uint8_t* base_ptr = smem_raw + (base - raw);

    const bool gen = (*prm.noniso != 0);
    if (gen && (prm.D > 128 || prm.x_no_sq)) __trap();            // isotropic sigma was promised (MGP_MATH_TC_ISO / staging): fail loudly
    if (LAYOUT == LAYOUT_TOP1 && prm.iso_elsewhere && !gen) return;   // isotropic: logprob_top1_wide_kernel has done the work
    const int nkb = (gen ? 2 * prm.D : prm.D) / KB;               // K blocks per tile
    const int kcol0 = gen ? 0 : prm.D;                            // isotropic: only the [x] / [-2 w mu] half
    // [B,P,HW] through TMA: one x tile = one image (nti = round_up(HW,32) patches) so that no 32-column chunk
    // crosses an image end.  The wider tile only fits when sigma is isotropic (K = D); otherwise this
    // instantiation falls back to 128-patch tiles and register stores.
    const bool img = BPHW_TMA && !gen;
    const int NT = img ? prm.nti : 128;                           // patches per tile
    const int nch = NT / 32;                                      // 32-patch MMA chunks (m64n32k16 each)
    const int row_step = img ? prm.HW : 128;                      // first patch row of x tile nt = nt * row_step
    const int n_ptiles = prm.n_ptiles, n_ntiles = img ? prm.B : prm.n_ntiles;
    const uint32_t xsub = (uint32_t)NT * KB * 2;                  // one [NT x 64] fp16 block of the x tile

    // carve-up: nbuf x tiles | S stages of (proto hi, proto lo) | staging (accumulator transpose + TMA stores) | barriers + sn tile
    const uint32_t x_bytes = (uint32_t)(2 * nkb) * xsub;          // hi blocks then lo blocks
    const uint32_t tile_budget = prm.smem_bytes - 1024u - 2048u - (uint32_t)STAGING_BYTES;
    const int nbuf = (2 * x_bytes + 2 * 2 * SUB_BYTES <= tile_budget) ? 2 : 1;   // double-buffer x when it fits
    int S = (int)((tile_budget - nbuf * x_bytes) / (2 * SUB_BYTES));
    if (S > 6) S = 6;
    const uint32_t x_base = base;
    const uint32_t st_base = x_base + nbuf * x_bytes;
    const uint32_t stg_base = st_base + (uint32_t)S * 2 * SUB_BYTES;
    const uint32_t misc = stg_base + (uint32_t)STAGING_BYTES;
    float* staging = reinterpret_cast<float*>(base_ptr + (stg_base - base));
    uint8_t* misc_ptr = base_ptr + (misc - base);
    const uint32_t bar0 = misc;                                   // full[6] empty[6] xfull[2] xempty[2]
    auto FULL = [&](int i) { return bar0 + 8u * i; };
    auto EMPTY = [&](int i) { return bar0 + 8u * (6 + i); };
    auto XFULL = [&](int i) { return bar0 + 8u * (12 + i); };
    auto XEMPTY = [&](int i) { return bar0 + 8u * (14 + i); };
    float* s_sn = reinterpret_cast<float*>(misc_ptr + 8 * 16);    // [256] |x|^2 of the current x tile, 16 B aligned

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;

    if (threadIdx.x == 0) {
        for (int i = 0; i < 6; ++i) { mbar_init(FULL(i), 1); mbar_init(EMPTY(i), 8); }   // empty: one arrive per consumer warp
        for (int i = 0; i < 2; ++i) { mbar_init(XFULL(i), 1); mbar_init(XEMPTY(i), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    // schedule: team t = blockIdx / team handles x tiles t, t + n_teams, ...; member k of the team takes the
    // prototype tiles k, k + team, ... of each of them
    const int TS = prm.team;
    const int n_teams = gridDim.x / TS, team = blockIdx.x / TS, k0 = blockIdx.x % TS;
    const bool has_work = (team < n_teams) && (k0 < n_ptiles);

    if (!has_work) {
        // nothing to do for this CTA (tiny problems)
    } else if (warp == 9 && lane == 0) {
        // =========================== x-tile TMA producer (next x tile prefetched when double-buffered) ===========
        int c = 0;
        for (int nt = team; nt < n_ntiles; nt += n_teams, ++c) {
            const int buf = c % nbuf;
            if (c >= nbuf) mbar_wait(XEMPTY(buf), (uint32_t)((c / nbuf - 1) & 1));
            mbar_expect_tx(XFULL(buf), x_bytes);
            const uint32_t xb = x_base + (uint32_t)buf * x_bytes;
            for (int kb = 0; kb < nkb; ++kb)
                for (int r = 0; r < NT; r += prm.xbox) {          // x-map box rows: 128 (128-patch tiles) or 32 (image tiles)
                    const uint32_t ro = (uint32_t)r * KB * 2;
                    tma_load_2d(xb + (uint32_t)kb * xsub + ro, &map_xh, kcol0 + kb * KB, nt * row_step + r, XFULL(buf));
                    tma_load_2d(xb + (uint32_t)(nkb + kb) * xsub + ro, &map_xl, kcol0 + kb * KB, nt * row_step + r, XFULL(buf));
                }
        }
    } else if (warp == 8 && lane == 0) {
        // =========================== prototype TMA producer ===========================
        int stage = 0;
        uint32_t phase = 0;
        for (int nt = team; nt < n_ntiles; nt += n_teams) {
            for (int pt = k0; pt < n_ptiles; pt += TS) {
                for (int kb = 0; kb < nkb; ++kb) {
                    mbar_wait(EMPTY(stage), phase ^ 1u);
                    if (prm.debug & 16) {
                        mbar_arrive(FULL(stage));
                    } else {
                        mbar_expect_tx(FULL(stage), 2 * SUB_BYTES);
                        const uint32_t dst = st_base + (uint32_t)stage * 2 * SUB_BYTES;
                        tma_load_2d(dst, &map_ph, kcol0 + kb * KB, pt * PT, FULL(stage));
                        tma_load_2d(dst + SUB_BYTES, &map_pl, kcol0 + kb * KB, pt * PT, FULL(stage));
                    }
                    if (++stage == S) { stage = 0; phase ^= 1u; }
                }
            }
        }
    } else if (warp < 8) {
        // =========================== consumers: MMA + epilogue ===========================
        // warpgroup wg multiplies prototype rows [64 wg, 64 wg + 64) of the tile with all NT patches (nch m64n32 MMAs
        // per K step, hi*hi + lo*hi + hi*lo into the same fp32 registers), then drains the accumulator 64 patches
        // at a time through its transpose block: thread u of the warpgroup takes prototype row u % 64, chunk u / 64
        // of the pass -- 32 consecutive prototypes per warp, 32 patches per thread, as epilogue_chunk expects.
        // The transpose block [64 prototypes][64 patches] fp32 is the warpgroup's four TMA-store blocks; float column c
        // of row r sits at c ^ 4 (r & 7) (conflict-free float4 reads).
        const int wg = warp >> 2, wq = warp & 3, u = threadIdx.x & 127;
        const int trow = u & 63, tsub = u >> 6;
        float* tp = staging + wg * 4096;
        float* stg = staging + warp * 1024;                       // this warp's 4 KiB TMA-store block
        const uint32_t wg_bar = 2 + wg;
        auto wg_sync = [&]() { asm volatile("bar.sync %0, 128;" ::"r"(wg_bar) : "memory"); };
        int stage = 0, c = 0;
        uint32_t phase = 0;
        for (int nt = team; nt < n_ntiles; nt += n_teams, ++c) {
            const int buf = c % nbuf;
            const int row0 = nt * row_step;
            asm volatile("bar.sync 1, 256;" ::: "memory");        // readers of the previous x tile's norms are done
            for (int i = threadIdx.x; i < NT; i += 256) {
                const int n = row0 + i;
                s_sn[i] = (n < prm.N) ? prm.sn[n] : 0.f;
            }
            asm volatile("bar.sync 1, 256;" ::: "memory");
            mbar_wait(XFULL(buf), (uint32_t)((c / nbuf) & 1));
            const uint32_t xb = x_base + (uint32_t)buf * x_bytes;
            for (int pt = k0; pt < n_ptiles; pt += TS) {
                float acc[NCH][16];
#pragma unroll
                for (int ch = 0; ch < NCH; ++ch)
#pragma unroll
                    for (int j = 0; j < 16; ++j) acc[ch][j] = 0.f;
                for (int kb = 0; kb < nkb; ++kb) {
                    mbar_wait(FULL(stage), phase);
                    const uint32_t ph = st_base + (uint32_t)stage * 2 * SUB_BYTES + (uint32_t)wg * 64u * 128u, pl = ph + SUB_BYTES;
                    const uint32_t xh = xb + (uint32_t)kb * xsub, xl = xb + (uint32_t)(nkb + kb) * xsub;
                    if (!(prm.debug & 4)) {
                        wg_fence();
#pragma unroll
                        for (int k = 0; k < KB / 16; ++k) {
                            const uint32_t off = (uint32_t)k * 32u;   // 16 fp16 = 32 B inside the 128 B swizzle row
                            const uint64_t a_h = gmma_desc(ph + off), a_l = gmma_desc(pl + off);
#pragma unroll
                            for (int ch = 0; ch < NCH; ++ch) {
                                if (ch < nch) {
                                    const uint32_t xo = (uint32_t)ch * 32u * 128u + off;   // 32 patch rows = 4 KiB
                                    const uint64_t b_h = gmma_desc(xh + xo), b_l = gmma_desc(xl + xo);
                                    wg_mma_n32<0>(acc[ch], a_h, b_h, 1u);
                                    wg_mma_n32<0>(acc[ch], a_l, b_h, 1u);
                                    wg_mma_n32<0>(acc[ch], a_h, b_l, 1u);
                                }
                            }
                        }
                        wg_commit();
                        wg_wait0();
                    }
                    __syncwarp();
                    if (lane == 0) mbar_arrive(EMPTY(stage));    // this warp no longer reads the stage
                    if (++stage == S) { stage = 0; phase ^= 1u; }
                }
                if (pt + TS >= n_ptiles) {                        // last prototype tile of this x tile: release the buffer
                    __syncwarp();
                    if (lane == 0) mbar_arrive(XEMPTY(buf));
                }
                if (prm.debug & 8) continue;
                const int p = pt * PT + wg * 64 + trow;
                const bool pok = p < prm.P;
                const float c0 = pok ? __ldg(prm.e0 + p) : 0.f;
                const float c1 = pok ? __ldg(prm.e1 + p) : 0.f;
                const float c2 = (pok && !gen) ? __ldg(prm.e2 + p) : 0.f;
#pragma unroll
                for (int pass = 0; pass < NCH / 2; ++pass) {
                    if (2 * pass >= nch) break;
                    // the TMA engine has read this warp's previous store block, and every reader of the previous pass is done
                    if (TMA_ST && lane == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
                    wg_sync();
                    const int r = 16 * wq + (lane >> 2), sw = 4 * (r & 7);    // (r + 8) & 7 == r & 7
#pragma unroll
                    for (int i = 0; i < 8; ++i) {                 // n8 block i of this pass -> chunk 2 pass + i / 4
                        const int ch = 2 * pass + (i >> 2), ib = i & 3;
                        if (ch < nch) {
                            const int col = (8 * i + 2 * (lane & 3)) ^ sw;
                            *reinterpret_cast<float2*>(tp + r * 64 + col) = make_float2(acc[ch][4 * ib], acc[ch][4 * ib + 1]);
                            *reinterpret_cast<float2*>(tp + (r + 8) * 64 + col) = make_float2(acc[ch][4 * ib + 2], acc[ch][4 * ib + 3]);
                        }
                    }
                    wg_sync();
                    const int ch = 2 * pass + tsub;
                    uint32_t rv[32];
                    if (ch < nch) {
                        const float4* src = reinterpret_cast<const float4*>(tp + trow * 64 + 32 * tsub);
#pragma unroll
                        for (int q = 0; q < 8; ++q) {
                            const float4 f = src[q ^ (trow & 7)];
                            rv[4 * q] = __float_as_uint(f.x); rv[4 * q + 1] = __float_as_uint(f.y);
                            rv[4 * q + 2] = __float_as_uint(f.z); rv[4 * q + 3] = __float_as_uint(f.w);
                        }
                    }
                    if (TMA_ST) wg_sync();                        // the store blocks are free for epilogue_chunk
                    if (ch < nch) {
                        if (!BPHW_TMA || img)
                            epilogue_chunk<LAYOUT>(rv, s_sn + ch * 32, c0, c1, c2, row0 + ch * 32, p, pok, prm, stg, &map_out,
                                                   nt, ch * 32);
                        else
                            epilogue_chunk<STG_LAYOUT>(rv, s_sn + ch * 32, c0, c1, c2, row0 + ch * 32, p, pok, prm);
                    }
                }
            }
        }
        if (TMA_ST && lane == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");   // stores landed
    }
}

// ------------------------------------------------------------------------------------------ top-1, image tiles
// Per (image, prototype) max / arg-max of log p for isotropic sigma, 32 <= HW <= 256, D in {64, 128}.  An x tile is
// one image, NI = HW rounded up to the next instantiated width; columns >= HW belong to the next image (or lie past
// N and read as zero) and are masked.  Same warp roles and team schedule as logprob_tc_kernel:
//   warp 9   TMA producer of the x tile: one NI-row box per K block and hi / lo half, each K block with its own
//            full / empty barrier pair, so the next image's first K block loads while the current image's last
//            prototype tile still multiplies its second one
//   warp 8   TMA producer of the prototype half tiles through an S-stage ring: a stage is one warpgroup's 64 rows of
//            one K block (hi and lo, 16 KiB through a 64-row box), loaded in the order the warpgroups consume them --
//            per prototype tile warpgroup 0's K blocks, then warpgroup 1's -- and released by the 4 warps that read it
//   warps 0-7  warpgroup g multiplies prototype rows [64 g, 64 g + 64) of the tile with the whole image: per k16
//            step one m64nNIk16 MMA per pass (hi*hi, lo*hi, hi*lo), one commit group per K block, the previous K
//            block's group retired (and its stage released) while the current one runs.  The warpgroups take turns
//            issuing (ping-pong, ordered by two named barriers): warpgroup 0 issues tile j while warpgroup 1 runs the
//            epilogue of tile j - 1, then warpgroup 1 issues tile j while warpgroup 0 runs the epilogue of tile j, so
//            the tensor cores always have the other warpgroup's MMAs queued behind the ones that finish.  The epilogue
//            reads the fragments in place: a thread holds 2 prototype rows x NI / 4 columns; it keeps the running (max,
//            first column) of each row, a quad of lanes merges its four by two shuffles, and lane 0 of the quad writes
//            the packed result with a plain 64-bit store -- every (image, prototype) pair has exactly one writer, so
//            `best` needs no zeroing and no atomics.  Turns change nothing a result depends on: each accumulator
//            element receives the same MMAs in the same order as without them.
// HW_MIN: the smallest HW this width serves; 8-column blocks below it need no mask.
template <int NI, int HW_MIN>
__global__ void __launch_bounds__(TC_THREADS, 1)
logprob_top1_wide_kernel(const __grid_constant__ CUtensorMap map_xh, const __grid_constant__ CUtensorMap map_xl,
                         const __grid_constant__ CUtensorMap map_ph, const __grid_constant__ CUtensorMap map_pl,
                         const TcParams prm) {
    static_assert(NI % 8 == 0 && NI >= 32 && NI <= 256 && HW_MIN <= NI, "wgmma N");
    constexpr int R = NI / 2;                                     // accumulator registers per thread
    constexpr uint32_t XSUB = (uint32_t)NI * KB * 2;              // one [NI x 64] fp16 block of the x tile
    constexpr uint32_t HSUB = 64u * KB * 2;                       // one warpgroup's [64 x 64] fp16 half of a K block
    constexpr int SMAX = 8;                                       // prototype stages at most (barrier slots)
    extern __shared__ uint8_t smem_raw[];
    const uint32_t raw = smem_u32(smem_raw);
    const uint32_t base = (raw + 1023u) & ~1023u;                 // SWIZZLE_128B tiles need 1024 B alignment
    uint8_t* base_ptr = smem_raw + (base - raw);

    if (*prm.noniso != 0) {                                       // anisotropic: the 128-patch-tile kernel runs instead
        if (!prm.iso_elsewhere) __trap();                         // ... unless isotropic sigma was promised: fail loudly
        return;
    }
    const int nkb = prm.D / KB;                                   // 1 or 2 K blocks, the [x] / [-2 w mu] half only
    const int kcol0 = prm.D;

    // carve-up: nbuf x tiles (hi blocks then lo blocks) | S prototype half-tile stages (hi, lo) | barriers | |x|^2 of
    // two images per warpgroup
    const uint32_t x_bytes = (uint32_t)(2 * nkb) * XSUB;
    const uint32_t misc_bytes = 256u + 2u * 2u * 256u * 4u;
    const uint32_t tile_budget = prm.smem_bytes - 1024u - misc_bytes;
    const int nbuf = (2 * x_bytes + 8 * 2 * HSUB <= tile_budget) ? 2 : 1;   // double-buffer x when 8 stages still fit
    int S = (int)((tile_budget - nbuf * x_bytes) / (2 * HSUB));
    if (S > SMAX) S = SMAX;
    const uint32_t x_base = base;
    const uint32_t st_base = x_base + nbuf * x_bytes;
    const uint32_t misc = st_base + (uint32_t)S * 2 * HSUB;
    const uint32_t bar0 = misc;                                   // full[8] empty[8] xfull[2][2] xempty[2][2]
    auto FULL = [&](int i) { return bar0 + 8u * i; };
    auto EMPTY = [&](int i) { return bar0 + 8u * (SMAX + i); };
    auto XFULL = [&](int b, int kb) { return bar0 + 8u * (2 * SMAX + 2 * b + kb); };
    auto XEMPTY = [&](int b, int kb) { return bar0 + 8u * (2 * SMAX + 4 + 2 * b + kb); };
    float* s_sn = reinterpret_cast<float*>(base_ptr + (misc - base) + 256);   // [2 warpgroups][2 images][256]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        // prototype empty: one arrive per warp of the warpgroup that read the stage; x empty: per consumer warp
        for (int i = 0; i < SMAX; ++i) { mbar_init(FULL(i), 1); mbar_init(EMPTY(i), 4); }
        for (int b = 0; b < 2; ++b)
            for (int kb = 0; kb < 2; ++kb) { mbar_init(XFULL(b, kb), 1); mbar_init(XEMPTY(b, kb), 8); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int TS = prm.team;
    const int n_teams = gridDim.x / TS, team = blockIdx.x / TS, k0 = blockIdx.x % TS;
    const int n_ptiles = prm.n_ptiles, B = prm.B, HW = prm.HW;
    if (team >= n_teams || k0 >= n_ptiles) return;                // nothing to do for this CTA (tiny problems)

    if (warp == 9) {
        // =========================== x-tile TMA producer ===========================
        if (lane == 0) {
            int c = 0;
            for (int nt = team; nt < B; nt += n_teams, ++c) {
                const int buf = c % nbuf, use = c / nbuf;
                const uint32_t xb = x_base + (uint32_t)buf * x_bytes;
                for (int kb = 0; kb < nkb; ++kb) {
                    if (use > 0) mbar_wait(XEMPTY(buf, kb), (uint32_t)((use - 1) & 1));
                    mbar_expect_tx(XFULL(buf, kb), 2 * XSUB);
                    tma_load_2d(xb + (uint32_t)kb * XSUB, &map_xh, kcol0 + kb * KB, nt * HW, XFULL(buf, kb));
                    tma_load_2d(xb + (uint32_t)(nkb + kb) * XSUB, &map_xl, kcol0 + kb * KB, nt * HW, XFULL(buf, kb));
                }
            }
        }
    } else if (warp == 8) {
        // =========================== prototype TMA producer ===========================
        // stage order per prototype tile: warpgroup 0's K blocks, then warpgroup 1's
        if (lane == 0) {
            int stage = 0;
            uint32_t phase = 0;
            for (int nt = team; nt < B; nt += n_teams)
                for (int pt = k0; pt < n_ptiles; pt += TS)
                    for (int h = 0; h < 2; ++h)
                        for (int kb = 0; kb < nkb; ++kb) {
                            const int r0 = pt * PT + 64 * h;
                            mbar_wait(EMPTY(stage), phase ^ 1u);
                            if ((prm.debug & 16) || r0 >= prm.P) {
                                // no load: switched off, or no prototype row in this half (its results are not stored)
                                mbar_arrive(FULL(stage));
                            } else {
                                mbar_expect_tx(FULL(stage), 2 * HSUB);
                                const uint32_t dst = st_base + (uint32_t)stage * 2 * HSUB;
                                tma_load_2d(dst, &map_ph, kcol0 + kb * KB, r0, FULL(stage));
                                tma_load_2d(dst + HSUB, &map_pl, kcol0 + kb * KB, r0, FULL(stage));
                            }
                            if (++stage == S) { stage = 0; phase ^= 1u; }
                        }
        }
    } else {
        // =========================== consumers: MMA + epilogue ===========================
        const int wg = warp >> 2, wq = warp & 3, q = lane & 3, u = threadIdx.x & 127;
        const int prow = wg * 64 + 16 * wq + (lane >> 2);         // this thread's prototype rows: prow and prow + 8
        unsigned long long* best = reinterpret_cast<unsigned long long*>(prm.out);
        // turns: named barrier 4 + g = "warpgroup g may issue its MMAs of the next tile" (one warpgroup arrives, the
        // other waits, 256 threads; 2 + g syncs warpgroup g alone); warpgroup 0 takes the first turn without waiting,
        // and warpgroup 1 hands a turn back only when another tile follows, so every arrive has its wait
        auto wait_turn = [&]() { if (wg) named_bar_sync<5, 256>(); else named_bar_sync<4, 256>(); };
        auto give_turn = [&]() { if (wg) named_bar_arrive<4, 256>(); else named_bar_arrive<5, 256>(); };
        // ring position: this warpgroup's stages of a tile follow nkb stages of warpgroup 0 (for warpgroup 1) and are
        // followed by nkb of warpgroup 1 (for warpgroup 0); nkb <= 2 < S
        int stage = wg * nkb, c = 0;
        uint32_t phase = 0;
        auto advance = [&](int n) { stage += n; if (stage >= S) { stage -= S; phase ^= 1u; } };
        bool first = true;
        for (int nt = team; nt < B; nt += n_teams, ++c) {
            const int buf = c % nbuf;
            const uint32_t xpar = (uint32_t)((c / nbuf) & 1);
            const uint32_t xb = x_base + (uint32_t)buf * x_bytes;
            // |x|^2 of this image, a copy per warpgroup so that neither waits for the other, double-buffered by image:
            // the readers of buffer c & 1 (image c - 2) are this warpgroup's threads, all past the previous image's barrier
            float* sn = s_sn + wg * 512 + (c & 1) * 256;
            for (int i = u; i < NI; i += 128) sn[i] = (i < HW) ? prm.sn[(size_t)nt * HW + i] : 0.f;
            if (wg) named_bar_sync<3, 128>(); else named_bar_sync<2, 128>();
            for (int pt = k0; pt < n_ptiles; pt += TS) {
                const bool last = pt + TS >= n_ptiles;            // last prototype tile of this image: release x
                const bool more = !last || nt + n_teams < B;      // another tile follows in this CTA
                const int p0 = pt * PT + prow, p1 = p0 + 8;
                const float c0a = p0 < prm.P ? __ldg(prm.e0 + p0) : 0.f, c0b = p1 < prm.P ? __ldg(prm.e0 + p1) : 0.f;
                const float c1a = p0 < prm.P ? __ldg(prm.e1 + p0) : 0.f, c1b = p1 < prm.P ? __ldg(prm.e1 + p1) : 0.f;
                const float c2a = p0 < prm.P ? __ldg(prm.e2 + p0) : 0.f, c2b = p1 < prm.P ? __ldg(prm.e2 + p1) : 0.f;
                float acc[R];
#pragma unroll
                for (int j = 0; j < R; ++j) acc[j] = 0.f;
                if (wg == 1 || !first) wait_turn();               // the other warpgroup has issued its MMAs
                first = false;
                int prev = 0;
                for (int kb = 0; kb < nkb; ++kb) {
                    mbar_wait(XFULL(buf, kb), xpar);
                    mbar_wait(FULL(stage), phase);
                    if (!(prm.debug & 4)) {
                        const uint32_t ph = st_base + (uint32_t)stage * 2 * HSUB;
                        const uint32_t pl = ph + HSUB;
                        const uint32_t xh = xb + (uint32_t)kb * XSUB, xl = xb + (uint32_t)(nkb + kb) * XSUB;
                        wg_fence();
#pragma unroll
                        for (int k = 0; k < KB / 16; ++k) {
                            const uint32_t off = (uint32_t)k * 32u;   // 16 fp16 = 32 B inside the 128 B swizzle row
                            const uint64_t a_h = gmma_desc(ph + off), a_l = gmma_desc(pl + off);
                            const uint64_t b_h = gmma_desc(xh + off), b_l = gmma_desc(xl + off);
                            wg_mma_ss<NI>(acc, a_h, b_h);
                            wg_mma_ss<NI>(acc, a_l, b_h);
                            wg_mma_ss<NI>(acc, a_h, b_l);
                        }
                        wg_commit();
                    }
                    // every MMA of this tile is issued: the other warpgroup's turn (its MMAs queue behind these)
                    if (kb == nkb - 1 && (wg == 0 || more)) give_turn();
                    if (kb > 0) {                                 // K block kb - 1 has retired: release what it read
                        wg_wait<1>();
                        __syncwarp();
                        if (lane == 0) {
                            mbar_arrive(EMPTY(prev));
                            if (last) mbar_arrive(XEMPTY(buf, kb - 1));
                        }
                    }
                    prev = stage;
                    advance(1);
                }
                advance(nkb);                                     // past the other warpgroup's stages of this tile
                wg_wait<0>();
                wg_fence_operands(acc);
                __syncwarp();
                if (lane == 0) {
                    mbar_arrive(EMPTY(prev));
                    if (last) mbar_arrive(XEMPTY(buf, nkb - 1));
                }
                if (prm.debug & 8) continue;
                // v = e0 + e1 acc + e2 |x|^2, the expression and rounding of epilogue_chunk; strict '>' over increasing
                // columns keeps the first of equal maxima
                float ma = -INFINITY, mb = -INFINITY;
                int ia = 0, ib = 0;
#pragma unroll
                for (int i = 0; i < NI / 8; ++i) {
                    const float2 s = *reinterpret_cast<const float2*>(sn + 8 * i + 2 * q);
#pragma unroll
                    for (int j = 0; j < 2; ++j) {
                        const int col = 8 * i + 2 * q + j;
                        const bool ok = (8 * i + 8 <= HW_MIN) || col < HW;
                        const float sj = j ? s.y : s.x;
                        const float va = fmaf(c1a, acc[4 * i + j], fmaf(c2a, sj, c0a));
                        const float vb = fmaf(c1b, acc[4 * i + 2 + j], fmaf(c2b, sj, c0b));
                        if (ok && va > ma) { ma = va; ia = col; }
                        if (ok && vb > mb) { mb = vb; ib = col; }
                    }
                }
#pragma unroll
                for (int o = 1; o <= 2; o <<= 1) {                // merge the quad: larger value, then smaller column
                    const float oa = __shfl_xor_sync(0xffffffffu, ma, o), ob = __shfl_xor_sync(0xffffffffu, mb, o);
                    const int ja = __shfl_xor_sync(0xffffffffu, ia, o), jb = __shfl_xor_sync(0xffffffffu, ib, o);
                    if (oa > ma || (oa == ma && ja < ia)) { ma = oa; ia = ja; }
                    if (ob > mb || (ob == mb && jb < ib)) { mb = ob; ib = jb; }
                }
                if (q == 0 && (!(prm.debug & 1) || ma + mb == 123.456f)) {
                    if (p0 < prm.P) best[(size_t)nt * prm.P + p0] = top1_pack(ma, ia);
                    if (p1 < prm.P) best[(size_t)nt * prm.P + p1] = top1_pack(mb, ib);
                }
            }
        }
    }
}

// ------------------------------------------------------------------------------------------ host
// output [N, P] fp32 row-major, box = 32 prototypes x 32 patches, no swizzle (TMA-store epilogue)
bool make_out_map(CUtensorMap* m, const void* ptr, uint64_t N, uint64_t P) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[2] = {P, N};
    cuuint64_t strides[1] = {P * sizeof(float)};
    cuuint32_t box[2] = {32, 32};
    cuuint32_t es[2] = {1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, const_cast<void*>(ptr), dims, strides, box, es,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_NONE,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

// output [B, P, HW] fp32, box = 32 patches x 32 prototypes x 1 image, 128B swizzle (inner box = 128 B)
bool make_out_map_bphw(CUtensorMap* m, const void* ptr, uint64_t B, uint64_t P, uint64_t HW) {
    EncodeTiledFn enc = get_encode();
    if (!enc) return false;
    cuuint64_t dims[3] = {HW, P, B};
    cuuint64_t strides[2] = {HW * sizeof(float), P * HW * sizeof(float)};
    cuuint32_t box[3] = {32, 32, 1};
    cuuint32_t es[3] = {1, 1, 1};
    return enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 3, const_cast<void*>(ptr), dims, strides, box, es,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_NONE,
               CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

struct WsLayout {
    size_t bh, bl, e0, e1, e2, flag, ah, al, sn, total;
};
WsLayout ws_layout(long long N, int P, int D) {
    WsLayout w;
    size_t o = 0;
    w.bh = o; o = align256(o + (size_t)P * 2 * D * 2);
    w.bl = o; o = align256(o + (size_t)P * 2 * D * 2);
    w.e0 = o; o = align256(o + (size_t)P * 4);
    w.e1 = o; o = align256(o + (size_t)P * 4);
    w.e2 = o; o = align256(o + (size_t)P * 4);
    w.flag = o; o = align256(o + 4);
    w.ah = o; o = align256(o + (size_t)N * 2 * D * 2);
    w.al = o; o = align256(o + (size_t)N * 2 * D * 2);
    w.sn = o; o = align256(o + (size_t)((N + 255) / 256 * 256) * 4);
    w.total = o;
    return w;
}

}  // namespace

// logprob_tcz.cu: [N,P] output, isotropic sigma, D <= 128: patch operands resident in registers, x split fused
bool mgp_logprob_tcz_supported(int P, int D);
int mgp_logprob_tcz_launch(const float* xhat, const void* bh, const void* bl, const float* e0, const float* e1,
                           const float* e2, const int* noniso, float* out, long long N, int P, int D, cudaStream_t st);
int mgp_opt_tc_z();   // abi.cu

bool mgp_logprob_tc_supported(int layout, int B, int HW, int P, int D, int assume_iso) {
    (void)layout;
    // K blocks of 64; the x tile (128 patches x K x 4 B, K = 2D when some sigma is anisotropic) must fit in
    // shared memory: D <= 128 always, D = 256 only when the caller asserts isotropic sigma (MGP_MATH_TC_ISO)
    if (!(D == 64 || D == 128 || (D == 256 && assume_iso))) return false;
    if ((long long)B * HW < 1 || P < 1) return false;
    return get_encode() != nullptr;
}

size_t mgp_logprob_tc_ws_bytes(long long N, int P, int D) { return ws_layout(N, P, D).total; }

// the patch-side operand slots of the workspace, for a producer that writes them itself (mgp_normalize_fwd_stage)
bool mgp_logprob_tc_stage_ptrs(void* ws, size_t ws_bytes, long long N, int P, int D, __half** ah, __half** al, float** sn) {
    const WsLayout w = ws_layout(N, P, D);
    if (!ws || ws_bytes < w.total) return false;
    uint8_t* wsb = reinterpret_cast<uint8_t*>(ws);
    *ah = reinterpret_cast<__half*>(wsb + w.ah);
    *al = reinterpret_cast<__half*>(wsb + w.al);
    *sn = reinterpret_cast<float*>(wsb + w.sn);
    return true;
}

// The prototype pre-pass alone (run != 0; else the operands are already there), into the prototype slots of a workspace
// of mgp_logprob_tc_ws_bytes(0, P, D) bytes or more; returns where they are (log_density.cu reads them)
int mgp_logprob_tc_proto_prep(const float* mu, const float* sigma, float eps, float eps_log, void* ws, int P, int D,
                              int run, void** bh, void** bl, float** e0, float** e1, float** e2, int** flag,
                              cudaStream_t st) {
    const WsLayout w = ws_layout(0, P, D);
    uint8_t* wsb = reinterpret_cast<uint8_t*>(ws);
    *bh = wsb + w.bh;
    *bl = wsb + w.bl;
    *e0 = reinterpret_cast<float*>(wsb + w.e0);
    *e1 = reinterpret_cast<float*>(wsb + w.e1);
    *e2 = reinterpret_cast<float*>(wsb + w.e2);
    *flag = reinterpret_cast<int*>(wsb + w.flag);
    if (run) {
        MGP_CUDA(cudaMemsetAsync(*flag, 0, 4, st));
        tc_proto_prep_kernel<<<(P + 7) / 8, 256, 0, st>>>(mu, sigma, eps, eps_log, reinterpret_cast<__half*>(*bh),
                                                          reinterpret_cast<__half*>(*bl), *e0, *e1, *e2, *flag, P, D);
        MGP_CHECK_LAUNCH();
    }
    return MGP_OK;
}

int mgp_logprob_tc_launch(const float* xhat, const float* mu, const float* sigma, float eps, float eps_log, float* out,
                          int layout, int B, int HW, int P, int D, void* ws, size_t ws_bytes, int reuse_operands,
                          int assume_iso, int x_staged, cudaStream_t st) {
    const long long N = (long long)B * HW;
    const WsLayout w = ws_layout(N, P, D);
    if (ws_bytes < w.total) return MGP_ERR_WORKSPACE;
    uint8_t* wsb = reinterpret_cast<uint8_t*>(ws);
    __half* bh = reinterpret_cast<__half*>(wsb + w.bh);
    __half* bl = reinterpret_cast<__half*>(wsb + w.bl);
    __half* ah = reinterpret_cast<__half*>(wsb + w.ah);
    __half* al = reinterpret_cast<__half*>(wsb + w.al);
    float* e0 = reinterpret_cast<float*>(wsb + w.e0);
    float* e1 = reinterpret_cast<float*>(wsb + w.e1);
    float* e2 = reinterpret_cast<float*>(wsb + w.e2);
    float* sn = reinterpret_cast<float*>(wsb + w.sn);
    int* flag = reinterpret_cast<int*>(wsb + w.flag);

    // [N,P] with isotropic sigma (asserted by the caller) and D <= 128: the register-resident kernel reads fp32 x itself
    const bool use_z = (layout == MGP_OUT_LOGP_NP) && assume_iso && mgp_opt_tc_z() && mgp_logprob_tcz_supported(P, D);
    // reuse_operands: 0 = prepare both operand sides, 1 = the prototype side is already in ws, 2 = both sides are
    if (reuse_operands == 0) {
        MGP_CUDA(cudaMemsetAsync(flag, 0, 4, st));
        tc_proto_prep_kernel<<<(P + 7) / 8, 256, 0, st>>>(mu, sigma, eps, eps_log, bh, bl, e0, e1, e2, flag, P, D);
        MGP_CHECK_LAUNCH();
    }
    if (!use_z && reuse_operands < 2 && !(x_staged & 1)) {
        tc_x_prep_kernel<<<(unsigned)((N + 7) / 8), 256, 0, st>>>(xhat, ah, al, sn, flag, (int)N, D);
        MGP_CHECK_LAUNCH();
    }
    if (use_z) return mgp_logprob_tcz_launch(xhat, bh, bl, e0, e1, e2, flag, out, N, P, D, st);

    CUtensorMap mxh, mxl, mph, mpl;
    CUtensorMap mout;
    const char* no_tma = getenv("MGP_TC_NO_TMA_STORE");
    const bool tma_ok = !(no_tma && atoi(no_tma));
    const bool tma_np = (layout == MGP_OUT_LOGP_NP) && (P % 4 == 0) && tma_ok;
    // [B,P,HW] through the 3-D map uses image-aligned x tiles (a chunk may not cross an image end)
    const bool tma_bphw = (layout != MGP_OUT_LOGP_NP) && (HW % 4 == 0) && HW >= 32 && HW <= 256 && tma_ok && D <= 128;
    const bool top1 = (layout == MGP_OUT_TOP1_BP);
    // top-1 with image tiles (logprob_top1_wide_kernel) unless sigma is known to be anisotropic (x staged with its x^2
    // half).  Whether sigma is isotropic is otherwise decided on the device (tc_proto_prep_kernel's flag): unless the
    // caller promised it, the 128-patch-tile kernel is launched behind the wide one and returns at once when it is.
    const bool iso_known = assume_iso || x_staged == 1;
    const bool top1_wide = top1 && HW >= 32 && HW <= 256 && (D == 64 || D == 128) && x_staged != 2;
    const bool top1_tiles = top1 && (!top1_wide || !iso_known);
    // image-aligned x tiles (box of 32 rows) for the [B,P,HW] TMA stores
    const bool img_tiles = tma_bphw && !top1;
    const uint32_t xbox = img_tiles ? 32u : 128u;
    if (top1_tiles) MGP_CUDA(cudaMemsetAsync(out, 0, (size_t)B * P * sizeof(unsigned long long), st));
    if (!make_map_f16(&mxh, ah, (uint64_t)N, 2 * D, xbox) || !make_map_f16(&mxl, al, (uint64_t)N, 2 * D, xbox) ||
        !make_map_f16(&mph, bh, (uint64_t)P, 2 * D, 128) || !make_map_f16(&mpl, bl, (uint64_t)P, 2 * D, 128))
        return MGP_ERR_UNSUPPORTED;
    if (tma_bphw && !top1) {
        if (!make_out_map_bphw(&mout, out, (uint64_t)B, (uint64_t)P, (uint64_t)HW)) return MGP_ERR_UNSUPPORTED;
    } else if (!make_out_map(&mout, tma_np ? out : (float*)ah, tma_np ? (uint64_t)N : 64, tma_np ? (uint64_t)P : 64)) {
        return MGP_ERR_UNSUPPORTED;
    }

    TcParams prm;
    prm.e0 = e0; prm.e1 = e1; prm.e2 = e2; prm.sn = sn; prm.noniso = flag; prm.out = out;
    prm.N = (int)N; prm.HW = HW; prm.P = P; prm.D = D;
    prm.x_no_sq = (x_staged == 1) ? 1 : 0;          // staged without the x^2 half: an anisotropic sigma must fault, not read stale data
    prm.iso_elsewhere = 0;
    {
        const char* dbg = getenv("MGP_TC_DEBUG");
        prm.debug = dbg ? atoi(dbg) : 0;
    }
    prm.n_ptiles = (P + PT - 1) / PT;
    prm.n_ntiles = (int)((N + 127) / 128);
    prm.B = B;
    prm.xbox = (int)xbox;
    prm.nti = ((HW + 31) / 32) * 32;
    int sms = 0;
    MGP_CUDA(mgp_sm_count(&sms));
    // teams of 4 CTAs (fewer when there are fewer prototype tiles) share an x tile and write adjacent tiles
    int team = 4;
    {
        const char* ts = getenv("MGP_TC_TEAM");
        if (ts && atoi(ts) > 0) team = atoi(ts);
    }
    if (team > prm.n_ptiles) team = prm.n_ptiles;
    if (team > sms) team = sms;
    const int n_teams_max = sms / team;
    prm.team = team;
    const size_t smem = (size_t)227 * 1024;
    prm.smem_bytes = (uint32_t)smem;

    if (top1_wide) {
        // the x map's box is the whole image tile (NI rows, NI = HW rounded up to an instantiated width); the prototype
        // maps' box is one warpgroup's 64 rows (the kernel's ring stages are half tiles)
        const int ni = HW <= 32 ? 32 : HW <= 56 ? 56 : HW <= 64 ? 64 : HW <= 128 ? 128 : HW <= 200 ? 200 : 256;
        CUtensorMap wxh, wxl, wph, wpl;
        if (!make_map_f16(&wxh, ah, (uint64_t)N, 2 * D, (uint32_t)ni) || !make_map_f16(&wxl, al, (uint64_t)N, 2 * D, (uint32_t)ni) ||
            !make_map_f16(&wph, bh, (uint64_t)P, 2 * D, 64) || !make_map_f16(&wpl, bl, (uint64_t)P, 2 * D, 64))
            return MGP_ERR_UNSUPPORTED;
        TcParams pw = prm;
        pw.iso_elsewhere = iso_known ? 0 : 1;
        const int grid_w = (n_teams_max < B ? n_teams_max : B) * team;
#define MGP_TOP1_WIDE(NI, LO)                                                                                      \
    do {                                                                                                           \
        MGP_CUDA(cudaFuncSetAttribute(logprob_top1_wide_kernel<NI, LO>, cudaFuncAttributeMaxDynamicSharedMemorySize, \
                                      (int)smem));                                                                 \
        logprob_top1_wide_kernel<NI, LO><<<grid_w, TC_THREADS, smem, st>>>(wxh, wxl, wph, wpl, pw);               \
    } while (0)
        switch (ni) {
            case 32: MGP_TOP1_WIDE(32, 32); break;
            case 56: MGP_TOP1_WIDE(56, 33); break;
            case 64: MGP_TOP1_WIDE(64, 57); break;
            case 128: MGP_TOP1_WIDE(128, 65); break;
            case 200: MGP_TOP1_WIDE(200, 129); break;
            default: MGP_TOP1_WIDE(256, 201); break;
        }
#undef MGP_TOP1_WIDE
        MGP_CHECK_LAUNCH();
        if (!top1_tiles) return MGP_OK;
        prm.iso_elsewhere = 1;
    }

    int n_teams = n_teams_max;
    {
        const int nt_min = (img_tiles && B < prm.n_ntiles) ? B : prm.n_ntiles;
        if (n_teams > nt_min) n_teams = nt_min;
    }
    const int grid = n_teams * team;
    // shared memory: 1 KiB alignment slack + x tile(s) + prototype stages + 32 KiB staging + 2 KiB misc
    const size_t x_max = (size_t)(assume_iso && D > 128 ? 512 : 1024) * D;   // general: 128 x 2D x 4 B (isotropic: half)
    if (1024 + x_max + (size_t)2 * 2 * SUB_BYTES + STAGING_BYTES + 2048 > smem)
        return MGP_ERR_UNSUPPORTED;

#define MGP_TC_LAUNCH(L)                                                                                           \
    do {                                                                                                           \
        MGP_CUDA(cudaFuncSetAttribute(logprob_tc_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)); \
        logprob_tc_kernel<L><<<grid, TC_THREADS, smem, st>>>(mxh, mxl, mph, mpl, mout, prm);                               \
    } while (0)
    if (top1) MGP_TC_LAUNCH(LAYOUT_TOP1);
    else if (tma_np) MGP_TC_LAUNCH(LAYOUT_NP_TMA);
    else if (tma_bphw && layout == MGP_OUT_LOGP_BPHW) MGP_TC_LAUNCH(LAYOUT_BPHW_TMA);
    else if (tma_bphw) MGP_TC_LAUNCH(LAYOUT_NEGP_TMA);
    else if (layout == MGP_OUT_LOGP_NP) MGP_TC_LAUNCH(MGP_OUT_LOGP_NP);
    else if (layout == MGP_OUT_LOGP_BPHW) MGP_TC_LAUNCH(MGP_OUT_LOGP_BPHW);
    else MGP_TC_LAUNCH(MGP_OUT_NEGP_BPHW);
#undef MGP_TC_LAUNCH
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}
