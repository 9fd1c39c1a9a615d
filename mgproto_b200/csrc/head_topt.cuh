// Register-resident warp top-T / top-1 over rows of log p, shared by the head's selection kernels (head.cu, head_long.cu).
#pragma once
#include "mgp_common.cuh"

namespace {

// One warp selects the T largest of NR [HW] rows at once (descending, ties -> smaller index).
// Each lane keeps R = ceil(HW/32) keys per row in registers; per level: warp REDUX.max on the lanes'
// local maxima, REDUX.min on the index among equal maxima, winner removed from its lane.  The NR rows
// are independent dependency chains, interleaved to hide the REDUX latency.
template <int R, int NR>
__device__ __forceinline__ void warp_topT(const float* const (&rows)[NR], int rs, int HW, int T, int lane,
                                          float (&out_v)[NR], int (&out_i)[NR]) {
    unsigned key[NR][R];
#pragma unroll
    for (int i = 0; i < NR; ++i) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int j = lane + 32 * r;
            key[i][r] = (j < HW) ? f2key(rows[i][(size_t)j * rs]) : 0u;  // 0 sorts below every real float (incl. -inf)
        }
        out_v[i] = 0.f;
        out_i[i] = 0;
    }
    for (int t = 0; t < T; ++t) {
#pragma unroll
        for (int i = 0; i < NR; ++i) {
            unsigned lm = key[i][0];
#pragma unroll
            for (int r = 1; r < R; ++r) lm = max(lm, key[i][r]);
            int li = 0x7fffffff;
#pragma unroll
            for (int r = R - 1; r >= 0; --r)
                if (key[i][r] == lm) li = lane + 32 * r;
            const unsigned best = __reduce_max_sync(0xffffffffu, lm);
            const int bi = __reduce_min_sync(0xffffffffu, (lm == best) ? li : 0x7fffffff);
#pragma unroll
            for (int r = 0; r < R; ++r)
                if (bi == lane + 32 * r) key[i][r] = 0u;
            if (lane == t) {
                out_v[i] = key2f(best);
                out_i[i] = bi;
            }
        }
    }
}

// Faster variant for R <= 8 (HW <= 256): every lane first sorts its R keys (descending, compile-time
// compare-exchange network), so a level costs one REDUX.max over the lanes' heads, a ballot to find the
// owner (lowest lane among equal heads) and a predicated pop of the owner's list -- ~15 instructions instead
// of ~45.  Indices are recovered at the end from the owner's unsorted copy: lane t fetches the owner's R
// original keys by shuffle and takes the position of its value; equal values picked twice from one lane
// are disambiguated by their rank among earlier identical picks (MATCH.ANY).
template <int R, int NR>
__device__ __forceinline__ void warp_topT_sorted(const float* const (&rows)[NR], int rs, int HW, int T, int lane,
                                                 float (&out_v)[NR], int (&out_i)[NR]) {
    unsigned orig[NR][R], key[NR][R];
#pragma unroll
    for (int i = 0; i < NR; ++i) {
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int j = lane + 32 * r;
            orig[i][r] = (j < HW) ? f2key(rows[i][(size_t)j * rs]) : 0u;
            key[i][r] = orig[i][r];
        }
#pragma unroll
        for (int a = 1; a < R; ++a)
#pragma unroll
            for (int b = a; b >= 1; --b) {
                const unsigned hi = max(key[i][b - 1], key[i][b]), lo = min(key[i][b - 1], key[i][b]);
                key[i][b - 1] = hi;
                key[i][b] = lo;
            }
    }
    unsigned my_key[NR];
    int my_owner[NR];
#pragma unroll
    for (int i = 0; i < NR; ++i) { my_key[i] = 0u; my_owner[i] = 0; }
    for (int t = 0; t < T; ++t) {
#pragma unroll
        for (int i = 0; i < NR; ++i) {
            const unsigned best = __reduce_max_sync(0xffffffffu, key[i][0]);
            const unsigned m = __ballot_sync(0xffffffffu, key[i][0] == best);
            const int owner = __ffs(m) - 1;
            if (lane == owner) {
#pragma unroll
                for (int r = 0; r + 1 < R; ++r) key[i][r] = key[i][r + 1];
                key[i][R - 1] = 0u;
            }
            if (lane == t) { my_key[i] = best; my_owner[i] = owner; }
        }
    }
#pragma unroll
    for (int i = 0; i < NR; ++i) {
        // rank of this pick among earlier picks of the same (value, lane)
        const unsigned long long tag = ((unsigned long long)my_key[i] << 8) | (unsigned)my_owner[i];
        const unsigned same = __match_any_sync(0xffffffffu, (lane < T) ? tag : (0xffffffffffffff00ull | (unsigned)lane));
        int skip = __popc(same & ((1u << lane) - 1u));
        int rr = 0;
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const unsigned o = __shfl_sync(0xffffffffu, orig[i][r], my_owner[i]);
            const bool hit = (o == my_key[i]);
            if (hit && skip == 0) rr = r;
            if (hit) --skip;
        }
        out_v[i] = key2f(my_key[i]);
        out_i[i] = my_owner[i] + 32 * rr;
    }
}

// Level 0 only (max and arg-max, ties -> smaller index) of NR rows: with labels the reference overwrites
// levels >= 1 of every wrong-class prototype with level 0 (model.py:218-221), so only the K rows of the
// image's own class need the full top-T.  ~40 instructions per row instead of ~540: the kernel becomes a
// streaming read of log p.
template <int R, int NR>
__device__ __forceinline__ void warp_top1(const float* const (&rows)[NR], int rs, int HW, int lane,
                                          float (&out_v)[NR], int (&out_i)[NR]) {
    float x[NR][R];
#pragma unroll
    for (int i = 0; i < NR; ++i)
#pragma unroll
        for (int r = 0; r < R; ++r) {
            const int j = lane + 32 * r;
            x[i][r] = (j < HW) ? rows[i][(size_t)j * rs] : -INFINITY;
        }
#pragma unroll
    for (int i = 0; i < NR; ++i) {
        float mv = x[i][0];
        int mr = 0;
#pragma unroll
        for (int r = 1; r < R; ++r)
            if (x[i][r] > mv) { mv = x[i][r]; mr = r; }
        const unsigned key = (lane < HW) ? f2key(mv) : 0u;
        const unsigned best = __reduce_max_sync(0xffffffffu, key);
        out_i[i] = __reduce_min_sync(0xffffffffu, (key == best) ? lane + 32 * mr : 0x7fffffff);
        out_v[i] = key2f(best);
    }
}
}  // namespace
