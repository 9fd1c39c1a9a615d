// a2/a3/a16: diagonal-Gaussian log-likelihood of every patch under every prototype,
// exact-form fp32 SIMT version (MGP_MATH_FP32).
// ref: model.py:256-275 (compute_log_prob), :323-336 (_estimate_log_prob), :429-438.
//
//   log p[n,p] = cst[p] - 1/2 sum_d ((x[n,d] - mu[p,d]) * rinv[p,d])^2
//   rinv = 1/(sigma+eps),  cst = -D/2 log 2pi - sum_d log(sigma+eps_log)      (prep kernel)
//
// Register-tiled like an SGEMM (128x128 CTA tile, 8x8 per thread, K-step 16), but the
// inner op is sub-mul-fma on the *difference* -- the same arithmetic form as the
// reference, so the result carries no cancellation error.  3 issue slots per pair-dim:
// this kernel is bound by the fp32 pipe, not by HBM;
// it is the exact path and the fallback for shapes the tensor-core kernel does not take.
#include "mgp_common.cuh"

namespace {

constexpr int BT = 128;  // tile edge (both sides)
constexpr int BK = 16;
constexpr int PITCH = BT + 4;

__global__ void proto_prep_kernel(const float* __restrict__ sigma, float eps, float eps_log, float* __restrict__ rinv,
                                  float* __restrict__ cst, int P, int D) {
    const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (p >= P) return;
    float ls = 0.f;
    for (int d = lane; d < D; d += 32) {
        float s = sigma[(size_t)p * D + d];
        rinv[(size_t)p * D + d] = 1.0f / (s + eps);
        ls += logf(s + eps_log) + 0.5f * MGP_LOG_2PI;   // per-dim terms: no 470 - 470 cancellation at D = 512
    }
    ls = warp_sum(ls);
    if (lane == 0) cst[p] = -ls;
}

// PROTO_ON_I: rows i of the tile are prototypes and columns j are patches (BPHW layouts);
// otherwise rows are patches and columns prototypes (NP layout).  Lanes run along j.
template <int LAYOUT>
__global__ void __launch_bounds__(256, 2)
logprob_simt_kernel(const float* __restrict__ x, const float* __restrict__ mu, const float* __restrict__ rinv,
                    const float* __restrict__ cst, float* __restrict__ out, int N, int HW, int P, int D) {
    constexpr bool PROTO_ON_I = (LAYOUT != MGP_OUT_LOGP_NP);
    __shared__ __align__(16) float Xs[BK][PITCH];
    __shared__ __align__(16) float Ms[BK][PITCH];
    __shared__ __align__(16) float Rs[BK][PITCH];

    const int tid = threadIdx.x;
    const int tj = tid & 15, ti = tid >> 4;
    const int i0 = blockIdx.y * BT, j0 = blockIdx.x * BT;
    const int n0 = PROTO_ON_I ? j0 : i0;
    const int p0 = PROTO_ON_I ? i0 : j0;

    float acc[8][8];
#pragma unroll
    for (int a = 0; a < 8; ++a)
#pragma unroll
        for (int c = 0; c < 8; ++c) acc[a][c] = 0.f;

    for (int k0 = 0; k0 < D; k0 += BK) {
        // global -> smem (transposed to [k][row]); 128 rows x 16 floats per operand
#pragma unroll
        for (int s = 0; s < 2; ++s) {
            const int f = tid + 256 * s;
            const int row = f >> 2, c4 = (f & 3) * 4;
            const int k = k0 + c4;
            float4 vx = make_float4(0.f, 0.f, 0.f, 0.f), vm = vx, vr = vx;
            if (k < D) {
                if (n0 + row < N) vx = __ldg(reinterpret_cast<const float4*>(x + (size_t)(n0 + row) * D + k));
                if (p0 + row < P) {
                    vm = __ldg(reinterpret_cast<const float4*>(mu + (size_t)(p0 + row) * D + k));
                    vr = __ldg(reinterpret_cast<const float4*>(rinv + (size_t)(p0 + row) * D + k));
                }
            }
            Xs[c4 + 0][row] = vx.x; Xs[c4 + 1][row] = vx.y; Xs[c4 + 2][row] = vx.z; Xs[c4 + 3][row] = vx.w;
            Ms[c4 + 0][row] = vm.x; Ms[c4 + 1][row] = vm.y; Ms[c4 + 2][row] = vm.z; Ms[c4 + 3][row] = vm.w;
            Rs[c4 + 0][row] = vr.x; Rs[c4 + 1][row] = vr.y; Rs[c4 + 2][row] = vr.z; Rs[c4 + 3][row] = vr.w;
        }
        __syncthreads();
#pragma unroll
        for (int k = 0; k < BK; ++k) {
            float xv[8], mv[8], rv[8];
            const int ox = (PROTO_ON_I ? tj : ti) * 4;  // patch-side offset
            const int op = (PROTO_ON_I ? ti : tj) * 4;  // prototype-side offset
            *reinterpret_cast<float4*>(&xv[0]) = *reinterpret_cast<const float4*>(&Xs[k][ox]);
            *reinterpret_cast<float4*>(&xv[4]) = *reinterpret_cast<const float4*>(&Xs[k][64 + ox]);
            *reinterpret_cast<float4*>(&mv[0]) = *reinterpret_cast<const float4*>(&Ms[k][op]);
            *reinterpret_cast<float4*>(&mv[4]) = *reinterpret_cast<const float4*>(&Ms[k][64 + op]);
            *reinterpret_cast<float4*>(&rv[0]) = *reinterpret_cast<const float4*>(&Rs[k][op]);
            *reinterpret_cast<float4*>(&rv[4]) = *reinterpret_cast<const float4*>(&Rs[k][64 + op]);
#pragma unroll
            for (int a = 0; a < 8; ++a)
#pragma unroll
                for (int c = 0; c < 8; ++c) {
                    const int ip = PROTO_ON_I ? a : c;
                    const int ix = PROTO_ON_I ? c : a;
                    const float t = (xv[ix] - mv[ip]) * rv[ip];
                    acc[a][c] = fmaf(t, t, acc[a][c]);
                }
        }
        __syncthreads();
    }

    // epilogue
    if (LAYOUT == MGP_OUT_LOGP_NP) {
        const bool vec = (P & 3) == 0;
#pragma unroll
        for (int a = 0; a < 8; ++a) {
            const int n = i0 + (a >> 2) * 64 + ti * 4 + (a & 3);
            if (n >= N) continue;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int p = j0 + h * 64 + tj * 4;
                if (p >= P) continue;
                float v[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) v[c] = (p + c < P) ? cst[p + c] - 0.5f * acc[a][h * 4 + c] : 0.f;
                float* dst = out + (size_t)n * P + p;
                if (vec) {
                    *reinterpret_cast<float4*>(dst) = make_float4(v[0], v[1], v[2], v[3]);
                } else {
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        if (p + c < P) dst[c] = v[c];
                }
            }
        }
    } else {
        const bool vec = (HW & 3) == 0;  // then 4 consecutive n (n % 4 == 0) share an image and are 16B-aligned
#pragma unroll
        for (int a = 0; a < 8; ++a) {
            const int p = i0 + (a >> 2) * 64 + ti * 4 + (a & 3);
            if (p >= P) continue;
            const float cp = cst[p];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int n = j0 + h * 64 + tj * 4;
                if (n >= N) continue;
                float v[4];
#pragma unroll
                for (int c = 0; c < 4; ++c) {
                    float lp = cp - 0.5f * acc[a][h * 4 + c];
                    v[c] = (LAYOUT == MGP_OUT_NEGP_BPHW) ? -expf(lp) : lp;
                }
                if (vec && n + 3 < N) {
                    const int b = n / HW, hw = n - b * HW;
                    *reinterpret_cast<float4*>(out + ((size_t)b * P + p) * HW + hw) = make_float4(v[0], v[1], v[2], v[3]);
                } else {
#pragma unroll
                    for (int c = 0; c < 4; ++c)
                        if (n + c < N) {
                            const int b = (n + c) / HW, hw = (n + c) - b * HW;
                            out[((size_t)b * P + p) * HW + hw] = v[c];
                        }
                }
            }
        }
    }
}

}  // namespace

// Exposed to logprob.cu (dispatcher)
int mgp_logprob_simt_launch(const float* xhat, const float* mu, const float* sigma, float eps, float eps_log,
                            float* out, int layout, int B, int HW, int P, int D, float* ws, cudaStream_t st) {
    float* rinv = ws;
    float* cst = ws + (size_t)P * D;
    proto_prep_kernel<<<(P + 7) / 8, 256, 0, st>>>(sigma, eps, eps_log, rinv, cst, P, D);
    MGP_CHECK_LAUNCH();
    const int N = B * HW;
    if (layout == MGP_OUT_LOGP_NP) {
        dim3 grid((P + BT - 1) / BT, (N + BT - 1) / BT);
        logprob_simt_kernel<MGP_OUT_LOGP_NP><<<grid, 256, 0, st>>>(xhat, mu, rinv, cst, out, N, HW, P, D);
    } else {
        dim3 grid((N + BT - 1) / BT, (P + BT - 1) / BT);
        if (layout == MGP_OUT_LOGP_BPHW)
            logprob_simt_kernel<MGP_OUT_LOGP_BPHW><<<grid, 256, 0, st>>>(xhat, mu, rinv, cst, out, N, HW, P, D);
        else
            logprob_simt_kernel<MGP_OUT_NEGP_BPHW><<<grid, 256, 0, st>>>(xhat, mu, rinv, cst, out, N, HW, P, D);
    }
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}
