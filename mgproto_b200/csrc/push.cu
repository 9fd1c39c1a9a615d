// Prototype projection on the device (ref push.py:125-200, numeric half): a per-prototype store of the K best candidates
// over the whole push set, and the greedy assignment from it.
//
// Prototype (c, k) only considers images labelled c, and the reference's has_pushed_img only couples prototypes of the
// same class.  Prototype k picks after prototypes 0..k-1 of its class, so at most k images are excluded when it picks:
// its pick is always among its own k + 1 best candidates over the push set.  Keeping the K best candidates per
// prototype (value, image id, patch, D-float row) is therefore enough for the exact greedy, and the store's size,
// C*K*K*(D + 4)*4 bytes, does not depend on the number of images.
//
// Every candidate is ordered by one total key, (-p ascending, image id ascending) = f2key(-p) << 32 | id, and ids are
// unique, so the store holds the K smallest keys of everything merged: a set that does not depend on the order in which
// batches or ranks deliver records.  That is what keeps image-sharded replicas identical.
//
//   push_records_kernel  per (image, k): the record fields [rows K*D | val K | patch K | label] (ops._push_rec_views)
//   push_merge_kernel    per prototype (c, k): fold n records of class c into the K slots (lane owns slots lane, lane+32)
//   push_assign_kernel   per class: k = 0..K-1 in order, the smallest key whose id no earlier prototype took -> mu[c,k]
#include "mgp_common.cuh"

namespace {

constexpr unsigned long long EMPTY = 0xffffffffffffffffull;
constexpr int WPB = 8;   // warps per block of the records / merge kernels
constexpr int APB = 4;   // warps (classes) per block of the assign kernel

__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w > v ? w : v;
    }
    return v;
}

__device__ __forceinline__ unsigned long long warp_min_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long w = __shfl_xor_sync(0xffffffffu, v, o);
        v = w < v ? w : v;
    }
    return v;
}

// lowest slot index (0..63) holding `v`; lane owns slots lane (s0) and lane + 32 (s1)
__device__ __forceinline__ int warp_find_slot(unsigned long long s0, unsigned long long s1, bool h0, bool h1,
                                              unsigned long long v) {
    const unsigned b0 = __ballot_sync(0xffffffffu, h0 && s0 == v);
    const unsigned b1 = __ballot_sync(0xffffffffu, h1 && s1 == v);
    return b0 ? __ffs(b0) - 1 : 31 + __ffs(b1);
}

__device__ __forceinline__ void warp_copy_row(float* __restrict__ dst, const float* __restrict__ src, int D, int lane) {
    const float4* s = reinterpret_cast<const float4*>(src);
    float4* d = reinterpret_cast<float4*>(dst);
    for (int i = lane; i < (D >> 2); i += 32) d[i] = s[i];
}

// One warp per (image b, k).  Records are rs fp32 words apart; every field pointer already points into record 0.  A
// label outside [0, C) is written as -1 (the record is ignored); a patch outside [0, HW) is written as -1 (that
// candidate is ignored) and its row is not read.
__global__ void push_records_kernel(const int32_t* __restrict__ arg, const float* __restrict__ val,
                                    const float* __restrict__ xhat, const int64_t* __restrict__ labels,
                                    float* __restrict__ r_rows, float* __restrict__ r_val, int32_t* __restrict__ r_patch,
                                    int64_t* __restrict__ r_label, int rs, int B, int HW, int C, int K, int D) {
    const int wg = blockIdx.x * WPB + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (wg >= B * K) return;
    const int b = wg / K, k = wg - b * K;
    const long long lab = labels[b];
    const bool ok = lab >= 0 && lab < C;
    const int a = ok ? arg[wg] : -1;
    const bool have = a >= 0 && a < HW;
    const size_t ro = (size_t)b * rs;
    float4* dst = reinterpret_cast<float4*>(r_rows + ro + (size_t)k * D);
    const float4* src = reinterpret_cast<const float4*>(xhat + ((size_t)b * HW + (have ? a : 0)) * D);
    for (int i = lane; i < (D >> 2); i += 32) dst[i] = have ? src[i] : make_float4(0.f, 0.f, 0.f, 0.f);
    if (lane == 0) {
        r_val[ro + k] = have ? val[wg] : 0.f;
        r_patch[ro + k] = have ? a : -1;
        if (k == 0) r_label[ro >> 1] = ok ? lab : -1;
    }
}

// One warp per prototype j = c*K + k.  Slot keys and patches live in registers for the whole merge; a replaced slot's
// row is copied at once (every slot of j belongs to this warp alone).  Records with label c are visited in index order,
// but the final set of keys is the K smallest of (store  U  candidates) whatever the order.
__global__ void push_merge_kernel(const float* __restrict__ r_rows, const float* __restrict__ r_val,
                                  const int32_t* __restrict__ r_patch, const int64_t* __restrict__ r_label, int rs,
                                  int n, unsigned id0, unsigned long long* __restrict__ key, int32_t* __restrict__ patch,
                                  float* __restrict__ row, int C, int K, int D) {
    const int j = blockIdx.x * WPB + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (j >= C * K) return;
    const int c = j / K, k = j - c * K;
    unsigned long long* ks = key + (size_t)j * K;
    int32_t* ps = patch + (size_t)j * K;
    float* rw = row + (size_t)j * K * D;
    const bool h0 = lane < K, h1 = lane + 32 < K;
    unsigned long long s0 = h0 ? ks[lane] : 0ull, s1 = h1 ? ks[lane + 32] : 0ull;
    int p0 = h0 ? ps[lane] : -1, p1 = h1 ? ps[lane + 32] : -1;
    unsigned long long mx = warp_max_u64(s0 > s1 ? s0 : s1);
    for (int base = 0; base < n; base += 32) {
        const int i = base + lane;
        const bool mine = i < n && r_label[((size_t)i * rs) >> 1] == c && r_patch[(size_t)i * rs + k] >= 0;
        unsigned todo = __ballot_sync(0xffffffffu, mine);
        while (todo) {
            const int r = base + __ffs(todo) - 1;
            todo &= todo - 1;
            const size_t ro = (size_t)r * rs;
            const unsigned long long cand =
                ((unsigned long long)f2key(r_val[ro + k]) << 32) | (unsigned long long)(id0 + (unsigned)r);
            if (cand >= mx) continue;                                     // warp-uniform
            const int slot = warp_find_slot(s0, s1, h0, h1, mx);
            const int pc = r_patch[ro + k];
            if (slot == lane) { s0 = cand; p0 = pc; }
            if (slot == lane + 32) { s1 = cand; p1 = pc; }
            warp_copy_row(rw + (size_t)slot * D, r_rows + ro + (size_t)k * D, D, lane);
            mx = warp_max_u64(s0 > s1 ? s0 : s1);
        }
    }
    if (h0) { ks[lane] = s0; ps[lane] = p0; }
    if (h1) { ks[lane + 32] = s1; ps[lane + 32] = p1; }
}

// One warp per class c: prototypes k = 0..K-1 in order (push.py:166-200).  Prototype k takes its smallest key whose
// image id none of prototypes 0..k-1 took (their ids in shared memory); without one, it writes id -1 and leaves mu.
__global__ void push_assign_kernel(const unsigned long long* __restrict__ key, const int32_t* __restrict__ patch,
                                   const float* __restrict__ row, float* __restrict__ mu,
                                   int64_t* __restrict__ chosen_id, int64_t* __restrict__ chosen_patch,
                                   float* __restrict__ chosen_val, int C, int K, int D) {
    __shared__ unsigned used_s[APB][64];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int c = blockIdx.x * APB + w;
    if (c >= C) return;
    unsigned* used = used_s[w];
    const bool h0 = lane < K, h1 = lane + 32 < K;
    for (int k = 0; k < K; ++k) {
        const int j = c * K + k;
        const unsigned long long* ks = key + (size_t)j * K;
        unsigned long long s0 = h0 ? ks[lane] : EMPTY, s1 = h1 ? ks[lane + 32] : EMPTY;
        for (int u = 0; u < k; ++u) {                 // an empty slot is EMPTY already: the id -1 mark matches nothing new
            const unsigned id = used[u];
            if ((unsigned)s0 == id) s0 = EMPTY;
            if ((unsigned)s1 == id) s1 = EMPTY;
        }
        const unsigned long long mn = warp_min_u64(s0 < s1 ? s0 : s1);
        if (mn == EMPTY) {
            if (lane == 0) {
                chosen_id[j] = -1;
                chosen_patch[j] = -1;
                chosen_val[j] = INFINITY;
                used[k] = 0xffffffffu;
            }
            __syncwarp();
            continue;
        }
        const int slot = warp_find_slot(s0, s1, h0, h1, mn);
        const unsigned id = (unsigned)mn;
        if (lane == 0) {
            chosen_id[j] = (int64_t)id;
            chosen_patch[j] = patch[(size_t)j * K + slot];
            chosen_val[j] = key2f((unsigned)(mn >> 32));
            used[k] = id;
        }
        warp_copy_row(mu + (size_t)j * D, row + ((size_t)j * K + slot) * D, D, lane);
        __syncwarp();
    }
}

static inline bool aligned8(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 7u) == 0; }

// shape checks shared by the three entry points
static inline int check_ckd(int C, int K, int D) {
    if (C <= 0 || K <= 0 || D <= 0) return MGP_ERR_INVALID;
    if (K > 64 || (D & 3)) return MGP_ERR_UNSUPPORTED;
    if ((long long)C * K > 0x7fffffffLL) return MGP_ERR_UNSUPPORTED;
    return MGP_OK;
}

// record pointers: the fields of record 0, rs fp32 words between records (rows 16-byte, label 8-byte aligned)
static inline int check_records(const float* r_rows, const float* r_val, const int32_t* r_patch, const int64_t* r_label,
                                int rs, int K, int D) {
    if (!r_rows || !r_val || !r_patch || !r_label) return MGP_ERR_INVALID;
    if (rs < (long long)K * D + 2 * K + 2 || (rs & 3) || !mgp_aligned16(r_rows) || !aligned8(r_label))
        return MGP_ERR_INVALID;
    return MGP_OK;
}

}  // namespace

extern "C" int mgp_push_records(const int32_t* arg, const float* val, const float* xhat_nd, const int64_t* labels,
                                float* rec_rows, float* rec_val, int32_t* rec_patch, int64_t* rec_label, int rec_stride,
                                int B, int HW, int C, int K, int D, void* stream) {
    if (!arg || !val || !xhat_nd || !labels) return MGP_ERR_INVALID;
    if (B <= 0 || HW <= 0) return MGP_ERR_INVALID;
    if (int e = check_ckd(C, K, D)) return e;
    if (int e = check_records(rec_rows, rec_val, rec_patch, rec_label, rec_stride, K, D)) return e;
    if (!mgp_aligned16(xhat_nd)) return MGP_ERR_INVALID;
    if ((long long)B * K > 0x7fffffffLL) return MGP_ERR_UNSUPPORTED;
    const int warps = B * K;
    push_records_kernel<<<(warps + WPB - 1) / WPB, WPB * 32, 0, (cudaStream_t)stream>>>(
        arg, val, xhat_nd, labels, rec_rows, rec_val, rec_patch, rec_label, rec_stride, B, HW, C, K, D);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" int mgp_push_merge(const float* rec_rows, const float* rec_val, const int32_t* rec_patch,
                              const int64_t* rec_label, int rec_stride, int n, size_t id0, unsigned long long* key,
                              int32_t* patch, float* row, int C, int K, int D, void* stream) {
    if (!key || !patch || !row) return MGP_ERR_INVALID;
    if (n <= 0 || id0 + (size_t)n > 0xffffffffull) return MGP_ERR_INVALID;    // id 0xffffffff: the empty slot
    if (int e = check_ckd(C, K, D)) return e;
    if (int e = check_records(rec_rows, rec_val, rec_patch, rec_label, rec_stride, K, D)) return e;
    if (!mgp_aligned16(row) || !aligned8(key)) return MGP_ERR_INVALID;
    const int warps = C * K;
    push_merge_kernel<<<(warps + WPB - 1) / WPB, WPB * 32, 0, (cudaStream_t)stream>>>(
        rec_rows, rec_val, rec_patch, rec_label, rec_stride, n, (unsigned)id0, key, patch, row, C, K, D);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}

extern "C" int mgp_push_assign(const unsigned long long* key, const int32_t* patch, const float* row, float* mu,
                               int64_t* chosen_id, int64_t* chosen_patch, float* chosen_val, int C, int K, int D,
                               void* stream) {
    if (!key || !patch || !row || !mu || !chosen_id || !chosen_patch || !chosen_val) return MGP_ERR_INVALID;
    if (int e = check_ckd(C, K, D)) return e;
    if (!mgp_aligned16(row) || !mgp_aligned16(mu) || !aligned8(key) || !aligned8(chosen_id) || !aligned8(chosen_patch))
        return MGP_ERR_INVALID;
    push_assign_kernel<<<(C + APB - 1) / APB, APB * 32, 0, (cudaStream_t)stream>>>(key, patch, row, mu, chosen_id,
                                                                                   chosen_patch, chosen_val, C, K, D);
    MGP_CHECK_LAUNCH();
    return MGP_OK;
}
