/*
 * mgproto_b200 -- C ABI of the CUDA-native (H100, sm_90a) MGProto Gaussian-prototype hot path.
 *
 * The reference (cwangrun/MGProto) has no FFI: its boundary is the Python surface of
 * model.MGProto (SURVEY.md section 8b).  Each entry point below replaces the reference code
 * cited beside it ("ref:" = file:line under /root/reference) and is what a binding of
 * that path calls.  Plain pointers and sizes only; no torch types.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer (fp32 unless stated), dense, row-major, 16-byte
 *     aligned; the caller (PyTorch) owns all memory, nothing is allocated or retained;
 *   - kernels are enqueued asynchronously on `stream` (a cudaStream_t passed as void*);
 *   - return value: 0 = launched; >0 = the cudaError_t of the failing call;
 *     <0 = an MGP_ERR_* argument error, nothing launched.  Nothing throws.
 *   - symbols: B images, HW patches/image, N = B*HW, C classes, K prototypes/class,
 *     P = C*K, D feature dim (D % 4 == 0), T mining levels (T <= 32, T <= HW), cap = bank
 *     rows per class.  "sigma" holds standard deviations (ref: model.py:272).
 */
#ifndef MGPROTO_B200_H_
#define MGPROTO_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MGP_ABI_VERSION 2   /* 2: Adam hyper-parameters and tau travel as double (see mgp_em_update) */

#define MGP_OK 0
#define MGP_ERR_INVALID (-1)      /* null pointer / non-positive size / misalignment      */
#define MGP_ERR_UNSUPPORTED (-2)  /* shape outside what the kernels are built for          */
#define MGP_ERR_WORKSPACE (-3)    /* workspace too small (see the *_ws_bytes queries)      */

/* math modes of the log-probability kernels */
#define MGP_MATH_FP32 0     /* exact-form fp32 SIMT: sum_d ((x-mu)/(sigma+eps))^2          */
#define MGP_MATH_TC 1       /* wgmma tensor cores, fp16 hi/lo split x3, fp32 accumulate    */
#define MGP_MATH_AUTO 2     /* TC when the shape qualifies, else FP32                      */
#define MGP_MATH_TC_REUSE 3 /* TC, operands (fp16 hi/lo split of x and of the prototypes) are
                               already staged in `ws` by the previous MGP_MATH_TC call with the
                               same shapes and pointers: only the GEMM kernel is launched       */
#define MGP_MATH_TC_ISO 4   /* TC; the caller asserts that sigma is constant over d inside every
                               prototype (true for every state the reference's loop reaches).
                               Extends the tensor-core path to D = 256; the kernel traps if the
                               assertion is false                                               */
#define MGP_MATH_TC_ISO_REUSE 5 /* TC_ISO with the prototype-side operands already in ws; the patch side is rebuilt */
/* OR-ed onto MGP_MATH_TC / _AUTO / _TC_ISO: the patch-side operands of `ws` (fp16 hi / lo split, |xhat|^2) were
 * written by mgp_normalize_fwd_stage for exactly this xhat_nd -- the tensor-core kernels that read staged patches skip
 * their own pre-pass (the register-resident kernel reads fp32 xhat_nd and ignores the flag).  _ISO: staged with
 * stage_aniso = 0, i.e. without the x^2 half an anisotropic sigma needs: the kernel faults if sigma turns out to be. */
#define MGP_MATH_X_STAGED 0x100
#define MGP_MATH_X_STAGED_ISO 0x200

/* output layouts of mgp_logprob_fwd */
#define MGP_OUT_LOGP_NP 0      /* out[n*P + p]           = log p      (ref: compute_log_prob)   */
#define MGP_OUT_LOGP_BPHW 1    /* out[(b*P + p)*HW + hw] = log p      (feeds mgp_head_select)    */
#define MGP_OUT_NEGP_BPHW 2    /* out[(b*P + p)*HW + hw] = -exp(log p) (ref: push_forward :437)  */
#define MGP_OUT_TOP1_BP 3      /* no log p output: `out` is uint64 [B,P], out[b*P + p] = packed
                                  (max_hw log p, arg max) -- ((monotone key of the float) << 32) |
                                  (0xffffffff - hw), ties -> smaller hw.  Tensor-core path only
                                  (MGP_ERR_UNSUPPORTED otherwise); feeds mgp_head_select_top1    */

/* feature formats of the add-on features x [B,D,H,W] (the x_fmt argument of the *_x entry points): element type,
 * OR-ed with MGP_X_NHWC when x is channels_last, i.e. [B,HW,D] = [N,D] row-major (NCHW, [B,D,HW], otherwise).
 * torch.autocast makes the add-on convolutions return bf16 / fp16.  Only x and its gradient take these formats:
 * xhat, inv_norm, the staged operands and the NCHW copy of xhat are fp32 in every format. */
#define MGP_X_F32 0
#define MGP_X_BF16 1
#define MGP_X_F16 2
#define MGP_X_NHWC 4

int mgp_abi_version(void);
const char* mgp_error_string(int code);
/* 1 if the library was built with the sm_90a tensor-core (wgmma) kernels */
int mgp_has_tensor_core_path(void);
/* Process-wide test / diagnosis switches (not part of the reference surface; the defaults are the product path).
 * key "tc_z": 1 (default; 0 if MGP_TC_NO_Z is set) = the [N,P] log-likelihood with isotropic sigma and D <= 128 takes the
 * register-resident kernel (csrc/logprob_tcz.cu), 0 = always csrc/logprob_tc.cu;
 * key "em_tc": 1 (default; 0 if MGP_EM_NO_TC is set) = mgp_update_gmm may take the tensor-core kernel;
 * key "em_fused": 1 (default; 0 if MGP_EM_UNFUSED is set in the environment) = mgp_update_gmm runs the single
 * cluster launch where the shape allows, 0 = always the multi-launch path (identical arithmetic, used by the
 * parity tests to cross-check the two).  Returns the previous value, or MGP_ERR_INVALID for an unknown key. */
int mgp_set_option(const char* key, int value);
/* Profiling hooks.  key "em_tc_prof": p = device buffer of 64*8 int64 (or NULL to stop) that the tensor-core EM kernel
 * fills with clock64 stamps of its pipeline phases for class `arg` (tools/em_tc_prof.py prints them). */
int mgp_debug_set_ptr(const char* key, void* p, int arg);

/* ---- a1  l2_normalize + rearrange -------------------------------------------------------
 * ref: model.py:40-41, :210-211, :431-432.
 * x_nchw [B,D,HW] -> xhat_nd [N,D] = x / max(||x||_2, 1e-12) over D; inv_norm [N] = 1/max(..).
 * xhat_nchw (optional, may be NULL) receives the same values in [B,D,HW] (push_forward's
 * first return value). */
int mgp_normalize_fwd(const float* x_nchw, float* xhat_nd, float* inv_norm, float* xhat_nchw,
                      int B, int D, int HW, void* stream);
/* The same pass, also writing the patch-side operands of the tensor-core log-likelihood kernels into `ws` (a workspace
 * of mgp_logprob_ws_bytes(B, HW, P, D, MGP_MATH_TC) bytes that the following mgp_logprob_fwd call receives with
 * MGP_MATH_X_STAGED[_ISO] OR-ed onto its math mode): one read of the features instead of two, one launch less.
 * stage_aniso = 0 skips the x^2 half (only needed when some sigma varies over d). */
int mgp_normalize_fwd_stage(const float* x_nchw, float* xhat_nd, float* inv_norm, float* xhat_nchw,
                            void* ws, size_t ws_bytes, int B, int D, int HW, int P, int stage_aniso,
                            void* stream);

/* Backward of the above: g_xhat_nd [N,D] -> g_x_nchw [B,D,HW]
 *   g_x = (g - xhat * <xhat, g>) * inv_norm. */
int mgp_normalize_bwd(const float* g_xhat_nd, const float* xhat_nd, const float* inv_norm,
                      float* g_x_nchw, int B, int D, int HW, void* stream);

/* Both of the above for features x in any MGP_X_* format (ref: model.py:210-211, :431-432 under torch.autocast,
 * where F.normalize of bf16 / fp16 add-on features yields fp32).  x_fmt = MGP_X_F32 is exactly mgp_normalize_fwd
 * (ws == NULL) or mgp_normalize_fwd_stage (ws != NULL; P and stage_aniso are read only then).  16-bit values are
 * widened on load; every output is fp32 and bit-identical to the MGP_X_F32 pass on the features converted to fp32
 * NCHW.  An unknown x_fmt returns MGP_ERR_INVALID. */
int mgp_normalize_fwd_x(const void* x, int x_fmt, float* xhat_nd, float* inv_norm, float* xhat_nchw,
                        void* ws, size_t ws_bytes, int B, int D, int HW, int P, int stage_aniso,
                        void* stream);
/* mgp_normalize_bwd writing g_x in x_fmt's type and layout (the gradient autograd hands back to the add-on
 * convolutions): the fp32 value of mgp_normalize_bwd, rounded to nearest-even for bf16 / fp16. */
int mgp_normalize_bwd_x(const float* g_xhat_nd, const float* xhat_nd, const float* inv_norm, void* g_x,
                        int x_fmt, int B, int D, int HW, void* stream);

/* ---- a2/a3/a16  diagonal-Gaussian log-likelihood -----------------------------------------
 * ref: model.py:256-275 (compute_log_prob, eps = 0), :323-336 (_estimate_log_prob,
 * eps = 1e-10, log(sigma+eps)), :429-438 (push_forward).
 *   log p[n,p] = -D/2 log 2pi - sum_d log(sigma+eps_log) - 1/2 sum_d ((x-mu)/(sigma+eps))^2
 * `eps` is added to sigma inside the quotient; `eps_log` inside the logarithm
 * (compute_log_prob: 0 / 0, _estimate_log_prob: 1e-10 / 1e-10).
 * xhat_nd [N,D] (N = B*HW; for MGP_OUT_LOGP_NP pass B = N, HW = 1 if there is no image
 * structure), mu/sigma [P,D]; `ws` is scratch of at least mgp_logprob_ws_bytes(B, HW, P, D, math)
 * bytes (the tensor-core path stages fp16 hi/lo operands there). */
size_t mgp_logprob_ws_bytes(int B, int HW, int P, int D, int math);
/* 1 if mgp_logprob_fwd with this layout / shape / math mode reads the fp32 patches itself (the register-resident
 * kernel, csrc/logprob_tcz.cu), so that its workspace holds prototype-side operands only: a caller whose mu / sigma
 * are unchanged since the previous call with the same workspace may then pass MGP_MATH_TC_ISO_REUSE and skip the
 * prototype pre-pass (with the other tensor-core kernels _ISO_REUSE rebuilds the patch side, *_TC_REUSE reuses it). */
int mgp_logprob_ws_is_prototype_only(int out_layout, int P, int D, int math);
int mgp_logprob_fwd(const float* xhat_nd, const float* mu, const float* sigma, float eps,
                    float eps_log, float* out, int out_layout, int B, int HW, int P, int D,
                    int math, void* ws, size_t ws_bytes, void* stream);

/* ---- a14 over feature maps: per-patch class log-densities -----------------------------------
 * ref: model.py:403-421 (_score, as_average=False), :323-336 (_estimate_log_prob, eps = 1e-10 in
 * (sigma+eps) and log(sigma+eps)), train_and_test.py:199 (sum_c p(x|c)).  For every patch n = b*HW + hw of
 * xhat_nd [N,D] (normalised rows, ref model.py:210-211) and every class c:
 *   out_bchw[(b*C + c)*HW + hw] = logsumexp_k( log p_ck(x_n) + log(pi_ck + 1e-10) )   ([B,C,HW], fp32)
 *   out_bhw[b*HW + hw]          = logsumexp_c out_bchw[...]                           ([B,HW]; may be NULL)
 * mu/sigma [P,D] (P = C*K, class-major), weight_cp = last_layer.weight [C,P]: pi_ck = weight_cp[c, c*K + k].
 * MGP_MATH_TC_ISO (the caller asserts sigma constant over d inside every prototype), D in {64, 128}, K <= 64:
 * one tensor-core kernel, the [N,P] log-likelihood never reaches HBM; MGP_MATH_TC_ISO_REUSE: the same with the
 * prototype-side operands of `ws` kept from the previous call with unchanged mu / sigma.  A false assertion yields
 * NaN outputs.  Every other math mode and shape: mgp_logprob_fwd into row chunks of `ws`, then a log-sum-exp
 * kernel.  No limit on HW; N < 2^31.  ws: mgp_log_density_ws_bytes(B, HW, C, K, D, math) bytes. */
size_t mgp_log_density_ws_bytes(int B, int HW, int C, int K, int D, int math);
int mgp_log_density(const float* xhat_nd, const float* mu, const float* sigma, const float* weight_cp,
                    float* out_bchw, float* out_bhw, int B, int HW, int C, int K, int D, int math,
                    void* ws, size_t ws_bytes, void* stream);

/* ---- a4-a7  top-T mining + mixture logits ------------------------------------------------
 * ref: model.py:188-206 (global_max_pooling_gmm_topT), :214-222, :254, NonNegLinear :54-74.
 * logp_bphw [B,P,HW] (MGP_OUT_LOGP_BPHW).  Per (b,p): the T largest over HW, descending
 * (ties: smaller index first) -> vals [B,P,T] = exp(log p) (BEFORE the wrong-class rule),
 * idx [B,P,T] int32.  Then logits[b,c,t] = log sum_k W[c, c*K+k] * v'[b,c*K+k,t] with
 * v'[.,t] = v[.,0] for prototypes of classes != gt[b] and t >= 1 (gt may be NULL: no rule).
 * weight_cp is last_layer.weight [C, P]; only its class-diagonal blocks are read. */
int mgp_head_select(const float* logp_bphw, const float* weight_cp, const int64_t* gt,
                    float* logits, float* vals, int32_t* idx, int B, int HW, int C, int K,
                    int T, void* stream);
/* Same, reading the [N,P] layout (MGP_OUT_LOGP_NP, N = B*HW) that compute_log_prob and the
 * tensor-core kernel produce at full speed: the block of an image and a group of classes is
 * staged through shared memory. */
int mgp_head_select_np(const float* logp_np, const float* weight_cp, const int64_t* gt,
                       float* logits, float* vals, int32_t* idx, int B, int HW, int C, int K,
                       int T, void* stream);

/* Labelled (training) variant that never materialises log p.  With labels the reference overwrites
 * levels t >= 1 of every wrong-class prototype with level 0 (model.py:218-221), so only
 * max/arg-max over the patches is needed for the C-1 other classes: `best` [B,P] uint64 is the
 * MGP_OUT_TOP1_BP output of mgp_logprob_fwd.  The K prototypes of each image's own class get the
 * full top-T from an exact fp32 evaluation of their K x HW log-likelihoods inside this call
 * (xhat_nd [N,D], mu/sigma [P,D], eps = eps_log = 0 as in compute_log_prob).
 * Outputs as mgp_head_select; of vals/idx [B,P,T] only level 0 (all prototypes) and levels
 * 0..T-1 of the own-class prototypes are written -- exactly the entries the logits, the enqueue
 * and mgp_head_bwd read when labels are given.  gt must not be NULL; gt[b] outside [0,C) makes
 * every class of image b a wrong class. */
int mgp_head_select_top1(const uint64_t* best, const float* xhat_nd, const float* mu,
                         const float* sigma, const float* weight_cp, const int64_t* gt,
                         float* logits, float* vals, int32_t* idx, int B, int HW, int C, int K,
                         int D, int T, void* stream);

/* Backward of mgp_head_select composed with the log-likelihood and the normalisation:
 * grad_logits [B,C,T] -> g_x_nchw [B,D,HW] (gradient w.r.t. the un-normalised features;
 * mu, sigma receive none: they are detached at ref model.py:264-265).  Autograd of the
 * reference saves N*P*D*4 bytes for this (51 GB at B=256); here only vals/idx/logits are
 * kept and the T selected patches per (b,p) are re-differentiated.
 * ws: scratch of mgp_head_bwd_ws_bytes(B, HW, P, D) bytes. */
size_t mgp_head_bwd_ws_bytes(int B, int HW, int P, int D);
int mgp_head_bwd(const float* grad_logits, const float* logits, const float* vals,
                 const int32_t* idx, const float* weight_cp, const int64_t* gt,
                 const float* xhat_nd, const float* inv_norm, const float* mu,
                 const float* sigma, void* ws, size_t ws_bytes, float* g_x_nchw, int B, int HW,
                 int C, int K, int D, int T, void* stream);
/* The same with g_x in the MGP_X_* format x_fmt of the features (ref: model.py:210-222 backward under
 * torch.autocast): the normalisation backward writes the gradient in x's type and layout (see mgp_normalize_bwd_x). */
int mgp_head_bwd_x(const float* grad_logits, const float* logits, const float* vals,
                   const int32_t* idx, const float* weight_cp, const int64_t* gt,
                   const float* xhat_nd, const float* inv_norm, const float* mu,
                   const float* sigma, void* ws, size_t ws_bytes, void* g_x, int x_fmt, int B,
                   int HW, int C, int K, int D, int T, void* stream);

/* ---- long feature maps: the head at 1 <= HW <= 4096 -----------------------------------------
 * ref: model.py:188-206 (global_max_pooling_gmm_topT: torch.topk over h*w of any size), :214-222, :254.
 * The entry points above refuse HW > 1024 (10-bit patch keys, [HW]-sized shared-memory tiles); these take any
 * HW <= 4096 (2048-px inputs at stride 32, 1024-px inputs with the x2 add-on upsample, model.py:138), with
 * T <= min(32, HW) and K <= 64, and compute the same outputs.  HW > 4096 returns MGP_ERR_UNSUPPORTED before any
 * launch.  Shared memory per block does not depend on HW.
 * mgp_head_select_long: as mgp_head_select (logp_bphw [B,P,HW]; gt may be NULL). */
int mgp_head_select_long(const float* logp_bphw, const float* weight_cp, const int64_t* gt,
                         float* logits, float* vals, int32_t* idx, int B, int HW, int C, int K,
                         int T, void* stream);
/* As mgp_head_select_top1 (ref model.py:218-221): `best` [B,P] from mgp_logprob_fwd(MGP_OUT_TOP1_BP), the own
 * class's exact fp32 log p evaluated in patch slices; gt = -1 for every image gives the level-0 head. */
int mgp_head_select_top1_long(const uint64_t* best, const float* xhat_nd, const float* mu,
                              const float* sigma, const float* weight_cp, const int64_t* gt,
                              float* logits, float* vals, int32_t* idx, int B, int HW, int C,
                              int K, int D, int T, void* stream);
/* As mgp_head_bwd_x (ref model.py:210-222 backward), for the outputs of the two calls above; deterministic and
 * atomics-free like it.  Also needs P = C*K < 2^20.  ws: mgp_head_bwd_long_ws_bytes(B, HW, P, D) bytes. */
size_t mgp_head_bwd_long_ws_bytes(int B, int HW, int P, int D);
int mgp_head_bwd_long_x(const float* grad_logits, const float* logits, const float* vals,
                        const int32_t* idx, const float* weight_cp, const int64_t* gt,
                        const float* xhat_nd, const float* inv_norm, const float* mu,
                        const float* sigma, void* ws, size_t ws_bytes, void* g_x, int x_fmt,
                        int B, int HW, int C, int K, int D, int T, void* stream);

/* ref: model.py:188-206 (global_max_pooling_gmm_topT) as a stand-alone call on PROBABILITIES sims [B,P,HW]:
 * vals [B,P,T] = the T largest over HW, descending; idx [B,P,T] their patch indices; feats [B,P,D,T] (optional, NULL
 * to skip; 4*B*P*D*T bytes) = x_nchw[b, :, idx[b,p,t]] -- the reference's max_feat, [B,C,K,D,T] once viewed. */
int mgp_topt_pool(const float* sims_bphw, const float* x_nchw, float* vals, int32_t* idx, float* feats,
                  int B, int HW, int C, int K, int D, int T, void* stream);

/* ---- f2  OoD / accuracy statistics of the test loop (ref train_and_test.py:184-199, :212-213) ---------------------
 * out0: level-0 log evidences, element (b, c) at out0[b*stride_b + c*stride_c] (the [B,C,T] logits with stride_c = T,
 * or a dense [B,C]).  p_sum[b] = sum_c exp(out0), p_mean[b] = p_sum / C, pred[b] = argmax_c (int64). */
int mgp_ood_score(const float* out0, int stride_b, int stride_c, float* p_sum, float* p_mean,
                  int64_t* pred, int B, int C, void* stream);

/* ---- a8/a9  enqueue into the per-class FIFO bank -----------------------------------------
 * ref: model.py:225-250, utils/memory.py:31-73.
 *
 * mgp_mined_gather: for every image, the top-1 patch (level 0 of idx [B,P,T]) of each of its
 * GT class's K prototypes: top1 [B,K] int32 spatial index, rows [B,K,D] feature rows.  (These
 * two small tensors are what a batch-sharded multi-GPU run all-gathers before the enqueue.)
 *
 * mgp_bank_enqueue: per image, the rows at the unique (ascending) spatial indices are appended
 * to the image's class FIFO (classes independent; within a class: image order, then ascending
 * index -- the reference's order).  The bank is a ring: bank [C,cap,D], logical row r of class c
 * lives at slot (head[c] + r) % cap, r < mem_len[c] (oldest first).  A single push larger than
 * cap keeps its first cap rows (the reference draws an unseeded random subset there).
 * updated[c] (uint8) is set for every class that received rows (ref model.py:250).
 * plan: int32 scratch of mgp_bank_enqueue_plan_ints(B, C, K) elements.  gt outside [0,C) skips the image. */
/* rows_stride / top1_stride / gt_stride: elements (fp32 / int32 / int64) between consecutive IMAGES of rows / top1 / gt;
 * 0 = dense (K*D / K / 1).  A batch-sharded run lets mgp_mined_gather write straight into packed per-image records
 * [rows K*D | top1 K | gt] that one all-gather exchanges, and mgp_bank_enqueue read the gathered records in place. */
int mgp_mined_gather(const float* xhat_nd, const int32_t* idx, const int64_t* gt, int32_t* top1,
                     float* rows, int rows_stride, int top1_stride, int B, int HW, int C, int K, int D,
                     int T, void* stream);
/* shadow_h / shadow_l [C,cap,D] fp16 and shadow_xx [C,cap] fp32 (all three or none): the tensor-core operand copy of
 * the bank -- hi / lo halves of 256 * row and |row|^2 -- kept in step by the scatter (see mgp_update_gmm). */
size_t mgp_bank_enqueue_plan_ints(int B, int C, int K);
int mgp_bank_enqueue(float* bank, int64_t* mem_len, int32_t* head, uint8_t* updated,
                     const float* rows, const int32_t* top1, const int64_t* gt, int rows_stride,
                     int top1_stride, int gt_stride, int32_t* plan,
                     void* shadow_h, void* shadow_l, float* shadow_xx,
                     int B, int C, int K, int D, int cap, void* stream);
/* (Re)builds the whole shadow from the fp32 bank: after the bank was written by anything but mgp_bank_enqueue
 * (checkpoint load, MemoryBank.push, direct tensor writes). */
int mgp_bank_shadow_sync(const float* bank, void* shadow_h, void* shadow_l, float* shadow_xx, int C, int cap, int D,
                         void* stream);

/* Copies the ring of every class into oldest->newest order: lin [C,cap,D] (rows >= mem_len
 * zero).  This is the layout of the reference's queue.cls%d buffers (state_dict wire format). */
int mgp_bank_linearize(const float* bank, const int64_t* mem_len, const int32_t* head,
                       float* lin, int C, int cap, int D, void* stream);

/* ---- a10-a12  memory-bank EM ---------------------------------------------------------------
 * ref: model.py:277-301 (update_GMM), :303-321 (_e_step), :367-401 (_m_step_diversified).
 *
 * mgp_em_plan: active[c] = updated[c] && mem_len[c] >= cap (ref :283,:289); order[c] = rank of
 * c among the active classes (ascending id) or -1; sched[0] = number of active classes,
 * sched[1] = Adam step count before this update (adam_step[0] if a device counter is given,
 * which is then advanced by num_em_loop * n_active; else the host value step0); updated[]
 * is cleared (ref :287,:301).  No host sync.
 *
 * mgp_em_stats: E-step + sufficient statistics of the smoothed responsibilities over bank
 * slots [row_begin, row_end) of every active class (a row shard; 0, cap = all):
 *   r_nk = (softmax_k(lp_nk + log(pi_k + 1e-10)) + alpha) / sum_k(.)
 *   stats[c][split] = { S0[K], S1[K][D], S2[K][D] (if with_s2), loglik }   (partial sums)
 * stats layout [C][n_split][stat_stride], stat_stride = mgp_em_stat_stride(K, D, with_s2);
 * partials are combined in split order by mgp_em_update (deterministic; a multi-GPU caller
 * all-reduces the whole buffer first).  pi is read from weight_cp's class-diagonal blocks.
 *
 * mgp_em_update: the diversified M-step with the reference's sequential semantics in one
 * launch for all classes.  The reference takes one Adam step on the WHOLE mu tensor per
 * (active class, EM loop) with a gradient that is zero outside that class, so per class the
 * timeline is: num_em_loop*order[c] zero-gradient steps (phase 0; inactive classes take all
 * their zero-gradient steps here), the EM-loop steps (phase 1, em_loop = 0..num_em_loop-1,
 * each after a fresh mgp_em_stats): gradient -(S1 - mu S0) w / n + lamda * diversity gradient,
 * Adam step, pi <- tau*pi + (1-tau)*(S0+1e-10)/n written into weight_cp; then the trailing
 * zero-gradient steps (phase 2).  Adam arithmetic is torch.optim.Adam's (no weight decay, no
 * amsgrad); exp_avg / exp_avg_sq [C,K,D].  With exp_avg == NULL no optimiser step is taken
 * (phase 1 then only writes grad_out [C,K,D] and pi: for a caller-owned optimiser);
 * only_class >= 0 restricts phase 1 to that class. */
size_t mgp_em_stat_stride(int K, int D, int with_s2);
int mgp_em_plan(uint8_t* updated, const int64_t* mem_len, int32_t* order, int32_t* sched,
                int32_t* adam_step, int step0, int C, int cap, int num_em_loop, void* stream);
int mgp_em_stats(const float* bank, const int32_t* order, const float* mu, const float* sigma,
                 const float* weight_cp, float alpha, int row_begin, int row_end, int n_split,
                 int with_s2, float* stats, int C, int K, int D, int cap, void* stream);
/* lr, beta1, beta2, adam_eps and tau are DOUBLES: torch.optim.Adam and momentum_update (model.py:44-50) hold them as
 * Python floats and form 1 - beta / 1 - tau in double before narrowing to fp32; a float parameter would bake
 * 1.0f - 0.999f (1.3e-5 off) into exp_avg_sq. */
int mgp_em_update(const float* stats, int n_split, int with_s2, int n_rows_total,
                  const int32_t* order, const int32_t* sched, float* mu, const float* sigma,
                  float* weight_cp, float* exp_avg, float* exp_avg_sq, int em_loop,
                  int num_em_loop, int phase, double lr, double beta1, double beta2, double adam_eps,
                  double tau, float lamda, float* grad_out, int only_class, int C, int K, int D,
                  void* stream);

/* The whole update_GMM (ref model.py:277-301) of a single-GPU replica in one call: mgp_em_plan (with the
 * device-resident Adam step counter adam_step[0]), phase 0, num_em_loop x (mgp_em_stats over all cap rows,
 * phase 1), phase 2 -- 3 + 2*num_em_loop launches enqueued on `stream`, nothing read back.  order [C] int32,
 * sched [2] int32 and stats [C][n_split][mgp_em_stat_stride(K,D,0)] fp32 are scratch.  (A batch-sharded
 * multi-GPU caller uses the individual entry points, with an all-reduce of stats between the two.) */
/* With the bank's shadow (shadow_h / shadow_l / shadow_xx, see mgp_bank_enqueue; may be NULL) and sigma_iso != 0 --
 * the caller's assertion that sigma is constant over d inside every prototype, which holds for every state the
 * reference's training loop reaches -- shapes K <= 16, D in {128, 256} run as ONE tensor-core launch after the planner
 * (csrc/em_tc.cu: both inner products as wgmma GEMMs on fp16 hi/lo splits).  The kernel re-checks sigma and sets
 * status[0] = 1 (leaving that class untouched) if the assertion was wrong.  Otherwise: K <= 16, D in {64, 128}: one
 * fp32 cluster launch; any other shape: the launches listed above. */
/* number of kernel launches mgp_update_gmm enqueues for this shape (2 = planner + single launch) */
int mgp_update_gmm_launches(int K, int D, int cap, int num_em_loop, int have_shadow_iso);
int mgp_update_gmm(const float* bank, const void* shadow_h, const void* shadow_l, const float* shadow_xx,
                   int sigma_iso, int32_t* status, uint8_t* updated, const int64_t* mem_len, float* mu,
                   const float* sigma, float* weight_cp, float* exp_avg, float* exp_avg_sq,
                   int32_t* adam_step, int32_t* order, int32_t* sched, float* stats, int n_split,
                   int num_em_loop, float alpha, double lr, double beta1, double beta2, double adam_eps,
                   double tau, float lamda, int C, int K, int D, int cap, void* stream);
/* The tensor-core update_GMM of mgp_update_gmm (planner + one kernel) with STAGED outputs: mu and weight_cp are only
 * read; the new means go to mu_stage [C,K,D] and the new class-diagonal pi to pi_stage [C,K] (pi_stage[c*K+k] is the
 * value for weight_cp[c][c*K+k]), for every class.  exp_avg / exp_avg_sq are updated in place as in mgp_update_gmm.
 * A caller can therefore run it on a second stream while other work still reads mu and pi, and then apply it with
 * mgp_em_commit on the stream that owns them.  Only the tensor-core path is staged: the same preconditions (shadow,
 * status, sigma isotropic -- asserted by calling this -- and a supported shape), else MGP_ERR_UNSUPPORTED with nothing
 * enqueued.  The staging buffers must not alias mu / weight_cp. */
int mgp_update_gmm_staged(const void* shadow_h, const void* shadow_l, const float* shadow_xx, int32_t* status,
                          uint8_t* updated, const int64_t* mem_len, const float* mu, const float* sigma,
                          const float* weight_cp, float* exp_avg, float* exp_avg_sq, int32_t* adam_step,
                          int32_t* order, int32_t* sched, float* stats, int n_split, int num_em_loop, float alpha,
                          double lr, double beta1, double beta2, double adam_eps, double tau, float lamda,
                          float* mu_stage, float* pi_stage, int C, int K, int D, int cap, void* stream);
/* mu [C,K,D] <- mu_stage, weight_cp[c][c*K+k] <- pi_stage[c*K+k]: applies mgp_update_gmm_staged's result (one launch).
 * D % 4 == 0, mu and mu_stage 16-byte aligned. */
int mgp_em_commit(const float* mu_stage, const float* pi_stage, float* mu, float* weight_cp, int C, int K, int D,
                  void* stream);

/* ---- a11/a13/a14  EM building blocks on explicit rows ---------------------------------------
 * ref: model.py:303-321 (_e_step), :338-365 (_m_step), :403-421 (_score).
 * x [n,D], mu/sigma [K,D], pi [K]  ->  log_resp [n,K], score [n] = logsumexp_k(lp+log(pi+1e-10)).
 * Either output may be NULL. */
int mgp_em_estep(const float* x, const float* mu, const float* sigma, const float* pi,
                 float* log_resp, float* score, int n, int K, int D, void* stream);
/* closed-form M-step from log_resp (the only sigma update in the reference):
 * pi_out [K], mu_out [K,D], sigma_out [K,D]. */
int mgp_em_mstep_closed(const float* x, const float* log_resp, float alpha, float* pi_out,
                        float* mu_out, float* sigma_out, int n, int K, int D, void* stream);
/* ref: model.py:367-401 (_m_step_diversified) on explicit rows: pi_out [K] = (sum_n r + 1e-10) / n and
 * grad_out [K,D] = d gmm_loss / d mu (weighted log-likelihood term + lamda * diversity term), r the smoothed
 * responsibilities of log_resp; ws_nk [n*K] fp32 scratch.  The caller feeds grad_out to the optimiser step. */
int mgp_em_mstep_div(const float* x, const float* log_resp, const float* mu, const float* sigma,
                     float alpha, float lamda, float* ws_nk, float* pi_out, float* grad_out, int n,
                     int K, int D, void* stream);

/* ---- a17  training loss on the head output (optional fused helper) ------------------------------
 * ref: train_and_test.py:37-41, :55.  out [B,C,T] log evidences, gt [B] ->
 *   loss_b [B] per-image shares of  CE(level 0) + mine_coef * mean_{t>=1} CE(level t)  (sum = the loss),
 *   grad [B,C,T] = d loss / d out.  gt must lie in [0, C). */
int mgp_mine_ce(const float* out, const int64_t* gt, float* loss_b, float* grad, int B, int C, int T,
                float mine_coef, void* stream);

/* ---- a17b  auxiliary loss on the embedding: the Proxy-Anchor criterion ---------------------------
 * ref: utils/losses.py:19-61 (l2_norm, Proxy_Anchor.forward), called at train_and_test.py:42; it replaces the host
 * one-hot encoding (:9-16), the host read of the number of positive proxies (:51-52) and autograd's backward.
 * x [B,E] embeddings of element type x_dtype (MGP_X_F32 / _BF16 / _F16, no layout flag), proxies [C,E] fp32,
 * labels [B] int64.  With xh_b = x_b / sqrt(|x_b|^2 + 1e-12), ph_c likewise and s_bc = xh_b . ph_c:
 *   loss [1] = (1/|C+|) sum_c log(1 + sum_{b: t_b = c} exp(-beta (s_bc - margin)))
 *            + (1/C)    sum_c log(1 + sum_{b: t_b != c} exp(beta (s_bc + margin))),   C+ = classes present in the batch;
 *   grad_x [B,E] = d loss / d x in x's element type (round to nearest even), grad_p [C,E] = d loss / d proxies, fp32,
 *   both through the normalisations; either may be NULL (then that pass is skipped);
 *   n_valid (int32 [1], may be NULL) = |C+|.
 * Beyond the reference: an image whose label is outside [0, C) contributes to no sum (and gets a zero gradient);
 * |C+| = 0 gives the second term alone; C = 2 is allowed.  One launch of one cluster, no atomics (bit-identical from
 * run to run), nothing read back by the host, safe under stream capture.
 * 1 <= B <= 4096, 2 <= C <= 4096, E % 4 == 0, E <= 512 (MGP_ERR_UNSUPPORTED otherwise); x, proxies, grad_x and
 * grad_p 16-byte aligned. */
int mgp_proxy_anchor(const void* x, int x_dtype, const float* proxies, const int64_t* labels, int B, int C, int E,
                     float margin, float beta, float* loss, void* grad_x, float* grad_p, int32_t* n_valid,
                     void* stream);

/* ---- f1  prototype projection search --------------------------------------------------------
 * ref: push.py:125-158.  For every image and the K prototypes of its label's class: flat HW
 * argmin of -p (= argmax of log p; ties: smaller index) and -p there.
 * logp_bphw [B,P,HW] -> arg [B,K] int32, val [B,K]. */
int mgp_push_argmin(const float* logp_bphw, const int64_t* labels, int32_t* arg, float* val,
                    int B, int HW, int C, int K, void* stream);
/* The same result from best_bp [B,P], the packed per-(image, prototype) max / arg-max of log p that
 * mgp_logprob_fwd(..., MGP_OUT_TOP1_BP) computes in the tensor-core epilogue: the [B,P,HW] map (401 MB per batch of
 * 256 at cfg2; the reference copies it to the host, push.py:109-118) is never formed. */
int mgp_push_argmin_top1(const unsigned long long* best_bp, const int64_t* labels, int32_t* arg,
                         float* val, int B, int C, int K, void* stream);

/* ---- f1  prototype projection: candidate store and greedy assignment ----------------------------
 * ref: push.py:125-200.  Prototype (c,k) picks among images labelled c, after prototypes 0..k-1 of its class, so its
 * pick is among its own k+1 best candidates: a store of the K best candidates per prototype (K <= 64) gives the
 * reference's greedy exactly, in C*K*K*(D+4)*4 bytes whatever the number of images.  Candidates are ordered by
 * (-p ascending, image id ascending); exact ties in -p go to the smaller id.  The store is the set of the K smallest
 * keys merged so far, independent of the order of the merges: image-sharded replicas that merge the same gathered
 * records end with identical stores.
 *
 * Records: one per image, rec_stride fp32 words apart (a multiple of 4, >= K*D + 2K + 2); rec_rows / rec_val /
 * rec_patch / rec_label point at the fields of record 0: rows [K*D] fp32 (16-byte aligned), val [K] fp32 (-p),
 * patch [K] int32, label int64 (8-byte aligned).  A record whose label is outside [0, C) is ignored; a candidate whose
 * patch is < 0 is ignored.
 *
 * mgp_push_records (ref push.py:125-158): per image b, from mgp_push_argmin(_top1)'s arg [B,K] / val [B,K] and the
 * normalised features xhat_nd [B*HW, D], the rows xhat_nd[b*HW + arg[b,k]], the values, the patches and the label
 * (written as -1 outside [0, C); then nothing is read from arg / val / xhat_nd for that image).
 *
 * mgp_push_merge: folds n records into the store, record i being image id0 + i (id0 + n <= 0xffffffff).  Store:
 * key [C,K,K] uint64 = (monotone key of -p) << 32 | id, empty slot = UINT64_MAX (fill it so before the first merge);
 * patch [C,K,K] int32; row [C,K,K,D] fp32 (16-byte aligned).  One image id must not be merged twice.
 *
 * mgp_push_assign (ref push.py:165-200): per class, k = 0..K-1 in order, the smallest key of prototype (c,k) whose id
 * no earlier prototype of the class took: its row is copied into mu [C,K,D] (16-byte aligned), chosen_id /
 * chosen_patch [C*K] int64 and chosen_val [C*K] fp32 (-p) receive the pick.  Without a candidate: id -1, patch -1,
 * val +inf, mu[c,k] untouched. */
int mgp_push_records(const int32_t* arg, const float* val, const float* xhat_nd, const int64_t* labels,
                     float* rec_rows, float* rec_val, int32_t* rec_patch, int64_t* rec_label, int rec_stride,
                     int B, int HW, int C, int K, int D, void* stream);
int mgp_push_merge(const float* rec_rows, const float* rec_val, const int32_t* rec_patch, const int64_t* rec_label,
                   int rec_stride, int n, size_t id0, unsigned long long* key, int32_t* patch, float* row,
                   int C, int K, int D, void* stream);
int mgp_push_assign(const unsigned long long* key, const int32_t* patch, const float* row, float* mu,
                    int64_t* chosen_id, int64_t* chosen_patch, float* chosen_val, int C, int K, int D, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MGPROTO_B200_H_ */
