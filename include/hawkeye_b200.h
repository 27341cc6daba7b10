/* hawkeye_b200 — C ABI of the H100-native high-order-pooling hot path.
 *
 * One shared library (hawkeye_b200/libhawkeye_b200.so), plain C types, no torch types.
 * Conventions:
 *   - return 0 = success; <0 = argument/shape/alignment error, nothing was launched;
 *     >0 = cudaError_t from a launch.  hk_last_error() gives the text (thread-local).
 *   - the caller owns every device buffer including workspaces (query *_workspace_bytes);
 *     the library allocates nothing and never synchronises; all work is enqueued on `stream`
 *     (a cudaStream_t passed as void*).  There is no library-owned device state: every entry point is re-entrant and
 *     may run concurrently with anything else on the GPU (no kernel waits on another thread-block cluster).
 *   - tensors are contiguous fp32; pointers 16-byte aligned; no CPU fallback: an unsupported
 *     shape is an error (-3), never a silent slow path.
 * Each entry point cites the reference interface it replaces (paths relative to the Hawkeye tree).
 */
#ifndef HAWKEYE_B200_H
#define HAWKEYE_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

const char* hk_version(void);
const char* hk_last_error(void);
long long hk_launch_count(void);      /* kernels launched by this library, counted over all host threads */
void hk_reset_launch_count(void);

/* ---- precision mode (process-wide; default 0, or $HK_PRECISE at first use) ---------------------------------------
 * 0: single-pass TF32 tensor-core products (the tf32 tensor-core MMA keeps 10 mantissa bits of each operand); every kernel
 *    that produces an operand of a later MMA rounds it to tf32 on store (round-to-nearest), so outputs of
 *    hk_conv3x3_*, hk_bn_*, hk_bilinear_pool_fwd, hk_cbp_fwd carry a 2^-11 relative quantisation.  Meets the 1e-3
 *    forward tolerance of the path; gradients below ReLU / max-pool kinks then differ from an fp32 run by branch
 *    flips (see tests/matched.py).
 * 1: 3xTF32 — every MMA operand is split into (hi, lo) tf32 halves and  A.B ~= Ah.Bh + Al.Bh + Ah.Bl  is accumulated
 *    by the same GEMM in one launch (all three products per k-step); nothing is rounded on store.  fp32-class results (for parity runs against
 *    the fp32 reference) at more than 3x the cost; this mode allocates stream-ordered scratch (cudaMallocAsync). */
void hk_set_precise(int on);
int hk_get_precise(void);

/* ---- generic batched TF32 tensor-core GEMM (wgmma + TMA) -------------------------------------
 * C[b] = alpha*alpha_vec[b] * A[b].B[b] + diag*I + beta*beta_vec[b] * D[b]   (ReLU optional; C optionally transposed)
 * A logical [M,K]: a_mn_major=0 -> A[m*lda+k]; 1 -> A[k*lda+m].   B logical [K,N]: b_mn_major=0 -> B[n*ldb+k]; 1 -> B[k*ldb+n].
 * Replaces torch.bmm call sites model/methods/MPNCOV.py:117,132,154-160,178-194 and 1x1 convs resnet.py:34-37. */
int hk_gemm_tf32(const float* A, int a_mn_major, long long lda, long long strideA, const float* B, int b_mn_major,
                 long long ldb, long long strideB, float* C, long long ldc, long long strideC, int trans_c, int M,
                 int N, int K, int batch, float alpha, const float* alpha_vec, float diag, const float* D,
                 long long ldd, long long strideD, float beta, const float* beta_vec, int relu, void* stream);

/* same product, always as 3xTF32 whatever the precision mode (results that feed an exponential, e.g. CIN's softmax(-Gram)) */
int hk_gemm_3xtf32(const float* A, int a_mn_major, long long lda, long long strideA, const float* B, int b_mn_major,
                   long long ldb, long long strideB, float* C, long long ldc, long long strideC, int trans_c, int M,
                   int N, int K, int batch, float alpha, const float* alpha_vec, float diag, const float* D,
                   long long ldd, long long strideD, float beta, const float* beta_vec, int relu, void* stream);

/* ---- BCNN bilinear pooling: model/methods/BCNN.py:13-27 (BilinearPooling.forward) ----------------
 * x [B,C,HW] (NCHW feature map viewed as in BCNN.py:17) -> y [B,C*C] = normalize(sqrt(x x^T/HW + 1e-5)).
 * inv_norm_out (optional, [B]) receives 1/||z||.  Requires C%128==0.  H*W need not be a multiple of 4 (7x7 maps of 224x224
 * inputs): the workspace then also holds a zero-padded copy of x (TMA needs a 16-byte row pitch).  H*W <= 58112 (the
 * channel sums of one image are reduced in shared memory): forward and backward reject a larger map with -3. */
size_t hk_bilinear_pool_fwd_workspace_bytes(int B, int C, int HW);
int hk_bilinear_pool_fwd(const float* x, float* y, float* inv_norm_out, int B, int C, int HW, void* workspace,
                         size_t workspace_bytes, void* stream);
/* backward of the same (what autograd derives for BCNN.py:13-27): dx [B,C,HW] from dy [B,C*C]; z is recomputed.
 * Default precision mode: y (forward) and dx (backward) are rounded to tf32 on store — they are operands of the next
 * MMA (classifier / last conv dgrad) — and the forward uses sqrt.approx (2^-22 rel.); hk_set_precise(1): fp32 as computed. */
size_t hk_bilinear_pool_bwd_workspace_bytes(int B, int C, int HW);
int hk_bilinear_pool_bwd(const float* x, const float* dy, float* dx, int B, int C, int HW, void* workspace,
                         size_t workspace_bytes, void* stream);

/* ---- CBCNN compact bilinear pooling: model/methods/CBCNN.py:96-135 (CompactBilinearPooling.forward) ------------
 * h1,h2 int32 [C] and s1,s2 fp32 [C] are the count-sketch hash / sign vectors of CBCNN.py:76-91 (numpy seeds 1/3/5/7,
 * generated bit-exactly on the host).  y [B,d] = normalize(signed_sqrt(tensor-sketch)); pre [B,d] (pre-sqrt sketch)
 * is saved for the backward.  Requires C%128==0; for H*W % 4 != 0 a zero-padded copy of x is made in stream-ordered
 * scratch (cudaMallocAsync) — the one case outside the precise mode where the library allocates. */
int hk_cbp_fwd(const float* x, const int* h1, const int* h2, const float* s1, const float* s2, float* y, float* pre,
               int B, int C, int HW, int d, void* stream);
size_t hk_cbp_bwd_workspace_bytes(int B, int C, int d);
int hk_cbp_bwd(const float* x, const float* pre, const float* dy, const int* h1, const int* h2, const float* s1,
               const float* s2, float* dx, int B, int C, int HW, int d, void* workspace, size_t workspace_bytes,
               void* stream);

/* ---- Fast MPN-COV pooling head: model/methods/MPNCOV.py:105-230 -----------------------------------------------
 * Covpool (:105-134): x [B,C,M] -> cov [B,C,C] = X I_hat X^T; xc [B,C,ceil4(M)] receives the centred features at a 16-byte row
 *   pitch (saved for bwd; equal to [B,C,M] whenever M % 4 == 0).
 * Sqrtm (:137-202): coupled Newton-Schulz, iterN >= 2, forward and the reference's hand-derived backward formulae,
 *   all products as 3xTF32 wgmma GEMMs.  `saved` (hk_sqrtm_saved_floats floats) carries A, Y_i, Z_i, normA.
 * Triuvec (:205-230): row-major upper triangle [B,n,n] <-> [B,n(n+1)/2]. */
int hk_covpool_fwd(const float* x, float* cov, float* xc, int B, int C, int M, void* stream);
int hk_covpool_bwd(const float* xc, const float* g, float* dx, int B, int C, int M, void* stream);
size_t hk_sqrtm_saved_floats(int B, int n, int iterN);
size_t hk_sqrtm_fwd_workspace_bytes(int B, int n);
size_t hk_sqrtm_bwd_workspace_bytes(int B, int n);
int hk_sqrtm_fwd(const float* x, float* y, float* saved, int B, int n, int iterN, void* workspace,
                 size_t workspace_bytes, void* stream);
int hk_sqrtm_bwd(const float* x, const float* y, const float* g, float* saved, float* grad_x, int B, int n, int iterN,
                 void* workspace, size_t workspace_bytes, void* stream);
int hk_triuvec_fwd(const float* x, float* y, int B, int n, void* stream);
int hk_triuvec_bwd(const float* g, float* dx, int B, int n, void* stream);

/* ---- VGG-16 backbone: model/backbone/vgg.py:56-70 (Conv2d 3x3 s1 p1 + bias, ReLU, MaxPool2d(2,2)) ----------
 * Activations are NHWC fp32 inside the backbone.  Weights keep the reference layout [Cout,Cin,3,3] in the
 * state_dict and are re-packed per step: w_fwd [9][Cout][Cin], w_dgrad [9][Cin][Cout] (taps flipped). */
int hk_conv3x3_pack_weights(const float* w, float* w_fwd, float* w_dgrad, int Cout, int Cin, void* stream);
/* y = relu?(conv3x3(x, w) + bias): implicit GEMM on wgmma, TMA zero-fill = padding.  Cin%32==0, Cout%32==0. */
int hk_conv3x3_fwd(const float* x_nhwc, const float* w_fwd_packed, const float* bias, float* y_nhwc, int N, int H,
                   int W, int Cin, int Cout, int relu, void* stream);
/* relu(conv3x3(x, w) + bias) followed by MaxPool2d(2,2) (vgg.py:59-68: every pool of VGG-16 follows a conv + ReLU) in ONE
 * kernel: the epilogue reduces the 2x2 windows across lanes and the full-resolution map is never written.
 * pooled: [N,H/2,W/2,Cout] NHWC, or [N,Cout,H/2,W/2] when out_nchw (the last pool feeds the pooling heads in NCHW);
 * code (optional, training): one byte per pooled element for hk_maxpool2x2_bwd_idx (bits 0-1 first arg-max in scan order,
 * bit 2 = max > 0).  Bit-identical to hk_conv3x3_fwd + hk_maxpool2x2_fwd_idx.  H, W even; single-pass TF32 mode only
 * (HK_ERR_UNSUPPORTED under hk_set_precise(1): the 3xTF32 passes chain through the full-resolution map). */
int hk_conv3x3_fwd_pool(const float* x_nhwc, const float* w_fwd_packed, const float* bias, float* pooled,
                        unsigned char* code, int N, int H, int W, int Cin, int Cout, int out_nchw, void* stream);
/* same with stride 2 (ResNet v1.5 down-sampling 3x3, resnet.py:116): H, W are the input dims, output is H/2 x W/2 */
int hk_conv3x3_s2_fwd(const float* x_nhwc, const float* w_fwd_packed, const float* bias, float* y_nhwc, int N, int H,
                      int W, int Cin, int Cout, int relu, void* stream);
/* dx = conv3x3^T(dy, w) * (relu_mask_act > 0)  (mask optional: the ReLU output that produced x) */
int hk_conv3x3_dgrad(const float* dy_nhwc, const float* w_dgrad_packed, const float* relu_mask_act, float* dx_nhwc,
                     int N, int H, int W, int Cin, int Cout, void* stream);
/* hk_conv3x3_dgrad (no mask) followed by hk_maxpool2x2_bwd_idx in ONE kernel: the data gradient of a conv whose input x
 * [N,H,W,Cin] is the output of a 2x2 max-pool goes straight to the pool's input.  code: the pool's bytes [N,H,W,Cin];
 * dx_full: [N,2H,2W,Cin], each window holding the gradient at its arg-max (zero where bit 2 is clear) and zeros elsewhere.
 * The pooled gradient is never written; dx_full is bit-identical to the two-launch sequence.  H % 8 == 0, W % 8 == 0,
 * Cin % 32 == 0, Cout % 32 == 0, 4*H*W*Cin < 2^31; single-pass TF32 only (HK_ERR_UNSUPPORTED otherwise). */
int hk_conv3x3_dgrad_unpool(const float* dy_nhwc, const float* w_dgrad_packed, const unsigned char* code, float* dx_full,
                            int N, int H, int W, int Cin, int Cout, void* stream);
/* VGG conv1_2's data gradient with conv1_1's weight gradient in its epilogue: dx1 = conv3x3^T(dy, w) * (relu_mask_act > 0)
 * (relu_mask_act optional: conv1_1's output) is never written; dw1 [64,3,3,3] and db1 [64] (optional) of the 3-channel
 * layer are computed from it and the NCHW image x_nchw [N,3,H,W], as hk_conv3x3_first_wgrad_direct_acc would from the
 * stored dx1 (the sums run in another order).  accumulate != 0 adds.  Cin = Cout = 64, W % 16 == 0, H % 8 == 0,
 * single-pass TF32 only (HK_ERR_UNSUPPORTED otherwise).  Deterministic: per-CTA partials in the workspace, reduced in a
 * fixed order. */
size_t hk_conv3x3_dgrad_first_wgrad_workspace_bytes(void);
int hk_conv3x3_dgrad_first_wgrad_acc(const float* dy_nhwc, const float* w_dgrad_packed, const float* relu_mask_act,
                                     const float* x_nchw, float* dw1, float* db1, int N, int H, int W, int Cin, int Cout,
                                     void* workspace, size_t workspace_bytes, int accumulate, void* stream);
/* dw [Cout,Cin,3,3] (reference layout), db [Cout] (optional) from x, dy (dy already ReLU-masked).  Cin%32==0, W%4==0. */
size_t hk_conv3x3_wgrad_workspace_bytes(int Cin, int Cout);
int hk_conv3x3_wgrad(const float* x_nhwc, const float* dy_nhwc, float* dw, float* db, int N, int H, int W, int Cin,
                     int Cout, void* workspace, size_t workspace_bytes, void* stream);
/* accumulate != 0: dw += ..., db += ... (gradient accumulation straight into a parameter's .grad buffer, no temporaries) */
int hk_conv3x3_wgrad_acc(const float* x_nhwc, const float* dy_nhwc, float* dw, float* db, int N, int H, int W, int Cin,
                         int Cout, void* workspace, size_t workspace_bytes, int accumulate, void* stream);
/* first layer (Cin=3, vgg.py:61): NCHW image in, NHWC out, bias+ReLU fused.  The 3x3x3 patches are materialised once
 * as X27 [N*H*W][32] (start of the fwd workspace) and reused by the weight/bias gradient. */
size_t hk_conv3x3_first_fwd_workspace_bytes(int N, int H, int W, int Cout);
int hk_conv3x3_first_fwd(const float* x_nchw, const float* w, const float* bias, float* y_nhwc, int N, int H, int W,
                         int Cout, void* workspace, size_t workspace_bytes, void* stream);
size_t hk_conv3x3_first_wgrad_workspace_bytes(int N, int H, int W, int Cout);
int hk_conv3x3_first_wgrad(const float* x27, const float* dy_nhwc, float* dw, float* db, int N, int H, int W,
                           int Cout, void* workspace, size_t workspace_bytes, void* stream);
int hk_conv3x3_first_wgrad_acc(const float* x27, const float* dy_nhwc, float* dw, float* db, int N, int H, int W,
                               int Cout, void* workspace, size_t workspace_bytes, int accumulate, void* stream);
/* first layer without X27 in memory (Cout = 64, single-pass TF32 only; HK_ERR_UNSUPPORTED in precise mode): each kernel
 * rebuilds the patches of its pixels from the NCHW image.  fwd_direct: y bit-identical to hk_conv3x3_first_fwd.
 * wgrad_direct_acc: dw [64,3,3,3], db [64] (optional) from the image and dy (ReLU-masked); accumulate != 0 adds. */
int hk_conv3x3_first_fwd_direct(const float* x_nchw, const float* w, const float* bias, float* y_nhwc, int N, int H, int W,
                                int Cout, void* stream);
size_t hk_conv3x3_first_wgrad_direct_workspace_bytes(void);
int hk_conv3x3_first_wgrad_direct_acc(const float* x_nchw, const float* dy_nhwc, float* dw, float* db, int N, int H, int W,
                                      int Cout, void* workspace, size_t workspace_bytes, int accumulate, void* stream);
/* MaxPool2d(2,2) on NHWC; out_nchw=1 writes the pooled map as NCHW (input of the pooling heads).
 * bwd routes dy to the first max (PyTorch semantics) and multiplies by (x>0), i.e. also applies the ReLU backward. */
int hk_maxpool2x2_fwd(const float* x_nhwc, float* y, int N, int H, int W, int C, int out_nchw, void* stream);
int hk_maxpool2x2_bwd(const float* x_nhwc, const float* dy, float* dx_nhwc, int N, int H, int W, int C, int dy_nchw,
                      void* stream);
/* training variants: fwd also records one byte per pooled element (bits 0-1 arg-max window position, bit 2 = max > 0);
 * bwd routes dy from that byte alone instead of re-reading the four pre-pool activations */
int hk_maxpool2x2_fwd_idx(const float* x_nhwc, float* y, unsigned char* code, int N, int H, int W, int C, int out_nchw,
                          void* stream);
int hk_maxpool2x2_bwd_idx(const unsigned char* code, const float* dy, float* dx_nhwc, int N, int H, int W, int C,
                          int dy_nchw, void* stream);

/* ---- ResNet-50 v1.5 trunk support (model/backbone/resnet.py:89-252); activations NHWC [P = N*H*W, C] -----------------
 * stem 7x7/s2/p3 (resnet.py:176): patches X147 [P][160] (+ packed weights [64][160]) feed one wgmma GEMM. */
int hk_stem_im2col(const float* x_nchw, float* x147, int N, int H, int W, void* stream);
int hk_pack_stem_weights(const float* w, float* w147, int Cout, void* stream);
/* nn.BatchNorm2d in train mode (batch statistics, running stats updated with momentum, eps inside the sqrt):
 * y = [relu]((x-mean)*invstd*gamma + beta [+ residual]);  backward returns dx, dgamma, dbeta and (optionally) the
 * ReLU-masked dy for the residual branch (resnet.py:141-142 `out += identity; relu`). */
size_t hk_bn_workspace_bytes(long long P, int C);
int hk_bn_fwd(const float* x, const float* gamma, const float* beta, const float* residual, float* y, float* save_mean,
              float* save_invstd, float* running_mean, float* running_var, float momentum, float eps, long long P, int C,
              int relu, void* workspace, size_t workspace_bytes, void* stream);
int hk_bn_apply(const float* x, const float* mean, const float* invstd, const float* gamma, const float* beta,
                const float* residual, float* y, long long P, int C, int relu, void* stream);
int hk_bn_bwd(const float* x, const float* y, const float* dy, const float* gamma, const float* save_mean,
              const float* save_invstd, float* dx, float* dres, float* dgamma, float* dbeta, long long P, int C, int relu,
              void* workspace, size_t workspace_bytes, void* stream);
/* hk_bn_bwd with the ReLU mask recomputed instead of read: when the forward was relu((x-mean)*invstd*gamma + beta) WITHOUT a
 * residual, pass that beta as beta_for_mask and the backward re-evaluates the forward's own expression on x (same operation
 * order, so the same mask) — y is not read (may be null): a third less HBM traffic in both backward passes.
 * beta_for_mask == null: identical to hk_bn_bwd (mask = y > 0). */
int hk_bn_bwd_ex(const float* x, const float* y, const float* dy, const float* gamma, const float* beta_for_mask,
                 const float* save_mean, const float* save_invstd, float* dx, float* dres, float* dgamma, float* dbeta,
                 long long P, int C, int relu, void* workspace, size_t workspace_bytes, void* stream);
/* hk_bn_bwd_ex for BatchNorm on frozen (running) statistics, i.e. backward through an eval-mode BatchNorm: mean / invstd are
 * the constants the forward used (running_mean, 1/sqrt(running_var + eps)); dx = dy'*gamma*invstd, dgamma = sum dy'*xhat,
 * dbeta = sum dy' (dy' = dy under the ReLU mask), with the same fixed-order workspace reduction.  The running statistics are
 * not arguments: nothing here touches them. */
int hk_bn_bwd_frozen(const float* x, const float* y, const float* dy, const float* gamma, const float* beta_for_mask,
                     const float* mean, const float* invstd, float* dx, float* dres, float* dgamma, float* dbeta, long long P,
                     int C, int relu, void* workspace, size_t workspace_bytes, void* stream);
/* nn.MaxPool2d(3, 2, 1) (resnet.py:180) */
/* argmax (optional, [N,Ho,Wo,C] bytes): window position of the first maximum, consumed by the backward */
int hk_maxpool3x3s2_fwd(const float* x, float* y, unsigned char* argmax, int N, int H, int W, int C, void* stream);
int hk_maxpool3x3s2_bwd(const unsigned char* argmax, const float* dy, float* dx, int N, int H, int W, int C,
                        void* stream);
/* stride-2 sampling of an NHWC map (1x1/s2 down-sample convs) and its adjoint (zero insertion); H, W = full-res dims */
int hk_subsample2(const float* x, float* y, int N, int H, int W, int C, void* stream);
int hk_upsample2_zero(const float* y, float* x, int N, int H, int W, int C, void* stream);
/* layers the methods share: a += b; NCHW <-> NHWC; ReLU (elu = 0) or ELU with alpha 1 (elu = 1) of n > 0 elements, whose
 * backward reads the output y */
int hk_add_inplace(float* a, const float* b, size_t n, void* stream);
int hk_nhwc_to_nchw(const float* x, float* y, int N, int HW, int C, void* stream);
int hk_nchw_to_nhwc(const float* x, float* y, int N, int HW, int C, void* stream);
int hk_act_fwd(const float* x, float* y, size_t n, int elu, void* stream);
int hk_act_bwd(const float* y, const float* dy, float* dx, size_t n, int elu, void* stream);
/* weight gradient of a matrix-form conv (1x1, or im2col'd stem): dw [Cout][K] = dY[P][Cout]^T . X[P][K] */
size_t hk_matconv_wgrad_workspace_bytes(long long P, int K, int Cout);
int hk_matconv_wgrad(const float* x, const float* dy, float* dw, long long P, int K, int Cout, void* workspace,
                     size_t workspace_bytes, void* stream);

/* ---- channel interaction: model/methods/CIN.py:24-60, ChannelInteractionModule ---------------------
 * The Gram (:31), W.X (:34,:55), the 3x3 conv (:36,:57) and fc (:47-48) use hk_gemm_tf32 / hk_conv3x3_* / hk_linear_*; these are
 * the pieces in between: W_SCI = softmax(-G) row-wise (:32) and its backward; W_CCI = |W_SCI - weight_b * W_SCI[(b+B/2)%B]|
 * (:50-53; `per` = C*C elements per sample, B even) and its backward (d_sci, d_weight [B]); AdaptiveAvgPool1d(1) (:71) as a
 * row mean over the first `cols` of `ld` entries. */
int hk_softmax_neg_rows_fwd(const float* g, float* w, long long rows, int cols, void* stream);
int hk_softmax_neg_rows_bwd(const float* w, const float* dw, float* dg, long long rows, int cols, void* stream);
int hk_cci_weight_fwd(const float* w_sci, const float* weight, float* w_cci, int B, long long per, void* stream);
int hk_cci_weight_bwd(const float* w_sci, const float* weight, const float* d_cci, float* d_sci, float* d_weight, int B,
                      long long per, void* stream);
int hk_row_mean_fwd(const float* x, float* y, long long rows, int cols, int ld, void* stream);
int hk_row_mean_bwd(const float* dy, float* dx, long long rows, int cols, int ld, void* stream);
/* ---- CIN's contrastive loss: model/loss/CIN_loss.py:26-46 ----------------------------------------------------------------
 * hk_cin_pair_diff_fwd: d [B/2, per] = z[:B/2] - z[B/2:] of z [B, per] (the bias of h cancels in h(a) - h(b), so the projection
 * runs once, on the difference, through hk_linear_*); hk_cin_pair_diff_bwd: dz = [dd; -dd].
 * hk_cin_contrastive_loss: p [B/2, R] projected differences, labels [B] int64 -> loss[0] = alpha (L1 + L1^2) with
 * L1 = sum_{i : labels[i] == labels[B/2]} ||p_i + 1e-6||^2, and dp [B/2, R] = alpha (1 + 2 L1) 2 (p_i + 1e-6) on those rows, 0 on
 * the others.  One launch, no read-back.  B even. */
int hk_cin_pair_diff_fwd(const float* z, float* d, int B, long long per, void* stream);
int hk_cin_pair_diff_bwd(const float* dd, float* dz, int B, long long per, void* stream);
int hk_cin_contrastive_loss(const float* p, const long long* labels, float* loss, float* dp, int B, int R, float alpha,
                            void* stream);

/* ---- OSME excitation: s = sigmoid(m)[n,c] * x[n,c,:] and its backward; the
 * squeeze (AdaptiveAvgPool2d) is hk_row_mean_*, the two Linear layers are hk_linear_*, ReLU on the bottleneck hk_act_* */
int hk_se_gate_fwd(const float* x, const float* m, float* s, long long rows, int hw, void* stream);
int hk_se_gate_bwd(const float* x, const float* m, const float* ds, float* dx, float* dm, long long rows, int hw,
                   void* stream);
/* ---- MAMC / N-pairs loss of OSMENet: model/loss/MAMC_loss.py:24-90 -------------------------------------------------------
 * hk_l2norm_rows_*: F.normalize(p=2, dim=1) of [rows, D] and its backward (inv_norm[r] = 1 / max(||x_r||, 1e-12)).
 * hk_npair_loss: prod [n,n] = F F^T of the n = batch x attention anchors (row-normalised features), cls[n] / part[n] the
 * label and attention index of each anchor.  Adds the N-pairs loss (sum of the three terms of eq. 11, divided by n) to the
 * pre-zeroed fp64 accumulator loss_acc[0] and writes d loss / d prod [n,n].  One launch, O(n) per anchor
 * (sum_k exp(neg_k - pos_j) = exp(-pos_j) * sum_k exp(neg_k)) instead of the reference's per-anchor Python loop. */
int hk_l2norm_rows_fwd(const float* x, float* y, float* inv_norm, int rows, int D, void* stream);
int hk_l2norm_rows_bwd(const float* y, const float* inv_norm, const float* dy, float* dx, int rows, int D, void* stream);
int hk_npair_loss(const float* prod, const int* cls, const int* part, double* loss_acc, float* dprod, int n, void* stream);

/* ---- APINet: model/methods/APINet.py:28-119, model/loss/APINet_loss.py:33-39 -------------------------------------------
 * hk_apinet_pairs (get_pairs + pdist, :76-119): pool [n,D], labels [n] -> intra[i] = argmin over j != i of the same label,
 *   inter[i] = argmin over other labels of dist(i,j) = (-2<x_i,x_j> + |x_j|^2) + |x_i|^2 (fp32, fixed order); ties go to
 *   the lowest index, a row without candidates gets 0 (np.argmin of an all-inf row).  labels1 / labels2 (optional, [2n])
 *   receive cat(labels, labels) and cat(labels[intra], labels[inter]).  2 <= n <= 4096; no host round trip.
 * hk_apinet_gather: mutual [2n, 2D] = [pool[r mod n] | pool[idx2[r]]] with idx2 = cat(intra, inter) (:36-43);
 *   hk_apinet_scatter is its adjoint: dpool[i] sums its sources in ascending row order (no atomics).  D % 4 == 0.
 * hk_dropout_*: nn.Dropout(p) in train mode, y = x * keep / (1 - p); keep is a stateless hash of (*seed, call, element index)
 *   (splitmix64; restated in oracle/hop_oracle.py), so the backward recomputes the mask.  The seed is a device int64, so a
 *   captured graph draws new masks on every replay.  p == 0: identity (seed may be null).
 * hk_apinet_gate_fwd (:46-61): m = map2 output [2n, D], f1 / f2 = the halves of mutual; g1 = sigmoid(m f1), g2 = sigmoid(m f2);
 *   out [8n, D] = [drop(g1 f1 + f1); drop(g2 f2 + f2); drop(g2 f1 + f1); drop(g1 f2 + f2)] (self_1, self_2, other_1, other_2:
 *   one hk_linear_fwd of fc over it gives cat(self_logits, other_logits), :63-69).  Dropout call ids call0 + 0..3 in the
 *   reference's order (f1 self, f1 other, f2 self, f2 other).  The backward writes dm and STORES df1 | df2 into dmutual
 *   (map1's dgrad then accumulates onto it).
 * hk_apinet_rank_loss: logits [2R, K] whose rows r and r + R are a (self, other) pair, targets [2R]; adds
 *   mean_r max(0, p_other[r] - p_self[r] + margin) (p = softmax probability of the row's target) to the fp64 accumulator
 *   loss_acc[0] and ADDS its gradient times grad_scale to dlogits (optional; which holds the cross-entropy gradient).  At the
 *   hinge the gradient passes, as torch's clamp_min does.  Default precision mode: the sums are rounded to tf32 on store. */
int hk_apinet_pairs(const float* pool, const long long* labels, long long* intra, long long* inter, long long* labels1,
                    long long* labels2, int n, int D, void* stream);
int hk_apinet_gather(const float* pool, const long long* idx2, float* mutual, int n, int D, void* stream);
int hk_apinet_scatter(const float* dmutual, const long long* idx2, float* dpool, int n, int D, void* stream);
int hk_dropout_fwd(const float* x, float* y, size_t n, float p, const long long* seed, int call, void* stream);
int hk_dropout_bwd(const float* dy, float* dx, size_t n, float p, const long long* seed, int call, void* stream);
int hk_apinet_gate_fwd(const float* m, const float* mutual, float* out, int rows, int D, float p, const long long* seed,
                       int call0, void* stream);
int hk_apinet_gate_bwd(const float* m, const float* mutual, const float* dout, float* dm, float* dmutual, int rows, int D,
                       float p, const long long* seed, int call0, void* stream);
int hk_apinet_rank_loss(const float* logits, const long long* targets, double* loss_acc, float* dlogits, int R, int K,
                        float margin, float grad_scale, void* stream);

/* ---- DCL: model/methods/DCL.py:31-45, model/loss/DCL_loss.py:16-21 ------------------------------------------------
 * hk_dcl_head_fwd (DCL.py:33-39): trunk map x [N,C,H,W] (NCHW), Convmask weight w [C] and bias b [1] ->
 *   pooled [N,C] = spatial mean of x, and mask [N,Q], Q = (H/2)(W/2), = tanh(avgpool2x2(w.x[n,:,p] + b)); an odd last row /
 *   column is dropped, as AvgPool2d(2) drops it.  x is read once; the per-block shares of the 1x1 conv go to the workspace
 *   (hk_dcl_head_workspace_bytes, serves both directions) and are added in a fixed order: no atomics, the same bits on every
 *   run.  Default precision mode: pooled is rounded to tf32 on store (operand of the classifier MMA); mask is not.
 * hk_dcl_head_bwd: dpooled [N,C], dmask [N,Q] -> dx [N,C,H,W] = dpooled/HW + w[c] dz[n,p] (dz: the tanh and 2x2-mean
 *   adjoint, 0 on a dropped row / column), dw [C], db [1]; one read of x, one write of dx, fixed-order sums.  H*W <= 1024.
 * hk_dcl_loss (DCLLoss): logits [R,ld] with the classifier in columns [0,K) and classifier_swap in [K,K+K2); labels /
 *   labels_swap int64 [R]; mask / law [R,Q].  ADDS alpha CE(0:K, labels) + beta CE(K:K+K2, labels_swap) + gamma L1(mask, law)
 *   (CE with label smoothing 0.1, means over rows / entries) to the fp64 accumulator loss_acc[0]; writes dlogits [R,ld] (pad
 *   columns zero; rounded to tf32 in the default mode, like hk_softmax_ce_ls), dmask [R,Q] = gamma sign(mask - law)/(R Q)
 *   (0 where equal) and correct (optional) = top-1 hits over columns [0,K), or with combine (cls_2xmul, K2 == 2K,
 *   Examples/DCL.py:104-107) over z[k] + z[K+k] + z[2K+k].  A label outside its segment gets no one-hot term and never
 *   counts as correct, as in hk_softmax_ce_ls.  Any R. */
size_t hk_dcl_head_workspace_bytes(int N, int C, int H, int W);
int hk_dcl_head_fwd(const float* x, const float* w, const float* b, float* pooled, float* mask, int N, int C, int H, int W,
                    void* workspace, size_t workspace_bytes, void* stream);
int hk_dcl_head_bwd(const float* x, const float* w, const float* mask, const float* dpooled, const float* dmask, float* dx,
                    float* dw, float* db, int N, int C, int H, int W, void* workspace, size_t workspace_bytes, void* stream);
int hk_dcl_loss(const float* logits, int ld, int K, int K2, const long long* labels, const long long* labels_swap,
                const float* mask, const float* law, int R, int Q, float alpha, float beta, float gamma, int combine,
                double* loss_acc, float* dlogits, float* dmask, int* correct, void* stream);

/* ---- ProtoTree: model/methods/ProtoTree/{l2conv,prototree,branch,leaf}.py, Examples/ProtoTreeNet.py ----------------------
 * Tree of height H (1 <= H <= 12): P = 2^H - 1 branches, L = 2^H leaves, 2^(H+1) - 1 nodes numbered in pre-order (root 0,
 * left child i + 1, right child i + 1 + size of the left subtree, prototree.py:275-287).  Prototype row k belongs to the k-th
 * branch in pre-order; leaf j is the j-th leaf from the left.  (The reference maps rows to branches through a set ordered by
 * object hash, prototree.py:51, which changes from process to process; this order is the package's fixed choice.)
 * hk_prototree_dist_fwd (l2conv.py:41-63, prototree.py:111-116): x [N,HW,D] (position-major), prototypes [P,D] ->
 *   mind [N,P] = min over positions of sqrt(sum_d (z - p)^2 + 1e-14), argmin [N,P] int32 = the first minimising position in
 *   row-major order (what max_pool2d of -d picks).  The squared distance is summed directly in fp32 in both precision modes:
 *   the reference's |x|^2 + |p|^2 - 2 x.p cancels at the minimum, the one position that gets a gradient.  act = 1: x is the
 *   neck's pre-activation, z = sigmoid(x) (ProtoTreeNet.py:24-27) is applied on load and stored to z [N,HW,D]; act = 0: z = x
 *   and the z argument is unused.  N <= 65535.
 * hk_prototree_dist_bwd: dmind [N,P] -> dx [N,HW,D] = sum over the prototypes j with argmin h of dmind (z - p_j) / mind, 0 at
 *   every other position (act = 1: times z (1 - z), and rounded to tf32 in the default mode: it is the neck GEMMs' operand);
 *   dprotos [P,D] = -sum_n dmind (z[argmin] - p) / mind.  z is the forward's z (act = 1) or x (act = 0).  Every sum has one
 *   owner and a fixed order: the same bits on every run.  HW + P <= 51199 (the per-image grouping of the prototypes by
 *   argmin position is kept in shared memory).
 * hk_prototree_route_fwd (branch.py:22-57, leaf.py:30-67): mind [N,P], theta [L,K] -> sm [L,K] = softmax of each leaf,
 *   ps [N,P] = exp(-mind) (by branch rank), pa [N, 2^(H+1) - 1] = probability of arriving at each node (pre-order; the left
 *   child gets (1 - ps) pa, the right ps pa), pred [N,K] = sum_l pa[leaf l] sm[l].
 * hk_prototree_route_bwd: dpred [N,K] -> dmind [N,P], bottom-up with u[leaf] = dpred . sm[leaf] and u = (1 - ps) u_l + ps u_r:
 *   dmind = -ps pa (u_r - u_l), with no division by ps or 1 - ps; dtheta [L,K] (optional, K <= 12288) = the softmax adjoint of
 *   sum_n pa[n, leaf] dpred[n].
 * hk_prototree_nll (Examples/ProtoTreeNet.py:109, F.nll_loss(torch.log(pred), labels)): labels int64 [N] -> loss[0] = mean of
 *   -log pred[n, y] over the V rows whose label is in [0, K), dpred [N,K] = -onehot(y) / (V pred[n, y]), correct (optional) =
 *   top-1 hits on pred.  A row with a label outside [0, K) gets no term, no gradient, never counts and is not in V, as
 *   F.nll_loss treats ignore_index rows (torch raises for other out-of-range labels; this does not).  V = 0 gives a NaN loss.
 * hk_prototree_leaf_update_sum / hk_prototree_leaf_update_apply (Examples/ProtoTreeNet.py:116-132), the derivative-free leaf
 *   update in two steps so that data-parallel ranks can all-reduce the sum in between:
 *   update [L,K] = sum_b [y_b = k] pa[b, leaf] softmax(theta)[k] / pred[b, k] from the step's pa, pred and labels (ascending
 *   b); then in place theta = relu(theta - theta0 / num_batches) + update, theta0 = the epoch-start snapshot. */
int hk_prototree_dist_fwd(const float* x, const float* protos, float* z, float* mind, int* argmin, int N, int HW, int D,
                          int P, int act, void* stream);
int hk_prototree_dist_bwd(const float* z, const float* protos, const float* mind, const int* argmin, const float* dmind,
                          float* dx, float* dprotos, int N, int HW, int D, int P, int act, void* stream);
int hk_prototree_route_fwd(const float* mind, const float* theta, float* sm, float* ps, float* pa, float* pred, int N,
                           int height, int K, void* stream);
int hk_prototree_route_bwd(const float* ps, const float* pa, const float* sm, const float* dpred, float* dmind,
                           float* dtheta, int N, int height, int K, void* stream);
int hk_prototree_nll(const float* pred, const long long* labels, float* loss, float* dpred, int* correct, int N, int K,
                     void* stream);
int hk_prototree_leaf_update_sum(const float* theta, const float* pa, const float* pred, const long long* labels,
                                 float* update, int N, int height, int K, void* stream);
int hk_prototree_leaf_update_apply(float* theta, const float* theta0, const float* update, int height, int K,
                                   float num_batches, void* stream);

/* ---- Interp-Parts: model/methods/Interp_Parts.py, model/loss/InterpParts_loss.py --------------------------------------
 * hk_ip_group_fwd (GroupingUnit.forward, Interp_Parts.py:56-122): trunk map x [N,HW,C] (NHWC, as the trunk produces it),
 *   centres [K,C] (the grouping weight [K,C,1,1]), smooth [K] -> with beta = sigmoid(smooth):
 *   dist [N,K,HW] = sum_c (x - c_k)^2, summed directly in fp32 in both precision modes (the reference's 2 c.x - |x|^2 - |c|^2
 *   cancels; a direct sum is never positive after the negation, so the reference's clamp(max=0) is the identity here);
 *   assign [N,K,HW] = softmax over k of -dist / beta; qx [N,K,C] = sum_p assign x; ssum [N,K] = sum_p assign;
 *   u = (qx / max(ssum, 1e-5) - c_k) / sqrt(beta / 2); nrm [N,K] = |u|; out [N,K,C] = u / max(|u|, 1e-12) (F.normalize over
 *   C; the NHWC [N,K,1,C] input of the 1x1 stacks; rounded to tf32 in the default mode, it is the next GEMM's operand).  One
 *   read of the map: partials per 32-pixel tile go to the workspace (hk_ip_group_workspace_bytes, serves both directions)
 *   and a second launch folds them in tile order.  1 <= K <= 32; C % 4 == 0 and C <= 1536; x 16-byte aligned.
 *   Replaces :67-122 (the bmm's, x_sq, the expanded c_sq and beta, the permuted x).
 * hk_ip_group_bwd: dout [N,K,C] -> dx [N,HW,C], dcentres [K,C], dsmooth [K] (through 1/beta in the softmax and through
 *   sqrt(beta / 2)).  The clamps' zero-gradient regions are honoured: no gradient through ssum where ssum < 1e-5, and
 *   dout / 1e-12 where |u| < 1e-12.  dassign (optional, [N,K,HW]) is a dense gradient of assign.  The shaping loss's gradient
 *   arrives as argmax [N,K] (hk_ip_occupancy) and coef [N,K] (optional): coef times the Gaussian taps gauss [(2r+1)^2] is added
 *   to d assign on the window under each blurred maximum, inside the same pass (no dense d assign).  One read of the map, one
 *   write of dx; every sum in a fixed order.
 * hk_ip_att_fwd (attconv[2:5] + softmax + pooling, :289-291,:349-361): f [P,C] (P = N K rows of the attconv stack output),
 *   1-channel conv w [C], b [1]; BatchNorm(1) gamma, beta [1] over the P values (training: batch statistics, running_mean /
 *   running_var updated with momentum and the unbiased variance, as hk_bn_fwd does; else the running statistics); ReLU;
 *   att [N,K] = softmax over the K parts; pooled [N,D] = sum_k att post[n,k,:] with post [P,D] the post_block output
 *   (avg_pool1d(K) * K).  conv [P] and stats [2] = (mean, invstd) are saved for the backward.  Training needs P > 1.
 * hk_ip_att_bwd: dpooled [N,D] and datt (optional, [N,K]) -> df [P,C], dw [C], db [1], dgamma [1], dbeta [1], dpost [P,D];
 *   scratch [P] floats.
 * hk_ip_occupancy (ShapingLoss steps 1-2, InterpParts_loss.py:114-124): assign [N,K,H,W], gauss [(2r+1)^2] (the normalised
 *   Gaussian; [1.0] for radius 0) -> occ [N,K] = max of the "valid" depthwise blur, argmax [N,K] int32 = its position in the
 *   (H - 2r) x (W - 2r) blurred map, the first maximum in row-major order on ties.  2r < H and 2r < W.
 * hk_ip_shaping_loss (:125-138): occ [R,K] (R = the global batch), prior [R] (the Beta prior's quantiles, on the device) ->
 *   loss[0] = mean over (i, k) of |log(occ + eps) - log(prior[rank] + eps)|, rank = the place of occ[i,k] in the ascending
 *   sort of its column (ties by row index); docc [R,K] = its gradient (sign(0) = 0, as torch's abs). */
size_t hk_ip_group_workspace_bytes(int N, int HW, int K, int C);
int hk_ip_group_fwd(const float* x, const float* centres, const float* smooth, float* assign, float* dist, float* out,
                    float* qx, float* ssum, float* nrm, int N, int HW, int K, int C, void* workspace,
                    size_t workspace_bytes, void* stream);
int hk_ip_group_bwd(const float* x, const float* centres, const float* smooth, const float* assign, const float* dist,
                    const float* qx, const float* ssum, const float* nrm, const float* dout, const float* dassign,
                    const int* argmax, const float* coef, const float* gauss, int radius, float* dx, float* dcentres,
                    float* dsmooth, int N, int H, int W, int K, int C, void* workspace, size_t workspace_bytes,
                    void* stream);
int hk_ip_att_fwd(const float* f, const float* w, const float* b, const float* gamma, const float* beta,
                  float* running_mean, float* running_var, float momentum, float eps, int training, const float* post,
                  float* conv, float* att, float* stats, float* pooled, int N, int K, int C, int D, void* stream);
int hk_ip_att_bwd(const float* f, const float* w, const float* gamma, const float* beta, const float* conv,
                  const float* att, const float* stats, const float* post, const float* dpooled, const float* datt,
                  int training, float* df,
                  float* dw, float* db, float* dgamma, float* dbeta, float* dpost, float* scratch, int N, int K, int C,
                  int D, void* stream);
int hk_ip_occupancy(const float* assign, const float* gauss, float* occ, int* argmax, int N, int K, int H, int W,
                    int radius, void* stream);
int hk_ip_shaping_loss(const float* occ, const float* prior, float* loss, float* docc, int R, int K, float eps,
                       void* stream);

/* ---- NTS-Net: model/methods/NTS_Net/NTSNet.py, anchors.py, model/loss/NTS_loss.py --------------------------------------
 * The proposal net's maps d1 [B,H1,W1,C], d2 [B,H2,W2,C], d3 [B,H3,W3,C] (NHWC ReLU outputs of down1..3, H2 = ceil(H1 / 2),
 * H3 = ceil(H2 / 2), likewise W) feed three 1x1 tidy convs with 6, 6 and 9 outputs.  Score a of an image is tidy_k channel ch
 * at position p with a = off_k + ch H_k W_k + p, off = (0, 6 H1 W1, 6 H1 W1 + 6 H2 W2): the reference's channel-major
 * flatten and concatenation (NTSNet.py:79-82), A = hk_nts_num_anchors(H1, W1) scores, which is also the anchor order.
 * hk_nts_score_fwd (ProposalNet tidy1..3, :79-82): w_k [A_k,C] (the tidy weight [A_k,C,1,1]), b_k [A_k] -> score [B,A] in one
 *   launch; one warp per score, fixed-order sums.
 * hk_nts_score_bwd: the sparse gradient of top_n_prob = gather(score, idx) (:42), dprob [B,T] at idx int64 [B,T] ->
 *   g_k [B,H_k,W_k,C] = (d_k > 0) (d score / d d_k): the gradient at down_k's pre-activation from the tidy path; dw_k [A_k,C],
 *   db_k [A_k].  Only the T kept scores of an image are read; an index outside [0, A) is skipped.  Fixed-order sums.
 * hk_nts_nms (hard_nms, anchors.py:63-90, per image, :35-42): scores [B,A], anchors int32 [A,4] = (y0, x0, y1, x1) ->
 *   idx int64 [B,T], prob [B,T] = scores at idx, boxes int32 [B,T,4] = anchors at idx.  Greedy: the highest-scoring alive
 *   candidate is kept, then every alive candidate whose IoU with it is >= 0.25 is dropped, the IoU tested exactly on the
 *   integer boxes as 4 inter >= union (inter = 0 when either overlap extent is negative).  Equal scores go to the lower
 *   index (the reference's np.argsort leaves that order undefined).  A row with fewer than T survivors gets idx -1, prob 0
 *   and box (0, 0, 1, 1) past its last survivor.  One block per image; A <= 2048; anchors and boxes 16-byte aligned.
 * hk_nts_crop (:43-49): img NCHW [B,C,H,W], boxes int32 [B*T,4] in the coordinates of the image zero-padded by pad on every
 *   side -> out NCHW [B*T,C,S,S] = F.interpolate(padded[n, :, y0:y1, x0:x1], (S, S), bilinear, align_corners=True) with
 *   ATen's upsample_bilinear2d arithmetic.  Pixels outside the image read as zero; no padded copy is made.  B T <= 65535.
 * hk_nts_rank_loss (list_loss + ranking_loss, NTS_loss.py:32-47): part_logits [B*T,K] (row n T + t), labels int64 [B],
 *   prob [B,T] -> L[n,t] = logsumexp - z[y_n] in fp32; ADDS sum_n sum_i sum_j relu(1 - prob[n,i] + prob[n,j]) [L[n,j] > L[n,i]]
 *   / B to the fp64 accumulator loss_acc[0] and writes dprob [B,T] (no gradient through L; none at the hinge).  B T <= 8192. */
int hk_nts_num_anchors(int H1, int W1);
int hk_nts_score_fwd(const float* d1, const float* d2, const float* d3, const float* w1, const float* b1, const float* w2,
                     const float* b2, const float* w3, const float* b3, float* score, int B, int H1, int W1, int H2, int W2,
                     int H3, int W3, int C, void* stream);
int hk_nts_score_bwd(const float* d1, const float* d2, const float* d3, const float* w1, const float* w2, const float* w3,
                     const long long* idx, const float* dprob, float* g1, float* g2, float* g3, float* dw1, float* db1,
                     float* dw2, float* db2, float* dw3, float* db3, int B, int T, int H1, int W1, int H2, int W2, int H3,
                     int W3, int C, void* stream);
int hk_nts_nms(const float* scores, const int* anchors, long long* idx, float* prob, int* boxes, int B, int A, int T,
               void* stream);
int hk_nts_crop(const float* img, const int* boxes, float* out, int B, int T, int C, int H, int W, int pad, int S,
                void* stream);
int hk_nts_rank_loss(const float* part_logits, const long long* labels, const float* prob, double* loss_acc, float* dprob,
                     int B, int T, int K, void* stream);

/* ---- AP-CNN (model/methods/APCNN.py): feature pyramid, pyramid attention, ROI selection, ROI-guided refinement ------------
 * All maps NHWC fp32, 16-byte aligned; every sum in a fixed order (no atomics), so results are bitwise repeatable.
 * hk_apcnn_lateral_fwd (PyramidFeatures.forward, :221-230): out [N,2h,2w,C] = nearest-2x(top [N,h,w,C]) + lat; _bwd: dtop =
 *   the 2x2 sums of dout (dlat is dout itself).  C % 4 == 0.
 * hk_apcnn_bcast (SimpleFPA's x_master + x_gpb, :197): y [N,HW,C] = a (optional, else 0) + scale b [N,C].
 * hk_apcnn_pool (AvgPool2d over the map, :194, and the adjoint of the broadcast): y [N,C] = scale sum_p x [N,HW,C].  C % 256.
 * hk_apcnn_att_fwd (SpatialGate :271-280 and the pools behind cls3/4/5 and Concate, :533-563): F [N,H,W,256], w [256,1,3,3]
 *   and bias [1] of the ConvTranspose2d(256, 1, 3, 1, 1) -> gate [N,H,W] = sigmoid(convT(F)), pool_f [N,256] = mean_hw F,
 *   pool_sf [N,256] = mean_hw(gate F).  With the channel gate ch [N,256], mean_hw((gate + ch) F) = pool_sf + ch pool_f, so the
 *   attended maps (:256-266) are never written.  F is read twice (tap products, then gate and pools).
 * hk_apcnn_att_bwd: dpool_f (optional) and dpool_sf [N,256] -> dF = dpool_f / HW + gate dpool_sf / HW + the gate's path,
 *   dw [256,1,3,3], db [1].  F is read twice and dF written once.  The gate itself carries no gradient (the reference uses it
 *   under no_grad for the ROIs and for visualisation).
 * hk_apcnn_roi (get_att_roi, :444-476, for the three levels in one launch): gates g3 [N,H3,W3], g4 [N,H3/2,W3/2], g5
 *   [N,H3/4,W3/4]; windows int32 [3,4] = (y0, y1, x0, x1) of each level's central window (host memory); keep uint8 [3,15,15] =
 *   1 where a cell at offset (dy + 7, dx + 7) from a pick survives it (device memory).  Cells outside the window count as 0;
 *   a cell is a candidate iff its value is strictly above the mean over all h w cells; greedy NMS up to 5 / 3 / 1 picks,
 *   equal scores to the highest flat index.  boxes fp32 [N,9,4] = (x1, y1, x2, y2) clamped to [0, img - 1], levels at rows
 *   0-4, 5-7, 8, zeros past the count; counts int32 [N,3].  H3, W3 % 4 == 0; H3 W3 <= 9830.
 * hk_apcnn_refine_fwd (get_roi_crop_feat, :478-531): x [N,H,W,C], boxes / counts as above, draws fp32 [N,2] in [0, 1) or null
 *   (eval mode: no drop, no rescale) -> y [N,H,W,C]: the union of the image's ROIs / 8, truncated, bilinearly resized
 *   (align_corners=False, ATen's arithmetic) to H x W.  draws[n,0] < 0.3 drops level-3 ROI floor(draws[n,1] count), < 0.6 a
 *   level-4 ROI; the crop is multiplied by the untruncated window area over its kept cells.  meta int32 [N,12] is written for
 *   the backward.  An image without any ROI keeps its whole map.  _bwd: dy -> dx (zero outside the window and in the dropped
 *   block), gather form.  C % 4 == 0.
 * hk_apcnn_mix_fwd / _bwd (PyramidAttentions.forward, :251-268, on vectors): z, pm, psf, v, ch [3,N,C] (levels 3, 4, 5);
 *   ch_3 = sig(z_3), ch_4 = (sig(z_4) + ch_3) / 2, ch_5 = (sig(z_5) + ch_4) / 2, v_l = psf_l + ch_l pm_l; the backward gives
 *   dz and dpm from dv (dpsf is dv).
 * hk_apcnn_mask_cat (:590-592): out [N,3,H3,W3] = (g3, nearest-2x g4, nearest-4x g5). */
int hk_apcnn_lateral_fwd(const float* top, const float* lat, float* out, int N, int h, int w, int C, void* stream);
int hk_apcnn_lateral_bwd(const float* dout, float* dtop, int N, int h, int w, int C, void* stream);
int hk_apcnn_bcast(const float* a, const float* b, float* y, int N, int HW, int C, float scale, void* stream);
size_t hk_apcnn_pool_workspace_bytes(int N, int HW, int C);
int hk_apcnn_pool(const float* x, float* y, int N, int HW, int C, float scale, void* workspace, size_t workspace_bytes,
                  void* stream);
size_t hk_apcnn_att_workspace_bytes(int N, int H, int W);
int hk_apcnn_att_fwd(const float* F, const float* w, const float* bias, float* gate, float* pool_f, float* pool_sf, int N,
                     int H, int W, int C, void* workspace, size_t workspace_bytes, void* stream);
int hk_apcnn_att_bwd(const float* F, const float* w, const float* gate, const float* dpool_f, const float* dpool_sf, float* dF,
                     float* dw, float* db, int N, int H, int W, int C, void* workspace, size_t workspace_bytes, void* stream);
int hk_apcnn_roi(const float* g3, const float* g4, const float* g5, const int* windows, const unsigned char* keep, float* boxes,
                 int* counts, int N, int H3, int W3, int img_h, int img_w, void* stream);
int hk_apcnn_refine_fwd(const float* x, const float* boxes, const int* counts, const float* draws, float* y, int* meta, int N,
                        int H, int W, int C, void* stream);
int hk_apcnn_refine_bwd(const float* dy, const int* meta, float* dx, int N, int H, int W, int C, void* stream);
int hk_apcnn_mix_fwd(const float* z, const float* pm, const float* psf, float* v, float* ch, int N, int C, void* stream);
int hk_apcnn_mix_bwd(const float* z, const float* pm, const float* ch, const float* dv, float* dz, float* dpm, int N, int C,
                     void* stream);
int hk_apcnn_mask_cat(const float* g3, const float* g4, const float* g5, float* out, int N, int H3, int W3, void* stream);

/* ---- MGE-CNN (model/methods/MGE_CNN/MGE.py, grad_cam.py): part head, Grad-CAM boxes, detached concatenation, gate -------
 * All maps NHWC fp32; every sum in a fixed order (no atomics), so results are bitwise repeatable.
 * hk_mge_part_fwd (conv6* + F.relu + pool_max, MGE.py:135, :166, :197): x [N,H,W,C] (layer3's map), w [O,C] (the weight
 *   [O,C,1,1] of Conv2d(C, O, 1, 1, padding 1)), bias [O] -> pooled [N,O] = max(relu(b_o), max_p relu(w_o . x_p + b_o)) (the
 *   padded border of the conv's output is its bias) and pos int32 [N,O], the winning pixel (first in row-major order) or -1
 *   when the border wins, ties included.  The product runs on the wgmma GEMM (bias in its epilogue) into the workspace
 *   (hk_mge_part_workspace_bytes); pooled is rounded to tf32 on store outside the precise mode.  C, O % 4 == 0.
 * hk_mge_part_bwd: dpooled [N,O] -> dw [O,C] = sum_n dpooled [pooled > 0] x[n, pos] (nothing for the border), db [O] =
 *   sum_n dpooled [pooled > 0], n ascending.  No dx: the head reads conv4.detach().
 * hk_mge_cam_box (GradCam, grad_cam.py:51-90, and get_bbox, MGE.py:48-72, for all images in one launch, one block each):
 *   the target is targets[n] (int64, may be null) or else the first maximum of logits [N,K]; the layer weights are
 *   relu(w_main[idx]) / (h w) (the closed form of the reference's backward: the hooked tensor is pooled and fed to the main
 *   classifier w_main [K,C]); a target outside [0, K) gives zero weights.  CAM = sum_c feat[n] [h,w,C] * weights, upsampled
 *   to S x S (bilinear, align_corners=True, ATen's fp32 arithmetic), min-max normalised and kept where !(m < rate) (a
 *   constant CAM gives 0 / 0 = NaN and keeps every pixel).  boxes int32 [N,4] = (y0, x0, y1, x1), the extents of the kept
 *   pixels with the end exclusive (x[:, y0:y1, x0:x1]), or (0, 0, S, S) when y0 == y1 or x0 == x1: what hk_nts_crop reads
 *   with pad 0.  C + h w <= 12288; boxes 16-byte aligned.
 * hk_mge_cat_l2n (pool_cat*, MGE.py:136, :167, :198): out [N, Da + Db] = (scale a / ||a||, scale b / ||b||) per row, without
 *   an epsilon (l2_norm_v2); rounded to tf32 on store outside the precise mode.
 * hk_mge_gate_fwd (cls_gate[1], softmax and the weighted sum, MGE.py:207-213): h [N,F] (cls_gate[0]'s output), w2 [3,F],
 *   b2 [3], the three cat logits c0, c1, c2 [N,K] -> pr [N,3] = softmax(h w2^T + b2), out [N,K] = c0 pr0 + c1 pr1 + c2 pr2.
 *   The 3-output linear lives here because the GEMM's operands need a 16-byte row pitch.
 * hk_mge_gate_bwd: dout [N,K] (and dpr [N,3], may be null) -> dz [N,3], the gradient of the gate logits; dh [N,F] (may be
 *   null); dw2 [3,F] and db2 [3] (both or neither), n ascending.  No gradient reaches c0..c2 (detached in the reference). */
size_t hk_mge_part_workspace_bytes(int N, int H, int W, int O);
int hk_mge_part_fwd(const float* x, const float* w, const float* bias, float* pooled, int* pos, int N, int H, int W, int C,
                    int O, void* workspace, size_t workspace_bytes, void* stream);
int hk_mge_part_bwd(const float* x, const int* pos, const float* pooled, const float* dpooled, float* dw, float* db, int N,
                    int H, int W, int C, int O, void* stream);
int hk_mge_cam_box(const float* logits, const long long* targets, const float* w_main, const float* feat, int* boxes, int N,
                   int K, int C, int h, int w, int S, float rate, void* stream);
int hk_mge_cat_l2n(const float* a, const float* b, float* out, int N, int Da, int Db, float scale, void* stream);
int hk_mge_gate_fwd(const float* h, const float* w2, const float* b2, const float* c0, const float* c1, const float* c2,
                    float* pr, float* out, int N, int F, int K, void* stream);
int hk_mge_gate_bwd(const float* h, const float* w2, const float* pr, const float* c0, const float* c1, const float* c2,
                    const float* dout, const float* dpr, float* dz, float* dh, float* dw2, float* db2, int N, int F, int K,
                    void* stream);

/* ---- classifier nn.Linear (BCNN.py:42, CBCNN.py:26, MPNCOV.py:31) as skinny wgmma GEMMs ------------------- */
size_t hk_linear_fwd_workspace_bytes(int B, int F, int N);
int hk_linear_fwd(const float* x, const float* w, const float* bias, float* y, int B, int F, int N, void* workspace,
                  size_t workspace_bytes, void* stream);
int hk_linear_dgrad(const float* dy, const float* w, float* dx, int B, int F, int N, void* stream);
int hk_linear_wgrad(const float* dy, const float* x, float* dw, float* db, int B, int F, int N, void* stream);

/* ---- nn.CrossEntropyLoss(label_smoothing) fwd+bwd (train.py:211-212, :315-319); labels int64 ----------------
 * loss[0] = mean loss; dlogits (optional) = dloss/dlogits * grad_scale; correct (optional) = #argmax==label.
 * A label outside [0, K) gets no one-hot term (its row adds eps (lse - mean(z)) and gets softmax - eps/K) and never counts.
 * In the default precision mode dlogits is rounded to tf32 on store (it is the operand of the classifier's dgrad / wgrad
 * MMAs, which would otherwise truncate it); hk_set_precise(1) stores it unrounded. */
int hk_softmax_ce_ls(const float* logits, const long long* labels, float* loss, float* dlogits, int* correct, int B,
                     int K, float label_smoothing, float grad_scale, void* stream);

/* ---- Pairwise Confusion: model/loss/pair_confusion.py (PairwiseConfusionLoss) ------------------------------------------
 * logits [B, K], labels int64 [B], B even.  loss[0] = CE_ls(z, y) + lambda_a * sum_{i < B/2} [y_i != y_{B/2+i}] ||d_i|| / B,
 * d_i = z_i - z_{B/2+i}; dlogits = (softmax - target) * grad_scale / B plus, on a pair with differing labels and
 * ||d_i|| > 0, +-(lambda_a / B) d_i / ||d_i|| * grad_scale on rows i and B/2+i (0 when ||d_i|| = 0, as torch's norm
 * backward gives); correct[0] = top-1 hits over the B rows, as hk_softmax_ce_ls counts them.  dlogits is rounded to tf32
 * once, in the default precision mode.  One launch, one block, fixed-order sums: the same bits on every run.
 * HK_ERR_ARG on a null pointer, B odd or below 2, or K <= 0. */
int hk_pc_loss(const float* logits, const long long* labels, float* loss, float* dlogits, int* correct, int B, int K,
               float label_smoothing, float lambda_a, float grad_scale, void* stream);

/* ---- CrossX: model/methods/CrossX.py (MELayer in Bottleneck, the conv2_i / conv3_i fusion), model/loss/CrossX_loss.py ---
 * Maps NHWC fp32, 16-byte aligned.  Part maps are [N, HW, P, C]: the P parts of a pixel side by side.  P in 1..3.  Every sum
 * runs in a fixed order, so results are bitwise repeatable.
 * hk_crossx_me_fwd (Bottleneck.forward with meflag, CrossX.py:110-123): c = bn3 output [N,HW,C], r = residual, m = the
 *   pre-sigmoid gate logits [N,P,C] -> out = relu(c + r) (optional: null skips it) and part p = relu(c sigmoid(m_p) + r).
 *   c and r are read once.  C % 128.
 * hk_crossx_me_bwd: dout (optional) and dparts [N,HW,P,C] -> dc, dr [N,HW,C] and dm [N,P,C] = g (1 - g) sum_hw dpart_p
 *   [part_p > 0] c, the ReLU masks recomputed from c, r and m.  The squeeze's gradient (mean_hw c feeds the gates) is not
 *   part of dc.  Workspace: hk_crossx_me_bwd_workspace_bytes.  C % 128.
 * hk_crossx_fuse_fwd (CrossX.py:211-225, part p): parts = the layer3 parts [N,H,W,P,C], R = conv2_p(layer4 part p)
 *   [N,H/2,W/2,C] -> S [N,H,W,C] = part_p + nearest-2x(R); pmax [N,P,C] (slice p) = the global max of part_p and pidx the
 *   pixel h W + w where AdaptiveMaxPool2d(1)'s h-major scan finds it: the first of equal maxima, the last NaN.  H, W even,
 *   C % 32.
 * hk_crossx_fuse_bwd: dS, dpmax [N,P,C], pidx -> dparts (slice p) = dS + dpmax at pidx, dR = the 2x2 sums of dS.  C % 4.
 * hk_crossx_reg_sums (RegularLoss, CrossX_loss.py:13-17): fu [N,P,Cu], fp and fc [N,P,Cp] -> s = (s_u [P,Cu], s_p [P,Cp],
 *   s_c [P,Cp]) concatenated, s_g[p] = sum_n x[n,p] / ||x[n,p]||.  An all-zero row adds nothing (the reference: NaN).
 * hk_crossx_loss (CrossXLoss.__call__, :44-64): logits xf, xp, xc [N,K], labels int64 [N], the features and s (summed over
 *   every rank's batch, n_total images) -> loss[0] = CE_ls(xf + xp + xc) + (KL(xp) + KL(xc)) / N + sum_g gamma_g
 *   sum(triu(corr_g)), KL(x) = sum q (log q - log_softmax x) with q = softmax xf (which receives gradient),
 *   corr_g[i,j] = s_i . s_j / n_total^2 with 1 - corr on the diagonal; dxf, dxp, dxc (rounded to tf32 once in the default
 *   mode) and dfu, dfp, dfc (the regularisers' gradient times reg_scale; zero for an all-zero row); correct[0] = top-1 hits
 *   of xf + xp + xc.  A class where softmax xf underflows to 0 adds 0 to the KL terms and to dxf (the reference's gradient
 *   through its target is log 0 there, so its dxf is NaN).  One launch, one block, no host read-back. */
int hk_crossx_me_fwd(const float* c, const float* r, const float* m, float* out, float* parts, int N, int HW, int P, int C,
                     void* stream);
size_t hk_crossx_me_bwd_workspace_bytes(int N, int HW, int P, int C);
int hk_crossx_me_bwd(const float* c, const float* r, const float* m, const float* dout, const float* dparts, float* dc,
                     float* dr, float* dm, int N, int HW, int P, int C, void* workspace, size_t workspace_bytes,
                     void* stream);
int hk_crossx_fuse_fwd(const float* parts, const float* R, float* S, float* pmax, int* pidx, int N, int H, int W, int P,
                       int C, int p, void* stream);
int hk_crossx_fuse_bwd(const float* dS, const float* dpmax, const int* pidx, float* dparts, float* dR, int N, int H, int W,
                       int P, int C, int p, void* stream);
int hk_crossx_reg_sums(const float* fu, const float* fp, const float* fc, float* s, int N, int P, int Cu, int Cp,
                       void* stream);
int hk_crossx_loss(const float* xf, const float* xp, const float* xc, const long long* labels, const float* fu,
                   const float* fp, const float* fc, const float* s, float* loss, float* dxf, float* dxp, float* dxc,
                   float* dfu, float* dfp, float* dfc, int* correct, int N, int K, int P, int Cu, int Cp,
                   float label_smoothing, float gamma_ulti, float gamma_plty, float gamma_cmbn, int n_total,
                   float reg_scale, void* stream);

/* ---- S3N: model/methods/S3N.py (grid_size 31, padding_size 30, a 61x61 filter) ---------------------------------------
 * hk_s3n_sample_maps (S3N.py:193-270, generate_map up to the two torch.cat): one block per image.  crm [N,h,w,K] are the
 *   class response maps as the 1x1 conv's NHWC rows (S3N.py:290-291 before the interpolation), rnd [N,961] uniform draws
 *   (a peak at grid position q uses rnd[n,q]), p int32 [1] on the device (0, 1 or 2, S3N.py:226-258), radius / radius_inv
 *   [1] (the ScaleLayer scales).  Interpolates to 31x31 (align_corners=True), takes softmax, top-5 and the gate of the maps'
 *   spatial means, the decision map, its min-max normalisation and its peaks (first maximum of the 3x3 window and >= the
 *   mean), assigns them by p and writes xs [2N,961]: rows [0,N) the zoom maps base + sum s G(radius sqrt s), rows [N,2N)
 *   the complementary maps base + sum (1/s) G(radius_inv sqrt s), G(t) = exp(-d^2 / 2(31 t)^2) (kernel_generate over its
 *   maximum).  The peak record for the backward: counts [N], peaks [N,961] int32 = position | flags << 16 (1: zoom map,
 *   2: complementary map) and scores [N,961], in row-major order.  An image without peaks keeps base in both maps.
 *   h, w <= 64, 5 <= K <= 4096; no host synchronisation.
 * hk_s3n_sample_maps_bwd: dxs [2N,961] and the peak record -> dradius [1], dradius_inv [1], one block, fixed order.
 * hk_s3n_grid_fwd (create_grid, S3N.py:156-183, after ReplicationPad2d(30) at :272/:277): maps [B,961] (B = 2N: zoom then
 *   complementary), filter [61,61] -> grid [B,31,31,2] = clamp(2 Sx / S0 - 1, -1, 1), clamp(2 Sy / S0 - 1, -1, 1), with S0,
 *   Sx, Sy the correlations of the padded map alone, times the x basis and times the y basis; sums [B,31,31,3] = (S0,Sx,Sy)
 *   for the backward.
 * hk_s3n_grid_bwd: dgrid [B,31,31,2] -> dmaps [B,961] (through the clamp, inclusive at the bounds, the quotient, the
 *   correlations and the replication pad) and dfilter [61,61] summed over the B maps in index order.  Workspace:
 *   hk_s3n_grid_bwd_workspace_bytes(B).
 * hk_s3n_warp_fwd (S3N.py:186 + :274/:279): x [N,C,H,W], grid [B,31,31,2] -> out [B,C,Ho,Wo] = grid_sample(x[b % N],
 *   interpolate(grid, (Ho,Wo), bilinear, align_corners=True), bilinear, zeros, align_corners=True); the Ho x Wo grid is
 *   never written.
 * hk_s3n_warp_bwd: dout [B,C,Ho,Wo] -> dgrid [B,31,31,2] (x gets no gradient); workspace
 *   hk_s3n_warp_bwd_workspace_bytes(B,Ho,Wo) holds the Ho x Wo grid gradient, which is gathered per coarse node.
 * hk_stem_dgrad (backbone/resnet.py:176, conv1 7x7 / 2, padding 3, 64 outputs): dc NHWC [N,Ho,Wo,64] (16-byte aligned),
 *   w [64,3,7,7] -> dx NCHW [N,3,H,W], a gather per input pixel: no atomics, no column workspace. */
int hk_s3n_sample_maps(const float* crm, const float* rnd, const int* p, const float* radius, const float* radius_inv,
                       float base_ratio, float* xs, int* peaks, float* scores, int* counts, int N, int h, int w, int K,
                       void* stream);
int hk_s3n_sample_maps_bwd(const float* dxs, const int* peaks, const float* scores, const int* counts,
                           const float* radius, const float* radius_inv, float* dradius, float* dradius_inv, int N,
                           void* stream);
int hk_s3n_grid_fwd(const float* maps, const float* filter, float* grid, float* sums, int B, void* stream);
size_t hk_s3n_grid_bwd_workspace_bytes(int B);
int hk_s3n_grid_bwd(const float* maps, const float* filter, const float* sums, const float* dgrid, float* dmaps,
                    float* dfilter, int B, void* workspace, size_t workspace_bytes, void* stream);
int hk_s3n_warp_fwd(const float* x, const float* grid, float* out, int N, int B, int C, int H, int W, int Ho, int Wo,
                    void* stream);
size_t hk_s3n_warp_bwd_workspace_bytes(int B, int Ho, int Wo);
int hk_s3n_warp_bwd(const float* x, const float* grid, const float* dout, float* dgrid, int N, int B, int C, int H, int W,
                    int Ho, int Wo, void* workspace, size_t workspace_bytes, void* stream);
int hk_stem_dgrad(const float* dc, const float* w, float* dx, int N, int H, int W, void* stream);

/* ---- input side: transforms.ToTensor + Normalize (dataset/transforms.py:14-19, test.py:80-85) fused on
 * the GPU: uint8 HWC batch [N,H,W,3] -> fp32 NCHW (x/255 - mean_c)/std_c; a quarter of the float pipeline's H2D bytes */
int hk_normalize_u8(const unsigned char* x_nhwc, float* y_nchw, int N, int H, int W, float mean0, float mean1, float mean2,
                    float std0, float std1, float std2, void* stream);

/* ---- input side: the default train / eval presets (dataset/transforms.py ClassificationPresetTrain: RandomResizedCrop,
 * flip, TrivialAugmentWide, ToTensor, Normalize, RandomErasing; ClassificationPresetEval: Resize, CenterCrop, ToTensor,
 * Normalize) on the GPU.  The input is a ragged batch of N decoded RGB images: uint8 HWC, image n at byte offsets[n] of
 * src with sizes[n] = (H, W).  params [N, hk_augment_params_cols()] (double) holds each image's draws, made on the host
 * (hawkeye_b200/ops_augment.py documents the columns).  Three launches, in order:
 * hk_augment_crop_resize: -> img [N,S,S,3] uint8, the source box resized to the virtual size with PIL's BILINEAR
 *   arithmetic (bit-identical to Image.resize), the S x S window kept, mirrored on request.  A box outside its image gives
 *   a zero image.
 * hk_augment_stats: img -> lut [N,3,256] uint8, the tables of the images whose op is Contrast, AutoContrast or Equalize
 *   (one block per image; the others' rows are not written).
 * hk_augment_apply: img, lut -> y [N,3,S,S] fp32 = the image's TrivialAugmentWide op, then (x/255 - mean_c)/std_c as
 *   hk_normalize_u8 computes it, 0 inside the erasing rectangle. */
int hk_augment_params_cols(void);
int hk_augment_crop_resize(const unsigned char* src, const long long* offsets, const int* sizes, const double* params,
                           unsigned char* img, int N, int S, void* stream);
int hk_augment_stats(const unsigned char* img, const double* params, unsigned char* lut, int N, int S, void* stream);
int hk_augment_apply(const unsigned char* img, const double* params, const unsigned char* lut, float* y, int N, int S,
                     float mean0, float mean1, float mean2, float std0, float std1, float std2, void* stream);

/* ---- input side: baseline JPEG decode, bit-identical to PIL's Image.open(path).convert('RGB') through libjpeg-turbo,
 * for the images the device presets leave encoded (dataset.transformer.decode: cuda).  hawkeye_b200/ops_jpeg.py parses
 * the markers on the host and documents the batch layout: J encoded images; scan = their unstuffed scans back to back
 * (4-byte aligned, scan_bytes including at least 8 bytes of padding); segs [G + 1] int32 = the byte offset of each
 * restart segment in scan, the last entry the end; header [J, hk_jpeg_header_cols()] int32 = each image's batch index,
 * size, components, luma sampling, MCUs, restart interval, first segment and count, first block, plane offset and its
 * quant / DC / AC table indices per component; qtabs [Q, 64] int32 in natural order; htabs = the Huffman tables, 1424
 * bytes each (canonical maxcode / valoffset / huffval and a 9-bit look-ahead).  Three launches, in order:
 * hk_jpeg_huffman: scan -> coef [blocks, 64] int16 in natural order, DC absolute, each image's blocks in decode order
 *   from its first block; status [J] int32 = 0 when the image decoded, else 1 invalid Huffman code, 2 the data ends
 *   early, 3 data past a segment's last block, 4 a restart segment count that does not match the frame, 5 a
 *   coefficient index beyond 63.  One CTA per image decodes chunks of chunk_bytes in parallel by self-synchronisation;
 *   the result does not depend on chunk_bytes.  workspace of hk_jpeg_workspace_bytes(J, G, scan_bytes, chunk_bytes)
 *   bytes (0 for bad arguments).  HK_ERR_ARG on a null pointer or a bad size, HK_ERR_ALIGN, HK_ERR_WORKSPACE.
 * hk_jpeg_idct: coef -> planes uint8: dequantisation and jpeg_idct_islow with its range limit, each component's plane at
 *   whole-MCU size from the image's plane offset (luma, then the chroma planes).
 * hk_jpeg_color: planes -> pixels uint8 HWC at offsets[batch index]: libjpeg-turbo's fancy upsampling (h2v1, h2v2; plain
 *   replication for chroma at most 2 samples wide) and its YCbCr -> RGB tables, or grey replicated, cropped to W x H. */
int hk_jpeg_header_cols(void);
size_t hk_jpeg_workspace_bytes(int J, int G, long long scan_bytes, int chunk_bytes);
int hk_jpeg_huffman(const unsigned char* scan, const int* segs, const int* header, const unsigned char* htabs,
                    short* coef, int* status, int J, int G, long long scan_bytes, int chunk_bytes, void* workspace,
                    size_t workspace_bytes, void* stream);
int hk_jpeg_idct(const short* coef, const int* header, const int* qtabs, unsigned char* planes, int J, void* stream);
int hk_jpeg_color(const unsigned char* planes, const int* header, const long long* offsets, unsigned char* pixels,
                  int J, void* stream);

/* ---- Mixup / CutMix: dataset/transforms.py RandomMixup, RandomCutmix; dataset/collate_fn.py MixupCutmixCollateFn -------
 * One batch's draws are a row of hk_mix_cols() doubles in device memory: kind (0 Mixup, 1 CutMix), lambda, the CutMix
 * box x1, y1, x2, y2 (columns [x1, x2), rows [y1, y2)) and the target weight w (hawkeye_b200/ops_mixup.py).  Image n is
 * paired with image n - 1 mod N, the reference's roll(1, 0).
 * hk_mix_check: validates a row in HOST memory for H x W images before it is staged: HK_ERR_ARG on a null pointer, H or
 *   W <= 0, an unknown kind, lambda or w outside [0, 1], or a box that is not integral or lies outside the image.
 * hk_mix_batch: x [N,C,H,W] fp32 -> y, out of place (y must not alias x).  Replaces transforms.py:129-135 (Mixup):
 *   y_n = fl(fl(x_n (float)lambda) + fl(x_{n-1} (float)(1 - lambda))), bit-identical to the reference; and
 *   transforms.py:206,225 (CutMix): y_n = x_n with the box copied from x_{n-1}.  Reads x once (image N-1 twice) and
 *   writes y once.  HK_ERR_ARG on a null pointer, a size <= 0 or y == x.
 * hk_softmax_ce_ls_mix: replaces transforms.py:123,130,137-138 / :228-229 (the rolled dense target) and train.py:211-212
 *   (nn.CrossEntropyLoss(label_smoothing) on it): the target of row b is w onehot(y_b) + (1 - w) onehot(y_{b-1 mod B}),
 *   loss[0] = mean over rows, dlogits (optional) = (softmax - ((1 - eps) target + eps / K)) * grad_scale / B (rounded to
 *   tf32 in the default mode, as hk_softmax_ce_ls), correct (optional) = rows whose first argmax is the target's argmax
 *   (the larger weight's label; the lower class index on a tie, as target.max(1)[1]).  One launch, fixed-order sums.
 *   HK_ERR_ARG on a null pointer, B <= 0 or K <= 0. */
int hk_mix_cols(void);
int hk_mix_check(const double* mix, int H, int W);
int hk_mix_batch(const float* x, const double* mix, float* y, int N, int C, int H, int W, void* stream);
int hk_softmax_ce_ls_mix(const float* logits, const long long* labels, const double* mix, float* loss, float* dlogits,
                         int* correct, int B, int K, float label_smoothing, float grad_scale, void* stream);

/* ---- model EMA: torch.optim.swa_utils.AveragedModel(model, avg_fn=d * avg + (1 - d) * p, use_buffers=True) with
 * torchvision's ExponentialMovingAverage (references/classification/utils.py) and the update of train_one_epoch.
 * table [nseg, hk_ema_cols()] int64 describes the tensors: model pointer, average pointer, elements, kind (0 float32,
 * 1 int64) and the segment's first chunk (hawkeye_b200/engine.py ModelEMA builds it once and keeps it on the device).
 * hk_ema_plan: validates a table in HOST memory and fills its chunk column; -> the chunk count (the grid of the two
 *   launches below), or HK_ERR_ARG on a null pointer, nseg <= 0, a null or self-aliased segment, a length <= 0 or an
 *   unknown kind, HK_ERR_ALIGN on a pointer not aligned to its elements.
 * hk_ema_update: with the device counter *n_averaged == 0, avg = p; otherwise avg = fl(fl(decay avg) + fl(one_minus_decay
 *   p)) with no fused multiply-add, torch's arithmetic for d * avg + (1 - d) * p (the caller computes 1 - d in double);
 *   int64 tensors in fp32 on the converted values, truncated toward zero.  A 16-byte-aligned float32 segment (the flat
 *   parameter buffer) is read as float4.  Then, in a second one-thread launch so that no block of the first reads it,
 *   the counter is incremented, or set to 0 when reset_after (torchvision's warm-up reset).  No host synchronisation.
 * hk_ema_swap: exchanges the contents of every model tensor and its average in place; two swaps restore every bit.
 * Both: HK_ERR_ARG on a null pointer, nseg <= 0 or a chunk count <= 0 or above INT_MAX; update also on a factor outside
 *   [0, 1]. */
int hk_ema_cols(void);
long long hk_ema_plan(long long* table, int nseg);
int hk_ema_update(const long long* table, int nseg, long long nchunks, long long* n_averaged, float decay,
                  float one_minus_decay, int reset_after, void* stream);
int hk_ema_swap(const long long* table, int nseg, long long nchunks, void* stream);

/* ---- optimizers over flat fp32 buffers: torch.optim.SGD (Examples/BCNN.py:40), Adam (Examples/MPN.py:14-18) */
int hk_sgd_momentum(float* p, const float* g, float* buf, size_t n, float lr, float momentum, float weight_decay,
                    float grad_scale, int first_step, void* stream);
int hk_adam(float* p, const float* g, float* m, float* v, size_t n, float lr, float beta1, float beta2, float eps,
            float weight_decay, float grad_scale, int step, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* HAWKEYE_B200_H */
