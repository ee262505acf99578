/*
 * bdbnn.h — C ABI of libbdbnn_b200.so (sm_90a).
 *
 * The reference (BlueAnon/BD-BNN) ships no native code: its hot path is Python calling
 * ATen/cuDNN.  Each entry point below therefore replaces a *Python* call site of the reference
 * (cited per function, paths relative to the reference root).  The binding a maintainer adds on the
 * reference side is a ctypes stub; see INTEGRATION.md.
 *
 * Conventions
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - activations are NHWC ("channels_last"): element (n,h,w,c) at ((n*H+h)*W+w)*C+c;
 *   - conv weights are OIHW fp32 exactly as torch stores nn.Conv2d.weight;
 *   - bit tensors are uint32 words; bit j of word k covers channel 32*k+j (LSB first);
 *     bit value 1 encodes +1 (x >= 0), bit value 0 encodes -1 (x < 0); channel padding bits are 0;
 *   - stream is a cudaStream_t passed as void*; all work is enqueued on it, nothing synchronises;
 *   - the caller owns every buffer incl. workspaces; the only device memory the library allocates is the
 *     scratch of its cross-block reductions (per-block partials summed in a fixed order, so results are
 *     the same in every run), stream-ordered (cudaMallocAsync / cudaFreeAsync on `stream`, capturable);
 *   - return value 0 = ok, negative = error (bdbnn_last_error_string() describes the last one on
 *     the calling thread).  Nothing throws across the ABI.
 */
#ifndef BDBNN_H_
#define BDBNN_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#if defined(__GNUC__)
#define BDBNN_API __attribute__((visibility("default")))
#else
#define BDBNN_API
#endif

/* +-1 / gradient operand element format fed to the tensor cores (both are exact for +-1) */
#define BDBNN_FMT_FP16 0
#define BDBNN_FMT_BF16 1
/* how gy*gscale is rounded for the tensor-core backward */
#define BDBNN_GRAD_BF16 1    /* bf16(v): 8 significand bits                                        */
#define BDBNN_GRAD_BF16X2 2  /* [bf16 hi | bf16 lo]: 16 bits, two MMAs per K step (fp32-class)      */
#define BDBNN_GRAD_FP16S 3   /* fp16(v * 2^e), e per call from max|v|: 11 bits (TF32-class), 1 MMA  */

#define BDBNN_OK 0
#define BDBNN_ERR_INVALID_ARG (-1)
#define BDBNN_ERR_CUDA (-2)
#define BDBNN_ERR_UNSUPPORTED (-3)
#define BDBNN_ERR_WORKSPACE (-4)

/* Geometry of one conv2d call (square or rectangular kernels, symmetric zero padding). */
typedef struct bdbnn_conv_shape {
  int32_t N, H, W, Cin;     /* input  [N,H,W,Cin]  */
  int32_t Cout, kh, kw;     /* weight [Cout,Cin,kh,kw] */
  int32_t stride, pad;      /* same in h and w */
  int32_t Ho, Wo;           /* output [N,Ho,Wo,Cout]; must equal (H+2*pad-kh)/stride+1 etc. */
} bdbnn_conv_shape;

/* Library ABI version (major*1000 + minor). */
BDBNN_API int bdbnn_version(void);
/* Thread-local description of the last error returned on this thread ("" if none). */
BDBNN_API const char* bdbnn_last_error_string(void);
/* Developer aid: when device_buf != NULL (3*2048 int64), CTA (0,0,0) of the weight-gradient kernel records
 * (event id, clock64) pairs of its TMA producer warp (row 0: ring-slot wait begin / end) into it.  NULL
 * disables. */
BDBNN_API int bdbnn_debug_trace(long long* device_buf);
/* Which wgmma/TMA implicit-GEMM kernels can serve this shape: bitmask
 * BDBNN_TC_FWD | BDBNN_TC_DGRAD | BDBNN_TC_WGRAD (0 = none: the CUDA-core kernels do all three). */
#define BDBNN_TC_FWD 1
#define BDBNN_TC_DGRAD 2
#define BDBNN_TC_WGRAD 4
#define BDBNN_TC_FWD8 8   /* fp8 (e4m3 +-1) forward: bdbnn_binconv_fwd_tc8 */
#define BDBNN_TC_FWD_I16 16 /* forward can store the integer accumulator as int16: bdbnn_binconv_fwd_tc_i16 */
BDBNN_API int bdbnn_tc_supported(const bdbnn_conv_shape* s);

/* ---- activation sign/pack ---------------------------------------------------------------------
 * Replaces the activation binarisation inside the (absent) HardBinaryConv*.forward invoked at
 * train.py:492 / train.py:602 (SURVEY.md §8a a1-a3; spec in DESIGN.md §2).
 *   sign_bits[p*Cw+k] bit j = (x[p*C+32k+j] >= 0)           (forward operand, bit-exact)
 *   mask_bits[p*Cw+k] bit j = (|x[p*C+32k+j]| <= 1)         (STE mask saved for backward)
 *   xb_bf16 [p*C+c]        = +1.0/-1.0 in `fmt` (bf16 0x3F80/0xBF80, fp16 0x3C00/0xBC00); may be NULL
 * n_pix = N*H*W, Cw = ceil(C/32).  NaN inputs: sign bit 0 (-1), mask bit 0. */
BDBNN_API int bdbnn_act_pack(const float* x, int64_t n_pix, int32_t C, uint32_t* sign_bits,
                   uint32_t* mask_bits, uint16_t* xb_bf16, int32_t fmt, void* stream);

/* ---- weight sign/pack -------------------------------------------------------------------------
 * Replaces the weight binarisation of HardBinaryConv*.forward (same call sites).
 *   alpha[o]                 = mean_{c,r,s} |W[o,c,r,s]|                       (fp32)
 *   wsign_bits[(o*T+t)*Cw+k] bit j = (W[o,32k+j,t] >= 0),  T = kh*kw, t = r*kw+s
 *   wmask_bits[e/32] bit e%32      = (|W.flat[e]| <= 1)   in OIHW flat order  (STE mask)
 *   wf_bf16[(o*T+t)*Cin+c]   = sign(W[o,c,t]) as bf16              (fwd  B operand; may be NULL)
 *   wt_bf16[(c*T+t)*Cout+o]  = alpha[o]>0 ? sign(W[o,c,T-1-t]) : 0 (dgrad B operand; may be NULL)
 *   wf_fp8 [(o*T+t)*Cin+c]   = sign(W[o,c,t]) as e4m3 byte           (fwd_tc8 B operand; may be NULL)
 *   gscale[o] = alpha[o] > 0 ? alpha[o] : 1 ;  inv_gscale[o] = 1/gscale[o]   (may be NULL) */
BDBNN_API int bdbnn_weight_pack(const float* W, int32_t Cout, int32_t Cin, int32_t kh, int32_t kw,
                      float* alpha, uint32_t* wsign_bits, uint32_t* wmask_bits,
                      uint16_t* wf_bf16, uint16_t* wt_bf16, uint8_t* wf_fp8, float* gscale,
                      float* inv_gscale, int32_t fmt, void* stream);
/* The same packing for ALL binary convs of a network in two launches (one grid of sum(Cout) filter blocks, one
 * of transpose tiles) instead of two small launches per layer; host tables of `count` entries, per-layer pointers
 * exactly as bdbnn_weight_pack takes them (wf / wf8 entries may be NULL).  Every layer needs Cin*kh*kw % 32 == 0
 * (3x3 convs on multiples of 32 channels); taps = kh*kw. */
BDBNN_API int bdbnn_weight_pack_multi(int32_t count, const float* const* W_host, const int32_t* Cout_host,
                            const int32_t* Cin_host, const int32_t* taps_host, float* const* alpha_host,
                            uint32_t* const* wsign_host, uint32_t* const* wmask_host, uint16_t* const* wf_host,
                            uint16_t* const* wt_host, uint8_t* const* wf8_host, float* const* gscale_host,
                            float* const* inv_gscale_host, int32_t fmt, void* stream);
/* sign bits -> fp8 e4m3 +-1 bytes [n_pix][C] (0x38 = +1, 0xB8 = -1), C % 32 == 0: operand of fwd_tc8. */
BDBNN_API int bdbnn_bits_to_fp8(const uint32_t* sign_bits, int64_t n_pix, int32_t C, uint8_t* xb_fp8, void* stream);

/* ---- EDE backward factor: g[i] *= k*t*(1 - tanh(t*v[i])^2), k,t 1-element DEVICE floats ---------
 * The soft-sign derivative the reference's --ede recipe uses instead of the hard-tanh indicator
 * (train.py:409-415 assigns module.k/.t each epoch; schedule utils/utils.py:8-14).  Applied to
 * gx (v = x) and gW (v = W) after the dgrad/wgrad kernels ran with all-ones masks. */
BDBNN_API int bdbnn_ede_scale(float* g, const float* v, const float* k, const float* t, int64_t n, void* stream);

/* ---- binary conv forward, XNOR-popcount (bit-serial, CUDA cores) -------------------------------
 * y[n,ho,wo,o] = alpha[o] * sum_{valid taps} (Cin - 2*popc(xbits ^ wbits)); zero padding
 * contributes 0.  Replaces F.conv2d on +-1 fp32 tensors inside HardBinaryConv*.forward
 * (train.py:492,602).  Integer part exact. */
BDBNN_API int bdbnn_binconv_fwd_xnor(const uint32_t* sign_bits, const uint32_t* wsign_bits,
                           const float* alpha, float* y, const bdbnn_conv_shape* s, void* stream);

/* ---- binary conv forward, wgmma implicit GEMM on +-1 bf16 operands (exact, fp32 accumulate) --
 * Same result as bdbnn_binconv_fwd_xnor.  Requires bdbnn_tc_supported(s).
 * bn_sums / bn_ymax (both or neither; also on fwd_tc8 and stem_conv_fwd): if non-NULL the kernel's
 * epilogue also accumulates the BatchNorm batch statistics of y — bn_sums = double[2*Cout] (sum y, then
 * sum y^2 per channel), bn_ymax = u32[Cout] (bits of max|y|) — so that bdbnn_bn_fwd / bdbnn_bn_pool_fwd can
 * be called with stats_ready = 1 and skip their own pass over y.  The buffers are zeroed here. */
BDBNN_API int bdbnn_binconv_fwd_tc(const uint16_t* xb_bf16, const uint16_t* wf_bf16, int32_t fmt,
                         const float* alpha, float* y, const bdbnn_conv_shape* s, double* bn_sums,
                         uint32_t* bn_ymax, void* stream);

/* Same forward on fp8 (e4m3) +-1 operands: half the operand bytes and twice the K per MMA of the
 * 16-bit kernel; still exact.  Requires bdbnn_tc_supported(s) & BDBNN_TC_FWD8. */
BDBNN_API int bdbnn_binconv_fwd_tc8(const uint8_t* xb_fp8, const uint8_t* wf_fp8, const float* alpha, float* y,
                          const bdbnn_conv_shape* s, double* bn_sums, uint32_t* bn_ymax, void* stream);

/* Forward with the result stored as the EXACT INTEGER accumulator, int16 NHWC [N,Ho,Wo,Cout]:
 * y = alpha[o] * y_int[o], |y_int| <= kh*kw*Cin <= 32767 — lossless, half the bytes of the fp32 y that the
 * fused BatchNorm units (bdbnn_bn_fwd_i16 / bdbnn_bn_bwd_pack_i16) read once in the forward and twice in the
 * backward.  fmt = BDBNN_FMT_FP16 / BDBNN_FMT_BF16 (16-bit +-1 operands) or -1 (fp8 e4m3 operands, needs
 * BDBNN_TC_FWD8).  The statistics (bn_sums / bn_ymax) are those of y = alpha * y_int, as in fwd_tc.
 * Requires bdbnn_tc_supported(s) & BDBNN_TC_FWD_I16 (GEMMs eligible in bdbnn_debug_conv_plan only). */
BDBNN_API int bdbnn_binconv_fwd_tc_i16(const void* xb, const void* wf, int32_t fmt, const float* alpha,
                             int16_t* y_int, const bdbnn_conv_shape* s, double* bn_sums, uint32_t* bn_ymax,
                             void* stream);

/* ---- backward: data gradient -------------------------------------------------------------------
 * gx[n,h,w,c] = mask(n,h,w,c) * sum_{t,o} gy[n,ho,wo,o] * alpha[o] * sign(W[o,c,t])
 * Replaces cuDNN dgrad + the STE mask multiply that autograd runs under loss.backward()
 * (train.py:528, train.py:650).  Generic kernel: fp32 CUDA cores, any shape. */
BDBNN_API int bdbnn_binconv_dgrad(const float* gy, const uint32_t* wsign_bits, const float* alpha,
                        const uint32_t* mask_bits, float* gx, const bdbnn_conv_shape* s,
                        void* stream);

/* ---- backward: weight gradient -----------------------------------------------------------------
 * gW[o,c,r,s] = wmask(o,c,r,s) * sum_{n,ho,wo} gy[n,ho,wo,o] * sign(x)[n,ho*st+r-p,wo*st+s-p,c]
 * (Bi-Real STE: gradient w.r.t. the scaled binary weight passed straight through where |W|<=1.)
 * gW is OVERWRITTEN, OIHW fp32.  Generic kernel: fp32 CUDA cores + atomics, any shape. */
BDBNN_API int bdbnn_binconv_wgrad(const float* gy, const uint32_t* sign_bits, const uint32_t* wmask_bits,
                        float* gW, const bdbnn_conv_shape* s, void* stream);

/* ---- backward on tensor cores (wgmma, 16-bit operands, fp32 accumulate) -----------------------
 * grad_pack: v = gy[p*Cout+o] * gscale[o], written per `mode` (BDBNN_GRAD_*):
 *              BF16   gys[p*Cout+o]             = bf16_rn(v)
 *              BF16X2 gys[p*2Cout+o] = hi = bf16_rn(v), gys[p*2Cout+Cout+o] = bf16_rn(v - hi)
 *              FP16S  gys[p*Cout+o]             = fp16_rn(v * 2^e), e = 13 - floor(log2 max|v|); the max is
 *                     reduced into the device word amax_bits (float bits) by the same call
 *            gys is shared by dgrad_tc (K-major) and wgrad_tc (MN-major).
 * dgrad_tc : gx = mask * 2^-e * conv_transpose(gys, wt) (+ add)      (sign-only weights, exact; `add`,
 *            if non-NULL, is an fp32 tensor shaped like gx — the shortcut branch's gradient — summed in
 *            the epilogue; add == gx accumulates in place: with stride > 1 only the positions a tap reaches
 *            are touched, which is how the strided 1x1 shortcut adds its gradient to the main branch's)
 * wgrad_tc : gW = wmask * inv_gscale[o] * 2^-e * sum_pix gys[pix,o]*xb[pix',c]
 * The +-1 operands (xb, wt) must be in the format matching the mode: fp16 for FP16S, bf16 otherwise.
 * wgrad_tc needs a workspace of bdbnn_wgrad_tc_workspace_bytes(s) bytes (split-K partials).
 * grad_mode / amax_bits must be the values grad_pack was called with (amax_bits may be NULL unless FP16S). */
BDBNN_API int bdbnn_grad_pack(const float* gy, const float* gscale, int64_t n_pix, int32_t Cout,
                    int32_t mode, uint32_t* amax_bits, uint16_t* gys, void* stream);
BDBNN_API int bdbnn_binconv_dgrad_tc(const uint16_t* gys, int32_t grad_mode, const uint32_t* amax_bits,
                           const uint16_t* wt, const uint32_t* mask_bits, const float* add, float* gx,
                           const bdbnn_conv_shape* s, void* stream);
BDBNN_API size_t bdbnn_wgrad_tc_workspace_bytes(const bdbnn_conv_shape* s);
/* Host-only: the forward/dgrad kernel's tiling for a shape (mode 0 = forward, 1 = first dgrad phase,
 * 2 = fp8 forward).  out[12] = {planned (0 = not eligible for the int16 result / fused dgrad statistics),
 * halo mode (0), M tiles per CTA (1), accumulator buffers (1), N tile, N tiles, M tiles, ring stages,
 * dynamic smem bytes, grid, stage bytes, patch bytes (0)}.  Makes no CUDA call. */
BDBNN_API int bdbnn_debug_conv_plan(const bdbnn_conv_shape* s, int32_t mode, int32_t grad_halves, int32_t* out,
                          int32_t n_out);
/* Host-only: the tiling bdbnn_binconv_wgrad_tc would use, for tests.  out[12] = {supported, ksplit, ks_cap,
 * m_groups, n_tiles, dynamic smem bytes, M tiles per CTA, N tile, unit width, halo mode, K rows per stage,
 * ring stages}.  Makes no CUDA call. */
BDBNN_API int bdbnn_debug_wgrad_plan(const bdbnn_conv_shape* s, int32_t grad_halves, int32_t* out, int32_t n_out);
BDBNN_API int bdbnn_binconv_wgrad_tc(const uint16_t* gys, int32_t grad_mode, const uint32_t* amax_bits,
                           const uint16_t* xb, const uint32_t* wmask_bits, const float* inv_gscale,
                           float* gW, const bdbnn_conv_shape* s, void* workspace, size_t workspace_bytes,
                           void* stream);

/* ---- kurtosis regulariser, multi-tensor --------------------------------------------------------
 * Replaces KurtosisWeight.kurtosis_calc (kurtosis.py:23-39) called per hooked layer at
 * train.py:501-504 / 622-625, and the scalar reduction at train.py:505-512.
 * For each tensor l<L (L <= BDBNN_MAX_TENSORS): mu=mean(w), s=std(w) UNBIASED (n-1),
 * K=mean(((w-mu)/s)^4), loss=(K-target)^2.
 *   w_ptrs_host / numel_host / targets_host : HOST arrays of length L
 *   moments  : device double[L*8] scratch that the backward reads (mu, s, K, mean z^3, ...)
 *   kurt_out, loss_out : device float[L]
 * bwd: grad_l[j] (+)= gout[l] * 2(K-T) * 4/(n s) * (z^3 - mean(z^3) - z K n/(n-1));
 *      gout is a DEVICE float[L]; accumulate!=0 adds into grad, else overwrites. */
#define BDBNN_MAX_TENSORS 64
BDBNN_API int bdbnn_kurtosis_multi_fwd(const float* const* w_ptrs_host, const int64_t* numel_host,
                             const float* targets_host, int32_t L, double* moments,
                             float* kurt_out, float* loss_out, void* stream);
BDBNN_API int bdbnn_kurtosis_multi_bwd(const float* const* w_ptrs_host, const int64_t* numel_host,
                             const float* targets_host, int32_t L, const double* moments,
                             const float* gout, float* const* grad_ptrs_host, int32_t accumulate,
                             void* stream);

/* ---- KD logits loss (DistributionLoss.forward, utils/KD_loss.py:16-43; train.py:612) -----------
 * loss = -(1/N) sum_n sum_c softmax(t)[n,c] * log_softmax(s)[n,c]
 * grad_s[n,c] = (softmax(s) - softmax(t))[n,c] / N          (written when grad_s != NULL)
 * row_ws: device float[N] scratch.  s,t row-major [N,C] fp32. */
BDBNN_API int bdbnn_kd_logits_fwd_bwd(const float* s, const float* t, int32_t N, int32_t C, float* row_ws,
                            float* loss_out, float* grad_s, void* stream);

/* ---- KD per-layer weight loss (DistributionLoss_layer.forward, utils/KD_loss.py:52-67) ---------
 * loss = sum_l mean_l( exp(Wt_l) * (Wt_l - Ws_l) )   == sum_l KLDivLoss(log_target=True)(Ws,Wt)
 * bwd : gWs_l[j] (+)= -gout[0] * exp(Wt_l[j]) / numel_l
 * partial: device double[L] scratch. */
BDBNN_API int bdbnn_kd_layer_multi_fwd(const float* const* ws_ptrs_host, const float* const* wt_ptrs_host,
                             const int64_t* numel_host, int32_t L, double* partial,
                             float* loss_out, void* stream);
BDBNN_API int bdbnn_kd_layer_multi_bwd(const float* const* wt_ptrs_host, const int64_t* numel_host,
                             int32_t L, const float* gout, float* const* grad_ptrs_host,
                             int32_t accumulate, void* stream);

/* ---- BatchNorm(train) + residual add (+ next conv's sign/pack) around the binary conv --------------
 * Caller side of the path (SURVEY.md §8f rank 1).  y = conv output fp32 NHWC [n_pix][C], C % 4 == 0.
 * bn_fwd : mean/var over n_pix per channel (biased var, eps), mean/invstd saved for backward,
 *          running_mean/var (may be NULL) updated with `momentum` (unbiased var), then
 *          z = gamma*(y-mean)*invstd + beta (+ residual if non-NULL).
 *          If sign_bits != NULL (needs C % 32 == 0) also emits what bdbnn_act_pack(z) would:
 *          sign_bits, mask_bits, xb (format fmt) and, if xb_fp8 != NULL, the e4m3 +-1 bytes — the next
 *          binary conv then skips its own pack.
 *          ymax_bits[C] receives max|y| per channel (float bits) for the backward's FP16S bound.
 *          Scratch: sums_ws double[2C], ab_ws float[2C].
 * bn_bwd_pack : from gz (grad of z) and the saved y/mean/invstd computes dgamma, dbeta and writes
 *          gys = packed(gy * gscale[c]) with gy = gamma*invstd*(gz - mean(gz) - yhat*mean(gz*yhat)),
 *          in the layout bdbnn_grad_pack produces for `grad_mode` (FP16S scale from an upper bound of
 *          max|gy*gscale|, written to amax_bits).  The residual branch's gradient is gz itself.
 *          Scratch: sums_ws double[2C], gmax_bits u32[C], consts_ws float[4C]. */
BDBNN_API int bdbnn_bn_fwd(const float* y, const float* residual, const float* gamma, const float* beta,
                 int64_t n_pix, int32_t C, float eps, float momentum, float* running_mean,
                 float* running_var, double* sums_ws, uint32_t* ymax_bits, float* mean, float* invstd,
                 float* ab_ws, float* z, uint32_t* sign_bits, uint32_t* mask_bits, uint16_t* xb,
                 uint8_t* xb_fp8, int32_t fmt, int32_t stats_ready, void* stream);
BDBNN_API int bdbnn_bn_bwd_pack(const float* gz, const float* y, const float* mean, const float* invstd,
                      const float* gamma, const float* gscale, const uint32_t* ymax_bits, int64_t n_pix,
                      int32_t C, int32_t grad_mode, double* sums_ws, uint32_t* gmax_bits, float* consts_ws,
                      float* dgamma, float* dbeta, uint32_t* amax_bits, uint16_t* gys, void* stream);

/* The same two passes on the int16 conv result of bdbnn_binconv_fwd_tc_i16 (y = alpha[c] * y_int): 2 instead of
 * 4 bytes per element for the one forward and the two backward reads of y.  The statistics always come from the
 * conv epilogue (stats_ready is implied). */
BDBNN_API int bdbnn_bn_fwd_i16(const int16_t* y_int, const float* alpha, const float* residual, const float* gamma,
                     const float* beta, int64_t n_pix, int32_t C, float eps, float momentum, float* running_mean,
                     float* running_var, double* sums_ws, uint32_t* ymax_bits, float* mean, float* invstd,
                     float* ab_ws, float* z, uint32_t* sign_bits, uint32_t* mask_bits, uint16_t* xb,
                     uint8_t* xb_fp8, int32_t fmt, void* stream);
BDBNN_API int bdbnn_bn_bwd_pack_i16(const float* gz, const int16_t* y_int, const float* alpha, const float* mean,
                          const float* invstd, const float* gamma, const float* gscale, const uint32_t* ymax_bits,
                          int64_t n_pix, int32_t C, int32_t grad_mode, double* sums_ws, uint32_t* gmax_bits,
                          float* consts_ws, float* dgamma, float* dbeta, uint32_t* amax_bits, uint16_t* gys,
                          int32_t stats_ready, void* stream);
/* bdbnn_bn_bwd_pack_i16(stats_ready = 1): sums_ws (sum gz | sum gz*yhat) and gmax_bits were already accumulated by
 * the kernel that PRODUCED gz — bdbnn_binconv_dgrad_tc_stats, the data-gradient kernel of the next unit, whose
 * result (dgrad + shortcut gradient) is this unit's gz: the separate reduction pass over gz and y is skipped.
 * dgrad_tc_stats = bdbnn_binconv_dgrad_tc (stride 1, eligible GEMMs, Cin <= 512) + those statistics of the
 * producing unit: prod_y_int int16 [N,H,W,Cin], prod_alpha / prod_mean / prod_invstd float[Cin];
 * prod_sums double[2*Cin] and prod_gmax u32[Cin] are zeroed here. */
BDBNN_API int bdbnn_binconv_dgrad_tc_stats(const uint16_t* gys_bf16, int32_t grad_mode, const uint32_t* amax_bits,
                                 const uint16_t* wt_bf16, const uint32_t* mask_bits, const float* add, float* gx,
                                 const bdbnn_conv_shape* s, const int16_t* prod_y_int, const float* prod_alpha,
                                 const float* prod_mean, const float* prod_invstd, double* prod_sums,
                                 uint32_t* prod_gmax, void* stream);

/* ---- stem: BatchNorm(train) + MaxPool fused (the BN output is never written) -----------------------
 * bn_pool_fwd: y fp32 NHWC [N,H,W,C] (stem conv output) -> z = maxpool_k,s,p(gamma*(y-mean)*invstd+beta)
 *              [N,Ho,Wo,C], idx = winning tap per output element (1 byte), y_sel = y at the winner;
 *              optional packs of z as in bdbnn_bn_fwd.  Scratch as bdbnn_bn_fwd.
 * bn_pool_bwd: g_pool = grad of z -> gy = grad of y [N,H,W,C] (BN backward with the pooled gradient
 *              scattered to the winners), dgamma, dbeta.  `ones` = float[C] of 1.0 (unit gradient scale);
 *              scratch: sums_ws double[2C], gmax_bits u32[C], consts_ws float[4C], amax_scratch u32[1].
 *              If `gys` is non-NULL the gradient is written ONLY as gys = fp16(gy * 2^e) [N,H,W,C] with
 *              amax_scratch holding the bound e was derived from (FP16S operand of bdbnn_stem_conv_wgrad);
 *              gy may then be NULL. */
BDBNN_API int bdbnn_bn_pool_fwd(const float* y, const float* gamma, const float* beta, int32_t N, int32_t H, int32_t W,
                      int32_t C, int32_t k, int32_t stride, int32_t pad, int32_t Ho, int32_t Wo, float eps,
                      float momentum, float* running_mean, float* running_var, double* sums_ws,
                      uint32_t* ymax_bits, float* mean, float* invstd, float* ab_ws, float* z, float* y_sel,
                      uint8_t* idx, uint32_t* sign_bits, uint32_t* mask_bits, uint16_t* xb, uint8_t* xb_fp8,
                      int32_t fmt, int32_t stats_ready, void* stream);
BDBNN_API int bdbnn_bn_pool_bwd(const float* g_pool, const uint8_t* idx, const float* y, const float* y_sel,
                      const float* mean, const float* invstd, const float* gamma, const float* ones,
                      const uint32_t* ymax_bits, int32_t N, int32_t H, int32_t W, int32_t C, int32_t k,
                      int32_t stride, int32_t pad, int32_t Ho, int32_t Wo, double* sums_ws, uint32_t* gmax_bits,
                      float* consts_ws, float* dgamma, float* dbeta, uint32_t* amax_scratch, float* gy,
                      uint16_t* gys, void* stream);

/* ---- NHWC max-pool (stem of the ImageNet shells; torch.nn.MaxPool2d semantics) --------------------
 * Caller side of the path (SURVEY.md §8f: the ops either side of the binary convs).  x,y,gy,gx fp32
 * NHWC, C % 4 == 0; idx = winning tap (r*k+s) per output element, one byte each [N,Ho,Wo,C].
 * First maximum in scan order wins, NaN propagates; backward is a gather (deterministic, no atomics). */
BDBNN_API int bdbnn_maxpool_fwd(const float* x, float* y, uint8_t* idx, int32_t N, int32_t H, int32_t W,
                      int32_t C, int32_t k, int32_t stride, int32_t pad, int32_t Ho, int32_t Wo,
                      void* stream);
BDBNN_API int bdbnn_maxpool_bwd(const float* gy, const uint8_t* idx, float* gx, int32_t N, int32_t H,
                      int32_t W, int32_t C, int32_t k, int32_t stride, int32_t pad, int32_t Ho, int32_t Wo,
                      void* stream);

/* ---- stem convolution: 7x7 / stride 2 / pad 3, 3 -> 64 channels, fp32 in / fp32 out, on wgmma --------
 * Replaces the fp32 nn.Conv2d `conv1` of the torchvision-style ResNet the reference trains
 * (model(images), train.py:492,602; its weight gradient under loss.backward(), train.py:528,650), which
 * cuDNN runs on TF32 tensor cores.  Operands here are fp16 after a per-call power-of-two scale
 * (11-bit significands like TF32, fp32 accumulation); see bdbnn_b200/csrc/stem.cu.
 *   stem_pack      : x (any dense NCHW / channels_last strides, in elements) -> xw fp16 [N][H+6][WP][4]
 *                    (bdbnn_stem_xw_bytes), x_amax_bits (1 word), wf fp16 [64][7][32], alpha[64]
 *   stem_conv_fwd  : y[N][Ho][Wo][64] fp32 NHWC = conv(x, W)
 *   stem_conv_wgrad: gW[64][3][7][7] from gys = fp16(gy * 2^e) [N][Ho][Wo][64] (bdbnn_grad_pack, FP16S,
 *                    gscale = 1) and the saved xw; workspace of bdbnn_stem_wgrad_workspace_bytes.
 * Supported when (W-1)/2 + 1 <= 128 (bdbnn_stem_supported). */
BDBNN_API int bdbnn_stem_supported(int32_t N, int32_t H, int32_t W);
BDBNN_API size_t bdbnn_stem_xw_bytes(int32_t N, int32_t H, int32_t W);
BDBNN_API size_t bdbnn_stem_wgrad_workspace_bytes(int32_t N, int32_t H, int32_t W);
BDBNN_API int bdbnn_stem_pack(const float* x, int32_t N, int32_t H, int32_t W, int64_t sN, int64_t sC, int64_t sH,
                    int64_t sW, const float* weight, uint16_t* xw, uint32_t* x_amax_bits, uint16_t* wf,
                    float* alpha, void* stream);
BDBNN_API int bdbnn_stem_conv_fwd(const uint16_t* xw, const uint16_t* wf, const float* alpha, float* y, int32_t N,
                        int32_t H, int32_t W, double* bn_sums, uint32_t* bn_ymax, void* stream);
BDBNN_API int bdbnn_stem_conv_wgrad(const uint16_t* gys, const uint32_t* g_amax_bits, const uint16_t* xw,
                          const uint32_t* x_amax_bits, float* gW, int32_t N, int32_t H, int32_t W,
                          void* workspace, size_t workspace_bytes, void* stream);

/* ---- step pieces either side of the path (SURVEY.md section 8f ranks 3, 4) -----------------------------
 * ce_topk_fwd_bwd : nn.CrossEntropyLoss()(logits, target) (train.py:493, 614), its gradient
 *                   (softmax - onehot)/N (written when grad_logits != NULL), accuracy(output, target,
 *                   topk=(k1, k2)) in percent (train.py:518, utils/utils.py:72-85) and, when `meters` is
 *                   non-NULL, the running AverageMeter sums {loss*N, acc_k1*N, acc_k2*N, N} as device
 *                   doubles (train.py:520-524 without the .item() syncs).  Two launches, nothing read
 *                   back.  logits fp32 [N,C] row-major, target int64 [N]; scratch row_loss_ws float[N],
 *                   row_rank_ws int32[N]; loss_out float[1], acc_out float[2].
 * optim_adam_multi: torch.optim.Adam step (train.py:331-335: betas, eps, L2 weight decay only on the
 *                   conv-weight group) for `count` tensors in one launch per 48 tensors; p/g/m/v share
 *                   one dense layout per tensor; `step` is the 1-based step count for the bias
 *                   corrections; every gradient is multiplied by grad_scale first (1/world after the
 *                   data-parallel all-reduce SUM).  Pointer / size / hyper-parameter tables are HOST arrays.
 * optim_sgd_multi : torch.optim.SGD step with momentum (train.py:319-321; dampening 0, no nesterov);
 *                   first_step != 0 initialises the momentum buffers with the gradient. */
BDBNN_API int bdbnn_ce_topk_fwd_bwd(const float* logits, const int64_t* target, int32_t N, int32_t C, int32_t k1,
                          int32_t k2, float* row_loss_ws, int32_t* row_rank_ws, float* loss_out,
                          float* acc_out, float* grad_logits, double* meters, void* stream);
BDBNN_API int bdbnn_optim_adam_multi(float* const* params_host, const float* const* grads_host,
                           float* const* exp_avg_host, float* const* exp_avg_sq_host,
                           const int64_t* numel_host, const float* weight_decay_host, const float* lr_host,
                           int32_t count, float beta1, float beta2, float eps, int64_t step,
                           float grad_scale, void* stream);
BDBNN_API int bdbnn_optim_sgd_multi(float* const* params_host, const float* const* grads_host,
                          float* const* momentum_buf_host, const int64_t* numel_host,
                          const float* weight_decay_host, const float* lr_host, int32_t count, float momentum,
                          int32_t first_step, float grad_scale, void* stream);
/* CUDA-graph variants (the whole step of train.py:492-529 captured once and replayed): everything that changes
 * from step to step is read from DEVICE memory so a captured launch stays valid —
 * step_dev  float[1], the 1-based Adam step count (bdbnn_optim_step_inc adds 1; launch it before the update);
 * lr_dev    float[count], one learning rate per tensor in table order (the LR scheduler of train.py:336 / 322
 *           rewrites it between replays).  SGD: momentum buffers must exist and start at zero (first step then
 *           equals torch's buf = g). */
BDBNN_API int bdbnn_optim_step_inc(float* step_dev, void* stream);
BDBNN_API int bdbnn_optim_adam_multi_graph(float* const* params_host, const float* const* grads_host,
                                 float* const* exp_avg_host, float* const* exp_avg_sq_host,
                                 const int64_t* numel_host, const float* weight_decay_host, int32_t count,
                                 float beta1, float beta2, float eps, const float* step_dev, const float* lr_dev,
                                 float grad_scale, void* stream);
BDBNN_API int bdbnn_optim_sgd_multi_graph(float* const* params_host, const float* const* grads_host,
                                float* const* momentum_buf_host, const int64_t* numel_host,
                                const float* weight_decay_host, int32_t count, float momentum,
                                const float* lr_dev, float grad_scale, void* stream);

/* ---- fp32 1x1 shortcut convolution (`downsample` of the ResNet shells) on the wgmma kernels -------------
 * Packing only (bdbnn_b200/csrc/real_conv.cu): xh = fp16(x[:, ::stride, ::stride, :] * 2^ex) dense NHWC
 * [N,Ho,Wo,Cin], wf = fp16(W * 2^ew) [Cout][Cin], wt = its transpose [Cin][Cout], and the scale vectors
 * alpha[o] = 2^-ew 2^-ex, gscale[o] = 2^-ew, inv_gscale[o] = 2^ew 2^-ex.  The convolution itself is
 * bdbnn_binconv_fwd_tc / _dgrad_tc / _wgrad_tc run as a 1x1 stride-1 conv over xh with these vectors and
 * all-ones STE masks (TF32-class operands, fp32 accumulate; replaces cuDNN's TF32 kernels under
 * model(images) / loss.backward()).  x fp32 NHWC, weight fp32 [Cout][Cin] (= [Cout,Cin,1,1]);
 * x_amax_bits: TWO words of scratch ([0] = bits of max|x| over the samples, [1] = of max|W|). */
BDBNN_API int bdbnn_real_conv_pack(const float* x, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t stride,
                         const float* weight, int32_t Cout, uint16_t* xh, uint32_t* x_amax_bits, uint16_t* wf,
                         uint16_t* wt, float* alpha, float* gscale, float* inv_gscale, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BDBNN_H_ */
