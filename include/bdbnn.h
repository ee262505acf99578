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
#define BDBNN_TC_EVAL 32    /* eval-mode forward of a grouped conv: bdbnn_real_gconv_supported only */
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
/* The inverse for the forward operands of a loaded 1-bit model (bdbnn_b200/export.py): per layer, the sign words
 * wsign_bits [Cout][T][ceil(Cin/32)] (bit j of word k = 1 for +1, as bdbnn_weight_pack writes them) become
 *   wf [(o*T+t)*Cin+c] = +-1 in format fmt (fp16 0x3C00/0xBC00, bf16 0x3F80/0xBF80)   or
 *   wf8[(o*T+t)*Cin+c] = +-1 as e4m3 byte (0x38 / 0xB8),
 * exactly one of wf_host[l] / wf8_host[l] non-NULL; byte-identical to bdbnn_weight_pack's wf / wf8 of a weight with
 * those signs.  Any Cin (also the 16-channel convs bdbnn_weight_pack_multi does not take); taps = kh*kw.  One launch
 * per 32 layers (one grid of sum(Cout) filter blocks). */
BDBNN_API int bdbnn_weight_unpack_multi(int32_t count, const uint32_t* const* wsign_host, const int32_t* Cout_host,
                              const int32_t* Cin_host, const int32_t* taps_host, uint16_t* const* wf_host,
                              uint8_t* const* wf8_host, int32_t fmt, void* stream);
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

/* ---- eval-mode forward: conv + BatchNorm(eval) + residual in one epilogue ------------------------------------
 * Replaces the module chain model.eval() under torch.no_grad() runs per binary conv in validate()
 * (train.py:677-714): act_pack, weight pack, conv, nn.BatchNorm2d(eval), residual add.
 * bn_eval_fold : per channel, in fp64 with every step rounded separately (no FMA),
 *                  k = gamma / sqrt(running_var + eps)    (eps: this fp32 value widened to double)
 *                  scale[c] = float(alpha[c] * k),  shift[c] = float(beta - running_mean * k)
 *                alpha may be NULL (= 1).  One launch, no scratch.
 * binconv_fwd_tc_eval : the forward implicit GEMM of bdbnn_binconv_fwd_tc (same operands, tiling and
 *                BDBNN_TC_CLUSTER behaviour) with, from the fp32 accumulator acc, rounding each step (no FMA):
 *                  z = fp32(fp32(acc * scale[o]) + shift[o]);  z = fp32(z + residual)  if residual != NULL
 *                z fp32 NHWC [N,Ho,Wo,Cout]; residual (may be NULL) has z's shape and must not alias it.
 *                Optional +-1 copies of z for the next conv (sign(v) = +1 iff v >= 0: -0.0 -> +1, NaN -> -1):
 *                zb  16-bit in format fmt (fp16 0x3C00/0xBC00, bf16 0x3F80/0xBF80), needs fmt >= 0;
 *                zb8 fp8 e4m3 bytes (0x38 / 0xB8); both NHWC like z, NULL = not written.
 *                fmt = BDBNN_FMT_FP16 / BDBNN_FMT_BF16 (16-bit operands) or -1 (fp8 operands, needs BDBNN_TC_FWD8).
 *                Writes no statistics and allocates nothing.  Requires bdbnn_tc_supported(s) & BDBNN_TC_FWD.
 *                The 1x1 `downsample` in eval: bdbnn_real_conv_pack, then this call as a 1x1 stride-1 conv over
 *                xh (fmt FP16) with scale folded from the pack's alpha, no residual and no copies.
 * stem_conv_fwd_eval : the stem GEMM of bdbnn_stem_conv_fwd with the same epilogue (no residual, no copies);
 *                scale is folded from bdbnn_stem_pack's alpha.  The max-pool after it is bdbnn_maxpool_fwd. */
BDBNN_API int bdbnn_bn_eval_fold(const float* alpha, const float* gamma, const float* beta, const float* running_mean,
                       const float* running_var, int32_t C, float eps, float* scale, float* shift, void* stream);
BDBNN_API int bdbnn_binconv_fwd_tc_eval(const void* xb, const void* wf, int32_t fmt, const float* scale,
                              const float* shift, const float* residual, float* z, uint16_t* zb, uint8_t* zb8,
                              const bdbnn_conv_shape* s, void* stream);

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
 * 2 = fp8 forward, 3 = eval forward, 4 = fp8 eval forward).  out[12] = {planned (modes 0-2: 0 = not eligible for the
 * int16 result / fused dgrad statistics; modes 3-4: 0 = the eval kernel cannot run the shape),
 * halo mode (0), M tiles per CTA (1), accumulator buffers (1), N tile, N tiles, M tiles, ring stages,
 * dynamic smem bytes, grid, stage bytes, patch bytes (0)}; with n_out >= 14 also out[12], out[13] = thread-block
 * cluster CTAs along M (sharing the weight box) and along N (sharing the activation box); 1 unless
 * BDBNN_TC_CLUSTER=1, and 1 on a grid side that is odd.  Makes no CUDA call. */
BDBNN_API int bdbnn_debug_conv_plan(const bdbnn_conv_shape* s, int32_t mode, int32_t grad_halves, int32_t* out,
                          int32_t n_out);
/* CTAs of the forward (mode 0) / dgrad (mode 1) / eval forward (mode 2) / eval forward with the option-A residual of
 * the *_pad_shortcut entry points (mode 3) / eval forward with the Hardtanh epilogue of bdbnn_real_conv_fwd_eval
 * (mode 5, BDBNN_FMT_FP16 only; 4 is not a mode) tensor-core kernel that fit on one SM of the current device, for
 * operand format fmt (BDBNN_FMT_FP16 / BDBNN_FMT_BF16, -1 = fp8: modes 0 and 2 only), N tile bn (16/32/64/128) and
 * `smem` bytes of dynamic shared memory (bdbnn_debug_conv_plan out[8]), from the CUDA occupancy calculator.  Needs a
 * CUDA device; sets that kernel's maximum dynamic shared memory attribute to `smem` (every launch sets it again). */
BDBNN_API int bdbnn_debug_tc_conv_ctas_per_sm(int32_t mode, int32_t fmt, int32_t bn, int32_t smem, int32_t* ctas);
/* Host-only: the tiling bdbnn_binconv_wgrad_tc would use, for tests.  out[12] = {supported, ksplit, ks_cap,
 * m_groups, n_tiles, dynamic smem bytes, M tiles per CTA, N tile, unit width, 0, K rows per stage,
 * ring stages}.  With n_out >= 16 also out[12..15] = {operand mode (0 one box per tap, 1 one patch per channel
 * chunk and filter column), patch width (0 in box mode), patches per stage (0 in box mode), L2->shared-memory operand
 * KiB of the launch}; with n_out >= 18 also out[16] = the operand KiB of the box-mode plan of the same shape and
 * out[17] = the longest fp32 accumulation chain of the launch in output pixels.  Makes no CUDA call. */
BDBNN_API int bdbnn_debug_wgrad_plan(const bdbnn_conv_shape* s, int32_t grad_halves, int32_t* out, int32_t n_out);
BDBNN_API int bdbnn_binconv_wgrad_tc(const uint16_t* gys, int32_t grad_mode, const uint32_t* amax_bits,
                           const uint16_t* xb, const uint32_t* wmask_bits, const float* inv_gscale,
                           float* gW, const bdbnn_conv_shape* s, void* workspace, size_t workspace_bytes,
                           void* stream);

/* ---- kurtosis regulariser, multi-tensor --------------------------------------------------------
 * Replaces KurtosisWeight.kurtosis_calc (kurtosis.py:23-39) called per hooked layer at
 * train.py:501-504 / 622-625, and the scalar reduction at train.py:505-512.
 * For each tensor l<L (any L >= 0): mu=mean(w), s=std(w) UNBIASED (n-1),
 * K=mean(((w-mu)/s)^4), loss=(K-target)^2.
 * The multi-tensor loss calls launch their kernels once per BDBNN_MAX_TENSORS tensors (one kernel-parameter
 * table each); with L <= BDBNN_MAX_TENSORS that is one set of launches.
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

/* ---- binary-weight statistics for the training log (DESIGN.md §4w) ----------------------------
 * Both take L >= 0 layers, launched once per BDBNN_MAX_TENSORS of them; the pointer / numel / Cout arrays are HOST
 * arrays of length L, each weight a dense fp32 tensor whose filters (dim 0) are contiguous runs of numel/Cout
 * elements (NCHW or channels_last).
 * sign_flips: the sign bits of each weight (bit 1 = -1: v < 0 or NaN; -0 is +1), packed 32 per uint32 word into
 *   bits[l] (device, ceil(numel/32) words, tail bits 0).  init != 0 writes the bits and counts nothing (flips and
 *   steps may be NULL).  Otherwise flips[l] (device uint64) += popcount(new bits ^ stored bits), the new bits are
 *   stored, and steps[0] (device uint64, may be NULL) += 1.  Allocates nothing and never synchronises, so it can be
 *   captured in a CUDA graph; the counts are integers, the same in every run.
 * weight_stats: one block per (layer, filter), alpha_o = mean|W_o| in fp64.  Per layer l:
 *   stats_out[l*3 + 0] = #(|W| <= 1) / numel,  [1] = mean_o alpha_o,
 *   [2] = sum (W - alpha_o sign W)^2 / sum W^2 (0 when sum W^2 == 0);
 *   hist_out[l*68 + c] (uint64): c < 64 counts q = fp32(W / alpha_o) with floor(8q) + 32 == c (q in [-4, 4)),
 *   64 q < -4, 65 q >= 4, 66 weights of filters with alpha_o == 0, 67 q NaN.
 *   filter_sums (double[F*4]) and filter_hist (uint32[F*68]) are device scratch, F = sum of Cout.  Filters are
 *   added in filter order, so every output has the same bits in every run. */
#define BDBNN_WSTAT_VALUES 3
#define BDBNN_WSTAT_HIST 68
BDBNN_API int bdbnn_sign_flips_multi(const float* const* w_ptrs_host, const int64_t* numel_host,
                                     uint32_t* const* bits_ptrs_host, int32_t L, uint64_t* flips, uint64_t* steps,
                                     int32_t init, void* stream);
BDBNN_API int bdbnn_weight_stats_multi(const float* const* w_ptrs_host, const int64_t* numel_host,
                                       const int32_t* cout_host, int32_t L, double* filter_sums,
                                       uint32_t* filter_hist, double* stats_out, uint64_t* hist_out, void* stream);

/* ---- KD logits loss (DistributionLoss.forward, utils/KD_loss.py:16-43; train.py:612) -----------
 * loss = -(1/N) sum_n sum_c softmax(t)[n,c] * log_softmax(s)[n,c]
 * grad_s[n,c] = (softmax(s) - softmax(t))[n,c] / N          (written when grad_s != NULL)
 * row_ws: device float[N] scratch.  s,t row-major [N,C] fp32. */
BDBNN_API int bdbnn_kd_logits_fwd_bwd(const float* s, const float* t, int32_t N, int32_t C, float* row_ws,
                            float* loss_out, float* grad_s, void* stream);

/* ---- KD per-layer weight loss (DistributionLoss_layer.forward, utils/KD_loss.py:52-67) ---------
 * loss = sum_l mean_l( exp(Wt_l) * (Wt_l - Ws_l) )   == sum_l KLDivLoss(log_target=True)(Ws,Wt)
 * bwd : gWs_l[j] (+)= -gout[0] * exp(Wt_l[j]) / numel_l
 * partial: device double[L] scratch, left holding mean_l(...) per layer; loss adds them in layer order, one sum
 * for any L (the same bits in every run). */
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

/* bdbnn_bn_fwd with C == 16 and sign_bits != NULL writes ONE sign / mask word per pixel (bits 0-15; bits 16-31
 * are 0, as bdbnn_act_pack writes them for 16 channels): the packs of the CIFAR stem's BatchNorm output for the
 * first 16-channel binary conv.  (fp32 y only; not with bdbnn_bn_fwd_i16.)
 *
 * Option-A shortcut of the CIFAR ResNets (stride-2 subsample + zero channel padding) as the residual, read in place:
 * bn_fwd_pad_shortcut / bn_fwd_i16_pad_shortcut = bdbnn_bn_fwd / bdbnn_bn_fwd_i16 with
 *   residual[n,i,j,c] = x[n,2i,2j,c-pad] for pad <= c < pad+Cin, else 0
 * x fp32 NHWC [N,H,W,Cin] (16-byte aligned); z [N,Ho,Wo,C] with Ho = ceil(H/2), Wo = ceil(W/2), n_pix = N*Ho*Wo.
 * Needs Cin % 4 == 0, pad % 4 == 0, pad + Cin <= C.  Results equal bn_fwd with that residual materialised.
 * pad_shortcut_bwd: the shortcut's gradient added in place to the block input's, gx fp32 NHWC [N,H,W,Cin]:
 *   gx[n,2i,2j,c] += gz[n,i,j,c+pad]   (gz fp32 NHWC [N,Ho,Wo,Cout]; same conditions, Cout % 4 == 0). */
BDBNN_API int bdbnn_bn_fwd_pad_shortcut(const float* y, const float* x, int32_t N, int32_t H, int32_t W, int32_t Cin,
                              int32_t pad, const float* gamma, const float* beta, int32_t C, float eps,
                              float momentum, float* running_mean, float* running_var, double* sums_ws,
                              uint32_t* ymax_bits, float* mean, float* invstd, float* ab_ws, float* z,
                              uint32_t* sign_bits, uint32_t* mask_bits, uint16_t* xb, uint8_t* xb_fp8, int32_t fmt,
                              int32_t stats_ready, void* stream);
BDBNN_API int bdbnn_bn_fwd_i16_pad_shortcut(const int16_t* y_int, const float* alpha, const float* x, int32_t N,
                                  int32_t H, int32_t W, int32_t Cin, int32_t pad, const float* gamma,
                                  const float* beta, int32_t C, float eps, float momentum, float* running_mean,
                                  float* running_var, double* sums_ws, uint32_t* ymax_bits, float* mean,
                                  float* invstd, float* ab_ws, float* z, uint32_t* sign_bits, uint32_t* mask_bits,
                                  uint16_t* xb, uint8_t* xb_fp8, int32_t fmt, void* stream);
BDBNN_API int bdbnn_pad_shortcut_bwd(const float* gz, float* gx, int32_t N, int32_t H, int32_t W, int32_t Cin,
                           int32_t Cout, int32_t pad, void* stream);

/* ---- Hardtanh and 2x2 max-pool units of the CIFAR VGG-Small (DESIGN.md §4n) -----------------------------------------
 * bn_fwd_hardtanh : bdbnn_bn_fwd without residual, then z = hardtanh(u) for the BatchNorm output u (torch.nn.Hardtanh:
 *          clamp to [-1, 1], NaN stays NaN).  y is int16 (y = alpha[c] * y_int, statistics ready: stats_ready must be 1)
 *          when alpha != NULL, else fp32.  The packs (needed: sign_bits, mask_bits, xb; C % 32 == 0) are sign(u) and
 *          mask = (-1 < u < 1), strictly and 0 at NaN: Hardtanh's gradient times the next conv's STE indicator.
 * bn_bwd_pack_hardtanh : bdbnn_bn_bwd_pack(_i16) of gz * mask, the mask recomputed from y and the forward's ab_ws
 *          (`ab`, float[2C]); the sums are always computed here.
 * pool2_i16 : p_int int16 NHWC [N,H/2,W/2,C] = 2x2 / stride-2 max of y_int [N,H,W,C] (H, W even, C % 32 == 0), idx
 *          uint8 [N,H/2,W/2,C] = the winner's tap dy*2 + dx (first maximum in scan order, as torch.nn.MaxPool2d), and
 *          the BatchNorm statistics of alpha*p into sums double[2C] / ymax_bits u32[C] (zeroed here; per-block
 *          partials summed in a fixed order) for bn_fwd_hardtanh(p_int, alpha, n_pix = N*H/2*W/2, stats_ready = 1).
 * pool2_bn_bwd_pack : the BatchNorm + Hardtanh backward of that unit over the pooled tensor (gz fp32 NHWC
 *          [N,H/2,W/2,C]), written as gys at the conv-output resolution [N,H,W,(2)C]: the packed value at the winner,
 *          0 elsewhere (the max-pool backward).  Scratch and outputs as bdbnn_bn_bwd_pack.
 * pool2_bn_eval_hardtanh : z fp32 NHWC [N,H/2,W/2,C] = hardtanh(fp32(fp32(m * scale[c]) + shift[c])) for m the 2x2
 *          max of y_int, scale / shift from bdbnn_bn_eval_fold with alpha; optionally the +-1 copy of z, 16-bit in
 *          format fmt (zb) and / or e4m3 (zb8).
 * real_pool2_bn_eval_hardtanh : the same unit after a real-valued conv (the fp32 VGG-Small teacher): y fp32 NHWC
 *          [N,H,W,C] (H, W even, C % 32 == 0), z fp32 NHWC [N,H/2,W/2,C] = hardtanh(fp32(fp32(m * scale[c]) +
 *          shift[c])) for m the 2x2 max of y (NaN if the window holds one, as F.max_pool2d), no +-1 copy;
 *          z_amax_bits (one word, zeroed here) receives the bits of max|z| (integer atomicMax, as
 *          bdbnn_real_conv_fwd_eval), for the next conv's bdbnn_real_act_pack. */
BDBNN_API int bdbnn_bn_fwd_hardtanh(const void* y, const float* alpha, const float* gamma, const float* beta,
                          int64_t n_pix, int32_t C, float eps, float momentum, float* running_mean,
                          float* running_var, double* sums_ws, uint32_t* ymax_bits, float* mean, float* invstd,
                          float* ab_ws, float* z, uint32_t* sign_bits, uint32_t* mask_bits, uint16_t* xb,
                          uint8_t* xb_fp8, int32_t fmt, int32_t stats_ready, void* stream);
BDBNN_API int bdbnn_bn_bwd_pack_hardtanh(const float* gz, const void* y, const float* alpha, const float* ab,
                               const float* mean, const float* invstd, const float* gamma, const float* gscale,
                               const uint32_t* ymax_bits, int64_t n_pix, int32_t C, int32_t grad_mode,
                               double* sums_ws, uint32_t* gmax_bits, float* consts_ws, float* dgamma, float* dbeta,
                               uint32_t* amax_bits, uint16_t* gys, void* stream);
BDBNN_API int bdbnn_pool2_i16(const int16_t* y_int, const float* alpha, int32_t N, int32_t H, int32_t W, int32_t C,
                    int16_t* p_int, uint8_t* idx, double* sums, uint32_t* ymax_bits, void* stream);
BDBNN_API int bdbnn_pool2_bn_bwd_pack(const float* gz, const int16_t* p_int, const uint8_t* idx, const float* alpha,
                            const float* ab, const float* mean, const float* invstd, const float* gamma,
                            const float* gscale, const uint32_t* ymax_bits, int32_t N, int32_t H, int32_t W, int32_t C,
                            int32_t grad_mode, double* sums_ws, uint32_t* gmax_bits, float* consts_ws, float* dgamma,
                            float* dbeta, uint32_t* amax_bits, uint16_t* gys, void* stream);
BDBNN_API int bdbnn_pool2_bn_eval_hardtanh(const int16_t* y_int, const float* scale, const float* shift, int32_t N,
                                 int32_t H, int32_t W, int32_t C, float* z, uint16_t* zb, uint8_t* zb8, int32_t fmt,
                                 void* stream);
BDBNN_API int bdbnn_real_pool2_bn_eval_hardtanh(const float* y, const float* scale, const float* shift, int32_t N,
                                      int32_t H, int32_t W, int32_t C, float* z, uint32_t* z_amax_bits,
                                      void* stream);

/* ---- Hardtanh units of the fp32 VGG-Small trained on the wgmma kernels (DESIGN.md §4u) ------------------------------
 * real_bn_fwd_hardtanh : BatchNorm(train) + Hardtanh on fp32 y NHWC [n_pix][C] (C % 4 == 0) with the statistics
 *          ready in sums_ws / ymax_bits (stats_ready must be 1: from the conv epilogue, real_pool2 or the stem):
 *          bn_finalize (mean, invstd, ab_ws, running statistics), then z = hardtanh(u) for u = fmaf(y, a, b), torch's
 *          Hardtanh (clamp to [-1, 1], NaN and -0.0 stay), no +-1 packs.  u is the u bn_bwd_pack_hardtanh recomputes
 *          from y and ab_ws, so its strict mask (-1 < u < 1, 0 at NaN) is this forward's decision.  z_amax_bits (one
 *          word, zeroed here) = bits of max|z| (integer atomicMax, NaN on top) for the next bdbnn_real_act_pack.
 * real_pool2 : pool2_i16 on the fp32 output of a real-valued conv: p fp32 NHWC [N,H/2,W/2,C] = 2x2 / stride-2 max of y
 *          [N,H,W,C] as F.max_pool2d takes it (scan order, `v > m || v is NaN`: the first of equal values, NaN wins),
 *          idx uint8 = the winner's tap dy*2 + dx (torch's index), the BatchNorm statistics of p into sums double[2C]
 *          and pmax_bits u32[C] = max|p| per channel (both zeroed here; per-block partials summed in a fixed order) for
 *          real_bn_fwd_hardtanh(p, n_pix = N*H/2*W/2, stats_ready = 1).  H, W even, C % 32 == 0.
 * real_pool2_bn_bwd_pack : pool2_bn_bwd_pack of that unit with fp32 p (no alpha), grad_mode FP16S: the BatchNorm +
 *          Hardtanh backward over the pooled tensor written as gys fp16 [N,H,W,C] at the conv-output resolution, the
 *          value at the winner and 0 elsewhere; pmax_bits is real_pool2's. */
BDBNN_API int bdbnn_real_bn_fwd_hardtanh(const float* y, const float* gamma, const float* beta, int64_t n_pix, int32_t C,
                               float eps, float momentum, float* running_mean, float* running_var, double* sums_ws,
                               uint32_t* ymax_bits, float* mean, float* invstd, float* ab_ws, float* z,
                               uint32_t* z_amax_bits, int32_t stats_ready, void* stream);
BDBNN_API int bdbnn_real_pool2(const float* y, int32_t N, int32_t H, int32_t W, int32_t C, float* p, uint8_t* idx,
                     double* sums, uint32_t* pmax_bits, void* stream);
BDBNN_API int bdbnn_real_pool2_bn_bwd_pack(const float* gz, const float* p, const uint8_t* idx, const float* ab,
                                 const float* mean, const float* invstd, const float* gamma, const float* gscale,
                                 const uint32_t* pmax_bits, int32_t N, int32_t H, int32_t W, int32_t C,
                                 double* sums_ws, uint32_t* gmax_bits, float* consts_ws, float* dgamma, float* dbeta,
                                 uint32_t* amax_bits, uint16_t* gys, void* stream);

/* ---- ReLU units of the fp32 ResNet trained on the wgmma kernels (DESIGN.md §4r) ------------------------------------
 * bn_fwd_relu : bdbnn_bn_fwd on fp32 y (residual may be NULL), then z = relu(u) for u = BatchNorm(y) (+ residual)
 *          (torch.relu bit for bit: NaN and -0.0 stay).  No +-1 packs; instead mask_bits u32 [n_pix][C/32]
 *          (C % 32 == 0) = ReLU's gradient mask, bit c % 32 of word c / 32 set <=> !(z <= 0) (so set at NaN: torch's
 *          relu backward passes the gradient there), and
 *          z_amax_bits (one word, zeroed here) = bits of max|z| (integer atomicMax, NaN above every number), the word
 *          bdbnn_real_act_pack takes for the next conv's fp16 operand.
 * bn_bwd_pack_relu : bdbnn_bn_bwd_pack (grad_mode FP16S) of g = gz where the mask bit is set, 0 elsewhere (a select:
 *          a NaN of gz where z <= 0 gives 0); the sums are always computed here.  g_out (may be NULL) receives g, fp32
 *          like gz: the gradient of the residual added before the ReLU.
 * bn_pool_fwd_relu : bdbnn_bn_pool_fwd with z = relu(maxpool(u)) = maxpool(relu(u)) and no +-1 packs; mask_bits and
 *          z_amax_bits as bn_fwd_relu (on the pooled z, C % 32 == 0); where the mask bit is 0 the winner byte is 0xff,
 *          so that bn_pool_bwd_relu sends that window's gradient nowhere (a NaN window keeps its winner).
 * bn_pool_bwd_relu : bdbnn_bn_pool_bwd with g_pool masked by mask_bits (bn_pool_fwd_relu's) in the sums and, through
 *          idx, in the scatter.
 * real_scale_fold : alpha[o] = alpha_w[o] * 2^-ex, inv_gscale[o] = inv_gscale_w[o] * 2^-ex for o < C, ex the exponent
 *          bdbnn_real_act_pack scales x by (x_amax_bits): the vectors bdbnn_binconv_fwd_tc and bdbnn_binconv_wgrad_tc
 *          take for a 3x3 conv of fp16 x by the weight pack of bdbnn_real_weight_pack_multi_grad.  One launch. */
BDBNN_API int bdbnn_bn_fwd_relu(const float* y, const float* residual, const float* gamma, const float* beta,
                      int64_t n_pix, int32_t C, float eps, float momentum, float* running_mean, float* running_var,
                      double* sums_ws, uint32_t* ymax_bits, float* mean, float* invstd, float* ab_ws, float* z,
                      uint32_t* mask_bits, uint32_t* z_amax_bits, int32_t stats_ready, void* stream);
BDBNN_API int bdbnn_bn_bwd_pack_relu(const float* gz, const uint32_t* mask_bits, const float* y, const float* mean,
                           const float* invstd, const float* gamma, const float* gscale, const uint32_t* ymax_bits,
                           int64_t n_pix, int32_t C, int32_t grad_mode, double* sums_ws, uint32_t* gmax_bits,
                           float* consts_ws, float* dgamma, float* dbeta, uint32_t* amax_bits, uint16_t* gys,
                           float* g_out, void* stream);
BDBNN_API int bdbnn_bn_pool_fwd_relu(const float* y, const float* gamma, const float* beta, int32_t N, int32_t H,
                           int32_t W, int32_t C, int32_t k, int32_t stride, int32_t pad, int32_t Ho, int32_t Wo,
                           float eps, float momentum, float* running_mean, float* running_var, double* sums_ws,
                           uint32_t* ymax_bits, float* mean, float* invstd, float* ab_ws, float* z, float* y_sel,
                           uint8_t* idx, uint32_t* mask_bits, uint32_t* z_amax_bits, int32_t stats_ready,
                           void* stream);
BDBNN_API int bdbnn_bn_pool_bwd_relu(const float* g_pool, const uint8_t* idx, const uint32_t* mask_bits, const float* y,
                           const float* y_sel, const float* mean, const float* invstd, const float* gamma,
                           const float* ones, const uint32_t* ymax_bits, int32_t N, int32_t H, int32_t W, int32_t C,
                           int32_t k, int32_t stride, int32_t pad, int32_t Ho, int32_t Wo, double* sums_ws,
                           uint32_t* gmax_bits, float* consts_ws, float* dgamma, float* dbeta,
                           uint32_t* amax_scratch, float* gy, uint16_t* gys, void* stream);
BDBNN_API int bdbnn_real_scale_fold(const uint32_t* x_amax_bits, const float* alpha_w, const float* inv_gscale_w,
                          int32_t C, float* alpha, float* inv_gscale, void* stream);

/* ---- CIFAR stem: 3x3 / stride 1 / pad 1, 3 -> Cout channels (Cout in {16, 32, 48, 64, 128}), fp32, CUDA cores -
 * Replaces the fp32 nn.Conv2d `conv1` of the CIFAR ResNets (models/cifar10; model(images), train.py:492 and its
 * weight gradient under loss.backward(), train.py:528), which the reference runs on cuDNN.
 *   cifar_stem_fwd   : y fp32 NHWC [N,H,W,Cout] = conv(x, W): one fp32 FMA per tap, taps in the order (c, r, s), no
 *                      reduced-precision operands.  x [N,3,H,W] through element strides (NCHW or channels_last),
 *                      weight contiguous [Cout][3][3][3]; y 16-byte aligned.  bn_sums / bn_ymax (both or neither):
 *                      the BatchNorm statistics of y as bdbnn_binconv_fwd_tc writes them (for bdbnn_bn_fwd with
 *                      stats_ready = 1), from per-block partials summed in a fixed order; zeroed here.
 *   cifar_stem_wgrad : gW fp32 [Cout][3][3][3] (overwritten) = 2^-e * sum_pix x_tap(pix) * gys[pix][o], gys =
 *                      fp16(gy * 2^e) [N,H,W,Cout] with e from g_amax_bits (bdbnn_bn_bwd_pack, FP16S, gscale = 1):
 *                      TF32-class.  fp32 sums per block, block partials (in the workspace, of
 *                      bdbnn_cifar_stem_wgrad_workspace_bytes) added in block order by a finalize kernel.
 * Two launches (+ the statistics' fixed-order sum) forward, two backward; no input gradient.
 *   cifar_stem_fwd_eval : the same conv (same taps, same FMA order, same strides rules) with BatchNorm(eval) in the
 *                      epilogue, each step rounded (no FMA): z = fp32(fp32(y * scale[o]) + shift[o]), (scale,
 *                      shift) = bdbnn_bn_eval_fold with alpha = NULL.  z fp32 NHWC [N,H,W,Cout], 16-byte aligned;
 *                      z_amax_bits (one word, zeroed here) receives the bits of max|z| (integer atomicMax).  One
 *                      launch; replaces the eval-mode conv1 + bn1 of an fp32 CIFAR ResNet (the KD teacher). */
BDBNN_API int bdbnn_cifar_stem_fwd(const float* x, int32_t N, int32_t H, int32_t W, int64_t sN, int64_t sC,
                         int64_t sH, int64_t sW, const float* weight, int32_t Cout, float* y, double* bn_sums,
                         uint32_t* bn_ymax, void* stream);
BDBNN_API int bdbnn_cifar_stem_fwd_eval(const float* x, int32_t N, int32_t H, int32_t W, int64_t sN, int64_t sC,
                              int64_t sH, int64_t sW, const float* weight, int32_t Cout, const float* scale,
                              const float* shift, float* z, uint32_t* z_amax_bits, void* stream);
/* cifar_stem_fwd_eval_hardtanh: the same with z = hardtanh(BN_eval(conv)) (torch.nn.Hardtanh, NaN stays NaN) and Cout
 * in {16, 32, 48, 64, 128}: the eval stem of VGG-Small (DESIGN.md §4n); z_amax_bits is max|z| after the clamp. */
BDBNN_API int bdbnn_cifar_stem_fwd_eval_hardtanh(const float* x, int32_t N, int32_t H, int32_t W, int64_t sN,
                                       int64_t sC, int64_t sH, int64_t sW, const float* weight, int32_t Cout,
                                       const float* scale, const float* shift, float* z, uint32_t* z_amax_bits,
                                       void* stream);
BDBNN_API size_t bdbnn_cifar_stem_wgrad_workspace_bytes(int32_t N, int32_t H, int32_t W, int32_t Cout);
BDBNN_API int bdbnn_cifar_stem_wgrad(const float* x, int32_t N, int32_t H, int32_t W, int64_t sN, int64_t sC,
                           int64_t sH, int64_t sW, const uint16_t* gys, const uint32_t* g_amax_bits, int32_t Cout,
                           float* gW, void* workspace, size_t workspace_bytes, void* stream);

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
BDBNN_API int bdbnn_stem_conv_fwd_eval(const uint16_t* xw, const uint16_t* wf, const float* scale, const float* shift,
                             float* z, int32_t N, int32_t H, int32_t W, void* stream);
/* stem_conv_fwd_eval followed by z = relu(z) in the same epilogue (torch.relu: NaN propagates), for an fp32 teacher
 * whose stem is conv1 -> bn1 -> relu -> maxpool.  z_amax_bits (one word, may be NULL) receives the bits of max|z|,
 * zeroed here; the max-pool after it keeps that maximum, so the first block's activation pack can take it. */
BDBNN_API int bdbnn_stem_conv_fwd_eval_relu(const uint16_t* xw, const uint16_t* wf, const float* scale,
                                  const float* shift, float* z, uint32_t* z_amax_bits, int32_t N, int32_t H,
                                  int32_t W, void* stream);
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

/* ---- eval-mode forward of real-valued k x k convs (the frozen fp32 teacher of the KD step) --------------------
 * Operands as for the stem and the shortcut: fp16 after power-of-two scales (amax_pow2_scale of common.cuh:
 * max * 2^e in [2^13, 2^14)), fp32 accumulation — TF32-class, the format cuDNN gives the reference by default.
 *   real_act_pack          : xh[p][c] = fp16(x[p][c] * 2^ex), x dense fp32 NHWC [n_pix][C], C % 4 == 0.  ex from
 *                            amax_bits (one word): computed here (bits of max|x|, non-finite clamped to 3e38) when
 *                            have_amax == 0, else read as given (e.g. the z_amax_bits of the conv that wrote x).
 *                            One launch with the amax given, two without.
 *   real_weight_pack_multi : for `count` fp32 weights W_l [Cout][Cin][k][k] (host tables: Cout, Cin, k = kw_host[l],
 *                            and strides_host[4l..4l+3] = W_l's element strides along Cout, Cin, kh, kw; W_l must be
 *                            dense in some dimension order, e.g. contiguous or channels_last), one scale per tensor:
 *                            wf_l[o][t][c] = fp16(W_l[o][c][t] * 2^ew_l) (the forward's [Cout][k*k][Cin] layout),
 *                            alpha_l[o] = 2^-ew_l for every o; amax_bits = device scratch of `count` words (bits of
 *                            max|W_l|, zeroed here).  Two launches per 48 tensors.
 *   real_conv_fwd_eval     : the forward implicit GEMM of bdbnn_binconv_fwd_tc over xh / wf (fp16), with, rounding
 *                            every step (no FMA):
 *                              z = fp32(fp32(fp32(acc * 2^-ex) * scale[o]) + shift[o])   (2^-ex from x_amax_bits)
 *                              z = fp32(z + residual)  if residual != NULL (z's shape, must not alias it)
 *                              then the activation code `act`:
 *                                BDBNN_ACT_NONE     (0) z as it is
 *                                BDBNN_ACT_RELU     (1) z = relu(z)             (torch.relu: NaN propagates)
 *                                BDBNN_ACT_HARDTANH (2) z = clamp(z, -1, 1)     (torch.nn.Hardtanh(): NaN stays NaN,
 *                                                                                -0.0 stays -0.0)
 *                              any other value is rejected (BDBNN_ERR_INVALID_ARG)
 *                            (scale, shift) = bdbnn_bn_eval_fold with the weight's alpha.  z fp32 NHWC; z_amax_bits
 *                            (one word, may be NULL; zeroed here) receives the bits of max|z| (integer atomicMax
 *                            of |z|'s bits: run-to-run identical, NaN above every number).  Requires
 *                            bdbnn_tc_supported(s) & BDBNN_TC_FWD.  One launch. */
#define BDBNN_ACT_NONE 0
#define BDBNN_ACT_RELU 1
#define BDBNN_ACT_HARDTANH 2
BDBNN_API int bdbnn_real_act_pack(const float* x, int64_t n_pix, int32_t C, uint32_t* amax_bits, int32_t have_amax,
                        uint16_t* xh, void* stream);
BDBNN_API int bdbnn_real_weight_pack_multi(int32_t count, const float* const* W_host, const int32_t* Cout_host,
                                 const int32_t* Cin_host, const int32_t* kw_host, const int64_t* strides_host,
                                 uint32_t* amax_bits,
                                 uint16_t* const* wf_host, float* const* alpha_host, void* stream);
/*   real_weight_pack_multi_grad : the same pack (same arguments, same launches, same wf / alpha bits) plus the
 *                            operands of the data and weight gradients of a conv with real weights and +-1
 *                            activations (the W32/A1 convs, DESIGN.md §4p), through the existing
 *                            bdbnn_binconv_dgrad_tc / _wgrad_tc epilogues:
 *                              wt_l[c][k*k-1-t][o] = wf_l[o][t][c]   (the dgrad operand [Cin][k*k flipped][Cout],
 *                                                                     wf's fp16 bits, same scale)
 *                              gscale_l[o] = 2^-ew_l,  inv_gscale_l[o] = 2^ew_l
 *                            so that grad_pack(gy, gscale) with B = wt gives conv_transpose(gy, W) and the wgrad
 *                            epilogue's * inv_gscale gives sum(xb * gy).  wt_host, gscale_host and inv_gscale_host
 *                            are all NULL (then this is bdbnn_real_weight_pack_multi: two launches per 48 tensors)
 *                            or all given with non-NULL entries (three launches per 48 tensors); anything else is
 *                            BDBNN_ERR_INVALID_ARG before any launch. */
BDBNN_API int bdbnn_real_weight_pack_multi_grad(int32_t count, const float* const* W_host, const int32_t* Cout_host,
                                      const int32_t* Cin_host, const int32_t* kw_host, const int64_t* strides_host,
                                      uint32_t* amax_bits, uint16_t* const* wf_host, float* const* alpha_host,
                                      uint16_t* const* wt_host, float* const* gscale_host,
                                      float* const* inv_gscale_host, void* stream);
BDBNN_API int bdbnn_real_conv_fwd_eval(const uint16_t* xh, const uint32_t* x_amax_bits, const uint16_t* wf,
                             const float* scale, const float* shift, const float* residual, int32_t act, float* z,
                             uint32_t* z_amax_bits, const bdbnn_conv_shape* s, void* stream);

/* ---- grouped 3x3 real-valued convs as banded GEMMs (ResNeXt conv2, DESIGN.md §4t) -------------------------------
 * A grouped conv with Cin = Cout = C, `groups` groups of Cg = C / groups channels, 3x3 / pad 1 / stride 1 or 2.  The
 * output channels are split into bands of B = max(16, Cg) channels (B in {16, 32, 64}, Cg divides B, B divides C);
 * every group lies inside one band, and a band is a dense B -> B conv whose weight is block-diagonal (exact zeros
 * between its groups).  x, gy: fp16 NHWC operands as for the dense kernels; fp16 weights as packed by
 * bdbnn_real_weight_pack_multi_grouped.  Since the band multiplies the other groups' activations by exact zeros, an
 * Inf or NaN of x (or of gy) in one group reaches the outputs of the other groups of its band (Inf * 0 = NaN), where
 * torch's grouped conv keeps it inside its group.
 *   real_gconv_supported   : host-only, no CUDA call: for a valid shape s (Cin = Cout = C) and `groups`,
 *                            BDBNN_TC_FWD (the training forward, statistics in the epilogue) | BDBNN_TC_EVAL |
 *                            BDBNN_TC_DGRAD | BDBNN_TC_WGRAD when the banded kernels take it, else 0.
 *   real_gconv_fwd         : y = acc * alpha[o] (fp32 NHWC [N][Ho][Wo][C]) of xh by wf [C][9][B], with the BatchNorm
 *                            statistics of y (sum y, sum y^2 as doubles [2C], max|y| bits [C], zeroed here) in the
 *                            epilogue when bn_sums / bn_ymax are given.  One launch (+ one statistics sum).
 *   real_gconv_fwd_eval    : bdbnn_real_conv_fwd_eval's epilogue (act BDBNN_ACT_NONE or BDBNN_ACT_RELU) on the
 *                            banded GEMM.  One launch.
 *   real_gconv_dgrad       : bdbnn_binconv_dgrad_tc in the BDBNN_GRAD_FP16S mode (gys fp16 [N][Ho][Wo][C] with its
 *                            amax word; mask_bits, add as there) with wt [C][9 flipped][B].  One launch per stride
 *                            phase.
 *   real_gconv_wgrad       : bdbnn_binconv_wgrad_tc in the BDBNN_GRAD_FP16S mode: gW [C][Cg][3][3] = the in-group
 *                            sums (wmask over gW's OIHW index), with a workspace of
 *                            real_gconv_wgrad_workspace_bytes(s, groups) bytes (0 = not supported).  Two launches. */
BDBNN_API int bdbnn_real_gconv_supported(const bdbnn_conv_shape* s, int32_t groups);
BDBNN_API int bdbnn_real_gconv_fwd(const uint16_t* xh, const uint16_t* wf, const float* alpha, float* y,
                                   const bdbnn_conv_shape* s, int32_t groups, double* bn_sums, uint32_t* bn_ymax,
                                   void* stream);
BDBNN_API int bdbnn_real_gconv_fwd_eval(const uint16_t* xh, const uint32_t* x_amax_bits, const uint16_t* wf,
                                        const float* scale, const float* shift, const float* residual, int32_t act,
                                        float* z, uint32_t* z_amax_bits, const bdbnn_conv_shape* s, int32_t groups,
                                        void* stream);
BDBNN_API int bdbnn_real_gconv_dgrad(const uint16_t* gys, const uint32_t* amax_bits, const uint16_t* wt,
                                     const uint32_t* mask_bits, const float* add, float* gx, const bdbnn_conv_shape* s,
                                     int32_t groups, void* stream);
BDBNN_API size_t bdbnn_real_gconv_wgrad_workspace_bytes(const bdbnn_conv_shape* s, int32_t groups);
BDBNN_API int bdbnn_real_gconv_wgrad(const uint16_t* gys, const uint32_t* amax_bits, const uint16_t* xh,
                                     const uint32_t* wmask_bits, const float* inv_gscale, float* gW,
                                     const bdbnn_conv_shape* s, int32_t groups, void* workspace,
                                     size_t workspace_bytes, void* stream);
/*   real_weight_pack_multi_grouped : bdbnn_real_weight_pack_multi_grad with a group count per tensor (groups_host[l]
 *                            >= 1; Cin_host[l] = the weight's second dimension, Cin / groups).  A tensor with groups 1
 *                            gets exactly that entry's wf / alpha / wt / gscale / inv_gscale bits.  A grouped tensor
 *                            (Cout = Cin_host * groups, k = 3, B = max(16, Cin_host) as in real_gconv_supported)
 *                            gets the banded operands
 *                              wf_l[o][t][cl] = fp16(W_l[o][c - g(o)][t] * 2^ew_l) if c and o share a group, else +0
 *                              wt_l[c][8-t][ol] = wf_l[b(c) + ol][t][c - b(c)]
 *                            for c = b(o) + cl, b(o) = o - o % B, g(o) = o - o % Cin_host, and the same alpha, gscale
 *                            and inv_gscale (the zeros do not move max|W_l|).  wt_host, gscale_host and
 *                            inv_gscale_host are all NULL (forward operands only) or all given.  amax_bits: device
 *                            scratch of `count` words.  Every tensor is checked before the first launch. */
BDBNN_API int bdbnn_real_weight_pack_multi_grouped(int32_t count, const float* const* W_host,
                                                   const int32_t* Cout_host, const int32_t* Cin_host,
                                                   const int32_t* kw_host, const int64_t* strides_host,
                                                   const int32_t* groups_host, uint32_t* amax_bits,
                                                   uint16_t* const* wf_host, float* const* alpha_host,
                                                   uint16_t* const* wt_host, float* const* gscale_host,
                                                   float* const* inv_gscale_host, void* stream);

/* ---- eval forward with the CIFAR option-A shortcut as the residual, read in place ------------------------------
 * Replaces F.pad(x[:, :, ::2, ::2], (0, 0, 0, 0, pad, pad)) (models/cifar10's LambdaLayer, the `shortcut` of a
 * stride-2 BasicBlock) and the residual add after it.  The same launches as bdbnn_binconv_fwd_tc_eval and
 * bdbnn_real_conv_fwd_eval, with `residual` replaced by
 *   r[n,i,j,c] = x_res[n, 2i, 2j, c - pad]   for pad <= c < pad + C_res,   +0.0 otherwise
 * x_res fp32 NHWC [N][H_res][W_res][C_res], 16-byte aligned, not aliasing z.  Outside the band +0.0 is still added,
 * so z is bit-identical to passing the materialised zero-padded tensor as `residual` (-0.0 + 0.0 = +0.0).  Needs a
 * stride-2 conv with Ho = ceil(H_res / 2), Wo = ceil(W_res / 2), Cout == C_res + 2 * pad, and C_res, pad multiples
 * of 4.  binconv_fwd_tc_eval_pad_shortcut takes 16-bit operands only (the fp8 forward starts at 128 channels). */
BDBNN_API int bdbnn_binconv_fwd_tc_eval_pad_shortcut(const void* xb, const void* wf, int32_t fmt, const float* scale,
                                           const float* shift, const float* x_res, int32_t H_res, int32_t W_res,
                                           int32_t C_res, int32_t pad, float* z, uint16_t* zb, uint8_t* zb8,
                                           const bdbnn_conv_shape* s, void* stream);
BDBNN_API int bdbnn_real_conv_fwd_eval_pad_shortcut(const uint16_t* xh, const uint32_t* x_amax_bits, const uint16_t* wf,
                                          const float* scale, const float* shift, const float* x_res, int32_t H_res,
                                          int32_t W_res, int32_t C_res, int32_t pad, int32_t relu, float* z,
                                          uint32_t* z_amax_bits, const bdbnn_conv_shape* s, void* stream);

/* ---- CIFAR input batch from the device-resident dataset --------------------------------------------------------
 * Replaces the CIFAR DataLoaders of loader.py:7-50 (torchvision RandomCrop(32, padding=4), RandomHorizontalFlip,
 * ToTensor, Normalize in CPU workers, then the H2D copy of train.py:488-491).  images uint8 [n][32][32][3] (HWC per
 * image, 16-byte aligned), labels int64 [n].  Output element (b, c, i, j), with idx = perm(seed, epoch, pos0 + b):
 *   (dy, dx, flip) = draw(seed, epoch, idx) if augment, else (4, 4, 0);
 *   u = pixel (i + dy - 4, (flip ? 31 - j : j) + dx - 4) of image idx, channel c, or 0 outside the image;
 *   out = fp32((fp32(u / 255) - mean[c]) / std[c]), every step rounded to nearest (to_tensor, then normalize);
 * written through the element strides (sN, sC, sH, sW) (NCHW or channels_last); target[b] = labels[idx].
 * perm is a keyed Feistel bijection of [0, n) and draw a Philox-4x32-10 draw keyed by the dataset index (DESIGN.md
 * §4l; oracle/cifar_data_ref.py restates both).  mean_host / std_host: 3 floats each, HOST memory.  Needs
 * 1 <= n < 2^31 and 0 <= pos0, pos0 + B <= n.  One launch, B blocks; nothing read back. */
BDBNN_API int bdbnn_cifar_batch(const uint8_t* images, const int64_t* labels, int64_t n, uint64_t seed,
                                uint32_t epoch, int64_t pos0, int32_t B, int32_t augment, const float* mean_host,
                                const float* std_host, float* out, int64_t sN, int64_t sC, int64_t sH, int64_t sW,
                                int64_t* target, void* stream);

/* ---- ImageNet input batch from decoded uint8 images (csrc/imagenet_data.cu) ---------------------------------------
 * Replaces the per-image PIL transforms of loader.py:52-85 (RandomResizedCrop(224) + RandomHorizontalFlip, or
 * Resize(256) + CenterCrop(224); then ToTensor, Normalize) for images already decoded to uint8 RGB on the device.
 * One descriptor per image (88 bytes):
 *   src            : device pointer to the decoded image; pixel (c, y, x) at src[c * sC + y * sH + x * sW] (uint8
 *                    element strides: CHW planar and HWC both work); H x W, each side in [1, 8192]
 *   x0, y0, w, h   : crop box inside the source
 *   RH, RW         : size the box is resized to, in [224, 2^22] per side
 *   oy0, ox0       : origin of the 224 x 224 output window inside the resized image
 *   flip           : 1 mirrors the output columns (after the resize, as torchvision's hflip)
 *   label          : written to target[b]
 * Training: box = the crop, resized = 224 x 224, window (0, 0).  Evaluation: box = the whole image, resized =
 * Resize(256)'s size, window = CenterCrop(224)'s offsets.  Output element (b, c, i, j) = fp32((fp32(u / 255) -
 * mean[c]) / std[c]), each step rounded, u = pixel (oy0 + i, ox0 + (flip ? 223 - j : j)) of Pillow's antialiased
 * bilinear resize (uint8, 22-bit fixed point, horizontal pass then vertical; DESIGN.md §4m,
 * oracle/imagenet_data_ref.py) of the box to RH x RW; written through the element strides (sN, sC, sH, sW).
 * desc_host: B descriptors in HOST memory (pinned, so that the copy is asynchronous: keep them unchanged until work
 * queued on `stream` after this call has run); desc_dev: device memory for B descriptors, 8-byte aligned.  Every
 * descriptor is validated on the host.  mean_host / std_host: 3 floats each, HOST memory.  One H2D copy and one
 * launch on `stream`; nothing read back. */
typedef struct bdbnn_imagenet_desc {
  const uint8_t* src;
  int64_t sC, sH, sW;
  int32_t H, W;
  int32_t x0, y0, w, h;
  int32_t RH, RW;
  int32_t oy0, ox0;
  int32_t flip, reserved;
  int64_t label;
} bdbnn_imagenet_desc;
BDBNN_API int bdbnn_imagenet_batch(const bdbnn_imagenet_desc* desc_host, bdbnn_imagenet_desc* desc_dev, int32_t B,
                                   const float* mean_host, const float* std_host, float* out, int64_t sN,
                                   int64_t sC, int64_t sH, int64_t sW, int64_t* target, void* stream);

/* ---- Baseline JPEG decode on the device (csrc/jpeg_decode.cu) -----------------------------------------------------
 * Replaces libjpeg-turbo's decode (torchvision.io.decode_jpeg on the host, mode RGB) of the files it takes, with the
 * same pixels: jpeg_idct_islow, fancy upsampling, ycc_rgb_convert (DESIGN.md §4m, oracle/jpeg_ref.py).  Taken:
 * SOF0, or SOF1 with 8-bit samples; Huffman; one scan with every component in frame order; 1 component, or 3 that
 * libjpeg treats as YCbCr (a JFIF marker, an Adobe marker with transform 1, or ids 1, 2, 3 without an Adobe marker);
 * luma sampling 1x1, 2x1 or 2x2 with chroma 1x1; any restart interval; sides in [1, 8192].
 *
 * bdbnn_jpeg_parse (host only, thread-safe, allocates nothing): reads file_host's markers up to SOS, fills *desc_host
 * and writes the entropy-coded data, with stuffed 0x00 bytes dropped and split at the RST markers, to data_host[0,
 * desc->data_bytes); segment k starts at data_host[seg_off_host[k]], k < desc->nseg.  Returns 0, or
 * BDBNN_ERR_UNSUPPORTED for a file it does not take (progressive, arithmetic, lossless, 12-bit, CMYK / RGB, other
 * sampling, several scans, DNL, an RST out of sequence, any marker but RSTn / EOI inside the scan, a missing EOI, a
 * header anomaly, or data_cap / seg_cap too small: data_cap >= file_bytes and seg_cap >= file_bytes / 3 + 2
 * suffice), BDBNN_ERR_INVALID_ARG for NULL pointers or negative sizes.  The caller sets data_off, coef_off and
 * rgb_off. */
typedef struct bdbnn_jpeg_huff {
  uint16_t lut[512];    /* 9-bit lookahead: (code length << 8) | symbol, 0 for longer (or invalid) codes */
  int32_t maxcode[18];  /* largest code of each length (index = length), -1 if none */
  int32_t valoff[17];   /* a length-l code's symbol is vals[code + valoff[l]] */
  uint8_t vals[256];
} bdbnn_jpeg_huff;
typedef struct bdbnn_jpeg_desc {
  int32_t H, W;
  int32_t ncomp;        /* 1 or 3 */
  int32_t hmax, vmax;   /* luma sampling factors (1, 1 for one component) */
  int32_t mcux, mcuy;   /* MCU grid */
  int32_t bpm;          /* blocks per MCU */
  int32_t restart;      /* restart interval in MCUs, 0 = none */
  int32_t nseg;         /* entropy-coded segments */
  int32_t data_bytes;   /* unstuffed bytes */
  int32_t reserved;
  int64_t data_off;     /* caller: offset of this image's data in data_dev */
  int64_t coef_off;     /* caller: first block of this image (sum of the earlier images' mcux * mcuy * bpm) */
  int64_t rgb_off;      /* caller: offset of this image's H x W x 3 output in rgb (3 x the earlier images' pixels) */
  uint8_t blk_comp[8];  /* component of each block of the MCU */
  uint8_t comp_dc[4], comp_ac[4];       /* Huffman table of each component: dc[] / ac[] index */
  uint16_t qt[3][64];   /* quantisation table of each component, natural order */
  bdbnn_jpeg_huff dc[2], ac[2];
} bdbnn_jpeg_desc;
BDBNN_API int bdbnn_jpeg_parse(const uint8_t* file_host, int64_t file_bytes, bdbnn_jpeg_desc* desc_host,
                               uint8_t* data_host, int64_t data_cap, uint32_t* seg_off_host, int32_t seg_cap);

/* One entropy-coded segment of a batch: bytes [off, off + nbytes) of data_dev, MCUs [mcu0, mcu0 + nmcu) of image img,
 * cut into nsub = max(1, ceil(8 nbytes / S)) subsequences of S = bdbnn_jpeg_subseq_bits() bits, the first being
 * sub0 = the earlier segments' nsub summed.  Segments are listed image by image, in order. */
typedef struct bdbnn_jpeg_seg {
  int64_t off;
  int32_t img, nbytes;
  int32_t mcu0, nmcu;
  int32_t sub0, nsub;
} bdbnn_jpeg_seg;
/* Status bits of an image (any one sends it to the host decoder) */
#define BDBNN_JPEG_PAST_END 1     /* a needed bit past the end of a segment */
#define BDBNN_JPEG_BAD_CODE 2     /* an invalid Huffman code */
#define BDBNN_JPEG_K_OVERFLOW 4   /* a coefficient or zero run past index 63 */
#define BDBNN_JPEG_DC_RANGE 8     /* a DC value outside int16 */
#define BDBNN_JPEG_PADDING 16     /* more than 7 bits left after a segment's last MCU */
#define BDBNN_JPEG_IDCT_RANGE 32  /* IDCT inputs or intermediates outside the range where libjpeg-turbo's SIMD and
                                     C paths agree (dequantised or pass-1 values outside int16, pass-2 outside
                                     [-512, 511]) */
#define BDBNN_JPEG_INDEX 64       /* bdbnn_jpeg_decode_batch_indexed: a subsequence's exit differs from the segment's
                                     next stored start, or a stored start is malformed */
#define BDBNN_JPEG_RECORD 128     /* bdbnn_jpeg_decode_batch_files: the file differs from its record (geometry,
                                     restart interval, segment count or lengths, data_bytes), or the host parse
                                     refuses it */
/* Subsequence length S in bits (1024, or the bdbnn_debug_jpeg_subseq_bits override). */
BDBNN_API int bdbnn_jpeg_subseq_bits(void);
/* Tests only: sets S to bits in [8, 2^20], 0 restores the default.  Process-wide. */
BDBNN_API int bdbnn_debug_jpeg_subseq_bits(int32_t bits);
/* Device workspace for a batch of n_blocks blocks (sum of mcux * mcuy * bpm) and n_sub subsequences.  The
 * workspace begins with the int16 coefficients [n_blocks][64] (natural order, blocks in MCU order, DC after
 * prediction), valid after bdbnn_jpeg_decode_batch. */
BDBNN_API size_t bdbnn_jpeg_workspace_bytes(int64_t n_blocks, int64_t n_sub);
/* Host only: the validation bdbnn_jpeg_decode_batch runs before it touches any device pointer, of n_img
 * descriptors and n_seg segments (offsets, MCU coverage, subsequence counts at the current S) against data_bytes,
 * rgb_bytes and work_bytes.  0 or BDBNN_ERR_INVALID_ARG. */
BDBNN_API int bdbnn_jpeg_check_batch(const bdbnn_jpeg_desc* desc_host, int32_t n_img, const bdbnn_jpeg_seg* seg_host,
                                     int32_t n_seg, int64_t data_bytes, int64_t rgb_bytes, size_t work_bytes);
/* Decodes n_img images into rgb (uint8 HWC, image i at rgb + desc[i].rgb_off).  desc_host, seg_host and data_host
 * (data_bytes bytes) are copied to desc_dev, seg_dev and data_dev (pass pinned host memory for asynchronous
 * copies); every descriptor and segment is validated on the host first.  work: 256-byte aligned, work_bytes >=
 * bdbnn_jpeg_workspace_bytes.  status_dev / status_host: n_img int32 each; status_host (pinned) receives each
 * image's BDBNN_JPEG_* bits by a copy queued last on `stream`; rounds_host (pinned, may be NULL) likewise receives
 * the most barrier rounds one block of the synchronisation phase took.  Everything is queued on `stream`; nothing
 * waits on the host.  Keep the host buffers unchanged, and read rgb, status_host and rounds_host, once work queued
 * on `stream` after this call has run. */
BDBNN_API int bdbnn_jpeg_decode_batch(const bdbnn_jpeg_desc* desc_host, bdbnn_jpeg_desc* desc_dev, int32_t n_img,
                                      const bdbnn_jpeg_seg* seg_host, bdbnn_jpeg_seg* seg_dev, int32_t n_seg,
                                      const uint8_t* data_host, uint8_t* data_dev, int64_t data_bytes, void* work,
                                      size_t work_bytes, uint8_t* rgb, int64_t rgb_bytes, int32_t* status_dev,
                                      int32_t* status_host, int32_t* rounds_host, void* stream);

/* ---- Index of the synchronisation points (DESIGN.md §4m) ------------------------------------------------------------
 * The state of the sequential decode at every subsequence boundary of a file, computed once on the host so that the
 * device needs no synchronisation pass.  One uint16 entry per subsequence j >= 1 of each segment, segments in order
 * (the first subsequence of a segment starts at bit 0, block 0, DC, and is not stored): the state (pos, b, k) where
 * the sequential decode crosses bit j S, i.e. its first codeword boundary at or past j S, as bits 0-4 pos - j S,
 * bits 5-7 the block in the MCU b, bits 8-13 the zig-zag index k; bits 14-15 zero.
 *
 * bdbnn_jpeg_index_file (host only, thread-safe, allocates nothing): the entries of file_host at subsequences of
 * S bits, S in [8, 2^20].  scratch: 8-byte aligned, scratch_cap >= bdbnn_jpeg_index_scratch_bytes(file_bytes);
 * entry_cap >= 8 file_bytes / S suffices.  On success *n_entries entries and *n_seg = desc->nseg of
 * bdbnn_jpeg_parse.  Returns 0; BDBNN_ERR_UNSUPPORTED for a file bdbnn_jpeg_parse does not take, a segment whose
 * sequential decode raises a BDBNN_JPEG_* status bit (a fault, fewer blocks than its MCUs hold, or more than 7 bits
 * after them), or a state that does not fit an entry; BDBNN_ERR_INVALID_ARG for NULL pointers, sizes out of range
 * or too small a scratch or entry_cap. */
BDBNN_API size_t bdbnn_jpeg_index_scratch_bytes(int64_t file_bytes);
/* Tests only: packs state (pos, b, k) as the entry of subsequence j at S bits into *entry and unpacks it into
 * state[0..2]; BDBNN_ERR_UNSUPPORTED if the state has no entry. */
BDBNN_API int bdbnn_debug_jpeg_index_entry(int32_t pos, int32_t b, int32_t k, int32_t j, int32_t S, uint16_t* entry,
                                           int32_t* state);
BDBNN_API int bdbnn_jpeg_index_file(const uint8_t* file_host, int64_t file_bytes, int32_t S, void* scratch,
                                    size_t scratch_cap, uint16_t* entries, int64_t entry_cap, int64_t* n_entries,
                                    int32_t* n_seg);
/* bdbnn_jpeg_decode_batch with the starts taken from an index instead of the synchronisation pass.  entries_host
 * (n_entries uint16, pinned for an asynchronous copy) holds, segment by segment in the order of seg_host, each
 * segment's nsub - 1 entries at the current S (segment s's begin at entry sub0 - s); they are copied to entries_dev
 * on `stream`.  Returns BDBNN_ERR_INVALID_ARG before any launch if n_entries is not the sum of nsub - 1.  One pass,
 * one thread per subsequence, decodes from each stored start and compares the exit with the next stored start: an
 * image with a mismatch or a malformed entry gets BDBNN_JPEG_INDEX (and its pixels are not to be used, as with any
 * status bit).  When no image is flagged, the coefficients and pixels are those of bdbnn_jpeg_decode_batch.
 * rounds_host (may be NULL) receives 0. */
BDBNN_API int bdbnn_jpeg_decode_batch_indexed(const bdbnn_jpeg_desc* desc_host, bdbnn_jpeg_desc* desc_dev,
                                              int32_t n_img, const bdbnn_jpeg_seg* seg_host, bdbnn_jpeg_seg* seg_dev,
                                              int32_t n_seg, const uint8_t* data_host, uint8_t* data_dev,
                                              int64_t data_bytes, const uint16_t* entries_host, uint16_t* entries_dev,
                                              int64_t n_entries, void* work, size_t work_bytes, uint8_t* rgb,
                                              int64_t rgb_bytes, int32_t* status_dev, int32_t* status_host,
                                              int32_t* rounds_host, void* stream);

/* ---- Decode from the original files (DESIGN.md §4m, bdbnn_b200/jpeg_pack.py) ----------------------------------------
 * bdbnn_jpeg_decode_batch_indexed with the header parse and the unstuffing on the device.  files_host (files_bytes,
 * pinned) holds the batch's original JPEG files; image i's is bytes [file[i].off, + file[i].size) (16-byte aligned
 * offsets read fastest).  desc_host holds the image's record: H, W, ncomp, hmax, vmax, mcux, mcuy, bpm, restart, nseg,
 * data_bytes, blk_comp as bdbnn_jpeg_check_batch requires, and the caller's data_off, coef_off and rgb_off; its
 * other tables are zero.  seg_host, entries and every other
 * argument as bdbnn_jpeg_decode_batch_indexed, except that data_dev is written by the device and has no host copy.
 * On `stream`: files_host and file_host are copied to files_dev and file_dev; jpeg_parse_kernel (one thread per image)
 * builds desc_dev's quantisation and Huffman tables, blk_comp, comp_dc and comp_ac from the file's markers and sets
 * file_dev[i].scan; jpeg_unstuff_kernel (one CUDA block per image) writes the scan's unstuffed bytes to data_dev at
 * data_off, segment k at the segment table's offset; then the indexed decode.  A file that the host parse refuses,
 * or that differs from its record in geometry, restart interval, RST sequence, segment lengths or data_bytes, gets
 * BDBNN_JPEG_RECORD; no kernel reads or writes outside the buffers whatever the records say.  When every record
 * is true, desc_dev equals bdbnn_jpeg_parse's descriptor with the caller's offsets, data_dev its data, and the
 * pixels those of bdbnn_jpeg_decode_batch. */
typedef struct bdbnn_jpeg_file {
  int64_t off;          /* caller: the file's first byte in files */
  int32_t size;         /* caller: its bytes */
  int32_t scan;         /* device: offset of its entropy-coded data, -1 if the parse flagged it */
} bdbnn_jpeg_file;
BDBNN_API int bdbnn_jpeg_decode_batch_files(const uint8_t* files_host, uint8_t* files_dev, int64_t files_bytes,
                                            const bdbnn_jpeg_file* file_host, bdbnn_jpeg_file* file_dev,
                                            const bdbnn_jpeg_desc* desc_host, bdbnn_jpeg_desc* desc_dev, int32_t n_img,
                                            const bdbnn_jpeg_seg* seg_host, bdbnn_jpeg_seg* seg_dev, int32_t n_seg,
                                            uint8_t* data_dev, int64_t data_bytes, const uint16_t* entries_host,
                                            uint16_t* entries_dev, int64_t n_entries, void* work, size_t work_bytes,
                                            uint8_t* rgb, int64_t rgb_bytes, int32_t* status_dev,
                                            int32_t* status_host, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* BDBNN_H_ */
