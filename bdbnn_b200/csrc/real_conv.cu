// fp32 1x1 shortcut convolutions (ResNet `downsample`: 1x1, stride 2, no bias) on the tensor-core kernels.
//
// The reference keeps these convs real-valued (fp32 nn.Conv2d; cuDNN runs them on TF32 tensor cores).
// Like the stem (stem.cu) both operands are rounded to fp16 after per-call power-of-two scales (11-bit
// significands = TF32's, fp32 accumulation).  This file only PACKS: the strided input samples become a
// dense fp16 NHWC tensor xh = fp16(x[:, ::s, ::s, :] * 2^ex), the weight becomes wf = fp16(W * 2^ew)
// [Cout][Cin] and its transpose wt [Cin][Cout]; the GEMMs are the existing implicit-GEMM kernels run as a
// 1x1 / stride-1 convolution over xh, with the scales folded into the per-channel vectors those kernels
// already take:
//   forward : bdbnn_binconv_fwd_tc(xh, wf, FP16, alpha)            alpha[o]      = 2^-ew * 2^-ex
//   backward: gys = fp16(gy * gscale[o] * 2^e)                      gscale[o]     = 2^-ew
//             bdbnn_binconv_dgrad_tc(gys, wt, all-ones mask)        (2^e undone in its epilogue)
//             bdbnn_binconv_wgrad_tc(gys, xh, all-ones mask)        inv_gscale[o] = 2^ew * 2^-ex
#include <cuda_fp16.h>

#include <vector>

#include "common.cuh"

namespace bdbnn {

// max|x| over the sampled positions; thread = one float4 channel quad of one output pixel
__global__ void __launch_bounds__(256)
real_amax_kernel(const float4* __restrict__ x, int H, int W, int C4, int Ho, int Wo, int s, int64_t total,
                 uint32_t* __restrict__ amax_bits) {
  float m = 0.f;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += int64_t(gridDim.x) * blockDim.x) {
    const int c = int(i % C4);
    int64_t q = i / C4;
    const int wo = int(q % Wo); q /= Wo;
    const int ho = int(q % Ho);
    const int64_t n = q / Ho;
    const float4 v = __ldg(x + ((n * H + int64_t(ho) * s) * W + int64_t(wo) * s) * C4 + c);
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  m = warp_max(m);
  if (!(m < 3.0e38f)) m = 3.0e38f;
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(amax_bits, __float_as_uint(m));
}

__global__ void __launch_bounds__(256)
real_pack_x_kernel(const float4* __restrict__ x, int H, int W, int C4, int Ho, int Wo, int s, int64_t total,
                   const uint32_t* __restrict__ amax_bits, uint2* __restrict__ xh) {
  const float scale = amax_pow2_scale(__ldg(amax_bits), false);
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += int64_t(gridDim.x) * blockDim.x) {
    const int c = int(i % C4);
    int64_t q = i / C4;
    const int wo = int(q % Wo); q /= Wo;
    const int ho = int(q % Ho);
    const int64_t n = q / Ho;
    const float4 v = __ldg(x + ((n * H + int64_t(ho) * s) * W + int64_t(wo) * s) * C4 + c);
    const __half2 a = __floats2half2_rn(v.x * scale, v.y * scale), b = __floats2half2_rn(v.z * scale, v.w * scale);
    xh[i] = make_uint2(*reinterpret_cast<const uint32_t*>(&a), *reinterpret_cast<const uint32_t*>(&b));
  }
}

// max|W| (flat) into w_amax_bits (pre-zeroed)
__global__ void __launch_bounds__(256)
real_amax_w_kernel(const float* __restrict__ Wt, int n, uint32_t* __restrict__ w_amax_bits) {
  float m = 0.f;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) m = fmaxf(m, fabsf(__ldg(Wt + i)));
  m = warp_max(m);
  if (!(m < 3.0e38f)) m = 3.0e38f;
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(w_amax_bits, __float_as_uint(m));
}

// This block's slice of wf (coalesced along c) and of wt (coalesced along o), and — block 0 — the
// per-output-channel scale vectors.
__global__ void __launch_bounds__(1024)
real_pack_w_kernel(const float* __restrict__ Wt, int Cout, int Cin, const uint32_t* __restrict__ x_amax_bits,
                   const uint32_t* __restrict__ w_amax_bits, __half* __restrict__ wf, __half* __restrict__ wt,
                   float* __restrict__ alpha, float* __restrict__ gscale, float* __restrict__ inv_gscale) {
  const int n = Cout * Cin;
  const uint32_t w_amax = __ldg(w_amax_bits);
  const float sw = amax_pow2_scale(w_amax, false);
  const int stride = gridDim.x * blockDim.x;
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) wf[i] = __float2half_rn(__ldg(Wt + i) * sw);
  for (int j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += stride) {
    const int c = j / Cout, o = j - c * Cout;
    wt[j] = __float2half_rn(__ldg(Wt + int64_t(o) * Cin + c) * sw);
  }
  if (blockIdx.x == 0) {
    const float isw = amax_pow2_scale(w_amax, true), isx = amax_pow2_scale(__ldg(x_amax_bits), true);
    for (int o = threadIdx.x; o < Cout; o += blockDim.x) {
      alpha[o] = isw * isx;
      gscale[o] = isw;
      inv_gscale[o] = sw * isx;
    }
  }
}

// k x k weights of many real-valued convs (the 3x3 convs of an fp32 ResNet teacher) in two launches: one scale per
// tensor, wf[o][t][c] = fp16(W[o][c][t] * 2^ew) in the forward's [Cout][k*k][Cin] layout, alpha[o] = 2^-ew.  W is
// read through its element strides, so a dense OIHW or channels_last weight needs no copy.
constexpr int kRealPackMax = 48;          // keeps the table (kernel parameter) under 4 KB
constexpr int kRealPackPerBlock = 4096;   // weights per block (256 threads x 16)
struct RealWPackTable {
  const float* W[kRealPackMax];
  uint16_t* wf[kRealPackMax];
  float* alpha[kRealPackMax];
  int32_t Cout[kRealPackMax], Cin[kRealPackMax], T[kRealPackMax], KW[kRealPackMax];
  int32_t sO[kRealPackMax], sC[kRealPackMax], sR[kRealPackMax], sS[kRealPackMax];   // element strides of W
  int32_t blk0[kRealPackMax + 1];         // first block of tensor l (prefix sums of ceil(numel / kRealPackPerBlock))
  int32_t n;
};

__device__ __forceinline__ int real_wpack_find(const RealWPackTable& tab, int b) {
  int l = 0;
  while (l + 1 < tab.n && b >= tab.blk0[l + 1]) ++l;
  return l;
}

// amax[l] (pre-zeroed) = bits of max|W_l|, clamped to a finite value like the activation amax; W_l is dense (any
// dimension order), so its numel elements are the first numel of its storage
__global__ void __launch_bounds__(256)
real_wamax_multi_kernel(const __grid_constant__ RealWPackTable tab, uint32_t* __restrict__ amax) {
  const int l = real_wpack_find(tab, int(blockIdx.x));
  const int n = tab.Cout[l] * tab.Cin[l] * tab.T[l];
  const int base = (int(blockIdx.x) - tab.blk0[l]) * kRealPackPerBlock;
  const int end = base + kRealPackPerBlock < n ? base + kRealPackPerBlock : n;
  const float* W = tab.W[l];
  float m = 0.f;
  for (int i = base + threadIdx.x; i < end; i += blockDim.x) m = fmaxf(m, fabsf(__ldg(W + i)));
  m = warp_max(m);
  if (!(m < 3.0e38f)) m = 3.0e38f;
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(amax + l, __float_as_uint(m));
}

// coalesced along the output (c fastest); an OIHW weight is read with stride k*k through L2, a channels_last one
// in order
__global__ void __launch_bounds__(256)
real_wpack_multi_kernel(const __grid_constant__ RealWPackTable tab, const uint32_t* __restrict__ amax) {
  const int l = real_wpack_find(tab, int(blockIdx.x));
  const int Cin = tab.Cin[l], T = tab.T[l], KW = tab.KW[l], n = tab.Cout[l] * Cin * T;
  const int sO = tab.sO[l], sC = tab.sC[l], sR = tab.sR[l], sS = tab.sS[l];
  const int base = (int(blockIdx.x) - tab.blk0[l]) * kRealPackPerBlock;
  const int end = base + kRealPackPerBlock < n ? base + kRealPackPerBlock : n;
  const uint32_t a = __ldg(amax + l);
  const float sw = amax_pow2_scale(a, false), isw = amax_pow2_scale(a, true);
  const float* W = tab.W[l];
  __half* wf = reinterpret_cast<__half*>(tab.wf[l]);
  for (int j = base + threadIdx.x; j < end; j += blockDim.x) {
    const int c = j % Cin, q = j / Cin;
    const int t = q % T, o = q / T;
    const int r = t / KW, sx = t - r * KW;
    wf[j] = __float2half_rn(__ldg(W + int64_t(o) * sO + int64_t(c) * sC + int64_t(r) * sR + int64_t(sx) * sS) * sw);
    if (c == 0 && t == 0) tab.alpha[l][o] = isw;
  }
}

// The dgrad operands of the same convs (the W32/A1 convs of DESIGN.md §4p): wt[c][k*k-1-t][o] = wf[o][t][c] and, per
// output channel, gscale = 2^-ew, inv_gscale = 2^ew.  A third launch rather than a store in real_wpack_multi_kernel:
// wt runs along o, wf along c, so one of the two would be written in scattered 2-byte stores; here each block moves a
// 32 x 32 (o, c) tile of one tap through shared memory, reading wf and writing wt in whole rows.  Copying wf's fp16
// bits (not rounding W again) makes wt exactly wf transposed and flipped.  grid = sum of the tensors' tiles,
// block = (32, 8).
struct RealWtTable {
  const uint16_t* wf[kRealPackMax];
  uint16_t* wt[kRealPackMax];
  float* gscale[kRealPackMax];
  float* inv_gscale[kRealPackMax];
  int32_t Cout[kRealPackMax], Cin[kRealPackMax], T[kRealPackMax];
  int32_t tile0[kRealPackMax + 1];        // first tile of tensor l (prefix sums of T * ceil(Cout/32) * ceil(Cin/32))
  int32_t n;
};

__global__ void __launch_bounds__(256)
real_wt_multi_kernel(const __grid_constant__ RealWtTable tab, const uint32_t* __restrict__ amax) {
  __shared__ uint16_t tile[32][33];
  const int b = int(blockIdx.x);
  int l = 0;
  while (l + 1 < tab.n && b >= tab.tile0[l + 1]) ++l;
  const int Cout = tab.Cout[l], Cin = tab.Cin[l], T = tab.T[l];
  const int tc = (Cin + 31) / 32, to = (Cout + 31) / 32;
  const int q = b - tab.tile0[l];
  const int t = q / (to * tc), r = q - t * (to * tc);
  const int o0 = (r / tc) * 32, c0 = (r % tc) * 32;
  const uint16_t* wf = tab.wf[l];
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int o = o0 + i, c = c0 + threadIdx.x;
    if (o < Cout && c < Cin) tile[i][threadIdx.x] = wf[(int64_t(o) * T + t) * Cin + c];
  }
  __syncthreads();
  uint16_t* wt = tab.wt[l];
  for (int i = threadIdx.y; i < 32; i += 8) {
    const int c = c0 + i, o = o0 + threadIdx.x;
    if (c < Cin && o < Cout) wt[(int64_t(c) * T + (T - 1 - t)) * Cout + o] = tile[threadIdx.x][i];
  }
  if (q == 0) {
    const uint32_t a = __ldg(amax + l);
    const float sw = amax_pow2_scale(a, false), isw = amax_pow2_scale(a, true);
    for (int o = threadIdx.y * 32 + threadIdx.x; o < Cout; o += 256) {
      tab.gscale[l][o] = isw;
      tab.inv_gscale[l][o] = sw;
    }
  }
}

// The activation's scale folded into a 3x3 real x real conv's weight vectors (DESIGN.md §4r): x's fp16 operand is
// fp16(x * 2^ex) with ex from x_amax_bits, so alpha[o] = alpha_w[o] * 2^-ex and inv_gscale[o] = inv_gscale_w[o] * 2^-ex
// (powers of two: exact).
__global__ void real_scale_fold_kernel(const uint32_t* __restrict__ x_amax_bits, const float* __restrict__ alpha_w,
                                       const float* __restrict__ inv_gscale_w, int C, float* __restrict__ alpha,
                                       float* __restrict__ inv_gscale) {
  const int o = blockIdx.x * blockDim.x + threadIdx.x;
  if (o >= C) return;
  const float isx = amax_pow2_scale(__ldg(x_amax_bits), true);
  alpha[o] = alpha_w[o] * isx;
  inv_gscale[o] = inv_gscale_w[o] * isx;
}

// Grouped 3x3 weights (DESIGN.md §4t): the banded operands of bdbnn_real_weight_pack_multi_grouped.  Tensor l has
// band B[l] and Cin[l] = Cg channels per group (the weight's second dimension); its wf and wt both have Cout*T*B
// entries, blk0 counts their blocks.
struct RealGroupTable {
  int32_t B[kRealPackMax];
  int32_t blk0[kRealPackMax + 1];
};

__device__ __forceinline__ int real_group_find(const RealGroupTable& gt, int n, int b) {
  int l = 0;
  while (l + 1 < n && b >= gt.blk0[l + 1]) ++l;
  return l;
}

// wf[o][t][cl] = fp16(W[o][c - g(o)][t] * 2^ew) for c = b(o) + cl in o's group, else +0 (b, g: o's band and group
// starts); alpha[o] = 2^-ew.  Coalesced along the output.
__global__ void __launch_bounds__(256)
real_gwpack_multi_kernel(const __grid_constant__ RealWPackTable tab, const __grid_constant__ RealGroupTable gt,
                         const uint32_t* __restrict__ amax) {
  const int l = real_group_find(gt, tab.n, int(blockIdx.x));
  const int Cg = tab.Cin[l], T = tab.T[l], KW = tab.KW[l], B = gt.B[l], n = tab.Cout[l] * T * B;
  const int sO = tab.sO[l], sC = tab.sC[l], sR = tab.sR[l], sS = tab.sS[l];
  const int base = (int(blockIdx.x) - gt.blk0[l]) * kRealPackPerBlock;
  const int end = base + kRealPackPerBlock < n ? base + kRealPackPerBlock : n;
  const uint32_t a = __ldg(amax + l);
  const float sw = amax_pow2_scale(a, false), isw = amax_pow2_scale(a, true);
  const float* W = tab.W[l];
  __half* wf = reinterpret_cast<__half*>(tab.wf[l]);
  for (int j = base + threadIdx.x; j < end; j += blockDim.x) {
    const int cl = j % B, q = j / B;
    const int t = q % T, o = q / T;
    const int cg = (o - o % B) + cl - (o - o % Cg);
    const int r = t / KW, sx = t - r * KW;
    __half v = __float2half_rn(0.f);
    if (cg >= 0 && cg < Cg)
      v = __float2half_rn(__ldg(W + int64_t(o) * sO + int64_t(cg) * sC + int64_t(r) * sR + int64_t(sx) * sS) * sw);
    wf[j] = v;
    if (cl == 0 && t == 0) tab.alpha[l][o] = isw;
  }
}

// wt[c][T-1-t][ol] = wf[b(c) + ol][t][c - b(c)] (wf's bits: the band's transpose, taps flipped); gscale[c] = 2^-ew,
// inv_gscale[c] = 2^ew (Cin = Cout).  Coalesced along the output; wf is read in 2-byte gathers (a band operand is at
// most C * 9 * 64 * 2 bytes).
__global__ void __launch_bounds__(256)
real_gwt_multi_kernel(const __grid_constant__ RealWtTable tab, const __grid_constant__ RealGroupTable gt,
                      const uint32_t* __restrict__ amax) {
  const int l = real_group_find(gt, tab.n, int(blockIdx.x));
  const int T = tab.T[l], B = gt.B[l], n = tab.Cout[l] * T * B;
  const int base = (int(blockIdx.x) - gt.blk0[l]) * kRealPackPerBlock;
  const int end = base + kRealPackPerBlock < n ? base + kRealPackPerBlock : n;
  const uint32_t a = __ldg(amax + l);
  const float sw = amax_pow2_scale(a, false), isw = amax_pow2_scale(a, true);
  const uint16_t* wf = tab.wf[l];
  uint16_t* wt = tab.wt[l];
  for (int j = base + threadIdx.x; j < end; j += blockDim.x) {
    const int ol = j % B, q = j / B;
    const int tt = q % T, c = q / T;
    const int b = c - c % B;
    wt[j] = wf[(int64_t(b + ol) * T + (T - 1 - tt)) * B + (c - b)];
    if (ol == 0 && tt == 0) {
      tab.gscale[l][c] = isw;
      tab.inv_gscale[l][c] = sw;
    }
  }
}

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_real_scale_fold(const uint32_t* x_amax_bits, const float* alpha_w, const float* inv_gscale_w,
                                     int32_t C, float* alpha, float* inv_gscale, void* stream) {
  BDBNN_REQUIRE(C > 0, "real_scale_fold: C must be positive");
  BDBNN_REQUIRE(x_amax_bits && alpha_w && inv_gscale_w && alpha && inv_gscale, "real_scale_fold: NULL pointer");
  real_scale_fold_kernel<<<(C + 127) / 128, 128, 0, cudaStream_t(stream)>>>(x_amax_bits, alpha_w, inv_gscale_w, C,
                                                                            alpha, inv_gscale);
  return check_launch("real_scale_fold_kernel");
}

extern "C" int bdbnn_real_act_pack(const float* x, int64_t n_pix, int32_t C, uint32_t* amax_bits, int32_t have_amax,
                                   uint16_t* xh, void* stream) {
  BDBNN_REQUIRE(n_pix > 0 && C > 0 && (C & 3) == 0, "real_act_pack: needs n_pix > 0 and C a positive multiple of 4");
  BDBNN_REQUIRE(x && amax_bits && xh, "real_act_pack: NULL pointer");
  cudaStream_t st = cudaStream_t(stream);
  // the strided-sample kernels of bdbnn_real_conv_pack at stride 1 over n_pix 1x1 "images"
  const int C4 = C / 4;
  const int64_t total = n_pix * C4;
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = int64_t(num_sms()) * 16;
  if (blocks > cap) blocks = cap;
  if (!have_amax) {
    BDBNN_CUDA(cudaMemsetAsync(amax_bits, 0, sizeof(uint32_t), st));
    real_amax_kernel<<<unsigned(blocks), 256, 0, st>>>(reinterpret_cast<const float4*>(x), 1, 1, C4, 1, 1, 1, total,
                                                       amax_bits);
    int rc = check_launch("real_amax_kernel");
    if (rc) return rc;
  }
  real_pack_x_kernel<<<unsigned(blocks), 256, 0, st>>>(reinterpret_cast<const float4*>(x), 1, 1, C4, 1, 1, 1, total,
                                                       amax_bits, reinterpret_cast<uint2*>(xh));
  return check_launch("real_pack_x_kernel");
}

// Tensor l of a pack's host tables: non-NULL pointers, positive dims and a dense weight.
static int check_weight_tensor(int l, const float* const* W_host, const int32_t* Cout_host, const int32_t* Cin_host,
                               const int32_t* kw_host, const int64_t* strides_host, uint16_t* const* wf_host,
                               float* const* alpha_host, uint16_t* const* wt_host, float* const* gscale_host,
                               float* const* inv_gscale_host) {
  const bool grad = wt_host != nullptr;
  const int k = kw_host[l];
  const int64_t n = int64_t(Cout_host[l]) * Cin_host[l] * k * k;
  const int64_t* st4 = strides_host + 4 * int64_t(l);
  BDBNN_REQUIRE(W_host[l] && wf_host[l] && alpha_host[l], "real_weight_pack_multi: NULL pointer in tensor %d", l);
  BDBNN_REQUIRE(!grad || (wt_host[l] && gscale_host[l] && inv_gscale_host[l]),
                "real_weight_pack_multi: NULL gradient output in tensor %d", l);
  BDBNN_REQUIRE(Cout_host[l] > 0 && Cin_host[l] > 0 && k > 0 && n < (int64_t(1) << 30),
                "real_weight_pack_multi: bad dims in tensor %d", l);
  // dense: the strides are a permutation of the contiguous strides of some dimension order
  int64_t dims[4] = {Cout_host[l], Cin_host[l], k, k}, span = 1;
  bool dense = true;
  for (int d = 0; d < 4; ++d) {
    BDBNN_REQUIRE(st4[d] >= 0 && st4[d] < (int64_t(1) << 30), "real_weight_pack_multi: bad strides in tensor %d", l);
    span += (dims[d] - 1) * st4[d];
  }
  for (int d = 0; d < 4 && dense; ++d)
    for (int e = d + 1; e < 4; ++e)
      if (dims[d] > 1 && dims[e] > 1 && st4[d] == st4[e]) dense = false;
  BDBNN_REQUIRE(dense && span == n, "real_weight_pack_multi: tensor %d is not dense", l);
  return BDBNN_OK;
}

// One host body for both entry points: the gradient outputs (wt, gscale, inv_gscale) come as a group, all NULL or
// all given.  NULL: the two launches and their results are those of the forward-only pack.
static int real_weight_pack_multi(int32_t count, const float* const* W_host, const int32_t* Cout_host,
                                  const int32_t* Cin_host, const int32_t* kw_host, const int64_t* strides_host,
                                  uint32_t* amax_bits, uint16_t* const* wf_host, float* const* alpha_host,
                                  uint16_t* const* wt_host, float* const* gscale_host, float* const* inv_gscale_host,
                                  void* stream) {
  BDBNN_REQUIRE(count >= 0, "real_weight_pack_multi: bad count");
  BDBNN_REQUIRE(count == 0 || (W_host && Cout_host && Cin_host && kw_host && strides_host && amax_bits && wf_host &&
                               alpha_host),
                "real_weight_pack_multi: NULL table");
  const bool grad = wt_host != nullptr;
  BDBNN_REQUIRE((gscale_host != nullptr) == grad && (inv_gscale_host != nullptr) == grad,
                "real_weight_pack_multi: wt, gscale and inv_gscale are given together or not at all");
  // every tensor is checked before the first launch
  for (int l = 0; l < count; ++l) {
    const int rc = check_weight_tensor(l, W_host, Cout_host, Cin_host, kw_host, strides_host, wf_host, alpha_host,
                                       wt_host, gscale_host, inv_gscale_host);
    if (rc) return rc;
  }
  cudaStream_t st = cudaStream_t(stream);
  if (count > 0) BDBNN_CUDA(cudaMemsetAsync(amax_bits, 0, size_t(count) * sizeof(uint32_t), st));
  for (int off = 0; off < count; off += kRealPackMax) {
    const int cnt = count - off < kRealPackMax ? count - off : kRealPackMax;
    RealWPackTable tab;
    memset(&tab, 0, sizeof(tab));
    RealWtTable gtab;
    memset(&gtab, 0, sizeof(gtab));
    tab.n = cnt;
    gtab.n = cnt;
    int64_t blocks = 0, tiles = 0;
    for (int i = 0; i < cnt; ++i) {
      const int l = off + i;
      const int k = kw_host[l];
      const int64_t n = int64_t(Cout_host[l]) * Cin_host[l] * k * k;
      const int64_t* st4 = strides_host + 4 * int64_t(l);
      tab.W[i] = W_host[l]; tab.wf[i] = wf_host[l]; tab.alpha[i] = alpha_host[l];
      tab.Cout[i] = Cout_host[l]; tab.Cin[i] = Cin_host[l]; tab.T[i] = k * k; tab.KW[i] = k;
      tab.sO[i] = int32_t(st4[0]); tab.sC[i] = int32_t(st4[1]); tab.sR[i] = int32_t(st4[2]); tab.sS[i] = int32_t(st4[3]);
      tab.blk0[i] = int32_t(blocks);
      blocks += (n + kRealPackPerBlock - 1) / kRealPackPerBlock;
      if (grad) {
        gtab.wf[i] = wf_host[l]; gtab.wt[i] = wt_host[l];
        gtab.gscale[i] = gscale_host[l]; gtab.inv_gscale[i] = inv_gscale_host[l];
        gtab.Cout[i] = Cout_host[l]; gtab.Cin[i] = Cin_host[l]; gtab.T[i] = k * k;
        gtab.tile0[i] = int32_t(tiles);
        tiles += int64_t(k) * k * ((Cout_host[l] + 31) / 32) * ((Cin_host[l] + 31) / 32);
      }
    }
    BDBNN_REQUIRE(blocks < (int64_t(1) << 31), "real_weight_pack_multi: too many weights");
    tab.blk0[cnt] = int32_t(blocks);
    gtab.tile0[cnt] = int32_t(tiles);
    real_wamax_multi_kernel<<<unsigned(blocks), 256, 0, st>>>(tab, amax_bits + off);
    int rc = check_launch("real_wamax_multi_kernel");
    if (rc) return rc;
    real_wpack_multi_kernel<<<unsigned(blocks), 256, 0, st>>>(tab, amax_bits + off);
    rc = check_launch("real_wpack_multi_kernel");
    if (rc) return rc;
    if (grad) {
      real_wt_multi_kernel<<<unsigned(tiles), dim3(32, 8), 0, st>>>(gtab, amax_bits + off);
      rc = check_launch("real_wt_multi_kernel");
      if (rc) return rc;
    }
  }
  return BDBNN_OK;
}

extern "C" int bdbnn_real_weight_pack_multi(int32_t count, const float* const* W_host, const int32_t* Cout_host,
                                            const int32_t* Cin_host, const int32_t* kw_host,
                                            const int64_t* strides_host, uint32_t* amax_bits,
                                            uint16_t* const* wf_host, float* const* alpha_host, void* stream) {
  return real_weight_pack_multi(count, W_host, Cout_host, Cin_host, kw_host, strides_host, amax_bits, wf_host,
                                alpha_host, nullptr, nullptr, nullptr, stream);
}

extern "C" int bdbnn_real_weight_pack_multi_grad(int32_t count, const float* const* W_host, const int32_t* Cout_host,
                                                 const int32_t* Cin_host, const int32_t* kw_host,
                                                 const int64_t* strides_host, uint32_t* amax_bits,
                                                 uint16_t* const* wf_host, float* const* alpha_host,
                                                 uint16_t* const* wt_host, float* const* gscale_host,
                                                 float* const* inv_gscale_host, void* stream) {
  return real_weight_pack_multi(count, W_host, Cout_host, Cin_host, kw_host, strides_host, amax_bits, wf_host,
                                alpha_host, wt_host, gscale_host, inv_gscale_host, stream);
}

extern "C" int bdbnn_real_conv_pack(const float* x, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t stride,
                                    const float* weight, int32_t Cout, uint16_t* xh, uint32_t* x_amax_bits,
                                    uint16_t* wf, uint16_t* wt, float* alpha, float* gscale, float* inv_gscale,
                                    void* stream) {
  BDBNN_REQUIRE(N > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0 && stride > 0, "real_conv_pack: bad dims");
  BDBNN_REQUIRE((Cin & 3) == 0, "real_conv_pack: Cin must be a multiple of 4");
  BDBNN_REQUIRE(int64_t(Cout) * Cin <= (int64_t(1) << 22), "real_conv_pack: weight too large for the single-block pack");
  BDBNN_REQUIRE(x && weight && xh && x_amax_bits && wf && wt && alpha && gscale && inv_gscale,
                "real_conv_pack: NULL pointer");
  cudaStream_t st = cudaStream_t(stream);
  const int Ho = (H - 1) / stride + 1, Wo = (W - 1) / stride + 1, C4 = Cin / 4;
  const int64_t total = int64_t(N) * Ho * Wo * C4;
  BDBNN_CUDA(cudaMemsetAsync(x_amax_bits, 0, 2 * sizeof(uint32_t), st));   // [0] = max|x|, [1] = max|W|
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = int64_t(num_sms()) * 16;
  if (blocks > cap) blocks = cap;
  real_amax_kernel<<<unsigned(blocks), 256, 0, st>>>(reinterpret_cast<const float4*>(x), H, W, C4, Ho, Wo, stride,
                                                     total, x_amax_bits);
  int rc = check_launch("real_amax_kernel");
  if (rc) return rc;
  real_pack_x_kernel<<<unsigned(blocks), 256, 0, st>>>(reinterpret_cast<const float4*>(x), H, W, C4, Ho, Wo, stride,
                                                       total, x_amax_bits, reinterpret_cast<uint2*>(xh));
  rc = check_launch("real_pack_x_kernel");
  if (rc) return rc;
  int wblocks = int((int64_t(Cout) * Cin + 4095) / 4096);
  if (wblocks > 64) wblocks = 64;
  real_amax_w_kernel<<<wblocks * 4, 256, 0, st>>>(weight, Cout * Cin, x_amax_bits + 1);
  rc = check_launch("real_amax_w_kernel");
  if (rc) return rc;
  real_pack_w_kernel<<<wblocks, 1024, 0, st>>>(weight, Cout, Cin, x_amax_bits, x_amax_bits + 1, reinterpret_cast<__half*>(wf),
                                         reinterpret_cast<__half*>(wt), alpha, gscale, inv_gscale);
  return check_launch("real_pack_w_kernel");
}

// Dense tensors (groups 1) go through real_weight_pack_multi in their order, their amax words first; the grouped ones
// through the banded kernels, their words after.
extern "C" int bdbnn_real_weight_pack_multi_grouped(int32_t count, const float* const* W_host,
                                                    const int32_t* Cout_host, const int32_t* Cin_host,
                                                    const int32_t* kw_host, const int64_t* strides_host,
                                                    const int32_t* groups_host, uint32_t* amax_bits,
                                                    uint16_t* const* wf_host, float* const* alpha_host,
                                                    uint16_t* const* wt_host, float* const* gscale_host,
                                                    float* const* inv_gscale_host, void* stream) {
  BDBNN_REQUIRE(count >= 0, "real_weight_pack_multi_grouped: bad count");
  BDBNN_REQUIRE(count == 0 || (W_host && Cout_host && Cin_host && kw_host && strides_host && groups_host && amax_bits &&
                               wf_host && alpha_host),
                "real_weight_pack_multi_grouped: NULL table");
  const bool grad = wt_host != nullptr;
  BDBNN_REQUIRE((gscale_host != nullptr) == grad && (inv_gscale_host != nullptr) == grad,
                "real_weight_pack_multi_grouped: wt, gscale and inv_gscale are given together or not at all");
  std::vector<int> dense, grouped;
  for (int l = 0; l < count; ++l) {
    const int g = groups_host[l];
    BDBNN_REQUIRE(g >= 1, "real_weight_pack_multi_grouped: groups must be >= 1 in tensor %d", l);
    if (g == 1) { dense.push_back(l); continue; }
    const int rc = check_weight_tensor(l, W_host, Cout_host, Cin_host, kw_host, strides_host, wf_host, alpha_host,
                                       wt_host, gscale_host, inv_gscale_host);
    if (rc) return rc;
    const int cg = Cin_host[l], B = cg < 16 ? 16 : cg;
    BDBNN_REQUIRE(kw_host[l] == 3 && int64_t(cg) * g == Cout_host[l] && (B == 16 || B == 32 || B == 64) &&
                      B % cg == 0 && Cout_host[l] % B == 0,
                  "real_weight_pack_multi_grouped: tensor %d ([%d, %d, %d, %d], groups %d) has no banded operand", l,
                  Cout_host[l], cg, kw_host[l], kw_host[l], g);
    grouped.push_back(l);
  }
  cudaStream_t st = cudaStream_t(stream);
  const int nd = int(dense.size());
  {
    // the dense tensors' host tables, in order (real_weight_pack_multi checks them before its first launch; a
    // grouped tensor launches nothing before that)
    std::vector<const float*> W(nd);
    std::vector<int32_t> co(nd), ci(nd), kw(nd);
    std::vector<int64_t> str(4 * size_t(nd));
    std::vector<uint16_t*> wf(nd), wt(nd);
    std::vector<float*> al(nd), gs(nd), igs(nd);
    for (int i = 0; i < nd; ++i) {
      const int l = dense[i];
      W[i] = W_host[l]; co[i] = Cout_host[l]; ci[i] = Cin_host[l]; kw[i] = kw_host[l];
      for (int d = 0; d < 4; ++d) str[4 * i + d] = strides_host[4 * int64_t(l) + d];
      wf[i] = wf_host[l]; al[i] = alpha_host[l];
      if (grad) { wt[i] = wt_host[l]; gs[i] = gscale_host[l]; igs[i] = inv_gscale_host[l]; }
    }
    const int rc = real_weight_pack_multi(nd, W.data(), co.data(), ci.data(), kw.data(), str.data(), amax_bits,
                                          wf.data(), al.data(), grad ? wt.data() : nullptr,
                                          grad ? gs.data() : nullptr, grad ? igs.data() : nullptr, stream);
    if (rc) return rc;
  }
  const int ng = int(grouped.size());
  uint32_t* gamax = amax_bits + nd;
  if (ng > 0) BDBNN_CUDA(cudaMemsetAsync(gamax, 0, size_t(ng) * sizeof(uint32_t), st));
  for (int off = 0; off < ng; off += kRealPackMax) {
    const int cnt = ng - off < kRealPackMax ? ng - off : kRealPackMax;
    RealWPackTable tab;
    memset(&tab, 0, sizeof(tab));
    RealWtTable wtab;
    memset(&wtab, 0, sizeof(wtab));
    RealGroupTable gt;
    memset(&gt, 0, sizeof(gt));
    tab.n = wtab.n = cnt;
    int64_t wblocks = 0, blocks = 0;
    for (int i = 0; i < cnt; ++i) {
      const int l = grouped[off + i];
      const int cg = Cin_host[l], B = cg < 16 ? 16 : cg;
      const int64_t* st4 = strides_host + 4 * int64_t(l);
      tab.W[i] = W_host[l]; tab.wf[i] = wf_host[l]; tab.alpha[i] = alpha_host[l];
      tab.Cout[i] = Cout_host[l]; tab.Cin[i] = cg; tab.T[i] = 9; tab.KW[i] = 3;
      tab.sO[i] = int32_t(st4[0]); tab.sC[i] = int32_t(st4[1]); tab.sR[i] = int32_t(st4[2]); tab.sS[i] = int32_t(st4[3]);
      tab.blk0[i] = int32_t(wblocks);
      wblocks += (int64_t(Cout_host[l]) * cg * 9 + kRealPackPerBlock - 1) / kRealPackPerBlock;
      gt.B[i] = B;
      gt.blk0[i] = int32_t(blocks);
      blocks += (int64_t(Cout_host[l]) * 9 * B + kRealPackPerBlock - 1) / kRealPackPerBlock;
      if (grad) {
        wtab.wf[i] = wf_host[l]; wtab.wt[i] = wt_host[l];
        wtab.gscale[i] = gscale_host[l]; wtab.inv_gscale[i] = inv_gscale_host[l];
        wtab.Cout[i] = Cout_host[l]; wtab.Cin[i] = cg; wtab.T[i] = 9;
      }
    }
    BDBNN_REQUIRE(blocks < (int64_t(1) << 31), "real_weight_pack_multi_grouped: too many weights");
    tab.blk0[cnt] = int32_t(wblocks);
    gt.blk0[cnt] = int32_t(blocks);
    real_wamax_multi_kernel<<<unsigned(wblocks), 256, 0, st>>>(tab, gamax + off);
    int rc = check_launch("real_wamax_multi_kernel");
    if (rc) return rc;
    real_gwpack_multi_kernel<<<unsigned(blocks), 256, 0, st>>>(tab, gt, gamax + off);
    rc = check_launch("real_gwpack_multi_kernel");
    if (rc) return rc;
    if (grad) {
      real_gwt_multi_kernel<<<unsigned(blocks), 256, 0, st>>>(wtab, gt, gamax + off);
      rc = check_launch("real_gwt_multi_kernel");
      if (rc) return rc;
    }
  }
  return BDBNN_OK;
}
