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

}  // namespace bdbnn

using namespace bdbnn;

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
