// Stem convolution (7x7, stride 2, pad 3, 3 -> 64 channels, fp32 in / fp32 out) on wgmma.
//
// The reference runs this layer as an fp32 nn.Conv2d, which cuDNN executes on TF32 tensor cores by
// default (11-bit significands, fp32 accumulate).  Here both operands are rounded to fp16 after a
// per-call power-of-two scale taken from max|x| / max|W| (11-bit significands again, the scale keeps
// every value in fp16's normal range) and accumulated in fp32; the scales are undone in the fp32
// epilogues.  Data layout: the input is repacked once per step as xw = fp16 [N][H+6][WP][4] (3 zero
// pixels on every side, channel 3 = 0), so that the 7x(7x3) receptive field of output pixel (oh, ow)
// is 7 "windows" of 32 consecutive halves starting at row 2*oh + r, pixel 2*ow: a TMA tensor map with
// a 16-byte window stride (overlapping windows) presents that directly as the [pixels][32] operand of
// a 7-tap implicit GEMM (tc_conv.cu) and of the weight-gradient GEMM (tc_wgrad.cu).
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace bdbnn {

__global__ void __launch_bounds__(256)
stem_amax_kernel(const float* __restrict__ x, int64_t n, uint32_t* __restrict__ amax_bits) {
  float m = 0.f;
  const int64_t n4 = n >> 2;
  const float4* x4 = reinterpret_cast<const float4*>(x);
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride) {
    const float4 v = __ldg(x4 + i);
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  for (int64_t i = (n4 << 2) + int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride)
    m = fmaxf(m, fabsf(__ldg(x + i)));
  m = warp_max(m);
  if (!(m < 3.0e38f)) m = 3.0e38f;                     // inf / NaN inputs: keep the scale finite
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(amax_bits, __float_as_uint(m));
}

// xw[n][hp][wp][0..3] = fp16(x[n][c][hp-3][wp-3] * 2^e) (0 outside the image and for channel 3).
// One thread per padded pixel; x is addressed through element strides (NCHW or channels_last).
__global__ void __launch_bounds__(256)
stem_pack_x_kernel(const float* __restrict__ x, int N, int H, int W, int64_t sN, int64_t sC, int64_t sH,
                   int64_t sW, int HP, int WP, const uint32_t* __restrict__ amax_bits, uint2* __restrict__ xw) {
  const float scale = amax_pow2_scale(__ldg(amax_bits), false);
  const int64_t total = int64_t(N) * HP * WP;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += int64_t(gridDim.x) * blockDim.x) {
    const int wp = int(i % WP);
    const int64_t q = i / WP;
    const int hp = int(q % HP), n = int(q / HP);
    const int h = hp - 3, w = wp - 3;
    uint2 out = make_uint2(0u, 0u);
    if (h >= 0 && h < H && w >= 0 && w < W) {
      const float* px = x + n * sN + h * sH + w * sW;
      const __half2 a = __floats2half2_rn(__ldg(px) * scale, __ldg(px + sC) * scale);
      const __half2 b = __floats2half2_rn(__ldg(px + 2 * sC) * scale, 0.f);
      out.x = *reinterpret_cast<const uint32_t*>(&a);
      out.y = *reinterpret_cast<const uint32_t*>(&b);
    }
    xw[i] = out;
  }
}

// One block: wf[o][r][s*4 + c] = fp16(W[o][c][r][s] * 2^ew) (0 for s == 7 or c == 3);
// alpha[o] = 2^-ew * 2^-ex (the forward epilogue's scale).
__global__ void __launch_bounds__(1024)
stem_pack_w_kernel(const float* __restrict__ Wt, const uint32_t* __restrict__ x_amax_bits,
                   __half* __restrict__ wf, float* __restrict__ alpha) {
  __shared__ float red[32];
  __shared__ uint32_t w_amax;
  const int n_w = kStemCout * 3 * 49;
  float m = 0.f;
  for (int i = threadIdx.x; i < n_w; i += blockDim.x) m = fmaxf(m, fabsf(Wt[i]));
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    m = threadIdx.x < (blockDim.x >> 5) ? red[threadIdx.x] : 0.f;
    m = warp_max(m);
    if (!(m < 3.0e38f)) m = 3.0e38f;
    if (threadIdx.x == 0) w_amax = __float_as_uint(m);
  }
  __syncthreads();
  const float sw = amax_pow2_scale(w_amax, false);
  for (int i = threadIdx.x; i < kStemCout * kStemTaps * kStemWin; i += blockDim.x) {
    const int j = i % kStemWin, r = (i / kStemWin) % kStemTaps, o = i / (kStemWin * kStemTaps);
    const int sI = j >> 2, c = j & 3;
    float v = 0.f;
    if (sI < 7 && c < 3) v = Wt[((o * 3 + c) * 7 + r) * 7 + sI] * sw;
    wf[i] = __float2half_rn(v);
  }
  const float inv = amax_pow2_scale(w_amax, true) * amax_pow2_scale(__ldg(x_amax_bits), true);
  for (int o = threadIdx.x; o < kStemCout; o += blockDim.x) alpha[o] = inv;
}

// gW[o][c][r][s] = 2^-ex * 2^-eg * sum_k ws[k][(r*32 + s*4 + c)][o], slices added in order.
__global__ void __launch_bounds__(256)
stem_wgrad_finalize_kernel(const float* __restrict__ ws, int ksplit, const uint32_t* __restrict__ x_amax_bits,
                           const uint32_t* __restrict__ g_amax_bits, float* __restrict__ gW) {
  const int n = kStemCout * 3 * 49;
  const int64_t slice = int64_t(kStemTaps) * kStemWin * kStemCout;
  const float post = amax_pow2_scale(__ldg(x_amax_bits), true) * amax_pow2_scale(__ldg(g_amax_bits), true);
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
    // consecutive threads take consecutive o for one (c, r, s): coalesced workspace reads
    const int o = i % kStemCout, q = i / kStemCout;
    const int sI = q % 7, r = (q / 7) % 7, c = q / 49;
    const int64_t src = (int64_t(r) * kStemWin + sI * 4 + c) * kStemCout + o;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int k = 0;
    for (; k + 3 < ksplit; k += 4) {
      a0 += ws[int64_t(k) * slice + src];
      a1 += ws[int64_t(k + 1) * slice + src];
      a2 += ws[int64_t(k + 2) * slice + src];
      a3 += ws[int64_t(k + 3) * slice + src];
    }
    for (; k < ksplit; ++k) a0 += ws[int64_t(k) * slice + src];
    gW[((o * 3 + c) * 7 + r) * 7 + sI] = ((a0 + a1) + (a2 + a3)) * post;
  }
}

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_stem_supported(int32_t N, int32_t H, int32_t W) {
  StemGeom g;
  return stem_geom(N, H, W, &g) ? 1 : 0;
}

extern "C" size_t bdbnn_stem_xw_bytes(int32_t N, int32_t H, int32_t W) {
  StemGeom g;
  if (!stem_geom(N, H, W, &g)) return 0;
  return size_t(g.img_stride) * size_t(N);
}

extern "C" size_t bdbnn_stem_wgrad_workspace_bytes(int32_t N, int32_t H, int32_t W) {
  StemGeom g;
  if (!stem_geom(N, H, W, &g)) return 0;
  return stem_wgrad_workspace_bytes(g);
}

extern "C" int bdbnn_stem_pack(const float* x, int32_t N, int32_t H, int32_t W, int64_t sN, int64_t sC, int64_t sH,
                               int64_t sW, const float* weight, uint16_t* xw, uint32_t* x_amax_bits,
                               uint16_t* wf, float* alpha, void* stream) {
  StemGeom g;
  BDBNN_REQUIRE(stem_geom(N, H, W, &g), "stem_pack: geometry (%d,%d,%d) not supported (needs (W-1)/2+1 <= 128)", N, H, W);
  BDBNN_REQUIRE(x && weight && xw && x_amax_bits && wf && alpha, "stem_pack: NULL pointer");
  BDBNN_REQUIRE((uintptr_t(xw) & 15) == 0 && (uintptr_t(x) & 15) == 0, "stem_pack: x and xw must be 16-byte aligned");
  cudaStream_t st = cudaStream_t(stream);
  const int64_t n = int64_t(N) * 3 * H * W;
  BDBNN_CUDA(cudaMemsetAsync(x_amax_bits, 0, sizeof(uint32_t), st));
  int64_t blocks = ((n >> 2) + 255) / 256;
  const int64_t cap = int64_t(num_sms()) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  stem_amax_kernel<<<unsigned(blocks), 256, 0, st>>>(x, n, x_amax_bits);
  int rc = check_launch("stem_amax_kernel");
  if (rc) return rc;
  const int64_t total = int64_t(N) * g.HP * g.WP;
  blocks = (total + 255) / 256;
  if (blocks > cap * 4) blocks = cap * 4;
  stem_pack_x_kernel<<<unsigned(blocks), 256, 0, st>>>(x, N, H, W, sN, sC, sH, sW, g.HP, g.WP, x_amax_bits,
                                                       reinterpret_cast<uint2*>(xw));
  rc = check_launch("stem_pack_x_kernel");
  if (rc) return rc;
  stem_pack_w_kernel<<<1, 1024, 0, st>>>(weight, x_amax_bits, reinterpret_cast<__half*>(wf), alpha);
  return check_launch("stem_pack_w_kernel");
}

extern "C" int bdbnn_stem_conv_fwd(const uint16_t* xw, const uint16_t* wf, const float* alpha, float* y, int32_t N,
                                   int32_t H, int32_t W, double* bn_sums, uint32_t* bn_ymax, void* stream) {
  StemGeom g;
  BDBNN_REQUIRE(stem_geom(N, H, W, &g), "stem_conv_fwd: geometry not supported");
  BDBNN_REQUIRE(xw && wf && alpha && y, "stem_conv_fwd: NULL pointer");
  BDBNN_REQUIRE((bn_sums == nullptr) == (bn_ymax == nullptr), "stem_conv_fwd: bn_sums and bn_ymax go together");
  return launch_stem_fwd(xw, wf, alpha, y, g, bn_sums, bn_ymax, cudaStream_t(stream));
}

extern "C" int bdbnn_stem_conv_fwd_eval(const uint16_t* xw, const uint16_t* wf, const float* scale,
                                        const float* shift, float* z, int32_t N, int32_t H, int32_t W, void* stream) {
  StemGeom g;
  BDBNN_REQUIRE(stem_geom(N, H, W, &g), "stem_conv_fwd_eval: geometry not supported");
  BDBNN_REQUIRE(xw && wf && scale && shift && z, "stem_conv_fwd_eval: NULL pointer");
  return launch_stem_eval(xw, wf, scale, shift, z, g, 0, nullptr, cudaStream_t(stream));
}

extern "C" int bdbnn_stem_conv_fwd_eval_relu(const uint16_t* xw, const uint16_t* wf, const float* scale,
                                             const float* shift, float* z, uint32_t* z_amax_bits, int32_t N,
                                             int32_t H, int32_t W, void* stream) {
  StemGeom g;
  BDBNN_REQUIRE(stem_geom(N, H, W, &g), "stem_conv_fwd_eval_relu: geometry not supported");
  BDBNN_REQUIRE(xw && wf && scale && shift && z, "stem_conv_fwd_eval_relu: NULL pointer");
  return launch_stem_eval(xw, wf, scale, shift, z, g, 1, z_amax_bits, cudaStream_t(stream));
}

extern "C" int bdbnn_stem_conv_wgrad(const uint16_t* gys, const uint32_t* g_amax_bits, const uint16_t* xw,
                                     const uint32_t* x_amax_bits, float* gW, int32_t N, int32_t H, int32_t W,
                                     void* workspace, size_t workspace_bytes, void* stream) {
  StemGeom g;
  BDBNN_REQUIRE(stem_geom(N, H, W, &g), "stem_conv_wgrad: geometry not supported");
  BDBNN_REQUIRE(gys && g_amax_bits && xw && x_amax_bits && gW && workspace, "stem_conv_wgrad: NULL pointer");
  cudaStream_t st = cudaStream_t(stream);
  int ksplit = 0;
  int rc = launch_stem_wgrad(gys, xw, static_cast<float*>(workspace), workspace_bytes, &ksplit, g, st);
  if (rc) return rc;
  stem_wgrad_finalize_kernel<<<(kStemCout * 147 + 255) / 256, 256, 0, st>>>(static_cast<const float*>(workspace),
                                                                          ksplit, x_amax_bits, g_amax_bits, gW);
  return check_launch("stem_wgrad_finalize_kernel");
}
