// CIFAR ResNet stem (3x3 / stride 1 / pad 1, 3 -> Cout channels, fp32) and the gradient of the option-A shortcut,
// on CUDA cores.  See include/bdbnn.h for the contracts and DESIGN.md §4i for the data flow.
//
//   cifar_stem_fwd   : y = conv(x, W) in fp32 (one fmaf per tap, taps in the fixed order c, r, s), with the
//                      BatchNorm batch statistics of y from the same pass (per-block partials, summed in block order)
//   cifar_stem_wgrad : gW = 2^-e * sum_pix x_tap(pix) * gys[pix] from the fp16 operand bn_bwd_pack writes, per-block
//                      partials summed in block order by a finalize kernel
//   pad_shortcut_bwd : gx[n, 2i, 2j, c] += gz[n, i, j, c + pad], the option-A shortcut's gradient added in place
// The stem is tiny (27 MACs per output) and its input has 3 channels: a direct conv on CUDA cores reads x once and
// keeps the reference's fp32 numerics, which the binary layers behind the stem are sensitive to.
#include <cuda_fp16.h>

#include "common.cuh"

namespace bdbnn {

constexpr int kCsThreads = 256;
constexpr int kCsTaps = 27;           // 3 input channels x 3 x 3, tap t = c*9 + r*3 + s (OIHW order)
constexpr int kCsGroup = 16;          // output channels per forward block (blockIdx.y)
constexpr int kCsMaxCout = 64;        // the ResNet stems: 16, 32, 48, 64; VGG-Small's 128 has instances of its own
constexpr int kCsChunk = 128;         // pixels per shared-memory stage of the weight gradient
constexpr int kCsWideCout = 128;

// The 27 taps of output pixel (n, h, w), zero outside the image; x addressed through element strides.
__device__ __forceinline__ void cifar_stem_taps(const float* __restrict__ x, int n, int h, int w, int H, int W,
                                                int64_t sN, int64_t sC, int64_t sH, int64_t sW, float* v) {
#pragma unroll
  for (int c = 0; c < 3; ++c)
#pragma unroll
    for (int r = 0; r < 3; ++r)
#pragma unroll
      for (int s = 0; s < 3; ++s) {
        const int hh = h + r - 1, ww = w + s - 1;
        v[c * 9 + r * 3 + s] = (hh >= 0 && hh < H && ww >= 0 && ww < W)
                                   ? __ldg(x + n * sN + c * sC + hh * sH + ww * sW) : 0.0f;
      }
}

// One thread per output pixel, kCsGroup output channels per block row (blockIdx.y).  If part != NULL, the block's
// per-channel sum y and sum y^2 (warp butterflies in fp32, then the warps in order in fp64) go to its row of part
// ([gridDim.x][2*Cout]) and max|y| to ymax (integer atomicMax of the bits: order-free).
// EVAL: the eval-mode BatchNorm folded into the epilogue instead, y = fp32(fp32(acc * scale[o]) + shift[o]) (no FMA
// contraction, as tc_conv_kernel's eval epilogue), and the bits of max|y| over all channels into ymax[0].
// HT (with EVAL): z = hardtanh(BN_eval(conv)), torch.nn.Hardtanh (NaN stays NaN) — the VGG-Small stem.
template <bool EVAL, bool HT = false>
__global__ void __launch_bounds__(kCsThreads)
cifar_stem_fwd_kernel(const float* __restrict__ x, int N, int H, int W, int64_t sN, int64_t sC, int64_t sH,
                      int64_t sW, const float* __restrict__ wt, int Cout, float* __restrict__ y,
                      double* __restrict__ part, uint32_t* __restrict__ ymax, const float* __restrict__ scale,
                      const float* __restrict__ shift) {
  __shared__ float ws[kCsGroup][kCsTaps];
  __shared__ float red_s[kCsThreads / 32][kCsGroup], red_q[kCsThreads / 32][kCsGroup];
  __shared__ float red_m[kCsThreads / 32][kCsGroup];
  const int o0 = blockIdx.y * kCsGroup;
  for (int i = threadIdx.x; i < kCsGroup * kCsTaps; i += blockDim.x)
    ws[i / kCsTaps][i % kCsTaps] = wt[int64_t(o0) * kCsTaps + i];
  __syncthreads();
  const int64_t n_pix = int64_t(N) * H * W;
  const int64_t p = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  float acc[kCsGroup];
#pragma unroll
  for (int o = 0; o < kCsGroup; ++o) acc[o] = 0.0f;
  const bool valid = p < n_pix;
  if (valid) {
    const int w = int(p % W);
    const int64_t q = p / W;
    const int h = int(q % H), n = int(q / H);
    float v[kCsTaps];
    cifar_stem_taps(x, n, h, w, H, W, sN, sC, sH, sW, v);
#pragma unroll
    for (int t = 0; t < kCsTaps; ++t)
#pragma unroll
      for (int o = 0; o < kCsGroup; ++o) acc[o] = fmaf(v[t], ws[o][t], acc[o]);
    if (EVAL) {
#pragma unroll
      for (int o = 0; o < kCsGroup; ++o)
        acc[o] = __fadd_rn(__fmul_rn(acc[o], __ldg(scale + o0 + o)), __ldg(shift + o0 + o));
      if (HT) {
#pragma unroll
        for (int o = 0; o < kCsGroup; ++o) acc[o] = acc[o] != acc[o] ? acc[o] : fminf(fmaxf(acc[o], -1.0f), 1.0f);
      }
    }
    float4* dst = reinterpret_cast<float4*>(y + p * Cout + o0);
#pragma unroll
    for (int k = 0; k < kCsGroup / 4; ++k)
      dst[k] = make_float4(acc[4 * k], acc[4 * k + 1], acc[4 * k + 2], acc[4 * k + 3]);
  }
  if (EVAL) {   // max|z| as integer bits (NaN above every number): order-free, the same bits every run
    uint32_t m = 0u;
    if (valid)
#pragma unroll
      for (int o = 0; o < kCsGroup; ++o) m = max(m, __float_as_uint(fabsf(acc[o])));
    m = __reduce_max_sync(0xffffffffu, m);
    if ((threadIdx.x & 31) == 0 && m != 0u) atomicMax(ymax, m);
    return;
  }
  if (part == nullptr) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
#pragma unroll
  for (int o = 0; o < kCsGroup; ++o) {
    const float a = valid ? acc[o] : 0.0f;
    const float s = warp_sum(a), q = warp_sum(a * a), m = warp_max(fabsf(a));
    if (lane == 0) { red_s[warp][o] = s; red_q[warp][o] = q; red_m[warp][o] = m; }
  }
  __syncthreads();
  if (threadIdx.x < kCsGroup) {
    const int o = threadIdx.x;
    double su = 0.0, sq = 0.0;
    float mx = 0.0f;
    for (int w = 0; w < kCsThreads / 32; ++w) {
      su += double(red_s[w][o]); sq += double(red_q[w][o]); mx = fmaxf(mx, red_m[w][o]);
    }
    double* row = part + int64_t(blockIdx.x) * 2 * Cout;
    row[o0 + o] = su;
    row[Cout + o0 + o] = sq;
    atomicMax(ymax + o0 + o, __float_as_uint(mx));
  }
}

static int cifar_stem_wgrad_grid(int64_t n_pix) {
  int64_t blocks = (n_pix + kCsChunk - 1) / kCsChunk;
  const int64_t cap = int64_t(num_sms()) * 4;
  if (blocks > cap) blocks = cap;
  return int(blocks < 1 ? 1 : blocks);
}

// Block b stages pixel chunks b, b + gridDim.x, ... (x taps [27][chunk] as floats, gradient [chunk][Cout] as GT: float
// for the ResNet stems, the fp16 values themselves for 128 channels, which keeps them under 48 KB) and every
// thread adds, in pixel order, the terms of the outputs idx = tid + k*256 (o = idx % Cout, t = idx / Cout) in fp32.
// The block's sums go to its row of part ([gridDim.x][Cout*27], index o*27 + t = OIHW).
template <int MAXC, typename GT>
__global__ void __launch_bounds__(kCsThreads)
cifar_stem_wgrad_kernel(const float* __restrict__ x, int N, int H, int W, int64_t sN, int64_t sC, int64_t sH,
                        int64_t sW, const __half* __restrict__ gys, int Cout, double* __restrict__ part) {
  constexpr int kCsOutPerThread = MAXC * kCsTaps / kCsThreads + 1;
  __shared__ float xs[kCsTaps][kCsChunk + 1];
  __shared__ GT gs[kCsChunk][MAXC];
  const int64_t n_pix = int64_t(N) * H * W;
  const int64_t n_chunks = (n_pix + kCsChunk - 1) / kCsChunk;
  const int n_out = Cout * kCsTaps;
  float acc[kCsOutPerThread];
#pragma unroll
  for (int k = 0; k < kCsOutPerThread; ++k) acc[k] = 0.0f;
  for (int64_t ch = blockIdx.x; ch < n_chunks; ch += gridDim.x) {
    const int64_t p0 = ch * kCsChunk;
    const int np = int(n_pix - p0 < kCsChunk ? n_pix - p0 : kCsChunk);
    __syncthreads();                     // the previous chunk's reads are done
    if (threadIdx.x < kCsChunk) {
      const int j = threadIdx.x;
      float v[kCsTaps];
      if (j < np) {
        const int64_t p = p0 + j;
        const int w = int(p % W);
        const int64_t q = p / W;
        cifar_stem_taps(x, int(q / H), int(q % H), w, H, W, sN, sC, sH, sW, v);
      } else {
#pragma unroll
        for (int t = 0; t < kCsTaps; ++t) v[t] = 0.0f;
      }
#pragma unroll
      for (int t = 0; t < kCsTaps; ++t) xs[t][j] = v[t];
    }
    for (int i = threadIdx.x; i < kCsChunk * Cout; i += blockDim.x) {
      const int j = i / Cout, o = i - j * Cout;
      gs[j][o] = j < np ? GT(gys[(p0 + j) * Cout + o]) : GT(0.0f);
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < kCsOutPerThread; ++k) {
      const int idx = threadIdx.x + k * kCsThreads;
      if (idx >= n_out) break;
      const int o = idx % Cout, t = idx / Cout;
      float a = acc[k];
      for (int j = 0; j < np; ++j) a = fmaf(xs[t][j], float(gs[j][o]), a);
      acc[k] = a;
    }
  }
  double* row = part + int64_t(blockIdx.x) * n_out;
#pragma unroll
  for (int k = 0; k < kCsOutPerThread; ++k) {
    const int idx = threadIdx.x + k * kCsThreads;
    if (idx >= n_out) break;
    const int o = idx % Cout, t = idx / Cout;
    row[o * kCsTaps + t] = double(acc[k]);
  }
}

// gW[i] = float(2^-e * sum over blocks b, in order, of part[b][i]); 2^-e undoes the scale of the fp16 operand.
__global__ void __launch_bounds__(kCsThreads)
cifar_stem_wgrad_finalize_kernel(const double* __restrict__ part, int nparts, int n_out,
                                 const uint32_t* __restrict__ g_amax_bits, float* __restrict__ gW) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_out) return;
  double s = 0.0;
  for (int b = 0; b < nparts; ++b) s += part[int64_t(b) * n_out + i];
  gW[i] = float(s * double(amax_pow2_scale(__ldg(g_amax_bits), true)));
}

// gx[n][2i][2j][c] += gz[n][i][j][c + pad], one float4 of channels per thread and step.
__global__ void __launch_bounds__(kCsThreads)
pad_shortcut_bwd_kernel(const float4* __restrict__ gz, float4* __restrict__ gx, int64_t total4, int H, int W, int Ho,
                        int Wo, int Cin4, int C4, int pad4) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total4;
       i += int64_t(gridDim.x) * blockDim.x) {
    const int c4 = int(i % Cin4);
    int64_t q = i / Cin4;
    const int j = int(q % Wo);
    q /= Wo;
    const int hi = int(q % Ho);
    const int64_t n = q / Ho;
    const float4 g = __ldg(gz + ((n * Ho + hi) * Wo + j) * C4 + pad4 + c4);
    float4* d = gx + ((n * H + 2 * hi) * int64_t(W) + 2 * j) * Cin4 + c4;
    float4 a = *d;
    a.x += g.x; a.y += g.y; a.z += g.z; a.w += g.w;
    *d = a;
  }
}

static bool cifar_stem_cout_ok(int Cout) {
  return Cout % kCsGroup == 0 && ((Cout >= kCsGroup && Cout <= kCsMaxCout) || Cout == kCsWideCout);
}

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_cifar_stem_fwd(const float* x, int32_t N, int32_t H, int32_t W, int64_t sN, int64_t sC,
                                    int64_t sH, int64_t sW, const float* weight, int32_t Cout, float* y,
                                    double* bn_sums, uint32_t* bn_ymax, void* stream) {
  BDBNN_REQUIRE(N > 0 && H > 0 && W > 0, "cifar_stem_fwd: non-positive dims");
  BDBNN_REQUIRE(cifar_stem_cout_ok(Cout), "cifar_stem_fwd: Cout must be 16, 32, 48, 64 or 128");
  BDBNN_REQUIRE(x && weight && y, "cifar_stem_fwd: NULL pointer");
  BDBNN_REQUIRE((bn_sums == nullptr) == (bn_ymax == nullptr), "cifar_stem_fwd: bn_sums and bn_ymax go together");
  BDBNN_REQUIRE((uintptr_t(y) & 15) == 0, "cifar_stem_fwd: y must be 16-byte aligned");
  cudaStream_t st = cudaStream_t(stream);
  const int64_t n_pix = int64_t(N) * H * W;
  const dim3 grid(unsigned((n_pix + kCsThreads - 1) / kCsThreads), unsigned(Cout / kCsGroup));
  double* part = nullptr;
  if (bn_sums != nullptr) {
    BDBNN_CUDA(cudaMemsetAsync(bn_sums, 0, size_t(2 * Cout) * sizeof(double), st));
    BDBNN_CUDA(cudaMemsetAsync(bn_ymax, 0, size_t(Cout) * sizeof(uint32_t), st));
    int rc = det_sums_alloc(&part, grid.x, 2 * Cout, st);
    if (rc) return rc;
  }
  cifar_stem_fwd_kernel<false><<<grid, kCsThreads, 0, st>>>(x, N, H, W, sN, sC, sH, sW, weight, Cout, y, part,
                                                            bn_ymax, nullptr, nullptr);
  int rc = check_launch("cifar_stem_fwd_kernel");
  if (part == nullptr) return rc;
  if (rc) { cudaFreeAsync(part, st); return rc; }
  return det_sums_finish(part, grid.x, 2 * Cout, bn_sums, st);
}

template <bool HT>
static int cifar_stem_eval_launch(const float* x, int32_t N, int32_t H, int32_t W, int64_t sN, int64_t sC, int64_t sH,
                                  int64_t sW, const float* weight, int32_t Cout, const float* scale, const float* shift,
                                  float* z, uint32_t* z_amax_bits, void* stream) {
  BDBNN_REQUIRE(x && weight && scale && shift && z && z_amax_bits, "cifar_stem_fwd_eval: NULL pointer");
  BDBNN_REQUIRE((uintptr_t(z) & 15) == 0, "cifar_stem_fwd_eval: z must be 16-byte aligned");
  cudaStream_t st = cudaStream_t(stream);
  const int64_t n_pix = int64_t(N) * H * W;
  const dim3 grid(unsigned((n_pix + kCsThreads - 1) / kCsThreads), unsigned(Cout / kCsGroup));
  BDBNN_CUDA(cudaMemsetAsync(z_amax_bits, 0, sizeof(uint32_t), st));
  cifar_stem_fwd_kernel<true, HT><<<grid, kCsThreads, 0, st>>>(x, N, H, W, sN, sC, sH, sW, weight, Cout, z, nullptr,
                                                               z_amax_bits, scale, shift);
  return check_launch("cifar_stem_fwd_eval_kernel");
}

extern "C" int bdbnn_cifar_stem_fwd_eval(const float* x, int32_t N, int32_t H, int32_t W, int64_t sN, int64_t sC,
                                         int64_t sH, int64_t sW, const float* weight, int32_t Cout, const float* scale,
                                         const float* shift, float* z, uint32_t* z_amax_bits, void* stream) {
  BDBNN_REQUIRE(N > 0 && H > 0 && W > 0, "cifar_stem_fwd_eval: non-positive dims");
  BDBNN_REQUIRE(cifar_stem_cout_ok(Cout) && Cout <= kCsMaxCout, "cifar_stem_fwd_eval: Cout must be 16, 32, 48 or 64");
  return cifar_stem_eval_launch<false>(x, N, H, W, sN, sC, sH, sW, weight, Cout, scale, shift, z, z_amax_bits, stream);
}

extern "C" int bdbnn_cifar_stem_fwd_eval_hardtanh(const float* x, int32_t N, int32_t H, int32_t W, int64_t sN,
                                                  int64_t sC, int64_t sH, int64_t sW, const float* weight, int32_t Cout,
                                                  const float* scale, const float* shift, float* z,
                                                  uint32_t* z_amax_bits, void* stream) {
  BDBNN_REQUIRE(N > 0 && H > 0 && W > 0, "cifar_stem_fwd_eval_hardtanh: non-positive dims");
  BDBNN_REQUIRE(cifar_stem_cout_ok(Cout), "cifar_stem_fwd_eval_hardtanh: Cout must be 16, 32, 48, 64 or 128");
  return cifar_stem_eval_launch<true>(x, N, H, W, sN, sC, sH, sW, weight, Cout, scale, shift, z, z_amax_bits, stream);
}

extern "C" size_t bdbnn_cifar_stem_wgrad_workspace_bytes(int32_t N, int32_t H, int32_t W, int32_t Cout) {
  if (N <= 0 || H <= 0 || W <= 0 || !cifar_stem_cout_ok(Cout)) return 0;
  return size_t(cifar_stem_wgrad_grid(int64_t(N) * H * W)) * size_t(Cout) * kCsTaps * sizeof(double);
}

extern "C" int bdbnn_cifar_stem_wgrad(const float* x, int32_t N, int32_t H, int32_t W, int64_t sN, int64_t sC,
                                      int64_t sH, int64_t sW, const uint16_t* gys, const uint32_t* g_amax_bits,
                                      int32_t Cout, float* gW, void* workspace, size_t workspace_bytes, void* stream) {
  BDBNN_REQUIRE(N > 0 && H > 0 && W > 0, "cifar_stem_wgrad: non-positive dims");
  BDBNN_REQUIRE(cifar_stem_cout_ok(Cout), "cifar_stem_wgrad: Cout must be 16, 32, 48, 64 or 128");
  BDBNN_REQUIRE(x && gys && g_amax_bits && gW && workspace, "cifar_stem_wgrad: NULL pointer");
  BDBNN_REQUIRE(workspace_bytes >= bdbnn_cifar_stem_wgrad_workspace_bytes(N, H, W, Cout),
                "cifar_stem_wgrad: workspace too small (needs bdbnn_cifar_stem_wgrad_workspace_bytes)");
  cudaStream_t st = cudaStream_t(stream);
  const int grid = cifar_stem_wgrad_grid(int64_t(N) * H * W);
  double* part = static_cast<double*>(workspace);
  const __half* gh = reinterpret_cast<const __half*>(gys);
  if (Cout <= kCsMaxCout)
    cifar_stem_wgrad_kernel<kCsMaxCout, float><<<grid, kCsThreads, 0, st>>>(x, N, H, W, sN, sC, sH, sW, gh, Cout, part);
  else
    cifar_stem_wgrad_kernel<kCsWideCout, __half><<<grid, kCsThreads, 0, st>>>(x, N, H, W, sN, sC, sH, sW, gh, Cout,
                                                                              part);
  int rc = check_launch("cifar_stem_wgrad_kernel");
  if (rc) return rc;
  const int n_out = Cout * kCsTaps;
  cifar_stem_wgrad_finalize_kernel<<<(n_out + kCsThreads - 1) / kCsThreads, kCsThreads, 0, st>>>(part, grid, n_out,
                                                                                                g_amax_bits, gW);
  return check_launch("cifar_stem_wgrad_finalize_kernel");
}

extern "C" int bdbnn_pad_shortcut_bwd(const float* gz, float* gx, int32_t N, int32_t H, int32_t W, int32_t Cin,
                                      int32_t Cout, int32_t pad, void* stream) {
  BDBNN_REQUIRE(N > 0 && H > 0 && W > 0 && Cin > 0 && Cout > 0, "pad_shortcut_bwd: non-positive dims");
  BDBNN_REQUIRE(Cin % 4 == 0 && Cout % 4 == 0 && pad >= 0 && pad % 4 == 0 && pad + Cin <= Cout,
                "pad_shortcut_bwd: needs Cin, Cout, pad multiples of 4 and pad + Cin <= Cout");
  BDBNN_REQUIRE(gz && gx, "pad_shortcut_bwd: NULL pointer");
  BDBNN_REQUIRE((uintptr_t(gz) & 15) == 0 && (uintptr_t(gx) & 15) == 0, "pad_shortcut_bwd: 16-byte alignment needed");
  cudaStream_t st = cudaStream_t(stream);
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const int64_t total4 = int64_t(N) * Ho * Wo * (Cin / 4);
  int64_t blocks = (total4 + kCsThreads - 1) / kCsThreads;
  const int64_t cap = int64_t(num_sms()) * 8;
  if (blocks > cap) blocks = cap;
  pad_shortcut_bwd_kernel<<<unsigned(blocks), kCsThreads, 0, st>>>(reinterpret_cast<const float4*>(gz),
                                                                   reinterpret_cast<float4*>(gx), total4, H, W, Ho, Wo,
                                                                   Cin / 4, Cout / 4, pad / 4);
  return check_launch("pad_shortcut_bwd_kernel");
}
