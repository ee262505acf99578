// Fused BatchNorm(train) + residual add + sign/pack around the binary conv (SURVEY.md §8f rank 1: "the
// step either side of the conv").  The binary conv writes y; these kernels replace the cuDNN BN
// forward/backward, the ATen residual adds and the separate act_pack / grad_amax / grad_pack passes:
//
//   forward : bn_stats (1 read of y)  ->  bn_finalize ([C] math + running stats)
//             bn_apply_add_pack: z = y*a[c] + b[c] (+ residual)  [+ sign bits, STE mask bits and the +-1
//             16-bit copy of z, i.e. the NEXT conv's act_pack, in the same pass]
//   backward: bn_bwd_reduce (1 read of gz,y: sum gz, sum gz*yhat, max|gz| per channel)
//             bn_bwd_bound  ([C] math: dgamma, dbeta, per-channel constants, FP16S scale from a bound)
//             bn_bwd_pack   (1 read of gz,y -> gys = 16-bit operand of dgrad_tc / wgrad_tc; the fp32
//                            conv-output gradient is never materialised)
// Per element: forward 4 + 12(+2.25) bytes instead of 12 (BN) + 12 (add) + 6.25 (pack);
//              backward 8 + 10 bytes instead of ~20 (BN bwd) + 4 (amax) + 6 (pack).
// All tensors fp32 NHWC [n_pix][C], C % 4 == 0 (packing: C % 32 == 0).
#include <cuda_fp16.h>

#include "common.cuh"

namespace bdbnn {

constexpr int kBnThreads = 256;

__device__ __forceinline__ uint32_t bn_pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ uint32_t bn_pack_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}
__device__ __forceinline__ float bn_bf16_round(float v) {
  return __uint_as_float(bn_pack_bf16x2(0.f, v) & 0xffff0000u);
}

// y operand of the fused units: fp32 (y itself) or the exact int16 accumulator y_int with y = alpha[c]*y_int
// (bdbnn_binconv_fwd_tc_i16).  The loaders return y_int as floats for I16 — callers fold alpha into their
// per-channel constants, which is exact in the same sense (one fp32 multiply either way).
template <bool I16>
__device__ __forceinline__ float4 load_y4(const void* __restrict__ y, int64_t i) {
  if (I16) {
    const uint2 r = __ldcs(reinterpret_cast<const uint2*>(y) + i);
    return make_float4(float(int16_t(r.x & 0xffffu)), float(int16_t(r.x >> 16)), float(int16_t(r.y & 0xffffu)),
                       float(int16_t(r.y >> 16)));
  }
  return __ldcs(reinterpret_cast<const float4*>(y) + i);
}

// Per-channel (sum a, sum b, max c) over pixels; thread = one float4 channel group, strided over pixels.
// Each block adds its threads' partials of a channel in thread order and writes them to its row of `part`
// ([gridDim.x][2C], summed in block order by det_sums_finish): the sums are the same in every run.
// The block tail shared with pool2_i16_kernel: thread partials (sa, sb) of channel group c4 and max bits mx go to the
// block's row of `part` (threads added in thread order) and to maxbits.  shs: [2][blockDim] float4, then [C] uint32
// zeroed by the caller before its first __syncthreads.
__device__ __forceinline__ void block_partials(float4* shs, uint32_t* shm, int C4, int c4, float4 sa, float4 sb,
                                               float4 mx, double* __restrict__ part, uint32_t* __restrict__ maxbits) {
  const int C = C4 * 4;
  const int c = c4 * 4;
  shs[threadIdx.x] = sa;
  shs[blockDim.x + threadIdx.x] = sb;
  atomicMax(&shm[c + 0], __float_as_uint(mx.x)); atomicMax(&shm[c + 1], __float_as_uint(mx.y));
  atomicMax(&shm[c + 2], __float_as_uint(mx.z)); atomicMax(&shm[c + 3], __float_as_uint(mx.w));
  __syncthreads();
  const int first = int((int64_t(blockIdx.x) * blockDim.x) % C4);     // channel group of thread 0
  double* row = part + int64_t(blockIdx.x) * 2 * C;
  for (int g = threadIdx.x; g < C4; g += blockDim.x) {
    float4 a = make_float4(0, 0, 0, 0), b = a;
    for (int t = (g - first + C4) % C4; t < int(blockDim.x); t += C4) {
      const float4 u = shs[t], v = shs[blockDim.x + t];
      a.x += u.x; a.y += u.y; a.z += u.z; a.w += u.w;
      b.x += v.x; b.y += v.y; b.z += v.z; b.w += v.w;
    }
    row[4 * g + 0] = a.x; row[4 * g + 1] = a.y; row[4 * g + 2] = a.z; row[4 * g + 3] = a.w;
    row[C + 4 * g + 0] = b.x; row[C + 4 * g + 1] = b.y; row[C + 4 * g + 2] = b.z; row[C + 4 * g + 3] = b.w;
  }
  for (int i = threadIdx.x; i < C; i += blockDim.x) atomicMax(maxbits + i, shm[i]);
}

// Hardtanh's gradient mask on the pre-activation u = fmaf(y, a, b) of the forward (the same fp32 operation, so the
// same u): gz passes where -1 < u < 1, strictly, and not at NaN (DESIGN.md §4n).
__device__ __forceinline__ float4 htanh_mask(float4 g, const float4 v, const float4 a, const float4 b) {
  const float ux = fmaf(v.x, a.x, b.x), uy = fmaf(v.y, a.y, b.y), uz = fmaf(v.z, a.z, b.z), uw = fmaf(v.w, a.w, b.w);
  g.x = (ux > -1.0f && ux < 1.0f) ? g.x : 0.0f;
  g.y = (uy > -1.0f && uy < 1.0f) ? g.y : 0.0f;
  g.z = (uz > -1.0f && uz < 1.0f) ? g.z : 0.0f;
  g.w = (uw > -1.0f && uw < 1.0f) ? g.w : 0.0f;
  return g;
}

// torch.nn.Hardtanh: clamp to [-1, 1], NaN stays NaN
__device__ __forceinline__ float htanh(float u) { return u != u ? u : fminf(fmaxf(u, -1.0f), 1.0f); }

// torch.relu bit for bit: 0 below 0, u itself otherwise (-0.0 and NaN stay)
__device__ __forceinline__ float relu_f(float u) { return u < 0.0f ? 0.0f : u; }

// ReLU's gradient bit as torch's threshold_backward takes it from z: 1 <=> !(z <= 0), so 1 at NaN too
__device__ __forceinline__ uint32_t relu_bits4(const float4 o) {
  return uint32_t(!(o.x <= 0.0f)) | (uint32_t(!(o.y <= 0.0f)) << 1) | (uint32_t(!(o.z <= 0.0f)) << 2) |
         (uint32_t(!(o.w <= 0.0f)) << 3);
}

// ReLU's gradient mask from the bit words [pix][C/32] the forward wrote (relu_bits4), for float4 element i of an
// NHWC tensor with C % 32 == 0: word i / 8, bits 4 * (i % 8) ..  A select, not a product, as torch's
// threshold_backward: a NaN or inf of gz where z <= 0 gives 0.
__device__ __forceinline__ float4 relu_mask(float4 g, const uint32_t* __restrict__ words, int64_t i) {
  const uint32_t m = __ldg(words + (i >> 3)) >> ((i & 7) * 4);
  g.x = (m & 1u) ? g.x : 0.0f;
  g.y = (m & 2u) ? g.y : 0.0f;
  g.z = (m & 4u) ? g.z : 0.0f;
  g.w = (m & 8u) ? g.w : 0.0f;
  return g;
}

// HT (backward only): gz is first multiplied by Hardtanh's mask on u = fmaf(y, ab[c], ab[C + c]) (ab: the forward's
// bn_finalize output, alpha folded in for I16).  RM (backward only): gz is first masked by relu_mask(rmask).
template <bool BWD, bool I16 = false, bool HT = false, bool RM = false>
__global__ void __launch_bounds__(kBnThreads)
bn_reduce_kernel(const float4* __restrict__ p0, const void* __restrict__ p1, const float* __restrict__ mean,
                 const float* __restrict__ invstd, int64_t n_pix, int C4, double* __restrict__ part,
                 uint32_t* __restrict__ maxbits, const float* __restrict__ alpha = nullptr,
                 const float* __restrict__ ab = nullptr, const uint32_t* __restrict__ rmask = nullptr) {
  extern __shared__ float4 shs[];             // [2][blockDim] per-thread partials, then [C] max bits
  const int C = C4 * 4;
  uint32_t* shm = reinterpret_cast<uint32_t*>(shs + 2 * blockDim.x);   // non-negative floats order like uints
  for (int i = threadIdx.x; i < C; i += blockDim.x) shm[i] = 0u;
  __syncthreads();
  const int64_t gtid = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t nthreads = int64_t(gridDim.x) * blockDim.x;   // multiple of C4 (host guarantees)
  const int c4 = int(gtid % C4);
  const int64_t p_step = nthreads / C4;
  float4 mu = make_float4(0, 0, 0, 0), is = make_float4(1, 1, 1, 1);
  if (BWD) {
    mu = *reinterpret_cast<const float4*>(mean + c4 * 4);
    is = *reinterpret_cast<const float4*>(invstd + c4 * 4);
    if (I16) {     // yhat = (alpha*yi - mean)*invstd = (yi - mean/alpha) * (alpha*invstd); alpha == 0 -> yhat = -mean*invstd
      const float4 al = *reinterpret_cast<const float4*>(alpha + c4 * 4);
      // keep the exact form: yhat = yi*(alpha*is) - mean*is, expressed through (v - mu')*is' with v = yi
      mu = make_float4(mu.x * is.x, mu.y * is.y, mu.z * is.z, mu.w * is.w);           // mean*invstd
      is = make_float4(al.x * is.x, al.y * is.y, al.z * is.z, al.w * is.w);           // alpha*invstd
    }
  }
  float4 ha = make_float4(0, 0, 0, 0), hb = ha;
  if (HT) {
    ha = *reinterpret_cast<const float4*>(ab + c4 * 4);
    hb = *reinterpret_cast<const float4*>(ab + C + c4 * 4);
  }
  float4 sa = make_float4(0, 0, 0, 0), sb = sa, mx = sa;
#pragma unroll 8
  for (int64_t p = gtid / C4; p < n_pix; p += p_step) {
    float4 u = __ldcs(p0 + p * C4 + c4);
    if (BWD) {   // u = gz, v = y:  a = gz, b = gz * yhat, c = |gz|
      const float4 v = load_y4<I16>(p1, p * C4 + c4);
      if (HT) u = htanh_mask(u, v, ha, hb);
      if (RM) u = relu_mask(u, rmask, p * C4 + c4);
      sa.x += u.x; sa.y += u.y; sa.z += u.z; sa.w += u.w;
      if (I16) {
        sb.x += u.x * fmaf(v.x, is.x, -mu.x); sb.y += u.y * fmaf(v.y, is.y, -mu.y);
        sb.z += u.z * fmaf(v.z, is.z, -mu.z); sb.w += u.w * fmaf(v.w, is.w, -mu.w);
      } else {
        sb.x += u.x * ((v.x - mu.x) * is.x); sb.y += u.y * ((v.y - mu.y) * is.y);
        sb.z += u.z * ((v.z - mu.z) * is.z); sb.w += u.w * ((v.w - mu.w) * is.w);
      }
    } else {     // u = y:  a = y, b = y*y, c = |y|
      sa.x += u.x; sa.y += u.y; sa.z += u.z; sa.w += u.w;
      sb.x += u.x * u.x; sb.y += u.y * u.y; sb.z += u.z * u.z; sb.w += u.w * u.w;
    }
    mx.x = fmaxf(mx.x, fabsf(u.x)); mx.y = fmaxf(mx.y, fabsf(u.y));
    mx.z = fmaxf(mx.z, fabsf(u.z)); mx.w = fmaxf(mx.w, fabsf(u.w));
  }
  block_partials(shs, shm, C4, c4, sa, sb, mx, part, maxbits);
}

// ---- run-to-run deterministic sums across blocks ----------------------------------------------------
// out[col] (+)= sum over parts p in [p0, p1) of in[p][col]: 32 columns x 32 part lanes per block; each lane adds its
// parts in order, the lanes are then added in lane order.  gridDim.y > 1: one output row per part chunk.
constexpr int kDetChunk = 1024;
__global__ void __launch_bounds__(1024)
det_reduce_kernel(const double* __restrict__ in, int64_t nparts, int width, double* __restrict__ out, int add) {
  __shared__ double red[32][33];
  const int col = blockIdx.x * 32 + threadIdx.x, lane = threadIdx.y;
  const int64_t p0 = int64_t(blockIdx.y) * kDetChunk;
  const int64_t p1 = p0 + kDetChunk < nparts ? p0 + kDetChunk : nparts;
  double acc = 0.0;
  if (col < width)
    for (int64_t p = p0 + lane; p < p1; p += 32) acc += in[p * width + col];
  red[lane][threadIdx.x] = acc;
  __syncthreads();
  if (lane == 0 && col < width) {
    double t = 0.0;
    for (int l = 0; l < 32; ++l) t += red[l][threadIdx.x];
    if (add) out[col] += t;
    else out[int64_t(blockIdx.y) * width + col] = t;
  }
}

int det_sums_alloc(double** part, int64_t nparts, int width, cudaStream_t st) {
  // keep freed scratch in the device's default pool instead of returning it at every synchronisation (release
  // threshold 0 would make each eager call map fresh memory)
  static const bool pool_ready = [] {
    int dev = 0;
    cudaMemPool_t pool;
    if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetDefaultMemPool(&pool, dev) != cudaSuccess) return false;
    uint64_t keep = UINT64_MAX;
    return cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep) == cudaSuccess;
  }();
  (void)pool_ready;
  BDBNN_CUDA(cudaMallocAsync(reinterpret_cast<void**>(part), size_t(nparts) * width * sizeof(double), st));
  return BDBNN_OK;
}

int det_sums_finish(double* part, int64_t nparts, int width, double* sums, cudaStream_t st) {
  double* cur = part;
  while (nparts > kDetChunk) {
    const int64_t m = (nparts + kDetChunk - 1) / kDetChunk;
    double* next = nullptr;
    const cudaError_t ea = cudaMallocAsync(reinterpret_cast<void**>(&next), size_t(m) * width * sizeof(double), st);
    if (ea != cudaSuccess) {
      cudaFreeAsync(cur, st);
      set_error("det_sums_finish: cudaMallocAsync failed: %s", cudaGetErrorString(ea));
      return BDBNN_ERR_CUDA;
    }
    det_reduce_kernel<<<dim3(unsigned((width + 31) / 32), unsigned(m)), dim3(32, 32), 0, st>>>(cur, nparts, width, next, 0);
    const int rc = check_launch("det_reduce_kernel");
    cudaFreeAsync(cur, st);
    if (rc) { cudaFreeAsync(next, st); return rc; }
    cur = next;
    nparts = m;
  }
  det_reduce_kernel<<<dim3(unsigned((width + 31) / 32), 1), dim3(32, 32), 0, st>>>(cur, nparts, width, sums, 1);
  const int rc = check_launch("det_reduce_kernel");
  BDBNN_CUDA(cudaFreeAsync(cur, st));
  return rc;
}

// bn_reduce_kernel over `grid` blocks with its partials summed into sums[2C] (pre-zeroed or accumulated)
template <bool BWD, bool I16 = false, bool HT = false, bool RM = false>
static int bn_reduce_launch(int grid, const float4* p0, const void* p1, const float* mean, const float* invstd,
                            int64_t n_pix, int C4, double* sums, uint32_t* maxbits, const float* alpha,
                            cudaStream_t st, const float* ab = nullptr, const uint32_t* rmask = nullptr) {
  double* part = nullptr;
  int rc = det_sums_alloc(&part, grid, 8 * C4, st);
  if (rc) return rc;
  bn_reduce_kernel<BWD, I16, HT, RM><<<grid, kBnThreads, 2 * kBnThreads * sizeof(float4) +
                                       size_t(4 * C4) * sizeof(uint32_t), st>>>(p0, p1, mean, invstd, n_pix, C4, part,
                                                                                maxbits, alpha, ab, rmask);
  rc = check_launch(BWD ? "bn_reduce_kernel<bwd>" : "bn_reduce_kernel<fwd>");
  if (rc) { cudaFreeAsync(part, st); return rc; }
  return det_sums_finish(part, grid, 8 * C4, sums, st);
}

// [C] math of the forward: mean, invstd, a = gamma*invstd, b = beta - mean*a, running statistics
// (torch.nn.BatchNorm2d: biased variance for normalisation, unbiased for running_var).
__global__ void bn_finalize_kernel(const double* __restrict__ sums, int64_t n_pix, int C, float eps,
                                   const float* __restrict__ gamma, const float* __restrict__ beta,
                                   float* __restrict__ mean, float* __restrict__ invstd, float* __restrict__ a,
                                   float* __restrict__ b, float* __restrict__ running_mean,
                                   float* __restrict__ running_var, float momentum,
                                   const float* __restrict__ alpha_i16 = nullptr) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double n = double(n_pix);
  const double m = sums[c] / n;
  double var = sums[C + c] / n - m * m;
  if (var < 0.0) var = 0.0;
  const float is = float(1.0 / sqrt(var + double(eps)));
  const float mf = float(m);
  mean[c] = mf;
  invstd[c] = is;
  const float av = gamma[c] * is;
  a[c] = alpha_i16 != nullptr ? av * alpha_i16[c] : av;     // int16 operand: z = y_int * (a*alpha) + b
  b[c] = beta[c] - mf * av;
  if (running_mean != nullptr) {
    const double unb = n > 1.0 ? var * n / (n - 1.0) : var;
    running_mean[c] = (1.0f - momentum) * running_mean[c] + momentum * mf;
    running_var[c] = (1.0f - momentum) * running_var[c] + momentum * float(unb);
  }
}

// Option-A (parameter-free) shortcut read in place as the residual: r[n,i,j,c] = x[n,2i,2j,c-pad] for
// pad <= c < pad+Cin, else 0; x fp32 NHWC [N,H,W,Cin], z [N,Ho,Wo,C] with Ho = ceil(H/2), Wo = ceil(W/2).
struct PadResidual {
  const float4* x;
  int H, W, Ho, Wo, Cin4, pad4;
};

// z = y*a + b (+ residual); optionally the sign / STE-mask bits and the +-1 16-bit copy of z.
// SUB: the residual is the option-A shortcut of `sub.x` (res is unused).  P16: C == 16, one sign / mask word per
// pixel from 4 lanes (bits 16-31 zero, as bdbnn_act_pack writes them) instead of one per 32 channels from 8 lanes.
// HT: z = hardtanh(u) for u = y*a + b, and the mask bits are Hardtanh's strict -1 < u < 1 (the product of its
// gradient and the next conv's STE indicator, which is 1 on hardtanh's range except at NaN).
// RELU (PACK false, fp32 y): z = relu(y*a + b (+ residual)), mask_bits = ReLU's gradient mask (relu_bits4, one bit per
// channel as the STE mask), and the bits of max|z| into z_amax (integer atomicMax, NaN on top: run-to-run identical),
// the word the next real-valued conv's real_act_pack scales its fp16 operand by.
// HT with PACK false (fp32 y, no residual, the real-valued Hardtanh units): z = hardtanh(u) for u = fmaf(y, a, b) as it
// stands (adding a zero residual would turn a -0.0 into +0.0), no mask words (the backward recomputes u with the same
// fmaf, htanh_mask), and max|z| into z_amax as RELU.
template <bool PACK, bool I16 = false, int U = 4, bool SUB = false, bool P16 = false, bool HT = false,
          bool RELU = false>
__global__ void __launch_bounds__(kBnThreads)
bn_apply_add_pack_kernel(const void* __restrict__ y, const float4* __restrict__ res,
                         const float* __restrict__ a, const float* __restrict__ b, int64_t n4, int C4,
                         float4* __restrict__ z, uint32_t* __restrict__ sign_bits,
                         uint32_t* __restrict__ mask_bits, uint2* __restrict__ xb4, uint32_t* __restrict__ xb8,
                         uint32_t one16, const PadResidual sub = PadResidual{}, uint32_t* __restrict__ z_amax = nullptr) {
  constexpr bool HT_REAL = HT && !PACK;
  constexpr int GL = P16 ? 4 : 8;                                 // lanes (float4 groups) per bit word
  const int lane = threadIdx.x & 31;
  const uint32_t group_mask = (P16 ? 0xfu : 0xffu) << (lane & (32 - GL));
  const int sh = (lane & (GL - 1)) * 4;
  const uint32_t pos = one16, neg = one16 | 0x8000u;
  const int64_t nthreads = int64_t(gridDim.x) * blockDim.x;       // multiple of C4 (host guarantees)
  int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int c4 = int(i % C4);                                     // constant per thread
  const float4 av = *reinterpret_cast<const float4*>(a + c4 * 4);
  const float4 bv = *reinterpret_cast<const float4*>(b + c4 * 4);
  const bool sub_on = SUB && c4 >= sub.pad4 && c4 < sub.pad4 + sub.Cin4;   // constant per thread too
  uint32_t zmax = 0u;
  auto emit = [&](int64_t i, const float4 v, const float4 r) {
    float4 o = make_float4(fmaf(v.x, av.x, bv.x), fmaf(v.y, av.y, bv.y), fmaf(v.z, av.z, bv.z),
                           fmaf(v.w, av.w, bv.w));
    if (!HT_REAL) { o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w; }
    if (HT) { o.x = htanh(o.x); o.y = htanh(o.y); o.z = htanh(o.z); o.w = htanh(o.w); }
    if (RELU) { o.x = relu_f(o.x); o.y = relu_f(o.y); o.z = relu_f(o.z); o.w = relu_f(o.w); }
    if (RELU || HT_REAL)
      zmax = max(zmax, max(max(__float_as_uint(fabsf(o.x)), __float_as_uint(fabsf(o.y))),
                           max(__float_as_uint(fabsf(o.z)), __float_as_uint(fabsf(o.w)))));
    if (RELU) {
      const uint32_t mw = __reduce_or_sync(group_mask, relu_bits4(o) << sh);
      if ((lane & (GL - 1)) == 0) mask_bits[i / GL] = mw;
    }
    // z (4 B/element, re-read only after the next conv has run) is stored evict-first so that the next conv's
    // operands written below (xb / xb8, 1-2 B/element) have a chance to stay in the 126 MB L2
    __stcs(z + i, o);
    if (PACK) {
      const uint32_t s0 = o.x >= 0.0f, s1 = o.y >= 0.0f, s2 = o.z >= 0.0f, s3 = o.w >= 0.0f;
      // HT: o is clamped, and clamp(u) lies strictly inside (-1, 1) exactly when u does
      const uint32_t m0 = HT ? (o.x > -1.0f && o.x < 1.0f) : fabsf(o.x) <= 1.0f,
                     m1 = HT ? (o.y > -1.0f && o.y < 1.0f) : fabsf(o.y) <= 1.0f,
                     m2 = HT ? (o.z > -1.0f && o.z < 1.0f) : fabsf(o.z) <= 1.0f,
                     m3 = HT ? (o.w > -1.0f && o.w < 1.0f) : fabsf(o.w) <= 1.0f;
      const uint32_t sw = __reduce_or_sync(group_mask, (s0 | (s1 << 1) | (s2 << 2) | (s3 << 3)) << sh);
      const uint32_t mw = __reduce_or_sync(group_mask, (m0 | (m1 << 1) | (m2 << 2) | (m3 << 3)) << sh);
      if ((lane & (GL - 1)) == 0) {
        sign_bits[i / GL] = sw;
        mask_bits[i / GL] = mw;
      }
      uint2 q;
      q.x = (s0 ? pos : neg) | ((s1 ? pos : neg) << 16);
      q.y = (s2 ? pos : neg) | ((s3 ? pos : neg) << 16);
      xb4[i] = q;
      if (xb8 != nullptr)   // e4m3 +-1 bytes for the fp8 forward of the next conv
        xb8[i] = 0x38383838u | ((s0 ? 0u : 0x80u) | (s1 ? 0u : 0x8000u) | (s2 ? 0u : 0x800000u) | (s3 ? 0u : 0x80000000u));
    }
  };
  const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
  auto load_r = [&](int64_t e) {
    if (SUB) {
      if (!sub_on) return zero4;
      int64_t q = e / C4;
      const int j = int(q % sub.Wo);
      q /= sub.Wo;
      const int hi = int(q % sub.Ho);
      const int64_t n = q / sub.Ho;
      return __ldg(sub.x + ((n * sub.H + 2 * hi) * int64_t(sub.W) + 2 * j) * sub.Cin4 + (c4 - sub.pad4));
    }
    return res != nullptr ? __ldcs(res + e) : zero4;
  };
  // two elements per thread and iteration: all four loads are issued before the first dependent instruction
  // (whole 8-lane pack groups take the same branch: n4 and nthreads are multiples of 8)
  for (; i + (U - 1) * nthreads < n4; i += U * nthreads) {
    float4 v[U], r[U];
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = load_y4<I16>(y, i + u * nthreads);       // I16: `a` already carries alpha
#pragma unroll
    for (int u = 0; u < U; ++u) r[u] = load_r(i + u * nthreads);
#pragma unroll
    for (int u = 0; u < U; ++u) emit(i + u * nthreads, v[u], r[u]);
  }
  for (; i < n4; i += nthreads) emit(i, load_y4<I16>(y, i), load_r(i));
  if (RELU || HT_REAL) {
    zmax = __reduce_max_sync(0xffffffffu, zmax);      // every lane of the (whole) warp gets here
    if (lane == 0 && zmax != 0u) atomicMax(z_amax, zmax);
  }
}

// [C] math of the backward.  consts[c] = {m1, m2*invstd, mean, a*gscale}; gy*gscale = (gz - m1 -
// (y-mean)*m2*invstd) * a*gscale.  FP16S scale from the bound
//   |gy*gscale| <= |a*gscale| * (max|gz| + |m1| + (max|y| + |mean|)*invstd*|m2|).
__global__ void bn_bwd_bound_kernel(const double* __restrict__ sums, const uint32_t* __restrict__ gmax_bits,
                                    const uint32_t* __restrict__ ymax_bits, int64_t n_pix, int C,
                                    const float* __restrict__ mean, const float* __restrict__ invstd,
                                    const float* __restrict__ gamma, const float* __restrict__ gscale,
                                    float4* __restrict__ consts, float* __restrict__ dgamma,
                                    float* __restrict__ dbeta, uint32_t* __restrict__ amax_bits,
                                    float gz_mult = 1.0f, const float* __restrict__ alpha_i16 = nullptr) {
  __shared__ float red[32];
  float bound = 0.f;
  const double n = double(n_pix);
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float s1 = float(sums[c]), s2 = float(sums[C + c]);
    dbeta[c] = s1;
    dgamma[c] = s2;
    const float m1 = float(sums[c] / n), m2 = float(sums[C + c] / n);
    const float is = invstd[c], mu = mean[c];
    const float A = gamma[c] * is * gscale[c];
    // pack kernel: (gz - k.x - (v - k.z)*k.y) * k.w with v = y; for the int16 operand v = y_int, so
    // (y - mu)*m2*is = (y_int - mu/alpha) * (alpha*m2*is)   (alpha == 0: y == 0 everywhere, term = -mu*m2*is)
    if (alpha_i16 != nullptr) {
      const float al = alpha_i16[c];
      if (al != 0.f) consts[c] = make_float4(m1, al * m2 * is, mu / al, A);
      else           consts[c] = make_float4(m1 - mu * m2 * is, 0.f, 0.f, A);
    } else {
      consts[c] = make_float4(m1, m2 * is, mu, A);
    }
    const float ymax = __uint_as_float(ymax_bits[c]), gmax = __uint_as_float(gmax_bits[c]);
    // gz_mult: how many gradient values can land on one position (pooled stem: windows per pixel)
    bound = fmaxf(bound, fabsf(A) * (gz_mult * gmax + fabsf(m1) + (ymax + fabsf(mu)) * is * fabsf(m2)));
  }
  bound = warp_max(bound);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = bound;
  __syncthreads();
  if (threadIdx.x == 0) {
    float m = 0.f;
    for (int i = 0; i < int(blockDim.x >> 5); ++i) m = fmaxf(m, red[i]);
    *amax_bits = __float_as_uint(m);
  }
}

// gys = 16-bit operand of the conv backward, straight from gz and y.  HT: gz times Hardtanh's mask (bn_reduce_kernel).
// RM: gz masked by relu_mask(rmask) first; the masked gradient is also written to g_out when that is non-NULL (the
// gradient of a residual added before the ReLU).
template <int MODE, bool I16 = false, int U = 4, bool HT = false, bool RM = false>
__global__ void __launch_bounds__(kBnThreads)
bn_bwd_pack_kernel(const float4* __restrict__ gz, const void* __restrict__ y, const float4* __restrict__ consts,
                   const uint32_t* __restrict__ amax_bits, int64_t n4, int C4, uint16_t* __restrict__ out,
                   const float* __restrict__ ab = nullptr, const uint32_t* __restrict__ rmask = nullptr,
                   float4* __restrict__ g_out = nullptr) {
  constexpr int HALVES = MODE == 2 ? 2 : 1;
  const int64_t nthreads = int64_t(gridDim.x) * blockDim.x;       // multiple of C4
  int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int c4 = int(i % C4);
  const float up = MODE == 3 ? amax_pow2_scale(*amax_bits, false) : 1.0f;
  const float4 k0 = consts[c4 * 4 + 0], k1 = consts[c4 * 4 + 1], k2 = consts[c4 * 4 + 2], k3 = consts[c4 * 4 + 3];
  const int C = C4 * 4;
  float4 ha = make_float4(0, 0, 0, 0), hb = ha;
  if (HT) {
    ha = *reinterpret_cast<const float4*>(ab + c4 * 4);
    hb = *reinterpret_cast<const float4*>(ab + C + c4 * 4);
  }
  int64_t pix = i / C4;
  const int64_t pix_step = nthreads / C4;
  auto emit = [&](int64_t e, int64_t pix, float4 g, const float4 v) {
    if (HT) g = htanh_mask(g, v, ha, hb);
    if (RM) {
      g = relu_mask(g, rmask, e);
      if (g_out != nullptr) __stcs(g_out + e, g);
    }
    const float a0 = (g.x - k0.x - (v.x - k0.z) * k0.y) * k0.w * up;
    const float a1 = (g.y - k1.x - (v.y - k1.z) * k1.y) * k1.w * up;
    const float a2 = (g.z - k2.x - (v.z - k2.z) * k2.y) * k2.w * up;
    const float a3 = (g.w - k3.x - (v.w - k3.z) * k3.y) * k3.w * up;
    uint2 r;
    if (MODE == 3) {
      r.x = bn_pack_f16x2(a0, a1);
      r.y = bn_pack_f16x2(a2, a3);
    } else {
      r.x = bn_pack_bf16x2(a0, a1);
      r.y = bn_pack_bf16x2(a2, a3);
    }
    uint16_t* dst = out + pix * (int64_t(HALVES) * C) + c4 * 4;
    *reinterpret_cast<uint2*>(dst) = r;
    if (MODE == 2) {
      uint2 l;
      l.x = bn_pack_bf16x2(a0 - bn_bf16_round(a0), a1 - bn_bf16_round(a1));
      l.y = bn_pack_bf16x2(a2 - bn_bf16_round(a2), a3 - bn_bf16_round(a3));
      *reinterpret_cast<uint2*>(dst + C) = l;
    }
  };
  // U elements per thread and iteration, loads first
  for (; i + (U - 1) * nthreads < n4; i += U * nthreads, pix += U * pix_step) {
    float4 g[U], v[U];
#pragma unroll
    for (int u = 0; u < U; ++u) g[u] = __ldcs(gz + i + u * nthreads);
#pragma unroll
    for (int u = 0; u < U; ++u) v[u] = load_y4<I16>(y, i + u * nthreads);
#pragma unroll
    for (int u = 0; u < U; ++u) emit(i + u * nthreads, pix + u * pix_step, g[u], v[u]);
  }
  for (; i < n4; i += nthreads, pix += pix_step) emit(i, pix, __ldcs(gz + i), load_y4<I16>(y, i));
}

// Hardtanh units after a 2x2 / stride-2 max-pool (DESIGN.md §4n), int16 conv results y_int [N][H][W][C] (H, W even):
//   pool2_i16_kernel      : p = 2x2 max of y_int (exact: alpha >= 0 and fp32 rounding are monotone), the winner's tap
//                           (dy*2 + dx, first maximum in scan order, one byte per channel), and the BatchNorm batch
//                           statistics of alpha*p (partials per block, summed in block order) with max|alpha*p|
//   pool2_bwd_pack_kernel : the BatchNorm backward on the pooled tensor (gz times Hardtanh's mask) written as the conv
//                           backward's 16-bit operand at the conv-output resolution: the value at the winner, 0 elsewhere
//   pool2_eval_kernel     : z = hardtanh(fp32(fp32(max * scale) + shift)) from the folded eval BatchNorm, + the +-1 copy
//   real_pool2_eval_kernel: the same on the fp32 output of a real-valued conv (the fp32 VGG-Small teacher), + max|z|
//   real_pool2_kernel     : pool2_i16_kernel on the fp32 output of a real-valued conv (the fp32 VGG-Small in training),
//                           F.max_pool2d's winner, statistics and max|p| of p itself; pool2_bwd_pack_kernel<MODE, false>
//                           is its backward
__device__ __forceinline__ int4 pool2_quad(const int16_t* __restrict__ y, int64_t off) {
  const uint2 r = __ldcs(reinterpret_cast<const uint2*>(y + off));
  return make_int4(int16_t(r.x & 0xffffu), int16_t(r.x >> 16), int16_t(r.y & 0xffffu), int16_t(r.y >> 16));
}

// max over the window at (n, 2ho, 2wo), channels 4*c4..4*c4+3; tap bytes in *win (strict > keeps the first maximum)
__device__ __forceinline__ int4 pool2_max(const int16_t* __restrict__ y, int64_t n, int ho, int wo, int H, int W,
                                          int C, int c4, uint32_t* win) {
  int4 m = make_int4(0, 0, 0, 0);
  uint32_t tx = 0, ty = 0, tz = 0, tw = 0;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int64_t off = ((n * H + 2 * ho + (t >> 1)) * W + 2 * wo + (t & 1)) * C + 4 * c4;
    const int4 v = pool2_quad(y, off);
    if (t == 0 || v.x > m.x) { m.x = v.x; tx = t; }
    if (t == 0 || v.y > m.y) { m.y = v.y; ty = t; }
    if (t == 0 || v.z > m.z) { m.z = v.z; tz = t; }
    if (t == 0 || v.w > m.w) { m.w = v.w; tw = t; }
  }
  *win = tx | (ty << 8) | (tz << 16) | (tw << 24);
  return m;
}

// fp32 y: the max of the window as F.max_pool2d takes it (scan order, `v > m || v is NaN`): NaN if the window holds
// one, and of equal values (+0.0 / -0.0) the first.  win != NULL: the winner's tap bytes as pool2_max (the last NaN
// of a window, as torch's index)
__device__ __forceinline__ bool pool2_wins(float m, float v) { return v > m || v != v; }

__device__ __forceinline__ float4 pool2_max_f32(const float* __restrict__ y, int64_t n, int ho, int wo, int H, int W,
                                                int C, int c4, uint32_t* win = nullptr) {
  float4 m;
  uint32_t tx = 0, ty = 0, tz = 0, tw = 0;
#pragma unroll
  for (int t = 0; t < 4; ++t) {
    const int64_t off = ((n * H + 2 * ho + (t >> 1)) * W + 2 * wo + (t & 1)) * C + 4 * c4;
    const float4 v = __ldcs(reinterpret_cast<const float4*>(y + off));
    if (t == 0) {
      m = v;
    } else {
      if (pool2_wins(m.x, v.x)) { m.x = v.x; tx = t; }
      if (pool2_wins(m.y, v.y)) { m.y = v.y; ty = t; }
      if (pool2_wins(m.z, v.z)) { m.z = v.z; tz = t; }
      if (pool2_wins(m.w, v.w)) { m.w = v.w; tw = t; }
    }
  }
  if (win != nullptr) *win = tx | (ty << 8) | (tz << 16) | (tw << 24);
  return m;
}

// thread = one channel group, strided over pooled pixels as bn_reduce_kernel (grid * blockDim a multiple of C4).
// F32: y and p fp32 (real_pool2_kernel, the statistics of p itself), else int16 (pool2_i16_kernel, those of alpha*p).
template <bool F32>
__device__ __forceinline__ void pool2_stats(const void* __restrict__ y, const float* __restrict__ alpha, int H, int W,
                                            int C4, int64_t n_pool, void* __restrict__ p, uint32_t* __restrict__ idx,
                                            double* __restrict__ part, uint32_t* __restrict__ maxbits) {
  extern __shared__ float4 shs[];
  const int C = C4 * 4;
  uint32_t* shm = reinterpret_cast<uint32_t*>(shs + 2 * blockDim.x);
  for (int i = threadIdx.x; i < C; i += blockDim.x) shm[i] = 0u;
  __syncthreads();
  const int Ho = H / 2, Wo = W / 2;
  const int64_t gtid = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t nthreads = int64_t(gridDim.x) * blockDim.x;
  const int c4 = int(gtid % C4);
  const int64_t p_step = nthreads / C4;
  const float4 al = F32 ? make_float4(1, 1, 1, 1) : *reinterpret_cast<const float4*>(alpha + c4 * 4);
  float4 sa = make_float4(0, 0, 0, 0), sb = sa, mx = sa;
  for (int64_t q = gtid / C4; q < n_pool; q += p_step) {
    const int wo = int(q % Wo);
    const int64_t r = q / Wo;
    const int ho = int(r % Ho);
    uint32_t win;
    const int64_t o = q * C4 + c4;
    float4 v;
    if (F32) {
      v = pool2_max_f32(static_cast<const float*>(y), r / Ho, ho, wo, H, W, C, c4, &win);
      static_cast<float4*>(p)[o] = v;
    } else {
      const int4 m = pool2_max(static_cast<const int16_t*>(y), r / Ho, ho, wo, H, W, C, c4, &win);
      *reinterpret_cast<uint2*>(static_cast<int16_t*>(p) + 4 * o) =
          make_uint2((uint32_t(m.x) & 0xffffu) | (uint32_t(m.y) << 16), (uint32_t(m.z) & 0xffffu) | (uint32_t(m.w) << 16));
      // alpha * p is the conv's fp32 output at the winner (one fp32 multiply, as the conv epilogue)
      v = make_float4(float(m.x) * al.x, float(m.y) * al.y, float(m.z) * al.z, float(m.w) * al.w);
    }
    idx[o] = win;
    sa.x += v.x; sa.y += v.y; sa.z += v.z; sa.w += v.w;
    sb.x += v.x * v.x; sb.y += v.y * v.y; sb.z += v.z * v.z; sb.w += v.w * v.w;
    mx.x = fmaxf(mx.x, fabsf(v.x)); mx.y = fmaxf(mx.y, fabsf(v.y));
    mx.z = fmaxf(mx.z, fabsf(v.z)); mx.w = fmaxf(mx.w, fabsf(v.w));
  }
  block_partials(shs, shm, C4, c4, sa, sb, mx, part, maxbits);
}

__global__ void __launch_bounds__(kBnThreads)
pool2_i16_kernel(const int16_t* __restrict__ y, const float* __restrict__ alpha, int H, int W, int C4, int64_t n_pool,
                 int16_t* __restrict__ p, uint32_t* __restrict__ idx, double* __restrict__ part,
                 uint32_t* __restrict__ maxbits) {
  pool2_stats<false>(y, alpha, H, W, C4, n_pool, p, idx, part, maxbits);
}

__global__ void __launch_bounds__(kBnThreads)
real_pool2_kernel(const float* __restrict__ y, int H, int W, int C4, int64_t n_pool, float* __restrict__ p,
                  uint32_t* __restrict__ idx, double* __restrict__ part, uint32_t* __restrict__ maxbits) {
  pool2_stats<true>(y, nullptr, H, W, C4, n_pool, p, idx, part, maxbits);
}

// I16: p is the int16 p_int of pool2_i16_kernel (consts carry alpha), else the fp32 p of real_pool2_kernel
template <int MODE, bool I16 = true>
__global__ void __launch_bounds__(kBnThreads)
pool2_bwd_pack_kernel(const float4* __restrict__ gz, const void* __restrict__ p, const uint32_t* __restrict__ idx,
                      const float4* __restrict__ consts, const float* __restrict__ ab,
                      const uint32_t* __restrict__ amax_bits, int H, int W, int C4, int64_t n4,
                      uint16_t* __restrict__ out) {
  constexpr int HALVES = MODE == 2 ? 2 : 1;
  const int64_t nthreads = int64_t(gridDim.x) * blockDim.x;       // multiple of C4
  int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int c4 = int(i % C4);
  const int C = C4 * 4, Ho = H / 2, Wo = W / 2;
  const float up = MODE == 3 ? amax_pow2_scale(*amax_bits, false) : 1.0f;
  const float4 k0 = consts[c4 * 4 + 0], k1 = consts[c4 * 4 + 1], k2 = consts[c4 * 4 + 2], k3 = consts[c4 * 4 + 3];
  const float4 ha = *reinterpret_cast<const float4*>(ab + c4 * 4);
  const float4 hb = *reinterpret_cast<const float4*>(ab + C + c4 * 4);
  for (; i < n4; i += nthreads) {
    const float4 v = load_y4<I16>(p, i);
    const float4 g = htanh_mask(__ldcs(gz + i), v, ha, hb);
    const uint32_t win = __ldcs(idx + i);
    const float a0 = (g.x - k0.x - (v.x - k0.z) * k0.y) * k0.w * up;
    const float a1 = (g.y - k1.x - (v.y - k1.z) * k1.y) * k1.w * up;
    const float a2 = (g.z - k2.x - (v.z - k2.z) * k2.y) * k2.w * up;
    const float a3 = (g.w - k3.x - (v.w - k3.z) * k3.y) * k3.w * up;
    const int64_t q = i / C4;
    const int wo = int(q % Wo);
    const int64_t r = q / Wo;
    const int ho = int(r % Ho);
    const int64_t n = r / Ho;
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float b0 = (win & 0xffu) == uint32_t(t) ? a0 : 0.0f;
      const float b1 = ((win >> 8) & 0xffu) == uint32_t(t) ? a1 : 0.0f;
      const float b2 = ((win >> 16) & 0xffu) == uint32_t(t) ? a2 : 0.0f;
      const float b3 = (win >> 24) == uint32_t(t) ? a3 : 0.0f;
      const int64_t pix = (n * H + 2 * ho + (t >> 1)) * W + 2 * wo + (t & 1);
      uint16_t* dst = out + pix * (int64_t(HALVES) * C) + c4 * 4;
      uint2 o;
      if (MODE == 3) {
        o.x = bn_pack_f16x2(b0, b1);
        o.y = bn_pack_f16x2(b2, b3);
      } else {
        o.x = bn_pack_bf16x2(b0, b1);
        o.y = bn_pack_bf16x2(b2, b3);
      }
      *reinterpret_cast<uint2*>(dst) = o;
      if (MODE == 2) {
        uint2 l;
        l.x = bn_pack_bf16x2(b0 - bn_bf16_round(b0), b1 - bn_bf16_round(b1));
        l.y = bn_pack_bf16x2(b2 - bn_bf16_round(b2), b3 - bn_bf16_round(b3));
        *reinterpret_cast<uint2*>(dst + C) = l;
      }
    }
  }
}

__global__ void __launch_bounds__(kBnThreads)
pool2_eval_kernel(const int16_t* __restrict__ y, const float* __restrict__ scale, const float* __restrict__ shift,
                  int H, int W, int C4, int64_t n4, float4* __restrict__ z, uint2* __restrict__ zb,
                  uint32_t* __restrict__ zb8, uint32_t one16) {
  const int64_t nthreads = int64_t(gridDim.x) * blockDim.x;       // multiple of C4
  int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int c4 = int(i % C4);
  const int Ho = H / 2, Wo = W / 2;
  const float4 sc = *reinterpret_cast<const float4*>(scale + c4 * 4);
  const float4 sf = *reinterpret_cast<const float4*>(shift + c4 * 4);
  const uint32_t pos = one16, neg = one16 | 0x8000u;
  for (; i < n4; i += nthreads) {
    const int64_t q = i / C4;
    const int wo = int(q % Wo);
    const int64_t r = q / Wo;
    uint32_t win;
    const int4 m = pool2_max(y, r / Ho, int(r % Ho), wo, H, W, C4 * 4, c4, &win);
    // one rounding per step, no FMA contraction (the eval epilogue of tc_conv_kernel)
    float4 o;
    o.x = htanh(__fadd_rn(__fmul_rn(float(m.x), sc.x), sf.x));
    o.y = htanh(__fadd_rn(__fmul_rn(float(m.y), sc.y), sf.y));
    o.z = htanh(__fadd_rn(__fmul_rn(float(m.z), sc.z), sf.z));
    o.w = htanh(__fadd_rn(__fmul_rn(float(m.w), sc.w), sf.w));
    z[i] = o;
    const bool s0 = o.x >= 0.0f, s1 = o.y >= 0.0f, s2 = o.z >= 0.0f, s3 = o.w >= 0.0f;
    if (zb != nullptr)
      zb[i] = make_uint2((s0 ? pos : neg) | ((s1 ? pos : neg) << 16), (s2 ? pos : neg) | ((s3 ? pos : neg) << 16));
    if (zb8 != nullptr)
      zb8[i] = 0x38383838u | ((s0 ? 0u : 0x80u) | (s1 ? 0u : 0x8000u) | (s2 ? 0u : 0x800000u) | (s3 ? 0u : 0x80000000u));
  }
}

// pool2_eval_kernel on an fp32 conv output (a kernel of its own, so that the int16 one keeps its code): no +-1 copy,
// the bits of max|z| into z_amax instead (integer atomicMax, NaN on top: run-to-run identical)
__global__ void __launch_bounds__(kBnThreads)
real_pool2_eval_kernel(const float* __restrict__ y, const float* __restrict__ scale, const float* __restrict__ shift,
                       int H, int W, int C4, int64_t n4, float4* __restrict__ z, uint32_t* __restrict__ z_amax) {
  const int64_t nthreads = int64_t(gridDim.x) * blockDim.x;       // multiple of C4
  int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int c4 = int(i % C4);
  const int Ho = H / 2, Wo = W / 2;
  const float4 sc = *reinterpret_cast<const float4*>(scale + c4 * 4);
  const float4 sf = *reinterpret_cast<const float4*>(shift + c4 * 4);
  uint32_t zmax = 0u;
  for (; i < n4; i += nthreads) {
    const int64_t q = i / C4;
    const int wo = int(q % Wo);
    const int64_t r = q / Wo;
    const float4 m = pool2_max_f32(y, r / Ho, int(r % Ho), wo, H, W, C4 * 4, c4);
    float4 o;
    o.x = htanh(__fadd_rn(__fmul_rn(m.x, sc.x), sf.x));
    o.y = htanh(__fadd_rn(__fmul_rn(m.y, sc.y), sf.y));
    o.z = htanh(__fadd_rn(__fmul_rn(m.z, sc.z), sf.z));
    o.w = htanh(__fadd_rn(__fmul_rn(m.w, sc.w), sf.w));
    z[i] = o;
    zmax = max(zmax, max(max(__float_as_uint(fabsf(o.x)), __float_as_uint(fabsf(o.y))),
                         max(__float_as_uint(fabsf(o.z)), __float_as_uint(fabsf(o.w)))));
  }
  zmax = __reduce_max_sync(0xffffffffu, zmax);      // every lane of the (whole) warp gets here
  if ((threadIdx.x & 31) == 0 && zmax != 0u) atomicMax(z_amax, zmax);
}

static int bn_grid(int64_t work, int C4, int per_sm = 8) {
  // grid whose thread count is a multiple of C4 (C4 in {4,..,128} divides 256*k); per_sm blocks per SM at most
  int64_t blocks = (work + kBnThreads - 1) / kBnThreads;
  const int64_t cap = int64_t(num_sms()) * per_sm;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  while ((blocks * kBnThreads) % C4 != 0) ++blocks;
  return int(blocks);
}

// Forward statistics pass (also the fallback of conv kernels without a statistics epilogue).
int bn_stats_launch(const float* y, int64_t n_pix, int C, double* sums, uint32_t* ymax, cudaStream_t st) {
  BDBNN_REQUIRE(C > 0 && (C & 3) == 0 && C <= 4096, "bn_stats: C must be a multiple of 4, <= 4096");
  const int C4 = C / 4;
  return bn_reduce_launch<false>(bn_grid(n_pix * C4 / 8, C4, n_pix * C4 > (int64_t(16) << 20) ? 8 : 3),
                                 reinterpret_cast<const float4*>(y), nullptr, nullptr, nullptr, n_pix, C4, sums, ymax,
                                 nullptr, st);
}

// Eval-mode BatchNorm folded into a per-channel affine map of the conv accumulator, in fp64 with every step rounded
// on its own (nvcc would otherwise contract a*b+c into an FMA):  k = gamma / sqrt(rv + eps),
// scale = float(alpha * k), shift = float(beta - rm * k).  oracle/eval_ref.py spells the same arithmetic.
__global__ void bn_eval_fold_kernel(const float* __restrict__ alpha, const float* __restrict__ gamma,
                                    const float* __restrict__ beta, const float* __restrict__ rm,
                                    const float* __restrict__ rv, int C, double eps, float* __restrict__ scale,
                                    float* __restrict__ shift) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double k = __ddiv_rn(double(gamma[c]), __dsqrt_rn(__dadd_rn(double(rv[c]), eps)));
  const double a = alpha != nullptr ? double(alpha[c]) : 1.0;
  scale[c] = __double2float_rn(__dmul_rn(a, k));
  shift[c] = __double2float_rn(__dsub_rn(double(beta[c]), __dmul_rn(double(rm[c]), k)));
}

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_bn_eval_fold(const float* alpha, const float* gamma, const float* beta, const float* running_mean,
                                  const float* running_var, int32_t C, float eps, float* scale, float* shift,
                                  void* stream) {
  BDBNN_REQUIRE(C > 0, "bn_eval_fold: C must be positive");
  BDBNN_REQUIRE(gamma && beta && running_mean && running_var && scale && shift, "bn_eval_fold: NULL pointer");
  bn_eval_fold_kernel<<<(C + 127) / 128, 128, 0, cudaStream_t(stream)>>>(alpha, gamma, beta, running_mean, running_var,
                                                                          C, double(eps), scale, shift);
  return check_launch("bn_eval_fold_kernel");
}

static int bn_dims_ok(int64_t n_pix, int32_t C, bool pack) {
  BDBNN_REQUIRE(n_pix > 0 && C > 0 && (C & 3) == 0, "bn: C must be a positive multiple of 4");
  BDBNN_REQUIRE(C <= 4096, "bn: C too large");
  BDBNN_REQUIRE(!pack || (C & 31) == 0, "bn: packing needs C %% 32 == 0");
  return BDBNN_OK;
}

static int bn_fwd_impl(const void* y, const float* alpha_i16, const float* residual, const float* gamma,
                       const float* beta, int64_t n_pix, int32_t C, float eps, float momentum, float* running_mean,
                       float* running_var, double* sums_ws, uint32_t* ymax_bits, float* mean, float* invstd,
                       float* ab_ws, float* z, uint32_t* sign_bits, uint32_t* mask_bits, uint16_t* xb,
                       uint8_t* xb_fp8, int32_t fmt, int32_t stats_ready, void* stream,
                       const PadResidual* sub = nullptr, bool ht = false, uint32_t* relu_amax = nullptr) {
  // bdbnn_real_bn_fwd_hardtanh: fp32 y, no +-1 packs and no mask words, max|z| into relu_amax
  const bool ht_real = ht && relu_amax != nullptr;
  if (relu_amax != nullptr && !ht) {      // bdbnn_bn_fwd_relu: fp32 y, no +-1 packs, the ReLU mask words instead
    BDBNN_REQUIRE(alpha_i16 == nullptr && sub == nullptr && !ht && sign_bits == nullptr && mask_bits != nullptr,
                  "bn_fwd_relu: needs fp32 y and mask_bits");
    BDBNN_REQUIRE((C & 31) == 0, "bn_fwd_relu: the mask words need C %% 32 == 0");
  }
  if (ht_real)
    BDBNN_REQUIRE(alpha_i16 == nullptr && sub == nullptr && residual == nullptr && sign_bits == nullptr &&
                      mask_bits == nullptr && stats_ready,
                  "real_bn_fwd_hardtanh: fp32 y, no residual, and the statistics ready (stats_ready = 1)");
  const bool pack = sign_bits != nullptr;
  const bool i16 = alpha_i16 != nullptr;
  // 16-channel packs (one word per pixel): the CIFAR stem's BatchNorm, fp32 y only
  const bool p16 = pack && C == 16;
  BDBNN_REQUIRE(!i16 || stats_ready, "bn_fwd_i16: the statistics must come from the conv epilogue (stats_ready = 1)");
  BDBNN_REQUIRE(!(p16 && (i16 || sub)), "bn_fwd: 16-channel packs only without int16 y and option-A residual");
  BDBNN_REQUIRE(!ht || ht_real || (pack && !p16 && !sub && !residual),
                "bn_fwd_hardtanh: needs the packs, C %% 32 == 0 and no residual");
  int rc = bn_dims_ok(n_pix, C, pack && !p16);
  if (rc) return rc;
  BDBNN_REQUIRE(y && gamma && beta && sums_ws && ymax_bits && mean && invstd && ab_ws && z, "bn_fwd: NULL pointer");
  BDBNN_REQUIRE(!pack || (mask_bits && xb), "bn_fwd: packing needs sign_bits, mask_bits and xb");
  BDBNN_REQUIRE((running_mean == nullptr) == (running_var == nullptr), "bn_fwd: running stats come in pairs");
  cudaStream_t st = cudaStream_t(stream);
  const int C4 = C / 4;
  if (!stats_ready) {          // else: sums_ws / ymax_bits were filled by the conv's epilogue
    BDBNN_CUDA(cudaMemsetAsync(sums_ws, 0, size_t(2 * C) * sizeof(double), st));
    BDBNN_CUDA(cudaMemsetAsync(ymax_bits, 0, size_t(C) * sizeof(uint32_t), st));
    rc = bn_stats_launch(static_cast<const float*>(y), n_pix, C, sums_ws, ymax_bits, st);
    if (rc) return rc;
  }
  float* a = ab_ws;
  float* b = ab_ws + C;
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(sums_ws, n_pix, C, eps, gamma, beta, mean, invstd, a, b,
                                                       running_mean, running_var, momentum, alpha_i16);
  rc = check_launch("bn_finalize_kernel");
  if (rc) return rc;
  const int64_t n4 = n_pix * C4;
  const int grid = bn_grid(n4, C4);
  const float4* r4 = reinterpret_cast<const float4*>(residual);
  float4* z4 = reinterpret_cast<float4*>(z);
  if (ht_real) {
    BDBNN_CUDA(cudaMemsetAsync(relu_amax, 0, sizeof(uint32_t), st));
    bn_apply_add_pack_kernel<false, false, 4, false, false, true><<<grid, kBnThreads, 0, st>>>(
        y, nullptr, a, b, n4, C4, z4, nullptr, nullptr, nullptr, nullptr, 0u, PadResidual{}, relu_amax);
  } else if (relu_amax != nullptr) {
    BDBNN_CUDA(cudaMemsetAsync(relu_amax, 0, sizeof(uint32_t), st));
    bn_apply_add_pack_kernel<false, false, 4, false, false, false, true><<<grid, kBnThreads, 0, st>>>(
        y, r4, a, b, n4, C4, z4, nullptr, mask_bits, nullptr, nullptr, 0u, PadResidual{}, relu_amax);
  } else if (sub != nullptr) {
    const uint32_t one16 = fmt == BDBNN_FMT_FP16 ? 0x3C00u : 0x3F80u;
    uint2* xb2 = reinterpret_cast<uint2*>(xb);
    uint32_t* xb8 = reinterpret_cast<uint32_t*>(xb_fp8);
    if (pack && i16)
      bn_apply_add_pack_kernel<true, true, 4, true><<<grid, kBnThreads, 0, st>>>(y, nullptr, a, b, n4, C4, z4, sign_bits,
                                                                                mask_bits, xb2, xb8, one16, *sub);
    else if (pack)
      bn_apply_add_pack_kernel<true, false, 4, true><<<grid, kBnThreads, 0, st>>>(y, nullptr, a, b, n4, C4, z4, sign_bits,
                                                                                 mask_bits, xb2, xb8, one16, *sub);
    else if (i16)
      bn_apply_add_pack_kernel<false, true, 4, true><<<grid, kBnThreads, 0, st>>>(y, nullptr, a, b, n4, C4, z4, nullptr,
                                                                                 nullptr, nullptr, nullptr, 0u, *sub);
    else
      bn_apply_add_pack_kernel<false, false, 4, true><<<grid, kBnThreads, 0, st>>>(y, nullptr, a, b, n4, C4, z4, nullptr,
                                                                                  nullptr, nullptr, nullptr, 0u, *sub);
  } else if (p16) {
    const uint32_t one16 = fmt == BDBNN_FMT_FP16 ? 0x3C00u : 0x3F80u;
    bn_apply_add_pack_kernel<true, false, 4, false, true><<<grid, kBnThreads, 0, st>>>(
        y, r4, a, b, n4, C4, z4, sign_bits, mask_bits, reinterpret_cast<uint2*>(xb),
        reinterpret_cast<uint32_t*>(xb_fp8), one16);
  } else if (ht) {
    const uint32_t one16 = fmt == BDBNN_FMT_FP16 ? 0x3C00u : 0x3F80u;
    uint2* xb2 = reinterpret_cast<uint2*>(xb);
    uint32_t* xb8 = reinterpret_cast<uint32_t*>(xb_fp8);
    if (i16)
      bn_apply_add_pack_kernel<true, true, 4, false, false, true><<<grid, kBnThreads, 0, st>>>(
          y, nullptr, a, b, n4, C4, z4, sign_bits, mask_bits, xb2, xb8, one16);
    else
      bn_apply_add_pack_kernel<true, false, 4, false, false, true><<<grid, kBnThreads, 0, st>>>(
          y, nullptr, a, b, n4, C4, z4, sign_bits, mask_bits, xb2, xb8, one16);
  } else if (pack) {
    const uint32_t one16 = fmt == BDBNN_FMT_FP16 ? 0x3C00u : 0x3F80u;
    uint2* xb2 = reinterpret_cast<uint2*>(xb);
    uint32_t* xb8 = reinterpret_cast<uint32_t*>(xb_fp8);
    // four float4 per thread and iteration (more loads in flight than two); BDBNN_BN_UNROLL=2
    static const int unroll2 = [] { const char* e = getenv("BDBNN_BN_UNROLL"); return e ? atoi(e) == 2 : 0; }();
    if (i16 && unroll2)
      bn_apply_add_pack_kernel<true, true, 2><<<grid, kBnThreads, 0, st>>>(y, r4, a, b, n4, C4, z4, sign_bits, mask_bits,
                                                                            xb2, xb8, one16);
    else if (i16)
      bn_apply_add_pack_kernel<true, true><<<grid, kBnThreads, 0, st>>>(y, r4, a, b, n4, C4, z4, sign_bits, mask_bits,
                                                                         xb2, xb8, one16);
    else
      bn_apply_add_pack_kernel<true, false><<<grid, kBnThreads, 0, st>>>(y, r4, a, b, n4, C4, z4, sign_bits, mask_bits,
                                                                          xb2, xb8, one16);
  } else {
    if (i16)
      bn_apply_add_pack_kernel<false, true><<<grid, kBnThreads, 0, st>>>(y, r4, a, b, n4, C4, z4, nullptr, nullptr,
                                                                          nullptr, nullptr, 0u);
    else
      bn_apply_add_pack_kernel<false, false><<<grid, kBnThreads, 0, st>>>(y, r4, a, b, n4, C4, z4, nullptr, nullptr,
                                                                           nullptr, nullptr, 0u);
  }
  return check_launch("bn_apply_add_pack_kernel");
}

extern "C" int bdbnn_bn_fwd(const float* y, const float* residual, const float* gamma, const float* beta,
                            int64_t n_pix, int32_t C, float eps, float momentum, float* running_mean,
                            float* running_var, double* sums_ws, uint32_t* ymax_bits, float* mean,
                            float* invstd, float* ab_ws, float* z, uint32_t* sign_bits, uint32_t* mask_bits,
                            uint16_t* xb, uint8_t* xb_fp8, int32_t fmt, int32_t stats_ready, void* stream) {
  return bn_fwd_impl(y, nullptr, residual, gamma, beta, n_pix, C, eps, momentum, running_mean, running_var, sums_ws,
                     ymax_bits, mean, invstd, ab_ws, z, sign_bits, mask_bits, xb, xb_fp8, fmt, stats_ready, stream);
}

extern "C" int bdbnn_bn_fwd_relu(const float* y, const float* residual, const float* gamma, const float* beta,
                                 int64_t n_pix, int32_t C, float eps, float momentum, float* running_mean,
                                 float* running_var, double* sums_ws, uint32_t* ymax_bits, float* mean, float* invstd,
                                 float* ab_ws, float* z, uint32_t* mask_bits, uint32_t* z_amax_bits,
                                 int32_t stats_ready, void* stream) {
  BDBNN_REQUIRE(z_amax_bits != nullptr, "bn_fwd_relu: NULL z_amax_bits");
  return bn_fwd_impl(y, nullptr, residual, gamma, beta, n_pix, C, eps, momentum, running_mean, running_var, sums_ws,
                     ymax_bits, mean, invstd, ab_ws, z, nullptr, mask_bits, nullptr, nullptr, BDBNN_FMT_FP16,
                     stats_ready, stream, nullptr, false, z_amax_bits);
}

extern "C" int bdbnn_bn_fwd_hardtanh(const void* y, const float* alpha, const float* gamma, const float* beta,
                                     int64_t n_pix, int32_t C, float eps, float momentum, float* running_mean,
                                     float* running_var, double* sums_ws, uint32_t* ymax_bits, float* mean,
                                     float* invstd, float* ab_ws, float* z, uint32_t* sign_bits, uint32_t* mask_bits,
                                     uint16_t* xb, uint8_t* xb_fp8, int32_t fmt, int32_t stats_ready, void* stream) {
  BDBNN_REQUIRE(sign_bits != nullptr, "bn_fwd_hardtanh: NULL sign_bits");
  return bn_fwd_impl(y, alpha, nullptr, gamma, beta, n_pix, C, eps, momentum, running_mean, running_var, sums_ws,
                     ymax_bits, mean, invstd, ab_ws, z, sign_bits, mask_bits, xb, xb_fp8, fmt, stats_ready, stream,
                     nullptr, true);
}

extern "C" int bdbnn_real_bn_fwd_hardtanh(const float* y, const float* gamma, const float* beta, int64_t n_pix,
                                          int32_t C, float eps, float momentum, float* running_mean,
                                          float* running_var, double* sums_ws, uint32_t* ymax_bits, float* mean,
                                          float* invstd, float* ab_ws, float* z, uint32_t* z_amax_bits,
                                          int32_t stats_ready, void* stream) {
  BDBNN_REQUIRE(z_amax_bits != nullptr, "real_bn_fwd_hardtanh: NULL z_amax_bits");
  return bn_fwd_impl(y, nullptr, nullptr, gamma, beta, n_pix, C, eps, momentum, running_mean, running_var, sums_ws,
                     ymax_bits, mean, invstd, ab_ws, z, nullptr, nullptr, nullptr, nullptr, BDBNN_FMT_FP16,
                     stats_ready, stream, nullptr, true, z_amax_bits);
}

extern "C" int bdbnn_bn_fwd_i16(const int16_t* y_int, const float* alpha, const float* residual, const float* gamma,
                                const float* beta, int64_t n_pix, int32_t C, float eps, float momentum,
                                float* running_mean, float* running_var, double* sums_ws, uint32_t* ymax_bits,
                                float* mean, float* invstd, float* ab_ws, float* z, uint32_t* sign_bits,
                                uint32_t* mask_bits, uint16_t* xb, uint8_t* xb_fp8, int32_t fmt, void* stream) {
  BDBNN_REQUIRE(alpha != nullptr, "bn_fwd_i16: NULL alpha");
  return bn_fwd_impl(y_int, alpha, residual, gamma, beta, n_pix, C, eps, momentum, running_mean, running_var, sums_ws,
                     ymax_bits, mean, invstd, ab_ws, z, sign_bits, mask_bits, xb, xb_fp8, fmt, 1, stream);
}

// Geometry of the option-A residual of bdbnn_bn_fwd_pad_shortcut / _i16_pad_shortcut; n_pix of z.
static int pad_residual(const float* x, int32_t N, int32_t H, int32_t W, int32_t Cin, int32_t pad, int32_t C,
                        PadResidual* r, int64_t* n_pix) {
  BDBNN_REQUIRE(x != nullptr, "bn_fwd_pad_shortcut: NULL x");
  BDBNN_REQUIRE(N > 0 && H > 0 && W > 0 && Cin > 0, "bn_fwd_pad_shortcut: non-positive dims");
  BDBNN_REQUIRE(Cin % 4 == 0 && pad >= 0 && pad % 4 == 0 && pad + Cin <= C,
                "bn_fwd_pad_shortcut: needs Cin and pad multiples of 4 and pad + Cin <= C");
  BDBNN_REQUIRE((uintptr_t(x) & 15) == 0, "bn_fwd_pad_shortcut: x must be 16-byte aligned");
  r->x = reinterpret_cast<const float4*>(x);
  r->H = H; r->W = W; r->Ho = (H + 1) / 2; r->Wo = (W + 1) / 2; r->Cin4 = Cin / 4; r->pad4 = pad / 4;
  *n_pix = int64_t(N) * r->Ho * r->Wo;
  return BDBNN_OK;
}

extern "C" int bdbnn_bn_fwd_pad_shortcut(const float* y, const float* x, int32_t N, int32_t H, int32_t W, int32_t Cin,
                                         int32_t pad, const float* gamma, const float* beta, int32_t C, float eps,
                                         float momentum, float* running_mean, float* running_var, double* sums_ws,
                                         uint32_t* ymax_bits, float* mean, float* invstd, float* ab_ws, float* z,
                                         uint32_t* sign_bits, uint32_t* mask_bits, uint16_t* xb, uint8_t* xb_fp8,
                                         int32_t fmt, int32_t stats_ready, void* stream) {
  PadResidual r;
  int64_t n_pix = 0;
  int rc = pad_residual(x, N, H, W, Cin, pad, C, &r, &n_pix);
  if (rc) return rc;
  return bn_fwd_impl(y, nullptr, nullptr, gamma, beta, n_pix, C, eps, momentum, running_mean, running_var, sums_ws,
                     ymax_bits, mean, invstd, ab_ws, z, sign_bits, mask_bits, xb, xb_fp8, fmt, stats_ready, stream, &r);
}

extern "C" int bdbnn_bn_fwd_i16_pad_shortcut(const int16_t* y_int, const float* alpha, const float* x, int32_t N,
                                             int32_t H, int32_t W, int32_t Cin, int32_t pad, const float* gamma,
                                             const float* beta, int32_t C, float eps, float momentum,
                                             float* running_mean, float* running_var, double* sums_ws,
                                             uint32_t* ymax_bits, float* mean, float* invstd, float* ab_ws, float* z,
                                             uint32_t* sign_bits, uint32_t* mask_bits, uint16_t* xb, uint8_t* xb_fp8,
                                             int32_t fmt, void* stream) {
  BDBNN_REQUIRE(alpha != nullptr, "bn_fwd_i16_pad_shortcut: NULL alpha");
  PadResidual r;
  int64_t n_pix = 0;
  int rc = pad_residual(x, N, H, W, Cin, pad, C, &r, &n_pix);
  if (rc) return rc;
  return bn_fwd_impl(y_int, alpha, nullptr, gamma, beta, n_pix, C, eps, momentum, running_mean, running_var, sums_ws,
                     ymax_bits, mean, invstd, ab_ws, z, sign_bits, mask_bits, xb, xb_fp8, fmt, 1, stream, &r);
}

static int bn_bwd_pack_impl(const float* gz, const void* y, const float* alpha_i16, const float* mean,
                            const float* invstd, const float* gamma, const float* gscale, const uint32_t* ymax_bits,
                            int64_t n_pix, int32_t C, int32_t grad_mode, double* sums_ws, uint32_t* gmax_bits,
                            float* consts_ws, float* dgamma, float* dbeta, uint32_t* amax_bits, uint16_t* gys,
                            int stats_ready, void* stream, const float* ab_ht = nullptr,
                            const uint32_t* rmask = nullptr, float* g_out = nullptr) {
  const bool i16 = alpha_i16 != nullptr;
  const bool ht = ab_ht != nullptr;
  const bool rm = rmask != nullptr;
  BDBNN_REQUIRE(!(ht && stats_ready), "bn_bwd_pack_hardtanh: the sums are of the masked gradient (stats_ready = 0)");
  BDBNN_REQUIRE(!rm || (!i16 && !ht && !stats_ready && (C & 31) == 0 && grad_mode == BDBNN_GRAD_FP16S),
                "bn_bwd_pack_relu: fp32 y, C %% 32 == 0, grad_mode FP16S, and the sums are of the masked gradient");
  int rc = bn_dims_ok(n_pix, C, false);
  if (rc) return rc;
  BDBNN_REQUIRE(gz && y && mean && invstd && gamma && gscale && ymax_bits && sums_ws && gmax_bits && consts_ws &&
                    dgamma && dbeta && amax_bits && gys,
                "bn_bwd_pack: NULL pointer");
  BDBNN_REQUIRE(grad_mode >= BDBNN_GRAD_BF16 && grad_mode <= BDBNN_GRAD_FP16S, "bn_bwd_pack: bad grad_mode");
  cudaStream_t st = cudaStream_t(stream);
  const int C4 = C / 4;
  if (!stats_ready) {       // else: sums_ws / gmax_bits were filled by the dgrad epilogue that produced gz
    BDBNN_CUDA(cudaMemsetAsync(sums_ws, 0, size_t(2 * C) * sizeof(double), st));
    BDBNN_CUDA(cudaMemsetAsync(gmax_bits, 0, size_t(C) * sizeof(uint32_t), st));
    const int rgrid = bn_grid(n_pix * C4 / 8, C4, n_pix * C4 > (int64_t(16) << 20) ? 8 : 3);
    const float4* g4 = reinterpret_cast<const float4*>(gz);
    if (rm)
      rc = bn_reduce_launch<true, false, false, true>(rgrid, g4, y, mean, invstd, n_pix, C4, sums_ws, gmax_bits,
                                                      nullptr, st, nullptr, rmask);
    else if (i16 && ht)
      rc = bn_reduce_launch<true, true, true>(rgrid, g4, y, mean, invstd, n_pix, C4, sums_ws, gmax_bits, alpha_i16, st,
                                              ab_ht);
    else if (ht)
      rc = bn_reduce_launch<true, false, true>(rgrid, g4, y, mean, invstd, n_pix, C4, sums_ws, gmax_bits, nullptr, st,
                                               ab_ht);
    else if (i16)
      rc = bn_reduce_launch<true, true>(rgrid, g4, y, mean, invstd, n_pix, C4, sums_ws, gmax_bits, alpha_i16, st);
    else
      rc = bn_reduce_launch<true, false>(rgrid, g4, y, mean, invstd, n_pix, C4, sums_ws, gmax_bits, nullptr, st);
    if (rc) return rc;
  }
  bn_bwd_bound_kernel<<<1, 256, 0, st>>>(sums_ws, gmax_bits, ymax_bits, n_pix, C, mean, invstd, gamma, gscale,
                                         reinterpret_cast<float4*>(consts_ws), dgamma, dbeta, amax_bits, 1.0f,
                                         alpha_i16);
  rc = check_launch("bn_bwd_bound_kernel");
  if (rc) return rc;
  const int64_t n4 = n_pix * C4;
  // BDBNN_BN_BWD_PER_SM: resident blocks per SM of the backward apply kernel (64 registers x 256 threads: 4 fill the
  // register file; 3 leave room for a side-stream wgrad CTA next to them)
  static const int bwd_per_sm = [] { const char* e = getenv("BDBNN_BN_BWD_PER_SM"); return e ? atoi(e) : 8; }();
  const int grid = bn_grid(n4, C4, bwd_per_sm);
  const float4* g4 = reinterpret_cast<const float4*>(gz);
  const float4* k4 = reinterpret_cast<const float4*>(consts_ws);
  if (rm) {
    bn_bwd_pack_kernel<3, false, 4, false, true><<<grid, kBnThreads, 0, st>>>(
        g4, y, k4, amax_bits, n4, C4, gys, nullptr, rmask, reinterpret_cast<float4*>(g_out));
  } else if (ht) {
    if (i16 && grad_mode == BDBNN_GRAD_FP16S)
      bn_bwd_pack_kernel<3, true, 4, true><<<grid, kBnThreads, 0, st>>>(g4, y, k4, amax_bits, n4, C4, gys, ab_ht);
    else if (i16 && grad_mode == BDBNN_GRAD_BF16X2)
      bn_bwd_pack_kernel<2, true, 4, true><<<grid, kBnThreads, 0, st>>>(g4, y, k4, amax_bits, n4, C4, gys, ab_ht);
    else if (i16)
      bn_bwd_pack_kernel<1, true, 4, true><<<grid, kBnThreads, 0, st>>>(g4, y, k4, amax_bits, n4, C4, gys, ab_ht);
    else if (grad_mode == BDBNN_GRAD_FP16S)
      bn_bwd_pack_kernel<3, false, 4, true><<<grid, kBnThreads, 0, st>>>(g4, y, k4, amax_bits, n4, C4, gys, ab_ht);
    else if (grad_mode == BDBNN_GRAD_BF16X2)
      bn_bwd_pack_kernel<2, false, 4, true><<<grid, kBnThreads, 0, st>>>(g4, y, k4, amax_bits, n4, C4, gys, ab_ht);
    else
      bn_bwd_pack_kernel<1, false, 4, true><<<grid, kBnThreads, 0, st>>>(g4, y, k4, amax_bits, n4, C4, gys, ab_ht);
  } else if (i16) {
    if (grad_mode == BDBNN_GRAD_FP16S)
      bn_bwd_pack_kernel<3, true><<<grid, kBnThreads, 0, st>>>(g4, y, k4, amax_bits, n4, C4, gys);
    else if (grad_mode == BDBNN_GRAD_BF16X2)
      bn_bwd_pack_kernel<2, true><<<grid, kBnThreads, 0, st>>>(g4, y, k4, amax_bits, n4, C4, gys);
    else
      bn_bwd_pack_kernel<1, true><<<grid, kBnThreads, 0, st>>>(g4, y, k4, amax_bits, n4, C4, gys);
  } else {
    if (grad_mode == BDBNN_GRAD_FP16S)
      bn_bwd_pack_kernel<3, false><<<grid, kBnThreads, 0, st>>>(g4, y, k4, amax_bits, n4, C4, gys);
    else if (grad_mode == BDBNN_GRAD_BF16X2)
      bn_bwd_pack_kernel<2, false><<<grid, kBnThreads, 0, st>>>(g4, y, k4, amax_bits, n4, C4, gys);
    else
      bn_bwd_pack_kernel<1, false><<<grid, kBnThreads, 0, st>>>(g4, y, k4, amax_bits, n4, C4, gys);
  }
  return check_launch("bn_bwd_pack_kernel");
}

extern "C" int bdbnn_bn_bwd_pack(const float* gz, const float* y, const float* mean, const float* invstd,
                                 const float* gamma, const float* gscale, const uint32_t* ymax_bits,
                                 int64_t n_pix, int32_t C, int32_t grad_mode, double* sums_ws,
                                 uint32_t* gmax_bits, float* consts_ws, float* dgamma, float* dbeta,
                                 uint32_t* amax_bits, uint16_t* gys, void* stream) {
  return bn_bwd_pack_impl(gz, y, nullptr, mean, invstd, gamma, gscale, ymax_bits, n_pix, C, grad_mode, sums_ws,
                          gmax_bits, consts_ws, dgamma, dbeta, amax_bits, gys, 0, stream);
}

extern "C" int bdbnn_bn_bwd_pack_relu(const float* gz, const uint32_t* mask_bits, const float* y, const float* mean,
                                      const float* invstd, const float* gamma, const float* gscale,
                                      const uint32_t* ymax_bits, int64_t n_pix, int32_t C, int32_t grad_mode,
                                      double* sums_ws, uint32_t* gmax_bits, float* consts_ws, float* dgamma,
                                      float* dbeta, uint32_t* amax_bits, uint16_t* gys, float* g_out, void* stream) {
  BDBNN_REQUIRE(mask_bits != nullptr, "bn_bwd_pack_relu: NULL mask_bits");
  return bn_bwd_pack_impl(gz, y, nullptr, mean, invstd, gamma, gscale, ymax_bits, n_pix, C, grad_mode, sums_ws,
                          gmax_bits, consts_ws, dgamma, dbeta, amax_bits, gys, 0, stream, nullptr, mask_bits, g_out);
}

extern "C" int bdbnn_bn_bwd_pack_hardtanh(const float* gz, const void* y, const float* alpha, const float* ab,
                                          const float* mean, const float* invstd, const float* gamma,
                                          const float* gscale, const uint32_t* ymax_bits, int64_t n_pix, int32_t C,
                                          int32_t grad_mode, double* sums_ws, uint32_t* gmax_bits, float* consts_ws,
                                          float* dgamma, float* dbeta, uint32_t* amax_bits, uint16_t* gys,
                                          void* stream) {
  BDBNN_REQUIRE(ab != nullptr, "bn_bwd_pack_hardtanh: NULL ab");
  return bn_bwd_pack_impl(gz, y, alpha, mean, invstd, gamma, gscale, ymax_bits, n_pix, C, grad_mode, sums_ws,
                          gmax_bits, consts_ws, dgamma, dbeta, amax_bits, gys, 0, stream, ab);
}

// ---- 2x2 max-pool units (pool2_* kernels) ----------------------------------------------------------------------------
static int pool2_dims_ok(const char* what, int32_t N, int32_t H, int32_t W, int32_t C) {
  BDBNN_REQUIRE(N > 0 && H > 0 && W > 0, "%s: non-positive dims", what);
  BDBNN_REQUIRE(H % 2 == 0 && W % 2 == 0, "%s: H and W must be even", what);
  BDBNN_REQUIRE(C > 0 && C % 32 == 0 && C <= 4096, "%s: C must be a positive multiple of 32, <= 4096", what);
  return BDBNN_OK;
}

// pool2_i16 (alpha != NULL: int16 y and p) and real_pool2 (alpha NULL: fp32 y and p)
static int pool2_stats_impl(const char* what, const void* y, const float* alpha, int32_t N, int32_t H, int32_t W,
                            int32_t C, void* p, uint8_t* idx, double* sums, uint32_t* ymax_bits, void* stream) {
  int rc = pool2_dims_ok(what, N, H, W, C);
  if (rc) return rc;
  BDBNN_REQUIRE(y && p && idx && sums && ymax_bits, "%s: NULL pointer", what);
  cudaStream_t st = cudaStream_t(stream);
  const int C4 = C / 4;
  const int64_t n_pool = int64_t(N) * (H / 2) * (W / 2);
  BDBNN_CUDA(cudaMemsetAsync(sums, 0, size_t(2 * C) * sizeof(double), st));
  BDBNN_CUDA(cudaMemsetAsync(ymax_bits, 0, size_t(C) * sizeof(uint32_t), st));
  const int grid = bn_grid(n_pool * C4 / 2, C4);
  double* part = nullptr;
  rc = det_sums_alloc(&part, grid, 2 * C, st);
  if (rc) return rc;
  const size_t smem = 2 * kBnThreads * sizeof(float4) + size_t(C) * sizeof(uint32_t);
  uint32_t* win = reinterpret_cast<uint32_t*>(idx);
  if (alpha != nullptr) {
    pool2_i16_kernel<<<grid, kBnThreads, smem, st>>>(static_cast<const int16_t*>(y), alpha, H, W, C4, n_pool,
                                                     static_cast<int16_t*>(p), win, part, ymax_bits);
    rc = check_launch("pool2_i16_kernel");
  } else {
    real_pool2_kernel<<<grid, kBnThreads, smem, st>>>(static_cast<const float*>(y), H, W, C4, n_pool,
                                                      static_cast<float*>(p), win, part, ymax_bits);
    rc = check_launch("real_pool2_kernel");
  }
  if (rc) { cudaFreeAsync(part, st); return rc; }
  return det_sums_finish(part, grid, 2 * C, sums, st);
}

extern "C" int bdbnn_pool2_i16(const int16_t* y_int, const float* alpha, int32_t N, int32_t H, int32_t W, int32_t C,
                               int16_t* p_int, uint8_t* idx, double* sums, uint32_t* ymax_bits, void* stream) {
  int rc = pool2_dims_ok("pool2_i16", N, H, W, C);
  if (rc) return rc;
  BDBNN_REQUIRE(y_int && alpha && p_int && idx && sums && ymax_bits, "pool2_i16: NULL pointer");
  return pool2_stats_impl("pool2_i16", y_int, alpha, N, H, W, C, p_int, idx, sums, ymax_bits, stream);
}

extern "C" int bdbnn_real_pool2(const float* y, int32_t N, int32_t H, int32_t W, int32_t C, float* p, uint8_t* idx,
                                double* sums, uint32_t* pmax_bits, void* stream) {
  return pool2_stats_impl("real_pool2", y, nullptr, N, H, W, C, p, idx, sums, pmax_bits, stream);
}

// pool2_bn_bwd_pack (alpha != NULL: int16 p) and real_pool2_bn_bwd_pack (alpha NULL: fp32 p)
static int pool2_bn_bwd_pack_impl(const char* what, const float* gz, const void* p, const uint8_t* idx,
                                  const float* alpha, const float* ab, const float* mean, const float* invstd,
                                  const float* gamma, const float* gscale, const uint32_t* ymax_bits, int32_t N,
                                  int32_t H, int32_t W, int32_t C, int32_t grad_mode, double* sums_ws,
                                  uint32_t* gmax_bits, float* consts_ws, float* dgamma, float* dbeta,
                                  uint32_t* amax_bits, uint16_t* gys, void* stream) {
  int rc = pool2_dims_ok(what, N, H, W, C);
  if (rc) return rc;
  BDBNN_REQUIRE(gz && p && idx && ab && mean && invstd && gamma && gscale && ymax_bits && sums_ws && gmax_bits &&
                    consts_ws && dgamma && dbeta && amax_bits && gys,
                "%s: NULL pointer", what);
  BDBNN_REQUIRE(grad_mode >= BDBNN_GRAD_BF16 && grad_mode <= BDBNN_GRAD_FP16S, "%s: bad grad_mode", what);
  const bool i16 = alpha != nullptr;
  cudaStream_t st = cudaStream_t(stream);
  const int C4 = C / 4;
  const int64_t n_pool = int64_t(N) * (H / 2) * (W / 2);
  BDBNN_CUDA(cudaMemsetAsync(sums_ws, 0, size_t(2 * C) * sizeof(double), st));
  BDBNN_CUDA(cudaMemsetAsync(gmax_bits, 0, size_t(C) * sizeof(uint32_t), st));
  // BatchNorm's backward over the pooled tensor (it normalised the pooled values); each conv-output position takes at
  // most one pooled gradient, so the FP16S bound needs no multiplier
  const int rgrid = bn_grid(n_pool * C4 / 8, C4, 3);
  const float4* g4 = reinterpret_cast<const float4*>(gz);
  if (i16)
    rc = bn_reduce_launch<true, true, true>(rgrid, g4, p, mean, invstd, n_pool, C4, sums_ws, gmax_bits, alpha, st, ab);
  else
    rc = bn_reduce_launch<true, false, true>(rgrid, g4, p, mean, invstd, n_pool, C4, sums_ws, gmax_bits, nullptr, st,
                                             ab);
  if (rc) return rc;
  bn_bwd_bound_kernel<<<1, 256, 0, st>>>(sums_ws, gmax_bits, ymax_bits, n_pool, C, mean, invstd, gamma, gscale,
                                         reinterpret_cast<float4*>(consts_ws), dgamma, dbeta, amax_bits, 1.0f, alpha);
  rc = check_launch("bn_bwd_bound_kernel");
  if (rc) return rc;
  const int64_t n4 = n_pool * C4;
  const int grid = bn_grid(n4, C4);
  const float4* k4 = reinterpret_cast<const float4*>(consts_ws);
  const uint32_t* w4 = reinterpret_cast<const uint32_t*>(idx);
  if (!i16)
    pool2_bwd_pack_kernel<3, false><<<grid, kBnThreads, 0, st>>>(g4, p, w4, k4, ab, amax_bits, H, W, C4, n4, gys);
  else if (grad_mode == BDBNN_GRAD_FP16S)
    pool2_bwd_pack_kernel<3><<<grid, kBnThreads, 0, st>>>(g4, p, w4, k4, ab, amax_bits, H, W, C4, n4, gys);
  else if (grad_mode == BDBNN_GRAD_BF16X2)
    pool2_bwd_pack_kernel<2><<<grid, kBnThreads, 0, st>>>(g4, p, w4, k4, ab, amax_bits, H, W, C4, n4, gys);
  else
    pool2_bwd_pack_kernel<1><<<grid, kBnThreads, 0, st>>>(g4, p, w4, k4, ab, amax_bits, H, W, C4, n4, gys);
  return check_launch("pool2_bwd_pack_kernel");
}

extern "C" int bdbnn_pool2_bn_bwd_pack(const float* gz, const int16_t* p_int, const uint8_t* idx, const float* alpha,
                                       const float* ab, const float* mean, const float* invstd, const float* gamma,
                                       const float* gscale, const uint32_t* ymax_bits, int32_t N, int32_t H, int32_t W,
                                       int32_t C, int32_t grad_mode, double* sums_ws, uint32_t* gmax_bits,
                                       float* consts_ws, float* dgamma, float* dbeta, uint32_t* amax_bits,
                                       uint16_t* gys, void* stream) {
  int rc = pool2_dims_ok("pool2_bn_bwd_pack", N, H, W, C);
  if (rc) return rc;
  BDBNN_REQUIRE(alpha != nullptr, "pool2_bn_bwd_pack: NULL pointer");
  return pool2_bn_bwd_pack_impl("pool2_bn_bwd_pack", gz, p_int, idx, alpha, ab, mean, invstd, gamma, gscale,
                                ymax_bits, N, H, W, C, grad_mode, sums_ws, gmax_bits, consts_ws, dgamma, dbeta,
                                amax_bits, gys, stream);
}

extern "C" int bdbnn_real_pool2_bn_bwd_pack(const float* gz, const float* p, const uint8_t* idx, const float* ab,
                                            const float* mean, const float* invstd, const float* gamma,
                                            const float* gscale, const uint32_t* pmax_bits, int32_t N, int32_t H,
                                            int32_t W, int32_t C, double* sums_ws, uint32_t* gmax_bits,
                                            float* consts_ws, float* dgamma, float* dbeta, uint32_t* amax_bits,
                                            uint16_t* gys, void* stream) {
  return pool2_bn_bwd_pack_impl("real_pool2_bn_bwd_pack", gz, p, idx, nullptr, ab, mean, invstd, gamma, gscale,
                                pmax_bits, N, H, W, C, BDBNN_GRAD_FP16S, sums_ws, gmax_bits, consts_ws, dgamma, dbeta,
                                amax_bits, gys, stream);
}

extern "C" int bdbnn_pool2_bn_eval_hardtanh(const int16_t* y_int, const float* scale, const float* shift, int32_t N,
                                            int32_t H, int32_t W, int32_t C, float* z, uint16_t* zb, uint8_t* zb8,
                                            int32_t fmt, void* stream) {
  int rc = pool2_dims_ok("pool2_bn_eval_hardtanh", N, H, W, C);
  if (rc) return rc;
  BDBNN_REQUIRE(y_int && scale && shift && z, "pool2_bn_eval_hardtanh: NULL pointer");
  cudaStream_t st = cudaStream_t(stream);
  const int C4 = C / 4;
  const int64_t n4 = int64_t(N) * (H / 2) * (W / 2) * C4;
  pool2_eval_kernel<<<bn_grid(n4, C4), kBnThreads, 0, st>>>(y_int, scale, shift, H, W, C4, n4,
                                                           reinterpret_cast<float4*>(z), reinterpret_cast<uint2*>(zb),
                                                           reinterpret_cast<uint32_t*>(zb8),
                                                           fmt == BDBNN_FMT_FP16 ? 0x3C00u : 0x3F80u);
  return check_launch("pool2_eval_kernel");
}

extern "C" int bdbnn_real_pool2_bn_eval_hardtanh(const float* y, const float* scale, const float* shift, int32_t N,
                                                 int32_t H, int32_t W, int32_t C, float* z, uint32_t* z_amax_bits,
                                                 void* stream) {
  int rc = pool2_dims_ok("real_pool2_bn_eval_hardtanh", N, H, W, C);
  if (rc) return rc;
  BDBNN_REQUIRE(y && scale && shift && z && z_amax_bits, "real_pool2_bn_eval_hardtanh: NULL pointer");
  cudaStream_t st = cudaStream_t(stream);
  const int C4 = C / 4;
  const int64_t n4 = int64_t(N) * (H / 2) * (W / 2) * C4;
  BDBNN_CUDA(cudaMemsetAsync(z_amax_bits, 0, sizeof(uint32_t), st));
  real_pool2_eval_kernel<<<bn_grid(n4, C4), kBnThreads, 0, st>>>(y, scale, shift, H, W, C4, n4,
                                                                 reinterpret_cast<float4*>(z), z_amax_bits);
  return check_launch("real_pool2_eval_kernel");
}

extern "C" int bdbnn_bn_bwd_pack_i16(const float* gz, const int16_t* y_int, const float* alpha, const float* mean,
                                     const float* invstd, const float* gamma, const float* gscale,
                                     const uint32_t* ymax_bits, int64_t n_pix, int32_t C, int32_t grad_mode,
                                     double* sums_ws, uint32_t* gmax_bits, float* consts_ws, float* dgamma,
                                     float* dbeta, uint32_t* amax_bits, uint16_t* gys, int32_t stats_ready,
                                     void* stream) {
  BDBNN_REQUIRE(alpha != nullptr, "bn_bwd_pack_i16: NULL alpha");
  return bn_bwd_pack_impl(gz, y_int, alpha, mean, invstd, gamma, gscale, ymax_bits, n_pix, C, grad_mode, sums_ws,
                          gmax_bits, consts_ws, dgamma, dbeta, amax_bits, gys, stats_ready, stream);
}

// ===================================================================================================
// Stem: BatchNorm(train) + MaxPool fused (the 112x112x64 stem activation is the largest tensor of the
// step: 822 MB at N=256).  The BN output is never materialised:
//   forward : bn_reduce<fwd>(y) -> bn_finalize -> bn_pool_fwd: z = maxpool(a*y+b) + winner index +
//             y at the winner (for the backward's yhat) [+ the first binary conv's sign/mask/+-1 packs]
//   backward: bn_reduce<bwd>(g_pool, y_sel) over the POOLED tensors (every pooled gradient lands on
//             exactly one input position, so sum gz = sum g_pool and sum gz*yhat = sum g_pool*yhat_sel)
//             -> bn_bwd_bound -> bn_pool_bwd: gy = a*(gz - m1 - yhat*m2) for every input position, with
//             gz gathered from the (<= 4) windows whose winner is that position.
// torch.nn.MaxPool2d semantics on the BN output (first maximum in scan order wins, NaN propagates).
// ===================================================================================================
namespace bdbnn {

// RELU of bn_pool_fwd_k3s2_kernel (PACK false): z = relu(max) = max(relu(v)); mask_bits = ReLU's gradient mask
// (relu_bits4) as bn_apply_add_pack's RELU words, the winner byte 0xff (no tap: the backward gives that window's
// gradient to no position) where the bit is 0, and the bits of max|z| into z_amax.
__device__ __forceinline__ void pool_relu(float4& m, uint32_t& w4, uint32_t& zmax, uint32_t* __restrict__ mask_bits,
                                          int64_t i, uint32_t group_mask, int sh, int lane) {
  const uint32_t m4 = relu_bits4(m);
  m.x = relu_f(m.x); m.y = relu_f(m.y); m.z = relu_f(m.z); m.w = relu_f(m.w);
  w4 |= (m4 & 1u ? 0u : 0xffu) | (m4 & 2u ? 0u : 0xff00u) | (m4 & 4u ? 0u : 0xff0000u) | (m4 & 8u ? 0u : 0xff000000u);
  zmax = max(zmax, max(max(__float_as_uint(fabsf(m.x)), __float_as_uint(fabsf(m.y))),
                       max(__float_as_uint(fabsf(m.z)), __float_as_uint(fabsf(m.w)))));
  const uint32_t mw = __reduce_or_sync(group_mask, m4 << sh);
  if ((lane & 7) == 0) mask_bits[i >> 3] = mw;
}

__device__ __forceinline__ void pool_relu_amax(uint32_t zmax, uint32_t* __restrict__ z_amax) {
  zmax = __reduce_max_sync(0xffffffffu, zmax);      // every lane of the (whole) warp gets here
  if ((threadIdx.x & 31) == 0 && zmax != 0u) atomicMax(z_amax, zmax);
}

template <bool PACK>
__global__ void __launch_bounds__(kBnThreads)
bn_pool_fwd_kernel(const float4* __restrict__ y, const float* __restrict__ a, const float* __restrict__ b,
                   int N, int H, int W, int C4, int Ho, int Wo, int k, int s, int p, int64_t total,
                   float4* __restrict__ z, float4* __restrict__ ysel, uint32_t* __restrict__ idx,
                   uint32_t* __restrict__ sign_bits, uint32_t* __restrict__ mask_bits, uint2* __restrict__ xb4,
                   uint32_t* __restrict__ xb8, uint32_t one16) {
  const int lane = threadIdx.x & 31;
  const uint32_t group_mask = 0xffu << (lane & 24);
  const int sh = (lane & 7) * 4;
  const uint32_t pos = one16, neg = one16 | 0x8000u;
  const int64_t nthreads = int64_t(gridDim.x) * blockDim.x;     // multiple of C4
  int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int c = int(i % C4);
  const float4 av = *reinterpret_cast<const float4*>(a + c * 4);
  const float4 bv = *reinterpret_cast<const float4*>(b + c * 4);
  for (; i < total; i += nthreads) {
    int64_t q = i / C4;
    const int wo = int(q % Wo); q /= Wo;
    const int ho = int(q % Ho);
    const int n = int(q / Ho);
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f), ys = m;
    uint32_t w4 = 0;
    bool first = true;
    for (int r = 0; r < k; ++r) {
      const int h = ho * s - p + r;
      if (h < 0 || h >= H) continue;
      for (int t = 0; t < k; ++t) {
        const int w = wo * s - p + t;
        if (w < 0 || w >= W) continue;
        const float4 yv = __ldg(y + ((int64_t(n) * H + h) * W + w) * C4 + c);
        const float4 v = make_float4(fmaf(yv.x, av.x, bv.x), fmaf(yv.y, av.y, bv.y), fmaf(yv.z, av.z, bv.z),
                                     fmaf(yv.w, av.w, bv.w));
        const uint32_t tap = uint32_t(r * k + t);
        if (first || v.x > m.x || v.x != v.x) { m.x = v.x; ys.x = yv.x; w4 = (w4 & 0xffffff00u) | tap; }
        if (first || v.y > m.y || v.y != v.y) { m.y = v.y; ys.y = yv.y; w4 = (w4 & 0xffff00ffu) | (tap << 8); }
        if (first || v.z > m.z || v.z != v.z) { m.z = v.z; ys.z = yv.z; w4 = (w4 & 0xff00ffffu) | (tap << 16); }
        if (first || v.w > m.w || v.w != v.w) { m.w = v.w; ys.w = yv.w; w4 = (w4 & 0x00ffffffu) | (tap << 24); }
        first = false;
      }
    }
    z[i] = m;
    ysel[i] = ys;
    idx[i] = w4;
    if (PACK) {
      const uint32_t s0 = m.x >= 0.0f, s1 = m.y >= 0.0f, s2 = m.z >= 0.0f, s3 = m.w >= 0.0f;
      const uint32_t m0 = fabsf(m.x) <= 1.0f, m1 = fabsf(m.y) <= 1.0f, m2 = fabsf(m.z) <= 1.0f,
                     m3 = fabsf(m.w) <= 1.0f;
      const uint32_t sw = __reduce_or_sync(group_mask, (s0 | (s1 << 1) | (s2 << 2) | (s3 << 3)) << sh);
      const uint32_t mw = __reduce_or_sync(group_mask, (m0 | (m1 << 1) | (m2 << 2) | (m3 << 3)) << sh);
      if ((lane & 7) == 0) {
        sign_bits[i >> 3] = sw;
        mask_bits[i >> 3] = mw;
      }
      uint2 o;
      o.x = (s0 ? pos : neg) | ((s1 ? pos : neg) << 16);
      o.y = (s2 ? pos : neg) | ((s3 ? pos : neg) << 16);
      xb4[i] = o;
      if (xb8 != nullptr)
        xb8[i] = 0x38383838u | ((s0 ? 0u : 0x80u) | (s1 ? 0u : 0x8000u) | (s2 ? 0u : 0x800000u) | (s3 ? 0u : 0x80000000u));
    }
  }
}

// 3x3 / stride-2 / pad-1 forward (the stem's pool) with one block per output row (n, ho): the three input
// row pointers and the row validity are per block, the tap loop is unrolled, and the winner index is kept
// as four small integers instead of read-modify-write byte lanes — about half the instructions of the
// generic kernel, which is bound by instruction issue rather than by memory.
// Same scan order and NaN rule, so outputs are bit-identical.  blockDim.x is a multiple of C4.
template <bool PACK, bool RELU = false>
__global__ void __launch_bounds__(kBnThreads)
bn_pool_fwd_k3s2_kernel(const float4* __restrict__ y, const float* __restrict__ a, const float* __restrict__ b,
                        int H, int W, int C4, int Ho, int Wo, float4* __restrict__ z, float4* __restrict__ ysel,
                        uint32_t* __restrict__ idx, uint32_t* __restrict__ sign_bits,
                        uint32_t* __restrict__ mask_bits, uint2* __restrict__ xb4, uint32_t* __restrict__ xb8,
                        uint32_t one16, uint32_t* __restrict__ z_amax = nullptr) {
  const int lane = threadIdx.x & 31;
  const uint32_t group_mask = 0xffu << (lane & 24);
  const int sh = (lane & 7) * 4;
  const uint32_t pos = one16, neg = one16 | 0x8000u;
  const int c = threadIdx.x % C4;
  const float4 av = *reinterpret_cast<const float4*>(a + c * 4);
  const float4 bv = *reinterpret_cast<const float4*>(b + c * 4);
  const int n = blockIdx.x / Ho, ho = blockIdx.x - n * Ho;
  const int h0 = 2 * ho - 1;
  const float4* rows[3];
  bool rok[3];
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int h = h0 + r;
    rok[r] = h >= 0 && h < H;
    rows[r] = y + (int64_t(n) * H + (rok[r] ? h : 0)) * W * C4 + c;
  }
  const int per_row = Wo * C4;               // multiple of 8 when PACK (C % 32 == 0)
  const int64_t out0 = (int64_t(n) * Ho + ho) * per_row;
  uint32_t zmax = 0u;
  for (int j = threadIdx.x; j < per_row; j += blockDim.x) {
    const int wo = j / C4;
    const int w0 = 2 * wo - 1;
    float4 m = make_float4(0.f, 0.f, 0.f, 0.f), ys = m;
    uint32_t tx = 0, ty = 0, tz = 0, tw = 0;
    bool first = true;
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      if (!rok[r]) continue;
#pragma unroll
      for (int t = 0; t < 3; ++t) {
        const int w = w0 + t;
        if (w < 0 || w >= W) continue;
        const float4 yv = __ldg(rows[r] + int64_t(w) * C4);
        const float4 v = make_float4(fmaf(yv.x, av.x, bv.x), fmaf(yv.y, av.y, bv.y), fmaf(yv.z, av.z, bv.z),
                                     fmaf(yv.w, av.w, bv.w));
        const uint32_t tap = uint32_t(r * 3 + t);
        if (first || v.x > m.x || v.x != v.x) { m.x = v.x; ys.x = yv.x; tx = tap; }
        if (first || v.y > m.y || v.y != v.y) { m.y = v.y; ys.y = yv.y; ty = tap; }
        if (first || v.z > m.z || v.z != v.z) { m.z = v.z; ys.z = yv.z; tz = tap; }
        if (first || v.w > m.w || v.w != v.w) { m.w = v.w; ys.w = yv.w; tw = tap; }
        first = false;
      }
    }
    const int64_t i = out0 + j;
    uint32_t w4 = tx | (ty << 8) | (tz << 16) | (tw << 24);
    if (RELU) pool_relu(m, w4, zmax, mask_bits, i, group_mask, sh, lane);
    z[i] = m;
    ysel[i] = ys;
    idx[i] = w4;
    if (PACK) {
      const uint32_t s0 = m.x >= 0.0f, s1 = m.y >= 0.0f, s2 = m.z >= 0.0f, s3 = m.w >= 0.0f;
      const uint32_t m0 = fabsf(m.x) <= 1.0f, m1 = fabsf(m.y) <= 1.0f, m2 = fabsf(m.z) <= 1.0f,
                     m3 = fabsf(m.w) <= 1.0f;
      const uint32_t sw = __reduce_or_sync(group_mask, (s0 | (s1 << 1) | (s2 << 2) | (s3 << 3)) << sh);
      const uint32_t mw = __reduce_or_sync(group_mask, (m0 | (m1 << 1) | (m2 << 2) | (m3 << 3)) << sh);
      if ((lane & 7) == 0) {
        sign_bits[i >> 3] = sw;
        mask_bits[i >> 3] = mw;
      }
      uint2 o;
      o.x = (s0 ? pos : neg) | ((s1 ? pos : neg) << 16);
      o.y = (s2 ? pos : neg) | ((s3 ? pos : neg) << 16);
      xb4[i] = o;
      if (xb8 != nullptr)
        xb8[i] = 0x38383838u | ((s0 ? 0u : 0x80u) | (s1 ? 0u : 0x8000u) | (s2 ? 0u : 0x800000u) | (s3 ? 0u : 0x80000000u));
    }
  }
  if (RELU) pool_relu_amax(zmax, z_amax);
}

// gy[n,h,w,c] = A*(gz - m1 - (y-mean)*m2'),  gz = sum of g_pool over the windows won by (h,w);
// consts[c] = {m1, m2*invstd, mean, A} from bn_bwd_bound_kernel (gscale = 1).
// HALF: write gys = fp16(gy * 2^e) (e from the bound in amax_bits: the stem conv's wgrad operand, so the
// 4-byte gradient of the largest activation of the step is never written) instead of fp32 gy.
template <bool HALF>
__global__ void __launch_bounds__(kBnThreads)
bn_pool_bwd_kernel(const float4* __restrict__ gpool, const uint32_t* __restrict__ idx, const float4* __restrict__ y,
                   const float4* __restrict__ consts, int N, int H, int W, int C4, int Ho, int Wo, int k, int s,
                   int p, int64_t total, float4* __restrict__ gy, const uint32_t* __restrict__ amax_bits,
                   uint2* __restrict__ gys) {
  const float up = HALF ? amax_pow2_scale(__ldg(amax_bits), false) : 1.0f;
  const int64_t nthreads = int64_t(gridDim.x) * blockDim.x;     // multiple of C4
  int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int c = int(i % C4);
  const float4 k0 = consts[c * 4 + 0], k1 = consts[c * 4 + 1], k2 = consts[c * 4 + 2], k3 = consts[c * 4 + 3];
  for (; i < total; i += nthreads) {
    int64_t q = i / C4;
    const int w = int(q % W); q /= W;
    const int h = int(q % H);
    const int n = int(q / H);
    float4 gz = make_float4(0.f, 0.f, 0.f, 0.f);
    int ho0 = (h + p - k + s) / s;
    if (h + p - k + 1 <= 0) ho0 = 0;
    int wo0 = (w + p - k + s) / s;
    if (w + p - k + 1 <= 0) wo0 = 0;
    const int ho1 = min((h + p) / s, Ho - 1), wo1 = min((w + p) / s, Wo - 1);
    for (int ho = ho0; ho <= ho1; ++ho) {
      const uint32_t r = uint32_t(h - (ho * s - p));
      for (int wo = wo0; wo <= wo1; ++wo) {
        const uint32_t tap = r * uint32_t(k) + uint32_t(w - (wo * s - p));
        const int64_t o = ((int64_t(n) * Ho + ho) * Wo + wo) * C4 + c;
        const uint32_t w4 = __ldg(idx + o);
        const float4 g = __ldg(gpool + o);
        if ((w4 & 0xffu) == tap) gz.x += g.x;
        if (((w4 >> 8) & 0xffu) == tap) gz.y += g.y;
        if (((w4 >> 16) & 0xffu) == tap) gz.z += g.z;
        if ((w4 >> 24) == tap) gz.w += g.w;
      }
    }
    const float4 v = __ldcs(y + i);
    float4 o;
    o.x = (gz.x - k0.x - (v.x - k0.z) * k0.y) * k0.w;
    o.y = (gz.y - k1.x - (v.y - k1.z) * k1.y) * k1.w;
    o.z = (gz.z - k2.x - (v.z - k2.z) * k2.y) * k2.w;
    o.w = (gz.w - k3.x - (v.w - k3.z) * k3.y) * k3.w;
    if (HALF) {
      const __half2 h0 = __floats2half2_rn(o.x * up, o.y * up), h1 = __floats2half2_rn(o.z * up, o.w * up);
      gys[i] = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
    } else {
      gy[i] = o;
    }
  }
}

// Same result for the 3x3 / stride-2 / pad-1 pool (the stem's), restructured so that one thread owns a 2x2
// block of input positions (rows 2a, 2a+1; columns 2b, 2b+1) of one channel quad: the four positions are
// covered by the same four pooling windows (a..a+1, b..b+1), so each window's winner word and gradient
// are loaded once for four outputs (the generic kernel re-reads them 2.25x per output on average) and
// the index arithmetic is per block, not per element.  Windows are visited in the generic kernel's
// order, so the sums are bit-identical.  blockDim.x must be a multiple of C4.
template <bool HALF>
__global__ void __launch_bounds__(kBnThreads)
bn_pool_bwd_k3s2_kernel(const float4* __restrict__ gpool, const uint32_t* __restrict__ idx,
                        const float4* __restrict__ y, const float4* __restrict__ consts, int H, int W, int C4,
                        int Ho, int Wo, int HB, int WB, float4* __restrict__ gy,
                        const uint32_t* __restrict__ amax_bits, uint2* __restrict__ gys) {
  const float up = HALF ? amax_pow2_scale(__ldg(amax_bits), false) : 1.0f;
  const int c = threadIdx.x % C4;
  const float4 k0 = consts[c * 4 + 0], k1 = consts[c * 4 + 1], k2 = consts[c * 4 + 2], k3 = consts[c * 4 + 3];
  const int n = blockIdx.x / HB, a = blockIdx.x - n * HB;
  const int h0 = 2 * a, h1 = 2 * a + 1;
  const int per_row = WB * C4;
  for (int j = threadIdx.x; j < per_row; j += blockDim.x) {
    const int b = j / C4;
    const int w0 = 2 * b, w1 = 2 * b + 1;
    // windows (a,b) (a,b+1) (a+1,b) (a+1,b+1)
    float4 g[4];
    uint32_t wd[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int ho = a + (q >> 1), wo = b + (q & 1);
      if (ho < Ho && wo < Wo) {
        const int64_t o = ((int64_t(n) * Ho + ho) * Wo + wo) * C4 + c;
        wd[q] = __ldg(idx + o);
        g[q] = __ldg(gpool + o);
      } else {
        wd[q] = 0xffffffffu;                      // tap 255 never matches
        g[q] = make_float4(0.f, 0.f, 0.f, 0.f);
      }
    }
    auto pick = [&](float4& acc, int q, uint32_t tap) {
      const uint32_t w4 = wd[q];
      if ((w4 & 0xffu) == tap) acc.x += g[q].x;
      if (((w4 >> 8) & 0xffu) == tap) acc.y += g[q].y;
      if (((w4 >> 16) & 0xffu) == tap) acc.z += g[q].z;
      if ((w4 >> 24) == tap) acc.w += g[q].w;
    };
    float4 z00 = make_float4(0.f, 0.f, 0.f, 0.f), z01 = z00, z10 = z00, z11 = z00;
    pick(z00, 0, 4u);                                             // (2a  , 2b  ): centre of window (a,b)
    pick(z01, 0, 5u); pick(z01, 1, 3u);                           // (2a  , 2b+1)
    pick(z10, 0, 7u); pick(z10, 2, 1u);                           // (2a+1, 2b  )
    pick(z11, 0, 8u); pick(z11, 1, 6u); pick(z11, 2, 2u); pick(z11, 3, 0u);
    auto emit = [&](int h, int w, const float4& gz) {
      if (h >= H || w >= W) return;
      const int64_t i = ((int64_t(n) * H + h) * W + w) * C4 + c;
      const float4 v = __ldcs(y + i);
      float4 o;
      o.x = (gz.x - k0.x - (v.x - k0.z) * k0.y) * k0.w;
      o.y = (gz.y - k1.x - (v.y - k1.z) * k1.y) * k1.w;
      o.z = (gz.z - k2.x - (v.z - k2.z) * k2.y) * k2.w;
      o.w = (gz.w - k3.x - (v.w - k3.z) * k3.y) * k3.w;
      if (HALF) {
        const __half2 p0 = __floats2half2_rn(o.x * up, o.y * up), p1 = __floats2half2_rn(o.z * up, o.w * up);
        gys[i] = make_uint2(*reinterpret_cast<const uint32_t*>(&p0), *reinterpret_cast<const uint32_t*>(&p1));
      } else {
        gy[i] = o;
      }
    };
    emit(h0, w0, z00);
    emit(h0, w1, z01);
    emit(h1, w0, z10);
    emit(h1, w1, z11);
  }
}

}  // namespace bdbnn

using namespace bdbnn;

static int pool_geom_ok(int N, int H, int W, int C, int k, int s, int p, int Ho, int Wo) {
  BDBNN_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && (C & 3) == 0 && C <= 4096, "bn_pool: bad N/H/W/C");
  BDBNN_REQUIRE(k > 0 && k <= 15 && s > 0 && p >= 0 && 2 * p <= k, "bn_pool: bad k/stride/pad");
  BDBNN_REQUIRE(Ho == (H + 2 * p - k) / s + 1 && Wo == (W + 2 * p - k) / s + 1 && Ho > 0 && Wo > 0,
                "bn_pool: inconsistent output size");
  return BDBNN_OK;
}

// relu_amax != NULL: bdbnn_bn_pool_fwd_relu (mask_bits are ReLU's, no +-1 packs)
static int bn_pool_fwd_impl(const float* y, const float* gamma, const float* beta, int32_t N, int32_t H, int32_t W,
                            int32_t C, int32_t k, int32_t stride, int32_t pad, int32_t Ho, int32_t Wo, float eps,
                            float momentum, float* running_mean, float* running_var, double* sums_ws,
                            uint32_t* ymax_bits, float* mean, float* invstd, float* ab_ws, float* z, float* y_sel,
                            uint8_t* idx, uint32_t* sign_bits, uint32_t* mask_bits, uint16_t* xb, uint8_t* xb_fp8,
                            int32_t fmt, int32_t stats_ready, void* stream, uint32_t* relu_amax = nullptr) {
  int rc = pool_geom_ok(N, H, W, C, k, stride, pad, Ho, Wo);
  if (rc) return rc;
  const bool pack = sign_bits != nullptr;
  const bool relu = relu_amax != nullptr;
  BDBNN_REQUIRE(y && gamma && beta && sums_ws && ymax_bits && mean && invstd && ab_ws && z && y_sel && idx,
                "bn_pool_fwd: NULL pointer");
  BDBNN_REQUIRE(!pack || ((C & 31) == 0 && mask_bits && xb), "bn_pool_fwd: packing needs C %% 32 == 0 and all pack outputs");
  BDBNN_REQUIRE(!relu || (!pack && (C & 31) == 0 && mask_bits), "bn_pool_fwd_relu: needs C %% 32 == 0 and mask_bits");
  // the ReLU is in the 3x3 / stride-2 / pad-1 kernel only (the pool of the torchvision ResNet stem)
  BDBNN_REQUIRE(!relu || (k == 3 && stride == 2 && pad == 1 && C <= 4 * kBnThreads && kBnThreads % (C / 4) == 0),
                "bn_pool_fwd_relu: needs the 3x3 / stride-2 / pad-1 pool and C dividing 1024");
  cudaStream_t st = cudaStream_t(stream);
  const int C4 = C / 4;
  const int64_t n_pix = int64_t(N) * H * W;
  if (!stats_ready) {
    BDBNN_CUDA(cudaMemsetAsync(sums_ws, 0, size_t(2 * C) * sizeof(double), st));
    BDBNN_CUDA(cudaMemsetAsync(ymax_bits, 0, size_t(C) * sizeof(uint32_t), st));
    rc = bn_stats_launch(y, n_pix, C, sums_ws, ymax_bits, st);
    if (rc) return rc;
  }
  float* a = ab_ws;
  float* b = ab_ws + C;
  bn_finalize_kernel<<<(C + 127) / 128, 128, 0, st>>>(sums_ws, n_pix, C, eps, gamma, beta, mean, invstd, a, b,
                                                       running_mean, running_var, momentum);
  rc = check_launch("bn_finalize_kernel");
  if (rc) return rc;
  const int64_t total = int64_t(N) * Ho * Wo * C4;
  const int grid = bn_grid(total, C4);
  const float4* y4 = reinterpret_cast<const float4*>(y);
  if (relu) BDBNN_CUDA(cudaMemsetAsync(relu_amax, 0, sizeof(uint32_t), st));
  // PACK (and RELU's mask words) need the 8 lanes of a 32-channel word inside one iteration of one warp: per-row work
  // and the block size must be multiples of 8 quads, which C % 32 == 0 gives when blockDim is a multiple of C4
  if (k == 3 && stride == 2 && pad == 1 && C4 <= kBnThreads &&
      (!(pack || relu) || (C4 % 8 == 0 && kBnThreads % C4 == 0))) {
    const int threads = (kBnThreads / C4) * C4;
    const unsigned rows_grid = unsigned(N) * unsigned(Ho);
    if (relu)
      bn_pool_fwd_k3s2_kernel<false, true><<<rows_grid, threads, 0, st>>>(
          y4, a, b, H, W, C4, Ho, Wo, reinterpret_cast<float4*>(z), reinterpret_cast<float4*>(y_sel),
          reinterpret_cast<uint32_t*>(idx), nullptr, mask_bits, nullptr, nullptr, 0u, relu_amax);
    else if (pack)
      bn_pool_fwd_k3s2_kernel<true><<<rows_grid, threads, 0, st>>>(
          y4, a, b, H, W, C4, Ho, Wo, reinterpret_cast<float4*>(z), reinterpret_cast<float4*>(y_sel),
          reinterpret_cast<uint32_t*>(idx), sign_bits, mask_bits, reinterpret_cast<uint2*>(xb),
          reinterpret_cast<uint32_t*>(xb_fp8), fmt == BDBNN_FMT_FP16 ? 0x3C00u : 0x3F80u);
    else
      bn_pool_fwd_k3s2_kernel<false><<<rows_grid, threads, 0, st>>>(
          y4, a, b, H, W, C4, Ho, Wo, reinterpret_cast<float4*>(z), reinterpret_cast<float4*>(y_sel),
          reinterpret_cast<uint32_t*>(idx), nullptr, nullptr, nullptr, nullptr, 0u);
    return check_launch("bn_pool_fwd_k3s2_kernel");
  }
  if (pack) {
    bn_pool_fwd_kernel<true><<<grid, kBnThreads, 0, st>>>(
        y4, a, b, N, H, W, C4, Ho, Wo, k, stride, pad, total, reinterpret_cast<float4*>(z),
        reinterpret_cast<float4*>(y_sel), reinterpret_cast<uint32_t*>(idx), sign_bits, mask_bits,
        reinterpret_cast<uint2*>(xb), reinterpret_cast<uint32_t*>(xb_fp8), fmt == BDBNN_FMT_FP16 ? 0x3C00u : 0x3F80u);
  } else {
    bn_pool_fwd_kernel<false><<<grid, kBnThreads, 0, st>>>(
        y4, a, b, N, H, W, C4, Ho, Wo, k, stride, pad, total, reinterpret_cast<float4*>(z),
        reinterpret_cast<float4*>(y_sel), reinterpret_cast<uint32_t*>(idx), nullptr, nullptr, nullptr, nullptr, 0u);
  }
  return check_launch("bn_pool_fwd_kernel");
}

extern "C" int bdbnn_bn_pool_fwd(const float* y, const float* gamma, const float* beta, int32_t N, int32_t H,
                                 int32_t W, int32_t C, int32_t k, int32_t stride, int32_t pad, int32_t Ho,
                                 int32_t Wo, float eps, float momentum, float* running_mean, float* running_var,
                                 double* sums_ws, uint32_t* ymax_bits, float* mean, float* invstd, float* ab_ws,
                                 float* z, float* y_sel, uint8_t* idx, uint32_t* sign_bits, uint32_t* mask_bits,
                                 uint16_t* xb, uint8_t* xb_fp8, int32_t fmt, int32_t stats_ready, void* stream) {
  return bn_pool_fwd_impl(y, gamma, beta, N, H, W, C, k, stride, pad, Ho, Wo, eps, momentum, running_mean, running_var,
                          sums_ws, ymax_bits, mean, invstd, ab_ws, z, y_sel, idx, sign_bits, mask_bits, xb, xb_fp8, fmt,
                          stats_ready, stream);
}

extern "C" int bdbnn_bn_pool_fwd_relu(const float* y, const float* gamma, const float* beta, int32_t N, int32_t H,
                                      int32_t W, int32_t C, int32_t k, int32_t stride, int32_t pad, int32_t Ho,
                                      int32_t Wo, float eps, float momentum, float* running_mean, float* running_var,
                                      double* sums_ws, uint32_t* ymax_bits, float* mean, float* invstd, float* ab_ws,
                                      float* z, float* y_sel, uint8_t* idx, uint32_t* mask_bits, uint32_t* z_amax_bits,
                                      int32_t stats_ready, void* stream) {
  BDBNN_REQUIRE(z_amax_bits != nullptr, "bn_pool_fwd_relu: NULL z_amax_bits");
  return bn_pool_fwd_impl(y, gamma, beta, N, H, W, C, k, stride, pad, Ho, Wo, eps, momentum, running_mean, running_var,
                          sums_ws, ymax_bits, mean, invstd, ab_ws, z, y_sel, idx, nullptr, mask_bits, nullptr, nullptr,
                          BDBNN_FMT_FP16, stats_ready, stream, z_amax_bits);
}

// relu_mask != NULL: bdbnn_bn_pool_bwd_relu (the pooled gradient masked by ReLU's words in the sums; the scatter needs
// no mask, the forward wrote no winner where z is not > 0)
static int bn_pool_bwd_impl(const float* g_pool, const uint8_t* idx, const float* y, const float* y_sel,
                            const float* mean, const float* invstd, const float* gamma, const float* ones,
                            const uint32_t* ymax_bits, int32_t N, int32_t H, int32_t W, int32_t C, int32_t k,
                            int32_t stride, int32_t pad, int32_t Ho, int32_t Wo, double* sums_ws, uint32_t* gmax_bits,
                            float* consts_ws, float* dgamma, float* dbeta, uint32_t* amax_scratch, float* gy,
                            uint16_t* gys, void* stream, const uint32_t* relu_mask = nullptr) {
  int rc = pool_geom_ok(N, H, W, C, k, stride, pad, Ho, Wo);
  if (rc) return rc;
  BDBNN_REQUIRE(g_pool && idx && y && y_sel && mean && invstd && gamma && ones && ymax_bits && sums_ws && gmax_bits &&
                    consts_ws && dgamma && dbeta && amax_scratch && (gy || gys),
                "bn_pool_bwd: NULL pointer");
  BDBNN_REQUIRE(relu_mask == nullptr || (C & 31) == 0, "bn_pool_bwd_relu: the mask words need C %% 32 == 0");
  cudaStream_t st = cudaStream_t(stream);
  const int C4 = C / 4;
  const int64_t n_pool = int64_t(N) * Ho * Wo, n_full = int64_t(N) * H * W;
  BDBNN_CUDA(cudaMemsetAsync(sums_ws, 0, size_t(2 * C) * sizeof(double), st));
  BDBNN_CUDA(cudaMemsetAsync(gmax_bits, 0, size_t(C) * sizeof(uint32_t), st));
  if (relu_mask != nullptr)
    rc = bn_reduce_launch<true, false, false, true>(bn_grid(n_pool * C4 / 8, C4, 3),
                                                    reinterpret_cast<const float4*>(g_pool),
                                                    reinterpret_cast<const float4*>(y_sel), mean, invstd, n_pool, C4,
                                                    sums_ws, gmax_bits, nullptr, st, nullptr, relu_mask);
  else
    rc = bn_reduce_launch<true>(bn_grid(n_pool * C4 / 8, C4, 3), reinterpret_cast<const float4*>(g_pool),
                                reinterpret_cast<const float4*>(y_sel), mean, invstd, n_pool, C4, sums_ws, gmax_bits,
                                nullptr, st);
  if (rc) return rc;
  // means are over the FULL-resolution element count; gscale = 1 (`ones`)
  const int per_dim = (k + stride - 1) / stride;          // pooling windows covering one position, per axis
  bn_bwd_bound_kernel<<<1, 256, 0, st>>>(sums_ws, gmax_bits, ymax_bits, n_full, C, mean, invstd, gamma, ones,
                                         reinterpret_cast<float4*>(consts_ws), dgamma, dbeta, amax_scratch,
                                         float(per_dim * per_dim));
  rc = check_launch("bn_bwd_bound_kernel");
  if (rc) return rc;
  const int64_t total = n_full * C4;
  if (k == 3 && stride == 2 && pad == 1 && C4 <= kBnThreads) {
    const int HB = (H + 1) / 2, WB = (W + 1) / 2;
    const int threads = (kBnThreads / C4) * C4;
    const unsigned grid = unsigned(N) * unsigned(HB);
    if (gys != nullptr)
      bn_pool_bwd_k3s2_kernel<true><<<grid, threads, 0, st>>>(
          reinterpret_cast<const float4*>(g_pool), reinterpret_cast<const uint32_t*>(idx),
          reinterpret_cast<const float4*>(y), reinterpret_cast<const float4*>(consts_ws), H, W, C4, Ho, Wo, HB, WB,
          nullptr, amax_scratch, reinterpret_cast<uint2*>(gys));
    else
      bn_pool_bwd_k3s2_kernel<false><<<grid, threads, 0, st>>>(
          reinterpret_cast<const float4*>(g_pool), reinterpret_cast<const uint32_t*>(idx),
          reinterpret_cast<const float4*>(y), reinterpret_cast<const float4*>(consts_ws), H, W, C4, Ho, Wo, HB, WB,
          reinterpret_cast<float4*>(gy), nullptr, nullptr);
    return check_launch("bn_pool_bwd_k3s2_kernel");
  }
  if (gys != nullptr)
    bn_pool_bwd_kernel<true><<<bn_grid(total, C4), kBnThreads, 0, st>>>(
        reinterpret_cast<const float4*>(g_pool), reinterpret_cast<const uint32_t*>(idx),
        reinterpret_cast<const float4*>(y), reinterpret_cast<const float4*>(consts_ws), N, H, W, C4, Ho, Wo, k,
        stride, pad, total, nullptr, amax_scratch, reinterpret_cast<uint2*>(gys));
  else
    bn_pool_bwd_kernel<false><<<bn_grid(total, C4), kBnThreads, 0, st>>>(
        reinterpret_cast<const float4*>(g_pool), reinterpret_cast<const uint32_t*>(idx),
        reinterpret_cast<const float4*>(y), reinterpret_cast<const float4*>(consts_ws), N, H, W, C4, Ho, Wo, k,
        stride, pad, total, reinterpret_cast<float4*>(gy), nullptr, nullptr);
  return check_launch("bn_pool_bwd_kernel");
}

extern "C" int bdbnn_bn_pool_bwd(const float* g_pool, const uint8_t* idx, const float* y, const float* y_sel,
                                 const float* mean, const float* invstd, const float* gamma, const float* ones,
                                 const uint32_t* ymax_bits, int32_t N, int32_t H, int32_t W, int32_t C, int32_t k,
                                 int32_t stride, int32_t pad, int32_t Ho, int32_t Wo, double* sums_ws,
                                 uint32_t* gmax_bits, float* consts_ws, float* dgamma, float* dbeta,
                                 uint32_t* amax_scratch, float* gy, uint16_t* gys, void* stream) {
  return bn_pool_bwd_impl(g_pool, idx, y, y_sel, mean, invstd, gamma, ones, ymax_bits, N, H, W, C, k, stride, pad, Ho,
                          Wo, sums_ws, gmax_bits, consts_ws, dgamma, dbeta, amax_scratch, gy, gys, stream);
}

extern "C" int bdbnn_bn_pool_bwd_relu(const float* g_pool, const uint8_t* idx, const uint32_t* mask_bits,
                                      const float* y, const float* y_sel, const float* mean, const float* invstd,
                                      const float* gamma, const float* ones, const uint32_t* ymax_bits, int32_t N,
                                      int32_t H, int32_t W, int32_t C, int32_t k, int32_t stride, int32_t pad,
                                      int32_t Ho, int32_t Wo, double* sums_ws, uint32_t* gmax_bits, float* consts_ws,
                                      float* dgamma, float* dbeta, uint32_t* amax_scratch, float* gy, uint16_t* gys,
                                      void* stream) {
  BDBNN_REQUIRE(mask_bits != nullptr, "bn_pool_bwd_relu: NULL mask_bits");
  return bn_pool_bwd_impl(g_pool, idx, y, y_sel, mean, invstd, gamma, ones, ymax_bits, N, H, W, C, k, stride, pad, Ho,
                          Wo, sums_ws, gmax_bits, consts_ws, dgamma, dbeta, amax_scratch, gy, gys, stream, mask_bits);
}
