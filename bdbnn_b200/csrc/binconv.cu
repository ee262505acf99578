// Binary convolution on CUDA cores: XNOR-popcount forward + generic (any-shape) backward kernels.
// The tensor-core (wgmma) implicit-GEMM versions live in tc_conv.cu; the kernels here are the
// bit-serial path BASELINE.json:north_star prescribes and the shape-generic fallback.
#include "common.cuh"

namespace bdbnn {

// -------------------------------------------------------------------------------------------------
// Forward: y[pix,o] = alpha[o] * ( Cin*nvalid - 2 * sum_{valid taps,k} popc(x[pix_t,k] ^ w[o,t,k]) )
//
// Block = 128 threads = 128 consecutive output pixels; each thread keeps TO accumulators (one per
// output channel of the tile) in registers.  The TO*T*Cw weight words of the tile are staged once in
// shared memory and read with warp-broadcast (all lanes same address) vector LDS; activation words
// are read straight from global with KC*32-bit vector loads (consecutive lanes = consecutive pixels,
// so a warp-load covers 32*Cw*4 contiguous bytes).  POPC issues at 16 lanes/clk/SM, so this kernel is
// POPC-pipe bound, not HBM bound (DESIGN.md §4.2); padding bits are 0 in both operands.
// -------------------------------------------------------------------------------------------------
template <int KC> struct WordVec;
template <> struct WordVec<1> { using type = uint32_t; };
template <> struct WordVec<2> { using type = uint2; };
template <> struct WordVec<4> { using type = uint4; };

template <int KC>
__device__ __forceinline__ int xor_popc(const typename WordVec<KC>::type& a,
                                        const typename WordVec<KC>::type& b);
template <> __device__ __forceinline__ int xor_popc<1>(const uint32_t& a, const uint32_t& b) {
  return __popc(a ^ b);
}
template <> __device__ __forceinline__ int xor_popc<2>(const uint2& a, const uint2& b) {
  return __popc(a.x ^ b.x) + __popc(a.y ^ b.y);
}
template <> __device__ __forceinline__ int xor_popc<4>(const uint4& a, const uint4& b) {
  return __popc(a.x ^ b.x) + __popc(a.y ^ b.y) + __popc(a.z ^ b.z) + __popc(a.w ^ b.w);
}

template <int TO, int KC>
__global__ void __launch_bounds__(128)
binconv_fwd_xnor_kernel(const uint32_t* __restrict__ xs, const uint32_t* __restrict__ ws,
                        const float* __restrict__ alpha, float* __restrict__ y,
                        bdbnn_conv_shape s, int32_t Cw, int64_t n_pix_out) {
  using V = typename WordVec<KC>::type;
  extern __shared__ __align__(16) uint32_t wsm[];  // [TO][T][Cw]
  const int T = s.kh * s.kw;
  const int o0 = blockIdx.y * TO;
  {
    const int n = TO * T * Cw;
    const uint32_t* src = ws + int64_t(o0) * T * Cw;
    for (int i = threadIdx.x; i < n; i += blockDim.x) wsm[i] = src[i];
  }
  __syncthreads();

  const int64_t pix = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const bool live = pix < n_pix_out;
  int wo = 0, ho = 0, n = 0;
  if (live) {
    wo = int(pix % s.Wo);
    const int64_t q = pix / s.Wo;
    ho = int(q % s.Ho);
    n = int(q / s.Ho);
  }

  int acc[TO];
#pragma unroll
  for (int o = 0; o < TO; ++o) acc[o] = 0;
  int nvalid = 0;

  for (int r = 0; r < s.kh; ++r) {
    const int h = ho * s.stride + r - s.pad;
    for (int q = 0; q < s.kw; ++q) {
      const int w = wo * s.stride + q - s.pad;
      const bool valid = live && h >= 0 && h < s.H && w >= 0 && w < s.W;
      if (!valid) continue;
      ++nvalid;
      const int t = r * s.kw + q;
      const V* xp = reinterpret_cast<const V*>(xs + ((int64_t(n) * s.H + h) * s.W + w) * Cw);
      for (int k = 0; k < Cw / KC; ++k) {
        const V xv = __ldg(xp + k);
#pragma unroll
        for (int o = 0; o < TO; ++o) {
          const V wv = *reinterpret_cast<const V*>(wsm + (o * T + t) * Cw + k * KC);
          acc[o] += xor_popc<KC>(xv, wv);
        }
      }
    }
  }
  if (!live) return;
  float* yp = y + pix * s.Cout + o0;
  const int base = s.Cin * nvalid;
  if constexpr (TO % 4 == 0) {
#pragma unroll
    for (int o = 0; o < TO; o += 4) {
      const float4 a = *reinterpret_cast<const float4*>(alpha + o0 + o);
      float4 v;
      v.x = a.x * float(base - 2 * acc[o + 0]);
      v.y = a.y * float(base - 2 * acc[o + 1]);
      v.z = a.z * float(base - 2 * acc[o + 2]);
      v.w = a.w * float(base - 2 * acc[o + 3]);
      *reinterpret_cast<float4*>(yp + o) = v;
    }
  } else {
#pragma unroll
    for (int o = 0; o < TO; ++o) yp[o] = alpha[o0 + o] * float(base - 2 * acc[o]);
  }
}

template <int TO>
static int launch_fwd_xnor(const uint32_t* xs, const uint32_t* ws, const float* alpha, float* y,
                           const bdbnn_conv_shape& s, cudaStream_t st) {
  const int32_t Cw = (s.Cin + 31) / 32;
  const int T = s.kh * s.kw;
  const int64_t n_pix = int64_t(s.N) * s.Ho * s.Wo;
  const size_t smem = size_t(TO) * T * Cw * 4;
  if (smem > 200 * 1024) {
    set_error("binconv_fwd_xnor: weight tile needs %zu B of shared memory", smem);
    return BDBNN_ERR_UNSUPPORTED;
  }
  dim3 grid(unsigned((n_pix + 127) / 128), unsigned(s.Cout / TO));
  auto go = [&](auto kern) -> int {
    if (smem > 48 * 1024)
      BDBNN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    kern<<<grid, 128, smem, st>>>(xs, ws, alpha, y, s, Cw, n_pix);
    return check_launch("binconv_fwd_xnor_kernel");
  };
  if (Cw % 4 == 0) return go(binconv_fwd_xnor_kernel<TO, 4>);
  if (Cw % 2 == 0) return go(binconv_fwd_xnor_kernel<TO, 2>);
  return go(binconv_fwd_xnor_kernel<TO, 1>);
}

// -------------------------------------------------------------------------------------------------
// Generic data gradient (any kernel size / stride / channel count).  One thread per (input pixel,
// channel); lanes of a warp share the pixel (when Cin >= 32) so gy / alpha / weight-word reads are
// warp-broadcast.  Correctness baseline and fallback for shapes the tensor-core path does not take.
// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
binconv_dgrad_generic_kernel(const float* __restrict__ gy, const uint32_t* __restrict__ ws,
                             const float* __restrict__ alpha, const uint32_t* __restrict__ mask_bits,
                             float* __restrict__ gx, bdbnn_conv_shape s, int32_t Cw, int64_t total) {
  const int64_t idx = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  const int c = int(idx % s.Cin);
  const int64_t pix = idx / s.Cin;
  const int w = int(pix % s.W);
  const int64_t q = pix / s.W;
  const int h = int(q % s.H);
  const int n = int(q / s.H);
  const int kword = c >> 5, kbit = c & 31;
  const bool pass = (mask_bits[pix * Cw + kword] >> kbit) & 1u;
  float acc = 0.f;
  if (pass) {
    const int T = s.kh * s.kw;
    for (int r = 0; r < s.kh; ++r) {
      const int hh = h + s.pad - r;
      if (hh < 0 || hh % s.stride != 0) continue;
      const int ho = hh / s.stride;
      if (ho >= s.Ho) continue;
      for (int qq = 0; qq < s.kw; ++qq) {
        const int ww = w + s.pad - qq;
        if (ww < 0 || ww % s.stride != 0) continue;
        const int wo = ww / s.stride;
        if (wo >= s.Wo) continue;
        const int t = r * s.kw + qq;
        const float* gyp = gy + ((int64_t(n) * s.Ho + ho) * s.Wo + wo) * s.Cout;
        const uint32_t* wp = ws + int64_t(t) * Cw + kword;
        for (int o = 0; o < s.Cout; ++o) {
          const float g = __ldg(gyp + o) * __ldg(alpha + o);
          const uint32_t bit = (__ldg(wp + int64_t(o) * T * Cw) >> kbit) & 1u;
          acc += bit ? g : -g;
        }
      }
    }
  }
  gx[idx] = acc;
}

// -------------------------------------------------------------------------------------------------
// Generic weight gradient.  One thread per weight element (o, t, c) (c fastest so lanes share the
// gy scalar and the activation word), grid.y splits the output pixels; partial sums are combined with
// fp32 atomics into the zero-initialised gW (summation order is therefore not fixed run to run).
// -------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
binconv_wgrad_generic_kernel(const float* __restrict__ gy, const uint32_t* __restrict__ xs,
                             const uint32_t* __restrict__ wmask, float* __restrict__ gW,
                             bdbnn_conv_shape s, int32_t Cw, int64_t n_pix_out, int64_t chunk) {
  const int T = s.kh * s.kw;
  const int64_t id = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t n_w = int64_t(s.Cout) * T * s.Cin;
  if (id >= n_w) return;
  const int c = int(id % s.Cin);
  const int64_t ot = id / s.Cin;
  const int t = int(ot % T);
  const int o = int(ot / T);
  const int r = t / s.kw, qq = t - r * s.kw;
  const int64_t e = (int64_t(o) * s.Cin + c) * T + t;  // OIHW flat index
  if (!((wmask[e >> 5] >> (e & 31)) & 1u)) return;      // STE: gradient blocked where |W| > 1
  const int kword = c >> 5, kbit = c & 31;

  const int64_t m0 = int64_t(blockIdx.y) * chunk;
  int64_t m1 = m0 + chunk;
  if (m1 > n_pix_out) m1 = n_pix_out;
  float acc = 0.f;
  for (int64_t m = m0; m < m1; ++m) {
    const int wo = int(m % s.Wo);
    const int64_t q = m / s.Wo;
    const int ho = int(q % s.Ho);
    const int n = int(q / s.Ho);
    const int h = ho * s.stride + r - s.pad;
    const int w = wo * s.stride + qq - s.pad;
    if (h < 0 || h >= s.H || w < 0 || w >= s.W) continue;
    const float g = __ldg(gy + m * s.Cout + o);
    const uint32_t bit = (__ldg(xs + ((int64_t(n) * s.H + h) * s.W + w) * Cw + kword) >> kbit) & 1u;
    acc += bit ? g : -g;
  }
  atomicAdd(gW + e, acc);
}

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_binconv_fwd_xnor(const uint32_t* sign_bits, const uint32_t* wsign_bits,
                                      const float* alpha, float* y, const bdbnn_conv_shape* s,
                                      void* stream) {
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(sign_bits && wsign_bits && alpha && y, "binconv_fwd_xnor: NULL pointer");
  cudaStream_t st = cudaStream_t(stream);
  if (s->Cout % 64 == 0) return launch_fwd_xnor<64>(sign_bits, wsign_bits, alpha, y, *s, st);
  if (s->Cout % 32 == 0) return launch_fwd_xnor<32>(sign_bits, wsign_bits, alpha, y, *s, st);
  if (s->Cout % 16 == 0) return launch_fwd_xnor<16>(sign_bits, wsign_bits, alpha, y, *s, st);
  if (s->Cout % 8 == 0) return launch_fwd_xnor<8>(sign_bits, wsign_bits, alpha, y, *s, st);
  return launch_fwd_xnor<1>(sign_bits, wsign_bits, alpha, y, *s, st);
}

extern "C" int bdbnn_binconv_dgrad(const float* gy, const uint32_t* wsign_bits, const float* alpha,
                                   const uint32_t* mask_bits, float* gx, const bdbnn_conv_shape* s,
                                   void* stream) {
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(gy && wsign_bits && alpha && mask_bits && gx, "binconv_dgrad: NULL pointer");
  const int32_t Cw = (s->Cin + 31) / 32;
  const int64_t total = int64_t(s->N) * s->H * s->W * s->Cin;
  const int64_t blocks = (total + 255) / 256;
  BDBNN_REQUIRE(blocks < (int64_t(1) << 31), "binconv_dgrad: tensor too large");
  binconv_dgrad_generic_kernel<<<unsigned(blocks), 256, 0, cudaStream_t(stream)>>>(
      gy, wsign_bits, alpha, mask_bits, gx, *s, Cw, total);
  return check_launch("binconv_dgrad_generic_kernel");
}

extern "C" int bdbnn_binconv_wgrad(const float* gy, const uint32_t* sign_bits,
                                   const uint32_t* wmask_bits, float* gW,
                                   const bdbnn_conv_shape* s, void* stream) {
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(gy && sign_bits && wmask_bits && gW, "binconv_wgrad: NULL pointer");
  const int32_t Cw = (s->Cin + 31) / 32;
  const int T = s->kh * s->kw;
  const int64_t n_w = int64_t(s->Cout) * T * s->Cin;
  const int64_t n_pix_out = int64_t(s->N) * s->Ho * s->Wo;
  BDBNN_CUDA(cudaMemsetAsync(gW, 0, size_t(n_w) * sizeof(float), cudaStream_t(stream)));
  const int64_t bx = (n_w + 255) / 256;
  // Enough pixel chunks to fill the machine a few times over, at least 64 pixels per chunk.
  int64_t by = (int64_t(num_sms()) * 16 + bx - 1) / bx;
  if (by < 1) by = 1;
  int64_t chunk = (n_pix_out + by - 1) / by;
  if (chunk < 64) chunk = 64;
  by = (n_pix_out + chunk - 1) / chunk;
  if (by > 65535) { by = 65535; chunk = (n_pix_out + by - 1) / by; }
  dim3 grid{unsigned(bx), unsigned(by)};
  binconv_wgrad_generic_kernel<<<grid, 256, 0, cudaStream_t(stream)>>>(gy, sign_bits, wmask_bits, gW,
                                                                      *s, Cw, n_pix_out, chunk);
  return check_launch("binconv_wgrad_generic_kernel");
}
