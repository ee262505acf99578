// Sign / bit-pack kernels (HBM-streaming).  See include/bdbnn.h for the contracts.
//
//   act_pack    : fp32 NHWC activations -> sign bits + STE mask bits (+ optional +-1 bf16 copy)
//   weight_pack : fp32 OIHW weights     -> alpha, sign bits [o][tap][cw], STE mask bits, bf16 operands
//   grad_pack   : fp32 NHWC grad        -> bf16(gy * gscale[o])
//
// Spec (DESIGN.md §2): sign(x) := (x >= 0) ? +1 : -1 ; STE mask := |x| <= 1.
#include "common.cuh"

namespace bdbnn {

constexpr int kPackUnroll = 8;

// One warp produces kPackUnroll words per iteration: lane j of the warp owns channel 32k+j of the
// word; __ballot_sync assembles the word.  Loads are issued kPackUnroll-deep before any ballot so
// each thread keeps 8 independent 4-byte requests in flight (enough bytes in flight to stream HBM at
// full occupancy; every warp-load is one 128-byte line).
__global__ void __launch_bounds__(256)
act_pack_kernel(const float* __restrict__ x, int64_t n_words, int32_t C, int32_t Cw,
                uint32_t* __restrict__ sign_bits, uint32_t* __restrict__ mask_bits,
                uint16_t* __restrict__ xb, uint16_t one16) {
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = (int64_t(gridDim.x) * blockDim.x) >> 5;
  const bool flat = (C & 31) == 0;

  for (int64_t w0 = warp_global * kPackUnroll; w0 < n_words; w0 += n_warps * kPackUnroll) {
    float v[kPackUnroll];
    int64_t idx[kPackUnroll];
    bool ok[kPackUnroll];
#pragma unroll
    for (int j = 0; j < kPackUnroll; ++j) {
      const int64_t wi = w0 + j;
      if (flat) {
        idx[j] = wi * 32 + lane;
        ok[j] = wi < n_words;
      } else {
        const int64_t p = wi / Cw;
        const int k = int(wi - p * Cw);
        const int c = k * 32 + lane;
        idx[j] = p * C + c;
        ok[j] = (wi < n_words) && (c < C);
      }
      v[j] = ok[j] ? __ldcs(x + idx[j]) : __int_as_float(0x7fc00000);  // NaN -> both bits 0
    }
    uint32_t my_sign = 0, my_mask = 0;
#pragma unroll
    for (int j = 0; j < kPackUnroll; ++j) {
      const uint32_t sb = __ballot_sync(0xffffffffu, v[j] >= 0.0f);
      const uint32_t mb = __ballot_sync(0xffffffffu, fabsf(v[j]) <= 1.0f);
      if (lane == j) { my_sign = sb; my_mask = mb; }
      if (xb != nullptr && ok[j]) xb[idx[j]] = (v[j] >= 0.0f) ? one16 : uint16_t(one16 | 0x8000u);
    }
    if (lane < kPackUnroll && (w0 + lane) < n_words) {
      sign_bits[w0 + lane] = my_sign;
      mask_bits[w0 + lane] = my_mask;
    }
  }
}

// One block per output channel (o).
__device__ __forceinline__ void
weight_pack_body(const float* __restrict__ W, int32_t Cout, int32_t Cin, int32_t T, int32_t Cw,
                 float* __restrict__ alpha, uint32_t* __restrict__ wsign,
                 uint16_t* __restrict__ wf, uint16_t* __restrict__ wt, uint8_t* __restrict__ wf8,
                 float* __restrict__ gscale, float* __restrict__ inv_gscale, uint16_t one16,
                 uint32_t* __restrict__ wmask_inline, int wt_inline, const int o) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nwarps = blockDim.x >> 5;
  const int per = Cin * T;
  const float* Wo = W + int64_t(o) * per;

  __shared__ float red[32];
  __shared__ float s_alpha;
  float a = 0.f;
  for (int i = tid; i < per; i += blockDim.x) a += fabsf(Wo[i]);
  a = warp_sum(a);
  if (lane == 0) red[warp] = a;
  __syncthreads();
  if (warp == 0) {
    float t = (lane < nwarps) ? red[lane] : 0.f;
    t = warp_sum(t);
    if (lane == 0) {
      const float al = t / float(per);
      s_alpha = al;
      alpha[o] = al;
      const float g = (al > 0.f) ? al : 1.f;
      if (gscale) gscale[o] = g;
      if (inv_gscale) inv_gscale[o] = 1.0f / g;
    }
  }
  __syncthreads();
  const bool live = s_alpha > 0.f;

  // sign words [o][t][k]
  for (int w = warp; w < T * Cw; w += nwarps) {
    const int t = w / Cw, k = w - t * Cw;
    const int c = k * 32 + lane;
    const bool ok = c < Cin;
    const float v = ok ? Wo[c * T + t] : -1.0f;
    const uint32_t sb = __ballot_sync(0xffffffffu, ok && (v >= 0.0f));
    if (lane == 0) wsign[(int64_t(o) * T + t) * Cw + k] = sb;
  }
  // bf16 operands for the tensor-core path
  if (wf != nullptr || wt != nullptr || wf8 != nullptr) {
    for (int i = tid; i < per; i += blockDim.x) {
      const int t = i / Cin, c = i - t * Cin;  // (t, c) with c fastest: coalesced wf writes
      const float v = Wo[c * T + t];
      const uint16_t sg = (v >= 0.0f) ? one16 : uint16_t(one16 | 0x8000u);
      if (wf) wf[(int64_t(o) * T + t) * Cin + c] = sg;
      if (wf8) wf8[(int64_t(o) * T + t) * Cin + c] = (v >= 0.0f) ? uint8_t(0x38) : uint8_t(0xB8);  // e4m3 +-1
      if (wt && wt_inline) wt[(int64_t(c) * T + (T - 1 - t)) * Cout + o] = live ? sg : uint16_t(0);
    }
  }
  // |W| <= 1 bits of this filter's slice of the flat OIHW mask (when the slice is word-aligned)
  if (wmask_inline != nullptr) {
    uint32_t* mo = wmask_inline + (int64_t(o) * per >> 5);
    for (int w = warp; w < (per >> 5); w += nwarps) {
      const uint32_t mb = __ballot_sync(0xffffffffu, fabsf(Wo[w * 32 + lane]) <= 1.0f);
      if (lane == 0) mo[w] = mb;
    }
  }
}

__global__ void __launch_bounds__(256)
weight_pack_kernel(const float* __restrict__ W, int32_t Cout, int32_t Cin, int32_t T, int32_t Cw,
                   float* __restrict__ alpha, uint32_t* __restrict__ wsign,
                   uint16_t* __restrict__ wf, uint16_t* __restrict__ wt, uint8_t* __restrict__ wf8,
                   float* __restrict__ gscale, float* __restrict__ inv_gscale, uint16_t one16,
                   uint32_t* __restrict__ wmask_inline, int wt_inline) {
  weight_pack_body(W, Cout, Cin, T, Cw, alpha, wsign, wf, wt, wf8, gscale, inv_gscale, one16, wmask_inline, wt_inline,
                   int(blockIdx.x));
}

// dgrad operand wt[c][T-1-t][o] = alpha[o] > 0 ? sign(W[o][c][t]) : 0 as a 32x32 tile transpose: reads run along
// (c,t) for one filter, writes run along o (the per-filter kernel's scattered 2-byte stores cost 50 us at
// 512x512x9).  grid = (ceil(per/32), ceil(Cout/32)), block = (32, 8).
__device__ __forceinline__ void
weight_wt_body(const float* __restrict__ W, const float* __restrict__ alpha, int32_t Cout, int32_t Cin, int32_t T,
               uint16_t* __restrict__ wt, uint16_t one16, const int bx, const int by) {
  __shared__ uint16_t tile[32][33];
  const int per = Cin * T;
  const int i0 = bx * 32, o0 = by * 32;
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int o = o0 + r, i = i0 + threadIdx.x;
    uint16_t sg = 0;
    if (o < Cout && i < per) {
      const float v = W[int64_t(o) * per + i];
      sg = __ldg(alpha + o) > 0.f ? ((v >= 0.0f) ? one16 : uint16_t(one16 | 0x8000u)) : uint16_t(0);
    }
    tile[r][threadIdx.x] = sg;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += 8) {
    const int i = i0 + r, o = o0 + threadIdx.x;
    if (i < per && o < Cout) {
      const int c = i / T, t = i - c * T;
      wt[(int64_t(c) * T + (T - 1 - t)) * Cout + o] = tile[threadIdx.x][r];
    }
  }
}

__global__ void __launch_bounds__(256)
weight_wt_kernel(const float* __restrict__ W, const float* __restrict__ alpha, int32_t Cout, int32_t Cin, int32_t T,
                 uint16_t* __restrict__ wt, uint16_t one16) {
  weight_wt_body(W, alpha, Cout, Cin, T, wt, one16, int(blockIdx.x), int(blockIdx.y));
}

// ---- all binary convs of a network in two launches (SURVEY.md §7.3: one multi-tensor pass over the weights) ----
// 16 + 16 per-layer launches of a ResNet-18 step each fill a fraction of the GPU (64..512 blocks of a few KB);
// batched, the same work is one grid of sum(Cout) filter blocks plus one grid of transpose tiles.
constexpr int kPackMaxLayers = 32;
struct WPackTable {
  const float* W[kPackMaxLayers];
  float* alpha[kPackMaxLayers];
  uint32_t* wsign[kPackMaxLayers];
  uint32_t* wmask[kPackMaxLayers];
  uint16_t* wf[kPackMaxLayers];
  uint16_t* wt[kPackMaxLayers];
  uint8_t* wf8[kPackMaxLayers];
  float* gscale[kPackMaxLayers];
  float* inv_gscale[kPackMaxLayers];
  int32_t Cout[kPackMaxLayers], Cin[kPackMaxLayers], T[kPackMaxLayers];
  int32_t blk0[kPackMaxLayers + 1];    // first filter block of layer l (prefix sums of Cout)
  int32_t tile0[kPackMaxLayers + 1];   // first transpose tile of layer l
  int32_t n;
};

__device__ __forceinline__ int wpack_find(const int32_t* start, int n, int b) {
  int l = 0;
  while (l + 1 < n && b >= start[l + 1]) ++l;
  return l;
}

__global__ void __launch_bounds__(256)
weight_pack_multi_kernel(const __grid_constant__ WPackTable tab, uint16_t one16) {
  const int l = wpack_find(tab.blk0, tab.n, int(blockIdx.x));
  const int Cin = tab.Cin[l];
  weight_pack_body(tab.W[l], tab.Cout[l], Cin, tab.T[l], (Cin + 31) / 32, tab.alpha[l], tab.wsign[l], tab.wf[l],
                   nullptr, tab.wf8[l], tab.gscale[l], tab.inv_gscale[l], one16, tab.wmask[l], 0,
                   int(blockIdx.x) - tab.blk0[l]);
}

__global__ void __launch_bounds__(256)
weight_wt_multi_kernel(const __grid_constant__ WPackTable tab, uint16_t one16) {
  const int l = wpack_find(tab.tile0, tab.n, int(blockIdx.x));
  const int t = int(blockIdx.x) - tab.tile0[l];
  const int tiles_x = (tab.Cin[l] * tab.T[l] + 31) / 32;
  weight_wt_body(tab.W[l], tab.alpha[l], tab.Cout[l], tab.Cin[l], tab.T[l], tab.wt[l], one16, t % tiles_x, t / tiles_x);
}

// ---- sign words of all binary convs of a loaded 1-bit model -> their forward operands, one launch ----
// One block per filter (blk0 as in WPackTable).  Element i = t*Cin + c of filter o reads bit c%32 of word
// [o][t][c/32]: the 32 lanes of a warp share one word, and the writes of a block run along the filter's row.
// Per layer exactly one of wf (16-bit, one16 / one16|0x8000) or wf8 (e4m3 0x38 / 0xB8) is non-NULL.
struct WUnpackTable {
  const uint32_t* wsign[kPackMaxLayers];
  uint16_t* wf[kPackMaxLayers];
  uint8_t* wf8[kPackMaxLayers];
  int32_t Cin[kPackMaxLayers], T[kPackMaxLayers];
  int32_t blk0[kPackMaxLayers + 1];
  int32_t n;
};

__global__ void __launch_bounds__(256)
weight_unpack_multi_kernel(const __grid_constant__ WUnpackTable tab, uint16_t one16) {
  const int l = wpack_find(tab.blk0, tab.n, int(blockIdx.x));
  const int o = int(blockIdx.x) - tab.blk0[l];
  const int Cin = tab.Cin[l], T = tab.T[l], Cw = (Cin + 31) / 32, per = Cin * T;
  const uint32_t* ws = tab.wsign[l] + int64_t(o) * T * Cw;
  uint16_t* wf = tab.wf[l];
  uint8_t* wf8 = tab.wf8[l];
  for (int i = threadIdx.x; i < per; i += blockDim.x) {
    const int t = i / Cin, c = i - t * Cin;
    const bool pos = (__ldg(ws + t * Cw + (c >> 5)) >> (c & 31)) & 1u;
    if (wf8) wf8[int64_t(o) * per + i] = pos ? uint8_t(0x38) : uint8_t(0xB8);
    else wf[int64_t(o) * per + i] = pos ? one16 : uint16_t(one16 | 0x8000u);
  }
}

// sign bits -> fp8 e4m3 +-1 bytes (0x38 / 0xB8), C % 32 == 0: word w expands to 32 consecutive bytes.
__global__ void __launch_bounds__(256)
bits_to_fp8_kernel(const uint32_t* __restrict__ bits, int64_t n_words, uint4* __restrict__ out) {
  // one thread per 16 output bytes (half a word is two threads)
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n_words * 2;
       i += int64_t(gridDim.x) * blockDim.x) {
    const uint32_t w = __ldg(bits + (i >> 1)) >> ((i & 1) * 16);
    uint32_t o[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const uint32_t nib = (w >> (4 * q)) & 0xfu;
      // byte j = 0x38 | (bit ? 0 : 0x80)
      o[q] = 0x38383838u | (((nib & 1u) ? 0u : 0x80u) | ((nib & 2u) ? 0u : 0x8000u) | ((nib & 4u) ? 0u : 0x800000u) |
                            ((nib & 8u) ? 0u : 0x80000000u));
    }
    out[i] = make_uint4(o[0], o[1], o[2], o[3]);
  }
}

// |W| <= 1 bits over the flat OIHW tensor.
__global__ void __launch_bounds__(256)
flat_mask_kernel(const float* __restrict__ W, int64_t n, uint32_t* __restrict__ mask_bits) {
  const int lane = threadIdx.x & 31;
  const int64_t warp_global = (int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5;
  const int64_t n_warps = (int64_t(gridDim.x) * blockDim.x) >> 5;
  const int64_t n_words = (n + 31) / 32;
  for (int64_t wi = warp_global; wi < n_words; wi += n_warps) {
    const int64_t e = wi * 32 + lane;
    const bool ok = e < n;
    const float v = ok ? W[e] : 2.0f;
    const uint32_t mb = __ballot_sync(0xffffffffu, ok && fabsf(v) <= 1.0f);
    if (lane == 0) mask_bits[wi] = mb;
  }
}

__device__ __forceinline__ uint32_t pack_bf16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

// ---- gradient operand packing -----------------------------------------------------------------------
// v = gy[i] * gscale[i % Cout]
//   MODE 1 (BF16)   : out[i] = bf16_rn(v)
//   MODE 2 (BF16X2) : out[pix*2C + o] = hi = bf16_rn(v), out[pix*2C + C + o] = bf16_rn(v - hi)
//   MODE 3 (FP16S)  : out[i] = fp16_rn(v * 2^e), e = 13 - floor(log2(amax)), amax = max|v| of this call
__device__ __forceinline__ float bf16_round(float v) {
  return __uint_as_float(pack_bf16x2(0.f, v) & 0xffff0000u);
}
__device__ __forceinline__ uint32_t pack_f16x2(float lo, float hi) {
  uint32_t r;
  asm("cvt.rn.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(hi), "f"(lo));
  return r;
}

__global__ void __launch_bounds__(256)
grad_amax_kernel(const float* __restrict__ gy, const float* __restrict__ gscale, int64_t n, int32_t Cout,
                 uint32_t* __restrict__ amax_bits) {
  const int64_t tid = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t nthreads = int64_t(gridDim.x) * blockDim.x;
  float m = 0.f;
  if ((Cout & 3) == 0) {
    const int64_t n4 = n >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(gy);
    for (int64_t i = tid; i < n4; i += nthreads) {
      const float4 v = __ldg(g4 + i);                    // keep in L2 for the pack pass that follows
      const int o = int((i * 4) % Cout);
      const float4 s = *reinterpret_cast<const float4*>(gscale + o);
      m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x * s.x), fabsf(v.y * s.y)), fmaxf(fabsf(v.z * s.z), fabsf(v.w * s.w))));
    }
  } else {
    for (int64_t i = tid; i < n; i += nthreads) m = fmaxf(m, fabsf(gy[i] * gscale[i % Cout]));
  }
  // NaN never wins fmaxf; an Inf does and yields scale 2^-115 (result stays Inf like the reference's)
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0 && m > 0.f) atomicMax(amax_bits, __float_as_uint(m));
}

template <int MODE>
__global__ void __launch_bounds__(256)
grad_pack_kernel(const float* __restrict__ gy, const float* __restrict__ gscale, int64_t n,
                 int32_t Cout, const uint32_t* __restrict__ amax_bits, uint16_t* __restrict__ out) {
  const int64_t tid = int64_t(blockIdx.x) * blockDim.x + threadIdx.x;
  const int64_t nthreads = int64_t(gridDim.x) * blockDim.x;
  constexpr int HALVES = MODE == 2 ? 2 : 1;
  const float up = MODE == 3 ? amax_pow2_scale(*amax_bits, false) : 1.0f;
  if ((Cout & 3) == 0) {
    const int64_t n4 = n >> 2;
    const float4* g4 = reinterpret_cast<const float4*>(gy);
    for (int64_t i = tid; i < n4; i += nthreads) {
      const float4 v = __ldcs(g4 + i);
      const int64_t e = i * 4;
      const int64_t pix = e / Cout;
      const int o = int(e - pix * Cout);
      const float4 s = *reinterpret_cast<const float4*>(gscale + o);
      const float a0 = v.x * s.x * up, a1 = v.y * s.y * up, a2 = v.z * s.z * up, a3 = v.w * s.w * up;
      uint2 r;
      if (MODE == 3) {
        r.x = pack_f16x2(a0, a1);
        r.y = pack_f16x2(a2, a3);
      } else {
        r.x = pack_bf16x2(a0, a1);
        r.y = pack_bf16x2(a2, a3);
      }
      uint16_t* dst = out + pix * (int64_t(HALVES) * Cout) + o;
      *reinterpret_cast<uint2*>(dst) = r;
      if (MODE == 2) {
        uint2 l;
        l.x = pack_bf16x2(a0 - bf16_round(a0), a1 - bf16_round(a1));
        l.y = pack_bf16x2(a2 - bf16_round(a2), a3 - bf16_round(a3));
        *reinterpret_cast<uint2*>(dst + Cout) = l;
      }
    }
  } else {
    for (int64_t i = tid; i < n; i += nthreads) {
      const int64_t pix = i / Cout;
      const int o = int(i - pix * Cout);
      const float v = gy[i] * gscale[o] * up;
      uint16_t* dst = out + pix * (int64_t(HALVES) * Cout) + o;
      if (MODE == 3) {
        *dst = uint16_t(pack_f16x2(v, 0.f) & 0xffffu);
      } else {
        *dst = uint16_t(pack_bf16x2(v, 0.f) & 0xffffu);
        if (MODE == 2) dst[Cout] = uint16_t(pack_bf16x2(v - bf16_round(v), 0.f) & 0xffffu);
      }
    }
  }
}

}  // namespace bdbnn

using namespace bdbnn;

static inline uint16_t one_bits(int fmt) { return fmt == BDBNN_FMT_FP16 ? uint16_t(0x3C00) : uint16_t(0x3F80); }

extern "C" int bdbnn_act_pack(const float* x, int64_t n_pix, int32_t C, uint32_t* sign_bits,
                              uint32_t* mask_bits, uint16_t* xb_bf16, int32_t fmt, void* stream) {
  BDBNN_REQUIRE(fmt == BDBNN_FMT_FP16 || fmt == BDBNN_FMT_BF16, "act_pack: bad operand format");
  BDBNN_REQUIRE(n_pix >= 0 && C > 0, "act_pack: bad n_pix/C");
  if (n_pix == 0) return BDBNN_OK;
  BDBNN_REQUIRE(x && sign_bits && mask_bits, "act_pack: NULL pointer");
  const int32_t Cw = (C + 31) / 32;
  const int64_t n_words = n_pix * Cw;
  const int threads = 256;
  const int64_t warps_needed = (n_words + kPackUnroll - 1) / kPackUnroll;
  int64_t blocks = (warps_needed * 32 + threads - 1) / threads;
  const int64_t cap = int64_t(num_sms()) * 8 * 4;  // a few waves of full-occupancy blocks
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  act_pack_kernel<<<unsigned(blocks), threads, 0, cudaStream_t(stream)>>>(
      x, n_words, C, Cw, sign_bits, mask_bits, xb_bf16, one_bits(fmt));
  return check_launch("act_pack_kernel");
}

extern "C" int bdbnn_weight_pack(const float* W, int32_t Cout, int32_t Cin, int32_t kh, int32_t kw,
                                 float* alpha, uint32_t* wsign_bits, uint32_t* wmask_bits,
                                 uint16_t* wf_bf16, uint16_t* wt_bf16, uint8_t* wf_fp8, float* gscale,
                                 float* inv_gscale, int32_t fmt, void* stream) {
  BDBNN_REQUIRE(fmt == BDBNN_FMT_FP16 || fmt == BDBNN_FMT_BF16, "weight_pack: bad operand format");
  BDBNN_REQUIRE(Cout > 0 && Cin > 0 && kh > 0 && kw > 0, "weight_pack: bad dims");
  BDBNN_REQUIRE(W && alpha && wsign_bits && wmask_bits, "weight_pack: NULL pointer");
  const int32_t T = kh * kw, Cw = (Cin + 31) / 32;
  const int per = Cin * T;
  const bool mask_inline = (per & 31) == 0;          // each filter's mask slice is whole words
  const bool wt_tiled = wt_bf16 != nullptr && int64_t(Cout) * per >= 32768;   // small layers: one launch less
  weight_pack_kernel<<<Cout, 256, 0, cudaStream_t(stream)>>>(W, Cout, Cin, T, Cw, alpha, wsign_bits,
                                                            wf_bf16, wt_bf16, wf_fp8, gscale, inv_gscale,
                                                            one_bits(fmt), mask_inline ? wmask_bits : nullptr,
                                                            wt_tiled ? 0 : 1);
  int rc = check_launch("weight_pack_kernel");
  if (rc) return rc;
  if (wt_tiled) {
    dim3 grid(unsigned((per + 31) / 32), unsigned((Cout + 31) / 32));
    weight_wt_kernel<<<grid, dim3(32, 8), 0, cudaStream_t(stream)>>>(W, alpha, Cout, Cin, T, wt_bf16, one_bits(fmt));
    rc = check_launch("weight_wt_kernel");
    if (rc) return rc;
  }
  if (mask_inline) return BDBNN_OK;
  const int64_t n = int64_t(Cout) * Cin * T;
  const int64_t n_words = (n + 31) / 32;
  int64_t blocks = (n_words * 32 + 255) / 256;
  if (blocks > 1024) blocks = 1024;
  flat_mask_kernel<<<unsigned(blocks), 256, 0, cudaStream_t(stream)>>>(W, n, wmask_bits);
  return check_launch("flat_mask_kernel");
}

extern "C" int bdbnn_weight_pack_multi(int32_t count, const float* const* W_host, const int32_t* Cout_host,
                                       const int32_t* Cin_host, const int32_t* taps_host, float* const* alpha_host,
                                       uint32_t* const* wsign_host, uint32_t* const* wmask_host,
                                       uint16_t* const* wf_host, uint16_t* const* wt_host, uint8_t* const* wf8_host,
                                       float* const* gscale_host, float* const* inv_gscale_host, int32_t fmt,
                                       void* stream) {
  BDBNN_REQUIRE(fmt == BDBNN_FMT_FP16 || fmt == BDBNN_FMT_BF16, "weight_pack_multi: bad operand format");
  BDBNN_REQUIRE(count >= 0, "weight_pack_multi: bad count");
  BDBNN_REQUIRE(count == 0 || (W_host && Cout_host && Cin_host && taps_host && alpha_host && wsign_host && wmask_host &&
                               wf_host && wt_host && wf8_host && gscale_host && inv_gscale_host),
                "weight_pack_multi: NULL table");
  cudaStream_t st = cudaStream_t(stream);
  for (int off = 0; off < count; off += kPackMaxLayers) {
    const int cnt = count - off < kPackMaxLayers ? count - off : kPackMaxLayers;
    WPackTable tab;
    memset(&tab, 0, sizeof(tab));
    tab.n = cnt;
    int blocks = 0, tiles = 0;
    for (int i = 0; i < cnt; ++i) {
      const int l = off + i;
      const int per = Cin_host[l] * taps_host[l];
      BDBNN_REQUIRE(W_host[l] && alpha_host[l] && wsign_host[l] && wmask_host[l] && wt_host[l] && gscale_host[l] &&
                        inv_gscale_host[l], "weight_pack_multi: NULL pointer in layer %d", l);
      BDBNN_REQUIRE(Cout_host[l] > 0 && per > 0 && (per & 31) == 0,
                    "weight_pack_multi: layer %d needs Cin*taps %% 32 == 0 (use bdbnn_weight_pack)", l);
      tab.W[i] = W_host[l]; tab.alpha[i] = alpha_host[l]; tab.wsign[i] = wsign_host[l]; tab.wmask[i] = wmask_host[l];
      tab.wf[i] = wf_host[l]; tab.wt[i] = wt_host[l]; tab.wf8[i] = wf8_host[l];
      tab.gscale[i] = gscale_host[l]; tab.inv_gscale[i] = inv_gscale_host[l];
      tab.Cout[i] = Cout_host[l]; tab.Cin[i] = Cin_host[l]; tab.T[i] = taps_host[l];
      tab.blk0[i] = blocks; tab.tile0[i] = tiles;
      blocks += Cout_host[l];
      tiles += ((per + 31) / 32) * ((Cout_host[l] + 31) / 32);
    }
    tab.blk0[cnt] = blocks; tab.tile0[cnt] = tiles;
    weight_pack_multi_kernel<<<unsigned(blocks), 256, 0, st>>>(tab, one_bits(fmt));
    int rc = check_launch("weight_pack_multi_kernel");
    if (rc) return rc;
    weight_wt_multi_kernel<<<unsigned(tiles), dim3(32, 8), 0, st>>>(tab, one_bits(fmt));
    rc = check_launch("weight_wt_multi_kernel");
    if (rc) return rc;
  }
  return BDBNN_OK;
}

extern "C" int bdbnn_weight_unpack_multi(int32_t count, const uint32_t* const* wsign_host, const int32_t* Cout_host,
                                         const int32_t* Cin_host, const int32_t* taps_host, uint16_t* const* wf_host,
                                         uint8_t* const* wf8_host, int32_t fmt, void* stream) {
  BDBNN_REQUIRE(fmt == BDBNN_FMT_FP16 || fmt == BDBNN_FMT_BF16, "weight_unpack_multi: bad operand format");
  BDBNN_REQUIRE(count >= 0, "weight_unpack_multi: bad count");
  BDBNN_REQUIRE(count == 0 || (wsign_host && Cout_host && Cin_host && taps_host && wf_host && wf8_host),
                "weight_unpack_multi: NULL table");
  cudaStream_t st = cudaStream_t(stream);
  for (int off = 0; off < count; off += kPackMaxLayers) {
    const int cnt = count - off < kPackMaxLayers ? count - off : kPackMaxLayers;
    WUnpackTable tab;
    memset(&tab, 0, sizeof(tab));
    tab.n = cnt;
    int blocks = 0;
    for (int i = 0; i < cnt; ++i) {
      const int l = off + i;
      BDBNN_REQUIRE(wsign_host[l] && ((wf_host[l] != nullptr) != (wf8_host[l] != nullptr)),
                    "weight_unpack_multi: layer %d needs its sign words and exactly one of wf / wf8", l);
      BDBNN_REQUIRE(Cout_host[l] > 0 && Cin_host[l] > 0 && taps_host[l] > 0 &&
                        int64_t(Cin_host[l]) * taps_host[l] <= INT32_MAX,
                    "weight_unpack_multi: bad dims in layer %d", l);
      BDBNN_REQUIRE(int64_t(blocks) + Cout_host[l] <= INT32_MAX, "weight_unpack_multi: too many filters");
      tab.wsign[i] = wsign_host[l]; tab.wf[i] = wf_host[l]; tab.wf8[i] = wf8_host[l];
      tab.Cin[i] = Cin_host[l]; tab.T[i] = taps_host[l];
      tab.blk0[i] = blocks;
      blocks += Cout_host[l];
    }
    tab.blk0[cnt] = blocks;
    weight_unpack_multi_kernel<<<unsigned(blocks), 256, 0, st>>>(tab, one_bits(fmt));
    const int rc = check_launch("weight_unpack_multi_kernel");
    if (rc) return rc;
  }
  return BDBNN_OK;
}

extern "C" int bdbnn_grad_pack(const float* gy, const float* gscale, int64_t n_pix, int32_t Cout,
                               int32_t mode, uint32_t* amax_bits, uint16_t* gys, void* stream) {
  BDBNN_REQUIRE(n_pix >= 0 && Cout > 0, "grad_pack: bad dims");
  BDBNN_REQUIRE(mode >= BDBNN_GRAD_BF16 && mode <= BDBNN_GRAD_FP16S, "grad_pack: bad mode %d", mode);
  if (n_pix == 0) return BDBNN_OK;
  BDBNN_REQUIRE(gy && gscale && gys, "grad_pack: NULL pointer");
  BDBNN_REQUIRE(mode != BDBNN_GRAD_FP16S || amax_bits, "grad_pack: FP16S mode needs the amax scratch word");
  cudaStream_t st = cudaStream_t(stream);
  const int64_t n = n_pix * Cout;
  int64_t blocks = ((n >> 2) + 255) / 256;
  const int64_t cap = int64_t(num_sms()) * 8 * 4;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  if (mode == BDBNN_GRAD_FP16S) {
    BDBNN_CUDA(cudaMemsetAsync(amax_bits, 0, sizeof(uint32_t), st));
    grad_amax_kernel<<<unsigned(blocks), 256, 0, st>>>(gy, gscale, n, Cout, amax_bits);
    int rc = check_launch("grad_amax_kernel");
    if (rc) return rc;
    grad_pack_kernel<3><<<unsigned(blocks), 256, 0, st>>>(gy, gscale, n, Cout, amax_bits, gys);
  } else if (mode == BDBNN_GRAD_BF16X2) {
    grad_pack_kernel<2><<<unsigned(blocks), 256, 0, st>>>(gy, gscale, n, Cout, nullptr, gys);
  } else {
    grad_pack_kernel<1><<<unsigned(blocks), 256, 0, st>>>(gy, gscale, n, Cout, nullptr, gys);
  }
  return check_launch("grad_pack_kernel");
}

extern "C" int bdbnn_bits_to_fp8(const uint32_t* sign_bits, int64_t n_pix, int32_t C, uint8_t* xb_fp8, void* stream) {
  BDBNN_REQUIRE(n_pix >= 0 && C > 0 && (C & 31) == 0, "bits_to_fp8: C must be a positive multiple of 32");
  if (n_pix == 0) return BDBNN_OK;
  BDBNN_REQUIRE(sign_bits && xb_fp8, "bits_to_fp8: NULL pointer");
  const int64_t n_words = n_pix * (C / 32);
  int64_t blocks = (n_words * 2 + 255) / 256;
  const int64_t cap = int64_t(num_sms()) * 8 * 4;
  if (blocks > cap) blocks = cap;
  bits_to_fp8_kernel<<<unsigned(blocks), 256, 0, cudaStream_t(stream)>>>(sign_bits, n_words,
                                                                         reinterpret_cast<uint4*>(xb_fp8));
  return check_launch("bits_to_fp8_kernel");
}

// ---- EDE backward factor (train.py:409-415, utils/utils.py:8-14) ------------------------------
// g[i] *= k * t * (1 - tanh(t * v[i])^2): the soft-sign derivative that replaces the hard-tanh STE
// indicator when the training loop has assigned .k/.t.  k and t stay on the device (1-element
// tensors written by the caller each epoch), so nothing here forces a host sync.
namespace bdbnn {
__global__ void __launch_bounds__(256)
ede_scale_kernel(float* __restrict__ g, const float* __restrict__ v, const float* __restrict__ kp,
                 const float* __restrict__ tp, int64_t n) {
  const float k = __ldg(kp), t = __ldg(tp), kt = k * t;
  const int64_t n4 = n >> 2;
  const int64_t stride = int64_t(gridDim.x) * blockDim.x;
  float4* g4 = reinterpret_cast<float4*>(g);
  const float4* v4 = reinterpret_cast<const float4*>(v);
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n4; i += stride) {
    float4 a = g4[i];
    const float4 b = __ldg(v4 + i);
    float th;
    th = tanhf(t * b.x); a.x *= kt * (1.0f - th * th);
    th = tanhf(t * b.y); a.y *= kt * (1.0f - th * th);
    th = tanhf(t * b.z); a.z *= kt * (1.0f - th * th);
    th = tanhf(t * b.w); a.w *= kt * (1.0f - th * th);
    g4[i] = a;
  }
  for (int64_t i = (n4 << 2) + int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
    const float th = tanhf(t * __ldg(v + i));
    g[i] *= kt * (1.0f - th * th);
  }
}
}  // namespace bdbnn

extern "C" int bdbnn_ede_scale(float* g, const float* v, const float* k, const float* t, int64_t n, void* stream) {
  BDBNN_REQUIRE(n >= 0, "ede_scale: negative n");
  if (n == 0) return BDBNN_OK;
  BDBNN_REQUIRE(g && v && k && t, "ede_scale: NULL pointer");
  BDBNN_REQUIRE(((uintptr_t(g) | uintptr_t(v)) & 15) == 0, "ede_scale: g and v must be 16-byte aligned");
  int64_t blocks = ((n >> 2) + 255) / 256;
  const int64_t cap = int64_t(bdbnn::num_sms()) * 8;
  if (blocks > cap) blocks = cap;
  if (blocks < 1) blocks = 1;
  bdbnn::ede_scale_kernel<<<unsigned(blocks), 256, 0, cudaStream_t(stream)>>>(g, v, k, t, n);
  return bdbnn::check_launch("ede_scale_kernel");
}
