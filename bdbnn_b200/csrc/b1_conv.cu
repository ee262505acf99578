// Binary 3x3 conv on the sm_90a binary tensor cores (DESIGN.md §4x):
//   wgmma.mma_async m64nNk256 .s32.b1.b1.and.popc  (SASS BGMMA), one instruction per 256 bits of K.
//
// Operands, both K-major with bit 1 = +1 and K index = tap * Cin + channel:
//   A = the activation sign bits of bdbnn_act_pack, [pixel][Cin/32] u32 (bit j of word k = channel 32k + j);
//   B = the stored sign words of bdbnn_weight_pack, [Cout][9][Cin/32] u32, read as they are.
// A tap outside the image loads zero bits.  The AND-popcount accumulator is turned into the +-1 dot product of the
// valid taps (padded taps contribute 0, DESIGN.md §2) by
//   sum_valid (2a-1)(2b-1) = 4 sum(a & b) - 2 sum_valid a - 2 sum_valid b + Cin * n_valid
// where sum_valid a is the popcount of the pixel's receptive field (pads are zero), sum_valid b sums the per-(filter,
// tap) popcount table (bdbnn_b1_popc_table) over the pixel's valid taps, and n_valid counts them.
//
// One CTA computes a 128-pixel x 64-filter tile over the whole K: every tap of the tile's A rows and B rows fits in
// shared memory (at most (128 + 64) x 9 x 64 bytes at Cin = 512), so there is no K loop to pipeline; the latency of
// one CTA's loads is hidden by the other CTAs on the SM.  Shared memory holds 16-byte K chunks as 8-row core
// matrices without swizzle: chunk kc of row m at ((m/8) * KCp + kc) * 128 + (m%8) * 16, KCp = the chunk count
// 9 * Cin / 128 rounded up to even, so one K = 256 step is two adjacent chunks (at Cin = 128 the two taps of a pair;
// the odd 9th tap is paired with a zero chunk in A and B).
#include "tc_common.cuh"

namespace bdbnn {

namespace {

constexpr int kB1TileM = 128, kB1TileN = 64, kB1Threads = 256, kB1Taps = 9;

__device__ __forceinline__ uint64_t b1_desc(uint32_t saddr, uint32_t sbo) {
  // layout type 0 (no swizzle), LBO = 128 bytes between the two K-adjacent core matrices, SBO between 8-row groups
  return uint64_t((saddr & 0x3FFFFu) >> 4) | (uint64_t(128u >> 4) << 16) | (uint64_t((sbo >> 4) & 0x3FFFu) << 32);
}

// D[64 x 64] (+)= popc(A[64 x 256] & B[64 x 256]^T), s32; accumulator layout as wgmma_ss's
__device__ __forceinline__ void bgmma_n64(int (&d)[32], uint64_t da, uint64_t db, int accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k256.s32.b1.b1.and.popc "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, "
      "%23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7]), "+r"(d[8]),
        "+r"(d[9]), "+r"(d[10]), "+r"(d[11]), "+r"(d[12]), "+r"(d[13]), "+r"(d[14]), "+r"(d[15]), "+r"(d[16]),
        "+r"(d[17]), "+r"(d[18]), "+r"(d[19]), "+r"(d[20]), "+r"(d[21]), "+r"(d[22]), "+r"(d[23]), "+r"(d[24]),
        "+r"(d[25]), "+r"(d[26]), "+r"(d[27]), "+r"(d[28]), "+r"(d[29]), "+r"(d[30]), "+r"(d[31])
      : "l"(da), "l"(db), "r"(accumulate)
      : "memory");
}

__device__ __forceinline__ void bgmma_n8(int (&d)[4], uint64_t da, uint64_t db) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 0, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n8k256.s32.b1.b1.and.popc {%0, %1, %2, %3}, %4, %5, p;\n\t}"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
      : "l"(da), "l"(db)
      : "memory");
}

// byte offset of K chunk kc of row m in a core-matrix tile with KCp chunks per row
__device__ __forceinline__ uint32_t b1_chunk_off(int m, int kc, int KCp) {
  return uint32_t(((m >> 3) * KCp + kc) * 128 + (m & 7) * 16);
}

struct B1Params {
  const uint32_t* x;       // [N*H*W][Cin/32]
  const uint32_t* w;       // [Cout][9][Cin/32]
  const int32_t* popc;     // [Cout][9]
  const float* scale; const float* shift; const float* res;   // eval
  float* z; uint32_t* zbits;                                  // eval (zbits may be NULL)
  int16_t* y;                                                 // int16 result
  int H, W, Cin, Cout, stride, Ho, Wo, KCp;
  int64_t P;
};

// valid-tap mask (bit r*3+q) of output pixel (oh, ow)
__device__ __forceinline__ uint32_t b1_tap_mask(int oh, int ow, int stride, int H, int W) {
  uint32_t rm = 0, cm = 0;
#pragma unroll
  for (int r = 0; r < 3; ++r) {
    const int ih = oh * stride - 1 + r, iw = ow * stride - 1 + r;
    rm |= uint32_t(ih >= 0 && ih < H) << r;
    cm |= uint32_t(iw >= 0 && iw < W) << r;
  }
  uint32_t m = 0;
#pragma unroll
  for (int r = 0; r < 3; ++r)
    if (rm >> r & 1u) m |= cm << (3 * r);
  return m;
}

// EVAL: z = fp32(fp32(y * scale) + shift) (+ residual), fp32 NHWC, and z's sign words (bit = z >= 0) if zbits.
// !EVAL: the exact integer y as int16 NHWC.
// CPT = Cin / 128, the 16-byte K chunks per tap: a compile-time K, so the wgmma chain is unrolled and not serialised.
template <bool EVAL, int CPT>
__global__ void __launch_bounds__(kB1Threads) b1_conv_kernel(const B1Params p) {
  extern __shared__ __align__(128) uint8_t smem[];
  constexpr int cpt = CPT, cw = 4 * CPT, KC = kB1Taps * CPT, KCp = (KC + 1) & ~1;
  uint8_t* sa = smem;                                                   // [128 rows][KCp chunks]
  uint8_t* sb = sa + kB1TileM * KCp * 16;                               // [64 rows][KCp chunks]
  int32_t* stab = reinterpret_cast<int32_t*>(sb + kB1TileN * KCp * 16);  // [64][9] popcount table
  int32_t* spop = stab + kB1TileN * kB1Taps;                            // [128] popcount of each A row
  const int tid = threadIdx.x;
  const int64_t m0 = int64_t(blockIdx.x) * kB1TileM;
  const int n0 = blockIdx.y * kB1TileN;
  const int hw = p.Ho * p.Wo;

  // A: thread item = (8-row group g, chunk kc, row r in group), r fastest so 8 threads fill one 128-byte core matrix
  for (int i = tid; i < kB1TileM * KCp; i += kB1Threads) {
    const int r = i & 7, rest = i >> 3, kc = rest % KCp, g = rest / KCp;
    const int m = g * 8 + r;
    const int64_t pix = m0 + m;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (kc < KC && pix < p.P) {
      const int t = kc / cpt, c = kc - t * cpt;
      const int n = int(pix / hw), rem = int(pix - int64_t(n) * hw), oh = rem / p.Wo, ow = rem - oh * p.Wo;
      const int ih = oh * p.stride - 1 + t / 3, iw = ow * p.stride - 1 + t % 3;
      if (ih >= 0 && ih < p.H && iw >= 0 && iw < p.W)
        v = __ldg(reinterpret_cast<const uint4*>(p.x + ((int64_t(n) * p.H + ih) * p.W + iw) * cw + 4 * c));
    }
    *reinterpret_cast<uint4*>(sa + b1_chunk_off(m, kc, KCp)) = v;
  }
  for (int i = tid; i < kB1TileN * KCp; i += kB1Threads) {
    const int r = i & 7, rest = i >> 3, kc = rest % KCp, g = rest / KCp;
    const int m = g * 8 + r;
    uint4 v = make_uint4(0u, 0u, 0u, 0u);
    if (kc < KC) {
      const int t = kc / cpt, c = kc - t * cpt;
      v = __ldg(reinterpret_cast<const uint4*>(p.w + (int64_t(n0 + m) * kB1Taps + t) * cw + 4 * c));
    }
    *reinterpret_cast<uint4*>(sb + b1_chunk_off(m, kc, KCp)) = v;
  }
  for (int i = tid; i < kB1TileN * kB1Taps; i += kB1Threads) stab[i] = __ldg(p.popc + n0 * kB1Taps + i);
  fence_proxy_async();   // the generic-proxy stores above are read by the wgmma (async proxy)
  __syncthreads();

  const int wg = tid >> 7, wt = tid & 127, warp = wt >> 5, lane = tid & 31;
  int acc[32];
#pragma unroll
  for (int i = 0; i < 32; ++i) acc[i] = 0;
  const uint32_t sbo = uint32_t(KCp) * 128u;
  const uint32_t a0 = smem_u32(sa) + uint32_t(wg) * 8u * sbo, b0 = smem_u32(sb);
  wgmma_fence();
#pragma unroll
  for (int ks = 0; ks < KCp / 2; ++ks) bgmma_n64(acc, b1_desc(a0 + ks * 256u, sbo), b1_desc(b0 + ks * 256u, sbo), ks);
  wgmma_commit();

  // while the tensor cores run: popcount of each of this warpgroup's 64 A rows, two threads per row
  {
    const int m = wg * 64 + (wt >> 1);
    int s = 0;
    for (int kc = wt & 1; kc < KCp; kc += 2) {
      const uint4 v = *reinterpret_cast<const uint4*>(sa + b1_chunk_off(m, kc, KCp));
      s += __popc(v.x) + __popc(v.y) + __popc(v.z) + __popc(v.w);
    }
    s += __shfl_xor_sync(0xffffffffu, s, 1);
    if ((wt & 1) == 0) spop[m] = s;
  }
  if (wg == 0)   // named barrier of the warpgroup's 128 threads (0 is __syncthreads')
    asm volatile("bar.sync 1, 128;" ::: "memory");
  else
    asm volatile("bar.sync 2, 128;" ::: "memory");
  wgmma_wait<0>();
#pragma unroll
  for (int i = 0; i < 32; ++i) asm volatile("" : "+r"(acc[i])::"memory");

  int64_t pix[2];
  bool valid[2];
  uint32_t tmask[2];
  int base[2];   // Cin * n_valid - 2 * sum_valid a
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int m = wg * 64 + 16 * warp + (lane >> 2) + 8 * h;
    pix[h] = m0 + m;
    valid[h] = pix[h] < p.P;
    tmask[h] = 0;
    if (valid[h]) {
      const int n = int(pix[h] / hw), rem = int(pix[h] - int64_t(n) * hw), oh = rem / p.Wo, ow = rem - oh * p.Wo;
      tmask[h] = b1_tap_mask(oh, ow, p.stride, p.H, p.W);
    }
    base[h] = p.Cin * __popc(tmask[h]) - 2 * spop[m];
  }
  uint32_t bits[2][2] = {{0u, 0u}, {0u, 0u}};
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const int col = 8 * j + 2 * (lane & 3);
    const int ch = n0 + col;
    int sbv[2][2] = {{0, 0}, {0, 0}};   // [row][column of the pair]: sum_valid b
#pragma unroll
    for (int t = 0; t < kB1Taps; ++t) {
      const int b0v = stab[col * kB1Taps + t], b1v = stab[(col + 1) * kB1Taps + t];
#pragma unroll
      for (int h = 0; h < 2; ++h)
        if (tmask[h] >> t & 1u) { sbv[h][0] += b0v; sbv[h][1] += b1v; }
    }
    float sc0 = 0.f, sc1 = 0.f, sh0 = 0.f, sh1 = 0.f;
    if (EVAL) {
      sc0 = __ldg(p.scale + ch); sc1 = __ldg(p.scale + ch + 1);
      sh0 = __ldg(p.shift + ch); sh1 = __ldg(p.shift + ch + 1);
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int y0 = 4 * acc[4 * j + 2 * h] + base[h] - 2 * sbv[h][0];
      const int y1 = 4 * acc[4 * j + 2 * h + 1] + base[h] - 2 * sbv[h][1];
      if (!valid[h]) continue;
      const int64_t off = pix[h] * p.Cout + ch;
      if (EVAL) {
        // one rounding per step, no FMA contraction: tc_conv_kernel<2>'s z
        float o0 = __fadd_rn(__fmul_rn(float(y0), sc0), sh0);
        float o1 = __fadd_rn(__fmul_rn(float(y1), sc1), sh1);
        if (p.res != nullptr) {
          const float2 r = __ldg(reinterpret_cast<const float2*>(p.res + off));
          o0 = __fadd_rn(o0, r.x); o1 = __fadd_rn(o1, r.y);
        }
        *reinterpret_cast<float2*>(p.z + off) = make_float2(o0, o1);
        // sign(v) = +1 iff v >= 0 (DESIGN.md §2): -0.0 -> 1, NaN -> 0, as bdbnn_act_pack
        bits[h][j >> 2] |= (uint32_t(o0 >= 0.f) | (uint32_t(o1 >= 0.f) << 1)) << (col & 31);
      } else {
        *reinterpret_cast<uint32_t*>(p.y + off) = (uint32_t(y0) & 0xffffu) | (uint32_t(y1) << 16);
      }
    }
  }
  if (EVAL && p.zbits != nullptr) {
    // a 32-channel word is spread over the four lanes of a quad: OR it together
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        uint32_t v = bits[h][k];
        v |= __shfl_xor_sync(0xffffffffu, v, 1);
        v |= __shfl_xor_sync(0xffffffffu, v, 2);
        if (valid[h] && (lane & 3) == 0) p.zbits[pix[h] * (p.Cout >> 5) + (n0 >> 5) + k] = v;
      }
  }
}

__global__ void b1_popc_table_kernel(const uint32_t* __restrict__ w, int rows, int cw, int32_t* __restrict__ table) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  int s = 0;
  for (int k = 0; k < cw; ++k) s += __popc(__ldg(w + int64_t(i) * cw + k));
  table[i] = s;
}

__global__ void b1_debug_mma_kernel(const uint32_t* a, const uint32_t* b, int32_t* d) {
  __shared__ __align__(128) uint8_t sa[64 * 32];
  __shared__ __align__(128) uint8_t sb[8 * 32];
  const int t = threadIdx.x;
  for (int i = t; i < 64 * 2; i += 128) {
    const int m = i >> 1, kc = i & 1;
    *reinterpret_cast<uint4*>(sa + b1_chunk_off(m, kc, 2)) = reinterpret_cast<const uint4*>(a)[i];
  }
  if (t < 16) {
    const int m = t >> 1, kc = t & 1;
    *reinterpret_cast<uint4*>(sb + b1_chunk_off(m, kc, 2)) = reinterpret_cast<const uint4*>(b)[t];
  }
  fence_proxy_async();
  __syncthreads();
  int acc[4] = {0, 0, 0, 0};
  wgmma_fence();
  bgmma_n8(acc, b1_desc(smem_u32(sa), 256u), b1_desc(smem_u32(sb), 256u));
  wgmma_commit();
  wgmma_wait<0>();
  const int w = t >> 5, l = t & 31, row = 16 * w + (l >> 2), col = 2 * (l & 3);
  d[row * 8 + col] = acc[0]; d[row * 8 + col + 1] = acc[1];
  d[(row + 8) * 8 + col] = acc[2]; d[(row + 8) * 8 + col + 1] = acc[3];
}

template <bool EVAL, int CPT>
int launch_b1_cpt(const B1Params& p, cudaStream_t st) {
  const size_t smem = size_t(kB1TileM + kB1TileN) * p.KCp * 16 + (kB1TileN * kB1Taps + kB1TileM) * 4;
  BDBNN_CUDA(cudaFuncSetAttribute(b1_conv_kernel<EVAL, CPT>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  int(smem)));
  const int64_t mt = (p.P + kB1TileM - 1) / kB1TileM;
  BDBNN_REQUIRE(mt < (int64_t(1) << 31), "binconv_fwd_b1: too many pixels");
  b1_conv_kernel<EVAL, CPT><<<dim3(unsigned(mt), unsigned(p.Cout / kB1TileN)), kB1Threads, smem, st>>>(p);
  return check_launch(EVAL ? "binconv_fwd_b1_eval" : "binconv_fwd_b1_i16");
}

template <bool EVAL>
int launch_b1(const B1Params& p, cudaStream_t st) {
  switch (p.Cin) {
    case 128: return launch_b1_cpt<EVAL, 1>(p, st);
    case 256: return launch_b1_cpt<EVAL, 2>(p, st);
    default: return launch_b1_cpt<EVAL, 4>(p, st);   // 384 is refused by b1_shape_ok
  }
}

int b1_params(B1Params* p, const uint32_t* xbits, const uint32_t* wsign, const int32_t* popc,
              const bdbnn_conv_shape* s, const char* what) {
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(xbits && wsign && popc, "%s: NULL pointer", what);
  BDBNN_REQUIRE(((reinterpret_cast<uintptr_t>(xbits) | reinterpret_cast<uintptr_t>(wsign)) & 15u) == 0,
                "%s: the bit operands must be 16-byte aligned", what);
  if (!b1_shape_ok(s)) {
    set_error("%s: shape not supported by the binary tensor-core kernel", what);
    return BDBNN_ERR_UNSUPPORTED;
  }
  memset(p, 0, sizeof(*p));
  p->x = xbits; p->w = wsign; p->popc = popc;
  p->H = s->H; p->W = s->W; p->Cin = s->Cin; p->Cout = s->Cout; p->stride = s->stride; p->Ho = s->Ho; p->Wo = s->Wo;
  p->KCp = (kB1Taps * (s->Cin / 128) + 1) & ~1;
  p->P = int64_t(s->N) * s->Ho * s->Wo;
  return BDBNN_OK;
}

}  // namespace

bool b1_shape_ok(const bdbnn_conv_shape* s) {
  return s->kh == 3 && s->kw == 3 && s->pad == 1 && (s->stride == 1 || s->stride == 2) &&
         (s->Cin == 128 || s->Cin == 256 || s->Cin == 512) && s->Cout % 64 == 0;
}

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_b1_popc_table(const uint32_t* wsign, int32_t Cout, int32_t Cin, int32_t T, int32_t* table,
                                   void* stream) {
  BDBNN_REQUIRE(wsign && table, "b1_popc_table: NULL pointer");
  BDBNN_REQUIRE(Cout > 0 && Cin > 0 && T > 0, "b1_popc_table: non-positive dims");
  const int rows = Cout * T;
  b1_popc_table_kernel<<<(rows + 255) / 256, 256, 0, cudaStream_t(stream)>>>(wsign, rows, (Cin + 31) / 32, table);
  return check_launch("b1_popc_table");
}

extern "C" int bdbnn_binconv_fwd_b1_eval(const uint32_t* xbits, const uint32_t* wsign, const int32_t* popc,
                                         const float* scale, const float* shift, const float* residual, float* z,
                                         uint32_t* zbits, const bdbnn_conv_shape* s, void* stream) {
  B1Params p;
  int rc = b1_params(&p, xbits, wsign, popc, s, "binconv_fwd_b1_eval");
  if (rc) return rc;
  BDBNN_REQUIRE(scale && shift && z, "binconv_fwd_b1_eval: NULL pointer");
  BDBNN_REQUIRE(residual != z, "binconv_fwd_b1_eval: residual must not alias z");
  p.scale = scale; p.shift = shift; p.res = residual; p.z = z; p.zbits = zbits;
  return launch_b1<true>(p, cudaStream_t(stream));
}

extern "C" int bdbnn_binconv_fwd_b1_i16(const uint32_t* xbits, const uint32_t* wsign, const int32_t* popc,
                                        int16_t* y_int, const bdbnn_conv_shape* s, void* stream) {
  B1Params p;
  int rc = b1_params(&p, xbits, wsign, popc, s, "binconv_fwd_b1_i16");
  if (rc) return rc;
  BDBNN_REQUIRE(y_int, "binconv_fwd_b1_i16: NULL pointer");
  p.y = y_int;
  return launch_b1<false>(p, cudaStream_t(stream));
}

extern "C" int bdbnn_debug_b1_mma(const uint32_t* a, const uint32_t* b, int32_t* d, void* stream) {
  BDBNN_REQUIRE(a && b && d, "debug_b1_mma: NULL pointer");
  BDBNN_REQUIRE(((reinterpret_cast<uintptr_t>(a) | reinterpret_cast<uintptr_t>(b)) & 15u) == 0,
                "debug_b1_mma: a and b must be 16-byte aligned");
  b1_debug_mma_kernel<<<1, 128, 0, cudaStream_t(stream)>>>(a, b, d);
  return check_launch("debug_b1_mma");
}
