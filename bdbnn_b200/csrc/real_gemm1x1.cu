// Eval-mode 1x1 conv of a real-valued teacher that reads its fp32 input directly (DESIGN.md §4q).
//
// bdbnn_real_act_pack + bdbnn_real_conv_fwd_eval read x as fp32, write it as fp16 and read the fp16 copy again; for a
// 1x1 conv (36 of ResNet-50's 53 convs) this kernel rounds x to fp16 on the way into shared memory instead:
//   warpgroup 2   : A producer.  Per 64-channel K block it loads the 128 x 64 fp32 tile of x (rows = output pixels,
//                   read at `stride`), rounds fp16(x * 2^ex) exactly as real_pack_x_kernel does, and stores it in the
//                   128-byte-swizzled K-major layout a TMA box would have; thread 0 also issues the TMA of the B box
//                   [BN x 64] of wf.  A ring slot is full when the 128 threads arrived (after a proxy fence) and the
//                   B bytes landed.
//   warpgroups 0/1: wgmma m64nNk16 over rows [0, 64) / [64, 128), the same four k16 steps per K block in ascending K
//                   from a zero accumulator as tc_conv_kernel, so the sums are bit-identical to the pack + GEMM pair;
//                   then real_conv_fwd_eval's epilogue unchanged (scale and shift rounded separately, residual,
//                   act code, max|z| word).
// Its own file: the existing kernels' code is untouched.
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace bdbnn {

constexpr int kG1Threads = 384;           // 2 consumer warpgroups + 1 producer warpgroup
constexpr int kG1KB = 64;                 // fp16 channels per K block: one 128-byte swizzled row
constexpr int kG1RowsPerThread = kTileM * kG1KB / 4 / 128;   // float4s of the A tile per producer thread (16)

struct Gemm1x1Params {
  const float4* x;                        // fp32 NHWC [N][H][W][Cin] as float4s
  int32_t H, W, Ho, Wo, stride, c4;       // c4 = Cin / 4
  int64_t M;                              // output pixels N * Ho * Wo
  int32_t n_kb, stages, Nout;
  const uint32_t* x_amax;
  const float* scale;
  const float* shift;
  const float* add;                       // optional residual [M][Nout]
  int32_t act;
  float* out;                             // [M][Nout]
  uint32_t* z_amax;                       // optional, pre-zeroed
};

template <int NW>
__global__ void __launch_bounds__(kG1Threads, 1)
real_gemm1x1_kernel(const __grid_constant__ CUtensorMap tmB, const Gemm1x1Params p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[kMaxStages];
  constexpr uint32_t a_bytes = kTileM * 128, stage_bytes = a_bytes + NW * 128;   // both multiples of 1024
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t tiles_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int64_t m0 = int64_t(blockIdx.x) * kTileM;
  const int nn0 = blockIdx.y * NW;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 128 + 1);   // 128 producer arrivals + thread 0's expect_tx
      mbar_init(smem_u32(&empty_bar[s]), 2);        // one arrival per consumer warpgroup
    }
    fence_barrier_init();
    prefetch_tmap(&tmB);
  }
  __syncthreads();

  if (warp >= 8) {
    const int t = threadIdx.x - 256;
    const int q = t & 15, r0 = t >> 4;     // float4 q of the K block, rows r0 + 8 i
    // input pixel of each of this thread's rows, -1 past the last output pixel
    int32_t ipix[kG1RowsPerThread];
#pragma unroll
    for (int i = 0; i < kG1RowsPerThread; ++i) {
      const int64_t m = m0 + r0 + 8 * i;
      if (m < p.M) {
        const int wo = int(m % p.Wo);
        const int64_t nh = m / p.Wo;
        const int ho = int(nh % p.Ho);
        const int n = int(nh / p.Ho);
        ipix[i] = (n * p.H + ho * p.stride) * p.W + wo * p.stride;
      } else {
        ipix[i] = -1;
      }
    }
    const float scale = amax_pow2_scale(__ldg(p.x_amax), false);
    for (int kb = 0; kb < p.n_kb; ++kb) {
      const int stage = kb % p.stages;
      const uint32_t phase = uint32_t(kb / p.stages) & 1u;
      float4 v[kG1RowsPerThread];
#pragma unroll
      for (int i = 0; i < kG1RowsPerThread; ++i)
        v[i] = ipix[i] >= 0 ? __ldg(p.x + int64_t(ipix[i]) * p.c4 + kb * (kG1KB / 4) + q) : make_float4(0.f, 0.f, 0.f, 0.f);
      mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1u);
      const uint32_t a_dst = tiles_base + stage * stage_bytes;
      const uint32_t fb = smem_u32(&full_bar[stage]);
      if (t == 0) {
        mbar_expect_tx(fb, NW * 128);
        tma_load_2d(a_dst + a_bytes, &tmB, fb, kb * kG1KB, nn0);
      }
#pragma unroll
      for (int i = 0; i < kG1RowsPerThread; ++i) {
        const int r = r0 + 8 * i;
        // real_pack_x_kernel's rounding: fp16(x * 2^ex), one product, round to nearest even
        const __half2 a = __floats2half2_rn(v[i].x * scale, v[i].y * scale);
        const __half2 b = __floats2half2_rn(v[i].z * scale, v[i].w * scale);
        // SWIZZLE_128B: 16-byte chunk j of row r sits at chunk j ^ (r % 8); float4 q is half of chunk q / 2
        const uint32_t addr = a_dst + uint32_t(r) * 128u + uint32_t(((q >> 1) ^ (r & 7)) << 4) + uint32_t(q & 1) * 8u;
        asm volatile("st.shared.v2.b32 [%0], {%1, %2};" ::"r"(addr), "r"(*reinterpret_cast<const uint32_t*>(&a)),
                     "r"(*reinterpret_cast<const uint32_t*>(&b))
                     : "memory");
      }
      fence_proxy_async();                 // the generic-proxy stores are visible to wgmma's async proxy
      mbar_arrive(fb);
    }
  } else {
    const int wg = warp >> 2, wq = warp & 3;
    float acc[NW / 2];
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) acc[i] = 0.f;
    for (int kb = 0; kb < p.n_kb; ++kb) {
      const int stage = kb % p.stages;
      mbar_wait(smem_u32(&full_bar[stage]), uint32_t(kb / p.stages) & 1u);
      const uint32_t a_src = tiles_base + stage * stage_bytes + uint32_t(wg * 64 * 128);
      const uint32_t b_src = tiles_base + stage * stage_bytes + a_bytes;
      wgmma_fence();
#pragma unroll
      for (int k = 0; k < 4; ++k)
        wgmma_ss<NW, 0>(acc, make_kmajor_desc(a_src + k * 32, 128), make_kmajor_desc(b_src + k * 32, 128));
      wgmma_commit();
      wgmma_wait<1>();
      if (kb > 0 && (threadIdx.x & 127) == 0) mbar_arrive(smem_u32(&empty_bar[(kb - 1) % p.stages]));
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);

    // ---- epilogue: real_conv_fwd_eval's; this thread holds rows r and r + 8 (r = 64 wg + 16 wq + lane/4) ----
    const float post = amax_pow2_scale(__ldg(p.x_amax), true);
    uint32_t zmax = 0u;
    int64_t pix[2];
    bool valid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      pix[h] = m0 + wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
      valid[h] = pix[h] < p.M;
    }
#pragma unroll
    for (int j = 0; j < NW / 8; ++j) {
      const int ch = nn0 + 8 * j + 2 * (lane & 3);
      const float a0 = __ldg(p.scale + ch), a1 = __ldg(p.scale + ch + 1);
      const float sb0 = __ldg(p.shift + ch), sb1 = __ldg(p.shift + ch + 1);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!valid[h]) continue;
        const int64_t off = pix[h] * p.Nout + ch;
        float o0 = __fadd_rn(__fmul_rn(__fmul_rn(acc[4 * j + 2 * h], post), a0), sb0);
        float o1 = __fadd_rn(__fmul_rn(__fmul_rn(acc[4 * j + 2 * h + 1], post), a1), sb1);
        if (p.add != nullptr) {
          const float2 r = __ldg(reinterpret_cast<const float2*>(p.add + off));
          o0 = __fadd_rn(o0, r.x); o1 = __fadd_rn(o1, r.y);
        }
        if (p.act == BDBNN_ACT_HARDTANH) {   // torch.nn.Hardtanh: NaN stays NaN, -0.0 stays -0.0
          o0 = o0 < -1.f ? -1.f : (o0 > 1.f ? 1.f : o0);
          o1 = o1 < -1.f ? -1.f : (o1 > 1.f ? 1.f : o1);
        } else if (p.act == BDBNN_ACT_RELU) {   // torch.relu: NaN stays NaN
          o0 = o0 != o0 ? o0 : fmaxf(o0, 0.f);
          o1 = o1 != o1 ? o1 : fmaxf(o1, 0.f);
        }
        *reinterpret_cast<float2*>(p.out + off) = make_float2(o0, o1);
        zmax = max(zmax, max(__float_as_uint(fabsf(o0)), __float_as_uint(fabsf(o1))));
      }
    }
    if (p.z_amax != nullptr) {
      zmax = __reduce_max_sync(0xffffffffu, zmax);
      if (lane == 0 && zmax != 0u) atomicMax(p.z_amax, zmax);
    }
  }
}

static bool gemm1x1_shape_ok(const bdbnn_conv_shape* s) {
  if (!s || s->kh != 1 || s->kw != 1 || s->pad != 0 || (s->stride != 1 && s->stride != 2)) return false;
  // the channel counts the pack + real_conv_fwd_eval pair takes with 128-byte K rows, so that both paths exist
  if (!(s->Cin == 64 || s->Cin % 128 == 0)) return false;
  if (!(s->Cout == 16 || s->Cout == 32 || s->Cout == 64 || s->Cout % 128 == 0)) return false;
  // the producer's input pixel index is 32-bit
  return int64_t(s->N) * s->H * s->W < INT32_MAX;
}

template <int NW>
static int launch_gemm1x1(const CUtensorMap& tmB, const Gemm1x1Params& p, cudaStream_t st) {
  const size_t smem = size_t(p.stages) * (kTileM + NW) * 128 + 1024;
  BDBNN_CUDA(cudaFuncSetAttribute(real_gemm1x1_kernel<NW>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  const dim3 grid(unsigned((p.M + kTileM - 1) / kTileM), unsigned(p.Nout / NW));
  real_gemm1x1_kernel<NW><<<grid, kG1Threads, smem, st>>>(tmB, p);
  return check_launch("real_gemm1x1_kernel");
}

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_real_gemm1x1_supported(const bdbnn_conv_shape* s) {
  if (!s || validate_shape(s) != BDBNN_OK) return 0;
  return gemm1x1_shape_ok(s) ? 1 : 0;
}

extern "C" int bdbnn_real_gemm1x1_fwd_eval(const float* x, const uint32_t* x_amax_bits, const uint16_t* wf,
                                           const float* scale, const float* shift, const float* residual,
                                           int32_t act, float* z, uint32_t* z_amax_bits, const bdbnn_conv_shape* s,
                                           void* stream) {
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(x && x_amax_bits && wf && scale && shift && z, "real_gemm1x1_fwd_eval: NULL pointer");
  BDBNN_REQUIRE(act >= BDBNN_ACT_NONE && act <= BDBNN_ACT_HARDTANH,
                "real_gemm1x1_fwd_eval: act must be 0 (none), 1 (ReLU) or 2 (Hardtanh), got %d", act);
  BDBNN_REQUIRE(residual != z && x != z, "real_gemm1x1_fwd_eval: x and residual must not alias z");
  BDBNN_REQUIRE((uintptr_t(x) & 15) == 0, "real_gemm1x1_fwd_eval: x must be 16-byte aligned");
  if (!gemm1x1_shape_ok(s)) {
    set_error("real_gemm1x1_fwd_eval: needs a 1x1 / pad-0 conv of stride 1 or 2, Cin 64 or a multiple of 128, "
              "Cout 16, 32, 64 or a multiple of 128");
    return BDBNN_ERR_UNSUPPORTED;
  }
  cudaStream_t st = cudaStream_t(stream);
  const int bn = s->Cout >= 128 ? 128 : s->Cout;
  CUtensorMap tmB;
  rc = make_weight_map(&tmB, wf, s->Cout, s->Cin, kG1KB, bn, 2);
  if (rc) return rc;
  Gemm1x1Params p;
  memset(&p, 0, sizeof(p));
  p.x = reinterpret_cast<const float4*>(x);
  p.H = s->H; p.W = s->W; p.Ho = s->Ho; p.Wo = s->Wo; p.stride = s->stride; p.c4 = s->Cin / 4;
  p.M = int64_t(s->N) * s->Ho * s->Wo;
  p.n_kb = s->Cin / kG1KB;
  const int stage_bytes = (kTileM + bn) * 128;
  int stages = (192 * 1024) / stage_bytes;
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages > p.n_kb) stages = p.n_kb;
  p.stages = stages;
  p.Nout = s->Cout;
  p.x_amax = x_amax_bits;
  p.scale = scale; p.shift = shift; p.add = residual; p.act = act;
  p.out = z; p.z_amax = z_amax_bits;
  if (z_amax_bits) BDBNN_CUDA(cudaMemsetAsync(z_amax_bits, 0, sizeof(uint32_t), st));
  switch (bn) {
    case 16: return launch_gemm1x1<16>(tmB, p, st);
    case 32: return launch_gemm1x1<32>(tmB, p, st);
    case 64: return launch_gemm1x1<64>(tmB, p, st);
    default: return launch_gemm1x1<128>(tmB, p, st);
  }
}
