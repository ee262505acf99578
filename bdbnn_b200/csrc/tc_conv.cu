// wgmma / TMA implicit-GEMM kernel for the binary convolution (sm_90a).
//
//   tc_conv_kernel  : D[pix, n] = sum_{tap t} sum_{k} A[pix shifted by t, k] * B[n, t*Kc + k]
//                     forward : A = sign(x)  (+-1 fp16/bf16/fp8, NHWC), B = sign(W) [Cout][T][Cin]; epilogue * alpha[n]
//                     dgrad   : A = gy*gscale (bf16/fp16,  NHWC), B = sign(W)^T [Cin][T'][Cout]; epilogue * STE mask bit
//                     eval    : the forward's operands; epilogue z = acc * scale[n] + shift[n] (+ residual), the
//                               eval-mode BatchNorm folded into one affine map, and the +-1 copy of z
//
// Dataflow per CTA (one 128-row output tile, one N tile of BN <= 128 columns):
//   warp 8 lane 0 : TMA producer. For every (tap, K-block) loads the activation box
//                   [BNI images][BH rows][BW=OW cols][KB channels] at coordinates shifted by the tap —
//                   TMA zero-fills out-of-image coordinates, which IS the conv's zero padding — and the
//                   matching [BN x KB] weight box, into a `stages`-deep ring of swizzled K-major tiles.
//   warpgroups 0/1: wgmma (fp32 accumulate in registers) for tile rows [0, 64) / [64, 128): per ring slot one wgmma
//                   as wide as the N tile for every 32 bytes of the K rows, an unbroken chain (the kernel is
//                   instantiated per N width, so the A tile is read from shared memory once per K step).  One wgmma
//                   group in flight: a ring slot is released once the group after it was issued and the one reading
//                   it retired.
//                   Then the epilogue from the same registers: alpha or STE mask, optional int16 result, additive
//                   tensor, and the per-channel BatchNorm statistics of the result (forward: sum y, sum y^2,
//                   max|y|; dgrad: the backward sums of the BatchNorm unit that produced the conv input).
// +-1 operands and fp32 accumulation make the forward integer-exact (|sum| <= 9*512 < 2^24).
#include "tc_common.cuh"

namespace bdbnn {

constexpr int kMaxBN = 128;

struct TcConvParams {
  int32_t OW, OH, NIMG;      // output pixel grid (one GEMM row per output pixel)
  int32_t BW, BH, BNI;       // tile = BNI images x BH rows x BW(=OW) cols  (<= 128 pixels)
  int32_t tiles_h;           // tiles per image group along h
  int32_t Kc, KB, n_kb;      // contraction channels, K-block elements, Kc/KB
  int32_t a_halves;          // 1: A has Kc channels; 2: A = [hi | lo] bf16 split, 2*Kc channels, B reused
  int32_t in_step;           // input coordinate = out coordinate * in_step + tap offset (2 for stride-2 fwd)
  int32_t n_taps;            // taps actually visited (subset for the stride-2 dgrad phases)
  int8_t tap_dh[kMaxTaps], tap_dw[kMaxTaps];   // input offset of tap i
  uint8_t tap_b[kMaxTaps];   // K-block row of B for tap i (B column = tap_b * Kc + k)
  int32_t out_step, out_off_h, out_off_w, OHf, OWf;  // out pixel = (oh*out_step+off_h, ow*out_step+off_w) in OHf x OWf
  int32_t Nout, BN;          // GEMM N total / per CTA
  int32_t stages;
  int32_t cm, cn;            // cluster: cm CTAs along M share the weight box, cn along N share the activation box
  int32_t row_bytes;         // KB * element size = swizzle span (32/64/128)
  const uint32_t* amax_bits; // MODE 1 FP16S / MODE 2 real operands: post-scale 2^-e of the A operand (NULL = 1)
  const float* add;          // dgrad: optional additive tensor; eval: optional residual
  const float* alpha;        // MODE 0: per-output-channel scale; MODE 2: folded BatchNorm scale
  const float* shift;        // MODE 2: folded BatchNorm shift
  int32_t relu;              // MODE 2: z = relu(z) after the residual (NaN propagates, as torch.relu)
  uint32_t* z_amax;          // MODE 2: optional bits of max|z| (pre-zeroed, integer atomicMax)
  uint16_t* zb;              // MODE 2: optional 16-bit +-1 copy of z (+1 = zb_one, -1 = zb_one | 0x8000)
  uint8_t* zb8;              // MODE 2: optional fp8 e4m3 +-1 copy of z
  uint32_t zb_one;           // MODE 2: 16-bit +1 (0x3C00 fp16, 0x3F80 bf16)
  const uint32_t* mask;      // MODE 1: STE mask words [pix][Nout/32 (ceil)]
  float* out;                // [pix][Nout] fp32
  int16_t* out_i16;          // MODE 0: the exact integer accumulator as int16 instead of out (y = alpha * int)
  double* bn_sums;           // per-channel statistics [2*Nout] (NULL = off), see TcConvLaunch
  double* stat_part;         // this launch's per-CTA statistics rows [gridDim.x][2*Nout] (det_sums_finish adds them)
  uint32_t* bn_ymax;
  const int16_t* st_y; const float* st_alpha; const float* st_mean; const float* st_invstd;   // MODE 1 statistics
  // PADRES instances: output pixel (n, oh, ow), channel ch reads the residual add[n][2*oh][2*ow][ch - res_coff] of an
  // NHWC [.][res_H][res_W][res_C] tensor inside the band res_coff <= ch < res_coff + res_C, +0.0 outside it
  int32_t res_H, res_W, res_C, res_coff;
};

// One K block of a ring slot: KS wgmmas back to back, each over 32 bytes of every row (row_bytes = 32 * KS).  KS and
// the N width are compile-time, so nothing stands between the wgmmas of a group: ptxas keeps the accumulator in place
// and issues them as one uninterrupted chain.
template <int NW, int KIND, int KS>
__device__ __forceinline__ void wgmma_k_block(float (&acc)[NW / 2], uint32_t a_src, uint32_t b_src) {
  wgmma_fence();
#pragma unroll
  for (int k = 0; k < KS; ++k)
    wgmma_ss<NW, KIND>(acc, make_kmajor_desc(a_src + k * 32, 32 * KS), make_kmajor_desc(b_src + k * 32, 32 * KS));
}

// MODE: 0 forward, 1 dgrad, 2 eval forward; KIND: 0 fp16, 1 bf16, 2 fp8 e4m3 operands; NW: the N tile (BN = 16, 32,
// 64 or 128), one wgmma wide.
// Two CTAs per SM need <= 96 registers per thread: registers are allocated per warp inside each of the SM's four
// 16K-register sub-partitions, and 2 x 9 warps put five warps on two of them.  The dgrad and eval instances ask for
// that bound (without it the 128-column dgrad ones took 102 registers and ran one CTA per SM); the forward ones fit at
// 96 without it (0 = no minimum).  bdbnn_debug_tc_conv_ctas_per_sm reports the residency.
// PADRES (MODE 2, 16-bit operands only): the residual is the CIFAR option-A shortcut read in place (res_* fields),
// an instance of its own so that the dense-residual instances keep their code.
// HARDTANH (MODE 2, fp16 operands, no PADRES): z = hardtanh(z) where relu would apply (p.relu is not read), the
// VGG-Small teacher's unpooled convs; instances of their own for the same reason.
// BANDED (fp16 operands, no PADRES / HARDTANH): a grouped conv as a banded GEMM (DESIGN.md §4t): the N tile is one
// band of BN = Kc channels and the activation box reads channels [nn0, nn0 + Kc) of A; instances of their own too.
template <int MODE, int KIND, int NW, bool PADRES = false, bool HARDTANH = false, bool BANDED = false>
__global__ void __launch_bounds__(kTcThreads, MODE == 0 ? 0 : 2)
tc_conv_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const TcConvParams p) {
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[kMaxStages];
  // per-warp statistics partials, summed in a fixed order at the end (run-to-run deterministic)
  __shared__ float stat_sum[kTcThreads / 32 - 1][kMaxBN], stat_sq[kTcThreads / 32 - 1][kMaxBN];
  __shared__ float stat_max[kTcThreads / 32 - 1][kMaxBN];

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t tiles_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const uint32_t a_bytes = kTileM * p.row_bytes;   // ring slot: A tile, then B tile
  const uint32_t stage_bytes = (a_bytes + uint32_t(p.BN) * p.row_bytes + 1023u) & ~1023u;
  const int tile_n = blockIdx.x / p.tiles_h, tile_h = blockIdx.x - tile_n * p.tiles_h;
  const int n0 = tile_n * p.BNI, h0 = tile_h * p.BH;
  const int nn0 = blockIdx.y * p.BN;
  const int kb_total = p.n_kb * p.a_halves;
  const int n_iters = p.n_taps * kb_total;
  const bool do_stats = MODE != 2 && p.bn_sums != nullptr;
  // cluster rank (x + y * cm); with cm * cn > 1 a ring slot is refilled only after the consumers of every CTA of the
  // cluster released it, since any of them may multicast into it
  const int cs = p.cm * p.cn;
  const int rx = int(blockIdx.x) % p.cm, ry = int(blockIdx.y) % p.cn;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), 2 * cs);   // one arrival per consumer warpgroup of the cluster
    }
    fence_barrier_init();
  }
  if (MODE != 2)
    for (int i = threadIdx.x; i < (kTcThreads / 32 - 1) * kMaxBN; i += blockDim.x) {
      (&stat_sum[0][0])[i] = 0.f; (&stat_sq[0][0])[i] = 0.f; (&stat_max[0][0])[i] = 0.f;
    }
  if (warp == kProducerWarp && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
  }
  if (cs > 1) cluster_sync();   // peers' barriers are initialised before anyone multicasts or arrives on them
  else __syncthreads();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      const uint32_t tx = uint32_t(p.BNI * p.BH * p.BW + p.BN) * uint32_t(p.row_bytes);
      // multicast groups: same M tile (column of the cluster) share A, same N tile (row) share B; the CTAs of a
      // group take turns loading the shared box, one iteration each
      uint16_t a_mask = 0, b_mask = 0;
      for (int y = 0; y < p.cn; ++y) a_mask |= uint16_t(1u << (rx + y * p.cm));
      for (int x = 0; x < p.cm; ++x) b_mask |= uint16_t(1u << (x + ry * p.cm));
      int it = 0;
      for (int ti = 0; ti < p.n_taps; ++ti) {
        const int dh = p.tap_dh[ti], dw = p.tap_dw[ti], tb = p.tap_b[ti];
        for (int kb = 0; kb < kb_total; ++kb, ++it) {
          const int stage = it % p.stages;
          const uint32_t phase = uint32_t(it / p.stages) & 1u;
          mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1u);
          const uint32_t fb = smem_u32(&full_bar[stage]);
          mbar_expect_tx(fb, tx);
          const uint32_t a_dst = tiles_base + stage * stage_bytes;
          const int kbb = kb >= p.n_kb ? kb - p.n_kb : kb;       // hi and lo halves share B
          if constexpr (BANDED) {   // this band's channels of A (no multicast: cn == 1)
            tma_load_4d(a_dst, &tmA, fb, nn0 + kb * p.KB, dw, h0 * p.in_step + dh, n0);
          } else {
            if (p.cn == 1) tma_load_4d(a_dst, &tmA, fb, kb * p.KB, dw, h0 * p.in_step + dh, n0);
            else if (it % p.cn == ry) tma_load_4d_mc(a_dst, &tmA, fb, kb * p.KB, dw, h0 * p.in_step + dh, n0, a_mask);
          }
          if (p.cm == 1) tma_load_2d(a_dst + a_bytes, &tmB, fb, tb * p.Kc + kbb * p.KB, nn0);
          else if (it % p.cm == rx) tma_load_2d_mc(a_dst + a_bytes, &tmB, fb, tb * p.Kc + kbb * p.KB, nn0, b_mask);
        }
      }
    }
  } else {
    const int wg = warp >> 2, wq = warp & 3;
    float acc[NW / 2];
#pragma unroll
    for (int i = 0; i < NW / 2; ++i) acc[i] = 0.f;
    for (int it = 0; it < n_iters; ++it) {
      const int stage = it % p.stages;
      mbar_wait(smem_u32(&full_bar[stage]), uint32_t(it / p.stages) & 1u);
      const uint32_t a_src = tiles_base + stage * stage_bytes + uint32_t(wg * 64 * p.row_bytes);
      const uint32_t b_src = tiles_base + stage * stage_bytes + a_bytes;
      if (p.row_bytes == 128) wgmma_k_block<NW, KIND, 4>(acc, a_src, b_src);
      else if (p.row_bytes == 64) wgmma_k_block<NW, KIND, 2>(acc, a_src, b_src);
      else wgmma_k_block<NW, KIND, 1>(acc, a_src, b_src);
      wgmma_commit();
      wgmma_wait<1>();
      if (it > 0 && (threadIdx.x & 127) == 0) {
        const uint32_t eb = smem_u32(&empty_bar[(it - 1) % p.stages]);
        if (cs == 1) mbar_arrive(eb);
        else
          for (int r = 0; r < cs; ++r) mbar_arrive_cluster(eb, uint32_t(r));
      }
    }
    wgmma_wait<0>();
    wgmma_fence_regs(acc);

    // ---- epilogue: this thread holds rows r and r + 8 (r = 64 wg + 16 wq + lane/4), column pairs 8j + 2(lane%4) ----
    const float post = (MODE != 0 && p.amax_bits) ? amax_pow2_scale(__ldg(p.amax_bits), true) : 1.0f;
    uint32_t zmax = 0u;                     // MODE 2: bits of this thread's max|z| (ordered as integers, NaN on top)
    const int mask_words = (p.Nout + 31) >> 5;
    int64_t pix[2];
    int32_t rpix[2];                        // PADRES residual pixel (32 bits, plan_tc_conv checks: keeps 96 registers)
    bool valid[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int m = wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
      const int wi = m % p.BW;
      const int q = m / p.BW;
      const int hi = q % p.BH, ni = q / p.BH;
      const int oh = (h0 + hi) * p.out_step + p.out_off_h, ow = wi * p.out_step + p.out_off_w;
      valid[h] = (ni < p.BNI) && (h0 + hi < p.OH) && (n0 + ni < p.NIMG) && oh < p.OHf && ow < p.OWf;
      pix[h] = (int64_t(n0 + ni) * p.OHf + oh) * p.OWf + ow;
      if (PADRES) rpix[h] = ((n0 + ni) * p.res_H + 2 * oh) * p.res_W + 2 * ow;
    }
#pragma unroll
    for (int j = 0; j < NW / 8; ++j) {
      // dgrad: `add` may alias `out`, so each pair's load of `add` waits for the previous pair's store.  Prefetching
      // the next 64 columns' `add` lines into L2 first turns that chain of HBM round trips into L2 hits (no
      // registers held).
      if (MODE == 1 && j % 8 == 0 && p.add != nullptr) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!valid[h]) continue;
          const float* row = p.add + pix[h] * p.Nout + nn0 + 8 * j;
#pragma unroll
          for (int f = 0; f < (NW < 64 ? NW : 64); f += 32) asm volatile("prefetch.global.L2 [%0];" ::"l"(row + f));
        }
      }
      const int col = 8 * j + 2 * (lane & 3);
      const int ch = nn0 + col;
      float a0 = 1.f, a1 = 1.f, sa0 = 0.f, sa1 = 0.f, sb0 = 0.f, sb1 = 0.f;
      if (MODE != 1) {
        a0 = __ldg(p.alpha + ch); a1 = __ldg(p.alpha + ch + 1);
        if (MODE == 2) { sb0 = __ldg(p.shift + ch); sb1 = __ldg(p.shift + ch + 1); }
      } else if (do_stats) {               // yhat = y_int * alpha * invstd - mean * invstd of the producing unit
        const float is0 = __ldg(p.st_invstd + ch), is1 = __ldg(p.st_invstd + ch + 1);
        sa0 = __ldg(p.st_alpha + ch) * is0; sa1 = __ldg(p.st_alpha + ch + 1) * is1;
        sb0 = __ldg(p.st_mean + ch) * is0; sb1 = __ldg(p.st_mean + ch + 1) * is1;
      }
      float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f, m0 = 0.f, m1 = 0.f;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        if (!valid[h]) continue;
        const float v0 = acc[4 * j + 2 * h], v1 = acc[4 * j + 2 * h + 1];
        const int64_t off = pix[h] * p.Nout + ch;
        float o0, o1;
        if (MODE == 0) {
          o0 = v0 * a0; o1 = v1 * a1;
          if (p.out_i16 != nullptr)        // exact: |v| <= taps * Kc <= 32767
            *reinterpret_cast<uint32_t*>(p.out_i16 + off) = (uint32_t(int(v0)) & 0xffffu) | (uint32_t(int(v1)) << 16);
          else
            *reinterpret_cast<float2*>(p.out + off) = make_float2(o0, o1);
        } else if (MODE == 2) {
          // one rounding per step, no FMA contraction: the CPU reference (oracle/eval_ref.py) matches bit for bit.
          // post = 2^-ex of real-valued operands (exact), 1 for the +-1 operands.
          o0 = __fadd_rn(__fmul_rn(__fmul_rn(v0, post), a0), sb0);
          o1 = __fadd_rn(__fmul_rn(__fmul_rn(v1, post), a1), sb1);
          if (PADRES) {
            // outside the channel band the residual is +0.0 and is still added: -0.0 + 0.0 = +0.0, as the
            // materialised zero-padded tensor gives (ch and the band edges are even, so a pair is in or out)
            float2 r = make_float2(0.f, 0.f);
            const int rc = ch - p.res_coff;
            if (unsigned(rc) < unsigned(p.res_C))
              r = __ldg(reinterpret_cast<const float2*>(p.add + int64_t(rpix[h]) * p.res_C + rc));
            o0 = __fadd_rn(o0, r.x); o1 = __fadd_rn(o1, r.y);
          } else if (p.add != nullptr) {   // the residual never aliases z (the entry points reject it)
            const float2 r = __ldg(reinterpret_cast<const float2*>(p.add + off));
            o0 = __fadd_rn(o0, r.x); o1 = __fadd_rn(o1, r.y);
          }
          if (HARDTANH) {                  // torch.nn.Hardtanh: NaN stays NaN, -0.0 stays -0.0
            o0 = o0 < -1.f ? -1.f : (o0 > 1.f ? 1.f : o0);
            o1 = o1 < -1.f ? -1.f : (o1 > 1.f ? 1.f : o1);
          } else if (p.relu) {             // torch.relu: NaN stays NaN (fmaxf alone would drop it)
            o0 = o0 != o0 ? o0 : fmaxf(o0, 0.f);
            o1 = o1 != o1 ? o1 : fmaxf(o1, 0.f);
          }
          *reinterpret_cast<float2*>(p.out + off) = make_float2(o0, o1);
          zmax = max(zmax, max(__float_as_uint(fabsf(o0)), __float_as_uint(fabsf(o1))));
          // sign(v) = +1 iff v >= 0 (DESIGN.md §2): -0.0 -> +1, NaN -> -1
          if (p.zb != nullptr)
            *reinterpret_cast<uint32_t*>(p.zb + off) =
                (o0 >= 0.f ? p.zb_one : p.zb_one | 0x8000u) | ((o1 >= 0.f ? p.zb_one : p.zb_one | 0x8000u) << 16);
          if (p.zb8 != nullptr)
            *reinterpret_cast<uint16_t*>(p.zb8 + off) = uint16_t((o0 >= 0.f ? 0x38u : 0xB8u) |
                                                                 ((o1 >= 0.f ? 0x38u : 0xB8u) << 8));
        } else {
          const uint32_t word = __ldg(p.mask + pix[h] * mask_words + (ch >> 5)) >> (ch & 31);
          o0 = (word & 1u) ? v0 * post : 0.0f;
          o1 = (word & 2u) ? v1 * post : 0.0f;
          if (p.add != nullptr) {          // plain load: add may alias out
            const float2 ad = *reinterpret_cast<const float2*>(p.add + off);
            o0 += ad.x; o1 += ad.y;
          }
          *reinterpret_cast<float2*>(p.out + off) = make_float2(o0, o1);
        }
        if (do_stats) {
          s0 += o0; s1 += o1;
          if (MODE == 1) {
            const uint32_t yr = __ldg(reinterpret_cast<const uint32_t*>(p.st_y + off));
            q0 += o0 * fmaf(float(int16_t(yr & 0xffffu)), sa0, -sb0);
            q1 += o1 * fmaf(float(int16_t(yr >> 16)), sa1, -sb1);
          } else {
            q0 += o0 * o0; q1 += o1 * o1;
          }
          m0 = fmaxf(m0, fabsf(o0)); m1 = fmaxf(m1, fabsf(o1));
        }
      }
      if (do_stats) {
        // lanes with the same lane % 4 hold the same two channels for different rows
#pragma unroll
        for (int d = 4; d <= 16; d <<= 1) {
          s0 += __shfl_xor_sync(0xffffffffu, s0, d); s1 += __shfl_xor_sync(0xffffffffu, s1, d);
          q0 += __shfl_xor_sync(0xffffffffu, q0, d); q1 += __shfl_xor_sync(0xffffffffu, q1, d);
          m0 = fmaxf(m0, __shfl_xor_sync(0xffffffffu, m0, d)); m1 = fmaxf(m1, __shfl_xor_sync(0xffffffffu, m1, d));
        }
        if (lane < 4) {            // each warp owns distinct rows: one writer per (warp, channel)
          stat_sum[warp][col] = s0; stat_sum[warp][col + 1] = s1;
          stat_sq[warp][col] = q0; stat_sq[warp][col + 1] = q1;
          stat_max[warp][col] = m0; stat_max[warp][col + 1] = m1;
        }
      }
    }
    if (MODE == 2 && p.z_amax != nullptr) {   // max is order-free: the same bits every run
      zmax = __reduce_max_sync(0xffffffffu, zmax);
      if (lane == 0 && zmax != 0u) atomicMax(p.z_amax, zmax);
    }
  }
  if (do_stats) {
    __syncthreads();
    // this CTA's row of the statistics partials (summed over CTAs in a fixed order after the kernel)
    double* row = p.stat_part + int64_t(blockIdx.x) * 2 * p.Nout;
    for (int i = threadIdx.x; i < p.BN; i += blockDim.x) {
      double su = 0.0, sq = 0.0;
      float mx = 0.f;
      for (int w = 0; w < kTcThreads / 32 - 1; ++w) {
        su += double(stat_sum[w][i]); sq += double(stat_sq[w][i]); mx = fmaxf(mx, stat_max[w][i]);
      }
      row[nn0 + i] = su;
      row[p.Nout + nn0 + i] = sq;
      atomicMax(p.bn_ymax + nn0 + i, __float_as_uint(mx));
    }
  }
  if (cs > 1) cluster_sync();   // no CTA exits while a peer may still multicast into it or arrive on its barriers
}

static bool chan_ok(int c) { return c == 16 || c == 32 || c == 64 || (c >= 128 && c % 128 == 0); }
static int pick_bn(int n) { return n >= 128 ? 128 : n; }   // n in {16,32,64} or multiple of 128

static bool tc_shape_ok(const bdbnn_conv_shape* s) {
  if (!s || (s->stride != 1 && s->stride != 2)) return false;
  if (!chan_ok(s->Cin) || !chan_ok(s->Cout)) return false;   // K blocks of 16/32/64, N tiles <= 128
  if (s->Wo > 128 || s->W > 128 * s->stride || s->W < 1) return false;
  if (s->kh != s->kw || s->kh > 7) return false;
  if (s->pad > s->kh - 1) return false;
  return true;
}

// GEMMs whose contraction is a whole number of 64-channel K blocks (stem windows: 32 halves) and whose N is 64 or a
// multiple of 128: the launches that may ask for the int16 result or for the dgrad's BatchNorm statistics.
static bool wide_gemm(const TcConvLaunch& L) {
  if (L.n_taps <= 0) return false;
  if (L.win ? (L.Kc != 32 || L.fmt < 0) : (L.Kc % 64 != 0)) return false;
  return L.Nout == 64 || L.Nout % 128 == 0;
}

// BDBNN_TC_CLUSTER=1: launch clusters that multicast the shared operand boxes.  Off by default: on an H100 the
// ResNet-18 step's conv kernels ran 1.7-2x slower with them (DESIGN.md §7), every CTA of a cluster waiting for the
// slowest one before a ring slot is refilled.
static bool tc_cluster_enabled() {
  const char* e = getenv("BDBNN_TC_CLUSTER");
  return e && strcmp(e, "1") == 0;
}

// Tiling of one launch; returns false when the launch asks for something this kernel cannot give.
static bool plan_tc_conv(const TcConvLaunch& L, int mode, TcConvParams* pp, size_t* smem_out, int* tiles_out) {
  if (L.n_taps <= 0 || L.OW > kTileM) return false;
  if ((L.out_i16 || (mode == 1 && L.bn_sums)) && !wide_gemm(L)) return false;
  if (L.out_i16 && (mode != 0 || L.n_taps * L.Kc * L.a_halves > 32767)) return false;
  if (mode == 1 && L.bn_sums && !(L.st_y && L.st_alpha && L.st_mean && L.st_invstd && L.out_step == 1)) return false;
  TcConvParams& p = *pp;
  memset(&p, 0, sizeof(p));
  const int esize = L.fmt < 0 ? 1 : 2;
  p.OW = L.OW; p.OH = L.OH; p.NIMG = L.NIMG;
  p.BW = L.OW;
  if (L.OH * L.OW <= kTileM) {
    p.BH = L.OH;
    p.BNI = kTileM / (L.OH * L.OW);
    if (p.BNI > L.NIMG) p.BNI = L.NIMG;
    if (p.BNI > 256) p.BNI = 256;
  } else {
    p.BH = kTileM / L.OW;
    p.BNI = 1;
  }
  p.tiles_h = (L.OH + p.BH - 1) / p.BH;
  p.Kc = L.Kc;
  p.KB = L.Kc * esize >= 128 ? 128 / esize : L.Kc;
  if (L.Kc % p.KB != 0) return false;
  p.n_kb = L.Kc / p.KB;
  p.a_halves = L.a_halves;
  p.in_step = L.in_step;
  p.row_bytes = p.KB * esize;
  p.n_taps = L.n_taps;
  memcpy(p.tap_dh, L.dh, sizeof(p.tap_dh));
  memcpy(p.tap_dw, L.dw, sizeof(p.tap_dw));
  memcpy(p.tap_b, L.tb, sizeof(p.tap_b));
  p.out_step = L.out_step; p.out_off_h = L.off_h; p.out_off_w = L.off_w; p.OHf = L.OHf; p.OWf = L.OWf;
  p.Nout = L.Nout;
  p.BN = pick_bn(L.Nout);
  if (L.fmt < 0 && p.BN < 64) return false;
  if (L.band) {   // one band per N tile: Kc = B channels of A starting at the tile's first output channel
    if (L.band != L.Kc || L.Nout % L.band != 0 || L.fmt != BDBNN_FMT_FP16 || L.a_halves != 1 || L.pad_res ||
        L.hardtanh || L.out_i16 || (mode == 1 && L.bn_sums) || L.win)
      return false;
    p.BN = L.band;
  }
  p.alpha = L.alpha; p.mask = L.mask; p.out = L.out; p.out_i16 = mode == 0 ? L.out_i16 : nullptr;
  p.shift = L.shift; p.zb = L.zb; p.zb8 = L.zb8; p.zb_one = L.fmt == BDBNN_FMT_BF16 ? 0x3F80u : 0x3C00u;
  p.amax_bits = L.amax_bits; p.add = L.add; p.relu = L.relu; p.z_amax = L.z_amax;
  if (L.pad_res) {
    if (mode != 2 || L.fmt < 0 || !L.add) return false;
    if (int64_t(L.NIMG) * L.res_H * L.res_W > INT32_MAX) return false;   // rpix is 32 bits
    p.res_H = L.res_H; p.res_W = L.res_W; p.res_C = L.res_C; p.res_coff = L.res_coff;
  }
  p.bn_sums = L.bn_sums; p.bn_ymax = L.bn_ymax;
  p.st_y = L.st_y; p.st_alpha = L.st_alpha; p.st_mean = L.st_mean; p.st_invstd = L.st_invstd;
  const uint32_t stage_bytes = (uint32_t(kTileM + p.BN) * p.row_bytes + 1023u) & ~1023u;
  const int n_iters = p.n_taps * p.n_kb * p.a_halves;
  // a 96 KB ring leaves room for two CTAs per SM
  int stages = int((96u * 1024u) / stage_bytes);
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages > n_iters) stages = n_iters;
  if (stages < 2) stages = 2;
  p.stages = stages;
  *smem_out = size_t(stages) * stage_bytes + 1024;
  *tiles_out = p.tiles_h * ((L.NIMG + p.BNI - 1) / p.BNI);
  // clusters of 2 neighbouring M tiles share the weight box, and of 2 N tiles (256 channels and up) the activation
  // box; a grid side that does not divide keeps cluster size 1 there (the grid is never padded)
  p.cm = p.cn = 1;
  if (tc_cluster_enabled()) {
    if (*tiles_out % 2 == 0) p.cm = 2;
    if ((L.Nout / p.BN) % 2 == 0 && !L.band) p.cn = 2;   // the bands of a row read different activation boxes
  }
  return true;
}

template <typename K>
static int launch_one(K kern, dim3 grid, size_t smem, cudaStream_t st, const CUtensorMap& tmA, const CUtensorMap& tmB,
                      const TcConvParams& p) {
  if (p.cm * p.cn == 1) {
    kern<<<grid, kTcThreads, smem, st>>>(tmA, tmB, p);
    return check_launch("tc_conv_kernel");
  }
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid; cfg.blockDim = dim3(kTcThreads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeClusterDimension;
  attr[0].val.clusterDim.x = unsigned(p.cm); attr[0].val.clusterDim.y = unsigned(p.cn); attr[0].val.clusterDim.z = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  BDBNN_CUDA(cudaLaunchKernelEx(&cfg, kern, tmA, tmB, p));
  return check_launch("tc_conv_kernel");
}

// The instance for an N tile of bn columns (16, 32, 64 or 128).
using TcConvKernel = decltype(&tc_conv_kernel<0, 0, 16, false>);
// The banded instance for a band of bn channels (16, 32 or 64), fp16 operands.
template <int MODE>
static TcConvKernel banded_kernel_for(int bn) {
  return bn == 16 ? tc_conv_kernel<MODE, 0, 16, false, false, true>
         : bn == 32 ? tc_conv_kernel<MODE, 0, 32, false, false, true>
                    : tc_conv_kernel<MODE, 0, 64, false, false, true>;
}
template <int MODE, int KIND, bool PADRES = false, bool HARDTANH = false>
static TcConvKernel kernel_for(int bn) {
  return bn == 16   ? tc_conv_kernel<MODE, KIND, 16, PADRES, HARDTANH>
         : bn == 32 ? tc_conv_kernel<MODE, KIND, 32, PADRES, HARDTANH>
         : bn == 64 ? tc_conv_kernel<MODE, KIND, 64, PADRES, HARDTANH>
                    : tc_conv_kernel<MODE, KIND, 128, PADRES, HARDTANH>;
}

template <int MODE, int KIND, bool PADRES = false, bool HARDTANH = false, bool BANDED = false>
static int launch_kind(const CUtensorMap& tmA, const CUtensorMap& tmB, const TcConvParams& p, size_t smem, dim3 grid,
                       cudaStream_t st) {
  const TcConvKernel kern = BANDED ? banded_kernel_for<MODE>(p.BN) : kernel_for<MODE, KIND, PADRES, HARDTANH>(p.BN);
  BDBNN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  if (p.bn_sums == nullptr) return launch_one(kern, grid, smem, st, tmA, tmB, p);
  TcConvParams q = p;
  int rc = det_sums_alloc(&q.stat_part, grid.x, 2 * p.Nout, st);
  if (rc) return rc;
  rc = launch_one(kern, grid, smem, st, tmA, tmB, q);
  if (rc) { cudaFreeAsync(q.stat_part, st); return rc; }
  return det_sums_finish(q.stat_part, grid.x, 2 * p.Nout, p.bn_sums, st);
}

template <int MODE>
static int launch_tc_conv(const TcConvLaunch& L, cudaStream_t st) {
  TcConvParams p;
  size_t smem = 0;
  int tiles = 0;
  if (!plan_tc_conv(L, MODE, &p, &smem, &tiles)) {
    set_error("tc_conv: launch geometry not supported");
    return BDBNN_ERR_UNSUPPORTED;
  }
  const int esize = L.fmt < 0 ? 1 : 2;
  CUtensorMap tmA, tmB;
  int rc;
  if (L.win)   // stem: overlapping windows, row step in_step, window step 1
    rc = make_window_map(&tmA, L.A, L.NIMG, L.IH, L.IW, p.KB, L.win_stride, L.win_row_stride, L.win_img_stride,
                         p.BW, p.BH, p.BNI, L.in_step);
  else
    rc = make_act_map(&tmA, L.A, L.NIMG, L.IH, L.IW, L.band ? L.a_chans : L.Kc * L.a_halves, p.KB, p.BW, p.BH, p.BNI,
                      L.in_step, esize);
  if (rc) return rc;
  rc = make_weight_map(&tmB, L.B, L.Nout, L.b_taps * L.Kc, p.KB, p.BN, esize);
  if (rc) return rc;
  const dim3 grid(unsigned(tiles), unsigned(L.Nout / p.BN));
  // forward statistics of the narrow (16/32-channel) GEMMs: one pass over the fp32 result after the kernel; the
  // banded GEMMs keep them in the epilogue (DESIGN.md §4t)
  const bool stats_pass = MODE == 0 && L.bn_sums != nullptr && !wide_gemm(L) && L.out != nullptr && !L.band;
  if (stats_pass) { p.bn_sums = nullptr; p.bn_ymax = nullptr; }
  if (L.band) return launch_kind<MODE, 0, false, false, true>(tmA, tmB, p, smem, grid, st);
  if (L.fmt < 0) {
    if constexpr (MODE == 1) {
      set_error("tc_conv: fp8 operands are forward only");
      return BDBNN_ERR_UNSUPPORTED;
    } else {
      return launch_kind<MODE, 2>(tmA, tmB, p, smem, grid, st);
    }
  }
  if constexpr (MODE == 2) {
    if (L.hardtanh) {
      if (L.pad_res || L.fmt != BDBNN_FMT_FP16) {
        set_error("tc_conv: the Hardtanh epilogue takes fp16 operands without the option-A residual");
        return BDBNN_ERR_UNSUPPORTED;
      }
      return launch_kind<2, 0, false, true>(tmA, tmB, p, smem, grid, st);
    }
    if (L.pad_res)
      return L.fmt == BDBNN_FMT_BF16 ? launch_kind<2, 1, true>(tmA, tmB, p, smem, grid, st)
                                     : launch_kind<2, 0, true>(tmA, tmB, p, smem, grid, st);
  }
  rc = L.fmt == BDBNN_FMT_BF16 ? launch_kind<MODE, 1>(tmA, tmB, p, smem, grid, st)
                               : launch_kind<MODE, 0>(tmA, tmB, p, smem, grid, st);
  if (rc || !stats_pass) return rc;
  return bn_stats_launch(L.out, int64_t(L.NIMG) * L.OHf * L.OWf, L.Nout, L.bn_sums, L.bn_ymax, st);
}

// Stem conv forward (7x7 / stride 2 / pad 3 on 3 channels) as a 7-tap implicit GEMM over the packed
// window view: tap r reads window row 2*oh + r, K = 32 values (8 pixels x 4 halves) per tap.
static void stem_launch(TcConvLaunch* Lp, const uint16_t* xw, const uint16_t* wf, const float* alpha, float* y,
                        const StemGeom& g) {
  TcConvLaunch& L = *Lp;
  memset(&L, 0, sizeof(L));
  L.A = xw; L.IH = g.HP; L.IW = g.Wo; L.Kc = kStemWin; L.a_halves = 1; L.in_step = 2;
  L.win = 1; L.win_stride = g.win_stride; L.win_row_stride = g.row_stride; L.win_img_stride = g.img_stride;
  L.B = wf; L.b_taps = kStemTaps; L.Nout = kStemCout;
  L.NIMG = g.N; L.OH = g.Ho; L.OW = g.Wo;
  for (int r = 0; r < kStemTaps; ++r) { L.dh[r] = int8_t(r); L.dw[r] = 0; L.tb[r] = uint8_t(r); }
  L.n_taps = kStemTaps;
  L.out_step = 1; L.OHf = g.Ho; L.OWf = g.Wo;
  L.alpha = alpha; L.out = y; L.fmt = BDBNN_FMT_FP16;
}

int launch_stem_fwd(const uint16_t* xw, const uint16_t* wf, const float* alpha, float* y, const StemGeom& g,
                    double* bn_sums, uint32_t* bn_ymax, cudaStream_t st) {
  TcConvLaunch L;
  stem_launch(&L, xw, wf, alpha, y, g);
  L.bn_sums = bn_sums; L.bn_ymax = bn_ymax;
  int rc = bn_stats_zero(bn_sums, bn_ymax, kStemCout, st);
  if (rc) return rc;
  return launch_tc_conv<0>(L, st);
}

// The same GEMM with the eval epilogue: z = acc * scale + shift (the folded eval-mode BatchNorm), no +-1 copy;
// optionally z = relu(z) and max|z| into z_amax (zeroed here).
int launch_stem_eval(const uint16_t* xw, const uint16_t* wf, const float* scale, const float* shift, float* z,
                     const StemGeom& g, int relu, uint32_t* z_amax, cudaStream_t st) {
  TcConvLaunch L;
  stem_launch(&L, xw, wf, scale, z, g);
  L.shift = shift; L.relu = relu; L.z_amax = z_amax;
  if (z_amax) BDBNN_CUDA(cudaMemsetAsync(z_amax, 0, sizeof(uint32_t), st));
  return launch_tc_conv<2>(L, st);
}

static long long* g_trace = nullptr;
void set_tc_trace(long long* buf) { g_trace = buf; }
long long* get_tc_trace() { return g_trace; }

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_debug_trace(long long* device_buf) {
  set_tc_trace(device_buf);
  return BDBNN_OK;
}

// Host-only: the kernel's tiling for the forward (mode 0: 16-bit operands, 2: fp8), the first dgrad phase
// (mode 1) or the eval forward (mode 3: 16-bit operands, 4: fp8) of a shape.  out[12] = {planned, halo, TS, NB, BN,
// n_tiles, supers, stages, dynamic smem, grid, stage bytes, patch bytes}; halo = 0, TS = NB = 1 (one 128-row tile
// per CTA, no patch), supers = M tiles.  With n_out >= 14 also out[12..13] = cluster CTAs along M and along N
// (BDBNN_TC_CLUSTER applies).  planned = 0 when the GEMM is not eligible for the int16 result / fused dgrad
// statistics (modes 0-2) or when the eval kernel cannot run the shape (modes 3-4).  No CUDA call.
extern "C" int bdbnn_debug_conv_plan(const bdbnn_conv_shape* s, int32_t mode, int32_t grad_halves, int32_t* out,
                                     int32_t n_out) {
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(out && n_out >= 12 && mode >= 0 && mode <= 4 && (grad_halves == 1 || grad_halves == 2),
                "debug_conv_plan: bad arguments");
  memset(out, 0, size_t(n_out >= 14 ? 14 : 12) * sizeof(int32_t));
  if (!tc_shape_ok(s)) return BDBNN_OK;
  TcConvLaunch L;
  memset(&L, 0, sizeof(L));
  const int T = s->kh * s->kw;
  if (mode == 1) {
    const int sd = s->stride;            // phase (0,0) of the stride decomposition
    for (int r = 0; r < s->kh; ++r) {
      if ((s->pad - r) % sd != 0) continue;
      for (int q = 0; q < s->kw; ++q) {
        if ((s->pad - q) % sd != 0) continue;
        L.dh[L.n_taps] = int8_t((s->pad - r) / sd); L.dw[L.n_taps] = int8_t((s->pad - q) / sd);
        L.tb[L.n_taps] = uint8_t(T - 1 - (r * s->kw + q));
        ++L.n_taps;
      }
    }
    L.OH = (s->H + sd - 1) / sd; L.OW = (s->W + sd - 1) / sd;
    L.IH = s->Ho; L.IW = s->Wo; L.Kc = s->Cout; L.a_halves = grad_halves; L.in_step = 1;
    L.b_taps = T; L.Nout = s->Cin; L.NIMG = s->N;
    L.out_step = sd; L.OHf = s->H; L.OWf = s->W;
    L.fmt = grad_halves == 1 ? BDBNN_FMT_FP16 : BDBNN_FMT_BF16;
  } else {
    L.IH = s->H; L.IW = s->W; L.Kc = s->Cin; L.a_halves = 1; L.in_step = s->stride;
    L.b_taps = T; L.Nout = s->Cout; L.NIMG = s->N; L.OH = s->Ho; L.OW = s->Wo;
    for (int r = 0; r < s->kh; ++r)
      for (int q = 0; q < s->kw; ++q) {
        const int t = r * s->kw + q;
        L.dh[t] = int8_t(r - s->pad); L.dw[t] = int8_t(q - s->pad); L.tb[t] = uint8_t(t);
      }
    L.n_taps = T;
    L.out_step = 1; L.OHf = s->Ho; L.OWf = s->Wo;
    L.fmt = (mode == 2 || mode == 4) ? -1 : BDBNN_FMT_FP16;
    if (L.fmt == -1 && s->Cin % 128 != 0) return BDBNN_OK;
  }
  if (L.n_taps == 0 || (mode <= 2 && !wide_gemm(L))) return BDBNN_OK;
  TcConvParams p;
  size_t smem = 0;
  int tiles = 0;
  if (!plan_tc_conv(L, mode == 1 ? 1 : (mode <= 2 ? 0 : 2), &p, &smem, &tiles)) return BDBNN_OK;
  const int32_t v[14] = {1, 0, 1, 1, p.BN, L.Nout / p.BN, tiles, p.stages, int32_t(smem), tiles * (L.Nout / p.BN),
                         int32_t((uint32_t(kTileM + p.BN) * p.row_bytes + 1023u) & ~1023u), 0, p.cm, p.cn};
  memcpy(out, v, size_t(n_out >= 14 ? 14 : 12) * sizeof(int32_t));
  return BDBNN_OK;
}

// CTAs of one tc_conv_kernel instance that fit on an SM with `smem` bytes of dynamic shared memory (the dynamic smem
// entry of bdbnn_debug_conv_plan).  mode 0 forward / 1 dgrad / 2 eval forward / 3 eval forward with the option-A
// residual / 5 eval forward with the Hardtanh epilogue (4 is not a mode), fmt BDBNN_FMT_FP16 / BF16 or -1 (fp8,
// forward and dense eval only; mode 5 takes fp16 only), bn = N tile (16, 32, 64 or 128).
extern "C" int bdbnn_debug_tc_conv_ctas_per_sm(int32_t mode, int32_t fmt, int32_t bn, int32_t smem, int32_t* ctas) {
  BDBNN_REQUIRE(ctas && ((mode >= 0 && mode <= 3) || mode == 5) && (bn == 16 || bn == 32 || bn == 64 || bn == 128) &&
                    smem >= 0 &&
                    (fmt == BDBNN_FMT_FP16 || fmt == BDBNN_FMT_BF16 || (fmt == -1 && (mode == 0 || mode == 2))) &&
                    (mode != 5 || fmt == BDBNN_FMT_FP16),
                "debug_tc_conv_ctas_per_sm: bad arguments");
  const int kind = fmt == -1 ? 2 : (fmt == BDBNN_FMT_BF16 ? 1 : 0);
  TcConvKernel kern;
  if (mode == 5) kern = kernel_for<2, 0, false, true>(bn);
  else if (mode == 3) kern = kind == 0 ? kernel_for<2, 0, true>(bn) : kernel_for<2, 1, true>(bn);
  else if (mode == 2) kern = kind == 2 ? kernel_for<2, 2>(bn) : kind == 0 ? kernel_for<2, 0>(bn) : kernel_for<2, 1>(bn);
  else if (mode == 0) kern = kind == 2 ? kernel_for<0, 2>(bn) : kind == 0 ? kernel_for<0, 0>(bn) : kernel_for<0, 1>(bn);
  else kern = kind == 0 ? kernel_for<1, 0>(bn) : kernel_for<1, 1>(bn);
  BDBNN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
  int n = 0;
  BDBNN_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, kern, kTcThreads, size_t(smem)));
  *ctas = n;
  return BDBNN_OK;
}

extern "C" int bdbnn_tc_supported(const bdbnn_conv_shape* s) {
  if (!tc_shape_ok(s)) return 0;
  // fp8 forward only with 128-byte K rows (Cin % 128 == 0)
  const bool v2 = s->Cin % 128 == 0 && (s->Cout == 64 || s->Cout % 128 == 0);
  // int16 forward output: the forward GEMM must be eligible (bdbnn_debug_conv_plan) and the integer result
  // must fit (|y_int| <= kh*kw*Cin)
  bool i16 = s->kh * s->kw * s->Cin <= 32767 && s->Cout <= 512;
  if (i16) {
    int32_t plan[12] = {0};
    i16 = bdbnn_debug_conv_plan(s, 0, 1, plan, 12) == BDBNN_OK && plan[0] == 1;
    if (i16 && v2) i16 = bdbnn_debug_conv_plan(s, 2, 1, plan, 12) == BDBNN_OK && plan[0] == 1;   // fp8 forward
  }
  return BDBNN_TC_FWD | BDBNN_TC_DGRAD | (wgrad_tc_ok(s) ? BDBNN_TC_WGRAD : 0) | (v2 ? BDBNN_TC_FWD8 : 0) |
         (i16 ? BDBNN_TC_FWD_I16 : 0) | (b1_shape_ok(s) ? BDBNN_TC_B1 : 0);
}

// The implicit GEMM of a forward conv: A = the +-1 activations (NHWC, fmt), B = the +-1 weights [Cout][T][Cin].
static void fwd_launch(TcConvLaunch* Lp, const void* xb, const void* wf, int fmt, const bdbnn_conv_shape* s) {
  TcConvLaunch& L = *Lp;
  memset(&L, 0, sizeof(L));
  L.A = static_cast<const uint16_t*>(xb); L.IH = s->H; L.IW = s->W; L.Kc = s->Cin; L.a_halves = 1; L.in_step = s->stride;
  L.B = static_cast<const uint16_t*>(wf); L.b_taps = s->kh * s->kw; L.Nout = s->Cout;
  L.NIMG = s->N; L.OH = s->Ho; L.OW = s->Wo;
  for (int r = 0; r < s->kh; ++r)
    for (int q = 0; q < s->kw; ++q) {
      const int t = r * s->kw + q;
      L.dh[t] = int8_t(r - s->pad); L.dw[t] = int8_t(q - s->pad); L.tb[t] = uint8_t(t);
    }
  L.n_taps = s->kh * s->kw;
  L.out_step = 1; L.OHf = s->Ho; L.OWf = s->Wo;
  L.fmt = fmt;
}

// Forward with the result stored as the exact integer accumulator (int16) — see include/bdbnn.h.
extern "C" int bdbnn_binconv_fwd_tc_i16(const void* xb, const void* wf, int32_t fmt, const float* alpha,
                                        int16_t* y_int, const bdbnn_conv_shape* s, double* bn_sums,
                                        uint32_t* bn_ymax, void* stream) {
  BDBNN_REQUIRE(fmt == BDBNN_FMT_FP16 || fmt == BDBNN_FMT_BF16 || fmt == -1, "binconv_fwd_tc_i16: bad operand format");
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(xb && wf && alpha && y_int, "binconv_fwd_tc_i16: NULL pointer");
  if (!tc_shape_ok(s) || (fmt == -1 && s->Cin % 128 != 0) || s->kh * s->kw * s->Cin > 32767) {
    set_error("binconv_fwd_tc_i16: shape not supported");
    return BDBNN_ERR_UNSUPPORTED;
  }
  TcConvLaunch L;
  fwd_launch(&L, xb, wf, fmt, s);
  L.alpha = alpha; L.out = nullptr; L.out_i16 = y_int;
  BDBNN_REQUIRE((bn_sums == nullptr) == (bn_ymax == nullptr), "binconv_fwd_tc_i16: bn_sums and bn_ymax go together");
  BDBNN_REQUIRE(bn_sums == nullptr || s->Cout <= 512, "binconv_fwd_tc_i16: statistics need Cout <= 512");
  L.bn_sums = bn_sums; L.bn_ymax = bn_ymax;
  rc = bn_stats_zero(bn_sums, bn_ymax, s->Cout, cudaStream_t(stream));
  if (rc) return rc;
  return launch_tc_conv<0>(L, cudaStream_t(stream));
}

extern "C" int bdbnn_binconv_fwd_tc(const uint16_t* xb_bf16, const uint16_t* wf_bf16, int32_t fmt,
                                    const float* alpha, float* y, const bdbnn_conv_shape* s, double* bn_sums,
                                    uint32_t* bn_ymax, void* stream) {
  BDBNN_REQUIRE(fmt == BDBNN_FMT_FP16 || fmt == BDBNN_FMT_BF16, "binconv_fwd_tc: bad operand format");
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(xb_bf16 && wf_bf16 && alpha && y, "binconv_fwd_tc: NULL pointer");
  if (!tc_shape_ok(s)) { set_error("binconv_fwd_tc: shape not supported by the tensor-core path"); return BDBNN_ERR_UNSUPPORTED; }
  TcConvLaunch L;
  fwd_launch(&L, xb_bf16, wf_bf16, fmt, s);
  L.alpha = alpha; L.out = y;
  BDBNN_REQUIRE((bn_sums == nullptr) == (bn_ymax == nullptr), "binconv_fwd_tc: bn_sums and bn_ymax go together");
  L.bn_sums = bn_sums; L.bn_ymax = bn_ymax;
  rc = bn_stats_zero(bn_sums, bn_ymax, s->Cout, cudaStream_t(stream));
  if (rc) return rc;
  return launch_tc_conv<0>(L, cudaStream_t(stream));
}

extern "C" int bdbnn_binconv_fwd_tc8(const uint8_t* xb_fp8, const uint8_t* wf_fp8, const float* alpha, float* y,
                                     const bdbnn_conv_shape* s, double* bn_sums, uint32_t* bn_ymax,
                                     void* stream) {
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(xb_fp8 && wf_fp8 && alpha && y, "binconv_fwd_tc8: NULL pointer");
  if (!tc_shape_ok(s) || s->Cin % 128 != 0) {
    set_error("binconv_fwd_tc8: shape not supported by the fp8 tensor-core path");
    return BDBNN_ERR_UNSUPPORTED;
  }
  TcConvLaunch L;
  fwd_launch(&L, xb_fp8, wf_fp8, -1, s);
  L.alpha = alpha; L.out = y;
  BDBNN_REQUIRE((bn_sums == nullptr) == (bn_ymax == nullptr), "binconv_fwd_tc8: bn_sums and bn_ymax go together");
  BDBNN_REQUIRE(bn_sums == nullptr || s->Cout <= 512, "binconv_fwd_tc8: statistics need Cout <= 512");
  L.bn_sums = bn_sums; L.bn_ymax = bn_ymax;
  rc = bn_stats_zero(bn_sums, bn_ymax, s->Cout, cudaStream_t(stream));
  if (rc) return rc;
  return launch_tc_conv<0>(L, cudaStream_t(stream));
}

// Eval-mode forward: z = alpha-folded BatchNorm of the conv (+ residual) and its +-1 copy — see include/bdbnn.h.
extern "C" int bdbnn_binconv_fwd_tc_eval(const void* xb, const void* wf, int32_t fmt, const float* scale,
                                         const float* shift, const float* residual, float* z, uint16_t* zb,
                                         uint8_t* zb8, const bdbnn_conv_shape* s, void* stream) {
  BDBNN_REQUIRE(fmt == BDBNN_FMT_FP16 || fmt == BDBNN_FMT_BF16 || fmt == -1, "binconv_fwd_tc_eval: bad operand format");
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(xb && wf && scale && shift && z, "binconv_fwd_tc_eval: NULL pointer");
  BDBNN_REQUIRE(residual != z, "binconv_fwd_tc_eval: residual must not alias z");
  BDBNN_REQUIRE(fmt != -1 || zb == nullptr, "binconv_fwd_tc_eval: the 16-bit copy needs 16-bit operands");
  if (!tc_shape_ok(s) || (fmt == -1 && s->Cin % 128 != 0)) {
    set_error("binconv_fwd_tc_eval: shape not supported by the tensor-core path");
    return BDBNN_ERR_UNSUPPORTED;
  }
  TcConvLaunch L;
  fwd_launch(&L, xb, wf, fmt, s);
  L.alpha = scale; L.shift = shift; L.add = residual; L.out = z; L.zb = zb; L.zb8 = zb8;
  return launch_tc_conv<2>(L, cudaStream_t(stream));
}

// Eval-mode forward of a real-valued conv on fp16 operands (xh = fp16(x * 2^ex), wf = fp16(W * 2^ew)) — see
// include/bdbnn.h.
extern "C" int bdbnn_real_conv_fwd_eval(const uint16_t* xh, const uint32_t* x_amax_bits, const uint16_t* wf,
                                        const float* scale, const float* shift, const float* residual, int32_t act,
                                        float* z, uint32_t* z_amax_bits, const bdbnn_conv_shape* s, void* stream) {
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(xh && x_amax_bits && wf && scale && shift && z, "real_conv_fwd_eval: NULL pointer");
  BDBNN_REQUIRE(act >= BDBNN_ACT_NONE && act <= BDBNN_ACT_HARDTANH,
                "real_conv_fwd_eval: act must be 0 (none), 1 (ReLU) or 2 (Hardtanh), got %d", act);
  BDBNN_REQUIRE(residual != z, "real_conv_fwd_eval: residual must not alias z");
  if (!tc_shape_ok(s)) {
    set_error("real_conv_fwd_eval: shape not supported by the tensor-core path");
    return BDBNN_ERR_UNSUPPORTED;
  }
  cudaStream_t st = cudaStream_t(stream);
  TcConvLaunch L;
  fwd_launch(&L, xh, wf, BDBNN_FMT_FP16, s);
  L.amax_bits = x_amax_bits;
  L.alpha = scale; L.shift = shift; L.add = residual; L.out = z; L.z_amax = z_amax_bits;
  L.relu = act == BDBNN_ACT_RELU; L.hardtanh = act == BDBNN_ACT_HARDTANH;
  if (z_amax_bits) BDBNN_CUDA(cudaMemsetAsync(z_amax_bits, 0, sizeof(uint32_t), st));
  return launch_tc_conv<2>(L, st);
}

// The option-A shortcut of a stride-2 conv as the eval epilogue's residual, read in place from x_res (NHWC fp32
// [N][H_res][W_res][C_res]): r[n,i,j,c] = x_res[n,2i,2j,c-pad] for pad <= c < pad + C_res, else +0.0.
static int pad_residual(TcConvLaunch* L, const float* x_res, int32_t H_res, int32_t W_res, int32_t C_res, int32_t pad,
                        const float* z, const bdbnn_conv_shape* s) {
  BDBNN_REQUIRE(x_res != nullptr, "pad_shortcut: NULL x_res");
  BDBNN_REQUIRE(x_res != z, "pad_shortcut: x_res must not alias z");
  BDBNN_REQUIRE((uintptr_t(x_res) & 15) == 0, "pad_shortcut: x_res must be 16-byte aligned");
  BDBNN_REQUIRE(H_res > 0 && W_res > 0 && C_res > 0 && pad >= 0, "pad_shortcut: non-positive x_res dims or pad < 0");
  BDBNN_REQUIRE(C_res % 4 == 0 && pad % 4 == 0, "pad_shortcut: C_res and pad must be multiples of 4");
  BDBNN_REQUIRE(s->Cout == C_res + 2 * pad, "pad_shortcut: Cout %d != C_res + 2 * pad = %d", s->Cout, C_res + 2 * pad);
  BDBNN_REQUIRE(s->stride == 2 && s->Ho == (H_res + 1) / 2 && s->Wo == (W_res + 1) / 2,
                "pad_shortcut: needs a stride-2 conv with Ho = ceil(H_res / 2), Wo = ceil(W_res / 2)");
  L->add = x_res;
  L->pad_res = 1; L->res_H = H_res; L->res_W = W_res; L->res_C = C_res; L->res_coff = pad;
  return BDBNN_OK;
}

extern "C" int bdbnn_binconv_fwd_tc_eval_pad_shortcut(const void* xb, const void* wf, int32_t fmt, const float* scale,
                                                      const float* shift, const float* x_res, int32_t H_res,
                                                      int32_t W_res, int32_t C_res, int32_t pad, float* z,
                                                      uint16_t* zb, uint8_t* zb8, const bdbnn_conv_shape* s,
                                                      void* stream) {
  BDBNN_REQUIRE(fmt == BDBNN_FMT_FP16 || fmt == BDBNN_FMT_BF16,
                "binconv_fwd_tc_eval_pad_shortcut: needs 16-bit operands (BDBNN_FMT_FP16 / BF16)");
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(xb && wf && scale && shift && z, "binconv_fwd_tc_eval_pad_shortcut: NULL pointer");
  TcConvLaunch L;
  fwd_launch(&L, xb, wf, fmt, s);
  rc = pad_residual(&L, x_res, H_res, W_res, C_res, pad, z, s);
  if (rc) return rc;
  if (!tc_shape_ok(s)) {
    set_error("binconv_fwd_tc_eval_pad_shortcut: shape not supported by the tensor-core path");
    return BDBNN_ERR_UNSUPPORTED;
  }
  L.alpha = scale; L.shift = shift; L.out = z; L.zb = zb; L.zb8 = zb8;
  return launch_tc_conv<2>(L, cudaStream_t(stream));
}

extern "C" int bdbnn_real_conv_fwd_eval_pad_shortcut(const uint16_t* xh, const uint32_t* x_amax_bits,
                                                     const uint16_t* wf, const float* scale, const float* shift,
                                                     const float* x_res, int32_t H_res, int32_t W_res, int32_t C_res,
                                                     int32_t pad, int32_t relu, float* z, uint32_t* z_amax_bits,
                                                     const bdbnn_conv_shape* s, void* stream) {
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(xh && x_amax_bits && wf && scale && shift && z, "real_conv_fwd_eval_pad_shortcut: NULL pointer");
  TcConvLaunch L;
  fwd_launch(&L, xh, wf, BDBNN_FMT_FP16, s);
  rc = pad_residual(&L, x_res, H_res, W_res, C_res, pad, z, s);
  if (rc) return rc;
  if (!tc_shape_ok(s)) {
    set_error("real_conv_fwd_eval_pad_shortcut: shape not supported by the tensor-core path");
    return BDBNN_ERR_UNSUPPORTED;
  }
  cudaStream_t st = cudaStream_t(stream);
  L.amax_bits = x_amax_bits;
  L.alpha = scale; L.shift = shift; L.out = z; L.relu = relu != 0; L.z_amax = z_amax_bits;
  if (z_amax_bits) BDBNN_CUDA(cudaMemsetAsync(z_amax_bits, 0, sizeof(uint32_t), st));
  return launch_tc_conv<2>(L, st);
}

struct DgradStats {      // backward statistics of the BatchNorm unit that produced this conv's input (see tc_common.cuh)
  const int16_t* y_int; const float* alpha; const float* mean; const float* invstd;
  double* sums; uint32_t* gmax;
};

// band > 0: the grouped conv's banded dgrad (DESIGN.md §4t), wt = [Cin][k*k flipped][band]
static int dgrad_tc_impl(const uint16_t* gys_bf16, int32_t grad_mode, const uint32_t* amax_bits,
                         const uint16_t* wt_bf16, const uint32_t* mask_bits, const float* add, float* gx,
                         const bdbnn_conv_shape* s, const DgradStats* stats, void* stream, int band = 0) {
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(gys_bf16 && wt_bf16 && mask_bits && gx, "binconv_dgrad_tc: NULL pointer");
  BDBNN_REQUIRE(grad_mode >= BDBNN_GRAD_BF16 && grad_mode <= BDBNN_GRAD_FP16S, "binconv_dgrad_tc: bad grad_mode");
  BDBNN_REQUIRE(grad_mode != BDBNN_GRAD_FP16S || amax_bits, "binconv_dgrad_tc: FP16S needs amax_bits");
  const int grad_halves = grad_mode == BDBNN_GRAD_BF16X2 ? 2 : 1;
  if (!tc_shape_ok(s)) { set_error("binconv_dgrad_tc: shape not supported by the tensor-core path"); return BDBNN_ERR_UNSUPPORTED; }
  cudaStream_t st = cudaStream_t(stream);
  const int T = s->kh * s->kw, sd = s->stride;
  // gx[h,w,c] = sum over taps (r,q) with (h+p-r) % sd == 0 (same in w) of
  //             gys[(h+p-r)/sd, (w+p-q)/sd, o] * wt[c][T-1-t][o]; one launch per (h%sd, w%sd) phase.
  TcConvLaunch Ls[4];
  int n_launch = 0;
  bool empty_phase = false;
  for (int a = 0; a < sd; ++a)
    for (int b = 0; b < sd; ++b) {
      TcConvLaunch& L = Ls[n_launch];
      memset(&L, 0, sizeof(L));
      for (int r = 0; r < s->kh; ++r) {
        const int nh = a + s->pad - r;
        if (nh % sd != 0) continue;
        for (int q = 0; q < s->kw; ++q) {
          const int nw = b + s->pad - q;
          if (nw % sd != 0) continue;
          L.dh[L.n_taps] = int8_t(nh / sd); L.dw[L.n_taps] = int8_t(nw / sd);
          L.tb[L.n_taps] = uint8_t(T - 1 - (r * s->kw + q));
          ++L.n_taps;
        }
      }
      L.OH = (s->H - a + sd - 1) / sd; L.OW = (s->W - b + sd - 1) / sd;
      if (L.OH <= 0 || L.OW <= 0) continue;
      if (L.n_taps == 0) { empty_phase = true; continue; }
      L.A = gys_bf16; L.IH = s->Ho; L.IW = s->Wo; L.Kc = band ? band : s->Cout; L.a_halves = grad_halves; L.in_step = 1;
      L.band = band; L.a_chans = s->Cout;
      L.B = wt_bf16; L.b_taps = T; L.Nout = s->Cin;
      L.NIMG = s->N;
      L.out_step = sd; L.off_h = a; L.off_w = b; L.OHf = s->H; L.OWf = s->W;
      L.mask = mask_bits; L.out = gx;
      L.fmt = grad_mode == BDBNN_GRAD_FP16S ? BDBNN_FMT_FP16 : BDBNN_FMT_BF16;
      L.amax_bits = grad_mode == BDBNN_GRAD_FP16S ? amax_bits : nullptr;
      L.add = add;
      if (stats) {
        L.bn_sums = stats->sums; L.bn_ymax = stats->gmax;
        L.st_y = stats->y_int; L.st_alpha = stats->alpha; L.st_mean = stats->mean; L.st_invstd = stats->invstd;
      }
      ++n_launch;
    }
  if (empty_phase) {
    const size_t bytes = size_t(s->N) * s->H * s->W * s->Cin * sizeof(float);
    // add == gx: accumulate in place (positions no phase writes keep their value, nothing to initialise)
    if (add != nullptr && add != gx) BDBNN_CUDA(cudaMemcpyAsync(gx, add, bytes, cudaMemcpyDeviceToDevice, st));
    else if (add == nullptr) BDBNN_CUDA(cudaMemsetAsync(gx, 0, bytes, st));
  }
  if (stats) {
    // one phase (stride 1): the epilogue owns the statistics
    if (n_launch != 1 || empty_phase) { set_error("binconv_dgrad_tc_stats: needs stride 1"); return BDBNN_ERR_UNSUPPORTED; }
    rc = bn_stats_zero(stats->sums, stats->gmax, s->Cin, st);
    if (rc) return rc;
    return launch_tc_conv<1>(Ls[0], st);
  }
  for (int i = 0; i < n_launch; ++i) {
    rc = launch_tc_conv<1>(Ls[i], st);
    if (rc) return rc;
  }
  return BDBNN_OK;
}

extern "C" int bdbnn_binconv_dgrad_tc(const uint16_t* gys_bf16, int32_t grad_mode, const uint32_t* amax_bits,
                                      const uint16_t* wt_bf16, const uint32_t* mask_bits, const float* add,
                                      float* gx, const bdbnn_conv_shape* s, void* stream) {
  return dgrad_tc_impl(gys_bf16, grad_mode, amax_bits, wt_bf16, mask_bits, add, gx, s, nullptr, stream);
}

extern "C" int bdbnn_binconv_dgrad_tc_stats(const uint16_t* gys_bf16, int32_t grad_mode, const uint32_t* amax_bits,
                                            const uint16_t* wt_bf16, const uint32_t* mask_bits, const float* add,
                                            float* gx, const bdbnn_conv_shape* s, const int16_t* prod_y_int,
                                            const float* prod_alpha, const float* prod_mean,
                                            const float* prod_invstd, double* prod_sums, uint32_t* prod_gmax,
                                            void* stream) {
  BDBNN_REQUIRE(prod_y_int && prod_alpha && prod_mean && prod_invstd && prod_sums && prod_gmax,
                "binconv_dgrad_tc_stats: NULL statistics pointer");
  BDBNN_REQUIRE(s && s->stride == 1 && s->Cin <= 512, "binconv_dgrad_tc_stats: needs stride 1 and Cin <= 512");
  const DgradStats stats = {prod_y_int, prod_alpha, prod_mean, prod_invstd, prod_sums, prod_gmax};
  return dgrad_tc_impl(gys_bf16, grad_mode, amax_bits, wt_bf16, mask_bits, add, gx, s, &stats, stream);
}


// ---- grouped 3x3 convs as banded GEMMs (DESIGN.md §4t) -------------------------------------------------------
// The band B = max(16, Cg) of a grouped conv the banded kernels take (Cin = Cout, Cg = Cin / groups divides B, B in
// {16, 32, 64} and divides Cout, 3x3 / pad 1, the dense kernels' spatial limits), else 0.  No CUDA call.
namespace bdbnn {
int gconv_band(const bdbnn_conv_shape* s, int groups) {
  if (!s || groups < 2 || s->Cin != s->Cout || s->Cin % groups != 0) return 0;
  const int cg = s->Cin / groups, B = cg < 16 ? 16 : cg;
  if ((B != 16 && B != 32 && B != 64) || B % cg != 0 || s->Cout % B != 0) return 0;
  if (s->kh != 3 || s->kw != 3 || s->pad != 1 || !tc_shape_ok(s)) return 0;
  return B;
}
}  // namespace bdbnn

// The forward GEMM of a grouped conv: A = xh (fp16 NHWC, Cin channels), B = wf [Cout][9][B] block-diagonal per band.
static void gconv_fwd_launch(TcConvLaunch* L, const void* xh, const void* wf, const bdbnn_conv_shape* s, int B) {
  fwd_launch(L, xh, wf, BDBNN_FMT_FP16, s);
  L->Kc = B; L->band = B; L->a_chans = s->Cin;
}

static int gconv_check(const bdbnn_conv_shape* s, int32_t groups, const char* what, int* band) {
  int rc = validate_shape(s);
  if (rc) return rc;
  *band = gconv_band(s, groups);
  if (*band == 0) {
    set_error("%s: grouped conv (Cin %d, Cout %d, groups %d, %dx%d, pad %d) not supported", what, s->Cin, s->Cout,
              groups, s->kh, s->kw, s->pad);
    return BDBNN_ERR_UNSUPPORTED;
  }
  return BDBNN_OK;
}

extern "C" int bdbnn_real_gconv_supported(const bdbnn_conv_shape* s, int32_t groups) {
  if (!s || s->N <= 0 || s->H <= 0 || s->W <= 0 || s->stride <= 0 || s->Ho != (s->H + 2 * s->pad - s->kh) / s->stride + 1 ||
      s->Wo != (s->W + 2 * s->pad - s->kw) / s->stride + 1 || s->Ho <= 0 || s->Wo <= 0)
    return 0;
  const int B = gconv_band(s, groups);
  if (B == 0) return 0;
  TcConvParams p;
  size_t smem = 0;
  int tiles = 0, caps = 0;
  TcConvLaunch L;
  gconv_fwd_launch(&L, nullptr, nullptr, s, B);
  double sums = 0.0;
  uint32_t ymax = 0;
  L.bn_sums = &sums; L.bn_ymax = &ymax;          // the training forward keeps its statistics in the epilogue
  if (plan_tc_conv(L, 0, &p, &smem, &tiles)) caps |= BDBNN_TC_FWD;
  L.bn_sums = nullptr; L.bn_ymax = nullptr;
  if (plan_tc_conv(L, 2, &p, &smem, &tiles)) caps |= BDBNN_TC_EVAL;
  // every phase of the dgrad (the taps of phase (a, b) as dgrad_tc_impl builds them)
  bool dg = true;
  const int sd = s->stride;
  for (int a = 0; a < sd; ++a)
    for (int b = 0; b < sd; ++b) {
      memset(&L, 0, sizeof(L));
      for (int r = 0; r < 3; ++r)
        for (int q = 0; q < 3; ++q)
          if ((a + 1 - r) % sd == 0 && (b + 1 - q) % sd == 0) {
            L.dh[L.n_taps] = int8_t((a + 1 - r) / sd); L.dw[L.n_taps] = int8_t((b + 1 - q) / sd);
            L.tb[L.n_taps] = uint8_t(8 - (r * 3 + q));
            ++L.n_taps;
          }
      L.OH = (s->H - a + sd - 1) / sd; L.OW = (s->W - b + sd - 1) / sd;
      if (L.OH <= 0 || L.OW <= 0) continue;
      L.IH = s->Ho; L.IW = s->Wo; L.Kc = B; L.a_halves = 1; L.in_step = 1; L.b_taps = 9; L.Nout = s->Cin;
      L.NIMG = s->N; L.out_step = sd; L.off_h = a; L.off_w = b; L.OHf = s->H; L.OWf = s->W;
      L.fmt = BDBNN_FMT_FP16; L.band = B; L.a_chans = s->Cout;
      dg = dg && plan_tc_conv(L, 1, &p, &smem, &tiles);
    }
  if (dg) caps |= BDBNN_TC_DGRAD;
  if (gwgrad_tc_ok(s, B)) caps |= BDBNN_TC_WGRAD;
  return caps;
}

extern "C" int bdbnn_real_gconv_fwd(const uint16_t* xh, const uint16_t* wf, const float* alpha, float* y,
                                    const bdbnn_conv_shape* s, int32_t groups, double* bn_sums, uint32_t* bn_ymax,
                                    void* stream) {
  int band = 0;
  int rc = gconv_check(s, groups, "real_gconv_fwd", &band);
  if (rc) return rc;
  BDBNN_REQUIRE(xh && wf && alpha && y, "real_gconv_fwd: NULL pointer");
  BDBNN_REQUIRE((bn_sums == nullptr) == (bn_ymax == nullptr), "real_gconv_fwd: bn_sums and bn_ymax go together");
  TcConvLaunch L;
  gconv_fwd_launch(&L, xh, wf, s, band);
  L.alpha = alpha; L.out = y;
  L.bn_sums = bn_sums; L.bn_ymax = bn_ymax;
  rc = bn_stats_zero(bn_sums, bn_ymax, s->Cout, cudaStream_t(stream));
  if (rc) return rc;
  return launch_tc_conv<0>(L, cudaStream_t(stream));
}

extern "C" int bdbnn_real_gconv_fwd_eval(const uint16_t* xh, const uint32_t* x_amax_bits, const uint16_t* wf,
                                         const float* scale, const float* shift, const float* residual, int32_t act,
                                         float* z, uint32_t* z_amax_bits, const bdbnn_conv_shape* s, int32_t groups,
                                         void* stream) {
  int band = 0;
  int rc = gconv_check(s, groups, "real_gconv_fwd_eval", &band);
  if (rc) return rc;
  BDBNN_REQUIRE(xh && x_amax_bits && wf && scale && shift && z, "real_gconv_fwd_eval: NULL pointer");
  BDBNN_REQUIRE(act == BDBNN_ACT_NONE || act == BDBNN_ACT_RELU,
                "real_gconv_fwd_eval: act must be 0 (none) or 1 (ReLU), got %d", act);
  BDBNN_REQUIRE(residual != z, "real_gconv_fwd_eval: residual must not alias z");
  cudaStream_t st = cudaStream_t(stream);
  TcConvLaunch L;
  gconv_fwd_launch(&L, xh, wf, s, band);
  L.amax_bits = x_amax_bits;
  L.alpha = scale; L.shift = shift; L.add = residual; L.out = z; L.z_amax = z_amax_bits;
  L.relu = act == BDBNN_ACT_RELU;
  if (z_amax_bits) BDBNN_CUDA(cudaMemsetAsync(z_amax_bits, 0, sizeof(uint32_t), st));
  return launch_tc_conv<2>(L, st);
}

extern "C" int bdbnn_real_gconv_dgrad(const uint16_t* gys, const uint32_t* amax_bits, const uint16_t* wt,
                                      const uint32_t* mask_bits, const float* add, float* gx,
                                      const bdbnn_conv_shape* s, int32_t groups, void* stream) {
  int band = 0;
  int rc = gconv_check(s, groups, "real_gconv_dgrad", &band);
  if (rc) return rc;
  return dgrad_tc_impl(gys, BDBNN_GRAD_FP16S, amax_bits, wt, mask_bits, add, gx, s, nullptr, stream, band);
}
