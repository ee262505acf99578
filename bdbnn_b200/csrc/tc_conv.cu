// wgmma / TMA implicit-GEMM kernel for the binary convolution (sm_90a).
//
//   tc_conv_kernel  : D[pix, n] = sum_{tap t} sum_{k} A[pix shifted by t, k] * B[n, t*Kc + k]
//                     forward : A = sign(x)  (+-1 fp16/bf16/fp8, NHWC), B = sign(W) [Cout][T][Cin]; epilogue * alpha[n]
//                     dgrad   : A = gy*gscale (bf16/fp16,  NHWC), B = sign(W)^T [Cin][T'][Cout]; epilogue * STE mask bit
//
// Dataflow per CTA (one 128-row output tile, one N tile of BN <= 128 columns):
//   warp 8 lane 0 : TMA producer. For every (tap, K-block) loads the activation box
//                   [BNI images][BH rows][BW=OW cols][KB channels] at coordinates shifted by the tap —
//                   TMA zero-fills out-of-image coordinates, which IS the conv's zero padding — and the
//                   matching [BN x KB] weight box, into a `stages`-deep ring of swizzled K-major tiles.
//   warpgroups 0/1: wgmma (fp32 accumulate in registers) for tile rows [0, 64) / [64, 128), one wgmma group in
//                   flight: a ring slot is released once the group after it was issued and the one reading it retired.
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
  int32_t row_bytes;         // KB * element size = swizzle span (32/64/128)
  const uint32_t* amax_bits; // FP16S: post-scale 2^-e (NULL otherwise)
  const float* add;          // dgrad: optional additive tensor
  const float* alpha;        // MODE 0: per-output-channel scale
  const uint32_t* mask;      // MODE 1: STE mask words [pix][Nout/32 (ceil)]
  float* out;                // [pix][Nout] fp32
  int16_t* out_i16;          // MODE 0: the exact integer accumulator as int16 instead of out (y = alpha * int)
  double* bn_sums;           // per-channel statistics [2*Nout] (NULL = off), see TcConvLaunch
  double* stat_part;         // this launch's per-CTA statistics rows [gridDim.x][2*Nout] (det_sums_finish adds them)
  uint32_t* bn_ymax;
  const int16_t* st_y; const float* st_alpha; const float* st_mean; const float* st_invstd;   // MODE 1 statistics
};

// KIND: 0 fp16, 1 bf16, 2 fp8 e4m3 operands; NW: wgmma N (16, 32, or 64 with BN/64 chunks)
template <int MODE, int KIND, int NW>
__global__ void __launch_bounds__(kTcThreads)
tc_conv_kernel(const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB,
               const TcConvParams p) {
  constexpr int NCH = NW == 64 ? kMaxBN / 64 : 1;
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
  const bool do_stats = p.bn_sums != nullptr;

  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), 2);      // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  for (int i = threadIdx.x; i < (kTcThreads / 32 - 1) * kMaxBN; i += blockDim.x) {
    (&stat_sum[0][0])[i] = 0.f; (&stat_sq[0][0])[i] = 0.f; (&stat_max[0][0])[i] = 0.f;
  }
  if (warp == kProducerWarp && lane == 0) {
    prefetch_tmap(&tmA);
    prefetch_tmap(&tmB);
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      const uint32_t tx = uint32_t(p.BNI * p.BH * p.BW + p.BN) * uint32_t(p.row_bytes);
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
          tma_load_4d(a_dst, &tmA, fb, kb * p.KB, dw, h0 * p.in_step + dh, n0);
          tma_load_2d(a_dst + a_bytes, &tmB, fb, tb * p.Kc + kbb * p.KB, nn0);
        }
      }
    }
  } else {
    const int wg = warp >> 2, wq = warp & 3;
    const int nch = p.BN / NW;
    float acc[NCH][NW / 2];
#pragma unroll
    for (int c = 0; c < NCH; ++c)
#pragma unroll
      for (int i = 0; i < NW / 2; ++i) acc[c][i] = 0.f;
    const int k_steps = p.row_bytes / 32;          // one wgmma consumes 32 bytes of every row
    for (int it = 0; it < n_iters; ++it) {
      const int stage = it % p.stages;
      mbar_wait(smem_u32(&full_bar[stage]), uint32_t(it / p.stages) & 1u);
      const uint32_t a_src = tiles_base + stage * stage_bytes + uint32_t(wg * 64 * p.row_bytes);
      const uint32_t b_src = tiles_base + stage * stage_bytes + a_bytes;
      wgmma_fence();
      for (int k = 0; k < k_steps; ++k) {
        const uint64_t ad = make_kmajor_desc(a_src + k * 32, p.row_bytes);
#pragma unroll
        for (int c = 0; c < NCH; ++c)
          if (c < nch)
            wgmma_ss<NW, KIND>(acc[c], ad, make_kmajor_desc(b_src + uint32_t(c * NW * p.row_bytes) + k * 32, p.row_bytes));
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (it > 0 && (threadIdx.x & 127) == 0) mbar_arrive(smem_u32(&empty_bar[(it - 1) % p.stages]));
    }
    wgmma_wait<0>();
#pragma unroll
    for (int c = 0; c < NCH; ++c) wgmma_fence_regs(acc[c]);

    // ---- epilogue: this thread holds rows r and r + 8 (r = 64 wg + 16 wq + lane/4), column pairs 8j + 2(lane%4) ----
    const float post = (MODE == 1 && p.amax_bits) ? amax_pow2_scale(__ldg(p.amax_bits), true) : 1.0f;
    const int mask_words = (p.Nout + 31) >> 5;
    int64_t pix[2];
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
    }
#pragma unroll
    for (int c = 0; c < NCH; ++c) {
      if (c >= nch) break;
#pragma unroll
      for (int j = 0; j < NW / 8; ++j) {
        const int col = c * NW + 8 * j + 2 * (lane & 3);
        const int ch = nn0 + col;
        float a0 = 1.f, a1 = 1.f, sa0 = 0.f, sa1 = 0.f, sb0 = 0.f, sb1 = 0.f;
        if (MODE == 0) {
          a0 = __ldg(p.alpha + ch); a1 = __ldg(p.alpha + ch + 1);
        } else if (do_stats) {               // yhat = y_int * alpha * invstd - mean * invstd of the producing unit
          const float is0 = __ldg(p.st_invstd + ch), is1 = __ldg(p.st_invstd + ch + 1);
          sa0 = __ldg(p.st_alpha + ch) * is0; sa1 = __ldg(p.st_alpha + ch + 1) * is1;
          sb0 = __ldg(p.st_mean + ch) * is0; sb1 = __ldg(p.st_mean + ch + 1) * is1;
        }
        float s0 = 0.f, s1 = 0.f, q0 = 0.f, q1 = 0.f, m0 = 0.f, m1 = 0.f;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          if (!valid[h]) continue;
          const float v0 = acc[c][4 * j + 2 * h], v1 = acc[c][4 * j + 2 * h + 1];
          const int64_t off = pix[h] * p.Nout + ch;
          float o0, o1;
          if (MODE == 0) {
            o0 = v0 * a0; o1 = v1 * a1;
            if (p.out_i16 != nullptr)        // exact: |v| <= taps * Kc <= 32767
              *reinterpret_cast<uint32_t*>(p.out_i16 + off) = (uint32_t(int(v0)) & 0xffffu) | (uint32_t(int(v1)) << 16);
            else
              *reinterpret_cast<float2*>(p.out + off) = make_float2(o0, o1);
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
  p.alpha = L.alpha; p.mask = L.mask; p.out = L.out; p.out_i16 = mode == 0 ? L.out_i16 : nullptr;
  p.amax_bits = L.amax_bits; p.add = L.add;
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
  return true;
}

template <int MODE, int KIND>
static int launch_kind(const CUtensorMap& tmA, const CUtensorMap& tmB, const TcConvParams& p, size_t smem, dim3 grid,
                       cudaStream_t st) {
  auto kern = p.BN == 16 ? tc_conv_kernel<MODE, KIND, 16>
                         : (p.BN == 32 ? tc_conv_kernel<MODE, KIND, 32> : tc_conv_kernel<MODE, KIND, 64>);
  BDBNN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  if (p.bn_sums == nullptr) {
    kern<<<grid, kTcThreads, smem, st>>>(tmA, tmB, p);
    return check_launch("tc_conv_kernel");
  }
  TcConvParams q = p;
  int rc = det_sums_alloc(&q.stat_part, grid.x, 2 * p.Nout, st);
  if (rc) return rc;
  kern<<<grid, kTcThreads, smem, st>>>(tmA, tmB, q);
  rc = check_launch("tc_conv_kernel");
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
    rc = make_act_map(&tmA, L.A, L.NIMG, L.IH, L.IW, L.Kc * L.a_halves, p.KB, p.BW, p.BH, p.BNI, L.in_step, esize);
  if (rc) return rc;
  rc = make_weight_map(&tmB, L.B, L.Nout, L.b_taps * L.Kc, p.KB, p.BN, esize);
  if (rc) return rc;
  const dim3 grid(unsigned(tiles), unsigned(L.Nout / p.BN));
  // forward statistics of the narrow (16/32-channel) GEMMs: one pass over the fp32 result after the kernel
  const bool stats_pass = MODE == 0 && L.bn_sums != nullptr && !wide_gemm(L) && L.out != nullptr;
  if (stats_pass) { p.bn_sums = nullptr; p.bn_ymax = nullptr; }
  if (L.fmt < 0) {
    if (MODE != 0) { set_error("tc_conv: fp8 operands are forward only"); return BDBNN_ERR_UNSUPPORTED; }
    return launch_kind<0, 2>(tmA, tmB, p, smem, grid, st);
  }
  rc = L.fmt == BDBNN_FMT_BF16 ? launch_kind<MODE, 1>(tmA, tmB, p, smem, grid, st)
                               : launch_kind<MODE, 0>(tmA, tmB, p, smem, grid, st);
  if (rc || !stats_pass) return rc;
  return bn_stats_launch(L.out, int64_t(L.NIMG) * L.OHf * L.OWf, L.Nout, L.bn_sums, L.bn_ymax, st);
}

// Stem conv forward (7x7 / stride 2 / pad 3 on 3 channels) as a 7-tap implicit GEMM over the packed
// window view: tap r reads window row 2*oh + r, K = 32 values (8 pixels x 4 halves) per tap.
int launch_stem_fwd(const uint16_t* xw, const uint16_t* wf, const float* alpha, float* y, const StemGeom& g,
                    double* bn_sums, uint32_t* bn_ymax, cudaStream_t st) {
  TcConvLaunch L;
  memset(&L, 0, sizeof(L));
  L.A = xw; L.IH = g.HP; L.IW = g.Wo; L.Kc = kStemWin; L.a_halves = 1; L.in_step = 2;
  L.win = 1; L.win_stride = g.win_stride; L.win_row_stride = g.row_stride; L.win_img_stride = g.img_stride;
  L.B = wf; L.b_taps = kStemTaps; L.Nout = kStemCout;
  L.NIMG = g.N; L.OH = g.Ho; L.OW = g.Wo;
  for (int r = 0; r < kStemTaps; ++r) { L.dh[r] = int8_t(r); L.dw[r] = 0; L.tb[r] = uint8_t(r); }
  L.n_taps = kStemTaps;
  L.out_step = 1; L.OHf = g.Ho; L.OWf = g.Wo;
  L.alpha = alpha; L.out = y; L.fmt = BDBNN_FMT_FP16;
  L.bn_sums = bn_sums; L.bn_ymax = bn_ymax;
  int rc = bn_stats_zero(bn_sums, bn_ymax, kStemCout, st);
  if (rc) return rc;
  return launch_tc_conv<0>(L, st);
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

// Host-only: the kernel's tiling for the forward (mode 0: 16-bit operands, 2: fp8) or the first dgrad phase
// (mode 1) of a shape.  out[12] = {planned, halo, TS, NB, BN, n_tiles, supers, stages, dynamic smem, grid,
// stage bytes, patch bytes}; halo = 0, TS = NB = 1 (one 128-row tile per CTA, no patch), supers = M tiles.
// planned = 0 when the GEMM is not eligible for the int16 result / fused dgrad statistics.  No CUDA call.
extern "C" int bdbnn_debug_conv_plan(const bdbnn_conv_shape* s, int32_t mode, int32_t grad_halves, int32_t* out,
                                     int32_t n_out) {
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(out && n_out >= 12 && mode >= 0 && mode <= 2 && (grad_halves == 1 || grad_halves == 2),
                "debug_conv_plan: bad arguments");
  memset(out, 0, 12 * sizeof(int32_t));
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
    L.fmt = mode == 2 ? -1 : BDBNN_FMT_FP16;
    if (mode == 2 && s->Cin % 128 != 0) return BDBNN_OK;
  }
  if (L.n_taps == 0 || !wide_gemm(L)) return BDBNN_OK;
  TcConvParams p;
  size_t smem = 0;
  int tiles = 0;
  if (!plan_tc_conv(L, mode == 1 ? 1 : 0, &p, &smem, &tiles)) return BDBNN_OK;
  const int32_t v[12] = {1, 0, 1, 1, p.BN, L.Nout / p.BN, tiles, p.stages, int32_t(smem), tiles * (L.Nout / p.BN),
                         int32_t((uint32_t(kTileM + p.BN) * p.row_bytes + 1023u) & ~1023u), 0};
  memcpy(out, v, sizeof(v));
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
         (i16 ? BDBNN_TC_FWD_I16 : 0);
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
  L.alpha = alpha; L.out = nullptr; L.out_i16 = y_int; L.fmt = fmt;
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
  memset(&L, 0, sizeof(L));
  L.A = xb_bf16; L.IH = s->H; L.IW = s->W; L.Kc = s->Cin; L.a_halves = 1; L.in_step = s->stride;
  L.B = wf_bf16; L.b_taps = s->kh * s->kw; L.Nout = s->Cout;
  L.NIMG = s->N; L.OH = s->Ho; L.OW = s->Wo;
  for (int r = 0; r < s->kh; ++r)
    for (int q = 0; q < s->kw; ++q) {
      const int t = r * s->kw + q;
      L.dh[t] = int8_t(r - s->pad); L.dw[t] = int8_t(q - s->pad); L.tb[t] = uint8_t(t);
    }
  L.n_taps = s->kh * s->kw;
  L.out_step = 1; L.OHf = s->Ho; L.OWf = s->Wo;
  L.alpha = alpha; L.out = y; L.fmt = fmt;
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
  memset(&L, 0, sizeof(L));
  L.A = reinterpret_cast<const uint16_t*>(xb_fp8); L.IH = s->H; L.IW = s->W; L.Kc = s->Cin; L.a_halves = 1;
  L.in_step = s->stride;
  L.B = reinterpret_cast<const uint16_t*>(wf_fp8); L.b_taps = s->kh * s->kw; L.Nout = s->Cout;
  L.NIMG = s->N; L.OH = s->Ho; L.OW = s->Wo;
  for (int r = 0; r < s->kh; ++r)
    for (int q = 0; q < s->kw; ++q) {
      const int t = r * s->kw + q;
      L.dh[t] = int8_t(r - s->pad); L.dw[t] = int8_t(q - s->pad); L.tb[t] = uint8_t(t);
    }
  L.n_taps = s->kh * s->kw;
  L.out_step = 1; L.OHf = s->Ho; L.OWf = s->Wo;
  L.alpha = alpha; L.out = y; L.fmt = -1;
  BDBNN_REQUIRE((bn_sums == nullptr) == (bn_ymax == nullptr), "binconv_fwd_tc8: bn_sums and bn_ymax go together");
  BDBNN_REQUIRE(bn_sums == nullptr || s->Cout <= 512, "binconv_fwd_tc8: statistics need Cout <= 512");
  L.bn_sums = bn_sums; L.bn_ymax = bn_ymax;
  rc = bn_stats_zero(bn_sums, bn_ymax, s->Cout, cudaStream_t(stream));
  if (rc) return rc;
  return launch_tc_conv<0>(L, cudaStream_t(stream));
}

struct DgradStats {      // backward statistics of the BatchNorm unit that produced this conv's input (see tc_common.cuh)
  const int16_t* y_int; const float* alpha; const float* mean; const float* invstd;
  double* sums; uint32_t* gmax;
};

static int dgrad_tc_impl(const uint16_t* gys_bf16, int32_t grad_mode, const uint32_t* amax_bits,
                         const uint16_t* wt_bf16, const uint32_t* mask_bits, const float* add, float* gx,
                         const bdbnn_conv_shape* s, const DgradStats* stats, void* stream) {
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
      L.A = gys_bf16; L.IH = s->Ho; L.IW = s->Wo; L.Kc = s->Cout; L.a_halves = grad_halves; L.in_step = 1;
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

