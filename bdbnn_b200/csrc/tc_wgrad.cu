// Weight gradient on tensor cores (wgmma + TMA, sm_90a).
//
//   D[(t,c), o] = sum_pix  xb[pix shifted by tap t, c] * gys[pix, o]          (K = output pixels)
//
// Both operands are "MN-major" for this GEMM: for a fixed pixel the M index (c) / N index (o) is the
// contiguous one in NHWC memory, so a TMA box [pixels][64 channels] lands in shared memory exactly in
// the canonical MN-major SWIZZLE_128B layout (8 pixel rows x 128 B per swizzle atom; SBO = 1024 B
// between 8-row K groups; LBO = distance between MN chunks).
// An M tile of 128 rows is two 64-channel "units" (tap, channel-chunk); unit u = tap * (Cin/64) + chunk.
// Per K stage one TMA box per unit is loaded (plus the gys boxes); warpgroup 0 multiplies rows [0, 64) of
// every M tile, warpgroup 1 rows [64, 128).
//
// Each CTA owns up to G accumulators (G*BN <= 256: 128 fp32 registers per thread) that share the gys stage,
// walks a contiguous range of K stages (split-K across CTAs) and writes its partial tiles to its own slice of
// an fp32 workspace [ksplit][T*Cin][Cout] (plain stores, no atomics); the finalize kernel sums the
// slices in a fixed order (run-to-run deterministic), applies 1/gscale[o], the FP16S 2^-e, the
// |W|<=1 STE mask and the [t][c][o] -> OIHW transposition.
#include "tc_common.cuh"

namespace bdbnn {

constexpr int kWgradWaves = 3;
constexpr int kMaxUnits = 16;      // units per CTA (G <= 4 M tiles of 2 units, or 2 tiles of 8 16-wide units)

struct TcWgradParams {
  int32_t OW, OH, NIMG;          // gy pixel grid
  int32_t BW, BH, BNI, tiles_h;  // K stage = BNI x BH x BW output pixels
  int32_t rows_a, rows_b;        // rows TMA writes per A box and per B box
  int32_t k_stage;               // K rows consumed per stage (multiple of 16)
  uint32_t a_box_bytes;          // smem footprint of one A box (1024-aligned)
  uint32_t b_box_bytes;
  int32_t n_a_boxes;             // A boxes per stage
  int32_t n_kboxes, kboxes_per_cta;
  int32_t Cin, Cout, kh, kw, pad, stride;
  int32_t g_halves;              // 1: gys = bf16(g); 2: gys = [hi | lo] split, both accumulated
  int32_t UW;                    // unit width in channels: 64 (128-byte rows, SWIZZLE_128B), 32 (64-byte rows,
                                 // SWIZZLE_64B; stem windows) or 16 (SWIZZLE_32B); an M tile is 128/UW units
  int32_t chunks_per_tap;        // Cin / 64
  int32_t n_units, G;            // (tap, chunk) units; M tiles (accumulators) per CTA
  int32_t BN;                    // N tile (output channels per CTA)
  int32_t stages;
  int32_t fmt;                   // operand format (BDBNN_FMT_*)
  float* ws;                     // [ksplit][T*Cin][Cout] fp32 partials (every valid entry is written)
  long long* trace;              // optional clock64 trace of CTA (0,0,0) (bdbnn_debug_trace)
};

#define BDBNN_WTR(r, ev)                                                                         \
  do {                                                                                           \
    if (p.trace != nullptr && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && tr_n < 1023) { \
      p.trace[(r) * 2048 + 2 * tr_n] = (ev);                                                     \
      p.trace[(r) * 2048 + 2 * tr_n + 1] = clock64();                                            \
      ++tr_n;                                                                                    \
    }                                                                                            \
  } while (0)

// NW: wgmma N (16 or 32 for the narrow N tiles, else 64 with BN/64 chunks).  Accumulator slot s = g * (BN/NW) + chunk.
template <int KIND, int NW>
__global__ void __launch_bounds__(kTcThreads)
tc_wgrad_kernel(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmG,
                const TcWgradParams p) {
  constexpr int kSlots = 256 / NW;                               // 128 accumulator floats per thread
  extern __shared__ uint8_t smem_raw[];
  __shared__ __align__(8) uint64_t full_bar[kMaxStages];
  __shared__ __align__(8) uint64_t empty_bar[kMaxStages];
  __shared__ uint32_t unit_off[kMaxUnits];   // byte offset of unit i's operand box inside a stage
  __shared__ int32_t unit_c[kMaxUnits], unit_dw[kMaxUnits], unit_dh[kMaxUnits];   // TMA coordinates of unit i

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const uint32_t tiles_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  const int mt0 = blockIdx.y * p.G;                               // first M tile of this CTA
  const int upt = kTileM / p.UW;                                  // units per M tile (2, 4 or 8)
  const uint32_t a_row = uint32_t(p.UW) * 2u;                     // bytes per A row
  const int n_mtiles = (p.n_units + upt - 1) / upt;
  const int g_cta = min(p.G, n_mtiles - mt0);
  const int nb_chunks = p.BN >= 64 ? p.BN / 64 : 1;               // 64-channel chunks of the N tile (or one narrow one)
  const uint32_t b_row = p.BN >= 64 ? 128u : uint32_t(p.BN) * 2u;  // bytes per gys row of one chunk
  const int nb_boxes = nb_chunks * p.g_halves;                    // hi (and lo) boxes of gys
  const uint32_t a_bytes = uint32_t(p.n_a_boxes) * p.a_box_bytes;
  const uint32_t stage_bytes = a_bytes + uint32_t(nb_boxes) * p.b_box_bytes;
  const int nn0 = blockIdx.z * p.BN;
  const int kb_begin = blockIdx.x * p.kboxes_per_cta;
  const int kb_end = min(kb_begin + p.kboxes_per_cta, p.n_kboxes);

  if (threadIdx.x < g_cta * upt) {
    int u = mt0 * upt + threadIdx.x;
    if (u >= p.n_units) u = p.n_units - 1;                         // odd unit count: rows ignored
    const int t = u / p.chunks_per_tap, j = u - t * p.chunks_per_tap;
    unit_off[threadIdx.x] = threadIdx.x * p.a_box_bytes;
    // the producer is ONE thread: everything per unit that needs a division is computed here, once
    const int r = t / p.kw, sx = t - r * p.kw;
    unit_c[threadIdx.x] = j * 64;
    unit_dw[threadIdx.x] = sx - p.pad;
    unit_dh[threadIdx.x] = r - p.pad;
  }
  if (threadIdx.x == 0) {
    for (int s = 0; s < p.stages; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), 2);                       // one arrival per consumer warpgroup
    }
    fence_barrier_init();
  }
  // Zero every row TMA never writes (A rows >= rows_a, B rows >= rows_b): they are read as K rows.
  {
    uint8_t* base_generic = smem_raw + (tiles_base - smem_u32(smem_raw));
    const int a_w16 = int(a_row / 16u);                            // 16-byte words per A row
    const int a_tail = int(p.a_box_bytes / 16) - p.rows_a * a_w16;
    const int b_w16 = int(b_row / 16u);
    const int b_tail = int(p.b_box_bytes / 16) - p.rows_b * b_w16;
    const int per_stage = p.n_a_boxes * a_tail + nb_boxes * b_tail;
    const int total = p.stages * per_stage;
    for (int i = threadIdx.x; i < total; i += blockDim.x) {
      const int s = i / per_stage;
      int r = i - s * per_stage;
      uint8_t* dst;
      if (r < p.n_a_boxes * a_tail) {
        const int b = r / a_tail, w = r - b * a_tail;
        dst = base_generic + size_t(s) * stage_bytes + size_t(b) * p.a_box_bytes + size_t(p.rows_a) * a_row +
              size_t(w) * 16u;
      } else {
        r -= p.n_a_boxes * a_tail;
        const int b = r / b_tail, w = r - b * b_tail;
        dst = base_generic + size_t(s) * stage_bytes + a_bytes + size_t(b) * p.b_box_bytes +
              size_t(p.rows_b) * b_row + size_t(w) * 16u;
      }
      *reinterpret_cast<uint4*>(dst) = make_uint4(0, 0, 0, 0);
    }
    fence_proxy_async();
  }
  if (warp == kProducerWarp && lane == 0) {
    prefetch_tmap(&tmX);
    prefetch_tmap(&tmG);
  }
  __syncthreads();

  if (warp == kProducerWarp) {
    if (lane == 0) {
      const int n_units_cta = g_cta * upt;
      const uint32_t tx = uint32_t(n_units_cta) * uint32_t(p.rows_a) * a_row +
                          uint32_t(nb_boxes) * uint32_t(p.rows_b) * b_row;
      int tr_n = 0;
      int stage = 0;
      uint32_t phase = 0;
      int tile_n = kb_begin / p.tiles_h, tile_h = kb_begin - tile_n * p.tiles_h;   // advanced incrementally
      for (int kb = kb_begin; kb < kb_end; ++kb) {
        BDBNN_WTR(0, 0);
        mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1u);
        BDBNN_WTR(0, 1);
        const uint32_t fb = smem_u32(&full_bar[stage]);
        mbar_expect_tx(fb, tx);
        const int n0 = tile_n * p.BNI, h0 = tile_h * p.BH;
        const uint32_t dst0 = tiles_base + stage * stage_bytes;
        const int hs = h0 * p.stride;
        for (int i = 0; i < n_units_cta; ++i)
          tma_load_4d(dst0 + unit_off[i], &tmX, fb, unit_c[i], unit_dw[i], hs + unit_dh[i], n0);
        uint32_t bdst = dst0 + a_bytes;
        for (int hf = 0; hf < p.g_halves; ++hf)
          for (int jb = 0; jb < nb_chunks; ++jb, bdst += p.b_box_bytes)
            tma_load_4d(bdst, &tmG, fb, hf * p.Cout + nn0 + jb * 64, 0, h0, n0);
        if (++stage == p.stages) { stage = 0; phase ^= 1u; }
        if (++tile_h == p.tiles_h) { tile_h = 0; ++tile_n; }
      }
    }
  } else if (kb_end > kb_begin) {
    const int wg = warp >> 2, wq = warp & 3;
    const int nch = p.BN / NW;                                     // wgmma chunks per M tile
    const int n_slots = g_cta * nch;
    const int u_wg = 64 / p.UW;                                    // units in this warpgroup's 64 rows
    float acc[kSlots][NW / 2];
#pragma unroll
    for (int s = 0; s < kSlots; ++s)
#pragma unroll
      for (int i = 0; i < NW / 2; ++i) acc[s][i] = 0.f;
    const int k_steps = p.k_stage / 16;
    const uint32_t lbo_a = p.a_box_bytes;                          // MN stride between the units of one wgmma
    int stage = 0;
    uint32_t phase = 0;
    int prev_stage = -1;
    for (int kb = kb_begin; kb < kb_end; ++kb) {
      mbar_wait(smem_u32(&full_bar[stage]), phase);
      const uint32_t a0 = tiles_base + stage * stage_bytes;
      const uint32_t b0 = a0 + a_bytes;
      wgmma_fence();
      for (int hf = 0; hf < p.g_halves; ++hf) {
        for (int k = 0; k < k_steps; ++k) {
          // 16 pixel rows per K step: 2 swizzle atoms of 8 rows
#pragma unroll
          for (int s = 0; s < kSlots; ++s) {
            if (s < n_slots) {
              const int g = s / nch, c = s - g * nch;
              const uint64_t ad = make_smem_desc(a0 + unit_off[g * upt + wg * u_wg] + uint32_t(k) * 16u * a_row, lbo_a, a_row);
              const uint64_t bd = make_smem_desc(b0 + uint32_t(hf * nb_chunks + c) * p.b_box_bytes + uint32_t(k) * 16u * b_row,
                                                 p.b_box_bytes, b_row);
              wgmma_ss<NW, KIND, 1, 1>(acc[s], ad, bd);
            }
          }
        }
      }
      wgmma_commit();
      wgmma_wait<1>();
      if (prev_stage >= 0 && (threadIdx.x & 127) == 0) mbar_arrive(smem_u32(&empty_bar[prev_stage]));
      prev_stage = stage;
      if (++stage == p.stages) { stage = 0; phase ^= 1u; }
    }
    wgmma_wait<0>();
#pragma unroll
    for (int s = 0; s < kSlots; ++s) wgmma_fence_regs(acc[s]);
    // ---- epilogue: rows m (and m + 8) of every M tile, column pairs 8j + 2(lane%4) of every chunk ----
    float* slice = p.ws + int64_t(blockIdx.x) * (int64_t(p.n_units) * p.UW * p.Cout);
#pragma unroll
    for (int s = 0; s < kSlots; ++s) {
      if (s >= n_slots) break;
      const int g = s / nch, c = s - g * nch;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int m = wg * 64 + wq * 16 + (lane >> 2) + 8 * h;
        const int u = (mt0 + g) * upt + m / p.UW;
        if (u >= p.n_units) continue;
        float* wrow = slice + (int64_t(u) * p.UW + (m % p.UW)) * p.Cout + nn0 + c * NW + 2 * (lane & 3);   // row t*Cin + c
#pragma unroll
        for (int j = 0; j < NW / 8; ++j)
          *reinterpret_cast<float2*>(wrow + 8 * j) = make_float2(acc[s][4 * j + 2 * h], acc[s][4 * j + 2 * h + 1]);
      }
    }
  }
}

// Launch with the template arguments of the plan (operand format, wgmma N).
static int launch_wgrad_kernel(const CUtensorMap& tmX, const CUtensorMap& tmG, const TcWgradParams& p, size_t smem,
                               dim3 grid, cudaStream_t st) {
  const int nw = p.BN >= 64 ? 64 : p.BN;
  auto pick = [&](auto k16, auto k32, auto k64) { return nw == 16 ? k16 : (nw == 32 ? k32 : k64); };
  auto kern = p.fmt == BDBNN_FMT_BF16 ? pick(tc_wgrad_kernel<1, 16>, tc_wgrad_kernel<1, 32>, tc_wgrad_kernel<1, 64>)
                                      : pick(tc_wgrad_kernel<0, 16>, tc_wgrad_kernel<0, 32>, tc_wgrad_kernel<0, 64>);
  BDBNN_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  kern<<<grid, kTcThreads, smem, st>>>(tmX, tmG, p);
  return check_launch("tc_wgrad_kernel");
}

// gW[o][c][t] = wmask ? inv_gscale[o] * 2^-e * sum_k ws[k][(t*Cin + c)*Cout + o] : 0
// One thread per [t*Cin+c][o] entry: the ksplit partials are read coalesced and added in slice order.
__global__ void __launch_bounds__(256)
wgrad_finalize_kernel(const float* __restrict__ ws, int ksplit, const uint32_t* __restrict__ wmask,
                      const float* __restrict__ inv_gscale, const uint32_t* __restrict__ amax_bits,
                      float* __restrict__ gW, int Cout, int Cin, int T) {
  const int64_t n = int64_t(Cout) * Cin * T;
  const float post = amax_bits ? amax_pow2_scale(__ldg(amax_bits), true) : 1.0f;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    const int o = int(i % Cout);
    const int64_t tc = i / Cout;
    const int c = int(tc % Cin), t = int(tc / Cin);
    const int64_t e = (int64_t(o) * Cin + c) * T + t;              // OIHW flat index
    float acc = 0.f;
    if ((wmask[e >> 5] >> (e & 31)) & 1u) {
      // fixed summation order (deterministic); four independent chains hide the load latency
      float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
      int k = 0;
      for (; k + 3 < ksplit; k += 4) {
        a0 += ws[int64_t(k) * n + i];
        a1 += ws[int64_t(k + 1) * n + i];
        a2 += ws[int64_t(k + 2) * n + i];
        a3 += ws[int64_t(k + 3) * n + i];
      }
      for (; k < ksplit; ++k) a0 += ws[int64_t(k) * n + i];
      acc = ((a0 + a1) + (a2 + a3)) * post * inv_gscale[o];
    }
    gW[e] = acc;
  }
}

struct WgradPlan {
  TcWgradParams p;
  int ksplit, ks_cap, mgroups, ntiles;
  size_t smem;
  bool ok;
};

static WgradPlan plan_wgrad_small(const bdbnn_conv_shape* s, int halves);

static WgradPlan plan_wgrad(const bdbnn_conv_shape* s, int halves) {
  WgradPlan pl;
  memset(&pl, 0, sizeof(pl));
  if (!s || (s->stride != 1 && s->stride != 2) || s->kh != s->kw || s->kh > 7 || s->pad > s->kh - 1) return pl;
  if (s->Cin == 16 || s->Cin == 32 || s->Cout == 16 || s->Cout == 32) return plan_wgrad_small(s, halves);
  if (s->Cin % 64 != 0 || s->Cout % 64 != 0) return pl;
  if (s->Cout > 128 && s->Cout % 256 != 0) return pl;
  if (s->Wo > 128 || s->W > 128 * s->stride) return pl;
  TcWgradParams& p = pl.p;
  const int T = s->kh * s->kw;
  p.OW = s->Wo; p.OH = s->Ho; p.NIMG = s->N;
  p.Cin = s->Cin; p.Cout = s->Cout; p.kh = s->kh; p.kw = s->kw; p.pad = s->pad; p.stride = s->stride;
  p.g_halves = halves;
  p.UW = 64;
  p.chunks_per_tap = s->Cin / 64;
  p.n_units = T * p.chunks_per_tap;
  const int n_mtiles = (p.n_units + 1) / 2;
  p.BN = s->Cout >= 256 ? 256 : s->Cout;
  p.G = 256 / p.BN;                                               // accumulator registers
  if (p.G > n_mtiles) p.G = n_mtiles;
  {  // balance the M groups (e.g. 9 M tiles with G<=4 -> 3 groups of 3, not 4+4+1)
    const int groups = (n_mtiles + p.G - 1) / p.G;
    p.G = (n_mtiles + groups - 1) / groups;
  }
  p.stages = 2;
  const uint32_t budget = 222u * 1024u;
  {
    // one [rows][64ch] box per unit
    const int row_bytes_all = p.G * 256 + p.BN * 2 * halves;      // smem bytes per pixel row per stage
    const int k_cap = int(budget / (unsigned(p.stages) * unsigned(row_bytes_all))) & ~15;
    if (k_cap < 16) return pl;
    const int kmax = k_cap > 128 ? 128 : k_cap;
    p.BW = s->Wo;
    double best = -1.0;
    int bBH = 0, bBNI = 0;
    if (s->Ho * s->Wo <= kmax) {
      for (int ni = 1; ni * s->Ho * s->Wo <= kmax && ni <= s->N && ni <= 256; ++ni) {
        const int rows = ni * s->Ho * s->Wo, ks = (rows + 15) & ~15;
        const double eff = double(rows) / ks * double(s->N) / (double((s->N + ni - 1) / ni) * ni);
        if (eff * (1.0 + 0.02 * ni) > best) { best = eff * (1.0 + 0.02 * ni); bBH = s->Ho; bBNI = ni; }
      }
    } else {
      for (int bh = 1; bh * s->Wo <= kmax && bh <= s->Ho; ++bh) {
        const int rows = bh * s->Wo, ks = (rows + 15) & ~15;
        const double eff = double(rows) / ks * double(s->Ho) / (double((s->Ho + bh - 1) / bh) * bh);
        if (eff * (1.0 + 0.01 * bh) > best) { best = eff * (1.0 + 0.01 * bh); bBH = bh; bBNI = 1; }
      }
    }
    if (bBH == 0) return pl;
    p.BH = bBH; p.BNI = bBNI;
    p.rows_a = p.rows_b = p.BNI * p.BH * p.BW;
    p.k_stage = (p.rows_a + 15) & ~15;
    p.a_box_bytes = p.b_box_bytes = uint32_t(p.k_stage) * 128u;
    p.n_a_boxes = p.G * 2;
    p.tiles_h = (s->Ho + p.BH - 1) / p.BH;
  }
  p.n_kboxes = p.tiles_h * ((s->N + p.BNI - 1) / p.BNI);
  pl.mgroups = (n_mtiles + p.G - 1) / p.G;
  pl.ntiles = s->Cout / p.BN;
  // split K over up to kWgradWaves waves of CTAs (1 CTA/SM by shared memory and registers): the register
  // accumulators hold at most 256 columns per CTA, so one wave would leave fp32 accumulation chains of up to a
  // whole layer's pixels in one CTA (bf16x2 wgrad error above 2e-5 of the L2 norm at N=256)
  int ks = kWgradWaves * num_sms() / (pl.mgroups * pl.ntiles);
  if (ks < 1) ks = 1;
  pl.ks_cap = ks;                       // upper bound of ksplit for any gradient mode (workspace sizing)
  if (ks > p.n_kboxes) ks = p.n_kboxes;
  p.kboxes_per_cta = (p.n_kboxes + ks - 1) / ks;
  pl.ksplit = (p.n_kboxes + p.kboxes_per_cta - 1) / p.kboxes_per_cta;
  const size_t stage_bytes = size_t(p.n_a_boxes) * p.a_box_bytes + size_t(p.BN / 64 * halves) * p.b_box_bytes;
  // stages are small (32-128 K rows) and the loop is bound by the TMA round trip, not by bytes: use every
  // stage the shared memory holds
  int stages = int(budget / stage_bytes);
  if (stages > kMaxStages) stages = kMaxStages;
  if (stages > p.kboxes_per_cta) stages = p.kboxes_per_cta;
  if (stages < 2) stages = 2;
  if (size_t(stages) * stage_bytes > budget) stages = 2;
  p.stages = stages;
  pl.smem = size_t(p.stages) * stage_bytes + 1024;
  pl.ok = pl.smem <= 227u * 1024u;
  return pl;
}

// CIFAR-sized layers (ResNet-20: 16/32/64 channels): box mode with narrow units — A rows of Cin*2 bytes
// (16 channels: SWIZZLE_32B, 32: SWIZZLE_64B, 64: SWIZZLE_128B), one gys box of Cout channels as the N
// tile.  All M tiles of the layer live in one CTA when they fit (T*Cin/128 accumulators of Cout columns).
static WgradPlan plan_wgrad_small(const bdbnn_conv_shape* s, int halves) {
  WgradPlan pl;
  memset(&pl, 0, sizeof(pl));
  auto ok_c = [](int c) { return c == 16 || c == 32 || c == 64; };
  if (!ok_c(s->Cin) || !ok_c(s->Cout)) return pl;
  if (s->Wo > 128 || s->W > 128 * s->stride) return pl;
  TcWgradParams& p = pl.p;
  const int T = s->kh * s->kw;
  p.OW = s->Wo; p.OH = s->Ho; p.NIMG = s->N;
  p.Cin = s->Cin; p.Cout = s->Cout; p.kh = s->kh; p.kw = s->kw; p.pad = s->pad; p.stride = s->stride;
  p.g_halves = halves;
  p.UW = s->Cin;
  p.chunks_per_tap = 1;
  p.n_units = T;
  const int upt = kTileM / p.UW;
  const int n_mtiles = (p.n_units + upt - 1) / upt;
  p.BN = s->Cout;
  p.G = kMaxUnits / upt;
  if (p.G > n_mtiles) p.G = n_mtiles;
  if (p.G * p.BN > 256) p.G = 256 / p.BN;
  p.BW = s->Wo;
  const int a_row = p.UW * 2, b_row = p.BN >= 64 ? 128 : p.BN * 2;
  // K stage: whole images when they are small, else rows of one image; <= 128 pixel rows
  if (s->Ho * s->Wo <= kTileM) {
    p.BH = s->Ho;
    p.BNI = kTileM / (s->Ho * s->Wo);
    if (p.BNI > s->N) p.BNI = s->N;
  } else {
    p.BH = kTileM / s->Wo;
    p.BNI = 1;
  }
  p.rows_a = p.rows_b = p.BNI * p.BH * p.BW;
  p.k_stage = (p.rows_a + 15) & ~15;
  p.a_box_bytes = (uint32_t(p.k_stage) * uint32_t(a_row) + 1023u) & ~1023u;
  p.b_box_bytes = (uint32_t(p.k_stage) * uint32_t(b_row) + 1023u) & ~1023u;
  p.tiles_h = (s->Ho + p.BH - 1) / p.BH;
  p.n_kboxes = p.tiles_h * ((s->N + p.BNI - 1) / p.BNI);
  // fewer M tiles per CTA until a 2-stage ring fits in shared memory
  size_t stage_bytes = 0;
  for (;; --p.G) {
    p.n_a_boxes = p.G * upt;
    stage_bytes = size_t(p.n_a_boxes) * p.a_box_bytes + size_t(halves) * p.b_box_bytes;
    p.stages = int((226u * 1024u) / stage_bytes);
    if (p.stages >= 2 || p.G == 1) break;
  }
  if (p.stages > 4) p.stages = 4;
  pl.mgroups = (n_mtiles + p.G - 1) / p.G;
  pl.ntiles = 1;
  int ks = kWgradWaves * num_sms() / pl.mgroups;
  if (ks < 1) ks = 1;
  pl.ks_cap = ks;
  if (ks > p.n_kboxes) ks = p.n_kboxes;
  p.kboxes_per_cta = (p.n_kboxes + ks - 1) / ks;
  pl.ksplit = (p.n_kboxes + p.kboxes_per_cta - 1) / p.kboxes_per_cta;
  pl.smem = size_t(p.stages) * stage_bytes + 1024;
  pl.ok = p.stages >= 2 && pl.smem <= 227u * 1024u;
  return pl;
}

bool wgrad_tc_ok(const bdbnn_conv_shape* s) { return s && plan_wgrad(s, 2).ok; }

// ---- stem conv weight gradient ------------------------------------------------------------------
// D[(r, j), o] = sum_pix xw[window(pix) of row 2*oh + r][j] * gys[pix, o]: 7 units (rows r of the 7x7
// filter) of 32 window values (8 pixels x 4 halves; j = s*4 + c), box mode, one K stage per output row
// group.  Both M tiles (units 0-3, 4-6 + one duplicate) live in every CTA, so gys is fetched once.
static WgradPlan plan_stem_wgrad(const StemGeom& g) {
  WgradPlan pl;
  memset(&pl, 0, sizeof(pl));
  TcWgradParams& p = pl.p;
  p.OW = g.Wo; p.OH = g.Ho; p.NIMG = g.N;
  p.Cin = kStemWin; p.Cout = kStemCout; p.kh = kStemTaps; p.kw = 1; p.pad = 0; p.stride = 2;
  p.g_halves = 1;
  p.UW = kStemWin;
  p.chunks_per_tap = 1;
  p.n_units = kStemTaps;
  p.BN = kStemCout;
  p.G = 2;
  p.stages = 3;
  p.BW = g.Wo;
  // K stage: BH output rows (or BNI whole images) of Wo pixels, <= 128 rows
  if (g.Ho * g.Wo <= kTileM) {
    p.BH = g.Ho;
    p.BNI = kTileM / (g.Ho * g.Wo);
    if (p.BNI > g.N) p.BNI = g.N;
  } else {
    p.BH = kTileM / g.Wo;
    p.BNI = 1;
  }
  p.rows_a = p.rows_b = p.BNI * p.BH * p.BW;
  p.k_stage = (p.rows_a + 15) & ~15;
  p.a_box_bytes = (uint32_t(p.k_stage) * 64u + 1023u) & ~1023u;
  p.b_box_bytes = uint32_t(p.k_stage) * 128u;
  p.n_a_boxes = p.G * (kTileM / p.UW);
  p.tiles_h = (g.Ho + p.BH - 1) / p.BH;
  p.n_kboxes = p.tiles_h * ((g.N + p.BNI - 1) / p.BNI);
  pl.mgroups = 1;
  pl.ntiles = 1;
  int ks = num_sms();
  pl.ks_cap = ks;
  if (ks > p.n_kboxes) ks = p.n_kboxes;
  p.kboxes_per_cta = (p.n_kboxes + ks - 1) / ks;
  pl.ksplit = (p.n_kboxes + p.kboxes_per_cta - 1) / p.kboxes_per_cta;
  const size_t stage_bytes = size_t(p.n_a_boxes) * p.a_box_bytes + p.b_box_bytes;
  p.stages = int((226u * 1024u) / stage_bytes);
  if (p.stages > 4) p.stages = 4;
  pl.smem = size_t(p.stages) * stage_bytes + 1024;
  pl.ok = p.stages >= 2 && pl.smem <= 227u * 1024u;
  return pl;
}

size_t stem_wgrad_workspace_bytes(const StemGeom& g) {
  const WgradPlan pl = plan_stem_wgrad(g);
  return pl.ok ? size_t(pl.ks_cap) * kStemTaps * kStemWin * kStemCout * sizeof(float) : 0;
}

int launch_stem_wgrad(const uint16_t* gys, const uint16_t* xw, float* ws, size_t ws_bytes, int* ksplit_out,
                      const StemGeom& g, cudaStream_t st) {
  WgradPlan pl = plan_stem_wgrad(g);
  if (!pl.ok) { set_error("stem_conv_wgrad: geometry not supported"); return BDBNN_ERR_UNSUPPORTED; }
  if (ws_bytes < stem_wgrad_workspace_bytes(g)) {
    set_error("stem_conv_wgrad: workspace %zu B too small", ws_bytes);
    return BDBNN_ERR_WORKSPACE;
  }
  pl.p.fmt = BDBNN_FMT_FP16;
  pl.p.ws = ws;
  pl.p.trace = get_tc_trace();
  CUtensorMap tmX, tmG;
  int rc = make_window_map(&tmX, xw, g.N, g.HP, g.Wo, kStemWin, g.win_stride, g.row_stride, g.img_stride, pl.p.BW,
                           pl.p.BH, pl.p.BNI, 2);
  if (rc) return rc;
  rc = make_act_map(&tmG, gys, g.N, g.Ho, g.Wo, kStemCout, 64, pl.p.BW, pl.p.BH, pl.p.BNI);
  if (rc) return rc;
  *ksplit_out = pl.ksplit;
  return launch_wgrad_kernel(tmX, tmG, pl.p, pl.smem, dim3(unsigned(pl.ksplit), 1, 1), st);
}

}  // namespace bdbnn

using namespace bdbnn;

// Host-only view of the wgrad tiling decision (no CUDA call): lets the CPU test-suite sweep shapes.
extern "C" int bdbnn_debug_wgrad_plan(const bdbnn_conv_shape* s, int32_t grad_halves, int32_t* out, int32_t n_out) {
  BDBNN_REQUIRE(s && out && n_out >= 12, "debug_wgrad_plan: need a shape and room for 12 ints");
  BDBNN_REQUIRE(grad_halves == 1 || grad_halves == 2, "debug_wgrad_plan: grad_halves must be 1 or 2");
  const WgradPlan pl = plan_wgrad(s, grad_halves);
  const int32_t v[12] = {pl.ok ? 1 : 0, pl.ksplit, pl.ks_cap, pl.mgroups, pl.ntiles, int32_t(pl.smem), pl.p.G, pl.p.BN,
                         pl.p.UW, 0, pl.p.k_stage, pl.p.stages};
  memcpy(out, v, sizeof(v));
  return BDBNN_OK;
}

extern "C" size_t bdbnn_wgrad_tc_workspace_bytes(const bdbnn_conv_shape* s) {
  if (!s) return 0;
  // the split count may depend on the gradient mode (narrow-channel plan): size for the larger one
  const WgradPlan p2 = plan_wgrad(s, 2), p1 = plan_wgrad(s, 1);
  if (!p2.ok) return 0;
  const int cap = p1.ok && p1.ks_cap > p2.ks_cap ? p1.ks_cap : p2.ks_cap;
  return size_t(cap) * s->kh * s->kw * s->Cin * s->Cout * sizeof(float);
}

extern "C" int bdbnn_binconv_wgrad_tc(const uint16_t* gys_bf16, int32_t grad_mode, const uint32_t* amax_bits,
                                      const uint16_t* xb_bf16,
                                      const uint32_t* wmask_bits, const float* inv_gscale, float* gW,
                                      const bdbnn_conv_shape* s, void* workspace, size_t workspace_bytes,
                                      void* stream) {
  int rc = validate_shape(s);
  if (rc) return rc;
  BDBNN_REQUIRE(gys_bf16 && xb_bf16 && wmask_bits && inv_gscale && gW && workspace,
                "binconv_wgrad_tc: NULL pointer");
  BDBNN_REQUIRE(grad_mode >= BDBNN_GRAD_BF16 && grad_mode <= BDBNN_GRAD_FP16S, "binconv_wgrad_tc: bad grad_mode");
  BDBNN_REQUIRE(grad_mode != BDBNN_GRAD_FP16S || amax_bits, "binconv_wgrad_tc: FP16S needs amax_bits");
  const int grad_halves = grad_mode == BDBNN_GRAD_BF16X2 ? 2 : 1;
  WgradPlan pl = plan_wgrad(s, grad_halves);
  pl.p.fmt = grad_mode == BDBNN_GRAD_FP16S ? BDBNN_FMT_FP16 : BDBNN_FMT_BF16;
  if (!pl.ok) { set_error("binconv_wgrad_tc: shape not supported by the tensor-core path"); return BDBNN_ERR_UNSUPPORTED; }
  const size_t need = bdbnn_wgrad_tc_workspace_bytes(s);
  if (workspace_bytes < need) {
    set_error("binconv_wgrad_tc: workspace %zu B < required %zu B", workspace_bytes, need);
    return BDBNN_ERR_WORKSPACE;
  }
  cudaStream_t st = cudaStream_t(stream);
  pl.p.ws = static_cast<float*>(workspace);
  pl.p.trace = get_tc_trace();
  CUtensorMap tmX, tmG;
  rc = make_act_map(&tmX, xb_bf16, s->N, s->H, s->W, s->Cin, pl.p.UW, pl.p.BW, pl.p.BH, pl.p.BNI, s->stride);
  if (rc) return rc;
  rc = make_act_map(&tmG, gys_bf16, s->N, s->Ho, s->Wo, s->Cout * grad_halves, pl.p.BN < 64 ? pl.p.BN : 64, pl.p.BW,
                    pl.p.BH, pl.p.BNI);
  if (rc) return rc;
  rc = launch_wgrad_kernel(tmX, tmG, pl.p, pl.smem, dim3(unsigned(pl.ksplit), unsigned(pl.mgroups), unsigned(pl.ntiles)),
                           st);
  if (rc) return rc;
  const int64_t n = int64_t(s->Cout) * s->Cin * s->kh * s->kw;
  int64_t blocks = (n + 255) / 256;
  if (blocks > 2048) blocks = 2048;
  wgrad_finalize_kernel<<<unsigned(blocks), 256, 0, st>>>(
      pl.p.ws, pl.ksplit, wmask_bits, inv_gscale, grad_mode == BDBNN_GRAD_FP16S ? amax_bits : nullptr, gW, s->Cout, s->Cin,
      s->kh * s->kw);
  return check_launch("wgrad_finalize_kernel");
}
