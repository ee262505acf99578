// Statistics of the binary layers' weights for the training log (DESIGN.md §4w): sign flips per optimizer step,
// counted inside the (graphed) step, and per-layer distribution statistics taken at epoch end.  Both take up to
// BDBNN_MAX_TENSORS layers per launch through one kernel-parameter table, as the loss kernels do.  Contracts:
// include/bdbnn.h.
#include "common.cuh"

namespace bdbnn {

// ---- sign flips ------------------------------------------------------------------------------------------------
struct FlipTable {
  const float* w[BDBNN_MAX_TENSORS];
  uint32_t* bits[BDBNN_MAX_TENSORS];
  int64_t n[BDBNN_MAX_TENSORS];
  int32_t L;
};

constexpr int kFlipThreads = 256;
constexpr int kFlipWords = 8;    // consecutive bit words per warp and iteration

// Bit j of word k is 1 when element 32k + j is -1 under DESIGN.md §2's rule (v >= 0, -0 included, is +1; NaN is -1).
// A warp takes kFlipWords consecutive words at a time: their 1 KB of weights in coalesced 128-byte loads and their
// stored bits in one load, all issued before the first ballot; lane u then compares and stores word u.
__global__ void __launch_bounds__(kFlipThreads)
sign_flips_kernel(FlipTable tab, unsigned long long* __restrict__ flips, unsigned long long* __restrict__ steps,
                  int init) {
  __shared__ unsigned long long red[kFlipThreads / 32];
  const int l = blockIdx.y;
  const float* __restrict__ w = tab.w[l];
  uint32_t* __restrict__ bits = tab.bits[l];
  const int64_t n = tab.n[l];
  const int64_t words = (n + 31) >> 5;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t nwarps = (int64_t(gridDim.x) * blockDim.x) >> 5;
  unsigned long long cnt = 0;
  for (int64_t w0 = ((int64_t(blockIdx.x) * blockDim.x + threadIdx.x) >> 5) * kFlipWords; w0 < words;
       w0 += nwarps * kFlipWords) {
    float v[kFlipWords];
#pragma unroll
    for (int u = 0; u < kFlipWords; ++u) {
      const int64_t i = ((w0 + u) << 5) + lane;
      v[u] = i < n ? w[i] : 0.f;
    }
    const int64_t word = w0 + lane;
    const bool owner = lane < kFlipWords && word < words;
    const uint32_t prev = owner && !init ? bits[word] : 0u;
    uint32_t mine = 0u;
#pragma unroll
    for (int u = 0; u < kFlipWords; ++u) {
      const uint32_t b = __ballot_sync(0xffffffffu, (((w0 + u) << 5) + lane < n) && !(v[u] >= 0.f));
      if (lane == u) mine = b;
    }
    if (owner) {
      cnt += __popc(mine ^ prev);
      bits[word] = mine;
    }
  }
  if (init) return;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
  if (lane == 0) red[warp] = cnt;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long t = 0;
    for (int i = 0; i < kFlipThreads / 32; ++i) t += red[i];
    if (t) atomicAdd(flips + l, t);                 // integer sums: the same total in any order
    if (steps && blockIdx.x == 0 && l == 0) steps[0] += 1ull;
  }
}

// ---- distribution statistics -----------------------------------------------------------------------------------
struct StatsTable {
  const float* w[BDBNN_MAX_TENSORS];
  int64_t n[BDBNN_MAX_TENSORS];
  int64_t foff[BDBNN_MAX_TENSORS];   // the layer's first filter row in the per-filter workspace
  int32_t cout[BDBNN_MAX_TENSORS];
  int32_t L;
};

constexpr int kStatThreads = 256;
constexpr int kHistCols = BDBNN_WSTAT_HIST;                      // 64 bins, underflow, overflow, alpha = 0, NaN
constexpr int kFilterSums = 4;                                   // alpha_o, sum W^2, sum (W - a sign W)^2, #|W| <= 1

__device__ __forceinline__ void block_sums(double* v, int k, double (*red)[kStatThreads / 32]) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int j = 0; j < k; ++j) {
    const double s = warp_sum(v[j]);
    if (lane == 0) red[j][warp] = s;
  }
  __syncthreads();
  for (int j = 0; j < k; ++j) {
    double t = 0.0;
    for (int i = 0; i < kStatThreads / 32; ++i) t += red[j][i];   // every thread, the same order
    v[j] = t;
  }
  __syncthreads();
}

// One block per (filter o, layer l).  Pass 1: sum|W|, sum W^2, the |W| <= 1 count -> alpha_o.  Pass 2, with alpha_o
// known: the binarisation error and the histogram of fp32(W / alpha_o).  Each thread's elements and the reduction
// tree are fixed, so the sums have the same bits in every run.
__global__ void __launch_bounds__(kStatThreads)
filter_stats_kernel(StatsTable tab, double* __restrict__ fsum, uint32_t* __restrict__ fhist) {
  __shared__ double red[kFilterSums][kStatThreads / 32];
  __shared__ uint32_t hist[kHistCols];
  const int l = blockIdx.y, o = blockIdx.x;
  if (o >= tab.cout[l]) return;
  const int64_t m = tab.n[l] / tab.cout[l];
  const float* __restrict__ w = tab.w[l] + int64_t(o) * m;
  for (int j = threadIdx.x; j < kHistCols; j += blockDim.x) hist[j] = 0u;
  double s[3] = {0.0, 0.0, 0.0};
  for (int64_t i = threadIdx.x; i < m; i += blockDim.x) {
    const float v = w[i];
    const double d = double(v);
    s[0] += fabs(d);
    s[1] += d * d;
    s[2] += fabsf(v) <= 1.f ? 1.0 : 0.0;
  }
  block_sums(s, 3, red);
  const double alpha = s[0] / double(m);
  double e[1] = {0.0};
  for (int64_t i = threadIdx.x; i < m; i += blockDim.x) {
    const float v = w[i];
    const double r = double(v) - (v >= 0.f ? alpha : -alpha);
    e[0] += r * r;
    int col;
    if (alpha == 0.0) {
      col = 66;
    } else {
      const float q = __double2float_rn(double(v) / alpha);
      col = q != q ? 67 : q < -4.f ? 64 : q >= 4.f ? 65 : int(floorf(8.f * q)) + 32;
    }
    atomicAdd(&hist[col], 1u);
  }
  block_sums(e, 1, red);
  const int64_t row = tab.foff[l] + o;
  if (threadIdx.x == 0) {
    double* f = fsum + row * kFilterSums;
    f[0] = alpha; f[1] = s[1]; f[2] = e[0]; f[3] = s[2];
  }
  for (int j = threadIdx.x; j < kHistCols; j += blockDim.x) fhist[row * kHistCols + j] = hist[j];
}

// One block per layer: thread j < 68 adds histogram column j over the filters, thread 68 the sums; filters in order.
__global__ void __launch_bounds__(128)
stats_finalize_kernel(StatsTable tab, const double* __restrict__ fsum, const uint32_t* __restrict__ fhist,
                      double* __restrict__ stats_out, unsigned long long* __restrict__ hist_out) {
  const int l = blockIdx.x, j = threadIdx.x;
  const int C = tab.cout[l];
  const int64_t base = tab.foff[l];
  if (j < kHistCols) {
    unsigned long long t = 0;
    for (int o = 0; o < C; ++o) t += fhist[(base + o) * kHistCols + j];
    hist_out[int64_t(l) * kHistCols + j] = t;
  } else if (j == kHistCols) {
    const double n = double(tab.n[l]);
    double a = 0.0, s2 = 0.0, se = 0.0, act = 0.0;
    for (int o = 0; o < C; ++o) {
      const double* f = fsum + (base + o) * kFilterSums;
      a += f[0];
      s2 += f[1];
      se += f[2];
      act += f[3];
    }
    double* out = stats_out + int64_t(l) * BDBNN_WSTAT_VALUES;
    out[0] = act / n;                          // ste_active
    out[1] = a / double(C);                    // alpha_mean
    out[2] = s2 == 0.0 ? 0.0 : se / s2;        // bin_error
  }
}

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_sign_flips_multi(const float* const* w_ptrs_host, const int64_t* numel_host,
                                      uint32_t* const* bits_ptrs_host, int32_t L, uint64_t* flips, uint64_t* steps,
                                      int32_t init, void* stream) {
  BDBNN_REQUIRE(L >= 0, "sign_flips_multi: tensor count %d", L);
  if (L == 0) return BDBNN_OK;
  BDBNN_REQUIRE(w_ptrs_host && numel_host && bits_ptrs_host, "sign_flips_multi: NULL pointer");
  BDBNN_REQUIRE(init || flips, "sign_flips_multi: NULL flips (needed unless init)");
  for (int i = 0; i < L; ++i) {
    BDBNN_REQUIRE(numel_host[i] > 0, "sign_flips_multi: tensor %d has numel %lld", i, (long long)numel_host[i]);
    BDBNN_REQUIRE(w_ptrs_host[i] && bits_ptrs_host[i], "sign_flips_multi: pointer %d is NULL", i);
  }
  cudaStream_t st = cudaStream_t(stream);
  for (int32_t off = 0; off < L; off += BDBNN_MAX_TENSORS) {
    FlipTable tab;
    memset(&tab, 0, sizeof(tab));
    tab.L = L - off < BDBNN_MAX_TENSORS ? L - off : BDBNN_MAX_TENSORS;
    int64_t mx = 0;
    for (int l = 0; l < tab.L; ++l) {
      tab.w[l] = w_ptrs_host[off + l];
      tab.bits[l] = bits_ptrs_host[off + l];
      tab.n[l] = numel_host[off + l];
      const int64_t words = (tab.n[l] + 31) / 32;
      if (words > mx) mx = words;
    }
    const int64_t per_block = int64_t(kFlipThreads / 32) * kFlipWords;
    int64_t bx = (mx + per_block - 1) / per_block;
    const int64_t cap = (int64_t(num_sms()) * 8 + tab.L - 1) / tab.L;
    if (bx > cap) bx = cap;
    if (bx < 1) bx = 1;
    sign_flips_kernel<<<dim3(unsigned(bx), unsigned(tab.L)), kFlipThreads, 0, st>>>(
        tab, reinterpret_cast<unsigned long long*>(flips ? flips + off : nullptr),
        reinterpret_cast<unsigned long long*>(off == 0 ? steps : nullptr), init);
    const int rc = check_launch("sign_flips_kernel");
    if (rc) return rc;
  }
  return BDBNN_OK;
}

extern "C" int bdbnn_weight_stats_multi(const float* const* w_ptrs_host, const int64_t* numel_host,
                                        const int32_t* cout_host, int32_t L, double* filter_sums,
                                        uint32_t* filter_hist, double* stats_out, uint64_t* hist_out, void* stream) {
  BDBNN_REQUIRE(L >= 0, "weight_stats_multi: tensor count %d", L);
  if (L == 0) return BDBNN_OK;
  BDBNN_REQUIRE(w_ptrs_host && numel_host && cout_host && filter_sums && filter_hist && stats_out && hist_out,
                "weight_stats_multi: NULL pointer");
  for (int i = 0; i < L; ++i) {
    BDBNN_REQUIRE(numel_host[i] > 0 && cout_host[i] > 0 && numel_host[i] % cout_host[i] == 0,
                  "weight_stats_multi: tensor %d: numel %lld is not a positive multiple of Cout %d", i,
                  (long long)numel_host[i], cout_host[i]);
    BDBNN_REQUIRE(w_ptrs_host[i] != nullptr, "weight_stats_multi: pointer %d is NULL", i);
  }
  cudaStream_t st = cudaStream_t(stream);
  int64_t foff = 0;
  for (int32_t off = 0; off < L; off += BDBNN_MAX_TENSORS) {
    StatsTable tab;
    memset(&tab, 0, sizeof(tab));
    tab.L = L - off < BDBNN_MAX_TENSORS ? L - off : BDBNN_MAX_TENSORS;
    int32_t mx = 0;
    for (int l = 0; l < tab.L; ++l) {
      tab.w[l] = w_ptrs_host[off + l];
      tab.n[l] = numel_host[off + l];
      tab.cout[l] = cout_host[off + l];
      tab.foff[l] = foff;
      foff += tab.cout[l];
      if (tab.cout[l] > mx) mx = tab.cout[l];
    }
    filter_stats_kernel<<<dim3(unsigned(mx), unsigned(tab.L)), kStatThreads, 0, st>>>(tab, filter_sums, filter_hist);
    int rc = check_launch("filter_stats_kernel");
    if (rc) return rc;
    stats_finalize_kernel<<<tab.L, 128, 0, st>>>(tab, filter_sums, filter_hist,
                                                 stats_out + int64_t(off) * BDBNN_WSTAT_VALUES,
                                                 reinterpret_cast<unsigned long long*>(hist_out) +
                                                     int64_t(off) * kHistCols);
    rc = check_launch("stats_finalize_kernel");
    if (rc) return rc;
  }
  return BDBNN_OK;
}
