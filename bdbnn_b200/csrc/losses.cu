// Fused multi-tensor loss kernels: kurtosis regulariser, KD logits loss, KD per-layer weight loss.
// All are tiny-tensor, launch-latency-bound in the reference (≈400 ATen launches per step, SURVEY.md
// §2.1); here each is 1-2 launches per BDBNN_MAX_TENSORS layers (one table).  Contracts: include/bdbnn.h.
#include "common.cuh"

namespace bdbnn {

struct TensorTable {
  const float* a[BDBNN_MAX_TENSORS];  // primary tensor (weights / teacher weights)
  const float* b[BDBNN_MAX_TENSORS];  // secondary tensor (student weights) or unused
  float* g[BDBNN_MAX_TENSORS];        // gradient destination or unused
  int64_t n[BDBNN_MAX_TENSORS];
  float target[BDBNN_MAX_TENSORS];
  int32_t L;
};

constexpr int kLossThreads = 256;
constexpr int kMomentStride = 8;  // doubles per tensor in the `moments` scratch

// Block sums of four values, stored to dst[0..3] (each block owns its dst: the cross-block sum is taken in a
// fixed order by det_sums_finish, so results are the same in every run).
__device__ __forceinline__ void block_store_sum4(double v0, double v1, double v2, double v3,
                                                 double* dst) {
  __shared__ double red[4][kLossThreads / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  v0 = warp_sum(v0); v1 = warp_sum(v1); v2 = warp_sum(v2); v3 = warp_sum(v3);
  if (lane == 0) { red[0][warp] = v0; red[1][warp] = v1; red[2][warp] = v2; red[3][warp] = v3; }
  __syncthreads();
  if (warp == 0) {
    const int nw = blockDim.x >> 5;
    double t0 = lane < nw ? red[0][lane] : 0.0, t1 = lane < nw ? red[1][lane] : 0.0;
    double t2 = lane < nw ? red[2][lane] : 0.0, t3 = lane < nw ? red[3][lane] : 0.0;
    t0 = warp_sum(t0); t1 = warp_sum(t1); t2 = warp_sum(t2); t3 = warp_sum(t3);
    if (lane == 0) {
      dst[0] = t0; dst[1] = t1; dst[2] = t2; dst[3] = t3;
    }
  }
}

// Pass 1: shifted raw power sums S_k = sum (w - w[0])^k, k=1..4, fp64 accumulation.
__global__ void __launch_bounds__(kLossThreads)
kurt_moments_kernel(TensorTable tab, double* __restrict__ part) {   // part: [gridDim.x][L][kMomentStride]
  const int l = blockIdx.y;
  const float* __restrict__ w = tab.a[l];
  const int64_t n = tab.n[l];
  const float pivot = n > 0 ? w[0] : 0.f;
  double s1 = 0, s2 = 0, s3 = 0, s4 = 0;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    const double d = double(w[i] - pivot);
    const double d2 = d * d;
    s1 += d; s2 += d2; s3 += d2 * d; s4 += d2 * d2;
  }
  block_store_sum4(s1, s2, s3, s4, part + (int64_t(blockIdx.x) * gridDim.y + l) * kMomentStride);
}

// Pass 2 (one thread per tensor): central moments -> mu, s (unbiased), K, mean z^3, loss.
__global__ void kurt_finalize_kernel(TensorTable tab, double* __restrict__ moments,
                                     float* __restrict__ kurt_out, float* __restrict__ loss_out) {
  const int l = threadIdx.x;
  if (l >= tab.L) return;
  double* m = moments + l * kMomentStride;
  const double n = double(tab.n[l]);
  const double pivot = tab.n[l] > 0 ? double(tab.a[l][0]) : 0.0;
  const double a1 = m[0] / n, r2 = m[1] / n, r3 = m[2] / n, r4 = m[3] / n;
  const double c2 = r2 - a1 * a1;
  const double c3 = r3 - 3.0 * a1 * r2 + 2.0 * a1 * a1 * a1;
  const double c4 = r4 - 4.0 * a1 * r3 + 6.0 * a1 * a1 * r2 - 3.0 * a1 * a1 * a1 * a1;
  const double var = c2 * n / (n - 1.0);  // torch.std default: unbiased (kurtosis.py:25)
  const double sd = sqrt(var);
  const double K = c4 / (var * var);      // mean(((w-mu)/s)^4)  (kurtosis.py:26)
  const double mz3 = c3 / (var * sd);
  const double diff = K - double(tab.target[l]);
  m[0] = pivot + a1;  // mu
  m[1] = sd;
  m[2] = K;
  m[3] = mz3;
  m[4] = n;
  kurt_out[l] = float(K);
  loss_out[l] = float(diff * diff);       // (kurtosis.py:28)
}

__global__ void __launch_bounds__(kLossThreads)
kurt_bwd_kernel(TensorTable tab, const double* __restrict__ moments, const float* __restrict__ gout,
                int accumulate) {
  const int l = blockIdx.y;
  const float* __restrict__ w = tab.a[l];
  float* __restrict__ g = tab.g[l];
  const int64_t n = tab.n[l];
  const double* m = moments + l * kMomentStride;
  const double mu = m[0], sd = m[1], K = m[2], mz3 = m[3], nn = m[4];
  // dL/dw_j = gout * 2(K-T) * 4/(n s) * ( z^3 - mean(z^3) - z K n/(n-1) )
  const double coef = double(gout[l]) * 2.0 * (K - double(tab.target[l])) * 4.0 / (nn * sd);
  const float fcoef = float(coef), fmu = float(mu), finv = float(1.0 / sd), fmz3 = float(mz3);
  const float fk = float(K * nn / (nn - 1.0));
  // residual of mu in fp32 keeps (w - mu) accurate when |mu| is not tiny
  const float fmu_lo = float(mu - double(fmu));
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    const float z = ((w[i] - fmu) - fmu_lo) * finv;
    const float v = fcoef * (z * z * z - fmz3 - z * fk);
    g[i] = accumulate ? g[i] + v : v;
  }
}

// ---- KD logits ---------------------------------------------------------------------------------
__device__ __forceinline__ float block_reduce_max(float v, float* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  v = warp_max(v);
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  float t = lane < nw ? sh[lane] : -INFINITY;
  t = warp_max(t);
  return t;
}
__device__ __forceinline__ float block_reduce_sum(float v, float* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  v = warp_sum(v);
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  float t = lane < nw ? sh[lane] : 0.f;
  t = warp_sum(t);
  return t;
}

// One block per row: loss_n = -sum_c softmax(t)_c * log_softmax(s)_c ; grad = (softmax(s)-softmax(t))/N
__global__ void __launch_bounds__(128)
kd_logits_row_kernel(const float* __restrict__ s, const float* __restrict__ t, int32_t N, int32_t C,
                     float* __restrict__ row_loss, float* __restrict__ grad_s) {
  __shared__ float sh[32];
  const int n = blockIdx.x;
  const float* sr = s + int64_t(n) * C;
  const float* tr = t + int64_t(n) * C;
  float ms = -INFINITY, mt = -INFINITY;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    ms = fmaxf(ms, sr[c]);
    mt = fmaxf(mt, tr[c]);
  }
  ms = block_reduce_max(ms, sh);
  mt = block_reduce_max(mt, sh);
  float es = 0.f, et = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    es += expf(sr[c] - ms);
    et += expf(tr[c] - mt);
  }
  es = block_reduce_sum(es, sh);
  et = block_reduce_sum(et, sh);
  const float lse_s = ms + logf(es);
  const float inv_et = 1.0f / et, inv_es = 1.0f / es, invN = 1.0f / float(N);
  float acc = 0.f;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const float pt = expf(tr[c] - mt) * inv_et;
    acc -= pt * (sr[c] - lse_s);
    if (grad_s) grad_s[int64_t(n) * C + c] = (expf(sr[c] - ms) * inv_es - pt) * invN;
  }
  acc = block_reduce_sum(acc, sh);
  if (threadIdx.x == 0) row_loss[n] = acc;
}

__global__ void __launch_bounds__(256)
mean_rows_kernel(const float* __restrict__ row_loss, int32_t N, float* __restrict__ out) {
  __shared__ double red[8];
  double a = 0.0;
  for (int i = threadIdx.x; i < N; i += blockDim.x) a += double(row_loss[i]);
  a = warp_sum(a);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = a;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < int(blockDim.x >> 5); ++i) t += red[i];
    out[0] = float(t / double(N));  // size_average=True (KD_loss.py:18,36)
  }
}

// ---- KD per-layer ------------------------------------------------------------------------------
__global__ void __launch_bounds__(kLossThreads)
kd_layer_fwd_kernel(TensorTable tab, double* __restrict__ part) {   // part: [gridDim.x][L]
  __shared__ double red[kLossThreads / 32];
  const int l = blockIdx.y;
  const float* __restrict__ wt = tab.a[l];
  const float* __restrict__ ws = tab.b[l];
  const int64_t n = tab.n[l];
  double acc = 0.0;
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    const float t = wt[i];
    acc += double(expf(t) * (t - ws[i]));  // KLDivLoss(log_target=True): exp(tgt)*(tgt-inp)
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double t = 0.0;
    for (int i = 0; i < int(blockDim.x >> 5); ++i) t += red[i];
    part[int64_t(blockIdx.x) * gridDim.y + l] = t;
  }
}

// partial[off + l] = sum of layer l of this table -> its mean (reduction='mean' per layer).  The call's last table
// (out != NULL) then adds the means of all off + L layers in layer order: one sum, whatever the number of tables.
__global__ void kd_layer_finalize_kernel(TensorTable tab, double* __restrict__ partial, int32_t off,
                                         float* __restrict__ out) {
  if (threadIdx.x != 0) return;
  for (int l = 0; l < tab.L; ++l) partial[off + l] /= double(tab.n[l]);
  if (out == nullptr) return;
  double t = 0.0;
  for (int l = 0; l < off + tab.L; ++l) t += partial[l];
  out[0] = float(t);
}

__global__ void __launch_bounds__(kLossThreads)
kd_layer_bwd_kernel(TensorTable tab, const float* __restrict__ gout, int accumulate) {
  const int l = blockIdx.y;
  const float* __restrict__ wt = tab.a[l];
  float* __restrict__ g = tab.g[l];
  const int64_t n = tab.n[l];
  const float coef = -gout[0] / float(n);
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n;
       i += int64_t(gridDim.x) * blockDim.x) {
    const float v = coef * expf(wt[i]);
    g[i] = accumulate ? g[i] + v : v;
  }
}

static unsigned blocks_for(int64_t max_n, int L) {
  int64_t bx = (max_n + int64_t(kLossThreads) * 4 - 1) / (int64_t(kLossThreads) * 4);
  const int64_t cap = (int64_t(num_sms()) * 8 + L - 1) / (L > 0 ? L : 1);
  if (bx > cap) bx = cap;
  if (bx < 1) bx = 1;
  return unsigned(bx);
}

// Every entry of a call's host arrays checked (b and g where given) before anything is enqueued.
static int check_entries(const float* const* a, const float* const* b, float* const* g, const int64_t* n,
                         int32_t L) {
  for (int i = 0; i < L; ++i) {
    BDBNN_REQUIRE(n[i] > 0, "tensor %d has numel %lld", i, (long long)n[i]);
    BDBNN_REQUIRE(a[i] != nullptr, "tensor %d pointer is NULL", i);
    BDBNN_REQUIRE(!b || b[i], "student pointer %d is NULL", i);
    BDBNN_REQUIRE(!g || g[i], "grad pointer %d is NULL", i);
  }
  return BDBNN_OK;
}

// Tensors [off, min(off + BDBNN_MAX_TENSORS, L)) as one table; returns its grid.x.  An entry point launches its
// kernels once per table, tables in order.
static unsigned fill_table(TensorTable& tab, const float* const* a, const float* const* b, float* const* g,
                           const int64_t* n, const float* targets, int32_t off, int32_t L) {
  memset(&tab, 0, sizeof(tab));
  tab.L = L - off < BDBNN_MAX_TENSORS ? L - off : BDBNN_MAX_TENSORS;
  int64_t mx = 0;
  for (int l = 0; l < tab.L; ++l) {
    const int i = off + l;
    tab.a[l] = a[i];
    tab.b[l] = b ? b[i] : nullptr;
    tab.g[l] = g ? g[i] : nullptr;
    tab.n[l] = n[i];
    tab.target[l] = targets ? targets[i] : 0.f;
    if (n[i] > mx) mx = n[i];
  }
  return blocks_for(mx, tab.L);
}

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_kurtosis_multi_fwd(const float* const* w_ptrs_host, const int64_t* numel_host,
                                        const float* targets_host, int32_t L, double* moments,
                                        float* kurt_out, float* loss_out, void* stream) {
  BDBNN_REQUIRE(L >= 0, "kurtosis_multi_fwd: tensor count %d", L);
  if (L == 0) return BDBNN_OK;
  BDBNN_REQUIRE(w_ptrs_host && numel_host && targets_host && moments && kurt_out && loss_out,
                "kurtosis_multi_fwd: NULL pointer");
  int rc = check_entries(w_ptrs_host, nullptr, nullptr, numel_host, L);
  if (rc) return rc;
  cudaStream_t st = cudaStream_t(stream);
  BDBNN_CUDA(cudaMemsetAsync(moments, 0, size_t(L) * kMomentStride * sizeof(double), st));
  for (int32_t off = 0; off < L; off += BDBNN_MAX_TENSORS) {
    TensorTable tab;
    const unsigned bx = fill_table(tab, w_ptrs_host, nullptr, nullptr, numel_host, targets_host, off, L);
    dim3 grid(bx, unsigned(tab.L));
    double* m = moments + int64_t(off) * kMomentStride;
    const int width = tab.L * kMomentStride;
    double* part = nullptr;
    rc = det_sums_alloc(&part, grid.x, width, st);
    if (rc) return rc;
    const cudaError_t em = cudaMemsetAsync(part, 0, size_t(grid.x) * width * sizeof(double), st);
    kurt_moments_kernel<<<grid, kLossThreads, 0, st>>>(tab, part);
    rc = em != cudaSuccess ? (set_error("kurtosis: cudaMemsetAsync failed: %s", cudaGetErrorString(em)), BDBNN_ERR_CUDA)
                           : check_launch("kurt_moments_kernel");
    if (rc) { cudaFreeAsync(part, st); return rc; }
    rc = det_sums_finish(part, grid.x, width, m, st);
    if (rc) return rc;
    kurt_finalize_kernel<<<1, BDBNN_MAX_TENSORS, 0, st>>>(tab, m, kurt_out + off, loss_out + off);
    rc = check_launch("kurt_finalize_kernel");
    if (rc) return rc;
  }
  return BDBNN_OK;
}

extern "C" int bdbnn_kurtosis_multi_bwd(const float* const* w_ptrs_host, const int64_t* numel_host,
                                        const float* targets_host, int32_t L, const double* moments,
                                        const float* gout, float* const* grad_ptrs_host,
                                        int32_t accumulate, void* stream) {
  BDBNN_REQUIRE(L >= 0, "kurtosis_multi_bwd: tensor count %d", L);
  if (L == 0) return BDBNN_OK;
  BDBNN_REQUIRE(w_ptrs_host && numel_host && targets_host && moments && gout && grad_ptrs_host,
                "kurtosis_multi_bwd: NULL pointer");
  int rc = check_entries(w_ptrs_host, nullptr, grad_ptrs_host, numel_host, L);
  if (rc) return rc;
  for (int32_t off = 0; off < L; off += BDBNN_MAX_TENSORS) {
    TensorTable tab;
    const unsigned bx = fill_table(tab, w_ptrs_host, nullptr, grad_ptrs_host, numel_host, targets_host, off, L);
    dim3 grid(bx, unsigned(tab.L));
    kurt_bwd_kernel<<<grid, kLossThreads, 0, cudaStream_t(stream)>>>(tab, moments + int64_t(off) * kMomentStride,
                                                                     gout + off, accumulate);
    rc = check_launch("kurt_bwd_kernel");
    if (rc) return rc;
  }
  return BDBNN_OK;
}

extern "C" int bdbnn_kd_logits_fwd_bwd(const float* s, const float* t, int32_t N, int32_t C,
                                       float* row_ws, float* loss_out, float* grad_s, void* stream) {
  BDBNN_REQUIRE(N > 0 && C > 0, "kd_logits: bad N/C");
  BDBNN_REQUIRE(s && t && row_ws && loss_out, "kd_logits: NULL pointer");
  cudaStream_t st = cudaStream_t(stream);
  kd_logits_row_kernel<<<N, 128, 0, st>>>(s, t, N, C, row_ws, grad_s);
  int rc = check_launch("kd_logits_row_kernel");
  if (rc) return rc;
  mean_rows_kernel<<<1, 256, 0, st>>>(row_ws, N, loss_out);
  return check_launch("mean_rows_kernel");
}

extern "C" int bdbnn_kd_layer_multi_fwd(const float* const* ws_ptrs_host,
                                        const float* const* wt_ptrs_host, const int64_t* numel_host,
                                        int32_t L, double* partial, float* loss_out, void* stream) {
  BDBNN_REQUIRE(loss_out != nullptr, "kd_layer_multi_fwd: NULL loss_out");
  BDBNN_REQUIRE(L >= 0, "kd_layer_multi_fwd: tensor count %d", L);
  cudaStream_t st = cudaStream_t(stream);
  if (L == 0) {
    BDBNN_CUDA(cudaMemsetAsync(loss_out, 0, sizeof(float), st));
    return BDBNN_OK;
  }
  BDBNN_REQUIRE(ws_ptrs_host && wt_ptrs_host && numel_host && partial,
                "kd_layer_multi_fwd: NULL pointer");
  int rc = check_entries(wt_ptrs_host, ws_ptrs_host, nullptr, numel_host, L);
  if (rc) return rc;
  BDBNN_CUDA(cudaMemsetAsync(partial, 0, size_t(L) * sizeof(double), st));
  for (int32_t off = 0; off < L; off += BDBNN_MAX_TENSORS) {
    TensorTable tab;
    const unsigned bx = fill_table(tab, wt_ptrs_host, ws_ptrs_host, nullptr, numel_host, nullptr, off, L);
    const int32_t cnt = tab.L;
    dim3 grid(bx, unsigned(cnt));
    double* part = nullptr;
    rc = det_sums_alloc(&part, grid.x, cnt, st);
    if (rc) return rc;
    kd_layer_fwd_kernel<<<grid, kLossThreads, 0, st>>>(tab, part);
    rc = check_launch("kd_layer_fwd_kernel");
    if (rc) { cudaFreeAsync(part, st); return rc; }
    rc = det_sums_finish(part, grid.x, cnt, partial + off, st);
    if (rc) return rc;
    kd_layer_finalize_kernel<<<1, 32, 0, st>>>(tab, partial, off, off + cnt == L ? loss_out : nullptr);
    rc = check_launch("kd_layer_finalize_kernel");
    if (rc) return rc;
  }
  return BDBNN_OK;
}

extern "C" int bdbnn_kd_layer_multi_bwd(const float* const* wt_ptrs_host, const int64_t* numel_host,
                                        int32_t L, const float* gout, float* const* grad_ptrs_host,
                                        int32_t accumulate, void* stream) {
  BDBNN_REQUIRE(L >= 0, "kd_layer_multi_bwd: tensor count %d", L);
  if (L == 0) return BDBNN_OK;
  BDBNN_REQUIRE(wt_ptrs_host && numel_host && gout && grad_ptrs_host,
                "kd_layer_multi_bwd: NULL pointer");
  int rc = check_entries(wt_ptrs_host, nullptr, grad_ptrs_host, numel_host, L);
  if (rc) return rc;
  for (int32_t off = 0; off < L; off += BDBNN_MAX_TENSORS) {
    TensorTable tab;
    const unsigned bx = fill_table(tab, wt_ptrs_host, nullptr, grad_ptrs_host, numel_host, nullptr, off, L);
    dim3 grid(bx, unsigned(tab.L));
    kd_layer_bwd_kernel<<<grid, kLossThreads, 0, cudaStream_t(stream)>>>(tab, gout, accumulate);
    rc = check_launch("kd_layer_bwd_kernel");
    if (rc) return rc;
  }
  return BDBNN_OK;
}
