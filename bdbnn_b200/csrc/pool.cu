// NHWC max-pool forward / backward (fp32).  Not part of the binary-conv maths, but it sits on the
// timed train step right after the stem (822 MB activation at ResNet-18 N=256), where ATen's
// max_pool_backward_nhwc scatters with atomics instead of reading each input position once.
//   forward : y = max over the k x k window (first maximum in scan order wins, NaN propagates — the
//             torch.nn.MaxPool2d rule), idx = winning tap (r*k+s) as one byte per element
//   backward: gather form, no atomics: gx[h,w] = sum of gy[ho,wo] over the (<= ceil(k/s)^2) windows
//             whose winner is (h,w)
#include "common.cuh"

namespace bdbnn {

__global__ void __launch_bounds__(256)
maxpool_fwd_kernel(const float4* __restrict__ x, float4* __restrict__ y, uint32_t* __restrict__ idx,
                   int N, int H, int W, int C4, int Ho, int Wo, int k, int s, int p, int64_t total) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += int64_t(gridDim.x) * blockDim.x) {
    const int c = int(i % C4);
    int64_t q = i / C4;
    const int wo = int(q % Wo); q /= Wo;
    const int ho = int(q % Ho);
    const int n = int(q / Ho);
    float4 m = make_float4(-INFINITY, -INFINITY, -INFINITY, -INFINITY);
    uint32_t w4 = 0;
    bool first = true;
    for (int r = 0; r < k; ++r) {
      const int h = ho * s - p + r;
      if (h < 0 || h >= H) continue;
      for (int t = 0; t < k; ++t) {
        const int w = wo * s - p + t;
        if (w < 0 || w >= W) continue;
        const float4 v = __ldg(x + ((int64_t(n) * H + h) * W + w) * C4 + c);
        const uint32_t tap = uint32_t(r * k + t);
        if (first || v.x > m.x || v.x != v.x) { m.x = v.x; w4 = (w4 & 0xffffff00u) | tap; }
        if (first || v.y > m.y || v.y != v.y) { m.y = v.y; w4 = (w4 & 0xffff00ffu) | (tap << 8); }
        if (first || v.z > m.z || v.z != v.z) { m.z = v.z; w4 = (w4 & 0xff00ffffu) | (tap << 16); }
        if (first || v.w > m.w || v.w != v.w) { m.w = v.w; w4 = (w4 & 0x00ffffffu) | (tap << 24); }
        first = false;
      }
    }
    y[i] = m;
    idx[i] = w4;
  }
}

__global__ void __launch_bounds__(256)
maxpool_bwd_kernel(const float4* __restrict__ gy, const uint32_t* __restrict__ idx, float4* __restrict__ gx,
                   int N, int H, int W, int C4, int Ho, int Wo, int k, int s, int p, int64_t total) {
  for (int64_t i = int64_t(blockIdx.x) * blockDim.x + threadIdx.x; i < total;
       i += int64_t(gridDim.x) * blockDim.x) {
    const int c = int(i % C4);
    int64_t q = i / C4;
    const int w = int(q % W); q /= W;
    const int h = int(q % H);
    const int n = int(q / H);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    int ho0 = (h + p - k + s) / s;           // ceil((h + p - k + 1) / s) for non-negative numerators
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
        const float4 g = __ldg(gy + o);
        if ((w4 & 0xffu) == tap) acc.x += g.x;
        if (((w4 >> 8) & 0xffu) == tap) acc.y += g.y;
        if (((w4 >> 16) & 0xffu) == tap) acc.z += g.z;
        if ((w4 >> 24) == tap) acc.w += g.w;
      }
    }
    gx[i] = acc;
  }
}

}  // namespace bdbnn

using namespace bdbnn;

static int pool_args_ok(int N, int H, int W, int C, int k, int s, int p, int Ho, int Wo) {
  BDBNN_REQUIRE(N > 0 && H > 0 && W > 0 && C > 0 && (C & 3) == 0, "maxpool: C must be a positive multiple of 4");
  BDBNN_REQUIRE(k > 0 && k <= 15 && s > 0 && p >= 0 && 2 * p <= k, "maxpool: bad k/stride/pad");
  BDBNN_REQUIRE(Ho == (H + 2 * p - k) / s + 1 && Wo == (W + 2 * p - k) / s + 1 && Ho > 0 && Wo > 0,
                "maxpool: inconsistent output size");
  return BDBNN_OK;
}

extern "C" int bdbnn_maxpool_fwd(const float* x, float* y, uint8_t* idx, int32_t N, int32_t H, int32_t W,
                                 int32_t C, int32_t k, int32_t stride, int32_t pad, int32_t Ho, int32_t Wo,
                                 void* stream) {
  int rc = pool_args_ok(N, H, W, C, k, stride, pad, Ho, Wo);
  if (rc) return rc;
  BDBNN_REQUIRE(x && y && idx, "maxpool_fwd: NULL pointer");
  const int64_t total = int64_t(N) * Ho * Wo * (C / 4);
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = int64_t(num_sms()) * 8 * 8;
  if (blocks > cap) blocks = cap;
  maxpool_fwd_kernel<<<unsigned(blocks), 256, 0, cudaStream_t(stream)>>>(
      reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y), reinterpret_cast<uint32_t*>(idx), N, H,
      W, C / 4, Ho, Wo, k, stride, pad, total);
  return check_launch("maxpool_fwd_kernel");
}

extern "C" int bdbnn_maxpool_bwd(const float* gy, const uint8_t* idx, float* gx, int32_t N, int32_t H,
                                 int32_t W, int32_t C, int32_t k, int32_t stride, int32_t pad, int32_t Ho,
                                 int32_t Wo, void* stream) {
  int rc = pool_args_ok(N, H, W, C, k, stride, pad, Ho, Wo);
  if (rc) return rc;
  BDBNN_REQUIRE(gy && idx && gx, "maxpool_bwd: NULL pointer");
  const int64_t total = int64_t(N) * H * W * (C / 4);
  int64_t blocks = (total + 255) / 256;
  const int64_t cap = int64_t(num_sms()) * 8 * 8;
  if (blocks > cap) blocks = cap;
  maxpool_bwd_kernel<<<unsigned(blocks), 256, 0, cudaStream_t(stream)>>>(
      reinterpret_cast<const float4*>(gy), reinterpret_cast<const uint32_t*>(idx), reinterpret_cast<float4*>(gx),
      N, H, W, C / 4, Ho, Wo, k, stride, pad, total);
  return check_launch("maxpool_bwd_kernel");
}
