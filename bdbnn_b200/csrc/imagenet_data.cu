// ImageNet input batch from decoded uint8 images: RandomResizedCrop(224) + RandomHorizontalFlip (training) or
// Resize(256) + CenterCrop(224) (evaluation), then ToTensor and Normalize, in one launch.  See include/bdbnn.h for the
// contract and DESIGN.md §4m for the spec; oracle/imagenet_data_ref.py restates it on the CPU bit for bit.
//
// The resize is Pillow's antialiased bilinear resample of a uint8 image (what torchvision runs on PIL images): per
// axis, coefficients in fp64 (Pillow's precompute_coeffs), rounded to int32 with 22 fractional bits; a horizontal
// pass into a uint8 intermediate, then a vertical pass, each accumulated in int32 from 2^21, shifted right by 22 and
// clipped to [0, 255].  Every fp64 step is an explicit __d*_rn so that nvcc cannot contract it into an FMA.
//
// Grid (bands, B): a block computes a band of TB output rows of one image, all 224 columns, 3 channels.  It computes
// the horizontal coefficients of the window's 224 columns and the vertical ones of its TB rows into shared memory,
// runs the horizontal pass over the source rows the band needs into a uint8 shared tile [rows][224][3], then the
// vertical pass, normalises and writes fp32 through the output's strides.  The host picks TB per launch from the
// largest filter support in the batch so that the tile fits (DESIGN.md §4m).
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace bdbnn {

constexpr int kInOut = 224;                       // output window side
constexpr int kInThreads = 256;
constexpr int kInPrec = 22;                       // Pillow's PRECISION_BITS for 8-bit images
constexpr int kInMaxSide = 8192;
constexpr int kInMaxResized = 1 << 22;
constexpr size_t kInSmemPreferred = 96 * 1024;    // two blocks per SM
constexpr size_t kInSmemMax = 227 * 1024;

struct InNorm {
  float mean[3], std[3];
};

struct InLayout {
  int TB, Kh, Kv, rows;                           // band rows, horizontal / vertical taps bound, tile rows bound
};

// Coefficients of output pixel xx of a 1-D resample in_size -> out_size (Pillow's precompute_coeffs with box
// (0, in_size), bilinear filter, support 1): first tap and tap count returned, int32 weights written to k[0, count).
__device__ int in_coeffs(int in_size, int out_size, int xx, int32_t* k, int* xmin_out) {
  const double scale = __ddiv_rn(double(in_size), double(out_size));
  const double fs = scale < 1.0 ? 1.0 : scale;    // filterscale; support = 1.0 * filterscale
  const double ss = __ddiv_rn(1.0, fs);
  const double center = __dmul_rn(__dadd_rn(double(xx), 0.5), scale);
  int xmin = int(__dadd_rn(__dadd_rn(center, -fs), 0.5));
  if (xmin < 0) xmin = 0;
  int xmax = int(__dadd_rn(__dadd_rn(center, fs), 0.5));
  if (xmax > in_size) xmax = in_size;
  const int n = xmax - xmin;
  double ww = 0.0;
  for (int x = 0; x < n; ++x) {
    const double v = fabs(__dmul_rn(__dadd_rn(__dadd_rn(double(x + xmin), -center), 0.5), ss));
    ww = __dadd_rn(ww, v < 1.0 ? __dadd_rn(1.0, -v) : 0.0);
  }
  for (int x = 0; x < n; ++x) {
    const double v = fabs(__dmul_rn(__dadd_rn(__dadd_rn(double(x + xmin), -center), 0.5), ss));
    double w = v < 1.0 ? __dadd_rn(1.0, -v) : 0.0;
    if (ww != 0.0) w = __ddiv_rn(w, ww);
    k[x] = int32_t(__dadd_rn(0.5, __dmul_rn(w, double(1 << kInPrec))));   // w >= 0: Pillow's (int)(0.5 + w * 2^22)
  }
  *xmin_out = xmin;
  return n;
}

__device__ __forceinline__ uint32_t in_clip8(int32_t acc) {
  const int32_t v = acc >> kInPrec;
  return uint32_t(v < 0 ? 0 : (v > 255 ? 255 : v));
}

__global__ void __launch_bounds__(kInThreads)
imagenet_batch_kernel(const bdbnn_imagenet_desc* __restrict__ descs, InLayout L, InNorm norm,
                      float* __restrict__ out, int64_t sN, int64_t sC, int64_t sH, int64_t sW,
                      int64_t* __restrict__ target) {
  extern __shared__ __align__(16) uint8_t in_smem[];
  int32_t* hw = reinterpret_cast<int32_t*>(in_smem);      // [224][Kh] horizontal weights
  int32_t* hx = hw + kInOut * L.Kh;                      // [224] first tap (crop column)
  int32_t* hn = hx + kInOut;                             // [224] tap count
  int32_t* vw = hn + kInOut;                             // [TB][Kv] vertical weights
  int32_t* vy = vw + L.TB * L.Kv;                        // [TB] first tap (crop row)
  int32_t* vn = vy + L.TB;                               // [TB] tap count
  uint8_t* tile = reinterpret_cast<uint8_t*>(vn + L.TB); // [rows][224][3] horizontal pass

  const int b = blockIdx.y;
  const bdbnn_imagenet_desc d = descs[b];
  const int r0 = blockIdx.x * L.TB;
  const int nr = min(L.TB, kInOut - r0);
  const int t = threadIdx.x;
  if (t < kInOut) {
    int xmin;
    hn[t] = in_coeffs(d.w, d.RW, d.ox0 + t, hw + t * L.Kh, &xmin);
    hx[t] = xmin;
  } else if (t - kInOut < nr) {
    const int r = t - kInOut;
    int ymin;
    vn[r] = in_coeffs(d.h, d.RH, d.oy0 + r0 + r, vw + r * L.Kv, &ymin);
    vy[r] = ymin;
  }
  if (blockIdx.x == 0 && t == 0) target[b] = d.label;
  __syncthreads();

  // Horizontal pass over crop rows [ybase, ybase + nrows): the rows the band's vertical taps read.
  const int ybase = vy[0];
  const int nrows = vy[nr - 1] + vn[nr - 1] - ybase;
  const uint8_t* src = d.src + int64_t(d.y0 + ybase) * d.sH + int64_t(d.x0) * d.sW;
  for (int e = t; e < nrows * kInOut; e += kInThreads) {
    const int yy = e / kInOut, q = e - yy * kInOut;
    const uint8_t* p = src + int64_t(yy) * d.sH + int64_t(hx[q]) * d.sW;
    const int32_t* k = hw + q * L.Kh;
    int32_t a0 = 1 << (kInPrec - 1), a1 = a0, a2 = a0;
    for (int x = 0; x < hn[q]; ++x, p += d.sW) {
      const int32_t w = k[x];
      a0 += int32_t(__ldg(p)) * w;
      a1 += int32_t(__ldg(p + d.sC)) * w;
      a2 += int32_t(__ldg(p + 2 * d.sC)) * w;
    }
    uint8_t* o = tile + e * 3;
    o[0] = uint8_t(in_clip8(a0));
    o[1] = uint8_t(in_clip8(a1));
    o[2] = uint8_t(in_clip8(a2));
  }
  __syncthreads();

  // Vertical pass, flip, to_tensor + normalize, fp32 store through the output strides.
  float* ob = out + int64_t(b) * sN;
  for (int e = t; e < nr * 3 * kInOut; e += kInThreads) {
    const int r = e / (3 * kInOut), c = (e / kInOut) % 3, j = e % kInOut;
    const int q = d.flip ? kInOut - 1 - j : j;
    const uint8_t* p = tile + ((vy[r] - ybase) * kInOut + q) * 3 + c;
    const int32_t* k = vw + r * L.Kv;
    int32_t acc = 1 << (kInPrec - 1);
    for (int y = 0; y < vn[r]; ++y) acc += int32_t(p[y * kInOut * 3]) * k[y];
    const float u = float(in_clip8(acc));
    ob[c * sC + (r0 + r) * sH + j * sW] = __fdiv_rn(__fsub_rn(__fdiv_rn(u, 255.0f), norm.mean[c]), norm.std[c]);
  }
}

// Upper bounds over the batch: taps per output pixel (2 ceil(support) + 1, Pillow's ksize) and, for a band of TB
// rows, source rows read: ymax(last) - ymin(first) <= (TB - 1) scale + 2 support + 1, plus a margin for rounding.
size_t in_smem_bytes(const InLayout& L) {
  return size_t(kInOut) * L.Kh * 4 + 2 * kInOut * 4 + size_t(L.TB) * L.Kv * 4 + 2 * L.TB * 4 +
         size_t(L.rows) * kInOut * 3;
}

InLayout in_layout(const bdbnn_imagenet_desc* d, int B) {
  InLayout best{0, 0, 0, 0};
  for (int TB : {32, 16, 8, 4, 2, 1}) {
    InLayout L{TB, 1, 1, 1};
    for (int i = 0; i < B; ++i) {
      const double sx = double(d[i].w) / d[i].RW, sy = double(d[i].h) / d[i].RH;
      const double fx = sx < 1.0 ? 1.0 : sx, fy = sy < 1.0 ? 1.0 : sy;
      L.Kh = std::max(L.Kh, 2 * int(ceil(fx)) + 1);
      L.Kv = std::max(L.Kv, 2 * int(ceil(fy)) + 1);
      L.rows = std::max(L.rows, std::min(int(floor((TB - 1) * sy + 2.0 * fy)) + 3, d[i].h));
    }
    best = L;
    if (in_smem_bytes(L) <= kInSmemPreferred) break;
  }
  return best;
}

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_imagenet_batch(const bdbnn_imagenet_desc* desc_host, bdbnn_imagenet_desc* desc_dev, int32_t B,
                                    const float* mean_host, const float* std_host, float* out, int64_t sN,
                                    int64_t sC, int64_t sH, int64_t sW, int64_t* target, void* stream) {
  BDBNN_REQUIRE(desc_host && desc_dev && mean_host && std_host && out && target, "imagenet_batch: NULL pointer");
  BDBNN_REQUIRE(B > 0 && B <= 65535, "imagenet_batch: B must be in [1, 65535], got %d", B);
  for (int i = 0; i < B; ++i) {
    const bdbnn_imagenet_desc& d = desc_host[i];
    BDBNN_REQUIRE(d.src != nullptr, "imagenet_batch: image %d: NULL source", i);
    BDBNN_REQUIRE(d.H >= 1 && d.W >= 1 && d.H <= kInMaxSide && d.W <= kInMaxSide,
                  "imagenet_batch: image %d: source %d x %d outside [1, %d] per side", i, d.H, d.W, kInMaxSide);
    BDBNN_REQUIRE(d.sC >= 0 && d.sH >= 0 && d.sW >= 0, "imagenet_batch: image %d: negative stride", i);
    BDBNN_REQUIRE(d.x0 >= 0 && d.y0 >= 0 && d.w >= 1 && d.h >= 1 && d.x0 + d.w <= d.W && d.y0 + d.h <= d.H,
                  "imagenet_batch: image %d: crop box (%d, %d, %d, %d) outside the %d x %d source", i, d.x0, d.y0,
                  d.w, d.h, d.H, d.W);
    BDBNN_REQUIRE(d.RH >= kInOut && d.RW >= kInOut && d.RH <= kInMaxResized && d.RW <= kInMaxResized,
                  "imagenet_batch: image %d: resized size %d x %d outside [224, 2^22]", i, d.RH, d.RW);
    BDBNN_REQUIRE(d.oy0 >= 0 && d.ox0 >= 0 && d.oy0 + kInOut <= d.RH && d.ox0 + kInOut <= d.RW,
                  "imagenet_batch: image %d: 224 x 224 window at (%d, %d) outside the %d x %d resized image", i,
                  d.oy0, d.ox0, d.RH, d.RW);
    BDBNN_REQUIRE(d.flip == 0 || d.flip == 1, "imagenet_batch: image %d: flip must be 0 or 1", i);
  }
  const InLayout L = in_layout(desc_host, B);
  const size_t smem = in_smem_bytes(L);
  BDBNN_REQUIRE(smem <= kInSmemMax, "imagenet_batch: %zu bytes of shared memory needed", smem);
  InNorm norm;
  for (int c = 0; c < 3; ++c) {
    norm.mean[c] = mean_host[c];
    norm.std[c] = std_host[c];
  }
  const cudaStream_t st = cudaStream_t(stream);
  BDBNN_CUDA(cudaMemcpyAsync(desc_dev, desc_host, size_t(B) * sizeof(bdbnn_imagenet_desc), cudaMemcpyHostToDevice,
                             st));
  BDBNN_CUDA(cudaFuncSetAttribute(imagenet_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
  const dim3 grid((kInOut + L.TB - 1) / L.TB, B);
  imagenet_batch_kernel<<<grid, kInThreads, smem, st>>>(desc_dev, L, norm, out, sN, sC, sH, sW, target);
  return check_launch("imagenet_batch_kernel");
}
