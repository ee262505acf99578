// Shared helpers for libbdbnn_b200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include "../../include/bdbnn.h"

namespace bdbnn {

// Thread-local last-error text behind bdbnn_last_error_string().
char* last_error_buf();
void set_error(const char* fmt, ...);

inline int check_launch(const char* what) {
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) {
    set_error("%s: %s", what, cudaGetErrorString(e));
    return BDBNN_ERR_CUDA;
  }
  return BDBNN_OK;
}

#define BDBNN_REQUIRE(cond, ...)      \
  do {                                \
    if (!(cond)) {                    \
      ::bdbnn::set_error(__VA_ARGS__); \
      return BDBNN_ERR_INVALID_ARG;   \
    }                                 \
  } while (0)

#define BDBNN_CUDA(call)                                                     \
  do {                                                                       \
    cudaError_t e__ = (call);                                                \
    if (e__ != cudaSuccess) {                                                \
      ::bdbnn::set_error("%s failed: %s", #call, cudaGetErrorString(e__));   \
      return BDBNN_ERR_CUDA;                                                 \
    }                                                                        \
  } while (0)

inline int validate_shape(const bdbnn_conv_shape* s) {
  BDBNN_REQUIRE(s != nullptr, "conv shape is NULL");
  BDBNN_REQUIRE(s->N > 0 && s->H > 0 && s->W > 0 && s->Cin > 0 && s->Cout > 0, "non-positive dims");
  BDBNN_REQUIRE(s->kh > 0 && s->kw > 0 && s->stride > 0 && s->pad >= 0, "bad kernel/stride/pad");
  BDBNN_REQUIRE(s->Ho == (s->H + 2 * s->pad - s->kh) / s->stride + 1 &&
                    s->Wo == (s->W + 2 * s->pad - s->kw) / s->stride + 1,
                "Ho/Wo (%d,%d) inconsistent with H,W,pad,k,stride", s->Ho, s->Wo);
  BDBNN_REQUIRE(s->Ho > 0 && s->Wo > 0, "empty output");
  return BDBNN_OK;
}

inline int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;
  }
  return n;
}

// Power-of-two scale for the FP16S gradient mode: amax * 2^e lands in [2^13, 2^14).
// inverse=false -> 2^e, inverse=true -> 2^-e (both exact).  amax == 0 / denormal -> 1.
__host__ __device__ inline float amax_pow2_scale(uint32_t amax_bits, bool inverse) {
  const int be = int((amax_bits >> 23) & 0xffu);
  if (be == 0) return 1.0f;
  int e = 13 - (be - 127);
  e = e > 120 ? 120 : (e < -120 ? -120 : e);
  const uint32_t bits = uint32_t(127 + (inverse ? -e : e)) << 23;
#ifdef __CUDA_ARCH__
  return __uint_as_float(bits);
#else
  float f;
  memcpy(&f, &bits, 4);
  return f;
#endif
}

// bn.cu: sum y, sum y^2, max|y| per channel of an NHWC fp32 tensor into (pre-zeroed) sums / ymax.
int bn_stats_launch(const float* y, int64_t n_pix, int C, double* sums, uint32_t* ymax, cudaStream_t st);
// bn.cu: run-to-run deterministic sums across blocks.  Block b writes its partial row part[b][0, width) (no
// atomics); det_sums_finish adds the column sums, taken in a fixed order, to sums[0, width) and frees `part`
// (also when it fails).
// Stream-ordered allocation, so both may be captured into a CUDA graph.
int det_sums_alloc(double** part, int64_t nparts, int width, cudaStream_t st);
int det_sums_finish(double* part, int64_t nparts, int width, double* sums, cudaStream_t st);

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace bdbnn
