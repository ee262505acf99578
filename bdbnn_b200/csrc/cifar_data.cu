// CIFAR input batch from the device-resident uint8 dataset: shuffle, RandomCrop(32, padding=4), RandomHorizontalFlip,
// ToTensor and Normalize in one launch.  See include/bdbnn.h for the contract and DESIGN.md §4l for the spec, which
// oracle/cifar_data_ref.py restates on the CPU bit for bit.
//
//   perm(seed, epoch, pos) : keyed Feistel bijection on [0, 2^m), 2^m the next power of two >= n, cycle-walked into
//                            [0, n); 8 rounds, round keys from Philox-4x32-10(seed, (epoch, 0, 1, 0 | 1))
//   draw(seed, epoch, idx) : Philox-4x32-10(seed, (epoch, idx, 0, 0)) -> dy = (w0*9)>>32, dx = (w1*9)>>32,
//                            flip = w2>>31
// One block per image: the 3 KB source image is staged in shared memory with 16-byte loads, then the block writes
// the 3x32x32 fp32 result through the output's strides.  ~0.4 MB in and 1.5 MB out per batch of 128: launch-bound.
#include "common.cuh"

namespace bdbnn {

constexpr int kCdThreads = 256;
constexpr int kCdImgBytes = 32 * 32 * 3;
constexpr int kCdFeistelRounds = 8;

struct CifarNorm {
  float mean[3], std[3];
};

struct Philox4 {
  uint32_t w[4];
};

// Philox-4x32-10 (Salmon et al., SC'11), key = (seed lo, seed hi), the constants of Random123 / cuRAND.
__device__ __forceinline__ Philox4 philox4x32_10(uint64_t seed, uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3) {
  uint32_t k0 = uint32_t(seed), k1 = uint32_t(seed >> 32);
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = uint64_t(0xD2511F53u) * c0, p1 = uint64_t(0xCD9E8D57u) * c2;
    const uint32_t n0 = uint32_t(p1 >> 32) ^ c1 ^ k0, n2 = uint32_t(p0 >> 32) ^ c3 ^ k1;
    c1 = uint32_t(p1);
    c3 = uint32_t(p0);
    c0 = n0;
    c2 = n2;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return Philox4{{c0, c1, c2, c3}};
}

// Feistel round function: a murmur3-style 32-bit mix of the right half and the round key.
__device__ __forceinline__ uint32_t feistel_f(uint32_t r, uint32_t k) {
  uint32_t h = (r ^ k) * 0x85EBCA6Bu;
  h ^= h >> 13;
  h *= 0xC2B2AE35u;
  h ^= h >> 16;
  return h;
}

// Epoch position pos (< n) -> dataset index, a bijection of [0, n).  The state x has m bits: a left (high) part of
// wl bits and a right (low) part of wr bits; a round maps (L, R) to (R, L ^ F(R, k)), so the widths swap each round.
__device__ uint32_t cifar_perm(uint32_t pos, uint32_t n, const uint32_t* keys) {
  int m = 0;
  while ((1u << m) < n) ++m;
  uint32_t x = pos;
  do {
    int wl = m - m / 2, wr = m / 2;
#pragma unroll
    for (int r = 0; r < kCdFeistelRounds; ++r) {
      const uint32_t L = x >> wr, R = x & ((1u << wr) - 1u);
      x = (R << wl) | ((L ^ feistel_f(R, keys[r])) & ((1u << wl) - 1u));
      const int t = wl; wl = wr; wr = t;
    }
  } while (x >= n);
  return x;
}

__global__ void __launch_bounds__(kCdThreads)
cifar_batch_kernel(const uint8_t* __restrict__ images, const int64_t* __restrict__ labels, uint32_t n, uint64_t seed,
                   uint32_t epoch, int64_t pos0, int augment, CifarNorm norm, float* __restrict__ out, int64_t sN,
                   int64_t sC, int64_t sH, int64_t sW, int64_t* __restrict__ target) {
  __shared__ __align__(16) uint8_t img[kCdImgBytes];
  __shared__ uint32_t meta[4];                          // idx, dy, dx, flip
  const int b = blockIdx.x;
  if (threadIdx.x == 0) {
    const Philox4 ka = philox4x32_10(seed, epoch, 0u, 1u, 0u), kb = philox4x32_10(seed, epoch, 0u, 1u, 1u);
    const uint32_t keys[kCdFeistelRounds] = {ka.w[0], ka.w[1], ka.w[2], ka.w[3], kb.w[0], kb.w[1], kb.w[2], kb.w[3]};
    const uint32_t idx = cifar_perm(uint32_t(pos0 + b), n, keys);
    uint32_t dy = 4, dx = 4, flip = 0;
    if (augment) {
      const Philox4 d = philox4x32_10(seed, epoch, idx, 0u, 0u);
      dy = uint32_t((uint64_t(d.w[0]) * 9u) >> 32);
      dx = uint32_t((uint64_t(d.w[1]) * 9u) >> 32);
      flip = d.w[2] >> 31;
    }
    meta[0] = idx; meta[1] = dy; meta[2] = dx; meta[3] = flip;
    target[b] = labels[idx];
  }
  __syncthreads();
  const uint32_t idx = meta[0];
  const int dy = int(meta[1]) - 4, dx = int(meta[2]) - 4;
  const bool flip = meta[3] != 0;
  const uint4* src = reinterpret_cast<const uint4*>(images + int64_t(idx) * kCdImgBytes);
  for (int t = threadIdx.x; t < kCdImgBytes / 16; t += blockDim.x) reinterpret_cast<uint4*>(img)[t] = __ldg(src + t);
  __syncthreads();
  float* o = out + int64_t(b) * sN;
  for (int t = threadIdx.x; t < kCdImgBytes; t += blockDim.x) {
    const int c = t >> 10, i = (t >> 5) & 31, j = t & 31;
    const int si = i + dy, sj = (flip ? 31 - j : j) + dx;        // source pixel of the unpadded image
    const uint32_t u = (si >= 0 && si < 32 && sj >= 0 && sj < 32) ? img[(si * 32 + sj) * 3 + c] : 0u;
    const float v = __fdiv_rn(__fsub_rn(__fdiv_rn(float(u), 255.0f), norm.mean[c]), norm.std[c]);
    o[c * sC + i * sH + j * sW] = v;
  }
}

}  // namespace bdbnn

using namespace bdbnn;

extern "C" int bdbnn_cifar_batch(const uint8_t* images, const int64_t* labels, int64_t n, uint64_t seed,
                                 uint32_t epoch, int64_t pos0, int32_t B, int32_t augment, const float* mean_host,
                                 const float* std_host, float* out, int64_t sN, int64_t sC, int64_t sH, int64_t sW,
                                 int64_t* target, void* stream) {
  BDBNN_REQUIRE(images && labels && mean_host && std_host && out && target, "cifar_batch: NULL pointer");
  BDBNN_REQUIRE(n > 0 && n < (int64_t(1) << 31), "cifar_batch: n must be in [1, 2^31)");
  BDBNN_REQUIRE(B > 0 && pos0 >= 0 && pos0 + B <= n, "cifar_batch: positions [pos0, pos0 + B) must lie in [0, n)");
  BDBNN_REQUIRE(augment == 0 || augment == 1, "cifar_batch: augment must be 0 or 1");
  BDBNN_REQUIRE((uintptr_t(images) & 15) == 0, "cifar_batch: images must be 16-byte aligned");
  CifarNorm norm;
  for (int c = 0; c < 3; ++c) {
    norm.mean[c] = mean_host[c];
    norm.std[c] = std_host[c];
  }
  cifar_batch_kernel<<<B, kCdThreads, 0, cudaStream_t(stream)>>>(images, labels, uint32_t(n), seed, epoch, pos0,
                                                                 augment, norm, out, sN, sC, sH, sW, target);
  return check_launch("cifar_batch_kernel");
}
