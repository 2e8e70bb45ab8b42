// The in-kernel minibatch draw of the dataset-backed producers (l2o_mnist_grad, l2o_mnist_conv_grad,
// l2o_cifar_conv_grad): all draw the same indices for the same (seed, counter, N), so the MNIST MLPs and ConvNet see
// one index stream, and the CIFAR-10 ConvNet draws from its split by the same rule.
//
// Batch row b of the evaluation at device counter c takes Philox4x32-10 keyed by the 64-bit seed at counter
// (b, 0, c_lo, c_hi); word 0 of the output is the draw r and idx_b = (r * N) >> 32 (a 64-bit multiply-high: each
// index has probability within N / 2^32 of 1 / N).
#pragma once
#include <cstdint>

namespace l2o {

// Philox4x32-10 (Salmon et al., SC'11), word 0 of the output block
__device__ __forceinline__ uint32_t philox_w0(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0,
                                              uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t hi0 = __umulhi(0xD2511F53u, c0), lo0 = 0xD2511F53u * c0;
    const uint32_t hi1 = __umulhi(0xCD9E8D57u, c2), lo1 = 0xCD9E8D57u * c2;
    const uint32_t n0 = hi1 ^ c1 ^ k0, n2 = hi0 ^ c3 ^ k1;
    c0 = n0;
    c1 = lo1;
    c2 = n2;
    c3 = lo0;
    k0 += 0x9E3779B9u;
    k1 += 0xBB67AE85u;
  }
  return c0;
}

// the example index of batch row `row` at counter `ctr`, uniform over [0, n)
__device__ __forceinline__ int batch_index(uint64_t seed, uint64_t ctr, int row, int n) {
  const uint32_t w = philox_w0((uint32_t)row, 0u, (uint32_t)ctr, (uint32_t)(ctr >> 32), (uint32_t)seed,
                               (uint32_t)(seed >> 32));
  return (int)(((uint64_t)w * (uint64_t)n) >> 32);
}

// read_data_sets: images.astype(float32) * (1.0 / 255.0), the double constant rounded to fp32 first
__device__ __forceinline__ float mnist_pixel(uint8_t v) { return __fmul_rn((float)v, (float)(1.0 / 255.0)); }

// the CIFAR-10 reader's tf.math.divide(image, 255) on a float32 image: a correctly rounded fp32 division
__device__ __forceinline__ float cifar_pixel(uint8_t v) { return __fdiv_rn((float)v, 255.f); }

}  // namespace l2o
