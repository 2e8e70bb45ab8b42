// Training-mode batch norm across a cooperative grid, for the ConvNet producers (l2o_mnist_conv_grad,
// l2o_cifar_conv_grad).  Each image writes its per-channel partials to the workspace; after a grid barrier every CTA
// merges them over b = 0..B-1 in an order that depends on B only, so every CTA holds bitwise the same batch constants
// and no atomics are needed.
//   statistics: per image (mean, M2) of its n positions, merged with Chan's formula for equal counts
//               (mu = sum mean_b / B, M2 = sum_b M2_b + n (mean_b - mu)^2), never E[z^2] - E[z]^2, which cancels when
//               |mu| >> sigma; the variance is biased, over all B * n positions, as fused training-mode batch norm;
//   backward:   per image (sum dy, sum dy * yhat); the means over all B * n positions.
#pragma once
#include <cuda_runtime.h>

namespace l2o {

// per-channel sum over the threads of one CTA, tid = q * C + c: red[tid] = v, then thread c < C adds q = 0.. in order
template <int kThreads>
__device__ __forceinline__ double chan_sum(double* red, double v, int C) {
  const int tid = threadIdx.x;
  red[tid] = v;
  __syncthreads();
  double s = 0.0;
  if (tid < C)
    for (int q = 0; q < kThreads / C; ++q) s += red[q * C + tid];
  __syncthreads();
  return s;   // meaningful in threads tid < C
}

// the BN statistics of the batch from the per-image (mean, M2) of n positions each: mu and 1 / sqrt(var + eps) in fp32
template <int kThreads>
__device__ void merge_stats(const double2* st, int B, int C, int n, float eps, double* red, float* mu_out,
                            float* rs_out, double* mu_tmp) {
  const int tid = threadIdx.x, c = tid % C, k = tid / C, K = kThreads / C;
  double s = 0.0;
  for (int b = k; b < B; b += K) s += __ldcg(&st[(size_t)b * C + c].x);
  s = chan_sum<kThreads>(red, s, C);
  if (tid < C) mu_tmp[tid] = s / (double)B;
  __syncthreads();
  const double mu = mu_tmp[c];
  double m2 = 0.0;
  for (int b = k; b < B; b += K) {
    const double2 v = __ldcg(&st[(size_t)b * C + c]);
    const double d = v.x - mu;
    m2 += v.y + (double)n * d * d;
  }
  m2 = chan_sum<kThreads>(red, m2, C);
  if (tid < C) {
    const double var = m2 / ((double)B * (double)n);   // biased, as fused training-mode batch norm
    mu_out[tid] = (float)mu_tmp[tid];
    rs_out[tid] = (float)(1.0 / sqrt(var + (double)eps));
  }
  __syncthreads();
}

// the BN backward means: sum_b (sum dy, sum dy * yhat) / (B n)
template <int kThreads>
__device__ void merge_back(const double2* bk, int B, int C, int n, double* red, float* ma, float* mb) {
  const int tid = threadIdx.x, c = tid % C, k = tid / C, K = kThreads / C;
  double s = 0.0, t = 0.0;
  for (int b = k; b < B; b += K) {
    const double2 v = __ldcg(&bk[(size_t)b * C + c]);
    s += v.x;
    t += v.y;
  }
  s = chan_sum<kThreads>(red, s, C);
  t = chan_sum<kThreads>(red, t, C);
  if (tid < C) {
    const double nn = (double)B * (double)n;
    ma[tid] = (float)(s / nn);
    mb[tid] = (float)(t / nn);
  }
  __syncthreads();
}

}  // namespace l2o
