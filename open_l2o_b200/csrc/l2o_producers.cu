// Fused gradient producers for the synthetic optimizee families (SURVEY.md 8(f) row 4): the optimizee step either side
// of the hot path.  The reference evaluates f and df/dx with ~15 TF ops per unroll step (DM/problems.py:103-175 +
// tf.gradients at DM/meta.py:322-329); here ONE launch per step produces both, so the step-at-a-time regime is
// producer kernel -> l2o_step, all inside one captured CUDA graph per unroll.
//
// Lasso (DM/problems.py:103-135 `lasso`, :137-175 `lasso_fixed`):
//   f = mean_b( 0.5 * ||A_b x_b - y_b||^2 + l * ||x_b||_1 ),   df/dx_b = ( A_b^T (A_b x_b - y_b) + l * sign(x_b) ) / B
// One CTA per batch row b.  Pass 1: the residual r = A_b x_b - y_b (a warp per matrix row, lanes striding over the
// columns: coalesced 128-byte reads, shuffle reduction).  Pass 2: g_j = sum_i A_ij r_i (a thread per column, the
// residual broadcast from shared memory, A read row by row: coalesced).  A_b (500 KB at m=250, n=500) is streamed from
// L2 twice per step; the whole batch (64 MB at B=128) stays L2-resident across the unroll.
// Random-scaling trick (DM/meta_dm_train.py:336-338,384-385): with `scale` the loss is evaluated at x (.) scale and the
// chain rule multiplies the gradient by scale.
//
// Confocal microscopy 3-D PSF fit (DM/problems.py:701-956, the simulated `inference=False` objective):
//   f = mean_b sum_v (pred_b[v] - t_b[v])^2,  pred = sum_p psf(theta_p) + bg,  t = l2_normalize(sum_p psf(sim_p) + bg_sim)
//   psf[i,j,k] = I0 ((Ex[i] Ey[j]) Ez[k]) / 8,  Ex[i] = -erf(((-0.5 - x0) + i) / (sqrt2 sxy)) + erf(((0.5 - x0) + i) / ...)
// The PSF is separable: a step needs 6 erf per axis index, point and batch row, not 6 per voxel.  One CTA per batch row b.
//   1. per-axis tables in shared memory: E, dE/dcentre, dE/dsigma of the fitted points, E of the simulated ones;
//   2. the target image into shared memory, its squared norm reduced in fp64;
//   3. the residual r = pred - t over that image, sum r^2 and sum r in fp64;
//   4. per point, sum_v r dpsf/dparam as a contraction over k (a thread per (i, j) row) and then over i, j.
// The image never leaves shared memory.  Every voxel value is formed with the reference's op order (_rn intrinsics keep
// the compiler from contracting it into FMAs); the quantile map U(lo, hi)(p) = lo + p (hi - lo) is tfd.Uniform.quantile.
#include <cuda_runtime.h>

#include "l2o_internal.h"

namespace {

constexpr int kConfThreads = 512;
constexpr int kConfWarps = kConfThreads / 32;
constexpr size_t kConfSmemLimit = 200 * 1024;

// floats of dynamic shared memory: the image, four [P][nx+ny+nz] tables and the 2P amplitudes
size_t confocal_smem_bytes(int P, const int32_t* roi) {
  const size_t V = (size_t)roi[0] * roi[1] * roi[2], L = (size_t)roi[0] + roi[1] + roi[2];
  return sizeof(float) * (V + 4 * (size_t)P * L + 2 * (size_t)P);
}

__device__ __forceinline__ float uniform_quantile(float p, float lo, float hi) {
  return __fadd_rn(lo, __fmul_rn(p, __fsub_rn(hi, lo)));
}

// sums K <= 6 doubles over the CTA; every thread gets the totals.  red: (kConfWarps + 1) * 6 doubles, the totals at a
// fixed offset past every per-warp slot, so the next call's per-warp writes never race a slow thread's read of them
template <int K>
__device__ __forceinline__ void block_sum(double (&v)[K], double* red) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int k = 0; k < K; ++k) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v[k] += __shfl_xor_sync(0xffffffffu, v[k], o);
    if (lane == 0) red[warp * K + k] = v[k];
  }
  __syncthreads();
  if (tid < K) {
    double t = 0.0;
    for (int w = 0; w < kConfWarps; ++w) t += red[w * K + tid];
    red[kConfWarps * 6 + tid] = t;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = red[kConfWarps * 6 + k];
}

__global__ void __launch_bounds__(kConfThreads) confocal_grad_kernel(l2o_confocal_args a) {
  extern __shared__ __align__(16) float sm[];
  __shared__ double red[(kConfWarps + 1) * 6];
  const int B = a.batch, P = a.num_points, b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int nx = a.roi[0], ny = a.roi[1], nz = a.roi[2];
  const int L = nx + ny + nz, rows = nx * ny, zo = nx + ny;
  float* img = sm;                    // [nx][ny][nz]: the target, then the residual
  float* tE = img + rows * nz;        // fitted points [P][L]: E, dE/dcentre, dE/dsigma (x, y, z axes concatenated)
  float* tC = tE + P * L;
  float* tS = tC + P * L;
  float* sE = tS + P * L;             // simulated points [P][L]: E
  float* amp = sE + P * L;            // [2P]: I0 of the fitted, then of the simulated points
  auto theta = [&](const float* src, int row) {   // x (.) scale, or a simulated constant
    const size_t o = (size_t)row * B + b;
    return src == a.x && a.scale ? a.x[o] * a.scale[o] : src[o];
  };

  // ---- 1. per-axis tables -------------------------------------------------------------------------------------------
  const float s2 = __fsqrt_rn(2.0f);
  constexpr float k2rpi = 1.1283791670955126f;   // 2 / sqrt(pi) = d erf / dz at 0
  for (int e = tid; e < 2 * P * L; e += kConfThreads) {
    const bool sim = e >= P * L;
    const int pe = sim ? e - P * L : e, p = pe / L, q = pe - p * L;
    const int ax = q < nx ? 0 : (q < zo ? 1 : 2);
    const int k = q - (ax == 0 ? 0 : (ax == 1 ? nx : zo));
    const float* src = sim ? a.sim : a.x;
    const int n = ax == 0 ? nx : (ax == 1 ? ny : nz);
    const float c = uniform_quantile(theta(src, 6 * p + 1 + ax), 0.5f, (float)(n - 1));
    const float sg = uniform_quantile(theta(src, 6 * p + (ax == 2 ? 5 : 4)), 2.0f, 4.0f);
    const float s = __fmul_rn(s2, sg);
    const float lo = __fdiv_rn(__fadd_rn(__fsub_rn(-0.5f, c), (float)k), s);
    const float hi = __fdiv_rn(__fadd_rn(__fsub_rn(0.5f, c), (float)k), s);
    const float E = __fadd_rn(-erff(lo), erff(hi));
    if (sim) {
      sE[pe] = E;
    } else {
      const float elo = expf(-lo * lo), ehi = expf(-hi * hi);
      tE[pe] = E;
      tC[pe] = k2rpi * (elo - ehi) / s;                // d lo / dc = d hi / dc = -1 / s
      tS[pe] = k2rpi * (lo * elo - hi * ehi) / sg;     // d lo / dsigma = -lo / sigma
    }
  }
  for (int e = tid; e < 2 * P; e += kConfThreads)
    amp[e] = uniform_quantile(theta(e < P ? a.x : a.sim, 6 * (e % P)), 0.5f, 2.0f);
  __syncthreads();

  // ---- 2. target image t = (sum_p psf(sim_p) + bg_sim) / ||.|| --------------------------------------------------------
  double nrm[1] = {0.0};
  const float bg_sim = a.sim[(size_t)6 * P * B + b];
  for (int q = warp; q < rows; q += kConfWarps) {
    const int i = q / ny, j = q - i * ny;
    for (int k = lane; k < nz; k += 32) {
      float y = 0.f;
      for (int p = 0; p < P; ++p) {
        const float* E = sE + p * L;
        y = __fadd_rn(y, __fmul_rn(__fmul_rn(amp[P + p], __fmul_rn(__fmul_rn(E[i], E[nx + j]), E[zo + k])), 0.125f));
      }
      y = __fadd_rn(y, bg_sim);
      img[q * nz + k] = y;
      nrm[0] += (double)y * (double)y;
    }
  }
  block_sum<1>(nrm, red);
  const float inv_norm = __frsqrt_rn(fmaxf((float)nrm[0], 1e-12f));   // tf.math.l2_normalize, epsilon 1e-12

  // ---- 3. residual r = (sum_p psf(theta_p) + bg) - t ------------------------------------------------------------------
  const float bg = theta(a.x, 6 * P);
  double res[2] = {0.0, 0.0};   // sum r^2, sum r
  for (int q = warp; q < rows; q += kConfWarps) {
    const int i = q / ny, j = q - i * ny;
    for (int k = lane; k < nz; k += 32) {
      float y = 0.f;
      for (int p = 0; p < P; ++p) {
        const float* E = tE + p * L;
        y = __fadd_rn(y, __fmul_rn(__fmul_rn(amp[p], __fmul_rn(__fmul_rn(E[i], E[nx + j]), E[zo + k])), 0.125f));
      }
      const float r = __fsub_rn(__fadd_rn(y, bg), __fmul_rn(img[q * nz + k], inv_norm));
      img[q * nz + k] = r;
      res[0] += (double)r * (double)r;
      res[1] += (double)r;
    }
  }
  block_sum<2>(res, red);
  const double gscale = 2.0 / (double)B;   // d/dpred of mean_b sum_v r^2
  if (tid == 0) {
    const size_t o = (size_t)6 * P * B + b;
    float g = (float)(gscale * res[1]);
    if (a.scale) g *= a.scale[o];
    a.g[o] = g;
    if (a.f) atomicAdd(a.f, res[0] / (double)B);
  }

  // ---- 4. per point: sum_v r * d psf / d(I0, x0, y0, z0, sxy, sz), k first, then (i, j) ------------------------------
  for (int p = 0; p < P; ++p) {
    const float *E = tE + p * L, *C = tC + p * L, *S = tS + p * L;
    double acc[6] = {0.0, 0.0, 0.0, 0.0, 0.0, 0.0};
    for (int q = tid; q < rows; q += kConfThreads) {
      const int i = q / ny, j = q - i * ny;
      const float* rr = img + q * nz;
      float a0 = 0.f, a1 = 0.f, a2 = 0.f;
      for (int k = 0; k < nz; ++k) {
        const float r = rr[k];
        a0 = fmaf(r, E[zo + k], a0);
        a1 = fmaf(r, C[zo + k], a1);
        a2 = fmaf(r, S[zo + k], a2);
      }
      const float ex = E[i], ey = E[nx + j], exy = ex * ey;
      acc[0] += (double)(a0 * exy);
      acc[1] += (double)(a0 * (C[i] * ey));
      acc[2] += (double)(a0 * (ex * C[nx + j]));
      acc[3] += (double)(a1 * exy);
      acc[4] += (double)(a0 * (S[i] * ey + ex * S[nx + j]));
      acc[5] += (double)(a2 * exy);
    }
    block_sum<6>(acc, red);
    if (tid < 6) {
      // d param / d theta: the quantile map's range; d psf / d param carries I0 / 8 (1 / 8 for I0 itself)
      const int n = tid == 1 ? nx : (tid == 2 ? ny : nz);
      const float range = tid == 0 ? 1.5f : (tid < 4 ? (float)(n - 1) - 0.5f : 2.0f);
      double v = 0.0;
#pragma unroll
      for (int m = 0; m < 6; ++m) v = m == tid ? acc[m] : v;
      const double amp_p = tid == 0 ? 1.0 : (double)amp[p];
      const size_t o = (size_t)(6 * p + tid) * B + b;
      float g = (float)(v * gscale * 0.125 * amp_p * (double)range);
      if (a.scale) g *= a.scale[o];
      a.g[o] = g;
    }
  }
}

constexpr int kLassoThreads = 512;

__global__ void __launch_bounds__(kLassoThreads) lasso_grad_kernel(l2o_lasso_args a) {
  extern __shared__ __align__(16) float sm[];
  const int m = a.m, n = a.n;
  float* sx = sm;                 // [n]  x (.) scale
  float* sr = sm + ((n + 3) & ~3);  // [m]  residual
  __shared__ double red[kLassoThreads / 32];
  const int b = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const float* __restrict__ A = a.A + (size_t)b * m * n;
  const float* __restrict__ x = a.x + (size_t)b * n;
  const float* __restrict__ sc = a.scale ? a.scale + (size_t)b * n : nullptr;
  double l1 = 0.0;
  for (int j = tid; j < n; j += kLassoThreads) {
    const float xv = sc ? x[j] * sc[j] : x[j];
    sx[j] = xv;
    l1 += (double)fabsf(xv);
  }
  __syncthreads();
  // ---- pass 1: r_i = sum_j A_ij x_j - y_i -------------------------------------------------------------------------
  double sq = 0.0;
  for (int i = warp; i < m; i += kLassoThreads / 32) {
    const float* __restrict__ row = A + (size_t)i * n;
    float acc0 = 0.f, acc1 = 0.f;
    int j = lane;
    for (; j + 32 < n; j += 64) {
      acc0 = fmaf(row[j], sx[j], acc0);
      acc1 = fmaf(row[j + 32], sx[j + 32], acc1);
    }
    if (j < n) acc0 = fmaf(row[j], sx[j], acc0);
    float acc = acc0 + acc1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) {
      const float r = acc - a.y[(size_t)b * m + i];
      sr[i] = r;
      sq += (double)r * (double)r;
    }
  }
  __syncthreads();
  // ---- pass 2: g_j = (sum_i A_ij r_i + l sign(x_j)) / B  [* scale_j] ----------------------------------------------------
  const float inv_b = 1.0f / (float)a.batch;
  for (int j = tid; j < n; j += kLassoThreads) {
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int i = 0;
    for (; i + 4 <= m; i += 4) {
      a0 = fmaf(A[(size_t)i * n + j], sr[i], a0);
      a1 = fmaf(A[(size_t)(i + 1) * n + j], sr[i + 1], a1);
      a2 = fmaf(A[(size_t)(i + 2) * n + j], sr[i + 2], a2);
      a3 = fmaf(A[(size_t)(i + 3) * n + j], sr[i + 3], a3);
    }
    for (; i < m; ++i) a0 = fmaf(A[(size_t)i * n + j], sr[i], a0);
    const float xv = sx[j];
    const float sgn = xv > 0.f ? 1.f : (xv < 0.f ? -1.f : 0.f);   // tf.abs'(0) = sign(0) = 0
    float g = ((a0 + a1) + (a2 + a3) + a.l1 * sgn) * inv_b;
    if (sc) g *= sc[j];
    a.g[(size_t)b * n + j] = g;
  }
  // ---- f += (0.5 sum r^2 + l sum |x|) / B -----------------------------------------------------------------------------------
  if (a.f) {
    double part = 0.5 * sq + (double)a.l1 * l1;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if (lane == 0) red[warp] = part;
    __syncthreads();
    if (tid == 0) {
      double tot = 0.0;
      for (int w = 0; w < kLassoThreads / 32; ++w) tot += red[w];
      atomicAdd(a.f, tot / (double)a.batch);
    }
  }
}

}  // namespace

extern "C" int l2o_lasso_grad(const l2o_lasso_args* a, void* stream) {
  if (!a || a->batch < 0 || a->m <= 0 || a->n <= 0 || !a->A || !a->y || !a->x || !a->g) return L2O_E_INVALID;
  if (a->batch == 0) return L2O_OK;
  const size_t smem = (size_t)(((a->n + 3) & ~3) + a->m) * sizeof(float);
  if (smem > 200 * 1024) return L2O_E_UNSUPPORTED;
  if (int rc = l2o::raise_smem_limit("l2o_lasso_grad", lasso_grad_kernel, smem)) return rc;
  lasso_grad_kernel<<<a->batch, kLassoThreads, smem, (cudaStream_t)stream>>>(*a);
  return l2o::after_launch("l2o_lasso_grad");
}

extern "C" int l2o_confocal_grad(const l2o_confocal_args* a, void* stream) {
  if (!a || !a->x || !a->sim || !a->g || a->batch < 0 || a->num_points < 1) return L2O_E_INVALID;
  for (int k = 0; k < 3; ++k)
    if (a->roi[k] < 1) return L2O_E_INVALID;
  for (int k = 0; k < 3; ++k)
    if (a->roi[k] > 65536) return L2O_E_UNSUPPORTED;   // keeps the size arithmetic below in 64 bits
  const size_t smem = confocal_smem_bytes(a->num_points, a->roi);
  if (smem > kConfSmemLimit) return L2O_E_UNSUPPORTED;
  if (a->batch == 0) return L2O_OK;
  if (int rc = l2o::raise_smem_limit("l2o_confocal_grad", confocal_grad_kernel, smem)) return rc;
  confocal_grad_kernel<<<a->batch, kConfThreads, smem, (cudaStream_t)stream>>>(*a);
  return l2o::after_launch("l2o_confocal_grad");
}
