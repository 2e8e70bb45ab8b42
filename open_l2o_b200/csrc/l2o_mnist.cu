// MNIST MLP producer (DM/problems.py:254-288 `mnist` + tf.gradients at DM/meta.py:322-329): f and df/dx of
//   f = mean_b xent(MLP(images[idx_b] / 255), labels[idx_b]),  idx_b ~ U[0, N) drawn afresh at every evaluation,
// in ONE launch.  The optimizee step feeding the hot path (SURVEY.md 8(f) row 4), like l2o_lasso_grad.
//
// Batch indices.  l2o_philox.cuh's draw at the device int64 *counter, which the kernel reads and CTA rank 0 advances by
// one after the last cluster barrier.  Because the counter lives on the device, a captured CUDA graph draws a fresh batch on every replay.
//
// Design.  One cluster of kCl = 8 CTAs, CTA rank s owning batch rows [s R, s R + R), R = ceil(B / 8) (the last CTAs
// may own fewer rows, or none).  Each CTA keeps its rows' hidden activations in shared memory, and later the dz of
// each layer in place of them.
//   forward  layer 0: the gathered uint8 pixels and the (scaled) weights staged in K-chunks of kKC features, one
//            thread per (row, unit) output accumulating in a fixed order; layers 1..: weights from L2.  Softmax cross
//            entropy one warp per row; the loss in fp64, summed over rows, then warps, then (rank 0) ranks in order.
//   backward dW_l[k][j] = sum_b A_l[b][k] dz_l[b][j] (A_0 = the pixels, A_l = h_{l-1}; the bias as a row of ones).
//            The K_l + 1 rows of dW_l / db_l are split across the CTAs; each CTA walks the rows of ranks 0..7 in
//            order, staging their dz (and A) through distributed shared memory, so every gradient element is one fp32
//            sum over b = 0..B-1 in the same order on every run: deterministic, no atomics.  Splitting by feature rather
//            than reducing per-CTA partial dW keeps shared memory small: a partial dW_0 alone is 784 x 64 floats
//            (200 KB) at the widest layer.
// Random scaling (DM/meta_dm_train.py:336-338,384-385) as l2o_lasso_grad: the loss at x (.) scale, g multiplied by scale.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include "l2o_internal.h"
#include "l2o_philox.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kCl = 8;          // CTAs per cluster
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kIn = L2O_MNIST_INPUT;
constexpr int kOut = L2O_MNIST_CLASSES;
constexpr int kKC = 56;         // layer-0 forward K-chunk (784 = 14 x 56)
constexpr int kRS = 32;         // rows staged per step of the weight-gradient sweep
constexpr size_t kSmemLimit = 227 * 1024;

struct Plan {
  int L;                        // linear layers (hidden + output)
  int K[L2O_MNIST_MAX_HIDDEN + 1], W[L2O_MNIST_MAX_HIDDEN + 1];   // layer l: [K_l] -> [W_l]
  int64_t off_w[L2O_MNIST_MAX_HIDDEN + 1], off_b[L2O_MNIST_MAX_HIDDEN + 1];
  int act_off[L2O_MNIST_MAX_HIDDEN];                              // floats: h_l [R][W_l]
  int R, dz_off, u_off, wmax, slice;                             // slice: rows of dW per CTA (max over layers)
  size_t smem;
};

__host__ __device__ inline int cdiv(int a, int b) { return (a + b - 1) / b; }

bool make_plan(const l2o_mnist_args& a, Plan& p) {
  const int nh = a.n_layers - 1;
  p.L = a.n_layers;
  int k = kIn;
  int64_t off = 0;
  p.wmax = kOut;
  for (int l = 0; l < p.L; ++l) {
    const int w = l < nh ? a.hidden[l] : kOut;
    p.K[l] = k;
    p.W[l] = w;
    p.off_w[l] = off;
    p.off_b[l] = off + (int64_t)k * w;
    off = p.off_b[l] + w;
    p.wmax = w > p.wmax ? w : p.wmax;
    k = w;
  }
  p.R = cdiv(a.batch, kCl);
  int f = 0;
  for (int l = 0; l < nh; ++l) {
    p.act_off[l] = f;
    f += p.R * p.W[l];
  }
  p.dz_off = f;
  f += p.R * kOut;
  p.slice = 0;
  for (int l = 0; l < p.L; ++l) p.slice = cdiv(p.K[l] + 1, kCl) > p.slice ? cdiv(p.K[l] + 1, kCl) : p.slice;
  f = (f + 3) & ~3;
  p.u_off = f;
  // the union region: forward chunk (weights [kKC][wmax] floats + pixels [R][kKC] bytes) or the backward sweep
  // (accumulators [slice][wmax], staged A [kRS][slice], staged dz [kRS][wmax] floats and kRS indices)
  const int fwd = kKC * p.wmax + cdiv(p.R * kKC, 4);
  const int bwd = p.slice * p.wmax + kRS * p.slice + kRS * p.wmax + kRS;
  f += fwd > bwd ? fwd : bwd;
  p.smem = sizeof(float) * (size_t)f + sizeof(int32_t) * (size_t)p.R;   // + the rows' indices
  return true;
}

__global__ void __cluster_dims__(kCl, 1, 1) __launch_bounds__(kThreads, 1) mnist_grad_kernel(const l2o_mnist_args a,
                                                                                          const Plan p) {
  extern __shared__ __align__(16) float sm[];
  __shared__ double red[kWarps];
  __shared__ double part;   // this CTA's sum of per-row losses
  cg::cluster_group cl = cg::this_cluster();
  const int rank = (int)cl.block_rank();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int B = a.batch, R = p.R, L = p.L;
  const int row0 = rank * R;
  const int nrows = max(0, min(R, B - row0));
  int32_t* sidx = reinterpret_cast<int32_t*>(sm + p.smem / sizeof(float) - R);
  float* u = sm + p.u_off;
  const float* __restrict__ x = a.x;
  const float* __restrict__ sc = a.scale;
  auto wv = [&](int64_t o) { return sc ? x[o] * sc[o] : x[o]; };

  // ---- batch indices -------------------------------------------------------------------------------------------------
  const uint64_t ctr = (uint64_t)*a.counter;
  for (int r = tid; r < nrows; r += kThreads) {
    const int idx = l2o::batch_index(a.seed, ctr, row0 + r, a.num_examples);
    sidx[r] = idx;
    if (a.idx_out) a.idx_out[row0 + r] = idx;
  }
  __syncthreads();

  // ---- forward, layer 0: z = pixels @ W0 over K-chunks, then h0 = act(z + b0) ----------------------------------------
  {
    const int W = p.W[0];
    float* z = sm + p.act_off[0];
    float* wc = u;
    uint8_t* xc = reinterpret_cast<uint8_t*>(u + kKC * p.wmax);
    for (int c0 = 0; c0 < kIn; c0 += kKC) {
      for (int e = tid; e < kKC * W; e += kThreads) wc[e] = wv(p.off_w[0] + (int64_t)c0 * W + e);
      for (int e = tid; e < nrows * kKC; e += kThreads) {
        const int r = e / kKC, kk = e - r * kKC;
        xc[e] = a.images[(size_t)sidx[r] * kIn + c0 + kk];
      }
      __syncthreads();
      for (int o = tid; o < nrows * W; o += kThreads) {
        const int r = o / W, j = o - r * W;
        const uint8_t* xr = xc + r * kKC;
        float acc = c0 == 0 ? 0.f : z[o];
#pragma unroll 8
        for (int kk = 0; kk < kKC; ++kk) acc = fmaf(l2o::mnist_pixel(xr[kk]), wc[kk * W + j], acc);
        z[o] = acc;
      }
      __syncthreads();
    }
  }
  // ---- hidden layers: bias + activation, then the next layer's z -------------------------------------------------------
  for (int l = 0; l < L - 1; ++l) {
    const int W = p.W[l];
    float* h = sm + p.act_off[l];
    for (int o = tid; o < nrows * W; o += kThreads) {
      const float v = h[o] + wv(p.off_b[l] + o % W);
      h[o] = a.activation == L2O_MNIST_RELU ? fmaxf(v, 0.f) : 1.f / (1.f + expf(-v));
    }
    __syncthreads();
    if (l + 1 < L - 1) {   // the next hidden layer's pre-activation (the output layer is fused into the loss below)
      const int K = W, Wn = p.W[l + 1];
      float* zn = sm + p.act_off[l + 1];
      for (int o = tid; o < nrows * Wn; o += kThreads) {
        const int r = o / Wn, j = o - r * Wn;
        float acc = 0.f;
        for (int k = 0; k < K; ++k) acc = fmaf(h[r * K + k], wv(p.off_w[l + 1] + (int64_t)k * Wn + j), acc);
        zn[o] = acc;
      }
      __syncthreads();
    }
  }
  // ---- output layer and softmax cross entropy, one warp per row; dz = (softmax - onehot) / B ---------------------------
  {
    const int l = L - 1, K = p.K[l];
    const float* hin = sm + p.act_off[L - 2];
    float* dz = sm + p.dz_off;
    double lsum = 0.0;
    for (int r = warp; r < nrows; r += kWarps) {
      float zj = -INFINITY;
      if (lane < kOut) {
        float acc = 0.f;
        for (int k = 0; k < K; ++k) acc = fmaf(hin[r * K + k], wv(p.off_w[l] + (int64_t)k * kOut + lane), acc);
        zj = acc + wv(p.off_b[l] + lane);
      }
      float m = zj;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
      const float e = lane < kOut ? expf(zj - m) : 0.f;
      float s = e;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      const int y = a.labels[sidx[r]];
      const float zy = __shfl_sync(0xffffffffu, zj, y);
      if (lane < kOut) dz[r * kOut + lane] = (e / s - (lane == y ? 1.f : 0.f)) / (float)B;
      if (lane == 0) lsum += (double)m + (double)logf(s) - (double)zy;
    }
    if (lane == 0) red[warp] = lsum;
    __syncthreads();
    if (tid == 0) {
      double t = 0.0;
      for (int w = 0; w < kWarps; ++w) t += red[w];
      part = t;
    }
  }

  // ---- backward: per layer, this CTA's rows of dW_l / db_l over all B rows in rank order, then dz_{l-1} ---------------
  for (int l = L - 1; l >= 0; --l) {
    const int K = p.K[l], W = p.W[l], Kp = K + 1;
    const int per = cdiv(Kp, kCl), k0 = rank * per, k1 = min(k0 + per, Kp), nk = max(0, k1 - k0);
    const int dzo = l == L - 1 ? p.dz_off : p.act_off[l];   // where dz_l lives (in place of h_l below the output)
    float* acc = u;
    float* sA = acc + p.slice * p.wmax;
    float* sD = sA + kRS * p.slice;
    int32_t* sI = reinterpret_cast<int32_t*>(sD + kRS * p.wmax);
    cl.sync();   // dz_l is complete in every CTA (and every CTA is past its forward use of the union region)
    for (int e = tid; e < nk * W; e += kThreads) acc[e] = 0.f;
    for (int s = 0; s < kCl; ++s) {
      const int nr = max(0, min(R, B - s * R));
      const float* rdz = cl.map_shared_rank(sm + dzo, s);
      const float* rA = l > 0 ? cl.map_shared_rank(sm + p.act_off[l - 1], s) : nullptr;
      const int32_t* rI = cl.map_shared_rank(reinterpret_cast<int32_t*>(sm + p.smem / sizeof(float) - R), s);
      for (int rb = 0; rb < nr; rb += kRS) {
        const int nb = min(kRS, nr - rb);
        if (l == 0)
          for (int e = tid; e < nb; e += kThreads) sI[e] = rI[rb + e];
        for (int e = tid; e < nb * W; e += kThreads) sD[e] = rdz[rb * W + e];
        if (l == 0) __syncthreads();
        for (int e = tid; e < nb * nk; e += kThreads) {
          const int r = e / nk, kk = e - r * nk, k = k0 + kk;
          float v = 1.f;
          if (k < K) v = l == 0 ? l2o::mnist_pixel(a.images[(size_t)sI[r] * kIn + k]) : rA[(rb + r) * K + k];
          sA[e] = v;
        }
        __syncthreads();
        for (int o = tid; o < nk * W; o += kThreads) {
          const int kk = o / W, j = o - kk * W;
          float t = acc[o];
          for (int r = 0; r < nb; ++r) t = fmaf(sA[r * nk + kk], sD[r * W + j], t);
          acc[o] = t;
        }
        __syncthreads();
      }
    }
    for (int o = tid; o < nk * W; o += kThreads) {
      const int kk = o / W, j = o - kk * W, k = k0 + kk;
      const int64_t off = k < K ? p.off_w[l] + (int64_t)k * W + j : p.off_b[l] + j;
      a.g[off] = sc ? acc[o] * sc[off] : acc[o];
    }
    if (l > 0) {
      cl.sync();   // every CTA is done reading this CTA's h_{l-1} and dz_l: dz_{l-1} may overwrite h_{l-1}
      const float* dz = sm + dzo;
      float* h = sm + p.act_off[l - 1];
      for (int o = tid; o < nrows * K; o += kThreads) {
        const int r = o / K, k = o - r * K;
        float t = 0.f;
        for (int j = 0; j < W; ++j) t = fmaf(dz[r * W + j], wv(p.off_w[l] + (int64_t)k * W + j), t);
        const float hv = h[o];
        h[o] = a.activation == L2O_MNIST_RELU ? (hv > 0.f ? t : 0.f) : t * hv * (1.f - hv);
      }
    }
  }

  // ---- f = (sum over ranks, in order) / B; the counter advances once per evaluation -----------------------------------
  cl.sync();
  if (rank == 0 && tid == 0) {
    double t = 0.0;
    for (int s = 0; s < kCl; ++s) t += *cl.map_shared_rank(&part, s);
    if (a.f) *a.f = t / (double)B;
    *a.counter = (int64_t)(ctr + 1);
  }
  cl.sync();   // no CTA leaves while rank 0 reads its shared memory
}

}  // namespace

extern "C" int l2o_mnist_grad(const l2o_mnist_args* a, void* stream) {
  if (!a || !a->images || !a->labels || !a->x || !a->g || !a->counter) return L2O_E_INVALID;
  if (a->batch < 1 || a->batch > L2O_MNIST_MAX_BATCH || a->num_examples < 1) return L2O_E_INVALID;
  if (a->n_layers < 2 || a->n_layers > L2O_MNIST_MAX_HIDDEN + 1) return L2O_E_INVALID;
  if (a->activation != L2O_MNIST_SIGMOID && a->activation != L2O_MNIST_RELU) return L2O_E_INVALID;
  for (int l = 0; l < a->n_layers - 1; ++l)
    if (a->hidden[l] < 1 || a->hidden[l] > L2O_MNIST_MAX_WIDTH) return L2O_E_INVALID;
  Plan p;
  make_plan(*a, p);
  if (p.smem > kSmemLimit) return L2O_E_UNSUPPORTED;   // not reached inside the limits above (at most ~180 KB)
  if (int rc = l2o::raise_smem_limit("l2o_mnist_grad", mnist_grad_kernel, p.smem)) return rc;
  mnist_grad_kernel<<<kCl, kThreads, p.smem, (cudaStream_t)stream>>>(*a, p);
  return l2o::after_launch("l2o_mnist_grad");
}
