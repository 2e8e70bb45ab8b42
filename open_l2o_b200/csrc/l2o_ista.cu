// Model-based L2O's LISTA family (MB/ = Model_Base_L2O/ of the reference) — sm_90a kernels + C-ABI.
//
// Four cell forms over a batch of rows, layers k = k0 .. k1-1 (row-major: y [B,M], x [B,N], A [M,N]):
//   LISTA   (MB/models/lista.py:32-45)        z_k = y B1^T + s_k x_k W_k^T       (layer 0: no W term)
//   coupled (lista_cp.py, lista_cpss.py, alista.py)  r_k = y - x_k A^T,  z_k = x_k + s_k r_k W_k
//   LFISTA and LAMP, which also carry x_{k-1} or v_{k-1}: their own kernels, further down
// then x_{k+1} = shrink(z_k): soft shrinkage sign(z) relu(|z| - theta_k) (MB/models/utils.py shrink_free), or support
// selection (shrink_ss): entries with |z| > theta_k and |z| > the row's rank-q_k magnitude pass through unshrunk.
//
// Design.  One thread-block cluster of kCl CTAs owns kR batch rows for the whole pass, so a forward or backward over
// any number of layers is ONE launch.  Each CTA of the cluster computes a 1/kCl column slice of every per-layer GEMM
// for the cluster's rows and writes it into every CTA's shared memory (distributed shared memory); a cluster barrier
// then makes the full rows visible to all of them.  The shrinkage, and the per-row rank selection of support
// selection (a radix select, one warp per row), run redundantly in every CTA on the full rows, so the next layer
// starts without another exchange.  The weights are read from global memory (they stay L2-resident across clusters).
// The GEMMs are fp32 FFMA on the CUDA cores.  A CTA's slice, computed transposed, is one m64n8 wgmma tile
// ((N / kCl) output columns x kR rows); running it on the tensor cores with the engine's 3xTF32 split and streaming the
// weights by TMA is the next step (DESIGN §3.12), and matters most for large batches.
//
// The backward is the same cluster recurrence run from k1-1 down to k0; it records dz_k and per-CTA partial sums of
// dtheta_k and ds_k.  A second launch forms the weight gradients from them (one GEMM per output, reducing over the
// batch and, for a shared W or B1, over the layers: dB1 = sum_k dz_k^T y), and reduces the partial sums.
#include <cooperative_groups.h>

#include <algorithm>
#include <cmath>
#include <cstdint>

#include "l2o_internal.h"

namespace cg = cooperative_groups;

namespace l2o {
namespace ista {

constexpr int kCl = 8;        // CTAs per cluster
constexpr int kR = 8;         // batch rows per cluster (one warp per row in the rank selection)
constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kMaxDim = kCl * kThreads;   // M, N <= 2048: a CTA's column slice is at most one thread per column
constexpr int kTile = 64;                 // weight-gradient output tile
constexpr int kChunk = 16;                // weight-gradient reduction chunk

struct Slice {
  int lo, hi;
};
__host__ __device__ inline Slice slice_of(int len, int c) {
  const int w = (len + kCl - 1) / kCl;
  const int lo = min(len, c * w);
  return {lo, min(len, lo + w)};
}

// The coupled form and LAMP apply W [M][N] to r_k (v_k); LISTA and LFISTA apply W [N][N] to x_k.
__host__ __device__ inline bool w_on_r(const l2o_ista_args& a) {
  return a.form == L2O_ISTA_COUPLED || a.form == L2O_ISTA_LAMP;
}
__device__ __forceinline__ const float* w_slot(const l2o_ista_args& a, int k) {
  if (a.form == L2O_ISTA_COUPLED) return a.W + (a.share_W ? 0 : (size_t)k * a.m * a.n);
  return a.W + (a.share_W ? 0 : (size_t)(k - 1) * a.n * a.n);
}
__device__ __forceinline__ float step_of(const l2o_ista_args& a, int k) { return a.step ? a.step[k] : 1.f; }

// out[b][j] = sum_t in[b][t] W[j][t] for j in [j0, j1): a warp per pair of outputs, lanes across t.
template <class F>
__device__ __forceinline__ void gemm_rows(const float* in, int ld_in, const float* __restrict__ W, int ldw, int T,
                                          int j0, int j1, F&& epi) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int j = j0 + 2 * w; j < j1; j += 2 * kWarps) {
    const bool two = j + 1 < j1;
    const float* w0 = W + (size_t)j * ldw;
    const float* w1 = two ? w0 + ldw : w0;
    float a0[kR], a1[kR];
#pragma unroll
    for (int b = 0; b < kR; ++b) a0[b] = a1[b] = 0.f;
    for (int t = lane; t < T; t += 32) {
      const float q0 = __ldg(w0 + t), q1 = __ldg(w1 + t);
#pragma unroll
      for (int b = 0; b < kR; ++b) {
        const float v = in[b * ld_in + t];
        a0[b] = fmaf(v, q0, a0[b]);
        a1[b] = fmaf(v, q1, a1[b]);
      }
    }
#pragma unroll
    for (int b = 0; b < kR; ++b)
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        a0[b] += __shfl_xor_sync(0xffffffffu, a0[b], o);
        a1[b] += __shfl_xor_sync(0xffffffffu, a1[b], o);
      }
#pragma unroll
    for (int b = 0; b < kR; ++b) {
      if (lane == b) epi(b, j, a0[b]);
      if (two && lane == kR + b) epi(b, j + 1, a1[b]);
    }
  }
}

// out[b][j] = sum_t in[b][t] W[t][j] for j in [j0, j1): a thread per (column, t-group), groups summed through red.
// Called by every thread of the CTA (it synchronises).
template <class F>
__device__ __forceinline__ void gemm_cols(const float* in, int ld_in, const float* __restrict__ W, int ldw, int T,
                                          int j0, int j1, float* red, F&& epi) {
  const int nj = j1 - j0;
  if (nj <= 0) return;
  const int G = kThreads / nj, jj = threadIdx.x % nj, g = threadIdx.x / nj;
  float acc[kR];
#pragma unroll
  for (int b = 0; b < kR; ++b) acc[b] = 0.f;
  if (g < G) {
    const float* wc = W + j0 + jj;
    for (int t = g; t < T; t += G) {
      const float q = __ldg(wc + (size_t)t * ldw);
#pragma unroll
      for (int b = 0; b < kR; ++b) acc[b] = fmaf(in[b * ld_in + t], q, acc[b]);
    }
#pragma unroll
    for (int b = 0; b < kR; ++b) red[(g * kR + b) * nj + jj] = acc[b];
  }
  __syncthreads();
  for (int o = threadIdx.x; o < nj * kR; o += kThreads) {
    const int b = o / nj, j = o % nj;
    float s = 0.f;
    for (int q = 0; q < G; ++q) s += red[(q * kR + b) * nj + j];
    epi(b, j0 + j, s);
  }
  __syncthreads();
}

// |z| at 0-based rank t in descending order over one row (MSB-first radix select on the fp32 bit patterns, which
// order like the values for |z| >= 0).  One warp; hist is the warp's 256 counters.
__device__ float row_rank_abs(const float* z, int n, int t, unsigned* hist) {
  const int lane = threadIdx.x & 31;
  unsigned prefix = 0, mask = 0;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = lane; i < 256; i += 32) hist[i] = 0;
    __syncwarp();
    for (int i = lane; i < n; i += 32) {
      const unsigned key = __float_as_uint(fabsf(z[i]));
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
    }
    __syncwarp();
    unsigned c[8], s = 0;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      c[q] = hist[255 - 8 * lane - q];
      s += c[q];
    }
    unsigned inc = s;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const unsigned v = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += v;
    }
    const unsigned exc = inc - s;
    const unsigned ball = __ballot_sync(0xffffffffu, exc <= (unsigned)t && (unsigned)t < inc);
    const int src = __ffs(ball) - 1;
    int bucket = 0;
    unsigned before = 0;
    if (lane == src) {
      unsigned acc = exc;
      bool found = false;
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        if (!found && (unsigned)t < acc + c[q]) {
          bucket = 255 - 8 * lane - q;
          before = acc;
          found = true;
        }
        acc += c[q];
      }
    }
    bucket = __shfl_sync(0xffffffffu, bucket, src);
    before = __shfl_sync(0xffffffffu, before, src);
    t -= (int)before;
    prefix |= (unsigned)bucket << shift;
    mask |= 255u << shift;
    __syncwarp();
  }
  return __uint_as_float(prefix);
}

// Shared-memory plan of one CTA, in floats.
struct Smem {
  int y, x, r, z, by, red, total;
};
__host__ __device__ inline Smem smem_plan(const l2o_ista_args& a) {
  Smem s;
  s.y = 0;
  s.x = s.y + kR * a.m;
  s.r = s.x + kR * a.n;
  s.z = s.r + (a.form == L2O_ISTA_COUPLED ? kR * a.m : 0);
  s.by = s.z + 2 * kR * a.n;
  s.red = s.by + (a.form == L2O_ISTA_LISTA ? kR * a.n : 0);
  s.total = s.red + kThreads * kR;   // also the rank selection's 8 x 256 counters
  return s;
}

__device__ __forceinline__ bool has_w_term(const l2o_ista_args& a, int k) {
  return a.form == L2O_ISTA_COUPLED || k >= 1;
}

__global__ void __cluster_dims__(kCl, 1, 1) __launch_bounds__(kThreads)
    ista_fwd_kernel(const l2o_ista_args a) {
  extern __shared__ float4 smem_f4[];
  float* sm = reinterpret_cast<float*>(smem_f4);
  cg::cluster_group cl = cg::this_cluster();
  const int c = (int)cl.block_rank();
  const int row0 = (blockIdx.x / kCl) * kR;
  const int M = a.m, N = a.n, tid = threadIdx.x;
  const Smem P = smem_plan(a);
  float *ys = sm + P.y, *xs = sm + P.x, *rb = sm + P.r, *by = sm + P.by, *red = sm + P.red;
  unsigned* hist = reinterpret_cast<unsigned*>(red);
  __shared__ float thr[kR];
  const Slice sm_ = slice_of(M, c), sn = slice_of(N, c);

  for (int e = tid; e < kR * M; e += kThreads) {
    const int b = e / M, i = e % M, row = row0 + b;
    ys[e] = row < a.batch ? a.y[(size_t)row * a.ldy + i] : 0.f;
  }
  for (int e = tid; e < kR * N; e += kThreads) {
    const int b = e / N, n = e % N, row = row0 + b;
    xs[e] = (a.x_in && row < a.batch) ? a.x_in[(size_t)row * N + n] : 0.f;
  }
  __syncthreads();
  if (a.form == L2O_ISTA_LISTA) {   // y B1^T is the same in every layer of the pass: own slice only
    gemm_rows(ys, M, a.B1, M, M, sn.lo, sn.hi, [&](int b, int n, float v) { by[b * N + n] = v; });
  }
  cl.sync();   // every CTA of the cluster has started (and finished its prologue) before any remote write

  for (int k = a.k0; k < a.k1; ++k) {
    const int l = k - a.k0;
    float* zb = sm + P.z + (l & 1) * kR * N;
    const float s = step_of(a, k), th = a.theta[k];
    auto put_z = [&](int b, int n, float z) {
      for (int q = 0; q < kCl; ++q) cl.map_shared_rank(zb, q)[b * N + n] = z;
    };
    if (a.form == L2O_ISTA_COUPLED) {
      const float* W = w_slot(a, k);
      gemm_rows(xs, N, a.A, N, N, sm_.lo, sm_.hi, [&](int b, int i, float v) {
        const float r = ys[b * M + i] - v;
        for (int q = 0; q < kCl; ++q) cl.map_shared_rank(rb, q)[b * M + i] = r;
        if (a.rs && row0 + b < a.batch) a.rs[((size_t)l * a.batch + row0 + b) * M + i] = r;
      });
      cl.sync();
      gemm_cols(rb, M, W, N, M, sn.lo, sn.hi, red, [&](int b, int n, float v) { put_z(b, n, xs[b * N + n] + s * v); });
    } else if (has_w_term(a, k)) {
      gemm_rows(xs, N, w_slot(a, k), N, N, sn.lo, sn.hi,
                [&](int b, int n, float v) { put_z(b, n, by[b * N + n] + s * v); });
    } else {
      for (int e = tid; e < kR * (sn.hi - sn.lo); e += kThreads) {
        const int b = e / (sn.hi - sn.lo), n = sn.lo + e % (sn.hi - sn.lo);
        put_z(b, n, by[b * N + n]);
      }
    }
    cl.sync();
    const int rank = a.ss_rank ? min(a.ss_rank[k], N - 1) : -1;   // negative: soft shrinkage in this layer
    if (rank >= 0) {
      const int w = tid >> 5;
      const float t = row_rank_abs(zb + w * N, N, rank, hist + w * 256);
      if ((tid & 31) == 0) thr[w] = t;
    }
    __syncthreads();
    for (int e = tid; e < kR * N; e += kThreads) {
      const int b = e / N, n = e % N, row = row0 + b;
      const float z = zb[e], az = fabsf(z);
      const bool pick = rank >= 0 && az > th && az > thr[b];
      const float m = fmaxf(az - th, 0.f);
      const float x = pick ? z : (z > 0.f ? m : (z < 0.f ? -m : 0.f));
      xs[e] = x;
      if (n >= sn.lo && n < sn.hi && row < a.batch) {
        const size_t o = ((size_t)l * a.batch + row) * N + n;
        a.xs[o] = x;
        if (a.zs) a.zs[o] = z;
        if (a.sel) a.sel[o] = pick;
      }
    }
    __syncthreads();
  }
  cl.sync();   // no CTA leaves while another may still write into its shared memory
}

struct Bwd {
  l2o_ista_args a;
  l2o_ista_grads g;
};

__device__ __forceinline__ float* dz_rec(const Bwd& p) { return reinterpret_cast<float*>(p.g.scratch); }
__device__ __forceinline__ float* part_rec(const Bwd& p) {
  return dz_rec(p) + (size_t)(p.a.k1 - p.a.k0) * p.a.batch * p.a.n;
}
__device__ __forceinline__ const float* layer_input(const l2o_ista_args& a, int l, int row) {
  if (l == 0) return a.x_in ? a.x_in + (size_t)row * a.n : nullptr;
  return a.xs + ((size_t)(l - 1) * a.batch + row) * a.n;
}

__device__ float block_sum(float v, float* scratch) {
  for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) scratch[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = 0.f;
  if (threadIdx.x == 0)
    for (int w = 0; w < kWarps; ++w) s += scratch[w];
  __syncthreads();
  return s;
}

__global__ void __cluster_dims__(kCl, 1, 1) __launch_bounds__(kThreads) ista_bwd_kernel(const Bwd p) {
  extern __shared__ float4 smem_f4[];
  float* sm = reinterpret_cast<float*>(smem_f4);
  const l2o_ista_args& a = p.a;
  cg::cluster_group cl = cg::this_cluster();
  const int c = (int)cl.block_rank();
  const int row0 = (blockIdx.x / kCl) * kR;
  const int M = a.m, N = a.n, tid = threadIdx.x;
  const Smem P = smem_plan(a);
  float *dx = sm + P.x, *rb = sm + P.r, *red = sm + P.red;
  __shared__ float wsum[kWarps];
  const Slice sm_ = slice_of(M, c), sn = slice_of(N, c);
  const int ns = sn.hi - sn.lo;
  float* dzr = dz_rec(p);
  float* part = part_rec(p);
  const int nblk = gridDim.x;

  for (int e = tid; e < kR * ns; e += kThreads) {
    const int b = e / ns, n = sn.lo + e % ns, row = row0 + b;
    dx[b * N + n] = row < a.batch ? p.g.d_xk[(size_t)row * N + n] : 0.f;
  }
  cl.sync();   // every CTA of the cluster has started before any remote write
  for (int k = a.k1 - 1; k >= a.k0; --k) {
    const int l = k - a.k0;
    float* zb = sm + P.z + (l & 1) * kR * N;
    const float s = step_of(a, k), th = a.theta[k];
    float dth = 0.f, ds = 0.f;
    for (int e = tid; e < kR * ns; e += kThreads) {
      const int b = e / ns, n = sn.lo + e % ns, row = row0 + b;
      float dz = 0.f;
      if (row < a.batch) {
        const size_t o = ((size_t)l * a.batch + row) * N + n;
        const float z = a.zs[o], az = fabsf(z), d = dx[b * N + n];
        const bool pick = a.sel && a.sel[o];
        const bool live = az > th && z != 0.f;   // relu'(0) = 0 and sign'(z) = 0
        dz = (pick || live) ? d : 0.f;
        if (!pick && live) dth -= (z > 0.f ? d : -d);
        dzr[o] = dz;
      }
      for (int q = 0; q < kCl; ++q) cl.map_shared_rank(zb, q)[b * N + n] = dz;
    }
    cl.sync();
    const bool wterm = has_w_term(a, k);
    if (a.form == L2O_ISTA_COUPLED) {
      const float* W = w_slot(a, k);
      gemm_rows(zb, N, W, N, N, sm_.lo, sm_.hi, [&](int b, int i, float u) {
        const int row = row0 + b;
        if (row < a.batch) ds += a.rs[((size_t)l * a.batch + row) * M + i] * u;
        for (int q = 0; q < kCl; ++q) cl.map_shared_rank(rb, q)[b * M + i] = s * u;
      });
      cl.sync();
      gemm_cols(rb, M, a.A, N, M, sn.lo, sn.hi, red, [&](int b, int n, float v) { dx[b * N + n] = zb[b * N + n] - v; });
    } else if (wterm) {
      gemm_cols(zb, N, w_slot(a, k), N, N, sn.lo, sn.hi, red, [&](int b, int j, float u) {
        const int row = row0 + b;
        if (row < a.batch) {
          const float* xin = layer_input(a, l, row);
          if (xin) ds += xin[j] * u;
        }
        dx[b * N + j] = s * u;
      });
    } else {
      for (int e = tid; e < kR * ns; e += kThreads) dx[(e / ns) * N + sn.lo + e % ns] = 0.f;
      __syncthreads();
    }
    const float sth = block_sum(dth, wsum), sds = block_sum(ds, wsum);
    if (tid == 0) {
      part[((size_t)l * nblk + blockIdx.x) * 2 + 0] = sth;
      part[((size_t)l * nblk + blockIdx.x) * 2 + 1] = sds;
    }
  }
  if (p.g.d_x_in)
    for (int e = tid; e < kR * ns; e += kThreads) {
      const int b = e / ns, n = sn.lo + e % ns, row = row0 + b;
      if (row < a.batch) p.g.d_x_in[(size_t)row * N + n] = dx[b * N + n];
    }
  cl.sync();
}

// Loss rows and dL/dx (MB/utils.py): sc  0.5 ||x - x_true||^2;  lasso 0.5 (0.5 ||x A^T - y||^2) + lam ||x||_1.
__global__ void __launch_bounds__(kThreads) ista_loss_kernel(const l2o_ista_loss_args a) {
  extern __shared__ float4 smem_f4[];
  float* xr = reinterpret_cast<float*>(smem_f4);
  float* er = xr + a.n;
  __shared__ float wsum[kWarps];
  const int row = blockIdx.x, N = a.n, M = a.m, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int n = threadIdx.x; n < N; n += kThreads) xr[n] = a.x[(size_t)row * N + n];
  __syncthreads();
  float f = 0.f;
  if (a.task == L2O_ISTA_TASK_SC) {
    for (int n = threadIdx.x; n < N; n += kThreads) {
      const float d = xr[n] - a.x_true[(size_t)row * a.ldx + n];
      a.d_x[(size_t)row * N + n] = d;
      f += 0.5f * d * d;
    }
  } else {
    for (int i = w; i < M; i += kWarps) {
      float v = 0.f;
      for (int n = lane; n < N; n += 32) v = fmaf(xr[n], a.A[(size_t)i * N + n], v);
      for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) er[i] = v - a.y[(size_t)row * a.ldy + i];
    }
    __syncthreads();
    for (int i = threadIdx.x; i < M; i += kThreads) f += 0.25f * er[i] * er[i];
    for (int n = threadIdx.x; n < N; n += kThreads) {
      float v = 0.f;
      for (int i = 0; i < M; ++i) v = fmaf(er[i], a.A[(size_t)i * N + n], v);
      const float x = xr[n];
      a.d_x[(size_t)row * N + n] = 0.5f * v + a.lam * (x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f));
      f += a.lam * fabsf(x);
    }
  }
  const float s = block_sum(f, wsum);
  if (threadIdx.x == 0 && a.loss) a.loss[row] = (double)s;
}

// ---------------------------------------------------------------------------------------------------------------
// The two-state recurrences: LFISTA carries x_{k-1} besides x_k, LAMP carries v_{k-1} and a per-row threshold.
// Their own forward and backward kernels, on the helpers above; the weight-gradient kernel further down serves every
// form.
//   LFISTA (MB/models/lfista.py)  z_k = y We^T + [k>=1] x_k Wg_k^T + [k>=2] x_{k-1} Wm_k^T,  x_{k+1} = shrink(z_k)
//   LAMP   (MB/models/lamp.py)    v_k = y - x_k A^T + b_k v_{k-1}  (b_k = ||x_k||_0 / M, b_0 = 0),
//                                 r_k = x_k + s_k v_k W_k,  x_{k+1} = shrink(r_k, max(sqrt(||v_k||^2 / M) lam_k, 0))
// One cluster owns kR rows for the pass, as above.  LFISTA: one exchange per layer (z_k), the x buffers rotate.
// LAMP: an exchange of v_k (M slice) and one of r_k (N slice); every CTA forms ||v_k||^2 and ||x_k||_0 of each row
// redundantly (a warp per row, in the same order everywhere), so all of them shrink with the same threshold.

// Shared-memory plan of the two-state forms, in floats.  LFISTA: y, x_k, x_{k-1}, z double buffer, y We^T.  LAMP:
// y, x_k, v (one buffer: a CTA writes v_k only into the other CTAs' slices of its own columns, after the barrier
// that ends every read of v_{k-1} there), r double buffer.
struct Smem2 {
  int y, x, s, z, by, red, total;
};
__host__ __device__ inline Smem2 smem_plan2(const l2o_ista_args& a) {
  Smem2 s;
  s.y = 0;
  s.x = s.y + kR * a.m;
  s.s = s.x + kR * a.n;
  s.z = s.s + kR * (a.form == L2O_ISTA_LFISTA ? a.n : a.m);
  s.by = s.z + 2 * kR * a.n;
  s.red = s.by + (a.form == L2O_ISTA_LFISTA ? kR * a.n : 0);
  s.total = s.red + kThreads * kR;
  return s;
}

__device__ __forceinline__ const float* wm_slot(const l2o_ista_args& a, int k) {
  return a.W2 + (size_t)(k - 1) * a.n * a.n;
}
__device__ __forceinline__ const float* lamp_w(const l2o_ista_args& a, int k) {   // [M][N] slot k, as coupled
  return a.W + (a.share_W ? 0 : (size_t)k * a.m * a.n);
}

// out[b][j] = sum_t (in0[b][t] W0[j][t] + in1[b][t] W1[j][t]): gemm_rows over two operand pairs in one loop.
template <class F>
__device__ __forceinline__ void gemm_rows2(const float* in0, const float* __restrict__ W0, const float* in1,
                                           const float* __restrict__ W1, int ld, int T, int j0, int j1, F&& epi) {
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  for (int j = j0 + 2 * w; j < j1; j += 2 * kWarps) {
    const bool two = j + 1 < j1;
    const float *p0 = W0 + (size_t)j * ld, *q0 = W1 + (size_t)j * ld;
    const float *p1 = two ? p0 + ld : p0, *q1 = two ? q0 + ld : q0;
    float a0[kR], a1[kR];
#pragma unroll
    for (int b = 0; b < kR; ++b) a0[b] = a1[b] = 0.f;
    for (int t = lane; t < T; t += 32) {
      const float u0 = __ldg(p0 + t), u1 = __ldg(p1 + t), v0 = __ldg(q0 + t), v1 = __ldg(q1 + t);
#pragma unroll
      for (int b = 0; b < kR; ++b) {
        const float x = in0[b * ld + t], xp = in1[b * ld + t];
        a0[b] = fmaf(xp, v0, fmaf(x, u0, a0[b]));
        a1[b] = fmaf(xp, v1, fmaf(x, u1, a1[b]));
      }
    }
#pragma unroll
    for (int b = 0; b < kR; ++b)
#pragma unroll
      for (int o = 16; o; o >>= 1) {
        a0[b] += __shfl_xor_sync(0xffffffffu, a0[b], o);
        a1[b] += __shfl_xor_sync(0xffffffffu, a1[b], o);
      }
#pragma unroll
    for (int b = 0; b < kR; ++b) {
      if (lane == b) epi(b, j, a0[b]);
      if (two && lane == kR + b) epi(b, j + 1, a1[b]);
    }
  }
}

// Soft shrinkage, as the four forms do it.
__device__ __forceinline__ float shrink1(float z, float th) {
  const float m = fmaxf(fabsf(z) - th, 0.f);
  return z > 0.f ? m : (z < 0.f ? -m : 0.f);
}

__global__ void __cluster_dims__(kCl, 1, 1) __launch_bounds__(kThreads)
    ista2_fwd_kernel(const l2o_ista_args a) {
  extern __shared__ float4 smem_f4[];
  float* sm = reinterpret_cast<float*>(smem_f4);
  cg::cluster_group cl = cg::this_cluster();
  const int c = (int)cl.block_rank();
  const int row0 = (blockIdx.x / kCl) * kR;
  const int M = a.m, N = a.n, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const bool lamp = a.form == L2O_ISTA_LAMP;
  const Smem2 P = smem_plan2(a);
  float *ys = sm + P.y, *xs = sm + P.x, *s2 = sm + P.s, *by = sm + P.by, *red = sm + P.red;
  __shared__ float thr[kR], bk[kR];
  const Slice sm_ = slice_of(M, c), sn = slice_of(N, c);
  const int S = lamp ? M : N;   // width of the second state

  for (int e = tid; e < kR * M; e += kThreads) {
    const int b = e / M, i = e % M, row = row0 + b;
    ys[e] = row < a.batch ? a.y[(size_t)row * a.ldy + i] : 0.f;
  }
  for (int e = tid; e < kR * N; e += kThreads) {
    const int b = e / N, n = e % N, row = row0 + b;
    xs[e] = (a.x_in && row < a.batch) ? a.x_in[(size_t)row * N + n] : 0.f;
  }
  for (int e = tid; e < kR * S; e += kThreads) {
    const int b = e / S, n = e % S, row = row0 + b;
    s2[e] = (a.s2_in && row < a.batch) ? a.s2_in[(size_t)row * S + n] : 0.f;
  }
  __syncthreads();
  if (!lamp) gemm_rows(ys, M, a.B1, M, M, sn.lo, sn.hi, [&](int b, int n, float v) { by[b * N + n] = v; });
  cl.sync();   // every CTA of the cluster has started (and finished its prologue) before any remote write

  for (int k = a.k0; k < a.k1; ++k) {
    const int l = k - a.k0;
    float* zb = sm + P.z + (l & 1) * kR * N;
    auto put_z = [&](int b, int n, float z) {
      for (int q = 0; q < kCl; ++q) cl.map_shared_rank(zb, q)[b * N + n] = z;
    };
    if (lamp) {
      if (lane == 0) bk[w] = 0.f;
      if (k > 0) {   // b_k = ||x_k||_0 / M, a warp per row
        int cnt = 0;
        for (int n = lane; n < N; n += 32) cnt += xs[w * N + n] != 0.f;
        for (int o = 16; o; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
        if (lane == 0) bk[w] = (float)cnt / (float)M;
      }
      __syncthreads();
      gemm_rows(xs, N, a.A, N, N, sm_.lo, sm_.hi, [&](int b, int i, float u) {
        const float v = ys[b * M + i] - u + bk[b] * s2[b * M + i];
        for (int q = 0; q < kCl; ++q) cl.map_shared_rank(s2, q)[b * M + i] = v;
        if (a.rs && row0 + b < a.batch) a.rs[((size_t)l * a.batch + row0 + b) * M + i] = v;
      });
      cl.sync();
      float ss = 0.f;   // ||v_k||^2 of row w
      for (int i = lane; i < M; i += 32) ss = fmaf(s2[w * M + i], s2[w * M + i], ss);
      for (int o = 16; o; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
      const float sq = sqrtf(ss / (float)M);
      if (lane == 0) {
        thr[w] = fmaxf(sq * a.theta[k], 0.f);
        if (a.rowrec && c == 0 && row0 + w < a.batch) {
          float* rr = a.rowrec + ((size_t)l * a.batch + row0 + w) * 2;
          rr[0] = sq;
          rr[1] = bk[w];
        }
      }
      const float s = step_of(a, k);
      gemm_cols(s2, M, lamp_w(a, k), N, M, sn.lo, sn.hi, red,
                [&](int b, int n, float u) { put_z(b, n, xs[b * N + n] + s * u); });
    } else {
      auto z_of = [&](int b, int n, float u) { put_z(b, n, by[b * N + n] + u); };
      if (k >= 2) gemm_rows2(xs, a.W + (size_t)(k - 1) * N * N, s2, wm_slot(a, k), N, N, sn.lo, sn.hi, z_of);
      else if (k == 1) gemm_rows(xs, N, a.W, N, N, sn.lo, sn.hi, z_of);
      else
        for (int e = tid; e < kR * (sn.hi - sn.lo); e += kThreads) {
          const int b = e / (sn.hi - sn.lo), n = sn.lo + e % (sn.hi - sn.lo);
          put_z(b, n, by[b * N + n]);
        }
      if (lane == 0) thr[w] = a.theta[k];
    }
    cl.sync();
    float* xn = lamp ? xs : s2;   // LFISTA: x_{k+1} replaces x_{k-1}, and the buffers swap roles
    for (int e = tid; e < kR * N; e += kThreads) {
      const int b = e / N, n = e % N, row = row0 + b;
      const float z = zb[e], x = shrink1(z, thr[b]);
      xn[e] = x;
      if (n >= sn.lo && n < sn.hi && row < a.batch) {
        const size_t o = ((size_t)l * a.batch + row) * N + n;
        a.xs[o] = x;
        if (a.zs) a.zs[o] = z;
      }
    }
    if (!lamp) {
      s2 = xs;
      xs = xn;
    }
    __syncthreads();
  }
  cl.sync();   // no CTA leaves while another may still write into its shared memory
}

// x_{k-1} of pass layer l, for LFISTA's Wm term: the layer input two layers back.
__device__ __forceinline__ const float* layer_input2(const l2o_ista_args& a, int l, int row) {
  if (l == 0) return a.s2_in ? a.s2_in + (size_t)row * a.n : nullptr;
  return layer_input(a, l - 1, row);
}

__global__ void __cluster_dims__(kCl, 1, 1) __launch_bounds__(kThreads) ista2_bwd_kernel(const Bwd p) {
  extern __shared__ float4 smem_f4[];
  float* sm = reinterpret_cast<float*>(smem_f4);
  const l2o_ista_args& a = p.a;
  cg::cluster_group cl = cg::this_cluster();
  const int c = (int)cl.block_rank();
  const int row0 = (blockIdx.x / kCl) * kR;
  const int M = a.m, N = a.n, tid = threadIdx.x, lane = tid & 31, w = tid >> 5;
  const bool lamp = a.form == L2O_ISTA_LAMP;
  const Smem2 P = smem_plan2(a);
  // dx: dL/dx_{k+1} on the N slice.  s2: LFISTA the carry dL/dx_k from layer k+1's Wm term (N slice); LAMP dv, the
  // full rows of dL/dv_k after the exchange (the own M slice holds the carry before it).
  float *dx = sm + P.x, *s2 = sm + P.s, *red = sm + P.red;
  __shared__ float wsum[kWarps], gpart[kCl][kR], gcoef[kR];
  const Slice sm_ = slice_of(M, c), sn = slice_of(N, c);
  const int ns = sn.hi - sn.lo;
  const Slice ss_ = lamp ? sm_ : sn;
  const int S = lamp ? M : N, nss = ss_.hi - ss_.lo;
  float* dzr = dz_rec(p);
  float* part = part_rec(p);
  const int nblk = gridDim.x;

  for (int e = tid; e < kR * ns; e += kThreads) {
    const int b = e / ns, n = sn.lo + e % ns, row = row0 + b;
    dx[b * N + n] = row < a.batch ? p.g.d_xk[(size_t)row * N + n] : 0.f;
  }
  for (int e = tid; e < kR * nss; e += kThreads) {
    const int b = e / nss, j = ss_.lo + e % nss, row = row0 + b;
    s2[b * S + j] = (p.g.d_s2 && row < a.batch) ? p.g.d_s2[(size_t)row * S + j] : 0.f;
  }
  cl.sync();   // every CTA of the cluster has started before any remote write
  for (int k = a.k1 - 1; k >= a.k0; --k) {
    const int l = k - a.k0;
    float* zb = sm + P.z + (l & 1) * kR * N;
    float dth = 0.f, ds = 0.f;
    if (lamp) {
      // dr = dx [r != 0, |r| >= theta_b] (tf.maximum sends the gradient to |r| - theta on ties); a warp per row, so
      // the row's partial of g = dL/dtheta_b is summed in a fixed order.
      const int row = row0 + w;
      const bool ok = row < a.batch;
      const float sq = ok ? a.rowrec[((size_t)l * a.batch + row) * 2] : 0.f;
      const float th = fmaxf(sq * a.theta[k], 0.f);
      float g = 0.f;
      for (int n = sn.lo + lane; n < sn.hi; n += 32) {
        float dr = 0.f;
        if (ok) {
          const size_t o = ((size_t)l * a.batch + row) * N + n;
          const float r = a.zs[o], d = dx[w * N + n];
          if (r != 0.f && fabsf(r) >= th) {
            dr = d;
            g -= r > 0.f ? d : -d;
          }
          dzr[o] = dr;
        }
        for (int q = 0; q < kCl; ++q) cl.map_shared_rank(zb, q)[w * N + n] = dr;
      }
      for (int o = 16; o; o >>= 1) g += __shfl_xor_sync(0xffffffffu, g, o);
      if (lane < kCl) cl.map_shared_rank(&gpart[0][0], lane)[c * kR + w] = g;
      cl.sync();
      if (lane == 0) {
        float gs = 0.f;
        for (int q = 0; q < kCl; ++q) gs += gpart[q][w];
        const float lk = a.theta[k];
        // theta = max(sqrt(rvar) lam, 0): d theta / d v = lam v / (M sqrt(rvar)) where sqrt(rvar) lam >= 0; a row
        // with rvar = 0 contributes nothing (TF's sqrt gradient would give inf * 0 there).
        gcoef[w] = (sq * lk >= 0.f && sq > 0.f) ? gs * lk / ((float)M * sq) : 0.f;
        if (c == 0 && sq * lk >= 0.f) dth = gs * sq;   // dlam_k, added by one CTA per cluster
      }
      __syncthreads();
      const float s = step_of(a, k);
      gemm_rows(zb, N, lamp_w(a, k), N, N, sm_.lo, sm_.hi, [&](int b, int i, float u) {
        const int rw = row0 + b;
        float dv = 0.f;
        if (rw < a.batch) {
          const float v = a.rs[((size_t)l * a.batch + rw) * M + i];
          const float carry = k + 1 < a.k1 ? a.rowrec[((size_t)(l + 1) * a.batch + rw) * 2 + 1] * s2[b * M + i]
                                           : s2[b * M + i];
          ds += v * u;
          dv = fmaf(s, u, fmaf(gcoef[b], v, carry));
        }
        for (int q = 0; q < kCl; ++q) cl.map_shared_rank(s2, q)[b * M + i] = dv;
      });
      cl.sync();
      gemm_cols(s2, M, a.A, N, M, sn.lo, sn.hi, red, [&](int b, int n, float v) { dx[b * N + n] = zb[b * N + n] - v; });
    } else {
      const float th = a.theta[k];
      for (int e = tid; e < kR * ns; e += kThreads) {
        const int b = e / ns, n = sn.lo + e % ns, row = row0 + b;
        float dz = 0.f;
        if (row < a.batch) {
          const size_t o = ((size_t)l * a.batch + row) * N + n;
          const float z = a.zs[o], d = dx[b * N + n];
          if (fabsf(z) > th && z != 0.f) {   // relu'(0) = 0 and sign'(z) = 0
            dz = d;
            dth -= z > 0.f ? d : -d;
          }
          dzr[o] = dz;
        }
        for (int q = 0; q < kCl; ++q) cl.map_shared_rank(zb, q)[b * N + n] = dz;
      }
      cl.sync();
      // dx_k = dz_k Wg_k + carry;  the carry for x_{k-1} is dz_k Wm_k, local to the slice.
      if (k >= 1)
        gemm_cols(zb, N, a.W + (size_t)(k - 1) * N * N, N, N, sn.lo, sn.hi, red,
                  [&](int b, int j, float u) { dx[b * N + j] = u + s2[b * N + j]; });
      else
        for (int e = tid; e < kR * ns; e += kThreads) dx[(e / ns) * N + sn.lo + e % ns] = s2[(e / ns) * N + sn.lo + e % ns];
      if (k >= 2)
        gemm_cols(zb, N, wm_slot(a, k), N, N, sn.lo, sn.hi, red, [&](int b, int j, float u) { s2[b * N + j] = u; });
      else
        for (int e = tid; e < kR * ns; e += kThreads) s2[(e / ns) * N + sn.lo + e % ns] = 0.f;
      __syncthreads();
    }
    const float sth = block_sum(dth, wsum), sds = block_sum(ds, wsum);
    if (tid == 0) {
      part[((size_t)l * nblk + blockIdx.x) * 2 + 0] = sth;
      part[((size_t)l * nblk + blockIdx.x) * 2 + 1] = sds;
    }
  }
  if (p.g.d_x_in)
    for (int e = tid; e < kR * ns; e += kThreads) {
      const int b = e / ns, n = sn.lo + e % ns, row = row0 + b;
      if (row < a.batch) p.g.d_x_in[(size_t)row * N + n] = dx[b * N + n];
    }
  if (p.g.d_s2_in)   // LFISTA: the carry dz_{k0} Wm_{k0};  LAMP: b_{k0} dv_{k0}
    for (int e = tid; e < kR * nss; e += kThreads) {
      const int b = e / nss, j = ss_.lo + e % nss, row = row0 + b;
      if (row < a.batch)
        p.g.d_s2_in[(size_t)row * S + j] = lamp ? a.rowrec[(size_t)row * 2 + 1] * s2[b * S + j] : s2[b * S + j];
    }
  cl.sync();
}

// The weight slots of the gradient launch, in blockIdx.y order: the W slots (nw), LFISTA's Wm slots (nw2), then B1
// (LFISTA: We).  Slot C [Pd][Qd] = gscale[birth] sum_{l in [la, lb)} c_l sum_b P_l[b][p] Q_l[b][q], c_l = s_k (1 for
// B1), over the pass layers [la, lb) that have the slot's term (la >= lb: the slot's gradient is 0 in this pass):
//   coupled, LAMP  dW_k = s_k r_k^T dz_k      (P = rs, Q = dz)
//   LISTA, LFISTA  dW_k = s_k dz_k^T x_k      (P = dz, Q = x_k);   LFISTA dWm_k = dz_k^T x_{k-1}  (Q = x_{k-1})
//   dB1 = sum_k dz_k^T y                      (P = dz, Q = y)
enum : int { kRsDz, kDzX, kDzXm, kDzY };
struct Slot {
  double* out;
  int Pd, Qd, la, lb, birth, op;
};
__host__ inline int w_slots(const l2o_ista_args& a) {
  if (a.share_W) return 1;
  return w_on_r(a) ? a.num_layers : a.num_layers - 1;
}
__device__ inline Slot grad_slot(const Bwd& p, int y, int nw, int nw2) {
  const l2o_ista_args& a = p.a;
  if (y >= nw + nw2) return {p.g.dB1, a.n, a.m, 0, a.k1 - a.k0, 0, kDzY};
  const bool on_r = w_on_r(a), wm = y >= nw;
  const int g = wm ? y - nw : y, first = on_r ? 0 : 1;   // first: the first layer with a W term
  Slot s;
  s.Pd = on_r ? a.m : a.n;
  s.Qd = a.n;
  s.op = on_r ? kRsDz : (wm ? kDzXm : kDzX);
  s.out = (wm ? p.g.dW2 : p.g.dW) + (size_t)g * s.Pd * s.Qd;
  if (a.share_W) {
    s.birth = first;
    s.la = max(a.k0, first) - a.k0;
    s.lb = a.k1 - a.k0;
  } else {
    const int k = g + first;
    const bool in = k >= a.k0 && k < a.k1 && (!wm || k >= 2);   // Wm_1 is never read
    s.birth = k;
    s.la = in ? k - a.k0 : 0;
    s.lb = in ? s.la + 1 : 0;
  }
  return s;
}

// blockIdx.y < nw + nw2 + nb1: a weight slot, 64 x 64 output tiles (4 x 4 per thread); the last: dtheta and ds
// (blockIdx.x = layer).  Held to 80 registers (3 CTAs per SM).
__global__ void __launch_bounds__(kThreads, 3) ista_grad_kernel(const Bwd p, int nblk_bwd, int nw, int nw2, int nb1) {
  const l2o_ista_args& a = p.a;
  const int M = a.m, N = a.n, B = a.batch;
  if ((int)blockIdx.y == nw + nw2 + nb1) {   // per-layer scalars (LAMP: dlam)
    const int k = blockIdx.x;
    if (k >= a.num_layers) return;
    const float* part = part_rec(p);
    __shared__ double acc[2][kWarps];
    double t = 0.0, s = 0.0;
    if (k >= a.k0 && k < a.k1)
      for (int i = threadIdx.x; i < nblk_bwd; i += kThreads) {
        t += part[((size_t)(k - a.k0) * nblk_bwd + i) * 2];
        s += part[((size_t)(k - a.k0) * nblk_bwd + i) * 2 + 1];
      }
    for (int o = 16; o; o >>= 1) {
      t += __shfl_xor_sync(0xffffffffu, t, o);
      s += __shfl_xor_sync(0xffffffffu, s, o);
    }
    if ((threadIdx.x & 31) == 0) acc[0][threadIdx.x >> 5] = t, acc[1][threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
      t = s = 0.0;
      for (int w = 0; w < kWarps; ++w) t += acc[0][w], s += acc[1][w];
      const double sc = p.g.gscale ? (double)p.g.gscale[k] : 1.0;
      p.g.dtheta[k] = sc * t;
      if (p.g.dstep) p.g.dstep[k] = sc * s;
    }
    return;
  }
  const Slot sl = grad_slot(p, blockIdx.y, nw, nw2);
  const int Pd = sl.Pd, Qd = sl.Qd;
  const float* dzr = dz_rec(p);
  const int tiles_q = (Qd + kTile - 1) / kTile, tiles = tiles_q * ((Pd + kTile - 1) / kTile);
  if ((int)blockIdx.x >= tiles) return;
  const int p0 = (blockIdx.x / tiles_q) * kTile, q0 = (blockIdx.x % tiles_q) * kTile;
  __shared__ float Ps[kChunk][kTile], Qs[kChunk][kTile];
  const int tp = threadIdx.x / 16, tq = threadIdx.x % 16;
  double acc[4][4] = {};   // per-layer fp32 sums, added across layers in fp64 (a shared W or B1 sums K of them)
  for (int l = sl.la; l < sl.lb; ++l) {
    float lacc[4][4] = {};
    const float coef = sl.op == kDzY ? 1.f : step_of(a, a.k0 + l);
    for (int b0 = 0; b0 < B; b0 += kChunk) {
      for (int e = threadIdx.x; e < kChunk * kTile; e += kThreads) {
        const int bb = e / kTile, j = e % kTile, row = b0 + bb;
        float pv = 0.f, qv = 0.f;
        if (row < B) {
          const float* dz = dzr + ((size_t)l * B + row) * N;
          if (sl.op == kRsDz) {
            if (p0 + j < Pd) pv = a.rs[((size_t)l * B + row) * M + p0 + j];
            if (q0 + j < Qd) qv = dz[q0 + j];
          } else {
            if (p0 + j < Pd) pv = dz[p0 + j];
            if (q0 + j < Qd) {
              if (sl.op == kDzY) qv = a.y[(size_t)row * a.ldy + q0 + j];
              else {
                const float* xin = sl.op == kDzX ? layer_input(a, l, row) : layer_input2(a, l, row);
                qv = xin ? xin[q0 + j] : 0.f;
              }
            }
          }
        }
        Ps[bb][j] = coef * pv;
        Qs[bb][j] = qv;
      }
      __syncthreads();
#pragma unroll
      for (int bb = 0; bb < kChunk; ++bb) {
        float pr[4], qr[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) pr[i] = Ps[bb][tp + 16 * i], qr[i] = Qs[bb][tq + 16 * i];
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) lacc[i][j] = fmaf(pr[i], qr[j], lacc[i][j]);
      }
      __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] += (double)lacc[i][j];
  }
  const double sc = p.g.gscale && sl.birth < a.num_layers ? (double)p.g.gscale[sl.birth] : 1.0;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int pp = p0 + tp + 16 * i, qq = q0 + tq + 16 * j;
      if (pp < Pd && qq < Qd) sl.out[(size_t)pp * Qd + qq] = sc * acc[i][j];
    }
}

inline bool two_state(const l2o_ista_args& a) { return a.form == L2O_ISTA_LFISTA || a.form == L2O_ISTA_LAMP; }
inline int plan_floats(const l2o_ista_args& a) { return two_state(a) ? smem_plan2(a).total : smem_plan(a).total; }

int check_args(const l2o_ista_args* a) {
  if (!a || a->form < L2O_ISTA_LISTA || a->form > L2O_ISTA_LAMP) return L2O_E_INVALID;
  if (a->batch <= 0 || a->m <= 0 || a->n <= 0 || a->num_layers <= 0 || a->k0 < 0 || a->k0 >= a->k1 ||
      a->k1 > a->num_layers || a->share_W < 0 || a->share_W > 1 || a->ldy < a->m)
    return L2O_E_INVALID;
  if (!a->theta || !a->y) return L2O_E_INVALID;
  if ((a->form == L2O_ISTA_COUPLED || a->form == L2O_ISTA_LAMP) && (!a->A || !a->W)) return L2O_E_INVALID;
  if (a->form == L2O_ISTA_LISTA && (!a->B1 || (a->k1 > 1 && !a->W))) return L2O_E_INVALID;
  if (a->form == L2O_ISTA_LFISTA &&
      (!a->B1 || (a->k1 > 1 && !a->W) || (a->k1 > 2 && !a->W2) || a->share_W || a->step))
    return L2O_E_INVALID;
  if (two_state(*a) && a->ss_rank) return L2O_E_INVALID;
  const void* ptrs[] = {a->A,  a->B1, a->W,  a->theta, a->step,  a->ss_rank, a->y,     a->x_in,
                        a->xs, a->zs, a->rs, a->W2,    a->s2_in, a->rowrec};
  for (const void* q : ptrs)
    if (misaligned(q, 4)) return L2O_E_INVALID;
  if (a->m > kMaxDim || a->n > kMaxDim) return L2O_E_UNSUPPORTED;
  if ((size_t)plan_floats(*a) * sizeof(float) > 200 * 1024) return L2O_E_UNSUPPORTED;
  return L2O_OK;
}

inline int clusters(const l2o_ista_args& a) { return (a.batch + kR - 1) / kR; }
inline int tiles_of(int len) { return (len + kTile - 1) / kTile; }

size_t scratch_bytes(const l2o_ista_args& a) {
  const size_t L = (size_t)(a.k1 - a.k0);
  return 4 * (L * a.batch * a.n + L * clusters(a) * kCl * 2);
}

}  // namespace ista
}  // namespace l2o

using namespace l2o::ista;

extern "C" {

int l2o_ista_workspace_bytes(const l2o_ista_args* a, size_t* bytes) {
  if (!bytes) return L2O_E_INVALID;
  if (int rc = check_args(a)) return rc;
  *bytes = scratch_bytes(*a);
  return L2O_OK;
}

int l2o_ista_fwd(const l2o_ista_args* a, void* stream) {
  if (int rc = check_args(a)) return rc;
  if (!a->xs) return L2O_E_INVALID;
  const auto kernel = two_state(*a) ? ista2_fwd_kernel : ista_fwd_kernel;
  const size_t smem = (size_t)plan_floats(*a) * sizeof(float);
  if (int rc = l2o::raise_smem_limit("l2o_ista_fwd", kernel, smem)) return rc;
  kernel<<<clusters(*a) * kCl, kThreads, smem, (cudaStream_t)stream>>>(*a);
  return l2o::after_launch("l2o_ista_fwd");
}

int l2o_ista_bwd(const l2o_ista_args* a, const l2o_ista_grads* g, void* stream) {
  if (int rc = check_args(a)) return rc;
  if (!g || !a->xs || !a->zs || !g->d_xk || !g->dtheta || !g->scratch) return L2O_E_INVALID;
  if (a->ss_rank && !a->sel) return L2O_E_INVALID;
  if (a->form == L2O_ISTA_COUPLED && !a->rs) return L2O_E_INVALID;
  if (a->form == L2O_ISTA_LISTA && !g->dB1) return L2O_E_INVALID;
  if (a->form == L2O_ISTA_LFISTA && !g->dB1) return L2O_E_INVALID;
  if (a->form == L2O_ISTA_LAMP && (!a->rs || !a->rowrec)) return L2O_E_INVALID;
  const void* f4[] = {g->d_xk, g->d_x_in, g->gscale, g->scratch, g->d_s2, g->d_s2_in};
  for (const void* q : f4)
    if (l2o::misaligned(q, 4)) return L2O_E_INVALID;
  const void* f8[] = {g->dW, g->dB1, g->dtheta, g->dstep, g->dW2};
  for (const void* q : f8)
    if (l2o::misaligned(q, 8)) return L2O_E_INVALID;
  Bwd p{*a, *g};
  const auto kernel = two_state(*a) ? ista2_bwd_kernel : ista_bwd_kernel;
  const size_t smem = (size_t)plan_floats(*a) * sizeof(float);
  if (int rc = l2o::raise_smem_limit("l2o_ista_bwd", kernel, smem)) return rc;
  const int nblk = clusters(*a) * kCl;
  kernel<<<nblk, kThreads, smem, (cudaStream_t)stream>>>(p);
  if (int rc = l2o::after_launch("l2o_ista_bwd")) return rc;
  const int nw = g->dW ? w_slots(*a) : 0, nw2 = a->form == L2O_ISTA_LFISTA && g->dW2 ? w_slots(*a) : 0;
  const int nb1 = a->form == L2O_ISTA_LISTA || a->form == L2O_ISTA_LFISTA ? 1 : 0;   // dB1 is required there
  int tiles = std::max(tiles_of(w_on_r(*a) ? a->m : a->n) * tiles_of(a->n), a->num_layers);
  if (nb1) tiles = std::max(tiles, tiles_of(a->n) * tiles_of(a->m));
  ista_grad_kernel<<<dim3(tiles, nw + nw2 + nb1 + 1), kThreads, 0, (cudaStream_t)stream>>>(p, nblk, nw, nw2, nb1);
  return l2o::after_launch("l2o_ista_bwd");
}

int l2o_ista_loss_grad(const l2o_ista_loss_args* a, void* stream) {
  if (!a || (a->task != L2O_ISTA_TASK_SC && a->task != L2O_ISTA_TASK_LASSO) || a->batch <= 0 || a->m <= 0 ||
      a->n <= 0 || !a->x || !a->d_x)
    return L2O_E_INVALID;
  if (a->task == L2O_ISTA_TASK_SC && (!a->x_true || a->ldx < a->n)) return L2O_E_INVALID;
  if (a->task == L2O_ISTA_TASK_LASSO && (!a->A || !a->y || a->ldy < a->m)) return L2O_E_INVALID;
  const void* f4[] = {a->A, a->y, a->x_true, a->x, a->d_x};
  for (const void* q : f4)
    if (l2o::misaligned(q, 4)) return L2O_E_INVALID;
  if (l2o::misaligned(a->loss, 8)) return L2O_E_INVALID;
  const size_t smem = (size_t)(a->n + a->m) * sizeof(float);
  if (smem > 200 * 1024) return L2O_E_UNSUPPORTED;
  if (int rc = l2o::raise_smem_limit("l2o_ista_loss_grad", ista_loss_kernel, smem)) return rc;
  ista_loss_kernel<<<a->batch, kThreads, smem, (cudaStream_t)stream>>>(*a);
  return l2o::after_launch("l2o_ista_loss_grad");
}

}  // extern "C"
