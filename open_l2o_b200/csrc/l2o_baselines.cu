// L2O-Scale's meta-trained hand-designed baselines — sm_90a CUDA kernels + C-ABI.
// SC/ = Model_Free_L2O/L2O-Scale/L2O-Scale-Training/ of the reference; TA = SC/optimizer/trainable_adam.py,
// GLR = global_learning_rate.py, LRS = learning_rate_schedule.py.
//
// All three are coordinate-wise, so one step over all optimizee tensors is ONE launch over the concatenated coordinates,
// and one backward step is one launch.  theta stays on the device: the kernels read TrainableAdam's four scalars and the
// schedule from device memory, and the schedule's step counter is read and advanced on the device, so a step captured
// in a CUDA graph replays with no host synchronisation and the schedule still advances.
//
// TrainableAdam (TA:95-175), theta = (log_learning_rate, beta1_logit, beta2_logit, log_epsilon), state planes m | t | v:
//   b1 = sigmoid(beta1_logit); b2 = sigmoid(beta2_logit); eps = exp(log_epsilon) + 1e-10; lr = exp(log_learning_rate)
//   t' = t + 1;  m' = b1 m + (1 - b1) g;  v' = v / (1 - pow(g^2, b2))      <- TA:133-134, arguments in the wrong slots
//   upd = lr (m' / (1 - b1^t')) / (sqrt(v' / (1 - b2^t') + 1e-10) + eps);  x' = x - upd
// The second moment is the reference as written: from v = 0 it stays 0 (or -0), except where g^2 == 1 rounds pow to
// exactly 1 and v' = 0/0 = NaN.  Both outcomes are computed literally (CUDA's powf is exact for base 1 and base 0).
//
// LearningRateSchedule (LRS:48-60): x' = x - rates[min(itr, n_steps - 1)] g, itr' = itr + 1.  GlobalLearningRate
// (GLR:38-39) is the same kernel with a one-entry table and no counter.
#include <cmath>
#include <cstdint>

#include "l2o_internal.h"

namespace l2o {
namespace baselines {

constexpr int kBlock = 256;
constexpr int kTheta = 4, kPlanes = 3;
constexpr int P_M = 0, P_T = 1, P_V = 2;   // sorted slot keys, the order flatten_and_sort uses (SC TO:85, 686-688)

// The four scalars, each computed in fp64 and rounded once: 1 - b1 and 1 - b1^t' cancel by 1000x at b1 = 0.999, so
// an fp32 sigmoid's last-ulp error would show at 1e-4 in the update.  The CPU oracle rounds the same way.
struct Scalars {
  float b1, b2, lr, eps, exp_le;
};
__device__ __forceinline__ Scalars scalars(const float* __restrict__ th) {
  Scalars s;
  s.lr = (float)exp((double)th[0]);
  s.b1 = (float)(1.0 / (1.0 + exp(-(double)th[1])));
  s.b2 = (float)(1.0 / (1.0 + exp(-(double)th[2])));
  s.exp_le = (float)exp((double)th[3]);
  s.eps = __fadd_rn(s.exp_le, 1e-10f);
  return s;
}

// 1 - b^t' with b^t' correctly rounded to fp32 (fp64 pow is accurate to < 1 ulp of fp64, far inside half an fp32 ulp,
// so the rounding is the correct one except where the fp64 value falls within 2^-29 relative of an fp32 tie).  Every
// coordinate of a run has the same t, so each thread recomputes the pair only when its t' changes.
struct Debias {
  float tp = -1.0f, c1 = 0.f, c2 = 0.f, p1 = 0.f, p2 = 0.f;
  __device__ __forceinline__ void at(float t_new, float b1, float b2) {
    if (t_new != tp) {
      tp = t_new;
      p1 = (float)pow((double)b1, (double)t_new);
      p2 = (float)pow((double)b2, (double)t_new);
      c1 = __fsub_rn(1.0f, p1);
      c2 = __fsub_rn(1.0f, p2);
    }
  }
};

struct TadamFwd {   // the forward values of one coordinate, every operation rounded on its own as TF's graph does
  float tn, mn, gg, q, one_q, vn, mh, vh, s, den, num, upd;
};
__device__ __forceinline__ TadamFwd tadam_fwd(const Scalars& k, Debias& db, float g, float m, float t, float v) {
  TadamFwd f;
  f.tn = __fadd_rn(t, 1.0f);
  f.mn = __fadd_rn(__fmul_rn(k.b1, m), __fmul_rn(__fsub_rn(1.0f, k.b1), g));
  f.gg = __fmul_rn(g, g);
  f.q = powf(f.gg, k.b2);
  f.one_q = __fsub_rn(1.0f, f.q);
  f.vn = __fdiv_rn(v, f.one_q);
  db.at(f.tn, k.b1, k.b2);
  f.mh = __fdiv_rn(f.mn, db.c1);
  f.vh = __fdiv_rn(f.vn, db.c2);
  f.s = __fsqrt_rn(__fadd_rn(f.vh, 1e-10f));
  f.den = __fadd_rn(f.s, k.eps);
  f.num = __fmul_rn(k.lr, f.mh);
  f.upd = __fdiv_rn(f.num, f.den);
  return f;
}

struct TadamStep {
  int64_t n;
  const float* theta;
  const float* g;
  const float* state_in;
  float* state_out;
  float* x;
  float* update;
};

// forward step: reads x g m t v, writes x m t v (36 B per coordinate)
__global__ void __launch_bounds__(kBlock) tadam_step_kernel(TadamStep a) {
  const Scalars k = scalars(a.theta);
  Debias db;
  const int64_t n = a.n;
  for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const float g = a.g[i];
    const float m = a.state_in[P_M * n + i], t = a.state_in[P_T * n + i], v = a.state_in[P_V * n + i];
    const TadamFwd f = tadam_fwd(k, db, g, m, t, v);
    a.state_out[P_M * n + i] = f.mn;
    a.state_out[P_T * n + i] = f.tn;
    a.state_out[P_V * n + i] = f.vn;
    if (a.x) a.x[i] = __fsub_rn(a.x[i], f.upd);
    if (a.update) a.update[i] = f.upd;
  }
}

// Block-wide sum of NV fp64 partials, then one fp64 atomic per entry per CTA (no per-coordinate global atomics).
template <int NV>
__device__ __forceinline__ void block_flush(double (&acc)[NV], const double (&scale)[NV], double* const (&dst)[NV]) {
  __shared__ double red[kBlock / 32][NV];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int j = 0; j < NV; ++j) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[j] += __shfl_xor_sync(0xffffffffu, acc[j], o);
    if (lane == 0) red[warp][j] = acc[j];
  }
  __syncthreads();
  if (threadIdx.x == 0) {   // (one thread, static indices: a thread-indexed pick would put the arrays on the stack)
#pragma unroll
    for (int j = 0; j < NV; ++j) {
      double s = 0.0;
#pragma unroll
      for (int w = 0; w < kBlock / 32; ++w) s += red[w][j];
      atomicAdd(dst[j], s * scale[j]);
    }
  }
}

struct TadamBwd {
  int64_t n;
  const float* theta;
  const float* g;
  const float* state_old;
  const float* d_state_new;
  const float* d_update;
  float* d_state_old;
  double* d_theta;
  float* d_g;
};

// backward: recompute the step from the old planes, then its adjoints.  t carries no adjoint (d t = 0).  Where v == 0
// (every reachable state but the NaN one) the v-chain contributes exactly 0 to theta and g: the g^2 and b2 terms of
// pow(g^2, b2) and the b2 term of the debias are not formed, because their literal form is 0 * inf at g = 0 (and, for
// the debias, once the adjoint of v^ overflows at |g| >~ 1e19).  See DESIGN §3.10.
__global__ void __launch_bounds__(kBlock) tadam_bwd_kernel(TadamBwd a) {
  const Scalars k = scalars(a.theta);
  Debias db;
  const int64_t n = a.n;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};   // sum d upd * upd | d eps | d b1 | d b2
  for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kBlock) {
    const float g = a.g[i];
    const float m = a.state_old[P_M * n + i], t = a.state_old[P_T * n + i], v = a.state_old[P_V * n + i];
    const TadamFwd f = tadam_fwd(k, db, g, m, t, v);
    const float du = a.d_update[i];
    // upd = num / den, num = lr mh, den = sqrt(vh + 1e-10) + eps
    const float dnum = du / f.den;
    const float dden = -du * f.upd / f.den;
    const float dmh = dnum * k.lr;
    const float dvh = dden * 0.5f / f.s;
    const float dmn = a.d_state_new[P_M * n + i] + dmh / db.c1;
    const float dvn = a.d_state_new[P_V * n + i] + dvh / db.c2;
    const float db1 = dmh * f.mh / db.c1 * f.tn * db.p1 / k.b1 + dmn * (m - g);   // through b1^t' and m'
    float db2 = 0.0f, dg = dmn * (1.0f - k.b1);
    if (v != 0.0f) {   // v' = v / (1 - q), q = pow(g^2, b2); v^ = v' / (1 - b2^t')
      db2 = dvh * f.vh / db.c2 * f.tn * db.p2 / k.b2;
      const float dq = dvn * f.vn / f.one_q;
      // at g^2 == 0 (g == 0, or |g| below ~1e-23 where g^2 underflows) pow's derivatives are taken as 0: the limit in
      // b2 always, in g for b2 > 1/2; the literal forms are inf * 0 and 0 * -inf
      if (f.gg != 0.0f) {
        dg += dq * k.b2 * powf(f.gg, k.b2 - 1.0f) * 2.0f * g;
        db2 += dq * f.q * logf(f.gg);
      }
    }
    a.d_state_old[P_M * n + i] = dmn * k.b1;
    a.d_state_old[P_T * n + i] = 0.0f;
    a.d_state_old[P_V * n + i] = dvn / f.one_q;
    if (a.d_g) a.d_g[i] = dg;
    acc[0] += (double)(du * f.upd);   // d log_lr = d upd * upd (upd is linear in lr = exp(log_lr))
    acc[1] += (double)dden;
    acc[2] += (double)db1;
    acc[3] += (double)db2;
  }
  const double scale[4] = {1.0, (double)k.exp_le, (double)k.b1 * (1.0 - (double)k.b1),
                           (double)k.b2 * (1.0 - (double)k.b2)};
  double* const dst[4] = {a.d_theta, a.d_theta + 1, a.d_theta + 2, a.d_theta + 3};
  // theta order: log_lr, beta1_logit, beta2_logit, log_epsilon; acc order: lr, eps, b1, b2
  double acc_t[4] = {acc[0], acc[2], acc[3], acc[1]};
  const double scale_t[4] = {scale[0], scale[2], scale[3], scale[1]};
  block_flush<4>(acc_t, scale_t, dst);
}

// ------------------------------------------------------------------------------------------------------------------
// LearningRateSchedule / GlobalLearningRate.  itr = {step index, CTA arrival count (0 between launches)}: every CTA reads
// the index before it arrives, and the last CTA to arrive writes index + 1 and resets the count, so the counter is
// advanced in place, race-free, within the one launch.
struct LrsStep {
  int64_t n;
  const float* rates;
  int32_t n_steps;
  int32_t* itr;
  const float* g;
  float* x;
  float* update;
};

__device__ __forceinline__ int lrs_index(int itr, int n_steps) {   // tf.minimum(itr, n_steps - 1) (LRS:54)
  return itr < n_steps - 1 ? (itr > 0 ? itr : 0) : n_steps - 1;
}

__global__ void __launch_bounds__(kBlock) lrs_step_kernel(LrsStep a) {
  __shared__ int s_itr;
  if (threadIdx.x == 0) s_itr = a.itr ? a.itr[0] : 0;
  __syncthreads();
  const float lr = a.rates[lrs_index(s_itr, a.n_steps)];
  for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * kBlock) {
    const float upd = __fmul_rn(lr, a.g[i]);
    if (a.x) a.x[i] = __fsub_rn(a.x[i], upd);
    if (a.update) a.update[i] = upd;
  }
  if (a.itr && threadIdx.x == 0) {
    __threadfence();   // this CTA's read of itr[0] is ordered before its arrival
    if (atomicAdd(&a.itr[1], 1) == (int)gridDim.x - 1) {
      a.itr[0] = s_itr + 1;
      a.itr[1] = 0;
    }
  }
}

struct LrsBwd {
  int64_t n;
  const float* rates;
  int32_t n_steps;
  const int32_t* itr;
  const float* g;
  const float* d_update;
  double* d_rates;
  float* d_g;
};

// d rates[index] += sum d_update g; d g = rate d_update
__global__ void __launch_bounds__(kBlock) lrs_bwd_kernel(LrsBwd a) {
  const int idx = lrs_index(a.itr ? a.itr[0] : 0, a.n_steps);
  const float lr = a.rates[idx];
  double acc[1] = {0.0};
  for (int64_t i = (int64_t)blockIdx.x * kBlock + threadIdx.x; i < a.n; i += (int64_t)gridDim.x * kBlock) {
    const float du = a.d_update[i];
    acc[0] += (double)(du * a.g[i]);
    if (a.d_g) a.d_g[i] = lr * du;
  }
  const double scale[1] = {1.0};
  double* const dst[1] = {a.d_rates + idx};
  block_flush<1>(acc, scale, dst);
}

}  // namespace baselines
}  // namespace l2o

using namespace l2o::baselines;

extern "C" {

int64_t l2o_tadam_theta_count(void) { return kTheta; }
int64_t l2o_tadam_state_floats(void) { return kPlanes; }

int l2o_tadam_step(const l2o_tadam_step_args* a, void* stream) {
  if (!a || a->n <= 0 || a->n > INT64_MAX / kPlanes || !a->theta || !a->g || !a->state_in || !a->state_out)
    return L2O_E_INVALID;
  const void* fp[] = {a->theta, a->g, a->state_in, a->state_out, a->x, a->update};
  for (const void* p : fp)
    if (l2o::misaligned(p, alignof(float))) return L2O_E_INVALID;
  TadamStep k{a->n, a->theta, a->g, a->state_in, a->state_out, a->x, a->update};
  return l2o::occupancy_launch("l2o_tadam_step", tadam_step_kernel, kBlock, 0, a->n, (cudaStream_t)stream, k);
}

int l2o_tadam_bwd(const l2o_tadam_bwd_args* a, void* stream) {
  if (!a || a->n <= 0 || a->n > INT64_MAX / kPlanes || !a->theta || !a->g || !a->state_old || !a->d_state_new ||
      !a->d_update || !a->d_state_old || !a->d_theta)
    return L2O_E_INVALID;
  const void* fp[] = {a->theta, a->g, a->state_old, a->d_state_new, a->d_update, a->d_state_old, a->d_g};
  for (const void* p : fp)
    if (l2o::misaligned(p, alignof(float))) return L2O_E_INVALID;
  if (l2o::misaligned(a->d_theta, alignof(double))) return L2O_E_INVALID;
  if (a->d_g) {
    const size_t n = (size_t)a->n, f = sizeof(float);
    const void* other[] = {a->theta, a->g, a->state_old, a->d_state_new, a->d_update, a->d_state_old, a->d_theta};
    const size_t bytes[] = {kTheta * f, n * f, kPlanes * n * f, kPlanes * n * f, n * f, kPlanes * n * f,
                            kTheta * sizeof(double)};
    if (l2o::overlaps_any(a->d_g, n * f, other, bytes, 7)) return L2O_E_INVALID;
  }
  TadamBwd k{a->n, a->theta, a->g, a->state_old, a->d_state_new, a->d_update, a->d_state_old, a->d_theta, a->d_g};
  return l2o::occupancy_launch("l2o_tadam_bwd", tadam_bwd_kernel, kBlock, 0, a->n, (cudaStream_t)stream, k);
}

int l2o_lrsgd_step(const l2o_lrsgd_step_args* a, void* stream) {
  if (!a || a->n <= 0 || a->n_steps <= 0 || !a->rates || !a->g) return L2O_E_INVALID;
  const void* fp[] = {a->rates, a->g, a->x, a->update, a->itr};
  for (const void* p : fp)
    if (l2o::misaligned(p, 4)) return L2O_E_INVALID;
  LrsStep k{a->n, a->rates, a->n_steps, a->itr, a->g, a->x, a->update};
  return l2o::occupancy_launch("l2o_lrsgd_step", lrs_step_kernel, kBlock, 0, a->n, (cudaStream_t)stream, k);
}

int l2o_lrsgd_bwd(const l2o_lrsgd_bwd_args* a, void* stream) {
  if (!a || a->n <= 0 || a->n_steps <= 0 || !a->rates || !a->g || !a->d_update || !a->d_rates) return L2O_E_INVALID;
  const void* fp[] = {a->rates, a->g, a->d_update, a->itr, a->d_g};
  for (const void* p : fp)
    if (l2o::misaligned(p, 4)) return L2O_E_INVALID;
  if (l2o::misaligned(a->d_rates, alignof(double))) return L2O_E_INVALID;
  if (a->d_g) {
    const size_t n = (size_t)a->n, f = sizeof(float);
    const void* other[] = {a->rates, a->g, a->d_update, a->itr, a->d_rates};
    const size_t bytes[] = {(size_t)a->n_steps * f, n * f, n * f, 2 * sizeof(int32_t), (size_t)a->n_steps * sizeof(double)};
    if (l2o::overlaps_any(a->d_g, n * f, other, bytes, 5)) return L2O_E_INVALID;
  }
  LrsBwd k{a->n, a->rates, a->n_steps, a->itr, a->g, a->d_update, a->d_rates, a->d_g};
  return l2o::occupancy_launch("l2o_lrsgd_bwd", lrs_bwd_kernel, kBlock, 0, a->n, (cudaStream_t)stream, k);
}

}  // extern "C"
