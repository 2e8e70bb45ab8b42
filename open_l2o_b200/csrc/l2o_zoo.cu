// The analytic families of L2O-Scale's problem zoo (SC/problems/problem_generator.py; SC/ =
// Model_Free_L2O/L2O-Scale/L2O-Scale-Training/): f(x) with df/dx, or H(x) v, at one parameter vector in ONE launch.
// The zoo's problems have 2 to a few thousand coordinates; through torch autograd one value-and-gradient is 10-40 tiny
// launches, and a second-order meta-step doubles that.
//
// Design.  One kernel template over (cluster size, value-and-gradient | Hessian-vector product); the family is a
// runtime switch.  Four kinds of family:
//   matrix (QUADRATIC, LASSO, BOWL, NORM, RASTRIGIN): r = A x - y.  A row-block GEMV: CTA k of the cluster owns rows
//     [r0, r1) of A.  Pass 1, a warp per row: the row dots A_i.x (and A_i.v) in fp64, a per-row weight w_i (r_i, or the norm's
//     a_i^(p-1) sign r_i, ...) and the row terms of f (sum r^2, sum a^p, ...) in fp64.  Pass 2, a thread per column:
//     the partial A^T w over the CTA's rows, fp64.  The partials go through distributed shared memory: after a cluster
//     barrier every CTA sums all CTAs' partials in rank order, then writes its own slice of the output.
//   data (PROJECTION_QUADRATIC, SUM_OF_QUADRATICS, OUTWARD_SNAKE): the objective only needs the column sums
//     sum_b A_bj^2 and sum_b A_bj of the data batch; the same row-block split and exchange.
//   elementwise (ISOTROPIC_QUADRATIC, DEPENDENCY_CHAIN, MIN_MAX_WELL) and the 2-D test functions: one CTA.
// Every sum has a fixed order (warp trees, per-warp slots, rank-ordered cluster sums): no atomics, so eager runs and
// graph replays give the same bits.  Element terms and the 2-D functions are formed in fp64.
#include <cooperative_groups.h>
#include <cuda_runtime.h>
#include <math.h>

#include "l2o_internal.h"

namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 512;
constexpr int kWarps = kThreads / 32;
constexpr int kCl = 8;                  // CTAs of the cluster for the large matrix and data problems
constexpr int64_t kClusterWork = 65536; // rows * n from which the cluster is used
constexpr double kPi = 3.14159265358979323846;

enum Kind { kMatrix, kData, kElement, kPlane };

__host__ __device__ inline int kind_of(int fam) {
  switch (fam) {
    case L2O_ZOO_QUADRATIC: case L2O_ZOO_LASSO: case L2O_ZOO_RASTRIGIN: case L2O_ZOO_BOWL: case L2O_ZOO_NORM:
      return kMatrix;
    case L2O_ZOO_PROJECTION_QUADRATIC: case L2O_ZOO_SUM_OF_QUADRATICS: case L2O_ZOO_OUTWARD_SNAKE:
      return kData;
    case L2O_ZOO_ISOTROPIC_QUADRATIC: case L2O_ZOO_DEPENDENCY_CHAIN: case L2O_ZOO_MIN_MAX_WELL:
      return kElement;
    default:
      return kPlane;
  }
}

// rows of A each CTA owns (matrix families keep a weight per owned row in shared memory)
__host__ __device__ inline int rows_per_cta(int rows, int cl) { return (rows + cl - 1) / cl; }

// bytes of dynamic shared memory: x, v [n] floats; the partial and the summed column sums [n] doubles (two each);
// the two row weights [rows_per_cta] floats of the matrix families
size_t smem_bytes(const l2o_zoo_args& a, int cl) {
  const int rb = kind_of(a.family) == kMatrix ? rows_per_cta(a.rows, cl) : 0;
  return 2 * sizeof(float) * (size_t)a.n + 4 * sizeof(double) * (size_t)a.n + 2 * sizeof(float) * (size_t)rb;
}

// sums K doubles over the CTA in a fixed order; every thread gets the totals.  red: kWarps * K + K doubles
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
    for (int w = 0; w < kWarps; ++w) t += red[w * K + tid];
    red[kWarps * K + tid] = t;
  }
  __syncthreads();
#pragma unroll
  for (int k = 0; k < K; ++k) v[k] = red[kWarps * K + k];
  __syncthreads();   // red is free again
}

__device__ __forceinline__ float sign_of(float v) { return v > 0.f ? 1.f : (v < 0.f ? -1.f : 0.f); }

// the 2-D test functions at (x, y): f, and g or H (vx, vy)
__device__ void plane(int fam, double x, double y, double vx, double vy, bool hvp, double& f, double& o0,
                      double& o1) {
  double gx = 0.0, gy = 0.0, hxx = 0.0, hxy = 0.0, hyy = 0.0;
  switch (fam) {
    case L2O_ZOO_ROSENBROCK: {
      const double u = y - x * x;
      f = (1.0 - x) * (1.0 - x) + 100.0 * u * u;
      gx = -2.0 * (1.0 - x) - 400.0 * x * u;
      gy = 200.0 * u;
      hxx = 2.0 - 400.0 * u + 800.0 * x * x;
      hxy = -400.0 * x;
      hyy = 200.0;
      break;
    }
    case L2O_ZOO_SADDLE:
      f = x * x - y * y;
      gx = 2.0 * x;
      gy = -2.0 * y;
      hxx = 2.0;
      hyy = -2.0;
      break;
    case L2O_ZOO_LOGSUMEXP: {
      const double e1 = exp(x + 3.0 * y - 0.1), e2 = exp(x - 3.0 * y - 0.1), e3 = exp(-x - 0.1);
      const double s = e1 + e2 + e3 + 1.0, sx = e1 + e2 - e3, sy = 3.0 * (e1 - e2);
      f = log(s);
      gx = sx / s;
      gy = sy / s;
      hxx = (e1 + e2 + e3) / s - gx * gx;
      hxy = sy / s - gx * gy;
      hyy = 9.0 * (e1 + e2) / s - gy * gy;
      break;
    }
    case L2O_ZOO_ACKLEY: {
      // sqrt at the origin: TensorFlow's sqrt' = 0.5 / 0 = inf times x = 0 gives NaN, and so does this order
      const double r = sqrt(0.5 * (x * x + y * y));
      const double er = exp(-0.2 * r), a1 = 4.0 * er, a2 = -0.8 * er;   // d/dr and d2/dr2 of -20 exp(-0.2 r)
      const double ca = cos(2.0 * kPi * x), cb = cos(2.0 * kPi * y);
      const double sa = sin(2.0 * kPi * x), sb = sin(2.0 * kPi * y);
      const double E = exp(0.5 * (ca + cb));
      f = -20.0 * er - E + exp(1.0) + 20.0;
      const double dr = a1 * (0.5 / r);     // d/dr times dr/d(x^2 + y^2) * 2
      gx = dr * x + kPi * E * sa;
      gy = dr * y + kPi * E * sb;
      const double rx = 0.5 * x / r, ry = 0.5 * y / r;
      const double r3 = 0.25 / (r * r * r);
      hxx = a2 * rx * rx + a1 * (0.5 / r - r3 * x * x) - kPi * kPi * E * sa * sa + 2.0 * kPi * kPi * E * ca;
      hyy = a2 * ry * ry + a1 * (0.5 / r - r3 * y * y) - kPi * kPi * E * sb * sb + 2.0 * kPi * kPi * E * cb;
      hxy = a2 * rx * ry - a1 * r3 * x * y - kPi * kPi * E * sa * sb;
      break;
    }
    case L2O_ZOO_BEALE: {
      const double y2 = y * y, y3 = y2 * y;
      const double t1 = 1.5 - x + x * y, t2 = 2.25 - x + x * y2, t3 = 2.625 - x + x * y3;
      const double ax = y - 1.0, ay = x, bx = y2 - 1.0, by = 2.0 * x * y, cx = y3 - 1.0, cy = 3.0 * x * y2;
      f = t1 * t1 + t2 * t2 + t3 * t3;
      gx = 2.0 * (t1 * ax + t2 * bx + t3 * cx);
      gy = 2.0 * (t1 * ay + t2 * by + t3 * cy);
      hxx = 2.0 * (ax * ax + bx * bx + cx * cx);
      hxy = 2.0 * (ax * ay + bx * by + cx * cy + t1 + t2 * 2.0 * y + t3 * 3.0 * y2);
      hyy = 2.0 * (ay * ay + by * by + cy * cy + t2 * 2.0 * x + t3 * 6.0 * x * y);
      break;
    }
    case L2O_ZOO_BOOTH: {
      const double a = x + 2.0 * y - 7.0, b = 2.0 * x + y - 5.0;
      f = a * a + b * b;
      gx = 2.0 * a + 4.0 * b;
      gy = 4.0 * a + 2.0 * b;
      hxx = 10.0;
      hxy = 8.0;
      hyy = 10.0;
      break;
    }
    case L2O_ZOO_STYBLINSKI_TANG:
      f = 0.5 * (x * x * x * x - 16.0 * x * x + 5.0 * x + y * y * y * y - 16.0 * y * y + 5.0 * y) + 80.0;
      gx = 0.5 * (4.0 * x * x * x - 32.0 * x + 5.0);
      gy = 0.5 * (4.0 * y * y * y - 32.0 * y + 5.0);
      hxx = 0.5 * (12.0 * x * x - 32.0);
      hyy = 0.5 * (12.0 * y * y - 32.0);
      break;
    case L2O_ZOO_MATYAS:
      f = 0.26 * (x * x + y * y) - 0.48 * x * y;
      gx = 0.52 * x - 0.48 * y;
      gy = 0.52 * y - 0.48 * x;
      hxx = 0.52;
      hxy = -0.48;
      hyy = 0.52;
      break;
    case L2O_ZOO_BRANIN: {
      const double b = 5.1 / (4.0 * kPi * kPi), c = 5.0 / kPi, r = 6.0, s = 10.0, t = 1.0 / (8.0 * kPi);
      const double u = y - b * x * x + c * x - r, du = -2.0 * b * x + c;
      f = u * u + s * (1.0 - t) * cos(x) + s;
      gx = 2.0 * u * du - s * (1.0 - t) * sin(x);
      gy = 2.0 * u;
      hxx = 2.0 * du * du - 4.0 * b * u - s * (1.0 - t) * cos(x);
      hxy = 2.0 * du;
      hyy = 2.0;
      break;
    }
    default: {   // MICHALEWICZ, m = 5: f = 2 - T(x, 1) - T(y, 2), T(z, k) = sin z sin(k z^2 / pi)^10
      double d1[2], d2[2], tv[2];
      const double zz[2] = {x, y};
#pragma unroll
      for (int q = 0; q < 2; ++q) {
        const double z = zz[q], k = (double)(q + 1), ph = k * z * z / kPi;
        const double S = sin(ph), Sd = cos(ph) * 2.0 * k * z / kPi;
        const double Sdd = -S * (2.0 * k * z / kPi) * (2.0 * k * z / kPi) + cos(ph) * 2.0 * k / kPi;
        const double S8 = pow(S, 8.0), S9 = S8 * S, S10 = S9 * S;
        tv[q] = sin(z) * S10;
        d1[q] = cos(z) * S10 + sin(z) * 10.0 * S9 * Sd;
        d2[q] = -sin(z) * S10 + 2.0 * cos(z) * 10.0 * S9 * Sd + sin(z) * (90.0 * S8 * Sd * Sd + 10.0 * S9 * Sdd);
      }
      f = 2.0 - (tv[0] + tv[1]);
      gx = -d1[0];
      gy = -d1[1];
      hxx = -d2[0];
      hyy = -d2[1];
      break;
    }
  }
  if (hvp) {
    o0 = hxx * vx + hxy * vy;
    o1 = hxy * vx + hyy * vy;
  } else {
    o0 = gx;
    o1 = gy;
  }
}

template <int CL, bool HVP>
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(kThreads) zoo_kernel(const l2o_zoo_args a) {
  extern __shared__ __align__(16) double smd[];
  __shared__ double part[2];                 // this CTA's row sums, read by every CTA of the cluster
  __shared__ double red[kWarps * 4 + 4];
  cg::cluster_group cl = cg::this_cluster();
  const int k = (int)cl.block_rank();
  const int n = a.n, fam = a.family, kind = kind_of(fam);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double* p1 = smd;            // [n] partial column sums of this CTA
  double* p2 = p1 + n;
  double* q1 = p2 + n;         // [n] the cluster's sums
  double* q2 = q1 + n;
  float* xs = reinterpret_cast<float*>(q2 + n);
  float* vs = xs + n;
  float* w1 = vs + n;          // [rb] the matrix families' row weights
  const int rows = (kind == kMatrix || kind == kData) ? a.rows : 0;
  const int rb = rows_per_cta(rows, CL);
  float* w2 = w1 + (kind == kMatrix ? rb : 0);
  const int r0 = min(rows, k * rb), r1 = min(rows, r0 + rb);
  const float p = a.p0;

  for (int j = tid; j < n; j += kThreads) {
    xs[j] = a.x[j];
    vs[j] = HVP ? a.v[j] : 0.f;
  }
  __syncthreads();

  // ---- row blocks: partial column sums and the row terms of f -------------------------------------------------------
  if (kind == kMatrix) {
    double s[2] = {0.0, 0.0};
    for (int i = r0 + warp; i < r1; i += kWarps) {
      const float* __restrict__ row = a.A + (size_t)i * n;
      double ax = 0.0, av = 0.0;
      for (int j = lane; j < n; j += 32) {
        const double u = (double)row[j];
        ax = fma(u, (double)xs[j], ax);
        if (HVP) av = fma(u, (double)vs[j], av);
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        ax += __shfl_xor_sync(0xffffffffu, ax, o);
        av += __shfl_xor_sync(0xffffffffu, av, o);
      }
      if (lane == 0) {
        const double r = fam == L2O_ZOO_BOWL ? ax : ax - (double)a.y[i];
        float u1 = (float)(HVP ? av : r), u2 = 0.f;
        if (fam == L2O_ZOO_NORM) {
          const double ab = fabs(r) + 1e-6;   // |diff| + EPSILON
          const double sg = r > 0.0 ? 1.0 : (r < 0.0 ? -1.0 : 0.0);
          const double w = pow(ab, (double)p - 1.0) * sg;
          u1 = (float)w;
          s[0] += pow(ab, (double)p);
          if (HVP) {
            u2 = (float)(pow(ab, (double)p - 2.0) * av);
            s[1] += w * av;
          }
        } else {
          s[0] += r * r;
          // tf.norm of the single-element rows: d|r| / dr = r / |r| is NaN at r = 0
          if (fam == L2O_ZOO_RASTRIGIN && r == 0.0) u1 = __int_as_float(0x7fc00000);
        }
        w1[i - r0] = u1;
        w2[i - r0] = u2;
      }
    }
    block_sum<2>(s, red);
    if (tid == 0) {
      part[0] = s[0];
      part[1] = s[1];
    }
    const bool two = HVP && fam == L2O_ZOO_NORM;
    for (int j = tid; j < n; j += kThreads) {
      double c1 = 0.0, c2 = 0.0;
      for (int i = r0; i < r1; ++i) {
        const double u = (double)a.A[(size_t)i * n + j];
        c1 = fma(u, (double)w1[i - r0], c1);
        if (two) c2 = fma(u, (double)w2[i - r0], c2);
      }
      p1[j] = c1;
      p2[j] = c2;
    }
  } else if (kind == kData) {
    for (int j = tid; j < n; j += kThreads) {
      double c1 = 0.0, c2 = 0.0;
      for (int i = r0; i < r1; ++i) {
        const double d = (double)a.A[(size_t)i * n + j];
        c1 = fma(d, d, c1);
        c2 += d;
      }
      p1[j] = c1;
      p2[j] = c2;
    }
  }
  cl.sync();   // every CTA's partials are written

  double S0 = 0.0, S1 = 0.0;
  if (kind == kMatrix || kind == kData) {
    for (int j = tid; j < n; j += kThreads) {
      double t1 = 0.0, t2 = 0.0;
      for (int q = 0; q < CL; ++q) {
        t1 += cl.map_shared_rank(p1, q)[j];
        t2 += cl.map_shared_rank(p2, q)[j];
      }
      q1[j] = t1;
      q2[j] = t2;
    }
    for (int q = 0; q < CL; ++q) {
      const double* pq = cl.map_shared_rank(part, q);
      S0 += pq[0];
      S1 += pq[1];
    }
  }
  cl.sync();   // no CTA leaves while another still reads its shared memory; q1, q2 complete

  // ---- the outputs --------------------------------------------------------------------------------------------------
  if (kind == kPlane) {
    if (tid == 0) {
      double f, o0, o1;
      plane(fam, (double)xs[0], (double)xs[1], (double)vs[0], (double)vs[1], HVP, f, o0, o1);
      a.out[0] = (float)o0;
      a.out[1] = (float)o1;
      if (!HVP && a.f) a.f[0] = (float)f;
    }
    return;
  }

  // global statistics over x (one CTA, or every CTA of the cluster alike)
  double st[2] = {0.0, 0.0};
  float mx = 0.f, mn = 0.f;
  int cmx = 0, cmn = 0;
  if (fam == L2O_ZOO_OUTWARD_SNAKE) {
    for (int j = tid; j < n; j += kThreads) {
      st[0] += (double)xs[j] * (double)xs[j];
      st[1] += (double)xs[j] * (double)vs[j];
    }
    block_sum<2>(st, red);
  } else if (fam == L2O_ZOO_MIN_MAX_WELL) {
    __shared__ float ext[2 * kWarps];
    __shared__ int cnt[2 * kWarps];
    mx = -INFINITY;
    mn = INFINITY;
    for (int j = tid; j < n; j += kThreads) {
      const float q = xs[j] * xs[j];
      mx = fmaxf(mx, q);
      mn = fminf(mn, q);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
      mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
    }
    if (lane == 0) {
      ext[warp] = mx;
      ext[kWarps + warp] = mn;
    }
    __syncthreads();
    for (int w = 0; w < kWarps; ++w) {
      mx = fmaxf(mx, ext[w]);
      mn = fminf(mn, ext[kWarps + w]);
    }
    int c0 = 0, c1 = 0;
    for (int j = tid; j < n; j += kThreads) {
      const float q = xs[j] * xs[j];
      c0 += q == mx;
      c1 += q == mn;
      if (q == mn) st[1] += (double)xs[j] * (double)vs[j];   // x.v over the minima
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      c0 += __shfl_xor_sync(0xffffffffu, c0, o);
      c1 += __shfl_xor_sync(0xffffffffu, c1, o);
    }
    if (lane == 0) {
      cnt[warp] = c0;
      cnt[kWarps + warp] = c1;
    }
    __syncthreads();
    for (int w = 0; w < kWarps; ++w) {
      cmx += cnt[w];
      cmn += cnt[kWarps + w];
    }
    block_sum<2>(st, red);
  }

  const int cb = (n + CL - 1) / CL, c0 = min(n, k * cb), c1 = min(n, c0 + cb);
  const double R = sqrt(st[0]), xv = st[1];
  const int nd = n - 1;   // DEPENDENCY_CHAIN's ndim
  auto qd = [&](int i) { return 1.0 / (double)(xs[i] * xs[i] + 1e-6f); };
  // f's element terms over all n (CTA 0 only), the outputs over this CTA's columns
  double fe[1] = {0.0};
  for (int j = (HVP || k != 0) ? c0 + tid : tid; j < ((HVP || k != 0) ? c1 : n); j += kThreads) {
    const double x = (double)xs[j], v = (double)vs[j];
    double o = 0.0, t = 0.0;
    switch (fam) {
      case L2O_ZOO_QUADRATIC: case L2O_ZOO_BOWL:
        o = q1[j];
        break;
      case L2O_ZOO_LASSO:
        o = HVP ? q1[j] : q1[j] + (double)p * (double)sign_of(xs[j]);
        t = (double)p * fabs(x);
        break;
      case L2O_ZOO_RASTRIGIN: {
        const double cj = (double)a.c[j], ph = 2.0 * kPi * x;
        o = HVP ? q1[j] / n + (double)p * 4.0 * kPi * kPi * cj * cos(ph) * v
                : q1[j] / n + (double)p * 2.0 * kPi * cj * sin(ph);
        t = -(double)p * cj * cos(ph);
        break;
      }
      case L2O_ZOO_NORM: {
        const double ip = 1.0 / (double)p;
        o = HVP ? (1.0 - p) * pow(S0, ip - 2.0) * S1 * q1[j] + (p - 1.0) * pow(S0, ip - 1.0) * q2[j]
                : pow(S0, ip - 1.0) * q1[j];
        break;
      }
      case L2O_ZOO_PROJECTION_QUADRATIC:
        o = 2.0 * q1[j] * (HVP ? v : x);
        t = q1[j] * x * x;
        break;
      case L2O_ZOO_SUM_OF_QUADRATICS:
        o = HVP ? 2.0 * rows * v : 2.0 * (rows * x - q2[j]);
        t = rows * x * x - 2.0 * x * q2[j];
        break;
      case L2O_ZOO_OUTWARD_SNAKE: {
        const double D0 = q2[0], re = R + 1e-6;
        const double h1 = -D0 / (re * re), h2 = 2.0 * D0 / (re * re * re);
        auto s_of = [&](int i) { return (double)xs[i] - kPi * cos((double)xs[i - 1]); };
        if (HVP) {
          auto jv = [&](int i) { return (double)vs[i] + kPi * sin((double)xs[i - 1]) * (double)vs[i - 1]; };
          o = (h2 / (R * R) - h1 / (R * R * R)) * xv * x + h1 / R * v;
          if (j >= 1) o += 2.0 * q1[j] * jv(j);
          if (j + 1 < n)
            o += 2.0 * q1[j + 1] * (jv(j + 1) * kPi * sin(x) + s_of(j + 1) * kPi * cos(x) * v);
        } else {
          o = h1 * (0.5 / R) * 2.0 * x;   // sqrt at |x| = 0: inf * 0 = NaN, as in TensorFlow
          if (j >= 1) o += 2.0 * q1[j] * s_of(j);
          if (j + 1 < n) o += 2.0 * q1[j + 1] * s_of(j + 1) * kPi * sin(x);
        }
        if (j >= 1) t = q1[j] * s_of(j) * s_of(j);
        if (j == 0) t = D0 / re;
        break;
      }
      case L2O_ZOO_ISOTROPIC_QUADRATIC:
        o = 2.0 * (HVP ? v : x);
        t = x * x;
        break;
      case L2O_ZOO_DEPENDENCY_CHAIN: {
        if (HVP) {
          if (j == 0) o = 2.0 * nd * v;
          if (j >= 1) {
            const double qp = qd(j - 1), xp = (double)xs[j - 1];
            o += 2.0 * qp * v - 4.0 * x * xp * qp * qp * (double)vs[j - 1];
          }
          if (j + 1 <= nd) {
            const double q = qd(j), xn = (double)xs[j + 1];
            o += -4.0 * xn * x * q * q * (double)vs[j + 1] + xn * xn * (8.0 * x * x * q * q * q - 2.0 * q * q) * v;
          }
        } else {
          if (j == 0) o = 2.0 * nd * x;
          if (j >= 1) o += 2.0 * x * qd(j - 1);
          if (j + 1 <= nd) {
            const double q = qd(j), xn = (double)xs[j + 1];
            o += -2.0 * xn * xn * x * q * q;
          }
        }
        t = j == 0 ? nd * x * x : x * x * qd(j - 1);
        break;
      }
      default: {   // MIN_MAX_WELL
        const float q = xs[j] * xs[j];
        const double m = (double)mn;
        if (q == mx) o += HVP ? 2.0 * v / cmx : 2.0 * x / cmx;
        if (q == mn)
          o += HVP ? 8.0 * x * xv / (m * m * m * (double)cmn * cmn) - 2.0 * v / (m * m * cmn)
                   : -2.0 * x / (m * m * cmn);
        break;
      }
    }
    if (j >= c0 && j < c1) a.out[j] = (float)o;
    fe[0] += t;
  }
  if (HVP || !a.f || k != 0) return;
  block_sum<1>(fe, red);
  if (tid == 0) {
    double f = fe[0];
    switch (fam) {
      case L2O_ZOO_QUADRATIC: case L2O_ZOO_BOWL: case L2O_ZOO_LASSO: f += 0.5 * S0; break;
      case L2O_ZOO_RASTRIGIN: f += 0.5 * S0 / n + (double)p * (double)n * (double)n; break;
      case L2O_ZOO_NORM: f = pow(S0, 1.0 / (double)p); break;
      case L2O_ZOO_SUM_OF_QUADRATICS: f += 1e-12; break;
      case L2O_ZOO_MIN_MAX_WELL: f = (double)mx + 1.0 / (double)mn - 2.0 + 1e-12; break;
      default: break;
    }
    a.f[0] = (float)f;
  }
}

int validate(const l2o_zoo_args* a, bool hvp) {
  if (!a || !a->x || !a->out || (hvp && !a->v)) return L2O_E_INVALID;
  if (a->family < 0 || a->family >= L2O_ZOO_NUM_FAMILIES || a->n < 1) return L2O_E_INVALID;
  const int fam = a->family, kind = kind_of(fam);
  if (kind == kMatrix) {
    if (!a->A) return L2O_E_INVALID;
    if (fam == L2O_ZOO_BOWL ? (a->n != 2 || a->rows != 2) : (a->rows != a->n || !a->y)) return L2O_E_INVALID;
    if (fam == L2O_ZOO_RASTRIGIN && !a->c) return L2O_E_INVALID;
    if (fam == L2O_ZOO_NORM && !(a->p0 > 0.f)) return L2O_E_INVALID;
  } else if (kind == kData) {
    if (!a->A || a->rows < 1) return L2O_E_INVALID;
    if (fam == L2O_ZOO_OUTWARD_SNAKE && a->n < 2) return L2O_E_INVALID;
  } else if (kind == kPlane) {
    if (a->n != 2) return L2O_E_INVALID;
  } else if (fam == L2O_ZOO_DEPENDENCY_CHAIN && a->n < 2) {
    return L2O_E_INVALID;
  }
  if (a->n > L2O_ZOO_MAX_N) return L2O_E_UNSUPPORTED;
  return L2O_OK;
}

template <bool HVP>
int launch(const l2o_zoo_args* a, void* stream, const char* fn) {
  if (int rc = validate(a, HVP)) return rc;
  const int kind = kind_of(a->family);
  const bool big = (kind == kMatrix || kind == kData) && (int64_t)a->rows * a->n >= kClusterWork;
  const int cl = big ? kCl : 1;
  const size_t smem = smem_bytes(*a, cl);
  const cudaStream_t st = (cudaStream_t)stream;
  if (big) {
    if (int rc = l2o::raise_smem_limit(fn, zoo_kernel<kCl, HVP>, smem)) return rc;
    zoo_kernel<kCl, HVP><<<kCl, kThreads, smem, st>>>(*a);
  } else {
    if (int rc = l2o::raise_smem_limit(fn, zoo_kernel<1, HVP>, smem)) return rc;
    zoo_kernel<1, HVP><<<1, kThreads, smem, st>>>(*a);
  }
  return l2o::after_launch(fn);
}

}  // namespace

extern "C" int l2o_zoo_value_grad(const l2o_zoo_args* a, void* stream) {
  return launch<false>(a, stream, "l2o_zoo_value_grad");
}

extern "C" int l2o_zoo_hvp(const l2o_zoo_args* a, void* stream) {
  return launch<true>(a, stream, "l2o_zoo_hvp");
}
