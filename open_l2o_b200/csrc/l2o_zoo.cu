// The analytic families of L2O-Scale's problem zoo (SC/problems/problem_generator.py; SC/ =
// Model_Free_L2O/L2O-Scale/L2O-Scale-Training/): f(x) with df/dx, H(x) v, or the Hessian form q = sum_k u_k^T H(x) v_k
// with its gradient dq/dx, at one parameter vector in ONE launch.
// The zoo's problems have 2 to a few thousand coordinates; through torch autograd one value-and-gradient is 10-40 tiny
// launches, and a second-order meta-step doubles that.
//
// Design.  One kernel template over (cluster size, mode: value-and-gradient | Hessian-vector product | Hessian form);
// the family is a runtime switch.  Four kinds of family:
//   matrix (QUADRATIC, LASSO, BOWL, NORM, RASTRIGIN): r = A x - y.  A row-block GEMV: CTA k of the cluster owns rows
//     [r0, r1) of A.  Pass 1, a warp per row: the row dots A_i.x (and A_i.v) in fp64, a per-row weight w_i (r_i, or the norm's
//     a_i^(p-1) sign r_i, ...) and the row terms of f (sum r^2, sum a^p, ...) in fp64.  Pass 2, a thread per column:
//     the partial A^T w over the CTA's rows, fp64.  The partials go through distributed shared memory: after a cluster
//     barrier every CTA sums all CTAs' partials in rank order, then writes its own slice of the output.
//     The Hessian form's pass 1 takes the 2k row dots A_i.u_k, A_i.v_k, streaming U and V from L2 (2 k n floats do
//     not fit next to x and the column sums in shared memory).  Only NORM has a non-constant A^T H A: its row weight
//     needs the cluster's sums over rows of w_i A_i.u_k, so NORM exchanges those, forms z = sum_k (Wv_k u_k + Wu_k v_k)
//     and takes one more row pass (A_i.z) before the single A^T w.
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
constexpr int kMaxPairs = L2O_ZOO_MAX_PAIRS;
constexpr int kRed = 2 * kMaxPairs + 2; // the Hessian form's per-CTA row sums: two scalars, then Wu_k, Wv_k
constexpr int kTile = 4;                // pairs whose row dots a warp accumulates at once

enum Kind { kMatrix, kData, kElement, kPlane };
enum Mode { kGrad, kHvp, kForm };

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
// the row weights [rows_per_cta] floats of the matrix families (two, three for the Hessian form)
size_t smem_bytes(const l2o_zoo_args& a, int cl, bool form) {
  const int rb = kind_of(a.family) == kMatrix ? rows_per_cta(a.rows, cl) : 0;
  return 2 * sizeof(float) * (size_t)a.n + 4 * sizeof(double) * (size_t)a.n + (form ? 3 : 2) * sizeof(float) * (size_t)rb;
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

// the 2-D test functions at (x, y): f, the gradient g, the Hessian h = (xx, xy, yy) and the third derivatives
// t = (xxx, xxy, xyy, yyy)
__device__ void plane(int fam, double x, double y, double& f, double (&g)[2], double (&h)[3], double (&t)[4]) {
  double gx = 0.0, gy = 0.0, hxx = 0.0, hxy = 0.0, hyy = 0.0;
  t[0] = t[1] = t[2] = t[3] = 0.0;
  switch (fam) {
    case L2O_ZOO_ROSENBROCK: {
      const double u = y - x * x;
      f = (1.0 - x) * (1.0 - x) + 100.0 * u * u;
      gx = -2.0 * (1.0 - x) - 400.0 * x * u;
      gy = 200.0 * u;
      hxx = 2.0 - 400.0 * u + 800.0 * x * x;
      hxy = -400.0 * x;
      hyy = 200.0;
      t[0] = 2400.0 * x;
      t[1] = -400.0;
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
      // the third central moment of the exponents' slopes under the softmax weights (the constant 1 has slope 0)
      const double pw[4] = {e1 / s, e2 / s, e3 / s, 1.0 / s};
      const double sl[4][2] = {{1.0, 3.0}, {1.0, -3.0}, {-1.0, 0.0}, {0.0, 0.0}};
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const double dx = sl[i][0] - gx, dy = sl[i][1] - gy;
        t[0] += pw[i] * dx * dx * dx;
        t[1] += pw[i] * dx * dx * dy;
        t[2] += pw[i] * dx * dy * dy;
        t[3] += pw[i] * dy * dy * dy;
      }
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
      // the radial term as P(x^2 + y^2): d3 = 8 P3 z_a z_b z_c + 4 P2 (d_ab z_c + d_ac z_b + d_bc z_a), with
      // P2, P3 its second and third derivatives; -E = -exp(e(x) + e(y)) with e's derivatives ps, ps1, ps2 (y: ch ..)
      const double a3 = 0.16 * er, r2 = r * r;
      const double P2 = (a2 / r2 - a1 / (r2 * r)) / 16.0;
      const double P3 = (a3 / (r2 * r) - 3.0 * a2 / (r2 * r2) + 3.0 * a1 / (r2 * r2 * r)) / 64.0;
      const double ps = -kPi * sa, ps1 = -2.0 * kPi * kPi * ca, ps2 = 4.0 * kPi * kPi * kPi * sa;
      const double ch = -kPi * sb, ch1 = -2.0 * kPi * kPi * cb, ch2 = 4.0 * kPi * kPi * kPi * sb;
      t[0] = 8.0 * P3 * x * x * x + 12.0 * P2 * x - (ps2 + 3.0 * ps * ps1 + ps * ps * ps) * E;
      t[1] = 8.0 * P3 * x * x * y + 4.0 * P2 * y - (ps1 + ps * ps) * ch * E;
      t[2] = 8.0 * P3 * x * y * y + 4.0 * P2 * x - ps * (ch1 + ch * ch) * E;
      t[3] = 8.0 * P3 * y * y * y + 12.0 * P2 * y - (ch2 + 3.0 * ch * ch1 + ch * ch * ch) * E;
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
      // f = sum_i s_i^2, s_i = c_i - x + x y^i: d3 f = 2 sum_i (s_bc s_a + s_b s_ac + s_c s_ab + s s_abc), s_xx = 0
      const double s[3] = {t1, t2, t3}, sx[3] = {ax, bx, cx}, sy[3] = {ay, by, cy};
      const double sxy[3] = {1.0, 2.0 * y, 3.0 * y2}, syy[3] = {0.0, 2.0 * x, 6.0 * x * y};
      const double sxyy[3] = {0.0, 2.0, 6.0 * y}, syyy[3] = {0.0, 0.0, 6.0 * x};
#pragma unroll
      for (int i = 0; i < 3; ++i) {
        t[1] += 4.0 * sx[i] * sxy[i];
        t[2] += 2.0 * (syy[i] * sx[i] + 2.0 * sy[i] * sxy[i] + s[i] * sxyy[i]);
        t[3] += 2.0 * (3.0 * syy[i] * sy[i] + s[i] * syyy[i]);
      }
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
      t[0] = 12.0 * x;
      t[3] = 12.0 * y;
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
      const double b = 5.1 / (4.0 * kPi * kPi), c = 5.0 / kPi, r = 6.0, s = 10.0, tt = 1.0 / (8.0 * kPi);
      const double u = y - b * x * x + c * x - r, du = -2.0 * b * x + c;
      f = u * u + s * (1.0 - tt) * cos(x) + s;
      gx = 2.0 * u * du - s * (1.0 - tt) * sin(x);
      gy = 2.0 * u;
      hxx = 2.0 * du * du - 4.0 * b * u - s * (1.0 - tt) * cos(x);
      hxy = 2.0 * du;
      hyy = 2.0;
      t[0] = -12.0 * b * du + s * (1.0 - tt) * sin(x);
      t[1] = -4.0 * b;
      break;
    }
    default: {   // MICHALEWICZ, m = 5: f = 2 - T(x, 1) - T(y, 2), T(z, k) = sin z sin(k z^2 / pi)^10
      double d1[2], d2[2], d3[2], tv[2];
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
        // the third derivative of sin z B, B = S^10: -cos z B - 3 sin z B1 + 3 cos z B2 + sin z B3 (Bi = B's i-th)
        const double p1 = 2.0 * k * z / kPi, p2 = 2.0 * k / kPi, S7 = pow(S, 7.0);
        const double Sddd = -cos(ph) * p1 * p1 * p1 - 3.0 * S * p1 * p2;
        const double B1 = 10.0 * S9 * Sd, B2 = 90.0 * S8 * Sd * Sd + 10.0 * S9 * Sdd;
        const double B3 = 720.0 * S7 * Sd * Sd * Sd + 270.0 * S8 * Sd * Sdd + 10.0 * S9 * Sddd;
        d3[q] = -cos(z) * S10 - 3.0 * sin(z) * B1 + 3.0 * cos(z) * B2 + sin(z) * B3;
      }
      f = 2.0 - (tv[0] + tv[1]);
      gx = -d1[0];
      gy = -d1[1];
      hxx = -d2[0];
      hyy = -d2[1];
      t[0] = -d3[0];
      t[3] = -d3[1];
      break;
    }
  }
  g[0] = gx;
  g[1] = gy;
  h[0] = hxx;
  h[1] = hxy;
  h[2] = hyy;
}

// sum_k u_k[i] v_k[i] of the Hessian form's pairs (U, V [K][n], streamed from L2)
__device__ __forceinline__ double pair_dot(const l2o_zoo_form_args& fa, int i) {
  const int n = fa.base.n;
  double s = 0.0;
  for (int q = 0; q < fa.k; ++q) s = fma((double)__ldg(fa.U + (size_t)q * n + i), (double)__ldg(fa.V + (size_t)q * n + i), s);
  return s;
}

template <int CL, int MODE>
__global__ void __cluster_dims__(CL, 1, 1) __launch_bounds__(kThreads) zoo_kernel(const l2o_zoo_form_args fa) {
  constexpr bool HVP = MODE == kHvp, FORM = MODE == kForm;
  const l2o_zoo_args& a = fa.base;
  extern __shared__ __align__(16) double smd[];
  __shared__ double part[FORM ? kRed : 2];   // this CTA's row sums, read by every CTA of the cluster
  __shared__ double red[FORM ? kWarps * kRed + kRed : kWarps * 4 + 4];
  cg::cluster_group cl = cg::this_cluster();
  const int k = (int)cl.block_rank();
  const int n = a.n, fam = a.family, kind = kind_of(fam);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  double* p1 = smd;            // [n] partial column sums of this CTA
  double* p2 = p1 + n;
  double* q1 = p2 + n;         // [n] the cluster's sums
  double* q2 = q1 + n;
  float* xs = reinterpret_cast<float*>(q2 + n);
  float* vs = xs + n;          // v; the Hessian form's NORM keeps z here
  float* w1 = vs + n;          // [rb] the matrix families' row weights
  const int rows = (kind == kMatrix || kind == kData) ? a.rows : 0;
  const int rb = rows_per_cta(rows, CL);
  float* w2 = w1 + (kind == kMatrix ? rb : 0);
  float* w3 = w2 + (kind == kMatrix ? rb : 0);   // the Hessian form's third row weight
  const int r0 = min(rows, k * rb), r1 = min(rows, r0 + rb);
  const float p = a.p0;
  const int K = FORM ? fa.k : 0;
  const bool same = fa.U == fa.V;

  for (int j = tid; j < n; j += kThreads) {
    xs[j] = a.x[j];
    vs[j] = HVP ? a.v[j] : 0.f;
  }
  __syncthreads();

  // ---- row blocks: partial column sums and the row terms of f -------------------------------------------------------
  if (FORM && kind == kMatrix) {
    // pass 1: du_k = A_i.u_k, dv_k = A_i.v_k; q's row term P_i = sum_k du_k dv_k (NORM: the per-CTA sums S, B.P and
    // Wu_k = sum_i w_i du_k, Wv_k in this warp's slots of red, the row weights w, b, c P)
    const bool norm = fam == L2O_ZOO_NORM;
    for (int t = tid; t < kWarps * kRed; t += kThreads) red[t] = 0.0;
    __syncthreads();
    double s[2] = {0.0, 0.0};
    for (int i = r0 + warp; i < r1; i += kWarps) {
      const float* __restrict__ row = a.A + (size_t)i * n;
      double w = 0.0, b = 0.0, c = 0.0, P = 0.0;
      // the pairs in tiles of kTile (the row is re-read from L1 / L2 per tile): fewer live accumulators
      for (int q0 = 0; q0 < K; q0 += kTile) {
        double ax = 0.0, du[kTile], dv[kTile];
#pragma unroll
        for (int q = 0; q < kTile; ++q) du[q] = dv[q] = 0.0;
        for (int j = lane; j < n; j += 32) {
          const double u = (double)row[j];
          if (norm && q0 == 0) ax = fma(u, (double)xs[j], ax);
#pragma unroll
          for (int q = 0; q < kTile; ++q) {
            if (q0 + q < K) {
              du[q] = fma(u, (double)__ldg(fa.U + (size_t)(q0 + q) * n + j), du[q]);
              if (!same) dv[q] = fma(u, (double)__ldg(fa.V + (size_t)(q0 + q) * n + j), dv[q]);
            }
          }
        }
#pragma unroll
        for (int q = 0; q < kTile; ++q) {
          if (q0 + q < K) {
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
              du[q] += __shfl_xor_sync(0xffffffffu, du[q], o);
              if (!same) dv[q] += __shfl_xor_sync(0xffffffffu, dv[q], o);
            }
            if (same) dv[q] = du[q];
            P = fma(du[q], dv[q], P);
          }
        }
        if (!norm) continue;
        if (q0 == 0) {
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) ax += __shfl_xor_sync(0xffffffffu, ax, o);
          const double r = ax - (double)a.y[i];
          const double ab = fabs(r) + 1e-6;   // |diff| + EPSILON
          const double sg = r > 0.0 ? 1.0 : (r < 0.0 ? -1.0 : 0.0);
          w = pow(ab, (double)p - 1.0) * sg;
          b = pow(ab, (double)p - 2.0);
          c = pow(ab, (double)p - 3.0) * sg;
          s[0] += pow(ab, (double)p);
        }
        if (lane == 0) {
#pragma unroll
          for (int q = 0; q < kTile; ++q) {
            if (q0 + q < K) {
              red[warp * kRed + 2 + q0 + q] += w * du[q];
              red[warp * kRed + 2 + kMaxPairs + q0 + q] += w * dv[q];
            }
          }
        }
      }
      if (!norm) {
        s[0] += P;   // lane 0's copy is the one summed
      } else if (lane == 0) {
        s[1] += b * P;
        w1[i - r0] = (float)w;
        w2[i - r0] = (float)b;
        w3[i - r0] = (float)(c * P);
      }
    }
    if (lane == 0) {
      red[warp * kRed] = s[0];
      red[warp * kRed + 1] = s[1];
    }
    __syncthreads();
    if (tid < kRed) {
      double t = 0.0;
      for (int w = 0; w < kWarps; ++w) t += red[w * kRed + tid];
      part[tid] = t;
    }
    cl.sync();   // every CTA's row sums are written
    if (tid < kRed) {
      double t = 0.0;
      for (int q = 0; q < CL; ++q) t += cl.map_shared_rank(part, q)[tid];
      red[tid] = t;   // red[0..kRed): the cluster's S (or sum P), B.P, Wu_k, Wv_k
    }
    __syncthreads();
    if (norm) {
      // d q / d r_i = al w_i + ga b_i A_i.z + de c_i P_i, z = sum_k (Wv_k u_k + Wu_k v_k)
      const double S = red[0], BP = red[1], ip = 1.0 / (double)p, pd = (double)p;
      double ww = 0.0;
      for (int q = 0; q < K; ++q) ww += red[2 + q] * red[2 + kMaxPairs + q];
      const double al = (1.0 - pd) * (1.0 - 2.0 * pd) * pow(S, ip - 3.0) * ww
                        - (pd - 1.0) * (pd - 1.0) * pow(S, ip - 2.0) * BP;
      const double ga = -(pd - 1.0) * (pd - 1.0) * pow(S, ip - 2.0), de = (pd - 1.0) * (pd - 2.0) * pow(S, ip - 1.0);
      for (int j = tid; j < n; j += kThreads) {
        double z = 0.0;
        for (int q = 0; q < K; ++q)
          z += red[2 + kMaxPairs + q] * (double)__ldg(fa.U + (size_t)q * n + j)
               + red[2 + q] * (double)__ldg(fa.V + (size_t)q * n + j);
        vs[j] = (float)z;
      }
      __syncthreads();
      for (int i = r0 + warp; i < r1; i += kWarps) {
        const float* __restrict__ row = a.A + (size_t)i * n;
        double az = 0.0;
        for (int j = lane; j < n; j += 32) az = fma((double)row[j], (double)vs[j], az);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) az += __shfl_xor_sync(0xffffffffu, az, o);
        if (lane == 0)
          w1[i - r0] = (float)(al * (double)w1[i - r0] + ga * (double)w2[i - r0] * az + de * (double)w3[i - r0]);
      }
      __syncthreads();
    }
  } else if (kind == kMatrix) {
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
  }
  // the column pass A^T w (the Hessian form: NORM only; the other matrix families have a constant A^T H A)
  if (kind == kMatrix && (!FORM || fam == L2O_ZOO_NORM)) {
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

  const bool cols = kind == kData || (kind == kMatrix && (!FORM || fam == L2O_ZOO_NORM));
  // the Hessian form's scalars, in shared memory to keep them out of the element loop's registers: sum_k Wu_k Wv_k
  // (NORM) or the radial q (OUTWARD_SNAKE); XX, UV, UM (OUTWARD_SNAKE, MIN_MAX_WELL, below)
  __shared__ double fs[FORM ? 4 : 1];
  double S0 = 0.0, S1 = 0.0;
  if (cols) {
    for (int j = tid; j < n; j += kThreads) {
      double t1 = 0.0, t2 = 0.0;
      for (int q = 0; q < CL; ++q) {
        t1 += cl.map_shared_rank(p1, q)[j];
        t2 += cl.map_shared_rank(p2, q)[j];
      }
      q1[j] = t1;
      q2[j] = t2;
    }
  }
  if (kind == kMatrix) {
    if (FORM) {
      S0 = red[0];
      S1 = red[1];
      if (tid == 0) {
        double ww = 0.0;
        for (int q = 0; q < K; ++q) ww += red[2 + q] * red[2 + kMaxPairs + q];
        fs[0] = ww;
      }
    } else {
      for (int q = 0; q < CL; ++q) {
        const double* pq = cl.map_shared_rank(part, q);
        S0 += pq[0];
        S1 += pq[1];
      }
    }
  }
  cl.sync();   // no CTA leaves while another still reads its shared memory; q1, q2 complete

  // ---- the outputs --------------------------------------------------------------------------------------------------
  if (kind == kPlane) {
    if (tid == 0) {
      double f, g[2], h[3], t3[4];
      plane(fam, (double)xs[0], (double)xs[1], f, g, h, t3);
      if (FORM) {
        double q = 0.0, o0 = 0.0, o1 = 0.0;
        for (int i = 0; i < K; ++i) {
          const double u0 = fa.U[2 * i], u1 = fa.U[2 * i + 1], v0 = fa.V[2 * i], v1 = fa.V[2 * i + 1];
          const double mxx = u0 * v0, mxy = u0 * v1 + u1 * v0, myy = u1 * v1;
          q += h[0] * mxx + h[1] * mxy + h[2] * myy;
          o0 += t3[0] * mxx + t3[1] * mxy + t3[2] * myy;
          o1 += t3[1] * mxx + t3[2] * mxy + t3[3] * myy;
        }
        a.out[0] = (float)o0;
        a.out[1] = (float)o1;
        if (fa.q) fa.q[0] = (float)q;
      } else {
        const double vx = (double)vs[0], vy = (double)vs[1];
        a.out[0] = (float)(HVP ? h[0] * vx + h[1] * vy : g[0]);
        a.out[1] = (float)(HVP ? h[1] * vx + h[2] * vy : g[1]);
        if (!HVP && a.f) a.f[0] = (float)f;
      }
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

  // the Hessian form's pair statistics over x: xu_k = x.u_k, xv_k = x.v_k (over the minima for MIN_MAX_WELL, all of
  // x for OUTWARD_SNAKE) in gk; XX = sum_k xu_k xv_k, UV = sum_k u_k.v_k over the same set, UM over the maxima
  __shared__ double gk[FORM ? 2 * kMaxPairs : 1];
  if (FORM && (fam == L2O_ZOO_OUTWARD_SNAKE || fam == L2O_ZOO_MIN_MAX_WELL)) {
    const bool mmw = fam == L2O_ZOO_MIN_MAX_WELL;
    double XX = 0.0, UV = 0.0, UM = 0.0;
    for (int q = 0; q < K; ++q) {
      double v4[4] = {0.0, 0.0, 0.0, 0.0};
      for (int j = tid; j < n; j += kThreads) {
        const float sq = xs[j] * xs[j];
        const double x = (double)xs[j], u = (double)fa.U[(size_t)q * n + j], v = (double)fa.V[(size_t)q * n + j];
        if (!mmw || sq == mn) {
          v4[0] += x * u;
          v4[1] += x * v;
          v4[2] += u * v;
        }
        if (mmw && sq == mx) v4[3] += u * v;
      }
      block_sum<4>(v4, red);
      if (tid == 0) {
        gk[q] = v4[0];
        gk[kMaxPairs + q] = v4[1];
      }
      XX += v4[0] * v4[1];
      UV += v4[2];
      UM += v4[3];
    }
    if (tid == 0) {
      fs[1] = XX;
      fs[2] = UV;
      fs[3] = UM;
      if (!mmw) {   // OUTWARD_SNAKE's radial part of q, A (x.u)(x.v) + B u.v (see the element loop)
        const double R = sqrt(st[0]), D0 = q2[0], re = R + 1e-6, h1 = -D0 / (re * re), h2 = 2.0 * D0 / (re * re * re);
        fs[0] = (h2 / (R * R) - h1 / (R * R * R)) * XX + h1 / R * UV;
      }
    }
    __syncthreads();
  }
  auto pair_x = [&](int j) {   // sum_k (xv_k u_k[j] + xu_k v_k[j])
    double s = 0.0;
    for (int q = 0; q < K; ++q)
      s += gk[kMaxPairs + q] * (double)fa.U[(size_t)q * n + j] + gk[q] * (double)fa.V[(size_t)q * n + j];
    return s;
  };

  const int cb = (n + CL - 1) / CL, c0 = min(n, k * cb), c1 = min(n, c0 + cb);
  const double R = sqrt(st[0]), xv = st[1];
  const int nd = n - 1;   // DEPENDENCY_CHAIN's ndim
  auto qd = [&](int i) { return 1.0 / (double)(xs[i] * xs[i] + 1e-6f); };
  // f's (or q's) element terms over all n (CTA 0 only), the outputs over this CTA's columns
  double fe[1] = {0.0};
  for (int j = (HVP || k != 0) ? c0 + tid : tid; j < ((HVP || k != 0) ? c1 : n); j += kThreads) {
    const double x = (double)xs[j], v = (double)vs[j];
    double o = 0.0, t = 0.0;
    switch (fam) {
      case L2O_ZOO_QUADRATIC: case L2O_ZOO_BOWL:
        o = FORM ? 0.0 : q1[j];
        break;
      case L2O_ZOO_LASSO:
        if (FORM) break;
        o = HVP ? q1[j] : q1[j] + (double)p * (double)sign_of(xs[j]);
        t = (double)p * fabs(x);
        break;
      case L2O_ZOO_RASTRIGIN: {
        const double cj = (double)a.c[j], ph = 2.0 * kPi * x;
        if (FORM) {
          const double P = pair_dot(fa, j);
          o = -(double)p * 8.0 * kPi * kPi * kPi * cj * sin(ph) * P;
          t = (double)p * 4.0 * kPi * kPi * cj * cos(ph) * P;
          break;
        }
        o = HVP ? q1[j] / n + (double)p * 4.0 * kPi * kPi * cj * cos(ph) * v
                : q1[j] / n + (double)p * 2.0 * kPi * cj * sin(ph);
        t = -(double)p * cj * cos(ph);
        break;
      }
      case L2O_ZOO_NORM: {
        if (FORM) {
          o = q1[j];
          break;
        }
        const double ip = 1.0 / (double)p;
        o = HVP ? (1.0 - p) * pow(S0, ip - 2.0) * S1 * q1[j] + (p - 1.0) * pow(S0, ip - 1.0) * q2[j]
                : pow(S0, ip - 1.0) * q1[j];
        break;
      }
      case L2O_ZOO_PROJECTION_QUADRATIC:
        if (FORM) {
          t = 2.0 * q1[j] * pair_dot(fa, j);
          break;
        }
        o = 2.0 * q1[j] * (HVP ? v : x);
        t = q1[j] * x * x;
        break;
      case L2O_ZOO_SUM_OF_QUADRATICS:
        if (FORM) {
          t = 2.0 * rows * pair_dot(fa, j);
          break;
        }
        o = HVP ? 2.0 * rows * v : 2.0 * (rows * x - q2[j]);
        t = rows * x * x - 2.0 * x * q2[j];
        break;
      case L2O_ZOO_OUTWARD_SNAKE: {
        const double D0 = q2[0], re = R + 1e-6;
        const double h1 = -D0 / (re * re), h2 = 2.0 * D0 / (re * re * re);
        auto s_of = [&](int i) { return (double)xs[i] - kPi * cos((double)xs[i - 1]); };
        if (FORM) {
          // radial D0 / (R + 1e-6): u^T H v = A (x.u)(x.v) + B u.v, A = h2 / R^2 - h1 / R^3, B = h1 / R
          const double h3 = -6.0 * D0 / (re * re * re * re), R2 = R * R;
          const double Ar = h2 / R2 - h1 / (R2 * R);
          const double dA = h3 / R2 - 3.0 * h2 / (R2 * R) + 3.0 * h1 / (R2 * R2), dB = h2 / R - h1 / R2;
          o = (dA * fs[1] + dB * fs[2]) / R * x + Ar * pair_x(j);
          // chain terms Q_i s_i^2, s_i = x_i - pi cos x_(i-1), Ju_i = u_i + pi sin(x_(i-1)) u_(i-1)
          auto chain = [&](int i, double& JJ, double& M) {   // sum_k Ju Jv and sum_k (u_(i-1) Jv_i + v_(i-1) Ju_i)
            const double sp = kPi * sin((double)xs[i - 1]);
            JJ = M = 0.0;
            for (int q = 0; q < K; ++q) {
              const float* u = fa.U + (size_t)q * n;
              const float* w = fa.V + (size_t)q * n;
              const double ju = (double)u[i] + sp * (double)u[i - 1], jv = (double)w[i] + sp * (double)w[i - 1];
              JJ += ju * jv;
              M += (double)u[i - 1] * jv + (double)w[i - 1] * ju;
            }
          };
          const double Pj = pair_dot(fa, j);
          double JJ, M;
          if (j >= 1) {
            const double cp = kPi * cos((double)xs[j - 1]), Pp = pair_dot(fa, j - 1);
            chain(j, JJ, M);
            o += 2.0 * q1[j] * cp * Pp;
            t = 2.0 * q1[j] * (JJ + s_of(j) * cp * Pp);
          }
          if (j + 1 < n) {
            chain(j + 1, JJ, M);
            const double cp = kPi * cos(x), sp = kPi * sin(x);
            o += 2.0 * q1[j + 1] * (cp * M + sp * cp * Pj - s_of(j + 1) * sp * Pj);
          }
          break;
        }
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
        if (FORM) {
          t = 2.0 * pair_dot(fa, j);
          break;
        }
        o = 2.0 * (HVP ? v : x);
        t = x * x;
        break;
      case L2O_ZOO_DEPENDENCY_CHAIN: {
        if (FORM) {
          // term i: a^2 phi(b), a = x_i, b = x_(i-1), phi = 1 / (b^2 + 1e-6) and its derivatives ph1 .. ph3;
          // C_i = sum_k (u_i v_(i-1) + u_(i-1) v_i)
          auto cross = [&](int i) {
            double s = 0.0;
            for (int q = 0; q < K; ++q) {
              const float* u = fa.U + (size_t)q * n;
              const float* w = fa.V + (size_t)q * n;
              s += (double)u[i] * (double)w[i - 1] + (double)u[i - 1] * (double)w[i];
            }
            return s;
          };
          auto phis = [&](int m, double& ph, double& ph1, double& ph2, double& ph3) {
            const double b = (double)xs[m], Q = qd(m);
            ph = Q;
            ph1 = -2.0 * b * Q * Q;
            ph2 = -2.0 * Q * Q + 8.0 * b * b * Q * Q * Q;
            ph3 = 24.0 * b * Q * Q * Q - 48.0 * b * b * b * Q * Q * Q * Q;
          };
          const double Pj = pair_dot(fa, j);
          double ph, ph1, ph2, ph3;
          if (j == 0) t = 2.0 * nd * Pj;
          if (j >= 1) {
            phis(j - 1, ph, ph1, ph2, ph3);
            const double C = cross(j), Pp = pair_dot(fa, j - 1);
            o += 2.0 * ph1 * C + 2.0 * x * ph2 * Pp;
            t += 2.0 * ph * Pj + 2.0 * x * ph1 * C + x * x * ph2 * Pp;
          }
          if (j + 1 <= nd) {
            phis(j, ph, ph1, ph2, ph3);
            const double an = (double)xs[j + 1];
            o += 2.0 * ph1 * pair_dot(fa, j + 1) + 2.0 * an * ph2 * cross(j + 1) + an * an * ph3 * Pj;
          }
          break;
        }
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
        if (FORM) {   // max x^2 has a constant Hessian; 1 / m with m the tie-averaged minimum
          if (q == mn) {
            const double c = (double)cmn;
            o = -48.0 * x * fs[1] / (m * m * m * m * c * c * c) + 8.0 * pair_x(j) / (m * m * m * c * c)
                + 8.0 * x * fs[2] / (m * m * m * c * c);
          }
          break;
        }
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
  if (FORM) {
    if (!fa.q || k != 0) return;
    block_sum<1>(fe, red);
    if (tid == 0) {
      double q = fe[0];
      switch (fam) {
        case L2O_ZOO_QUADRATIC: case L2O_ZOO_BOWL: case L2O_ZOO_LASSO: q += S0; break;
        case L2O_ZOO_RASTRIGIN: q += S0 / n; break;
        case L2O_ZOO_NORM: {
          const double pd = (double)p, ip = 1.0 / pd;
          q = (1.0 - pd) * pow(S0, ip - 2.0) * fs[0] + (pd - 1.0) * pow(S0, ip - 1.0) * S1;
          break;
        }
        case L2O_ZOO_OUTWARD_SNAKE: q += fs[0]; break;
        case L2O_ZOO_MIN_MAX_WELL: {
          const double m = (double)mn, c = (double)cmn;
          q = 2.0 * fs[3] / cmx + 8.0 * fs[1] / (m * m * m * c * c) - 2.0 * fs[2] / (m * m * c);
          break;
        }
        default: break;
      }
      fa.q[0] = (float)q;
    }
    return;
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

template <int MODE>
int launch(const l2o_zoo_form_args& fa, void* stream, const char* fn) {
  const l2o_zoo_args* a = &fa.base;
  const int kind = kind_of(a->family);
  const bool big = (kind == kMatrix || kind == kData) && (int64_t)a->rows * a->n >= kClusterWork;
  const int cl = big ? kCl : 1;
  const size_t smem = smem_bytes(*a, cl, MODE == kForm);
  const cudaStream_t st = (cudaStream_t)stream;
  if (big) {
    if (int rc = l2o::raise_smem_limit(fn, zoo_kernel<kCl, MODE>, smem)) return rc;
    zoo_kernel<kCl, MODE><<<kCl, kThreads, smem, st>>>(fa);
  } else {
    if (int rc = l2o::raise_smem_limit(fn, zoo_kernel<1, MODE>, smem)) return rc;
    zoo_kernel<1, MODE><<<1, kThreads, smem, st>>>(fa);
  }
  return l2o::after_launch(fn);
}

template <int MODE>
int launch_plain(const l2o_zoo_args* a, void* stream, const char* fn) {
  if (int rc = validate(a, MODE == kHvp)) return rc;
  l2o_zoo_form_args fa = {};
  fa.base = *a;
  return launch<MODE>(fa, stream, fn);
}

}  // namespace

extern "C" int l2o_zoo_value_grad(const l2o_zoo_args* a, void* stream) {
  return launch_plain<kGrad>(a, stream, "l2o_zoo_value_grad");
}

extern "C" int l2o_zoo_hvp(const l2o_zoo_args* a, void* stream) {
  return launch_plain<kHvp>(a, stream, "l2o_zoo_hvp");
}

extern "C" int l2o_zoo_hess_form(const l2o_zoo_form_args* a, void* stream) {
  if (!a || !a->U || !a->V || a->k < 1) return L2O_E_INVALID;
  if (int rc = validate(&a->base, false)) return rc;
  if (a->k > L2O_ZOO_MAX_PAIRS) return L2O_E_UNSUPPORTED;
  return launch<kForm>(*a, stream, "l2o_zoo_hess_form");
}
