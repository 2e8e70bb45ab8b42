// L2O-Minimax's Twin-L2O (include/l2o_b200.h, l2o_minimax_*): the min/max LSTM optimizer pair unrolled over a
// batch of saddle-point problems.
//
// Mapping.  Both nets' weights are L2-streamed, not held in shared memory: one net is 12 H^2 + 25 H + 1 floats
// (315 KB at H = 80, 788 KB at H = 128), so the pair never fits a CTA, and a cluster slicing them would leave half of
// it idle on every iteration (only one net runs per iteration).  The pair (<= 1.6 MB) stays resident in the 50 MB L2.
// A CTA owns whole problems (a loss-4 gradient couples a problem's dim rows), up to kCap rows, and runs every
// iteration of the launch for them: each weight it reads from L2 serves all its rows.  Gate unit j of a layer is
// thread j, reading the transposed image row by row (coalesced) and accumulating one sum per row.
//
// Backward.  mm_chain_kernel walks [t0, t1) in reverse for a few rows per CTA in fp64, recomputing each iteration's
// cells from the forward's checkpoint, and writes the gate adjoints and the layer inputs of every (iteration, row).
// mm_dw_kernel then forms each weight gradient as a tiled product over (iteration, row) in a fixed order: one owner
// per output, no atomics, so the result is bit-identical run to run.
#include <math.h>

#include <algorithm>

#include "l2o_internal.h"

namespace l2o {
namespace minimax {

constexpr int kBwdRows = 4;   // rows per CTA of the backward chain
constexpr int kTile = 32;     // weight-gradient output tile (kTile x kTile), items staged kTile at a time
constexpr double kPi = 3.14159265358979323846;

// torch-layout offsets inside one net's theta
struct Off {
  int64_t wih1, whh1, bih1, bhh1, wih2, whh2, bih2, bhh2, wout, bout, total;
  __host__ __device__ explicit Off(int H) {
    const int64_t G = 4 * (int64_t)H;
    wih1 = 0;
    whh1 = wih1 + G * 2;
    bih1 = whh1 + G * H;
    bhh1 = bih1 + G;
    wih2 = bhh1 + G;
    whh2 = wih2 + G * H;
    bih2 = whh2 + G * H;
    bhh2 = bih2 + G;
    wout = bhh2 + G;
    bout = wout + H;
    total = bout + 1;
  }
};

// forward image of one net: W1T [(H+2)][4H] (weight_ih rows, then weight_hh rows), b1 [4H] (bias_ih + bias_hh),
// W2T [2H][4H] (weight_ih rows, then weight_hh rows), b2 [4H], wout [H], bout
struct Img {
  int64_t w1, b1, w2, b2, wout, bout, total;
  __host__ __device__ explicit Img(int H) {
    const int64_t G = 4 * (int64_t)H;
    w1 = 0;
    b1 = w1 + (H + 2) * G;
    w2 = b1 + G;
    b2 = w2 + 2 * (int64_t)H * G;
    wout = b2 + G;
    bout = wout + H;
    total = bout + 1;
  }
};

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }
__device__ __forceinline__ double sigm(double x) { return 1.0 / (1.0 + exp(-x)); }

__global__ void mm_image_kernel(const float* __restrict__ theta, float* __restrict__ image, int H) {
  const Off o(H);
  const Img m(H);
  const int G = 4 * H, net = blockIdx.y;
  const float* th = theta + net * o.total;
  float* im = image + net * m.total;
  for (int64_t e = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; e < m.total; e += (int64_t)gridDim.x * blockDim.x) {
    float val;
    if (e < m.b1) {
      const int k = (int)(e / G), j = (int)(e % G);
      val = k < 2 ? th[o.wih1 + j * 2 + k] : th[o.whh1 + (int64_t)j * H + (k - 2)];
    } else if (e < m.w2) {
      const int j = (int)(e - m.b1);
      val = th[o.bih1 + j] + th[o.bhh1 + j];
    } else if (e < m.b2) {
      const int k = (int)((e - m.w2) / G), j = (int)((e - m.w2) % G);
      val = k < H ? th[o.wih2 + (int64_t)j * H + k] : th[o.whh2 + (int64_t)j * H + (k - H)];
    } else if (e < m.wout) {
      const int j = (int)(e - m.b2);
      val = th[o.bih2 + j] + th[o.bhh2 + j];
    } else if (e < m.bout) {
      val = th[o.wout + (e - m.wout)];
    } else {
      val = th[o.bout];
    }
    im[e] = val;
  }
}

// ---------------------------------------------------------------------------------------------------------------
// forward

struct FwdSmem {
  float *g, *h1, *c1, *h2, *c2, *u, *v, *gu, *gv, *d, *A, *f;
};

__device__ __forceinline__ FwdSmem carve_fwd(float* s, int cap, int H, int np, int dim) {
  FwdSmem m;
  m.g = s;
  m.h1 = m.g + cap * 4 * H;
  m.c1 = m.h1 + cap * H;
  m.h2 = m.c1 + cap * H;
  m.c2 = m.h2 + cap * H;
  m.u = m.c2 + cap * H;
  m.v = m.u + cap;
  m.gu = m.v + cap;
  m.gv = m.gu + cap;
  m.d = m.gv + cap;
  m.f = m.d + cap;
  m.A = m.f + cap;   // np * dim * dim (loss 4) or np * 2 (a, b)
  (void)np;
  (void)dim;
  return m;
}

inline size_t fwd_smem_bytes(int cap, int H, int np, int dim) {
  return sizeof(float) * ((size_t)cap * (8 * H) + 6 * (size_t)cap + (size_t)np * std::max(2, dim * dim));
}

// df/du and df/dv of local row r (problem p = r / dim, coordinate i) at the shared (u, v): MM ToyLoss.get_grad_*
__device__ __forceinline__ void loss_grads(int loss, int dim, const FwdSmem& m, int r, float& gu, float& gv) {
  const float u = m.u[r], v = m.v[r];
  if (loss == 4) {
    const int p = r / dim, i = r % dim;
    const float* A = m.A + p * dim * dim;
    const float* up = m.u + p * dim;
    const float* vp = m.v + p * dim;
    float su = 0.f, sv = 0.f;
    for (int k = 0; k < dim; ++k) {
      su = fmaf(A[i * dim + k], vp[k], su);   // (A v)_i
      sv = fmaf(A[k * dim + i], up[k], sv);   // (A^T u)_i
    }
    gu = su;
    gv = sv;
    return;
  }
  const float a = m.A[2 * r], b = m.A[2 * r + 1];
  if (loss == 1) {
    gu = 2.f * u * a;
    gv = -2.f * b * v;
  } else if (loss == 2) {
    gu = 2.f * u * a + 2.f * v;
    gv = -2.f * b * v + 2.f * u;
  } else {
    const float ang = a * (float)kPi * u;
    gu = -b * v * cosf(ang) * a * (float)kPi;
    gv = -b * sinf(ang);
  }
}

template <int CAP>
__global__ void __launch_bounds__(512) mm_fwd_kernel(const l2o_minimax_args a, int np) {
  extern __shared__ float smem[];
  const int H = a.hidden, G = 4 * H, dim = a.dim;
  const int R = a.batch * dim;
  const int p0 = blockIdx.x * np;
  const int npb = min(np, a.batch - p0);   // problems of this CTA
  const int nr = npb * dim, r0 = p0 * dim;
  const FwdSmem m = carve_fwd(smem, CAP, H, np, dim);
  const int tid = threadIdx.x, nt = blockDim.x;
  const int warp = tid >> 5, lane = tid & 31, nw = nt >> 5;
  const float al = a.rescale;

  for (int r = tid; r < nr; r += nt) {
    m.u[r] = a.u[r0 + r];
    m.v[r] = a.v[r0 + r];
  }
  const int nA = a.loss == 4 ? npb * dim * dim : npb * 2;
  const int64_t aoff = a.loss == 4 ? (int64_t)p0 * dim * dim : (int64_t)p0 * 2;
  for (int e = tid; e < nA; e += nt) m.A[e] = a.data[aoff + e];
  __syncthreads();
  for (int r = tid; r < nr; r += nt) loss_grads(a.loss, dim, m, r, m.gu[r], m.gv[r]);
  __syncthreads();

  for (int t = a.t0; t < a.t1; ++t) {
    const int net = (t & 1) ? 0 : 1;
    const float* im = a.image + net * Img(H).total;
    const Img io(H);
    float* st = a.state + (int64_t)net * 4 * R * H;
    const int64_t tl = t - a.t0;
    // this net's states of our rows, and their checkpoint
    for (int e = tid; e < nr * H; e += nt) {
      const int r = e / H, k = e % H;
      const int64_t gi = (int64_t)(r0 + r) * H + k;
      const float h1 = st[gi], c1 = st[(int64_t)R * H + gi], h2 = st[2 * (int64_t)R * H + gi],
                  c2 = st[3 * (int64_t)R * H + gi];
      m.h1[r * H + k] = h1;
      m.c1[r * H + k] = c1;
      m.h2[r * H + k] = h2;
      m.c2[r * H + k] = c2;
      if (a.ckpt) {
        float* ck = a.ckpt + (tl * R + r0 + r) * (int64_t)(G + 2) + 2;
        ck[k] = h1;
        ck[H + k] = c1;
        ck[2 * H + k] = h2;
        ck[3 * H + k] = c2;
      }
    }
    if (a.ckpt)
      for (int r = tid; r < nr; r += nt) {
        float* ck = a.ckpt + (tl * R + r0 + r) * (int64_t)(G + 2);
        ck[0] = net ? m.gv[r] : m.gu[r];
        ck[1] = net ? m.gu[r] : m.gv[r];
      }
    __syncthreads();

    // layer 1 gates: [x0, x1, rescale h1] W1^T + b1
    for (int j = tid; j < G; j += nt) {
      const float* w = im + io.w1 + j;
      float acc[CAP];
      const float w0 = w[0], w1v = w[G], b = im[io.b1 + j];
#pragma unroll
      for (int r = 0; r < CAP; ++r) {
        const float x0 = net ? m.gv[r] : m.gu[r], x1 = net ? m.gu[r] : m.gv[r];
        acc[r] = r < nr ? fmaf(w0, x0, fmaf(w1v, x1, b)) : 0.f;
      }
#pragma unroll (CAP <= 8 ? 8 : 2)
      for (int k = 0; k < H; ++k) {
        const float wk = __ldg(w + (int64_t)(k + 2) * G);
#pragma unroll
        for (int r = 0; r < CAP; ++r)
          if (r < nr) acc[r] = fmaf(wk, al * m.h1[r * H + k], acc[r]);
      }
#pragma unroll
      for (int r = 0; r < CAP; ++r)
        if (r < nr) m.g[r * G + j] = acc[r];
    }
    __syncthreads();
    for (int e = tid; e < nr * H; e += nt) {
      const int r = e / H, k = e % H;
      const float* g = m.g + r * G;
      const float ig = sigm(g[k]), fg = sigm(g[H + k]), gg = tanhf(g[2 * H + k]), og = sigm(g[3 * H + k]);
      const float c = fmaf(fg, al * m.c1[e], ig * gg);
      m.c1[e] = c;
      m.h1[e] = og * tanhf(c);
    }
    __syncthreads();
    // layer 2 gates: [h1, rescale h2] W2^T + b2
    for (int j = tid; j < G; j += nt) {
      const float* w = im + io.w2 + j;
      float acc[CAP];
      const float b = im[io.b2 + j];
#pragma unroll
      for (int r = 0; r < CAP; ++r) acc[r] = b;
#pragma unroll (CAP <= 8 ? 8 : 2)
      for (int k = 0; k < H; ++k) {
        const float wa = __ldg(w + (int64_t)k * G), wb = __ldg(w + (int64_t)(H + k) * G);
#pragma unroll
        for (int r = 0; r < CAP; ++r)
          if (r < nr) acc[r] = fmaf(wb, al * m.h2[r * H + k], fmaf(wa, m.h1[r * H + k], acc[r]));
      }
#pragma unroll
      for (int r = 0; r < CAP; ++r)
        if (r < nr) m.g[r * G + j] = acc[r];
    }
    __syncthreads();
    for (int e = tid; e < nr * H; e += nt) {
      const int r = e / H, k = e % H;
      const float* g = m.g + r * G;
      const float ig = sigm(g[k]), fg = sigm(g[H + k]), gg = tanhf(g[2 * H + k]), og = sigm(g[3 * H + k]);
      const float c = fmaf(fg, al * m.c2[e], ig * gg);
      m.c2[e] = c;
      m.h2[e] = og * tanhf(c);
    }
    __syncthreads();
    for (int e = tid; e < nr * H; e += nt) {
      const int r = e / H, k = e % H;
      const int64_t gi = (int64_t)(r0 + r) * H + k;
      st[gi] = m.h1[e];
      st[(int64_t)R * H + gi] = m.c1[e];
      st[2 * (int64_t)R * H + gi] = m.h2[e];
      st[3 * (int64_t)R * H + gi] = m.c2[e];
    }
    // output layer and update, one warp per row
    for (int r = warp; r < nr; r += nw) {
      float s = 0.f;
      for (int k = lane; k < H; k += 32) s = fmaf(im[io.wout + k], m.h2[r * H + k], s);
#pragma unroll
      for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) {
        const float delta = s + im[io.bout];
        float* x = net ? m.v : m.u;
        if (t < a.warm_end) {
          const float sg = delta > 0.f ? 1.f : (delta < 0.f ? -1.f : 0.f);
          x[r] = x[r] + sg * a.lr[t - 1];
        } else {
          x[r] = x[r] + delta * a.out_mul;
        }
      }
    }
    __syncthreads();
    for (int r = tid; r < nr; r += nt) {
      float gu, gv;
      loss_grads(a.loss, dim, m, r, gu, gv);
      m.gu[r] = gu;
      m.gv[r] = gv;
      if (a.dl) a.dl[tl * R + r0 + r] = net ? -gv : gu;
      if (a.traj) {
        a.traj[(tl * R + r0 + r) * 2] = m.u[r];
        a.traj[(tl * R + r0 + r) * 2 + 1] = m.v[r];
      }
    }
    if (a.lval) {
      __syncthreads();
      for (int p = tid; p < npb; p += nt) {
        float f;
        if (a.loss == 4) {
          f = 0.f;
          for (int i = 0; i < dim; ++i) f = fmaf(m.u[p * dim + i], m.gu[p * dim + i], f);
        } else {
          const float u = m.u[p], v = m.v[p], aa = m.A[2 * p], b = m.A[2 * p + 1];
          if (a.loss == 1)
            f = aa * u * u - b * v * v;
          else if (a.loss == 2)
            f = aa * u * u - b * v * v + 2.f * v * u;
          else
            f = -b * v * sinf((float)kPi * u * aa);
        }
        a.lval[tl * a.batch + p0 + p] = net ? -f : f;
      }
    }
    __syncthreads();
  }
  for (int r = tid; r < nr; r += nt) {
    a.u[r0 + r] = m.u[r];
    a.v[r0 + r] = m.v[r];
  }
}

// ---------------------------------------------------------------------------------------------------------------
// backward

__host__ __device__ inline int64_t dg_width(int H) { return 8 * (int64_t)H + 1; }   // dz1 [4H], dz2 [4H], d delta
__host__ __device__ inline int64_t act_width(int H) { return 4 * (int64_t)H + 5; }  // [x0, x1, 1, al h1p | 1, h1n, al h2p | 1, h2n]

struct Bwd {
  l2o_minimax_args a;
  l2o_minimax_grads g;
};

__global__ void __launch_bounds__(512) mm_chain_kernel(const Bwd P) {
  extern __shared__ double dsm[];
  const l2o_minimax_args& a = P.a;
  const int H = a.hidden, G = 4 * H, R = a.batch * a.dim;
  const int r0 = blockIdx.x * kBwdRows, nr = min(kBwdRows, R - r0);
  const int tid = threadIdx.x, nt = blockDim.x;
  const double al = a.rescale;
  const int64_t DW = dg_width(H), AW = act_width(H);
  double* carry = dsm;                             // [2 nets][4: dh1, dc1, dh2, dc2][kBwdRows][H]
  double* z1 = carry + 8 * kBwdRows * H;           // [rows][4H] layer-1 gate activations i, f, g, o
  double* z2 = z1 + kBwdRows * G;                  // layer 2
  double* dz = z2 + kBwdRows * G;                  // [rows][4H] gate pre-activation adjoints of the current layer
  double* in = dz + kBwdRows * G;                  // [rows][2]
  double* h1p = in + kBwdRows * 2;                 // [rows][H] x6: al h1p, c1p, al h2p, c2p, c1n, h1n
  double* c1p = h1p + kBwdRows * H;
  double* h2p = c1p + kBwdRows * H;
  double* c2p = h2p + kBwdRows * H;
  double* c1n = c2p + kBwdRows * H;
  double* h1n = c1n + kBwdRows * H;
  double* c2n = h1n + kBwdRows * H;
  double* h2n = c2n + kBwdRows * H;
  double* dd = h2n + kBwdRows * H;                 // [rows] d delta

  for (int e = tid; e < 8 * kBwdRows * H; e += nt) carry[e] = 0.0;
  const Img io(H);
  const Off oo(H);
  for (int t = a.t1 - 1; t >= a.t0; --t) {
    const int net = (t & 1) ? 0 : 1;
    const float* im = a.image + net * io.total;
    const float* th = a.theta + net * oo.total;
    double* cy = carry + net * 4 * kBwdRows * H;
    const int64_t tl = t - a.t0;
    __syncthreads();
    for (int e = tid; e < nr * H; e += nt) {
      const int r = e / H, k = e % H;
      const float* ck = a.ckpt + (tl * R + r0 + r) * (int64_t)(G + 2) + 2;
      h1p[e] = al * (double)ck[k];
      c1p[e] = ck[H + k];
      h2p[e] = al * (double)ck[2 * H + k];
      c2p[e] = ck[3 * H + k];
    }
    for (int r = tid; r < nr; r += nt) {
      const float* ck = a.ckpt + (tl * R + r0 + r) * (int64_t)(G + 2);
      in[2 * r] = ck[0];
      in[2 * r + 1] = ck[1];
      const int p = (r0 + r) / a.dim;
      const double w = P.g.weight ? (double)P.g.weight[p] : 1.0;
      // the sign step passes no gradient; after it x += delta out_mul
      dd[r] = t < a.warm_end ? 0.0 : (double)P.g.coef[tl] * w * (double)a.dl[tl * R + r0 + r] * (double)a.out_mul;
    }
    __syncthreads();
    // recompute layer 1
    for (int j = tid; j < G; j += nt) {
      const float* w = im + io.w1 + j;
      double acc[kBwdRows];
#pragma unroll
      for (int r = 0; r < kBwdRows; ++r)
        acc[r] = r < nr ? (double)th[oo.bih1 + j] + (double)th[oo.bhh1 + j] + (double)w[0] * in[2 * r] +
                              (double)w[G] * in[2 * r + 1]
                        : 0.0;
#pragma unroll 2
      for (int k = 0; k < H; ++k) {
        const double wk = __ldg(w + (int64_t)(k + 2) * G);
#pragma unroll
        for (int r = 0; r < kBwdRows; ++r)
          if (r < nr) acc[r] = fma(wk, h1p[r * H + k], acc[r]);
      }
#pragma unroll
      for (int r = 0; r < kBwdRows; ++r)
        if (r < nr) z1[r * G + j] = j >= 2 * H && j < 3 * H ? tanh(acc[r]) : sigm(acc[r]);
    }
    __syncthreads();
    for (int e = tid; e < nr * H; e += nt) {
      const int r = e / H, k = e % H;
      const double* z = z1 + r * G;
      const double c = z[H + k] * c1p[e] * al + z[k] * z[2 * H + k];
      c1n[e] = c;
      h1n[e] = z[3 * H + k] * tanh(c);
    }
    __syncthreads();
    // recompute layer 2
    for (int j = tid; j < G; j += nt) {
      const float* w = im + io.w2 + j;
      double acc[kBwdRows];
#pragma unroll
      for (int r = 0; r < kBwdRows; ++r) acc[r] = (double)th[oo.bih2 + j] + (double)th[oo.bhh2 + j];
#pragma unroll 2
      for (int k = 0; k < H; ++k) {
        const double wa = __ldg(w + (int64_t)k * G), wb = __ldg(w + (int64_t)(H + k) * G);
#pragma unroll
        for (int r = 0; r < kBwdRows; ++r)
          if (r < nr) acc[r] = fma(wb, h2p[r * H + k], fma(wa, h1n[r * H + k], acc[r]));
      }
#pragma unroll
      for (int r = 0; r < kBwdRows; ++r)
        if (r < nr) z2[r * G + j] = j >= 2 * H && j < 3 * H ? tanh(acc[r]) : sigm(acc[r]);
    }
    __syncthreads();
    for (int e = tid; e < nr * H; e += nt) {
      const int r = e / H, k = e % H;
      const double* z = z2 + r * G;
      const double c = z[H + k] * c2p[e] * al + z[k] * z[2 * H + k];
      c2n[e] = c;
      h2n[e] = z[3 * H + k] * tanh(c);
    }
    __syncthreads();
    // layer 2 cell backward: dh2 = d delta wout + carried dh2
    for (int e = tid; e < nr * H; e += nt) {
      const int r = e / H, k = e % H;
      const double* z = z2 + r * G;
      const double ig = z[k], fg = z[H + k], gg = z[2 * H + k], og = z[3 * H + k];
      const double dh = dd[r] * (double)th[oo.wout + k] + cy[(2 * kBwdRows + r) * H + k];
      const double tc = tanh(c2n[e]);
      const double dc = cy[(3 * kBwdRows + r) * H + k] + dh * og * (1.0 - tc * tc);
      double* d = dz + r * G;
      d[k] = dc * gg * ig * (1.0 - ig);
      d[H + k] = dc * c2p[e] * al * fg * (1.0 - fg);
      d[2 * H + k] = dc * ig * (1.0 - gg * gg);
      d[3 * H + k] = dh * tc * og * (1.0 - og);
      cy[(3 * kBwdRows + r) * H + k] = dc * fg * al;
    }
    __syncthreads();
    // dh1n = dz2 W_ih2 (written to c1p's slot after use: c1p is not needed again), carried dh2 = al dz2 W_hh2
    for (int k = tid; k < 2 * H; k += nt) {
      const float* w = th + (k < H ? oo.wih2 + k : oo.whh2 + (k - H));
      double acc[kBwdRows];
#pragma unroll
      for (int r = 0; r < kBwdRows; ++r) acc[r] = 0.0;
      for (int j = 0; j < G; ++j) {
        const double wj = __ldg(w + (int64_t)j * H);
#pragma unroll
        for (int r = 0; r < kBwdRows; ++r)
          if (r < nr) acc[r] = fma(wj, dz[r * G + j], acc[r]);
      }
#pragma unroll
      for (int r = 0; r < kBwdRows; ++r)
        if (r < nr) {
          if (k < H)
            c2n[r * H + k] = acc[r];   // c2n is dead past the cell backward: reuse it for dh1n
          else
            cy[(2 * kBwdRows + r) * H + (k - H)] = al * acc[r];
        }
    }
    // record layer-2 and output-layer adjoints and inputs
    for (int e = tid; e < nr * (G + 1); e += nt) {
      const int r = e / (G + 1), j = e % (G + 1);
      double* o = (double*)P.g.scratch + (tl * R + r0 + r) * DW;
      if (j < G)
        o[G + j] = dz[r * G + j];
      else
        o[2 * G] = dd[r];
    }
    __syncthreads();
    // layer 1 cell backward
    for (int e = tid; e < nr * H; e += nt) {
      const int r = e / H, k = e % H;
      const double* z = z1 + r * G;
      const double ig = z[k], fg = z[H + k], gg = z[2 * H + k], og = z[3 * H + k];
      const double dh = c2n[e] + cy[r * H + k];
      const double tc = tanh(c1n[e]);
      const double dc = cy[(kBwdRows + r) * H + k] + dh * og * (1.0 - tc * tc);
      double* d = dz + r * G;
      d[k] = dc * gg * ig * (1.0 - ig);
      d[H + k] = dc * c1p[e] * al * fg * (1.0 - fg);
      d[2 * H + k] = dc * ig * (1.0 - gg * gg);
      d[3 * H + k] = dh * tc * og * (1.0 - og);
      cy[(kBwdRows + r) * H + k] = dc * fg * al;
    }
    __syncthreads();
    // carried dh1 = al dz1 W_hh1
    for (int k = tid; k < H; k += nt) {
      const float* w = th + oo.whh1 + k;
      double acc[kBwdRows];
#pragma unroll
      for (int r = 0; r < kBwdRows; ++r) acc[r] = 0.0;
      for (int j = 0; j < G; ++j) {
        const double wj = __ldg(w + (int64_t)j * H);
#pragma unroll
        for (int r = 0; r < kBwdRows; ++r)
          if (r < nr) acc[r] = fma(wj, dz[r * G + j], acc[r]);
      }
#pragma unroll
      for (int r = 0; r < kBwdRows; ++r)
        if (r < nr) cy[r * H + k] = al * acc[r];
    }
    for (int e = tid; e < nr * G; e += nt) {
      const int r = e / G, j = e % G;
      ((double*)P.g.scratch)[(tl * R + r0 + r) * DW + j] = dz[e];
    }
    double* act = (double*)P.g.scratch + (int64_t)(a.t1 - a.t0) * R * DW;
    for (int e = tid; e < nr * (int)AW; e += nt) {
      const int r = e / (int)AW, c = e % (int)AW;
      double val;
      if (c < 2)
        val = in[2 * r + c];
      else if (c == 2 || c == H + 3 || c == 3 * H + 4)
        val = 1.0;
      else if (c < H + 3)
        val = h1p[r * H + c - 3];
      else if (c < 2 * H + 4)
        val = h1n[r * H + c - (H + 4)];
      else if (c < 3 * H + 4)
        val = h2p[r * H + c - (2 * H + 4)];
      else
        val = h2n[r * H + c - (3 * H + 5)];
      act[(tl * R + r0 + r) * AW + c] = val;
    }
  }
}

// dtheta of net blockIdx.z, layer blockIdx.y: sum over that net's (iteration, row) items of dz^T [inputs]
__global__ void __launch_bounds__(256) mm_dw_kernel(const Bwd P) {
  const l2o_minimax_args& a = P.a;
  const int H = a.hidden, G = 4 * H, R = a.batch * a.dim;
  const int net = blockIdx.z, job = blockIdx.y;
  const int64_t DW = dg_width(H), AW = act_width(H);
  const int Pd = job == 2 ? 1 : G;
  const int Qd = job == 0 ? H + 3 : (job == 1 ? 2 * H + 1 : H + 1);
  const int acol = job == 0 ? 0 : (job == 1 ? G : 2 * G);
  const int bcol = job == 0 ? 0 : (job == 1 ? H + 3 : 3 * H + 4);
  const int tq = (Qd + kTile - 1) / kTile;
  const int tile = blockIdx.x;
  if (tile >= tq * ((Pd + kTile - 1) / kTile)) return;
  const int p0 = (tile / tq) * kTile, q0 = (tile % tq) * kTile;
  const double* dg = (const double*)P.g.scratch;
  const double* act = dg + (int64_t)(a.t1 - a.t0) * R * DW;
  // items: iterations of this net's parity inside [t0, t1), all rows, in increasing order
  const int tfirst = ((a.t0 & 1) == (net == 0 ? 1 : 0)) ? a.t0 : a.t0 + 1;
  const int nts = tfirst < a.t1 ? (a.t1 - tfirst + 1) / 2 : 0;
  const int64_t n_items = (int64_t)nts * R;
  __shared__ double sA[kTile][kTile + 1], sB[kTile][kTile + 1];
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  double acc[4] = {0.0, 0.0, 0.0, 0.0};
  for (int64_t n0 = 0; n0 < n_items; n0 += kTile) {
    for (int e = threadIdx.x; e < kTile * kTile; e += blockDim.x) {
      const int i = e / kTile, c = e % kTile;
      const int64_t n = n0 + i;
      double va = 0.0, vb = 0.0;
      if (n < n_items) {
        const int64_t row = (int64_t)(tfirst - a.t0 + 2 * (n / R)) * R + n % R;
        if (p0 + c < Pd) va = dg[row * DW + acol + p0 + c];
        if (q0 + c < Qd) vb = act[row * AW + bcol + q0 + c];
      }
      sA[i][c] = va;
      sB[i][c] = vb;
    }
    __syncthreads();
#pragma unroll 8
    for (int i = 0; i < kTile; ++i) {
      const double b = sB[i][tx];
#pragma unroll
      for (int s = 0; s < 4; ++s) acc[s] = fma(sA[i][ty + 8 * s], b, acc[s]);
    }
    __syncthreads();
  }
  const Off oo(H);
  double* out = P.g.dtheta + net * oo.total;
  const int q = q0 + tx;
  if (q >= Qd) return;
#pragma unroll
  for (int s = 0; s < 4; ++s) {
    const int p = p0 + ty + 8 * s;
    if (p >= Pd) continue;
    const double val = acc[s];
    if (job == 0) {
      if (q < 2)
        out[oo.wih1 + p * 2 + q] = val;
      else if (q == 2) {
        out[oo.bih1 + p] = val;
        out[oo.bhh1 + p] = val;
      } else {
        out[oo.whh1 + (int64_t)p * H + (q - 3)] = val;
      }
    } else if (job == 1) {
      if (q == 0) {
        out[oo.bih2 + p] = val;
        out[oo.bhh2 + p] = val;
      } else if (q <= H) {
        out[oo.wih2 + (int64_t)p * H + (q - 1)] = val;
      } else {
        out[oo.whh2 + (int64_t)p * H + (q - 1 - H)] = val;
      }
    } else {
      if (q == 0)
        out[oo.bout] = val;
      else
        out[oo.wout + q - 1] = val;
    }
  }
}

// ---------------------------------------------------------------------------------------------------------------
// host side

inline int rows(const l2o_minimax_args& a) { return a.batch * a.dim; }
inline int fwd_cap(const l2o_minimax_args& a) { return a.dim <= 8 ? 8 : 32; }
inline int fwd_np(const l2o_minimax_args& a) { return std::max(1, fwd_cap(a) / a.dim); }
inline int threads_for(int H) { return std::max(128, (4 * H + 31) / 32 * 32); }
inline size_t bwd_smem_bytes(int H) {
  return sizeof(double) * ((size_t)8 * kBwdRows * H + 3 * (size_t)kBwdRows * 4 * H + 2 * kBwdRows +
                           8 * (size_t)kBwdRows * H + kBwdRows);
}

int check_args(const l2o_minimax_args* a) {
  if (!a || a->loss < 1 || a->loss > 4 || a->batch <= 0 || a->dim <= 0 || a->hidden <= 0) return L2O_E_INVALID;
  if (a->t0 < 1 || a->t1 <= a->t0 || a->warm_end < 1) return L2O_E_INVALID;
  if (!a->image || !a->data || !a->u || !a->v || !a->state) return L2O_E_INVALID;
  if (a->t0 < a->warm_end && !a->lr) return L2O_E_INVALID;
  const void* ptrs[] = {a->lr, a->theta, a->image, a->data, a->u, a->v, a->state, a->traj, a->ckpt, a->dl, a->lval};
  for (const void* q : ptrs)
    if (misaligned(q, 4)) return L2O_E_INVALID;
  if (a->hidden > L2O_MINIMAX_MAX_HIDDEN || a->dim > L2O_MINIMAX_MAX_DIM) return L2O_E_UNSUPPORTED;
  if (a->loss != 4 && a->dim != 1) return L2O_E_UNSUPPORTED;
  return L2O_OK;
}

size_t scratch_bytes(const l2o_minimax_args& a) {
  return sizeof(double) * (size_t)(a.t1 - a.t0) * rows(a) * (size_t)(dg_width(a.hidden) + act_width(a.hidden));
}

}  // namespace minimax
}  // namespace l2o

using namespace l2o::minimax;

extern "C" {

int64_t l2o_minimax_theta_count(int32_t hidden) { return hidden > 0 ? Off(hidden).total : 0; }
int64_t l2o_minimax_image_floats(int32_t hidden) { return hidden > 0 ? Img(hidden).total : 0; }

int l2o_minimax_image(const float* theta, float* image, int32_t hidden, void* stream) {
  if (!theta || !image || hidden <= 0 || l2o::misaligned(theta, 4) || l2o::misaligned(image, 4)) return L2O_E_INVALID;
  if (hidden > L2O_MINIMAX_MAX_HIDDEN) return L2O_E_UNSUPPORTED;
  const int blocks = (int)std::min<int64_t>((Img(hidden).total + 255) / 256, 1024);
  mm_image_kernel<<<dim3(blocks, 2), 256, 0, (cudaStream_t)stream>>>(theta, image, hidden);
  return l2o::after_launch("l2o_minimax_image");
}

int l2o_minimax_workspace_bytes(const l2o_minimax_args* a, size_t* bytes) {
  if (!bytes) return L2O_E_INVALID;
  if (int rc = check_args(a)) return rc;
  *bytes = scratch_bytes(*a);
  return L2O_OK;
}

int l2o_minimax_fwd(const l2o_minimax_args* a, void* stream) {
  if (int rc = check_args(a)) return rc;
  const int cap = fwd_cap(*a), np = fwd_np(*a);
  const size_t smem = fwd_smem_bytes(cap, a->hidden, np, a->dim);
  const int grid = (a->batch + np - 1) / np, nt = threads_for(a->hidden);
  if (cap == 8) {
    if (int rc = l2o::raise_smem_limit("l2o_minimax_fwd", mm_fwd_kernel<8>, smem)) return rc;
    mm_fwd_kernel<8><<<grid, nt, smem, (cudaStream_t)stream>>>(*a, np);
  } else {
    if (int rc = l2o::raise_smem_limit("l2o_minimax_fwd", mm_fwd_kernel<32>, smem)) return rc;
    mm_fwd_kernel<32><<<grid, nt, smem, (cudaStream_t)stream>>>(*a, np);
  }
  return l2o::after_launch("l2o_minimax_fwd");
}

int l2o_minimax_bwd(const l2o_minimax_args* a, const l2o_minimax_grads* g, void* stream) {
  if (int rc = check_args(a)) return rc;
  if (!g || !a->theta || !a->ckpt || !a->dl || !g->coef || !g->dtheta || !g->scratch) return L2O_E_INVALID;
  if (l2o::misaligned(g->coef, 4) || l2o::misaligned(g->weight, 4) || l2o::misaligned(g->dtheta, 8) ||
      l2o::misaligned(g->scratch, 8))
    return L2O_E_INVALID;
  Bwd p{*a, *g};
  const int H = a->hidden;
  const size_t smem = bwd_smem_bytes(H);
  if (int rc = l2o::raise_smem_limit("l2o_minimax_bwd", mm_chain_kernel, smem)) return rc;
  mm_chain_kernel<<<(rows(*a) + kBwdRows - 1) / kBwdRows, threads_for(H), smem, (cudaStream_t)stream>>>(p);
  if (int rc = l2o::after_launch("l2o_minimax_bwd")) return rc;
  const int tiles = ((4 * H + kTile - 1) / kTile) * ((2 * H + 1 + kTile - 1) / kTile);
  mm_dw_kernel<<<dim3(tiles, 3, 2), 256, 0, (cudaStream_t)stream>>>(p);
  return l2o::after_launch("l2o_minimax_bwd");
}

}  // extern "C"
