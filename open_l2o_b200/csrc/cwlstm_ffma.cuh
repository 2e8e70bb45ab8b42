// Exact-fp32 CUDA-core engine: one thread owns one coordinate; the shared [K x 4H] gate weights
// live in shared memory and are read with warp-uniform 128-bit loads; the coordinate's (h, c)
// state stays in registers across the whole T-step unroll.  This engine is the always-available
// parity anchor for the tensor-core engine (cwlstm_tc.cuh) and serves the small test-only net shapes.
//
// Reference semantics: DM/networks.py:207-232, DM/meta.py:319-376 (forward); SURVEY.md Appendix B
// (backward, derived from DM/meta.py:319-376 with second_derivatives=False).
#pragma once
#include "cwlstm_common.cuh"

namespace l2o {

constexpr int kTile = 128;  // coordinates (= threads) per CTA tile

// ------------------------------------------------------------------------------------------
// per-coordinate building blocks (all loops fully unrolled => arrays live in registers)
// ------------------------------------------------------------------------------------------
template <int KIN, int H>
__device__ __forceinline__ void gate_preact(const float* __restrict__ sW, const float* __restrict__ sB,
                                            const float* in, const float* h, float* z) {
  constexpr int NG = 4 * H;
#pragma unroll
  for (int q = 0; q < H; ++q) {
    const float4 b = *reinterpret_cast<const float4*>(sB + 4 * q);
    z[4 * q + 0] = b.x; z[4 * q + 1] = b.y; z[4 * q + 2] = b.z; z[4 * q + 3] = b.w;
  }
#pragma unroll
  for (int k = 0; k < KIN + H; ++k) {
    const float a = (k < KIN) ? in[k < KIN ? k : 0] : h[k >= KIN ? k - KIN : 0];
    const float4* row = reinterpret_cast<const float4*>(sW + k * NG);
#pragma unroll
    for (int q = 0; q < H; ++q) {
      const float4 w = row[q];
      z[4 * q + 0] = fmaf(a, w.x, z[4 * q + 0]);
      z[4 * q + 1] = fmaf(a, w.y, z[4 * q + 1]);
      z[4 * q + 2] = fmaf(a, w.z, z[4 * q + 2]);
      z[4 * q + 3] = fmaf(a, w.w, z[4 * q + 3]);
    }
  }
}

// snt.LSTM pointwise part: z -> activated gates in place (i | j | f | o); c: prev -> new; h out.
template <int H>
__device__ __forceinline__ void lstm_pointwise(float* z, float* c, float* h, float* tc /*nullable*/) {
#pragma unroll
  for (int u = 0; u < H; ++u) {
    const float i = sigmoid_acc(z[u]);
    const float j = tanh_acc(z[H + u]);
    const float f = sigmoid_acc(z[2 * H + u] + 1.0f);
    const float o = sigmoid_acc(z[3 * H + u]);
    z[u] = i; z[H + u] = j; z[2 * H + u] = f; z[3 * H + u] = o;
    const float cn = fmaf(f, c[u], i * j);
    const float t = tanh_acc(cn);
    c[u] = cn;
    h[u] = t * o;
    if (tc) tc[u] = t;
  }
}

template <class C>
__device__ __forceinline__ void preprocess(const float* __restrict__ sT, const NetRt& rt, float raw0, float raw1,
                                           float* u) {
  if constexpr (C::FC) {
#pragma unroll
    for (int j = 0; j < C::F; ++j) {
      float a = sT[C::O_BIN + j];
      a = fmaf(raw0, sT[C::O_WIN + j], a);
      if constexpr (C::NIN == 2) a = fmaf(raw1, sT[C::O_WIN + C::F + j], a);
      u[j] = elu_acc(a);
    }
  } else if constexpr (C::PRE == L2O_PRE_LOGSIGN) {
    static_assert(C::PRE != L2O_PRE_LOGSIGN || C::NIN == 1, "LogAndSign is coordinate-wise single-input");
    log_and_sign(raw0, rt.logsign_k, rt.logsign_ek, u[0], u[1]);
  } else {
    u[0] = raw0;
    if constexpr (C::NIN == 2) u[1] = raw1;
  }
}

template <int H>
__device__ __forceinline__ void load_vec(const float* __restrict__ p, float* v) {
  if constexpr (H % 4 == 0) {
#pragma unroll
    for (int q = 0; q < H / 4; ++q) {
      const float4 t = reinterpret_cast<const float4*>(p)[q];
      v[4 * q] = t.x; v[4 * q + 1] = t.y; v[4 * q + 2] = t.z; v[4 * q + 3] = t.w;
    }
  } else {
#pragma unroll
    for (int k = 0; k < H; ++k) v[k] = p[k];
  }
}
template <int H>
__device__ __forceinline__ void store_vec(float* __restrict__ p, const float* v) {
  if constexpr (H % 4 == 0) {
#pragma unroll
    for (int q = 0; q < H / 4; ++q)
      reinterpret_cast<float4*>(p)[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
  } else {
#pragma unroll
    for (int k = 0; k < H; ++k) p[k] = v[k];
  }
}

template <class C>
struct CoordState {
  float h1[cmax(C::H1, 1)], c1[cmax(C::H1, 1)], h2[cmax(C::H2, 1)], c2[cmax(C::H2, 1)];
  __device__ __forceinline__ void load(const float* __restrict__ arena, int64_t n, int64_t i) {
    if constexpr (C::H1 > 0) {
      load_vec<C::H1>(arena + i * C::H1, h1);
      load_vec<C::H1>(arena + (n + i) * C::H1, c1);
    }
    if constexpr (C::H2 > 0) {
      const float* b2 = arena + 2 * n * C::H1;
      load_vec<C::H2>(b2 + i * C::H2, h2);
      load_vec<C::H2>(b2 + (n + i) * C::H2, c2);
    }
  }
  __device__ __forceinline__ void store(float* __restrict__ arena, int64_t n, int64_t i) const {
    if constexpr (C::H1 > 0) {
      store_vec<C::H1>(arena + i * C::H1, h1);
      store_vec<C::H1>(arena + (n + i) * C::H1, c1);
    }
    if constexpr (C::H2 > 0) {
      float* b2 = arena + 2 * n * C::H1;
      store_vec<C::H2>(b2 + i * C::H2, h2);
      store_vec<C::H2>(b2 + (n + i) * C::H2, c2);
    }
  }
};

// One time step of the net for one coordinate; state updated in place; returns delta.
template <class C>
__device__ __forceinline__ float net_forward(const float* __restrict__ sT, const NetRt& rt, const float* u,
                                             CoordState<C>& s) {
  const float* top = u;
  if constexpr (C::H1 > 0) {
    float z[cmax(C::G1, 1)];
    gate_preact<C::F, C::H1>(sT + C::O_W1, sT + C::O_B1, u, s.h1, z);
    lstm_pointwise<C::H1>(z, s.c1, s.h1, nullptr);
    top = s.h1;
  }
  if constexpr (C::H2 > 0) {
    float z[cmax(C::G2, 1)];
    gate_preact<C::H1, C::H2>(sT + C::O_W2, sT + C::O_B2, s.h1, s.h2, z);
    lstm_pointwise<C::H2>(z, s.c2, s.h2, nullptr);
    top = s.h2;
  }
  float y = sT[C::O_BO];
#pragma unroll
  for (int k = 0; k < C::TOP; ++k) y = fmaf(top[k], sT[C::O_WO + k], y);
  return rt.tanh_output ? tanh_acc(y) * rt.scale : y * rt.scale;
}

template <class C>
__device__ __forceinline__ void stage_theta(float* sT, const float* __restrict__ theta) {
  for (int k = threadIdx.x; k < C::P; k += blockDim.x) sT[k] = theta[k];
  __syncthreads();
}

__host__ __device__ constexpr int round4(int x) { return (x + 3) / 4 * 4; }

// ------------------------------------------------------------------------------------------
// K1: one step, state in HBM (the external-gradient regime: autograd runs between steps).
// Algorithmic HBM traffic per coordinate: 2*SF*4 (state r+w) + 4 (g) + 8 (x r+w)  [= 652 B, H=20x2]
// ------------------------------------------------------------------------------------------
template <class C>
__global__ void __launch_bounds__(kTile) step_kernel(l2o_step_args a, NetRt rt) {
  extern __shared__ __align__(16) float smem[];
  float* sT = smem;
  stage_theta<C>(sT, a.theta);
  const int64_t n = a.n;
  for (int64_t tile = blockIdx.x; tile * kTile < n; tile += gridDim.x) {
    const int64_t i = tile * kTile + threadIdx.x;
    if (i >= n) continue;
    float raw0 = a.in0[i], raw1 = 0.f;
    if constexpr (C::NIN == 2) {
      if (a.m != nullptr) {
        float m = a.m[i], v = a.v[i];
        const float p = a.step_ptr ? (float)(*a.step_ptr + a.t_offset) : a.p;
        adam_features(raw0, m, v, a.beta1, a.beta2, p, raw0, raw1);
        a.m[i] = m; a.v[i] = v;
      } else {
        raw1 = a.in1[i];
      }
      if (a.feat_out) { a.feat_out[i] = raw0; a.feat_out[n + i] = raw1; }
    }
    float u[C::F];
    preprocess<C>(sT, rt, raw0, raw1, u);
    CoordState<C> s;
    s.load(a.state_in, n, i);
    const float d = net_forward<C>(sT, rt, u, s);
    s.store(a.state_out, n, i);
    if (a.delta) a.delta[i] = d;
    if (a.x) a.x[i] += d;
  }
}

// ------------------------------------------------------------------------------------------
// K2: fused T-step unroll; state in registers for all T steps.
// ------------------------------------------------------------------------------------------
// L2O_OPT_QUADRATIC_BATCH (DM/problems.py:73-101): f = fscale * sum_b ||W_b x_b - y_b||^2 with a dense W_b [d,d] per
// group of d consecutive coordinates; g = 2 fscale W_b^T (W_b x_b - y_b).  Called by every thread of the CTA: the group
// members exchange x, then the residuals, through shared memory.  Thread = coordinate k of group b owns residual row k.
__device__ __forceinline__ void quadratic_batch_eval(const l2o_unroll_args& a, int gd, bool act, int64_t i, float x,
                                                     float* sX, float* sR, float& f, float& g) {
  const int tid = threadIdx.x;
  sX[tid] = x;
  __syncthreads();
  float r = 0.f;
  int k = 0, t0 = 0;
  if (act) {
    k = (int)(i % gd);
    t0 = tid - k;  // first thread of this group inside the tile
    const float* __restrict__ wrow = a.opt_a + i * gd;   // W[b][k][:]
    float acc = 0.f;
    for (int j = 0; j < gd; ++j) acc = fmaf(wrow[j], sX[t0 + j], acc);
    r = acc - a.opt_b[i];
  }
  sR[tid] = r;
  __syncthreads();
  f = 0.f;
  g = 0.f;
  if (act) {
    const float* __restrict__ wcol = a.opt_a + (i - k) * gd + k;  // W[b][:][k], stride d
    float acc = 0.f;
    for (int j = 0; j < gd; ++j) acc = fmaf(wcol[(int64_t)j * gd], sR[t0 + j], acc);
    g = a.opt_fscale * (2.0f * acc);
    f = a.opt_fscale * (r * r);
  }
}

template <class C>
__global__ void __launch_bounds__(kTile) unroll_fwd_kernel(l2o_unroll_args a, NetRt rt) {
  extern __shared__ __align__(16) float smem[];
  float* sT = smem;
  double* sFx = reinterpret_cast<double*>(smem + round4(C::P) + 4);  // 16B-aligned, [T+1]
  const int T = a.T;
  const bool in_kernel_opt = a.opt_kind != L2O_OPT_NONE;
  const bool want_fx = in_kernel_opt && a.fx != nullptr;
  // dense grouped optimizee (L2O_OPT_QUADRATIC_BATCH): the d coordinates of a group exchange x and residuals through
  // shared memory, so a tile holds whole groups only
  const bool grouped = a.opt_kind == L2O_OPT_QUADRATIC_BATCH;
  const int gd = grouped ? a.opt_group : 1;
  const int tile_n = grouped ? (kTile / gd) * gd : kTile;
  __shared__ float sXg[kTile], sRg[kTile];
  if (want_fx)
    for (int t = threadIdx.x; t <= T; t += blockDim.x) sFx[t] = 0.0;
  stage_theta<C>(sT, a.theta);
  const int64_t n = a.n;
  const int64_t slot = n * C::SF;
  const int lane = threadIdx.x & 31;
  double imit = 0.0;
  for (int64_t tile = blockIdx.x; tile * tile_n < n; tile += gridDim.x) {
    const int64_t i = tile * tile_n + threadIdx.x;
    const bool act = (int)threadIdx.x < tile_n && i < n;
    CoordState<C> s;
    float x = 0.f, oa = 0.f, ob = 0.f, m = 0.f, v = 0.f;
    if (act) {
      s.load(a.state, n, i);
      if (a.ckpt) s.store(a.ckpt, n, i);
      if (a.x) x = a.x[i];
      if (in_kernel_opt && !grouped) { oa = a.opt_a[i]; ob = a.opt_b[i]; }
      if (a.m) { m = a.m[i]; v = a.v[i]; }
    }
    for (int t = 0; t < T; ++t) {
      float fval = 0.f;
      float fq = 0.f, gq = 0.f;
      if (grouped) quadratic_batch_eval(a, gd, act, i, x, sXg, sRg, fq, gq);   // block-wide (two barriers)
      if (act) {
        float raw0, raw1 = 0.f;
        if (grouped) {
          fval = fq;
          raw0 = gq;
          if (a.g_rec) a.g_rec[(int64_t)t * n + i] = raw0;
        } else if (in_kernel_opt) {
          optimizee_eval(a.opt_kind, x, oa, ob, a.opt_alpha, a.opt_fscale, fval, raw0);
          if (a.g_rec) a.g_rec[(int64_t)t * n + i] = raw0;
        } else if (C::NIN == 2 && a.m == nullptr) {
          raw0 = a.in_seq[((int64_t)t * 2) * n + i];
          raw1 = a.in_seq[((int64_t)t * 2 + 1) * n + i];
        } else {
          raw0 = a.in_seq[(int64_t)t * n + i];
        }
        if constexpr (C::NIN == 2) {
          if (a.m != nullptr) adam_features(raw0, m, v, a.beta1, a.beta2, (float)(a.step0 + t), raw0, raw1);
          if (a.feat_rec) {
            a.feat_rec[((int64_t)t * 2) * n + i] = raw0;
            a.feat_rec[((int64_t)t * 2 + 1) * n + i] = raw1;
          }
        }
        float u[C::F];
        preprocess<C>(sT, rt, raw0, raw1, u);
        const float d = net_forward<C>(sT, rt, u, s);
        x += d;
        if (a.ckpt) s.store(a.ckpt + (int64_t)(t + 1) * slot, n, i);
        if (a.delta_seq) a.delta_seq[(int64_t)t * n + i] = d;
        if (a.labels) {
          const float r = a.labels[(int64_t)t * n + i] - d;
          imit += 0.5 * (double)r * (double)r;
        }
      }
      if (want_fx) {
        const double ws = warp_sum_d((double)fval);
        if (lane == 0) atomicAdd(&sFx[t], ws);
      }
    }
    float fval = 0.f;
    float fqT = 0.f, gqT = 0.f;
    if (grouped) quadratic_batch_eval(a, gd, act, i, x, sXg, sRg, fqT, gqT);
    if (act) {
      if (grouped) {
        fval = fqT;
        if (a.g_rec) a.g_rec[(int64_t)T * n + i] = gqT;
      } else if (in_kernel_opt) {
        float gT;
        optimizee_eval(a.opt_kind, x, oa, ob, a.opt_alpha, a.opt_fscale, fval, gT);
        if (a.g_rec) a.g_rec[(int64_t)T * n + i] = gT;
      }
      s.store(a.state, n, i);
      if (a.x) a.x[i] = x;
      if (a.m) { a.m[i] = m; a.v[i] = v; }
    }
    if (want_fx) {
      const double ws = warp_sum_d((double)fval);
      if (lane == 0) atomicAdd(&sFx[T], ws);
    }
  }
  if (a.labels && a.imit_loss) {
    const double ws = warp_sum_d(imit);
    if (lane == 0) atomicAdd(a.imit_loss, ws / (double)a.n_total);
  }
  if (want_fx) {
    __syncthreads();
    for (int t = threadIdx.x; t <= T; t += blockDim.x) atomicAdd(&a.fx[t], sFx[t]);
  }
}

// ------------------------------------------------------------------------------------------
// K3: BPTT.  Reverse-time sweep; gates recomputed from the checkpointed (h, c); per-coordinate
// vectors staged to shared memory so the CTA can reduce dW = X^T dZ over its 128 coordinates with
// a (row-group x col-group) thread tiling whose accumulators persist (in smem slots) over all
// steps and tiles; flushed once per CTA with fp64 atomics.
// ------------------------------------------------------------------------------------------
__host__ __device__ constexpr int conflict_free_stride(int x) {  // multiple of 4 whose quarter is odd => float4 rows of
  int s = round4(x);                          // consecutive threads hit disjoint bank groups
  return ((s / 4) % 2 == 0) ? s + 4 : s;
}

template <int KR, int NC>
struct PassGeom {
  static constexpr int NCG = (NC + 3) / 4;
  static constexpr int RG = (kTile / NCG) < KR ? (kTile / NCG) : KR;
  static constexpr int RPG = (KR + RG - 1) / RG;
  static constexpr int NACC = RPG * 4;
  static constexpr int ROWS_TOUCHED = RG * RPG;
};

template <int KR, int NC, int INS, int DZS>
__device__ __forceinline__ void dw_pass(const float* __restrict__ sIN, const float* __restrict__ sDZ, float* sAcc,
                                        int tid) {
  using G = PassGeom<KR, NC>;
  static_assert(G::ROWS_TOUCHED <= INS, "IN stride too small");
  if (tid >= G::RG * G::NCG) return;
  const int r = tid / G::NCG, q = tid % G::NCG;
  float acc[G::RPG][4];
#pragma unroll
  for (int rr = 0; rr < G::RPG; ++rr)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[rr][j] = sAcc[(rr * 4 + j) * kTile + tid];
#pragma unroll 4
  for (int c = 0; c < kTile; ++c) {
    const float4 d = *reinterpret_cast<const float4*>(sDZ + c * DZS + 4 * q);
    const float* in = sIN + c * INS + r * G::RPG;
#pragma unroll
    for (int rr = 0; rr < G::RPG; ++rr) {
      const float av = in[rr];
      acc[rr][0] = fmaf(av, d.x, acc[rr][0]);
      acc[rr][1] = fmaf(av, d.y, acc[rr][1]);
      acc[rr][2] = fmaf(av, d.z, acc[rr][2]);
      acc[rr][3] = fmaf(av, d.w, acc[rr][3]);
    }
  }
#pragma unroll
  for (int rr = 0; rr < G::RPG; ++rr)
#pragma unroll
    for (int j = 0; j < 4; ++j) sAcc[(rr * 4 + j) * kTile + tid] = acc[rr][j];
}

// rows 0..KR-2 -> W[row][col] (row-major, NC columns) ; row KR-1 -> bias[col]
template <int KR, int NC>
__device__ __forceinline__ void dw_flush(const float* sAcc, double* __restrict__ dtheta, int o_w, int o_b, int tid) {
  using G = PassGeom<KR, NC>;
  if (tid >= G::RG * G::NCG) return;
  const int r = tid / G::NCG, q = tid % G::NCG;
#pragma unroll
  for (int rr = 0; rr < G::RPG; ++rr) {
    const int row = r * G::RPG + rr;
    if (row >= KR) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int col = 4 * q + j;
      if (col >= NC) continue;
      const float v = sAcc[(rr * 4 + j) * kTile + tid];
      const int idx = (row < KR - 1) ? o_w + row * NC + col : o_b + col;
      atomicAdd(&dtheta[idx], (double)v);
    }
  }
}

template <int N>
__device__ __forceinline__ void stage_row(float* row, const float* v) {  // N multiple of 4
#pragma unroll
  for (int q = 0; q < N / 4; ++q)
    reinterpret_cast<float4*>(row)[q] = make_float4(v[4 * q], v[4 * q + 1], v[4 * q + 2], v[4 * q + 3]);
}

// LSTM pointwise backward for one layer.  act = activated gates (i|j|f|o) -> overwritten by dz.
// dh: total gradient wrt h' ; dc: carry in (from step t+1) -> carry out (to step t-1).
template <int H>
__device__ __forceinline__ void lstm_pointwise_bwd(float* act, const float* cprev, const float* tc, const float* dh,
                                                   float* dc) {
#pragma unroll
  for (int u = 0; u < H; ++u) {
    const float i = act[u], j = act[H + u], f = act[2 * H + u], o = act[3 * H + u];
    const float t = tc[u];
    const float d_o = dh[u] * t;
    const float dcv = fmaf(dh[u] * o, 1.0f - t * t, dc[u]);
    act[u] = dcv * j * i * (1.0f - i);
    act[H + u] = dcv * i * (1.0f - j * j);
    act[2 * H + u] = dcv * cprev[u] * f * (1.0f - f);
    act[3 * H + u] = d_o * o * (1.0f - o);
    dc[u] = dcv * f;
  }
}

// din[k] = sum_n W[k][n] dz[n], k in [K0, K0+NK)
template <int NG, int K0, int NK>
__device__ __forceinline__ void matvec_wt(const float* __restrict__ sW, const float* dz, float* out) {
#pragma unroll
  for (int k = 0; k < NK; ++k) {
    const float4* row = reinterpret_cast<const float4*>(sW + (K0 + k) * NG);
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
    for (int q = 0; q < NG / 4; ++q) {
      const float4 w = row[q];
      s0 = fmaf(w.x, dz[4 * q], s0);
      s1 = fmaf(w.y, dz[4 * q + 1], s1);
      s2 = fmaf(w.z, dz[4 * q + 2], s2);
      s3 = fmaf(w.w, dz[4 * q + 3], s3);
    }
    out[k] = (s0 + s1) + (s2 + s3);
  }
}

template <class C>
struct BwdGeom {
  static constexpr int KR1 = C::H1 > 0 ? C::K1 + 1 : 1;
  static constexpr int KR2 = C::H2 > 0 ? C::K2 + 1 : 1;
  static constexpr int KRO = C::TOP + 1;
  static constexpr int KRF = C::NIN + 1;
  using P1 = PassGeom<KR1, cmax(C::G1, 4)>;
  using P2 = PassGeom<KR2, cmax(C::G2, 4)>;
  using PO = PassGeom<KRO, 1>;
  using PF = PassGeom<KRF, cmax(C::F, 4)>;
  static constexpr int INS = conflict_free_stride(cmax(cmax(P1::ROWS_TOUCHED, P2::ROWS_TOUCHED), 4));
  static constexpr int DZS = conflict_free_stride(cmax(cmax(C::G1, C::G2), 4));
  static constexpr int INO = conflict_free_stride(PO::ROWS_TOUCHED);
  static constexpr int DZO = 4;
  static constexpr int INF = conflict_free_stride(cmax(PF::ROWS_TOUCHED, 4));
  static constexpr int DZF = conflict_free_stride(cmax(C::F, 4));
  static constexpr int SCR = conflict_free_stride(cmax(C::G1 + 2 * C::H1, 4));  // act1 | c1p | tc1
  static constexpr int ACC1 = 0;
  static constexpr int ACC2 = ACC1 + (C::H1 > 0 ? P1::NACC : 0);
  static constexpr int ACCO = ACC2 + (C::H2 > 0 ? P2::NACC : 0);
  static constexpr int ACCF = ACCO + PO::NACC;
  static constexpr int NACC = ACCF + (C::FC ? PF::NACC : 0);
  // smem layout (floats)
  static constexpr int S_T = 0;
  static constexpr int S_IN = S_T + round4(C::P) + 4;
  static constexpr int S_DZ = S_IN + kTile * INS;
  static constexpr int S_INO = S_DZ + kTile * DZS;
  static constexpr int S_DZO = S_INO + kTile * INO;
  static constexpr int S_INF = S_DZO + kTile * DZO;
  static constexpr int S_DZF = S_INF + (C::FC ? kTile * INF : 0);
  static constexpr int S_SCR = S_DZF + (C::FC ? kTile * DZF : 0);
  static constexpr int S_ACC = S_SCR + (C::H2 > 0 ? kTile * SCR : 0);
  static constexpr int S_END = S_ACC + NACC * kTile;
  static constexpr size_t BYTES = (size_t)S_END * sizeof(float);
};

// CARRY: one segment of a longer unroll (l2o_unroll_bwd_carry): the carries start from cy and are written back there
template <class C, bool CARRY>
__global__ void __launch_bounds__(kTile) unroll_bwd_kernel(l2o_bwd_args a, NetRt rt, l2o_bwd_carry cy) {
  using B = BwdGeom<C>;
  static_assert(!(C::FC && C::H1 == 0), "fc preprocessing needs at least one LSTM layer");
  extern __shared__ __align__(16) float smem[];
  float* sT = smem + B::S_T;
  float* sIN = smem + B::S_IN;
  float* sDZ = smem + B::S_DZ;
  float* sINO = smem + B::S_INO;
  float* sDZO = smem + B::S_DZO;
  float* sINF = smem + B::S_INF;
  float* sDZF = smem + B::S_DZF;
  float* sSCR = smem + B::S_SCR;
  float* sACC = smem + B::S_ACC;
  const int tid = threadIdx.x;
  for (int k = tid; k < B::NACC * kTile; k += kTile) sACC[k] = 0.f;
  stage_theta<C>(sT, a.theta);

  const int64_t n = a.n;
  const int64_t slot = n * C::SF;
  const int T = a.T;
  float* myIN = sIN + tid * B::INS;
  float* myDZ = sDZ + tid * B::DZS;
  float* myINO = sINO + tid * B::INO;
  float* myDZO = sDZO + tid * B::DZO;
  float* myINF = sINF + tid * B::INF;
  float* myDZF = sDZF + tid * B::DZF;
  float* mySCR = sSCR + tid * B::SCR;

  for (int64_t tile = blockIdx.x; tile * kTile < n; tile += gridDim.x) {
    const int64_t i = tile * kTile + tid;
    const bool act = i < n;
    // carries from step t+1 (zero at t = T-1: the state handed to the next unroll is a constant,
    // DM/meta.py:385-389)
    float dh1c[cmax(C::H1, 1)], dc1c[cmax(C::H1, 1)], dh2c[cmax(C::H2, 1)], dc2c[cmax(C::H2, 1)];
#pragma unroll
    for (int k = 0; k < cmax(C::H1, 1); ++k) { dh1c[k] = 0.f; dc1c[k] = 0.f; }
#pragma unroll
    for (int k = 0; k < cmax(C::H2, 1); ++k) { dh2c[k] = 0.f; dc2c[k] = 0.f; }
    float lam = (act && a.g_rec) ? a.g_rec[(int64_t)T * n + i] : 0.f;
    if constexpr (CARRY) {   // the adjoint of the state after the segment, and lambda = carry + g_t1 (same order)
      if (act) {
        if constexpr (C::H1 > 0) {
          load_vec<C::H1>(cy.d_state + i * C::H1, dh1c);
          load_vec<C::H1>(cy.d_state + (n + i) * C::H1, dc1c);
        }
        if constexpr (C::H2 > 0) {
          load_vec<C::H2>(cy.d_state + 2 * n * C::H1 + i * C::H2, dh2c);
          load_vec<C::H2>(cy.d_state + 2 * n * C::H1 + (n + i) * C::H2, dc2c);
        }
        lam = cy.lam[i] + a.g_rec[(int64_t)T * n + i];
      }
    }

    for (int t = T - 1; t >= 0; --t) {
      // ---------------- phase A: forward recompute + out layer + layer-2 backward ----------------
      float u[C::F];
      float raw0 = 0.f, raw1 = 0.f;
      float h1n[cmax(C::H1, 1)];
      float dtop[C::TOP];     // gradient wrt the top vector coming from the output Linear
      float dh1_from2[cmax(C::H1, 1)];
      float y = 0.f, dy = 0.f;
      if (act) {
        if constexpr (C::NIN == 2) {
          raw0 = a.in_seq[((int64_t)t * 2) * n + i];
          raw1 = a.in_seq[((int64_t)t * 2 + 1) * n + i];
        } else {
          raw0 = a.in_seq[(int64_t)t * n + i];
        }
        preprocess<C>(sT, rt, raw0, raw1, u);
        const float* arena = a.ckpt + (int64_t)t * slot;
        const float* top = u;
        float h2n[cmax(C::H2, 1)];
        float act2[cmax(C::G2, 1)], c2p[cmax(C::H2, 1)], tc2[cmax(C::H2, 1)], h2p[cmax(C::H2, 1)];
        if constexpr (C::H1 > 0) {
          float act1[C::G1], c1p[C::H1], c1[C::H1], tc1[C::H1], h1p[C::H1];
          load_vec<C::H1>(arena + i * C::H1, h1p);
          load_vec<C::H1>(arena + (n + i) * C::H1, c1p);
#pragma unroll
          for (int k = 0; k < C::H1; ++k) c1[k] = c1p[k];
          gate_preact<C::F, C::H1>(sT + C::O_W1, sT + C::O_B1, u, h1p, act1);
          lstm_pointwise<C::H1>(act1, c1, h1n, tc1);
          top = h1n;
          if constexpr (C::H2 > 0) {  // park layer-1 values in this thread's smem scratch row
            stage_row<C::G1>(mySCR, act1);
#pragma unroll
            for (int k = 0; k < C::H1; ++k) { mySCR[C::G1 + k] = c1p[k]; mySCR[C::G1 + C::H1 + k] = tc1[k]; }
          } else {
            // single layer: finish here (needs act1/c1p/tc1 live)
            y = sT[C::O_BO];
#pragma unroll
            for (int k = 0; k < C::H1; ++k) y = fmaf(h1n[k], sT[C::O_WO + k], y);
            const float th = rt.tanh_output ? tanh_acc(y) : y;
            const float delta = th * rt.scale;
            const float dd = a.g_rec ? lam : (delta - a.labels[(int64_t)t * n + i]) / (float)a.n_total;
            dy = rt.scale * dd * (rt.tanh_output ? (1.0f - th * th) : 1.0f);
            float dh1[C::H1];
#pragma unroll
            for (int k = 0; k < C::H1; ++k) dh1[k] = fmaf(sT[C::O_WO + k], dy, dh1c[k]);
            lstm_pointwise_bwd<C::H1>(act1, c1p, tc1, dh1, dc1c);
            // stage IN = [u, h1p, 1], DZ = dz1
            float inrow[B::INS];
#pragma unroll
            for (int k = 0; k < B::INS; ++k)
              inrow[k] = k < C::F ? u[k < C::F ? k : 0]
                                  : (k < C::K1 ? h1p[(k >= C::F && k < C::K1) ? k - C::F : 0] : (k == C::K1 ? 1.f : 0.f));
            stage_row<B::INS>(myIN, inrow);
            float dzrow[B::DZS];
#pragma unroll
            for (int k = 0; k < B::DZS; ++k) dzrow[k] = k < C::G1 ? act1[k < C::G1 ? k : 0] : 0.f;
            stage_row<B::DZS>(myDZ, dzrow);
            matvec_wt<C::G1, C::F, C::H1>(sT + C::O_W1, act1, dh1c);
            // out layer staging
            float orow[B::INO];
#pragma unroll
            for (int k = 0; k < B::INO; ++k) orow[k] = k < C::H1 ? h1n[k < C::H1 ? k : 0] : (k == C::H1 ? 1.f : 0.f);
            stage_row<B::INO>(myINO, orow);
            *reinterpret_cast<float4*>(myDZO) = make_float4(dy, 0.f, 0.f, 0.f);
          }
        }
        if constexpr (C::H2 > 0) {
          float c2[C::H2];
          const float* b2 = arena + 2 * n * C::H1;
          load_vec<C::H2>(b2 + i * C::H2, h2p);
          load_vec<C::H2>(b2 + (n + i) * C::H2, c2p);
#pragma unroll
          for (int k = 0; k < C::H2; ++k) c2[k] = c2p[k];
          gate_preact<C::H1, C::H2>(sT + C::O_W2, sT + C::O_B2, h1n, h2p, act2);
          lstm_pointwise<C::H2>(act2, c2, h2n, tc2);
          y = sT[C::O_BO];
#pragma unroll
          for (int k = 0; k < C::H2; ++k) y = fmaf(h2n[k], sT[C::O_WO + k], y);
          const float th = rt.tanh_output ? tanh_acc(y) : y;
          const float delta = th * rt.scale;
          const float dd = a.g_rec ? lam : (delta - a.labels[(int64_t)t * n + i]) / (float)a.n_total;
          dy = rt.scale * dd * (rt.tanh_output ? (1.0f - th * th) : 1.0f);
          float dh2[C::H2];
#pragma unroll
          for (int k = 0; k < C::H2; ++k) dh2[k] = fmaf(sT[C::O_WO + k], dy, dh2c[k]);
          lstm_pointwise_bwd<C::H2>(act2, c2p, tc2, dh2, dc2c);
          float inrow[B::INS];
#pragma unroll
          for (int k = 0; k < B::INS; ++k)
            inrow[k] = k < C::H1 ? h1n[k < C::H1 ? k : 0]
                                 : (k < C::K2 ? h2p[(k >= C::H1 && k < C::K2) ? k - C::H1 : 0] : (k == C::K2 ? 1.f : 0.f));
          stage_row<B::INS>(myIN, inrow);
          float dzrow[B::DZS];
#pragma unroll
          for (int k = 0; k < B::DZS; ++k) dzrow[k] = k < C::G2 ? act2[k < C::G2 ? k : 0] : 0.f;
          stage_row<B::DZS>(myDZ, dzrow);
          matvec_wt<C::G2, 0, C::H1>(sT + C::O_W2, act2, dh1_from2);
          matvec_wt<C::G2, C::H1, C::H2>(sT + C::O_W2, act2, dh2c);
          float orow[B::INO];
#pragma unroll
          for (int k = 0; k < B::INO; ++k) orow[k] = k < C::H2 ? h2n[k < C::H2 ? k : 0] : (k == C::H2 ? 1.f : 0.f);
          stage_row<B::INO>(myINO, orow);
          *reinterpret_cast<float4*>(myDZO) = make_float4(dy, 0.f, 0.f, 0.f);
        }
        if constexpr (C::H1 == 0) {  // layers=(): Linear acts on the preprocessed input directly
          y = sT[C::O_BO];
#pragma unroll
          for (int k = 0; k < C::F; ++k) y = fmaf(u[k], sT[C::O_WO + k], y);
          const float th = rt.tanh_output ? tanh_acc(y) : y;
          const float delta = th * rt.scale;
          const float dd = a.g_rec ? lam : (delta - a.labels[(int64_t)t * n + i]) / (float)a.n_total;
          dy = rt.scale * dd * (rt.tanh_output ? (1.0f - th * th) : 1.0f);
          float orow[B::INO];
#pragma unroll
          for (int k = 0; k < B::INO; ++k) orow[k] = k < C::F ? u[k < C::F ? k : 0] : (k == C::F ? 1.f : 0.f);
          stage_row<B::INO>(myINO, orow);
          *reinterpret_cast<float4*>(myDZO) = make_float4(dy, 0.f, 0.f, 0.f);
        }
        (void)top; (void)dtop;
        // a segment hands sum_{tau > t0} on: g_t0 is the previous segment's last row
        if (a.g_rec && (!CARRY || t > 0)) lam += a.g_rec[(int64_t)t * n + i];
      } else {
        float zrow[B::INS];
#pragma unroll
        for (int k = 0; k < B::INS; ++k) zrow[k] = 0.f;
        stage_row<B::INS>(myIN, zrow);
        float zd[B::DZS];
#pragma unroll
        for (int k = 0; k < B::DZS; ++k) zd[k] = 0.f;
        stage_row<B::DZS>(myDZ, zd);
        float zo[B::INO];
#pragma unroll
        for (int k = 0; k < B::INO; ++k) zo[k] = 0.f;
        stage_row<B::INO>(myINO, zo);
        *reinterpret_cast<float4*>(myDZO) = make_float4(0.f, 0.f, 0.f, 0.f);
      }
      __syncthreads();
      if constexpr (C::H2 > 0)
        dw_pass<B::KR2, cmax(C::G2, 4), B::INS, B::DZS>(sIN, sDZ, sACC + B::ACC2 * kTile, tid);
      else if constexpr (C::H1 > 0)
        dw_pass<B::KR1, cmax(C::G1, 4), B::INS, B::DZS>(sIN, sDZ, sACC + B::ACC1 * kTile, tid);
      dw_pass<B::KRO, 1, B::INO, B::DZO>(sINO, sDZO, sACC + B::ACCO * kTile, tid);
      __syncthreads();
      // ---------------- phase B (two-layer nets): layer-1 backward ----------------
      if constexpr (C::H2 > 0) {
        if (act) {
          float act1[C::G1], c1p[C::H1], tc1[C::H1], h1p[C::H1];
          load_vec<C::G1>(mySCR, act1);
#pragma unroll
          for (int k = 0; k < C::H1; ++k) { c1p[k] = mySCR[C::G1 + k]; tc1[k] = mySCR[C::G1 + C::H1 + k]; }
          float dh1[C::H1];
#pragma unroll
          for (int k = 0; k < C::H1; ++k) dh1[k] = dh1_from2[k] + dh1c[k];
          lstm_pointwise_bwd<C::H1>(act1, c1p, tc1, dh1, dc1c);
          load_vec<C::H1>(a.ckpt + (int64_t)t * slot + i * C::H1, h1p);
          float inrow[B::INS];
#pragma unroll
          for (int k = 0; k < B::INS; ++k)
            inrow[k] = k < C::F ? u[k < C::F ? k : 0]
                                : (k < C::K1 ? h1p[(k >= C::F && k < C::K1) ? k - C::F : 0] : (k == C::K1 ? 1.f : 0.f));
          stage_row<B::INS>(myIN, inrow);
          float dzrow[B::DZS];
#pragma unroll
          for (int k = 0; k < B::DZS; ++k) dzrow[k] = k < C::G1 ? act1[k < C::G1 ? k : 0] : 0.f;
          stage_row<B::DZS>(myDZ, dzrow);
          matvec_wt<C::G1, C::F, C::H1>(sT + C::O_W1, act1, dh1c);
          if constexpr (C::FC) {
            float du[C::F];
            matvec_wt<C::G1, 0, C::F>(sT + C::O_W1, act1, du);
            float darow[B::DZF];
#pragma unroll
            for (int k = 0; k < B::DZF; ++k) {
              // elu'(a) = 1 (a > 0) else exp(a) = u + 1
              const float uk = u[k < C::F ? k : 0];
              darow[k] = k < C::F ? du[k < C::F ? k : 0] * (uk > 0.f ? 1.0f : uk + 1.0f) : 0.f;
            }
            stage_row<B::DZF>(myDZF, darow);
            float frow[B::INF];
#pragma unroll
            for (int k = 0; k < B::INF; ++k) frow[k] = k == 0 ? raw0 : (k == 1 && C::NIN == 2 ? raw1 : (k == C::NIN ? 1.f : 0.f));
            stage_row<B::INF>(myINF, frow);
          }
        } else {
          float zrow[B::INS];
#pragma unroll
          for (int k = 0; k < B::INS; ++k) zrow[k] = 0.f;
          stage_row<B::INS>(myIN, zrow);
          float zd[B::DZS];
#pragma unroll
          for (int k = 0; k < B::DZS; ++k) zd[k] = 0.f;
          stage_row<B::DZS>(myDZ, zd);
          if constexpr (C::FC) {
            float zf[B::DZF];
#pragma unroll
            for (int k = 0; k < B::DZF; ++k) zf[k] = 0.f;
            stage_row<B::DZF>(myDZF, zf);
            float zi[B::INF];
#pragma unroll
            for (int k = 0; k < B::INF; ++k) zi[k] = 0.f;
            stage_row<B::INF>(myINF, zi);
          }
        }
        __syncthreads();
        dw_pass<B::KR1, cmax(C::G1, 4), B::INS, B::DZS>(sIN, sDZ, sACC + B::ACC1 * kTile, tid);
        if constexpr (C::FC) dw_pass<B::KRF, cmax(C::F, 4), B::INF, B::DZF>(sINF, sDZF, sACC + B::ACCF * kTile, tid);
        __syncthreads();
      }
    }
    if constexpr (CARRY) {
      if (act) {
        if constexpr (C::H1 > 0) {
          store_vec<C::H1>(cy.d_state + i * C::H1, dh1c);
          store_vec<C::H1>(cy.d_state + (n + i) * C::H1, dc1c);
        }
        if constexpr (C::H2 > 0) {
          store_vec<C::H2>(cy.d_state + 2 * n * C::H1 + i * C::H2, dh2c);
          store_vec<C::H2>(cy.d_state + 2 * n * C::H1 + (n + i) * C::H2, dc2c);
        }
        cy.lam[i] = lam;
      }
    }
  }
  // flush the CTA's accumulators
  if constexpr (C::H1 > 0) dw_flush<B::KR1, cmax(C::G1, 4)>(sACC + B::ACC1 * kTile, a.dtheta, C::O_W1, C::O_B1, tid);
  if constexpr (C::H2 > 0) dw_flush<B::KR2, cmax(C::G2, 4)>(sACC + B::ACC2 * kTile, a.dtheta, C::O_W2, C::O_B2, tid);
  dw_flush<B::KRO, 1>(sACC + B::ACCO * kTile, a.dtheta, C::O_WO, C::O_BO, tid);
  if constexpr (C::FC) dw_flush<B::KRF, cmax(C::F, 4)>(sACC + B::ACCF * kTile, a.dtheta, C::O_WIN, C::O_BIN, tid);
}

}  // namespace l2o
