// L2O-Scale CoordinatewiseRNN update step and its backward — sm_90a CUDA kernels + C-ABI.
// SC/ = Model_Free_L2O/L2O-Scale/L2O-Scale-Training/ of the reference; CR = SC/optimizer/coordinatewise_rnn.py.
//
// The optimizer is fully coordinate-wise (no per-tensor or global reduction), so one step over all optimizee tensors is
// ONE launch over the concatenated coordinates:
//   ms'    = (1-d)(g^2 + 1e-12) + d ms                         (SC/optimizer/utils.py:108-134, d = OLD decay state)
//   s      = asinh(g / sqrt(ms' + 1e-16))                        (utils.py:31-33,137-160)
//   h3     = LSTM(20)(LSTM(20)(LSTM(10)(s)))                     (CR:80-83,205-207; TF LSTMCell, forget bias 1.0)
//   delta  = h3 Wu ; decay' = sigmoid(h3 Wd + bd) ; lr' = 2 sigmoid(h3 Wl + bl) lr     (CR:209-223)
//   x'     = x - lr' delta                                       (CR:226,240)
// The reference's "decay := 0 if ALL(ms == 0) over the tensor" (utils.py:129-130) is not evaluated: ms starts at 1
// (CR:169) and ms' >= min(d ms, (1-d) 1e-12) > 0, so the predicate is false in every state this optimizer produces.
//
// State: 103 fp32 planes of [N] (SoA, every access coalesced): 0..99 the "rnn" slot packed as the reference packs it
// (CR:306-315), c1 h1 c2 h2 c3 h3 — c BEFORE h; 100 rms; 101 decay; 102 learning_rate.
// theta: 6402 fp32 in TF variable creation order (open_l2o_b200/coordinatewise_rnn.py THETA_SPEC).
//
// Activations: sigmoid as ex2.approx + rcp.approx (relative error ~1e-7 everywhere); tanh as libdevice tanhf, because
// the same two-MUFU form of tanh has ~1e-7 ABSOLUTE error near 0, and a hidden unit whose |c'| stays small then misses
// 1e-5 relative parity.
//
// Engine: exact-fp32 FFMA, one thread per coordinate.  The cell weights are staged once per CTA in shared memory as a
// gate-interleaved image: element (k, u) is the float4 (W[k][i_u], W[k][j_u], W[k][f_u], W[k][o_u]), so one broadcast
// LDS.128 feeds the four FFMAs of one input row of one unit.
#include <cstdint>

#include "l2o_internal.h"

namespace l2o {
namespace crnn {

constexpr int H1 = 10, H2 = 20, H3 = 20;
constexpr int P_C1 = 0, P_H1 = 10, P_C2 = 20, P_H2 = 40, P_C3 = 60, P_H3 = 80, P_RMS = 100, P_DECAY = 101, P_LR = 102;
constexpr int kPlanes = 103;
// flat theta offsets (TF creation order: __init__ CR:90-102, then the cells on the first call CR:206)
constexpr int O_WU = 0, O_WD = 20, O_BD = 40, O_WL = 41, O_BL = 61, O_INIT = 62;
constexpr int O_K1 = 162, O_K2 = 642, O_K3 = 3122;   // cell_l kernel [KIN+H][4H] followed by its bias [4H]
constexpr int kTheta = 6402;
constexpr int kRo = 62;                              // readout block theta[0..62)
// shared weight image offsets (float4 units): layer l holds (KIN+H+1) x H entries, the bias row last
constexpr int S1 = 0, S2 = S1 + (1 + H1 + 1) * H1, S3 = S2 + (H1 + H2 + 1) * H2, kImgF4 = S3 + (H2 + H3 + 1) * H3;
static_assert(O_K2 == O_K1 + (1 + H1 + 1) * 4 * H1 && O_K3 == O_K2 + (H1 + H2 + 1) * 4 * H2 &&
                  kTheta == O_K3 + (H2 + H3 + 1) * 4 * H3, "theta layout");

constexpr int kFwdBlock = 64;
constexpr int kBwdBlock = 128;   // = coordinates per backward tile
constexpr int XS = 44;           // backward tile row strides (floats): x rows <= 41 (+pad), dz rows 80 (+pad);
constexpr int ZS = 84;           // 44 and 84 make the per-thread float4 row writes bank-conflict-free
constexpr int HS = 53, DS = 21;  // scratch row strides (odd: conflict-free scalar access)
constexpr int R_S = 0, R_H1 = 1, R_H2 = R_H1 + H1, R_H3 = R_H2 + H2;

struct StepArgs {
  int64_t n;
  const float* theta;
  const float* g;
  const float* state_in;
  float* state_out;
  float* x;
  float* update;
};

struct BwdArgs {
  int64_t n;
  const float* theta;
  const float* g;
  const float* state_old;
  const float* d_state_new;
  const float* d_update;
  float* d_state_old;
  double* d_theta;
  float* d_g;   // [n] or null
};

__device__ __forceinline__ float dsig(float s) { return s * (1.0f - s); }
// the reference's asinh, log(v + sqrt(1 + v^2)) (utils.py:31-33), evaluated as written, with its cancellation for v << 0
__device__ __forceinline__ float asinh_ref(float v) { return logf(v + sqrtf(__fadd_rn(1.0f, __fmul_rn(v, v)))); }

// theta -> gate-interleaved shared image of the three cells, plus the readout block
__device__ __forceinline__ void stage_weights(const float* __restrict__ theta, float4* sW, float* sRo) {
  auto stage = [&](int so, int to, int rows, int H) {
    for (int e = threadIdx.x; e < rows * H; e += blockDim.x) {
      const int k = e / H, u = e - k * H;
      const float* r = theta + to + k * 4 * H + u;
      sW[so + e] = make_float4(r[0], r[H], r[2 * H], r[3 * H]);
    }
  };
  stage(S1, O_K1, 1 + H1 + 1, H1);
  stage(S2, O_K2, H1 + H2 + 1, H2);
  stage(S3, O_K3, H2 + H3 + 1, H3);
  for (int e = threadIdx.x; e < kRo; e += blockDim.x) sRo[e] = theta[e];
}

// Weight-image read.  The image is invariant across the coordinate loop, so plain loads get hoisted out of it into
// registers (25 KB of them) and spill; a volatile load stays where the FFMAs use it.
__device__ __forceinline__ float4 lds4(const float4* p) {
  float4 v;
  asm volatile("ld.shared.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
               : "r"((unsigned)__cvta_generic_to_shared(p)));
  return v;
}

// gate pre-activations (i, j, f, o) of unit u for the input row x = [inp | h].  The weight rows are read in chunks of
// kChunk, and each chunk's address goes through an empty asm that consumes the running sums: ptxas cannot issue a
// chunk's loads before the previous chunk's FFMAs, so at most kChunk float4 are in flight (instead of all K of them,
// which needs > 200 registers at K = 40).
constexpr int kChunk = 8;
template <int K, int H>
__device__ __forceinline__ float4 gates(const float4* W, const float (&x)[K], int u) {
  float4 z = lds4(W + K * H + u);
#pragma unroll
  for (int k0 = 0; k0 < K; k0 += kChunk) {
    const float4* Wc = W + k0 * H + u;
    asm volatile("" : "+l"(Wc) : "f"(z.x), "f"(z.y), "f"(z.z), "f"(z.w));
#pragma unroll
    for (int k = k0; k < (k0 + kChunk < K ? k0 + kChunk : K); ++k) {
      const float4 w = lds4(Wc + (k - k0) * H);
      z.x = fmaf(x[k], w.x, z.x);
      z.y = fmaf(x[k], w.y, z.y);
      z.z = fmaf(x[k], w.z, z.z);
      z.w = fmaf(x[k], w.w, z.w);
    }
  }
  return z;
}

// ms' = (1-d)(g^2 + 1e-12) + d ms, every operation rounded on its own as the reference's graph does (no FMA
// contraction); q = g^2 + 1e-12
__device__ __forceinline__ float ms_update(float g, float d, float ms, float& q) {
  q = __fadd_rn(__fmul_rn(g, g), 1e-12f);
  return __fadd_rn(__fmul_rn(__fsub_rn(1.0f, d), q), __fmul_rn(d, ms));
}

// TF LSTMCell (forget bias 1.0) for one coordinate: x = [inp | h_PH], c_PC read from `in`; c', h' written to `out` and
// h' returned in hn.  Each plane element is loaded before the same thread stores it, so `out` may be `in` (in place).
template <int KIN, int H, int PC, int PH>
__device__ __forceinline__ void cell_fwd(const float4* W, const float* inp, const float* __restrict__ in,
                                         float* __restrict__ out, int64_t n, int64_t i, float (&hn)[H]) {
  float x[KIN + H], c[H];
#pragma unroll
  for (int k = 0; k < KIN; ++k) x[k] = inp[k];
#pragma unroll
  for (int k = 0; k < H; ++k) {
    x[KIN + k] = in[(PH + k) * n + i];
    c[k] = in[(PC + k) * n + i];
  }
#pragma unroll
  for (int u = 0; u < H; ++u) {
    const float4 z = gates<KIN + H, H>(W, x, u);
    const float cn = sigmoid_fast(z.z + 1.0f) * c[u] + sigmoid_fast(z.x) * tanh_acc(z.y);
    hn[u] = sigmoid_fast(z.w) * tanh_acc(cn);
    out[(PC + u) * n + i] = cn;
    out[(PH + u) * n + i] = hn[u];
  }
}

// ------------------------------------------------------------------------------------------------------------------
// forward step: thread = coordinate; every state byte read once and written once (836 B per coordinate with x)
__global__ void __launch_bounds__(kFwdBlock) step_kernel(StepArgs a) {
  __shared__ float4 sW[kImgF4];
  __shared__ float sRo[kRo];
  stage_weights(a.theta, sW, sRo);
  __syncthreads();
  const int64_t n = a.n;
  const float* __restrict__ in = a.state_in;
  float* __restrict__ out = a.state_out;
  for (int64_t i = (int64_t)blockIdx.x * kFwdBlock + threadIdx.x; i < n; i += (int64_t)gridDim.x * kFwdBlock) {
    const float g = a.g[i];
    const float ms = in[P_RMS * n + i], d = in[P_DECAY * n + i], lr = in[P_LR * n + i];
    float q;
    const float msn = ms_update(g, d, ms, q);
    const float s = asinh_ref(g / sqrtf(msn + 1e-16f));
    float h1n[H1], h2n[H2], h3n[H3];
    cell_fwd<1, H1, P_C1, P_H1>(sW + S1, &s, in, out, n, i, h1n);
    cell_fwd<H1, H2, P_C2, P_H2>(sW + S2, h1n, in, out, n, i, h2n);
    cell_fwd<H2, H3, P_C3, P_H3>(sW + S3, h2n, in, out, n, i, h3n);
    float delta = 0.f, zd = sRo[O_BD], zl = sRo[O_BL];
#pragma unroll
    for (int k = 0; k < H3; ++k) {
      delta = fmaf(h3n[k], sRo[O_WU + k], delta);
      zd = fmaf(h3n[k], sRo[O_WD + k], zd);
      zl = fmaf(h3n[k], sRo[O_WL + k], zl);
    }
    const float lrn = 2.0f * sigmoid_fast(zl) * lr;
    const float upd = lrn * delta;
    out[P_RMS * n + i] = msn;
    out[P_DECAY * n + i] = sigmoid_fast(zd);
    out[P_LR * n + i] = lrn;
    if (a.x) a.x[i] -= upd;
    if (a.update) a.update[i] = upd;
  }
}

// ------------------------------------------------------------------------------------------------------------------
// backward: recompute the step from the old planes and g, then walk it backwards (readouts, LSTM 3 -> 1, asinh and the
// ms chain).  g enters through ms' and v = g / sqrt(ms' + 1e-16) only, so with a non-null d_g the kernel also writes
// d g = dv / sqrt(ms' + 1e-16) + dms' (1 - d) 2g (second-order meta-gradients).  d theta of each cell is the tile contraction X^T dZ over the CTA's 128 coordinates (X = [inp | h | 1] rows,
// dZ = gate adjoints), done from shared memory into a per-CTA image of d theta that is flushed once per CTA with fp64
// atomics; the readout weights go through warp sums into the same image.
struct BwdSmem {
  float4 W[kImgF4];
  float ro[kRo + 2];
  float img[kTheta + 2];        // d theta, flat theta order
  float4 X[kBwdBlock * XS / 4];
  float4 Z[kBwdBlock * ZS / 4];
  float H[kBwdBlock * HS];      // per-thread scratch rows: s | h1' | h2' | h3'
  float D[kBwdBlock * DS];      // per-thread adjoint handed from one cell to the one below
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The backward keeps each coordinate's h' of the recompute and the adjoint handed from one cell to the next in the
// thread's shared scratch rows, and runs the unit loops rolled: fully unrolled, the independent units get interleaved
// by the scheduler and the kernel spills at 255 registers.

// x = [inp | h_old] from the thread's row of the X tile: [x | 1 | 0 pad] (the backward keeps x there, not in registers)
template <int KIN, int H>
__device__ __forceinline__ void store_xrow(float4* xrow, const float* inp, const float* h, int64_t n, int64_t i, bool act) {
  constexpr int K = KIN + H;
#pragma unroll
  for (int q = 0; q < (K + 4) / 4; ++q) {
    float v[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      const int k = 4 * q + r;
      v[r] = k < KIN ? inp[k] : k < K ? (act ? h[(k - KIN) * n + i] : 0.f) : (k == K ? 1.0f : 0.0f);
    }
    xrow[q] = make_float4(v[0], v[1], v[2], v[3]);
  }
}
template <int K, int H>
__device__ __forceinline__ float4 gates_row(const float4* W, const float4* xrow, int u) {
  float4 z = lds4(W + K * H + u);
#pragma unroll
  for (int q = 0; q < (K + 3) / 4; ++q) {
    const float4 xv = xrow[q];
    const float xs[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
    for (int r = 0; r < 4; ++r) {
      if (4 * q + r < K) {
        const float4 w = lds4(W + (4 * q + r) * H + u);
        z.x = fmaf(xs[r], w.x, z.x);
        z.y = fmaf(xs[r], w.y, z.y);
        z.z = fmaf(xs[r], w.z, z.z);
        z.w = fmaf(xs[r], w.w, z.w);
      }
    }
  }
  return z;
}

// one cell's forward recompute from the old planes: h' to hn (c' is not needed outside the cell)
template <int KIN, int H, int PC, int PH>
__device__ __forceinline__ void cell_recompute(const float4* W, const float* inp, const float* st, int64_t n, int64_t i,
                                               bool act, float4* xrow, float* hn) {
  store_xrow<KIN, H>(xrow, inp, st + PH * n, n, i, act);
#pragma unroll 1
  for (int u = 0; u < H; ++u) {
    const float4 z = gates_row<KIN + H, H>(W, xrow, u);
    const float c = act ? st[(PC + u) * n + i] : 0.f;
    const float cn = sigmoid_fast(z.z + 1.0f) * c + sigmoid_fast(z.x) * tanh_acc(z.y);
    hn[u] = sigmoid_fast(z.w) * tanh_acc(cn);
  }
}

// one cell's backward.  dh: in, the adjoint of h' from above (the d_state_new plane is added here); out, the adjoint
// of the cell input in dh[0..KIN).  Writes the old c / h adjoints and the thread's X and dZ rows of the tile.
template <int KIN, int H, int PC, int PH>
__device__ __forceinline__ void cell_bwd(const float4* W, const float* inp, float* dh, const BwdArgs& a, int64_t i,
                                         bool act, float4* xrow, float4* zrow) {
  constexpr int K = KIN + H;
  const int64_t n = a.n;
  store_xrow<KIN, H>(xrow, inp, a.state_old + PH * n, n, i, act);
#pragma unroll 1
  for (int u = 0; u < H; ++u) {
    const float4 z = gates_row<K, H>(W, xrow, u);
    const float c = act ? a.state_old[(PC + u) * n + i] : 0.f;
    const float dhu = dh[u] + (act ? a.d_state_new[(PH + u) * n + i] : 0.f);
    const float dcu = act ? a.d_state_new[(PC + u) * n + i] : 0.f;
    const float si = sigmoid_fast(z.x), tj = tanh_acc(z.y), sf = sigmoid_fast(z.z + 1.0f), so = sigmoid_fast(z.w);
    const float cn = sf * c + si * tj;
    const float tc = tanh_acc(cn);
    const float dcn = dcu + dhu * so * (1.0f - tc * tc);
    zrow[u] = make_float4(dcn * tj * dsig(si), dcn * si * (1.0f - tj * tj), dcn * c * dsig(sf), dhu * tc * dsig(so));
    if (act) a.d_state_old[(PC + u) * n + i] = dcn * sf;
  }
  // dx = W dz from the thread's own dZ row
  float dx[K];
#pragma unroll
  for (int k = 0; k < K; ++k) dx[k] = 0.f;
#pragma unroll 1
  for (int u = 0; u < H; ++u) {
    const float4 dz = zrow[u];
#pragma unroll
    for (int k = 0; k < K; ++k) {
      const float4 w = lds4(W + k * H + u);
      dx[k] = fmaf(w.x, dz.x, fmaf(w.y, dz.y, fmaf(w.z, dz.z, fmaf(w.w, dz.w, dx[k]))));
    }
  }
  if (act) {
#pragma unroll
    for (int k = 0; k < H; ++k) a.d_state_old[(PH + k) * n + i] = dx[KIN + k];
  }
#pragma unroll
  for (int k = 0; k < KIN; ++k) dh[k] = dx[k];
}

// img[k][g*H + u] += sum_t X[t][k] dZ[t][4u + g] over the tile; thread block = RK rows x 8 columns (two units)
template <int K1, int H, int RK>
__device__ __forceinline__ void contract(const BwdSmem& S, float* img) {
  constexpr int NKB = (K1 + RK - 1) / RK, NCB = H / 2;
  for (int b = threadIdx.x; b < NKB * NCB; b += kBwdBlock) {
    const int kb = b / NCB, cb = b - kb * NCB;
    float acc[RK][8];
#pragma unroll
    for (int r = 0; r < RK; ++r)
#pragma unroll
      for (int q = 0; q < 8; ++q) acc[r][q] = 0.f;
    const float* X = reinterpret_cast<const float*>(S.X);
#pragma unroll 4
    for (int t = 0; t < kBwdBlock; ++t) {
      const float4 z0 = S.Z[t * (ZS / 4) + 2 * cb], z1 = S.Z[t * (ZS / 4) + 2 * cb + 1];
      const float zz[8] = {z0.x, z0.y, z0.z, z0.w, z1.x, z1.y, z1.z, z1.w};
#pragma unroll
      for (int r = 0; r < RK; ++r) {
        const float xv = X[t * XS + kb * RK + r];
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[r][q] = fmaf(xv, zz[q], acc[r][q]);
      }
    }
#pragma unroll
    for (int r = 0; r < RK; ++r) {
      const int k = kb * RK + r;
      if (k < K1) {
#pragma unroll
        for (int q = 0; q < 8; ++q) {
          const int u = 2 * cb + q / 4, g = q % 4;
          img[k * 4 * H + g * H + u] += acc[r][q];
        }
      }
    }
  }
}

__global__ void __launch_bounds__(kBwdBlock, 1) bwd_kernel(BwdArgs a) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  BwdSmem& S = *reinterpret_cast<BwdSmem*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31;
  stage_weights(a.theta, S.W, S.ro);
  for (int e = tid; e < kTheta; e += kBwdBlock) S.img[e] = 0.f;
  __syncthreads();
  const int64_t n = a.n;
  const int64_t ntiles = (n + kBwdBlock - 1) / kBwdBlock;
  float4* xrow = S.X + tid * (XS / 4);
  float4* zrow = S.Z + tid * (ZS / 4);
  float* hr = S.H + tid * HS;
  float* dr = S.D + tid * DS;
  auto add_img = [&](int slot, float v) {
    v = warp_sum(v);
    if (lane == 0) atomicAdd(&S.img[slot], v);
  };
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int64_t i = tile * kBwdBlock + tid;
    const bool act = i < n;
    const float* so = a.state_old;
    // ---------------------------------------------------------------- forward recompute
    const float g = act ? a.g[i] : 0.f;
    const float ms = act ? so[P_RMS * n + i] : 0.f, d = act ? so[P_DECAY * n + i] : 0.f, lr = act ? so[P_LR * n + i] : 0.f;
    float q;
    const float msn = ms_update(g, d, ms, q);
    const float v = g / sqrtf(msn + 1e-16f);
    hr[R_S] = asinh_ref(v);
    cell_recompute<1, H1, P_C1, P_H1>(S.W + S1, hr + R_S, so, n, i, act, xrow, hr + R_H1);
    cell_recompute<H1, H2, P_C2, P_H2>(S.W + S2, hr + R_H1, so, n, i, act, xrow, hr + R_H2);
    cell_recompute<H2, H3, P_C3, P_H3>(S.W + S3, hr + R_H2, so, n, i, act, xrow, hr + R_H3);
    float delta = 0.f, zd = S.ro[O_BD], zl = S.ro[O_BL];
#pragma unroll
    for (int k = 0; k < H3; ++k) {
      delta = fmaf(hr[R_H3 + k], S.ro[O_WU + k], delta);
      zd = fmaf(hr[R_H3 + k], S.ro[O_WD + k], zd);
      zl = fmaf(hr[R_H3 + k], S.ro[O_WL + k], zl);
    }
    const float sd = sigmoid_fast(zd), sl = sigmoid_fast(zl);
    const float lrn = 2.0f * sl * lr;
    // ---------------------------------------------------------------- readouts
    const float dupd = act ? a.d_update[i] : 0.f;
    const float dlrn = (act ? a.d_state_new[P_LR * n + i] : 0.f) + dupd * delta;
    const float ddelta = dupd * lrn;
    const float dzl = dlrn * 2.0f * lr * dsig(sl);
    const float dlr = dlrn * 2.0f * sl;
    const float dzd = (act ? a.d_state_new[P_DECAY * n + i] : 0.f) * dsig(sd);
#pragma unroll 1
    for (int k = 0; k < H3; ++k) {
      const float h = hr[R_H3 + k];
      dr[k] = ddelta * S.ro[O_WU + k] + dzd * S.ro[O_WD + k] + dzl * S.ro[O_WL + k];
      add_img(O_WU + k, ddelta * h);
      add_img(O_WD + k, dzd * h);
      add_img(O_WL + k, dzl * h);
    }
    add_img(O_BD, dzd);
    add_img(O_BL, dzl);
    // ---------------------------------------------------------------- cells, top to bottom
    cell_bwd<H2, H3, P_C3, P_H3>(S.W + S3, hr + R_H2, dr, a, i, act, xrow, zrow);
    __syncthreads();
    contract<H2 + H3 + 1, H3, 4>(S, S.img + O_K3);
    __syncthreads();
    cell_bwd<H1, H2, P_C2, P_H2>(S.W + S2, hr + R_H1, dr, a, i, act, xrow, zrow);
    __syncthreads();
    contract<H1 + H2 + 1, H2, 4>(S, S.img + O_K2);
    __syncthreads();
    cell_bwd<1, H1, P_C1, P_H1>(S.W + S1, hr + R_S, dr, a, i, act, xrow, zrow);
    __syncthreads();
    contract<1 + H1 + 1, H1, 2>(S, S.img + O_K1);
    __syncthreads();
    // ---------------------------------------------------------------- asinh and the ms chain (and d g when asked)
    const float dv = dr[0] * rsqrtf(fmaf(v, v, 1.0f));
    const float dmsn = (act ? a.d_state_new[P_RMS * n + i] : 0.f) - 0.5f * dv * v / (msn + 1e-16f);
    if (act) {
      a.d_state_old[P_RMS * n + i] = dmsn * d;
      a.d_state_old[P_DECAY * n + i] = dmsn * (ms - q);
      a.d_state_old[P_LR * n + i] = dlr;
      if (a.d_g) a.d_g[i] = dv / sqrtf(msn + 1e-16f) + dmsn * (1.0f - d) * 2.0f * g;
    }
  }
  __syncthreads();
  for (int e = tid; e < kTheta; e += kBwdBlock)
    if (e < O_INIT || e >= O_K1) atomicAdd(&a.d_theta[e], (double)S.img[e]);
}

}  // namespace crnn
}  // namespace l2o

using namespace l2o::crnn;

extern "C" {

int64_t l2o_crnn_theta_count(void) { return kTheta; }
int64_t l2o_crnn_state_floats(void) { return kPlanes; }

int l2o_crnn_step(const l2o_crnn_step_args* a, void* stream) {
  if (!a || a->n <= 0 || a->n > INT64_MAX / kPlanes || !a->theta || !a->g || !a->state_in || !a->state_out)
    return L2O_E_INVALID;
  const void* fp[] = {a->theta, a->g, a->state_in, a->state_out, a->x, a->update};
  for (const void* p : fp)
    if (l2o::misaligned(p, alignof(float))) return L2O_E_INVALID;
  StepArgs k{a->n, a->theta, a->g, a->state_in, a->state_out, a->x, a->update};
  return l2o::occupancy_launch("l2o_crnn_step", step_kernel, kFwdBlock, 0, a->n, (cudaStream_t)stream, k);
}

int l2o_crnn_bwd(const l2o_crnn_bwd_args* a, void* stream) {
  if (!a || a->n <= 0 || a->n > INT64_MAX / kPlanes || !a->theta || !a->g || !a->state_old || !a->d_state_new ||
      !a->d_update || !a->d_state_old || !a->d_theta)
    return L2O_E_INVALID;
  const void* fp[] = {a->theta, a->g, a->state_old, a->d_state_new, a->d_update, a->d_state_old};
  for (const void* p : fp)
    if (l2o::misaligned(p, alignof(float))) return L2O_E_INVALID;
  if (l2o::misaligned(a->d_theta, alignof(double))) return L2O_E_INVALID;
  if (a->d_g) {
    if (l2o::misaligned(a->d_g, alignof(float))) return L2O_E_INVALID;
    const size_t n = (size_t)a->n, f = sizeof(float);
    const void* other[] = {a->theta, a->g, a->state_old, a->d_state_new, a->d_update, a->d_state_old, a->d_theta};
    const size_t bytes[] = {kTheta * f, n * f, kPlanes * n * f, kPlanes * n * f, n * f, kPlanes * n * f,
                            kTheta * sizeof(double)};
    if (l2o::overlaps_any(a->d_g, n * f, other, bytes, 7)) return L2O_E_INVALID;
  }
  BwdArgs k{a->n, a->theta, a->g, a->state_old, a->d_state_new, a->d_update, a->d_state_old, a->d_theta, a->d_g};
  return l2o::occupancy_launch("l2o_crnn_bwd", bwd_kernel, kBwdBlock, sizeof(BwdSmem), a->n, (cudaStream_t)stream, k);
}

}  // extern "C"
