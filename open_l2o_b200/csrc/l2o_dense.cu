// Row-wise dense LSTM optimizer net with RUN-TIME shapes: StandardDeepLSTM with output_size > 1, i.e. the reference's
// KernelDeepLSTM (DM/networks.py:303-351): a convolution kernel [kw, kh, cin, cout] is viewed as R = cin*cout rows of
// K = kw*kh inputs (tf.transpose(inputs, [2,3,0,1]) -> reshape [-1, K]), one LSTM stack runs per ROW, the output
// Linear has K columns and the result is transposed back.  With the variable flat in its own [kw,kh,cin,cout] order,
// element (k, r) sits at k*R + r, so the "transpose" is strided indexing and every access is coalesced over rows.
//
// Shapes are run-time (any kernel_shape / layers the reference's tests use: (1,), (1,1), (5,), (20,20); K up to 64),
// thread = row, weights read through the read-only cache (warp-uniform addresses).  This is the compatibility path of
// SURVEY.md 8(f) row 3 - correctness first; the coordinate-wise nets are where the tuned kernels are.
// Semantics: DM/networks.py:207-232 (net), DM/preprocess.py:52-70, Sonnet-1.11 snt.LSTM / Linear; backward = SURVEY.md
// Appendix B with a vector-valued output.
#include <cuda_runtime.h>

#include <cmath>
#include <new>

#include "l2o_internal.h"

struct l2o_dense {
  l2o_dense_desc d;
  int F;          // features after preprocessing
  int64_t P;      // theta count
  int SF;         // state floats per row
  int o_w[2], o_b[2], o_wo, o_bo, top;
};

namespace {
constexpr int kMaxF = 128, kMaxH = 32, kMaxO = 64, kRows = 128;

struct Shape {
  int L, H[2], K, F, O, pre, tanh_out;
  float k, ek, scale;
  int o_w[2], o_b[2], o_wo, o_bo, top;
};

__device__ __forceinline__ void preprocess_row(const Shape& s, const float* __restrict__ in, int64_t R, int64_t r, float* u) {
  for (int k = 0; k < s.K; ++k) {
    const float g = in[(int64_t)k * R + r];
    if (s.pre == L2O_PRE_LOGSIGN) l2o::log_and_sign(g, s.k, s.ek, u[2 * k], u[2 * k + 1]);
    else u[k] = g;
  }
}

// one LSTM layer forward for one row: z (activated gates i|j|f|o), c -> c', h -> h'
__device__ __forceinline__ void lstm_fwd(const float* __restrict__ W, const float* __restrict__ B, int kin, int H,
                                         const float* in, const float* hprev, const float* cprev, float* gates, float* cn,
                                         float* hn, float* tc) {
  const int G = 4 * H;
  for (int n = 0; n < G; ++n) gates[n] = __ldg(B + n);
  for (int k = 0; k < kin + H; ++k) {
    const float a = k < kin ? in[k] : hprev[k - kin];
    const float* row = W + (int64_t)k * G;
    for (int n = 0; n < G; ++n) gates[n] = fmaf(a, __ldg(row + n), gates[n]);
  }
  for (int u = 0; u < H; ++u) {
    const float i = l2o::sigmoid_acc(gates[u]), j = l2o::tanh_acc(gates[H + u]);
    const float f = l2o::sigmoid_acc(gates[2 * H + u] + 1.0f), o = l2o::sigmoid_acc(gates[3 * H + u]);
    gates[u] = i; gates[H + u] = j; gates[2 * H + u] = f; gates[3 * H + u] = o;
    const float c = fmaf(f, cprev[u], i * j);
    const float t = l2o::tanh_acc(c);
    cn[u] = c;
    hn[u] = t * o;
    if (tc) tc[u] = t;
  }
}

__global__ void __launch_bounds__(kRows) dense_step_kernel(Shape s, l2o_dense_step_args a) {
  const int64_t R = a.rows;
  const int64_t r = (int64_t)blockIdx.x * kRows + threadIdx.x;
  if (r >= R) return;
  float u[kMaxF], gates[4 * kMaxH], h0[kMaxH], c0[kMaxH], hn[kMaxH], cn[kMaxH], top[kMaxF];
  preprocess_row(s, a.in, R, r, u);
  const float* cur = u;
  int kin = s.F;
  int64_t off = 0;
  for (int l = 0; l < s.L; ++l) {
    const int H = s.H[l];
    for (int k = 0; k < H; ++k) { h0[k] = a.state_in[off + r * H + k]; c0[k] = a.state_in[off + (R + r) * H + k]; }
    lstm_fwd(a.theta + s.o_w[l], a.theta + s.o_b[l], kin, H, cur, h0, c0, gates, cn, hn, nullptr);
    for (int k = 0; k < H; ++k) { a.state_out[off + r * H + k] = hn[k]; a.state_out[off + (R + r) * H + k] = cn[k]; top[k] = hn[k]; }
    cur = top;
    kin = H;
    off += 2 * R * H;
  }
  for (int o = 0; o < s.O; ++o) {
    float y = __ldg(a.theta + s.o_bo + o);
    for (int k = 0; k < s.top; ++k) y = fmaf(cur[k], __ldg(a.theta + s.o_wo + k * s.O + o), y);
    const float d = s.tanh_out ? l2o::tanh_acc(y) * s.scale : y * s.scale;
    if (a.delta) a.delta[(int64_t)o * R + r] = d;
    if (a.x) a.x[(int64_t)o * R + r] += d;
  }
}

// warp-reduced accumulation into the CTA's shared dtheta image
__device__ __forceinline__ void acc(float* sD, int idx, float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(sD + idx, v);
}

__global__ void __launch_bounds__(kRows) dense_bwd_kernel(Shape s, l2o_dense_bwd_args a, int P) {
  extern __shared__ float sD[];   // [P] per-CTA dtheta
  for (int k = threadIdx.x; k < P; k += kRows) sD[k] = 0.f;
  __syncthreads();
  const int64_t R = a.rows;
  const int64_t r = (int64_t)blockIdx.x * kRows + threadIdx.x;
  const bool act = r < R;
  const int64_t rr = act ? r : 0;
  int64_t slot = 0;
  for (int l = 0; l < s.L; ++l) slot += 2 * R * s.H[l];
  float u[kMaxF], g1[4 * kMaxH], g2[4 * kMaxH], hp[2][kMaxH], cp[2][kMaxH], hn[2][kMaxH], tcs[2][kMaxH];
  float dh[2][kMaxH], dc[2][kMaxH], lam[kMaxO], dy[kMaxO], din[kMaxF + kMaxH];
  for (int l = 0; l < 2; ++l)
    for (int k = 0; k < kMaxH; ++k) { dh[l][k] = 0.f; dc[l][k] = 0.f; }
  for (int o = 0; o < s.O; ++o) lam[o] = (act && a.g_rec) ? a.g_rec[((int64_t)a.T * s.O + o) * R + rr] : 0.f;
  const float inv_nt = a.labels ? 1.0f / (float)a.n_total : 0.f;
  for (int t = a.T - 1; t >= 0; --t) {
    // ---- forward recompute from checkpoint slot t ----------------------------------------------------------------------
    preprocess_row(s, a.in_seq + (int64_t)t * s.K * R, R, rr, u);
    const float* ck = a.ckpt + (int64_t)t * slot;
    const float* cur = u;
    int kin = s.F;
    int64_t off = 0;
    for (int l = 0; l < s.L; ++l) {
      const int H = s.H[l];
      for (int k = 0; k < H; ++k) { hp[l][k] = ck[off + rr * H + k]; cp[l][k] = ck[off + (R + rr) * H + k]; }
      float cn[kMaxH];
      lstm_fwd(a.theta + s.o_w[l], a.theta + s.o_b[l], kin, H, cur, hp[l], cp[l], l == 0 ? g1 : g2, cn, hn[l], tcs[l]);
      cur = hn[l];
      kin = H;
      off += 2 * R * H;
    }
    // ---- output layer ---------------------------------------------------------------------------------------------------
    for (int o = 0; o < s.O; ++o) {
      float y = __ldg(a.theta + s.o_bo + o);
      for (int k = 0; k < s.top; ++k) y = fmaf(cur[k], __ldg(a.theta + s.o_wo + k * s.O + o), y);
      const float th = s.tanh_out ? l2o::tanh_acc(y) : y;
      const float dd = a.g_rec ? lam[o] : (th * s.scale - a.labels[((int64_t)t * s.O + o) * R + rr]) * inv_nt;
      dy[o] = act ? s.scale * dd * (s.tanh_out ? 1.0f - th * th : 1.0f) : 0.f;
      acc(sD, s.o_bo + o, dy[o]);
      for (int k = 0; k < s.top; ++k) acc(sD, s.o_wo + k * s.O + o, cur[k] * dy[o]);
    }
    // gradient wrt the top vector
    float dtop[kMaxF];
    for (int k = 0; k < s.top; ++k) {
      float v = 0.f;
      for (int o = 0; o < s.O; ++o) v = fmaf(__ldg(a.theta + s.o_wo + k * s.O + o), dy[o], v);
      dtop[k] = v;
    }
    // ---- LSTM layers, top down -------------------------------------------------------------------------------------------
    for (int l = s.L - 1; l >= 0; --l) {
      const int H = s.H[l], G = 4 * H;
      float* g = l == 0 ? g1 : g2;
      const float* in = l == 0 ? u : hn[l - 1];
      const int kl = l == 0 ? s.F : s.H[l - 1];
      for (int k = 0; k < H; ++k) {
        const float dhk = dtop[k] + dh[l][k];
        const float i = g[k], j = g[H + k], f = g[2 * H + k], o = g[3 * H + k], tc = tcs[l][k];
        const float dcv = fmaf(dhk * o, 1.0f - tc * tc, dc[l][k]);
        g[k] = act ? dcv * j * i * (1.0f - i) : 0.f;
        g[H + k] = act ? dcv * i * (1.0f - j * j) : 0.f;
        g[2 * H + k] = act ? dcv * cp[l][k] * f * (1.0f - f) : 0.f;
        g[3 * H + k] = act ? dhk * tc * o * (1.0f - o) : 0.f;
        dc[l][k] = dcv * f;
      }
      const float* W = a.theta + s.o_w[l];
      for (int n = 0; n < G; ++n) acc(sD, s.o_b[l] + n, g[n]);
      for (int k = 0; k < kl + H; ++k) {
        const float av = k < kl ? in[k] : hp[l][k - kl];
        float v = 0.f;
        for (int n = 0; n < G; ++n) {
          acc(sD, s.o_w[l] + k * G + n, av * g[n]);
          v = fmaf(__ldg(W + (int64_t)k * G + n), g[n], v);
        }
        din[k] = v;
      }
      for (int k = 0; k < H; ++k) dh[l][k] = din[kl + k];      // carry to step t-1
      for (int k = 0; k < kl; ++k) dtop[k] = din[k];           // to the layer below (unused for l == 0)
    }
    if (s.L == 0) { /* Linear on the preprocessed input only: nothing recurrent */ }
    if (a.g_rec)
      for (int o = 0; o < s.O; ++o) lam[o] += act ? a.g_rec[((int64_t)t * s.O + o) * R + rr] : 0.f;
  }
  __syncthreads();
  for (int k = threadIdx.x; k < P; k += kRows) atomicAdd(&a.dtheta[k], (double)sD[k]);
}

Shape make_shape(const l2o_dense* h) {
  Shape s{};
  s.L = h->d.n_layers; s.H[0] = h->d.hidden[0]; s.H[1] = h->d.hidden[1];
  s.K = h->d.n_in; s.F = h->F; s.O = h->d.n_out; s.pre = h->d.preprocess; s.tanh_out = h->d.tanh_output;
  s.k = h->d.logsign_k; s.ek = (float)std::exp((double)h->d.logsign_k); s.scale = h->d.scale;
  s.o_w[0] = h->o_w[0]; s.o_w[1] = h->o_w[1]; s.o_b[0] = h->o_b[0]; s.o_b[1] = h->o_b[1];
  s.o_wo = h->o_wo; s.o_bo = h->o_bo; s.top = h->top;
  return s;
}
}  // namespace

extern "C" {

int l2o_dense_create(l2o_dense_handle* out, const l2o_dense_desc* d) {
  if (!out || !d || d->n_layers < 0 || d->n_layers > 2 || d->n_in < 1 || d->n_out < 1) return L2O_E_INVALID;
  if (d->preprocess != L2O_PRE_IDENTITY && d->preprocess != L2O_PRE_LOGSIGN) return L2O_E_UNSUPPORTED;
  const int F = d->preprocess == L2O_PRE_LOGSIGN ? 2 * d->n_in : d->n_in;
  if (F > kMaxF || d->n_out > kMaxO) return L2O_E_UNSUPPORTED;
  for (int l = 0; l < d->n_layers; ++l)
    if (d->hidden[l] < 1 || d->hidden[l] > kMaxH) return L2O_E_UNSUPPORTED;
  l2o_dense* h = new (std::nothrow) l2o_dense();
  if (!h) return L2O_E_NOMEM;
  h->d = *d;
  h->F = F;
  int off = 0, kin = F;
  h->SF = 0;
  for (int l = 0; l < 2; ++l) { h->o_w[l] = 0; h->o_b[l] = 0; }
  for (int l = 0; l < d->n_layers; ++l) {
    const int H = d->hidden[l];
    h->o_w[l] = off; off += (kin + H) * 4 * H;
    h->o_b[l] = off; off += 4 * H;
    kin = H;
    h->SF += 2 * H;
  }
  h->top = kin;
  h->o_wo = off; off += kin * d->n_out;
  h->o_bo = off; off += d->n_out;
  h->P = off;
  *out = h;
  return L2O_OK;
}
void l2o_dense_destroy(l2o_dense_handle h) { delete h; }
int64_t l2o_dense_theta_count(l2o_dense_handle h) { return h ? h->P : L2O_E_INVALID; }
int64_t l2o_dense_state_floats(l2o_dense_handle h) { return h ? h->SF : L2O_E_INVALID; }

int l2o_dense_step(l2o_dense_handle h, const l2o_dense_step_args* a, void* stream) {
  if (!h || !a || a->rows < 0 || !a->theta || !a->in) return L2O_E_INVALID;
  if (h->SF > 0 && (!a->state_in || !a->state_out)) return L2O_E_INVALID;
  if (a->rows == 0) return L2O_OK;
  dense_step_kernel<<<(int)((a->rows + kRows - 1) / kRows), kRows, 0, (cudaStream_t)stream>>>(make_shape(h), *a);
  return l2o::after_launch("l2o_dense_step");
}

int l2o_dense_unroll_bwd(l2o_dense_handle h, const l2o_dense_bwd_args* a, void* stream) {
  if (!h || !a || a->rows < 0 || a->T < 0 || !a->theta || !a->dtheta) return L2O_E_INVALID;
  if (a->T > 0 && !a->in_seq) return L2O_E_INVALID;
  if (h->SF > 0 && !a->ckpt) return L2O_E_INVALID;
  if (!a->g_rec && (!a->labels || a->n_total <= 0)) return L2O_E_INVALID;
  if (a->rows == 0 || a->T == 0) return L2O_OK;
  const size_t smem = (size_t)h->P * sizeof(float);
  if (smem > 200 * 1024) return L2O_E_UNSUPPORTED;
  if (int rc = l2o::raise_smem_limit("l2o_dense_unroll_bwd", dense_bwd_kernel, smem)) return rc;
  dense_bwd_kernel<<<(int)((a->rows + kRows - 1) / kRows), kRows, smem, (cudaStream_t)stream>>>(make_shape(h), *a, (int)h->P);
  return l2o::after_launch("l2o_dense_unroll_bwd");
}

}  // extern "C"
