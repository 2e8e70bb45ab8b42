// Shared device code of the coordinate-wise LSTM engine: compile-time net configuration, flat
// theta offsets, activation / preprocessing math.  Semantics follow the reference
// (DM/ = Model_Free_L2O/L2O-DM and L2O-RNNProp/): DM/networks.py:207-232 (net), DM/preprocess.py:52-70
// (LogAndSign), DM/meta_rnnprop_train.py:383-388 (Adam features), Sonnet-1.11 snt.LSTM (gate order
// i|j|f|o, forget bias +1.0, state (hidden, cell)).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "l2o_b200.h"

namespace l2o {

template <int PRE_, int NIN_, int F_, int H1_, int H2_>
struct Cfg {
  static constexpr int PRE = PRE_, NIN = NIN_, F = F_, H1 = H1_, H2 = H2_;
  static constexpr int G1 = 4 * H1, G2 = 4 * H2;
  static constexpr int K1 = F + H1;   // rows of lstm_1/w_gates
  static constexpr int K2 = H1 + H2;  // rows of lstm_2/w_gates
  static constexpr int TOP = H2 > 0 ? H2 : (H1 > 0 ? H1 : F);
  static constexpr bool FC = (PRE == L2O_PRE_FC);
  // flat theta offsets (Sonnet creation order, DM/networks.py:47-62)
  static constexpr int O_WIN = 0;
  static constexpr int O_BIN = O_WIN + (FC ? NIN * F : 0);
  static constexpr int O_W1 = O_BIN + (FC ? F : 0);
  static constexpr int O_B1 = O_W1 + (H1 > 0 ? K1 * G1 : 0);
  static constexpr int O_W2 = O_B1 + G1;
  static constexpr int O_B2 = O_W2 + (H2 > 0 ? K2 * G2 : 0);
  static constexpr int O_WO = O_B2 + G2;
  static constexpr int O_BO = O_WO + TOP;
  static constexpr int P = O_BO + 1;
  static constexpr int SF = 2 * (H1 + H2);  // state floats per coordinate
};

__host__ __device__ constexpr int cmax(int a, int b) { return a > b ? a : b; }

struct NetRt {  // run-time scalars of the net
  float scale;
  float logsign_k;
  float logsign_ek;  // (float)exp((double)k)   DM/preprocess.py:67
  int tanh_output;
};

// ---- activations: accurate fp32 (parity bar is 1e-5 relative against the CPU oracle) ----------
__device__ __forceinline__ float sigmoid_acc(float x) { return __frcp_rn(1.0f + expf(-x)); }
__device__ __forceinline__ float tanh_acc(float x) { return tanhf(x); }
__device__ __forceinline__ float elu_acc(float a) { return a > 0.f ? a : expm1f(a); }

// ---- fast activations for the tensor-core engine: branch-free, 2 MUFU each (ex2.approx 2^-22 rel, rcp.approx 1 ulp);
// measured against the oracle the end-to-end error stays ~1e-6 (tests/test_tc_gpu.py) -----------------------------
__device__ __forceinline__ float ex2_approx(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rcp_approx(float x) {
  float y;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sigmoid_fast(float x) { return rcp_approx(1.0f + ex2_approx(-1.4426950408889634f * x)); }
__device__ __forceinline__ float tanh_fast(float x) {
  return fmaf(2.0f, rcp_approx(1.0f + ex2_approx(-2.8853900817779268f * x)), -1.0f);
}

// DM/preprocess.py:63-68
__device__ __forceinline__ void log_and_sign(float g, float k, float ek, float& lo, float& sg) {
  lo = fmaxf(logf(fabsf(g) + 1.1920929e-7f) / k, -1.0f);
  sg = fminf(fmaxf(g * ek, -1.0f), 1.0f);
}

// DM/meta_rnnprop_train.py:383-388
__device__ __forceinline__ void adam_features(float g, float& m, float& v, float beta1, float beta2, float p,
                                              float& mt, float& gt) {
  m = beta1 * m + (1.0f - beta1) * g;
  v = beta2 * v + (1.0f - beta2) * g * g;
  const float mh = m / (1.0f - powf(beta1, p));
  const float vh = v / (1.0f - powf(beta2, p));
  const float den = sqrtf(vh) + 1e-8f;
  mt = mh / den;
  gt = g / den;
}

// In-kernel separable optimizees (include/l2o_b200.h L2O_OPT_*).
__device__ __forceinline__ void optimizee_eval(int kind, float x, float a, float b, float alpha, float fscale,
                                               float& f, float& g) {
  if (kind == L2O_OPT_RASTRIGIN_SEP) {
    const float two_pi = 6.2831855f;
    float s, c;
    sincosf(two_pi * x, &s, &c);
    const float d = x - a;
    f = fscale * (0.5f * d * d - alpha * b * c + alpha);
    g = fscale * (d + (two_pi * alpha) * b * s);
  } else {  // L2O_OPT_QUADRATIC_DIAG
    const float r = a * x - b;
    f = fscale * (r * r);
    g = fscale * (2.0f * a * r);
  }
}

__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

}  // namespace l2o
