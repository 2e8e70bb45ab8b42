// Tensor-core engine (sm_90a): the [coords x K] x [K x 4H] gate contractions of the LSTM-20x2 on Hopper's warpgroup
// MMA (wgmma), forward unroll / single step.  The BPTT kernel (cwlstm_tc_bwd.cuh) shares the operand layout below.
//
// Design (DESIGN.md "tensor-core engine"):
//  * A warpgroup (128 threads) owns a tile of 64 coordinates = the M of one wgmma.  Thread (warp w, lane l) holds the
//    coordinates 16w + l/4 and 16w + l/4 + 8 (the rows of its accumulator fragment); the four threads of a quad
//    (q = l % 4) split the hidden units: thread q owns units [5q, 5q + 5) of both layers.
//  * A operand = the coordinate's [features | 1 | h1 | h2] row, kept IN REGISTERS as wgmma A fragments (register-A
//    mode): fragment column c belongs to thread c % 4, so a 20-vector starting at column `base` stores unit 5q + s at
//    column base + 4s + q.  The thread that produced h' writes it straight into its own fragment registers; the
//    recurrent state never touches shared or global memory between unroll steps, the cell state c stays in registers.
//  * B operand = gate weights in shared memory (K-major, no swizzle, 8x16-byte core matrices), staged once per CTA
//    with one TMA bulk copy (cp.async.bulk + mbarrier) of a pre-arranged image.  Gate column order: unit 5q + s has
//    its (i, j) pre-activations in accumulator columns 16s + 2q + {0, 1} and (f, o) in 16s + 8 + 2q + {0, 1}, i.e. in
//    the accumulator registers of the thread that owns the unit.
//  * fp32 parity on tf32 tensor cores: error-compensated 3xTF32 -- A = Ah + Al, B = Bh + Bl; D = Al.Bh + Ah.Bl + Ah.Bh
//    accumulated in fp32.  Biases ride along as a constant-1 column of A.
//  * sigmoid / tanh / c / h / output linear / x += delta are fused in the epilogue; the output layer's partial sums
//    over the thread's 5 units are combined with two quad shuffles.
#pragma once
#include "cwlstm_common.cuh"
#include "l2o_internal.h"

namespace l2o {
namespace tc {

constexpr int kH = 20;
constexpr int kN = 4 * kH;        // 80 gate columns
constexpr int kTile = 64;         // coordinates per warpgroup tile (wgmma M)
constexpr int kU = 5;             // hidden units per thread
constexpr int kFwdWG = 3;         // warpgroups per forward CTA (they share the weight image)
constexpr int kFwdThreads = 128 * kFwdWG;
template <int N>
struct IC {
  static constexpr int value = N;
};

// Operand-row geometry.  LSTM-20x2 with <= 3 features (identity, LogAndSign): [f0..f(F-1), 1, 0.. | h1 | h2 | 0 0 0 0]
// = 48 columns, layer 1 contracts k-blocks 0..2 (columns 0..23), layer 2 k-blocks 0..5 (the feature columns meet zero
// rows, the constant 1 carries b2).  RNNProp (fc(2->20)+ELU, DM/networks.py:180-183,219): [u(20) | 1 0 0 0 | h1 | h2] =
// 64 columns, layer 1 contracts columns 0..47 (h2 units in 44..47 meet zero rows), layer 2 columns 16..63 (u in 16..19
// meet zero rows, the 1 at column 20 carries b2).  BPTT dX widths: 24 columns per 20-vector (slot 2j + e of thread q =
// accumulator column 8j + 2q + e, slot 5 is padding); dX2 = [dh1n | dh2p], dX1 = [dh1p] (+ [de] for fc nets).
template <class C>
struct Geo {
  static constexpr bool FC = C::FC;
  static constexpr int ColH1 = FC ? 24 : 4, ColH2 = FC ? 44 : 24;
  static constexpr int ColOne = FC ? 20 : C::F;
  static constexpr int KB = FC ? 8 : 6;                        // k-blocks of 8 columns in the operand row
  static constexpr int L1Lo = 0, L1Hi = FC ? 6 : 3;           // layer-1 k-blocks [L1Lo, L1Hi)
  static constexpr int L2Lo = FC ? 2 : 0, L2Hi = KB;          // layer-2 k-blocks
  static constexpr int K1 = 8 * (L1Hi - L1Lo), K2 = 8 * (L2Hi - L2Lo);
  static constexpr int N1 = FC ? 48 : 24, N2 = 48;
  static constexpr int B1Floats = K1 * kN, B2Floats = K2 * kN, T1Floats = kN * N1, T2Floats = kN * N2;
  static constexpr int FwdFloats = 2 * (B1Floats + B2Floats);                 // B1h | B1l | B2h | B2l
  static constexpr int AllFloats = FwdFloats + 2 * (T1Floats + T2Floats);     // + T1h | T1l | T2h | T2l
  static_assert(!FC || C::F == 20, "fc preprocessing: dim 20");
  static_assert(FC || C::F <= 3, "feature chunk: at most 3 features");
};
constexpr int kImgMaxFloats = Geo<Cfg<L2O_PRE_FC, 2, 20, 20, 20>>::AllFloats;

// ------------------------------------------------------------------ PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void tma_bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
                   smem_u32(dst)),
               "l"(src), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// One thread stages `bytes` (multiple of 16, 16-byte aligned) of global memory into shared memory with the TMA engine;
// every thread of the CTA then waits on the barrier.  `bar` must have been initialised (count 1) and fenced.
__device__ __forceinline__ void stage_image(float* dst, const float* src, uint32_t bytes, uint64_t* bar) {
  if (threadIdx.x == 0) {
    mbar_expect_tx(bar, bytes);
    tma_bulk_g2s(dst, src, bytes, bar);
  }
  mbar_wait(bar, 0);
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// shared-memory matrix descriptor (wgmma), no swizzle: start >> 4 | LBO >> 4 << 16 | SBO >> 4 << 32
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo, uint32_t sbo) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo >> 4) << 16) | ((uint64_t)(sbo >> 4) << 32);
}
// descriptor of a K-major tf32 image with N columns (core matrices: 8 rows of N x 16 bytes of K; N-groups 128 B apart,
// K-chunks of 4 (N/8) * 128 B apart) and its start-address increment per K = 8 step (descriptor units of 16 B)
__device__ __forceinline__ uint64_t img_desc(const float* p, int ncols) {
  return make_desc(smem_u32(p), (uint32_t)(ncols / 8) * 128u, 128u);
}
__host__ __device__ constexpr uint64_t img_kstep(int ncols) { return (uint64_t)((2 * (ncols / 8) * 128) >> 4); }

#define L2O_ACC8(b) "+f"(d[b]), "+f"(d[b + 1]), "+f"(d[b + 2]), "+f"(d[b + 3]), "+f"(d[b + 4]), "+f"(d[b + 5]), \
                    "+f"(d[b + 6]), "+f"(d[b + 7])
// D[64 x 80] (+)= A[64 x 8] (registers, tf32) . B[8 x 80] (shared, tf32, K-major)
__device__ __forceinline__ void mma_rs_n80(float* d, const uint32_t* a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %45, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,"
      "%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, "
      "{%40,%41,%42,%43}, %44, p, 1, 1;\n\t}\n"
      : L2O_ACC8(0), L2O_ACC8(8), L2O_ACC8(16), L2O_ACC8(24), L2O_ACC8(32)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
}
// D[64 x 48] (+)= A[64 x 8] (registers) . B[8 x 48]
__device__ __forceinline__ void mma_rs_n48(float* d, const uint32_t* a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %29, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, "
      "{%24,%25,%26,%27}, %28, p, 1, 1;\n\t}\n"
      : L2O_ACC8(0), L2O_ACC8(8), L2O_ACC8(16)
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
}
// D[64 x 24] (+)= A[64 x 8] (registers) . B[8 x 24]
__device__ __forceinline__ void mma_rs_n24(float* d, const uint32_t* a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %17, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n24k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11}, "
      "{%12,%13,%14,%15}, %16, p, 1, 1;\n\t}\n"
      : L2O_ACC8(0), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
}
template <int N>
__device__ __forceinline__ void mma_rs(float* d, const uint32_t* a, uint64_t b, uint32_t acc) {
  static_assert(N == 80 || N == 48 || N == 24, "wgmma width");
  if constexpr (N == 80) mma_rs_n80(d, a, b, acc);
  else if constexpr (N == 48) mma_rs_n48(d, a, b, acc);
  else mma_rs_n24(d, a, b, acc);
}

__device__ __forceinline__ float to_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
// Error-compensated operand split for 3xTF32: hi = x truncated to tf32 (sign, 8 exponent, 10 mantissa bits), lo = the
// exact remainder (|lo| < 2^-10 |x|; its own truncation leaves a 2^-21 relative residual).  hi + lo == x exactly.
__device__ __forceinline__ void split_tf32(float x, uint32_t& hi, uint32_t& lo) {
  hi = __float_as_uint(x) & 0xFFFFE000u;
  lo = __float_as_uint(x - __uint_as_float(hi));
}

// ------------------------------------------------------------------ operand / accumulator maps
// 20-vector slot s of thread q at column base + 4s + q  <->  unit 5q + s
__host__ __device__ constexpr int vec_unit(int c, int base) { return 5 * ((c - base) & 3) + ((c - base) >> 2); }
__host__ __device__ constexpr int unit_col(int u, int base) { return base + 4 * (u % 5) + u / 5; }
// MMA gate column n -> reference gate column (gate * 20 + unit, snt.LSTM i|j|f|o blocks)
__host__ __device__ constexpr int gate_ref_col(int n) {
  return (2 * ((n >> 3) & 1) + (n & 1)) * kH + 5 * ((n & 7) >> 1) + (n >> 4);
}
// physical K index of the dX contractions -> MMA gate column.  The dZ accumulators are reused as A fragments
// (k-block j: a0|a1 = accumulator column 8j + 2q, a2|a3 = 8j + 2q + 1), so physical k = 8j + p carries gate column
// 8j + 2 (p % 4) + p / 4.
__host__ __device__ constexpr int dx_gate_col(int k) { return (k & ~7) + 2 * (k & 3) + ((k >> 2) & 1); }
// dX output column -> (20-vector group, unit), unit -1 = padding slot
__host__ __device__ constexpr int dx_group(int c) { return c / 24; }
__host__ __device__ constexpr int dx_unit(int c) {
  return 2 * ((c % 24) >> 3) + (c & 1) >= 5 ? -1 : 5 * ((c & 7) >> 1) + 2 * ((c % 24) >> 3) + (c & 1);
}
// index of (k, n) in a K-major tf32 image with ncols columns
__host__ __device__ constexpr int img_index(int k, int n, int ncols) {
  return ((k >> 2) * (ncols / 8) + (n >> 3)) * 32 + (n & 7) * 4 + (k & 3);
}

// value of the extended weight matrix of layer `l2` at (operand-row column c, MMA gate column n)
template <class C>
__device__ __forceinline__ float ext_weight(const float* __restrict__ theta, bool l2, int c, int n) {
  using G = Geo<C>;
  const int col = gate_ref_col(n);
  if (c == G::ColOne) return theta[(l2 ? C::O_B2 : C::O_B1) + col];
  const bool in_h1 = c >= G::ColH1 && c < G::ColH1 + kH, in_h2 = c >= G::ColH2 && c < G::ColH2 + kH;
  if (!l2) {
    if (in_h1) return theta[C::O_W1 + (C::F + vec_unit(c, G::ColH1)) * C::G1 + col];
    if (G::FC && c < kH) return theta[C::O_W1 + vec_unit(c, 0) * C::G1 + col];
    if (!G::FC && c < C::F) return theta[C::O_W1 + c * C::G1 + col];
    return 0.f;
  }
  if (in_h1) return theta[C::O_W2 + vec_unit(c, G::ColH1) * C::G2 + col];
  if (in_h2) return theta[C::O_W2 + (kH + vec_unit(c, G::ColH2)) * C::G2 + col];
  return 0.f;
}
// Gate scales folded into the forward images B1 / B2: MMA gate column n delivers z' = -s_g (z + delta_g), the exponent
// of sigma(z) = 1 / (1 + 2^(-log2e z)) and tanh(z) = 2 / (1 + 2^(-2 log2e z)) - 1, so the epilogues feed the
// accumulators to ex2 without a multiply.  s_g = log2e for i, f, o and 2 log2e for j; delta_f = 1 is snt.LSTM's
// forget bias (delta = 0 for the other gates), added to the bias row.  The dX images T1 / T2 stay unscaled: dZ is the
// gradient with respect to the unscaled pre-activation z.
constexpr float kLog2e = 1.4426950408889634f;
__host__ __device__ constexpr float gate_scale(int gate) { return gate == 1 ? -2.f * kLog2e : -kLog2e; }
constexpr int kGateF = 2;
// sigma(z) and tanh(z) from the scaled pre-activations sigma: z' = -log2e z, tanh: z' = -2 log2e z
__device__ __forceinline__ float sigmoid_scaled(float zs) { return rcp_approx(1.0f + ex2_approx(zs)); }
__device__ __forceinline__ float tanh_scaled(float zs) { return fmaf(2.0f, rcp_approx(1.0f + ex2_approx(zs)), -1.0f); }

// operand-row column of dX output column c of layer l2
template <class C>
__host__ __device__ constexpr int dx_operand_col(bool l2, int c) {
  using G = Geo<C>;
  return l2 ? unit_col(dx_unit(c), dx_group(c) == 0 ? G::ColH1 : G::ColH2)
            : unit_col(dx_unit(c), dx_group(c) == 0 ? G::ColH1 : 0);
}

// Weight image: B1h | B1l | B2h | B2l (forward) and, with_transposed, T1h | T1l | T2h | T2l (BPTT dX contractions,
// K = 80 gates in the physical order of dx_gate_col, N = N1 / N2 dX columns).  B_l rows = operand-row columns
// 8 L_lLo .. 8 L_lHi - 1, scaled by gate_scale (each value rounded once in fp32, then split into hi + lo).
template <class C>
__global__ void prep_weights_kernel(const float* __restrict__ theta, float* __restrict__ img, int with_transposed) {
  static_assert(C::H1 == kH && C::H2 == kH && (C::F <= 3 || C::FC), "tc engine: LSTM-20x2, F <= 3 or fc(20)");
  using G = Geo<C>;
  const int nb = (G::K1 + G::K2) * kN;
  const int nt = with_transposed ? kN * (G::N1 + G::N2) : 0;
  for (int e = blockIdx.x * blockDim.x + threadIdx.x; e < nb + nt; e += gridDim.x * blockDim.x) {
    float w;
    float* hi;
    int off, idx;
    if (e < nb) {
      const bool l2 = e >= G::K1 * kN;
      const int ee = l2 ? e - G::K1 * kN : e;
      const int k = ee / kN, n = ee % kN;
      const int c = 8 * (l2 ? G::L2Lo : G::L1Lo) + k, gate = gate_ref_col(n) / kH;
      w = ext_weight<C>(theta, l2, c, n);
      if (c == G::ColOne && gate == kGateF) w += 1.0f;
      w *= gate_scale(gate);
      hi = img + (l2 ? 2 * G::B1Floats : 0);
      off = l2 ? G::B2Floats : G::B1Floats;
      idx = img_index(k, n, kN);
    } else {
      const int e2 = e - nb;
      const bool l2 = e2 >= kN * G::N1;
      const int nc = l2 ? G::N2 : G::N1;
      const int ee = l2 ? e2 - kN * G::N1 : e2;
      const int k = ee / nc, n = ee % nc;
      w = dx_unit(n) < 0 ? 0.f : ext_weight<C>(theta, l2, dx_operand_col<C>(l2, n), dx_gate_col(k));
      hi = img + G::FwdFloats + (l2 ? 2 * G::T1Floats : 0);
      off = l2 ? G::T2Floats : G::T1Floats;
      idx = img_index(k, n, nc);
    }
    const float h = to_tf32(w);
    hi[idx] = h;
    hi[off + idx] = to_tf32(w - h);
  }
}

// ------------------------------------------------------------------ operand fragments
// Register-A fragments of one operand row: f[kb][hf * 2 + rh] = column 8 kb + 4 hf + q of row rh (rh 0: coordinate
// 16w + l/4, rh 1: + 8).
template <int KB>
struct Frag {
  uint32_t hi[KB][4], lo[KB][4];
  __device__ __forceinline__ void zero() {
#pragma unroll
    for (int k = 0; k < KB; ++k)
#pragma unroll
      for (int r = 0; r < 4; ++r) { hi[k][r] = 0u; lo[k][r] = 0u; }
  }
  // this thread's column of the 4-column group starting at column c (c % 4 == 0; a compile-time value after
  // unrolling, so the register index is static)
  __device__ __forceinline__ void put_at(int c, int rh, float v) {
    split_tf32(v, hi[c / 8][((c / 4) & 1) * 2 + rh], lo[c / 8][((c / 4) & 1) * 2 + rh]);
  }
  __device__ __forceinline__ float get_at(int c, int rh) const {   // hi + lo == the value put
    return __uint_as_float(hi[c / 8][((c / 4) & 1) * 2 + rh]) + __uint_as_float(lo[c / 8][((c / 4) & 1) * 2 + rh]);
  }
  template <int COL>
  __device__ __forceinline__ void put(int rh, float v) {
    static_assert(COL % 4 == 0 && COL / 8 < KB, "fragment column");
    put_at(COL, rh, v);
  }
  // the thread's 5 units of a 20-vector starting at column BASE
  template <int BASE>
  __device__ __forceinline__ void put_vec(int rh, const float* v) {
    static_assert(BASE % 4 == 0 && (BASE + 19) / 8 < KB, "fragment column");
#pragma unroll
    for (int s = 0; s < kU; ++s) put_at(BASE + 4 * s, rh, v[s]);
  }
};

// 3xTF32 contraction of k-blocks [LO, HI) of the operand row against a K-major image (hi at bh, lo at bl)
template <int N, int KB, int LO, int HI>
__device__ __forceinline__ void mma3(float* d, const Frag<KB>& f, uint64_t bh, uint64_t bl) {
  constexpr uint64_t step = img_kstep(N);
#pragma unroll
  for (int kb = LO; kb < HI; ++kb) {
    const uint64_t o = (uint64_t)(kb - LO) * step;
    mma_rs<N>(d, f.lo[kb], bh + o, kb > LO ? 1u : 0u);
    mma_rs<N>(d, f.hi[kb], bl + o, 1u);
    mma_rs<N>(d, f.hi[kb], bh + o, 1u);
  }
}

// accumulator register of (unit slot s, gate g in i|j|f|o, row rh)
__host__ __device__ constexpr int acc_idx(int s, int g, int rh) { return 4 * (2 * s + (g >> 1)) + 2 * rh + (g & 1); }

// ------------------------------------------------------------------ epilogue helpers
// One LSTM unit, pointwise, from the scaled pre-activations (i', j', f', o') of the unit (gate_scale: Ei = 2^i' etc.).
// 7 MUFU ops (5 ex2 + 2 rcp) instead of the 10 of five separate sigmoid/tanh evaluations: the whole cell update shares
// ONE reciprocal,
//   c' = sigma(f+1) c + sigma(i) tanh(j) = [c (1+Ei)(1+Ej) + (1-Ej)(1+Ef)] / [(1+Ei)(1+Ej)(1+Ef)],
// and tanh(c') sigma(o) = (1-Ec) / ((1+Ec)(1+Eo)) another.  The exponents are clamped to 2^40 so the triple product
// stays finite (sigma / tanh are saturated to 1e-12 there).
__device__ __forceinline__ void lstm_point_fwd(float zi, float zj, float zf, float zo, float& c, float& h) {
  const float Ei = ex2_approx(fminf(zi, 40.f));
  const float Ej = ex2_approx(fminf(zj, 40.f));
  const float Qf = 1.0f + ex2_approx(fminf(zf, 40.f));
  const float Pij = (1.0f + Ei) * (1.0f + Ej);
  const float cn = fmaf(c, Pij, (1.0f - Ej) * Qf) * rcp_approx(Pij * Qf);
  c = cn;
  const float Ec = ex2_approx(fminf(-2.f * kLog2e * cn, 63.f));
  const float Eo = ex2_approx(fminf(zo, 63.f));
  h = (1.0f - Ec) * rcp_approx((1.0f + Ec) * (1.0f + Eo));
}
// elu as the forward and backward kernels both evaluate it: a (a > 0) | expm1(a), with a short Taylor sum near zero
// where 2^x - 1 cancels
__device__ __forceinline__ float elu_fast(float av) {
  const float em = ex2_approx(kLog2e * av) - 1.0f;
  const float ep = av * fmaf(av, fmaf(av, fmaf(av, 1.0f / 24.0f, 1.0f / 6.0f), 0.5f), 1.0f);
  return av > 0.f ? av : (av > -0.0625f ? ep : em);
}

// the thread's 5 units of a [n][20] row-major array (p already points at the coordinate's row)
__device__ __forceinline__ void load5(const float* __restrict__ p, int q, float* v) {
#pragma unroll
  for (int s = 0; s < kU; ++s) v[s] = p[5 * q + s];
}
__device__ __forceinline__ void store5(float* __restrict__ p, int q, const float* v) {
#pragma unroll
  for (int s = 0; s < kU; ++s) p[5 * q + s] = v[s];
}
__device__ __forceinline__ float quad_sum(float v) {
  v += __shfl_xor_sync(0xffffffffu, v, 1);
  return v + __shfl_xor_sync(0xffffffffu, v, 2);
}
// value of row rh (0 | 1) from the quad thread that computed it (threads q = 0 / 1 of the quad; 2 / 3 duplicate them)
__device__ __forceinline__ float from_row(float v, int lane, int rh) {
  return __shfl_sync(0xffffffffu, v, (lane & ~3) | rh);
}

// internal (non-ABI) extras of a launch: RNNProp's bias-correction exponent p = float(step0 + t) may come from a
// DEVICE scalar (l2o_step_args::step_ptr, CUDA-graph friendly) or a fixed float (l2o_step_args::p)
struct FwdExtra {
  const int32_t* step_ptr;   // non-NULL: step0 = *step_ptr + t_offset
  int32_t t_offset;
  float p_fixed;             // used when > 0 and step_ptr == NULL (single step)
};

template <class C>
struct SmemF {
  float img[Geo<C>::FwdFloats];   // must stay first (16-byte aligned TMA destination)
  float wo[kH + 4];               // linear/w, linear/b
  float win[64];                  // fc nets: input_projection/w [2][20] then /b [20]
  uint64_t wbar;
};
// dynamic tail after SmemF<C>: (fc nets) Adam bias corrections [T][2] floats
template <class C>
__host__ __device__ constexpr size_t adamc_offset() {
  return (sizeof(SmemF<C>) + 15) & ~(size_t)15;
}
template <class C>
__host__ __device__ constexpr size_t fwd_smem_bytes(int T) {
  return adamc_offset<C>() + (C::FC ? (size_t)T * 2 * sizeof(float) : 0);
}
// fx partial sum of a warp whose lanes q = 2, 3 of every quad hold 0: warp_sum_d without its xor-2 level, which would
// only add those zeros
__device__ __forceinline__ double warp_sum_pairs_d(double v) {
  v += __shfl_xor_sync(0xffffffffu, v, 16);
  v += __shfl_xor_sync(0xffffffffu, v, 8);
  v += __shfl_xor_sync(0xffffffffu, v, 4);
  return v + __shfl_xor_sync(0xffffffffu, v, 1);
}

// ------------------------------------------------------------------ forward kernel
// Forward unroll of T steps (T = 1 with an out-of-place state_out: the l2o_step regime).  Per warpgroup tile: state
// rows in, then per step  features -> layer-1 MMAs -> layer-1 epilogue -> layer-2 MMAs -> layer-2 epilogue + output
// layer + parameter add.  The three warpgroups of a CTA run independent tiles, so one warpgroup's MMA round trip
// overlaps the others' epilogues.
//
// FAST (tc_fwd_fast: DM nets, n a multiple of 64, in-kernel optimizee, plain output layer, T >= 1, state in place) is
// the full-tile instantiation: no row tests, the optimizee kind OPT is a compile-time constant, CKPT says whether the
// checkpoints and g_rec are written (both or neither), and the tanh output, recorded deltas, imitation labels and Adam
// features are compiled out.  Its arithmetic is the general instantiation's, operation for operation.
template <class C, bool FAST = false, int OPT = L2O_OPT_NONE, bool CKPT = false>
__global__ void __launch_bounds__(kFwdThreads, 1) unroll_fwd_kernel(l2o_unroll_args a, NetRt rt, const float* __restrict__ img,
                                                                     float* __restrict__ state_out, FwdExtra ex) {
  static_assert(!FAST || (!C::FC && OPT != L2O_OPT_NONE), "the full-tile forward is the DM nets' with an optimizee");
  using G = Geo<C>;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  SmemF<C>& S = *reinterpret_cast<SmemF<C>*>(smem_raw);
  const int T = a.T;
  const int64_t n = a.n;
  const bool in_kernel_opt = FAST || a.opt_kind != L2O_OPT_NONE;
  const int opt_kind = FAST ? OPT : a.opt_kind;
  const bool want_fx = in_kernel_opt && a.fx != nullptr;
  const bool adam_mode = C::NIN == 2 && a.m != nullptr;   // fused RNNProp features (DM/meta_rnnprop_train.py:383-388)
  const bool has_ckpt = FAST ? CKPT : a.ckpt != nullptr;
  const bool has_grec = FAST ? CKPT : a.g_rec != nullptr;
  const bool tanh_out = !FAST && rt.tanh_output;
  const bool has_delta = !FAST && a.delta_seq != nullptr;
  const bool has_labels = !FAST && a.labels != nullptr;
  float* adamc = reinterpret_cast<float*>(smem_raw + adamc_offset<C>());

  if (threadIdx.x < kH) S.wo[threadIdx.x] = a.theta[C::O_WO + threadIdx.x];
  if (threadIdx.x == kH) S.wo[kH] = a.theta[C::O_BO];
  if constexpr (C::FC) {
    static_assert(!C::FC || C::NIN == 2, "fc nets here are RNNprop nets (two inputs)");
    if (threadIdx.x >= 32 && threadIdx.x < 92) S.win[threadIdx.x - 32] = a.theta[C::O_WIN + threadIdx.x - 32];
    if (adam_mode) {   // 1 - beta^p per step, p = float(step + t) (DM/meta_rnnprop_train.py:384,386)
      const int step0 = ex.step_ptr ? *ex.step_ptr + ex.t_offset : a.step0;
      for (int t = threadIdx.x; t < T; t += blockDim.x) {
        const float p = (ex.step_ptr == nullptr && ex.p_fixed > 0.f) ? ex.p_fixed : (float)(step0 + t);
        adamc[2 * t] = 1.0f - powf(a.beta1, p);
        adamc[2 * t + 1] = 1.0f - powf(a.beta2, p);
      }
    }
  }
  if (threadIdx.x == 0) {
    mbar_init(&S.wbar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  stage_image(S.img, img, G::FwdFloats * 4, &S.wbar);

  // the warpgroup index through lane 0, so the compiler can prove the tile indices warp-uniform
  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0), warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int g = lane >> 2, q = lane & 3, own = q & 1;
  const uint64_t b1h = img_desc(S.img, kN), b1l = img_desc(S.img + G::B1Floats, kN);
  const uint64_t b2h = img_desc(S.img + 2 * G::B1Floats, kN), b2l = img_desc(S.img + 2 * G::B1Floats + G::B2Floats, kN);
  const int64_t ntiles = (n + kTile - 1) / kTile;
  const int64_t slot = n * C::SF;
  const int64_t nk = n * kH;   // one [n][20] block of the state arena
  const float bo = S.wo[kH];
  float wo[kU];
#pragma unroll
  for (int s = 0; s < kU; ++s) wo[s] = S.wo[5 * q + s];
  double imit = 0.0;
  float d[kN / 2];   // gate accumulators (the first MMA of each layer overwrites them)
#pragma unroll
  for (int k = 0; k < kN / 2; ++k) d[k] = 0.f;

  for (int64_t tile = (int64_t)blockIdx.x * kFwdWG + wg; tile < ntiles; tile += (int64_t)gridDim.x * kFwdWG) {
    const int64_t r0 = tile * kTile + warp * 16 + g;
    const int64_t row[2] = {r0, r0 + 8};
    const bool act[2] = {FAST || row[0] < n, FAST || row[1] < n};
    const int64_t io = own ? row[1] : row[0];   // the row whose per-coordinate scalars this thread computes
    const bool oact = FAST || io < n;
    const bool writer = q < 2 && oact;
    // checkpoint rows of the thread's first coordinate (the second is 8 rows on) and its g_rec entry, stepped by one
    // slot / one row per step
    float* ck = has_ckpt ? a.ckpt + r0 * kH : nullptr;
    float* gr = has_grec ? a.g_rec + io : nullptr;
    Frag<G::KB> A;
    A.zero();
    float c1[2][kU], c2[2][kU];
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      float h1[kU] = {0.f, 0.f, 0.f, 0.f, 0.f}, h2[kU] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int s = 0; s < kU; ++s) { c1[rh][s] = 0.f; c2[rh][s] = 0.f; }
      if (act[rh]) {
        const int64_t i = row[rh];
        load5(a.state + i * kH, q, h1);
        load5(a.state + (n + i) * kH, q, c1[rh]);
        load5(a.state + 2 * n * kH + i * kH, q, h2);
        load5(a.state + 2 * n * kH + (n + i) * kH, q, c2[rh]);
        if (has_ckpt) {
          float* p = ck + rh * 8 * kH;
          store5(p, q, h1);
          store5(p + nk, q, c1[rh]);
          store5(p + 2 * nk, q, h2);
          store5(p + 3 * nk, q, c2[rh]);
        }
        if (!FAST && T == 0 && state_out != a.state) {
          store5(state_out + i * kH, q, h1);
          store5(state_out + (n + i) * kH, q, c1[rh]);
          store5(state_out + 2 * n * kH + i * kH, q, h2);
          store5(state_out + 2 * n * kH + (n + i) * kH, q, c2[rh]);
        }
      }
      A.template put_vec<G::ColH1>(rh, h1);
      A.template put_vec<G::ColH2>(rh, h2);
    }
    if constexpr (G::FC) {   // the constant 1 of the fc row; DM rows carry theirs in the feature chunk
      A.template put<G::ColOne>(0, q == 0 ? 1.0f : 0.f);
      A.template put<G::ColOne>(1, q == 0 ? 1.0f : 0.f);
    }
    float x = 0.f, oa = 0.f, ob = 0.f, am = 0.f, av = 0.f;
    if (oact) {
      if (FAST || a.x) x = a.x[io];
      if (in_kernel_opt) { oa = a.opt_a[io]; ob = a.opt_b[io]; }
      if (adam_mode) { am = a.m[io]; av = a.v[io]; }
    }

    for (int t = 0; t < T; ++t) {
      if (has_ckpt) ck += slot;   // slot t + 1
      // ---- gradient + preprocessing of the own row, then the feature columns of both rows -------------------------
      float fval = 0.f, raw0 = 0.f, raw1 = 0.f;
      if (oact) {
        if (in_kernel_opt) {
          optimizee_eval(opt_kind, x, oa, ob, a.opt_alpha, a.opt_fscale, fval, raw0);
          if (has_grec) {
            if (q < 2) *gr = raw0;
            gr += n;
          }
        } else if (C::NIN == 2 && !adam_mode) {   // operator surface: (m~, g~) given
          raw0 = a.in_seq[((int64_t)t * 2) * n + io];
          raw1 = a.in_seq[((int64_t)t * 2 + 1) * n + io];
        } else {
          raw0 = a.in_seq[(int64_t)t * n + io];
        }
      }
      if constexpr (G::FC) {
        if (adam_mode) {   // m' = b1 m + (1-b1) g ; v' = b2 v + (1-b2) g^2 ; m~ = m^/(sqrt(v^)+1e-8) ; g~ = g/(sqrt(v^)+1e-8)
          const float gg = raw0;
          am = a.beta1 * am + (1.0f - a.beta1) * gg;
          av = a.beta2 * av + (1.0f - a.beta2) * gg * gg;
          const float mh = am / adamc[2 * t], vh = av / adamc[2 * t + 1];
          const float den = sqrtf(vh) + 1e-8f;
          raw0 = mh / den;
          raw1 = gg / den;
        }
        if (writer && a.feat_rec) {
          a.feat_rec[((int64_t)t * 2) * n + io] = raw0;
          a.feat_rec[((int64_t)t * 2 + 1) * n + io] = raw1;
        }
        // u = elu([m~, g~] Win + bin) (DM/networks.py:219) for the thread's 5 fc outputs of both rows
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
          const float m0 = from_row(raw0, lane, rh), m1 = from_row(raw1, lane, rh);
          float u[kU];
#pragma unroll
          for (int s = 0; s < kU; ++s) {
            const int j = 5 * q + s;
            u[s] = elu_fast(fmaf(m1, S.win[kH + j], fmaf(m0, S.win[j], S.win[2 * kH + j])));
          }
          A.template put_vec<0>(rh, u);
        }
      } else {
        float f[C::F];
        preprocess<C>(nullptr, rt, raw0, raw1, f);
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
          float v = q == C::F ? 1.0f : 0.f;
#pragma unroll
          for (int k = 0; k < C::F; ++k) {
            const float fk = from_row(f[k], lane, rh);
            if (q == k) v = fk;
          }
          A.template put<0>(rh, v);
        }
      }
      if (want_fx) {
        // straight to global memory: a fire-and-forget reduction, where a shared-memory fp64 atomicAdd is a
        // compare-and-swap loop that the warps of the CTA contend for every step
        const double ws = warp_sum_pairs_d(q < 2 ? (double)fval : 0.0);
        if (lane == 0) atomicAdd(&a.fx[t], ws);
      }
      // ---- layer 1 ---------------------------------------------------------------------------------------------------
      wg_fence();
      mma3<kN, G::KB, G::L1Lo, G::L1Hi>(d, A, b1h, b1l);
      wg_commit();
      wg_wait<0>();
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        float h[kU];
#pragma unroll
        for (int s = 0; s < kU; ++s)
          lstm_point_fwd(d[acc_idx(s, 0, rh)], d[acc_idx(s, 1, rh)], d[acc_idx(s, 2, rh)], d[acc_idx(s, 3, rh)], c1[rh][s], h[s]);
        A.template put_vec<G::ColH1>(rh, h);
        if (act[rh] && has_ckpt) {
          store5(ck + rh * 8 * kH, q, h);
          store5(ck + nk + rh * 8 * kH, q, c1[rh]);
        }
        // without a branch around them, ptxas would sink the stores behind the layer-2 MMAs and issue all 40 of the
        // step at its end; the warp barrier keeps them where the epilogue produced their values.  It sits outside the
        // row test, so every lane reaches it on a ragged tile too.
        if (has_ckpt) __syncwarp();
      }
      // ---- layer 2 + output layer + parameter add --------------------------------------------------------------------
      wg_fence();
      mma3<kN, G::KB, G::L2Lo, G::L2Hi>(d, A, b2h, b2l);
      wg_commit();
      wg_wait<0>();
      float y[2];
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        float h[kU];
        float yp = 0.f;
#pragma unroll
        for (int s = 0; s < kU; ++s) {
          lstm_point_fwd(d[acc_idx(s, 0, rh)], d[acc_idx(s, 1, rh)], d[acc_idx(s, 2, rh)], d[acc_idx(s, 3, rh)], c2[rh][s], h[s]);
          yp = fmaf(h[s], wo[s], yp);
        }
        A.template put_vec<G::ColH2>(rh, h);
        y[rh] = quad_sum(yp) + bo;
        if (act[rh] && has_ckpt) {
          store5(ck + 2 * nk + rh * 8 * kH, q, h);
          store5(ck + 3 * nk + rh * 8 * kH, q, c2[rh]);
        }
        if (has_ckpt) __syncwarp();
      }
      const float yo = own ? y[1] : y[0];
      // __fmul_rn: Delta is rounded before x += Delta in every instantiation (an fma here would change x)
      const float dl = tanh_out ? tanh_acc(yo) * rt.scale : __fmul_rn(yo, rt.scale);
      x += dl;
      if (writer) {
        if (has_delta) a.delta_seq[(int64_t)t * n + io] = dl;
        if (has_labels) {
          const float r = a.labels[(int64_t)t * n + io] - dl;
          imit += 0.5 * (double)r * (double)r;
        }
      }
    }
    // ---- tile epilogue: final state (h exactly as hi + lo of its fragment), x, f(x_T), g_T, Adam moments ----------
    if (FAST || T > 0) {
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        if (!act[rh]) continue;
        float h1[kU], h2[kU];
#pragma unroll
        for (int s = 0; s < kU; ++s) {
          h1[s] = A.get_at(G::ColH1 + 4 * s, rh);
          h2[s] = A.get_at(G::ColH2 + 4 * s, rh);
        }
        float* p = state_out + row[rh] * kH;
        store5(p, q, h1);
        store5(p + nk, q, c1[rh]);
        store5(p + 2 * nk, q, h2);
        store5(p + 3 * nk, q, c2[rh]);
      }
    }
    float fval = 0.f;
    if (writer) {
      if (in_kernel_opt) {
        float gT;
        optimizee_eval(opt_kind, x, oa, ob, a.opt_alpha, a.opt_fscale, fval, gT);
        if (has_grec) *gr = gT;
      }
      if (FAST || a.x) a.x[io] = x;
      if (adam_mode) { a.m[io] = am; a.v[io] = av; }
    }
    if (want_fx) {
      const double ws = warp_sum_pairs_d((double)fval);
      if (lane == 0) atomicAdd(&a.fx[T], ws);
    }
  }
  if (has_labels && a.imit_loss) {
    const double ws = warp_sum_d(imit);
    if (lane == 0) atomicAdd(a.imit_loss, ws / (double)a.n_total);
  }
}

}  // namespace tc

// ------------------------------------------------------------------ host side (called from l2o_tc.cu)
// Whether a forward call runs the full-tile instantiation of unroll_fwd_kernel (FAST): a DM net (not fc) on an in-kernel
// Rastrigin or diagonal quadratic, n a multiple of 64, T >= 1, the state updated in place, checkpoints and g_rec both
// recorded or neither, and a plain output layer (no tanh, recorded deltas or imitation labels).
inline bool tc_fwd_fast(bool fc, const NetRt& rt, const l2o_unroll_args& a, const float* state_out) {
  return !fc && (a.opt_kind == L2O_OPT_RASTRIGIN_SEP || a.opt_kind == L2O_OPT_QUADRATIC_DIAG) && a.n > 0 &&
         a.n % tc::kTile == 0 && a.T > 0 && (state_out == nullptr || state_out == a.state) && a.x != nullptr &&
         (a.ckpt == nullptr) == (a.g_rec == nullptr) && !rt.tanh_output && a.delta_seq == nullptr && a.labels == nullptr;
}

template <class C, bool FAST, int OPT, bool CKPT>
int tc_run_fwd(const char* fn, const NetRt& rt, const l2o_unroll_args& a, float* img, cudaStream_t st, int sms,
               float* state_out, tc::FwdExtra ex) {
  auto k = tc::unroll_fwd_kernel<C, FAST, OPT, CKPT>;
  const size_t smem = tc::fwd_smem_bytes<C>(a.T);
  if (smem > 227 * 1024) return L2O_E_INVALID;
  if (int rc = raise_smem_limit(fn, k, smem)) return rc;
  const int64_t ntiles = (a.n + tc::kTile - 1) / tc::kTile;
  const int64_t ctas = (ntiles + tc::kFwdWG - 1) / tc::kFwdWG;
  const int grid = (int)(ctas < sms ? ctas : sms);
  k<<<grid, tc::kFwdThreads, smem, st>>>(a, rt, img, state_out ? state_out : a.state, ex);
  return after_launch(fn);
}

template <class C>
int tc_launch_fwd(const char* fn, const NetRt& rt, const l2o_unroll_args& a, float* img, cudaStream_t st, int sms,
                  float* state_out = nullptr, tc::FwdExtra ex = tc::FwdExtra{nullptr, 0, 0.f}, bool prep = true) {
  if (prep) {
    tc::prep_weights_kernel<C><<<16, 256, 0, st>>>(a.theta, img, 0);
    if (int rc = after_launch(fn)) return rc;
  }
  if constexpr (!C::FC) {
    if (tc_fwd_fast(false, rt, a, state_out)) {
      constexpr int R = L2O_OPT_RASTRIGIN_SEP, Q = L2O_OPT_QUADRATIC_DIAG;
      if (a.opt_kind == R)
        return a.ckpt ? tc_run_fwd<C, true, R, true>(fn, rt, a, img, st, sms, state_out, ex)
                      : tc_run_fwd<C, true, R, false>(fn, rt, a, img, st, sms, state_out, ex);
      return a.ckpt ? tc_run_fwd<C, true, Q, true>(fn, rt, a, img, st, sms, state_out, ex)
                    : tc_run_fwd<C, true, Q, false>(fn, rt, a, img, st, sms, state_out, ex);
    }
  }
  return tc_run_fwd<C, false, L2O_OPT_NONE, false>(fn, rt, a, img, st, sms, state_out, ex);
}

}  // namespace l2o
