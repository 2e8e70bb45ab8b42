// Tensor-core BPTT kernel (sm_90a, wgmma) through a T-step unroll of the LSTM-20x2 (cwlstm_tc.cuh operand layout).
//
// Per warpgroup tile of 64 coordinates, walking t = T-1 .. 0 from the checkpoints:
//   layer 2:  Z2 = [1 | h1n | h2p] . B2  (3xTF32, register-A)  -> gates, output layer, LSTM backward -> dZ2
//             dX2 = dZ2 . W2^T           (3xTF32, the dZ2 accumulators reused as A fragments)  -> dh1n(t), dh2p carry
//   layer 1:  Z1 = [u, 1 | h1p] . B1 -> LSTM backward with dh1 = carry + dh1n(t) -> dZ1;  dX1 = dZ1 . W1^T -> dh1p carry
//   dW:       dW^T rows += X^T . dZ over the tile's coordinates, on the bf16 tensor cores from shared-memory staging
//             (x = hi + lo, hi = bf16_rn(x), lo = bf16_rn(x - hi); products hi.hi + hi.lo + lo.hi, fp32 accumulate).
//             Both layers share ONE 64 x 80 accumulator: the operand rows of layer 2 ([h1n | h2p] in rows 0..39, 1 in
//             row 63) and of layer 1 ([h1p | feature chunk] in rows 40..62) are disjoint (dw_row), and each layer's
//             staged X^T keeps the other layer's rows at zero, so the two K = 64 contractions add into disjoint
//             accumulator rows.  The accumulators are drained into the fp64 dtheta after every tile (bounded fp32
//             accumulation length).  Both operands are staged as packed bf16 pairs with stmatrix (stage_x, stage_dz).
// DM nets take the checkpoint rows from a shared-memory ring that TMA bulk copies fill one layer phase ahead (CkRing).
// fc(20) nets (RNNProp) run the two layers as two passes over time (MODE 1: layer 2, exporting dX2[h1n] to the
// caller's hand-over buffer; MODE 2: layer 1 with the fc layer's own gradient), DM nets both layers in one pass (MODE 0).
// Semantics: SURVEY.md Appendix B (derived from DM/meta.py:319-376, second_derivatives=False); imitation mode
// DM/meta_dm_train.py:472-475.
#pragma once
#include <type_traits>
#include "cwlstm_tc.cuh"

namespace l2o {
namespace tcb {

using namespace tc;

constexpr int kBwdWG = 2;                       // warpgroups per CTA (they share the weight image)
constexpr int kBwdThreads = 128 * kBwdWG;
// staged dW operands per warpgroup (bf16, K-major: the 64 coordinates of the tile are the contraction index)
constexpr uint32_t kXaLBO = 8 * 128;            // X^T: 64 rows (8 core-matrix groups) per 8 coordinates
constexpr uint32_t kXbLBO = 10 * 128;           // dZ^T: 80 rows
constexpr uint32_t kXaBytes = 8 * kXaLBO;       // per hi / lo
constexpr uint32_t kXbBytes = 8 * kXbLBO;
// dW accumulator rows: 8-row blocks 0..4 hold layer 2 (MODE 2: layer 1's [h1p | e]), 5..7 layer 1 of DM nets (MODE 0),
// row 63 the constant 1 of the blocks 0..4 operand (dw_row)
constexpr int kBlkL1 = 5, kRowOne2 = 63;

// x = hi + lo for a pair of values (v0 in the low half): hi = bf16_rn(x), lo = bf16_rn(x - hi)
__device__ __forceinline__ void split_bf16x2(float v0, float v1, uint32_t& hi, uint32_t& lo) {
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(hi) : "f"(v1), "f"(v0));
  const float r0 = v0 - __uint_as_float(hi << 16), r1 = v1 - __uint_as_float(hi & 0xFFFF0000u);
  asm("cvt.rn.bf16x2.f32 %0, %1, %2;" : "=r"(lo) : "f"(r1), "f"(r0));
}
// four 8x8 b16 blocks, transposed: register i of lane l holds (row l / 4, columns 2 (l % 4) + {0, 1}) of block i, which
// land in the 16-byte rows 2 (l % 4) + {0, 1} at 2-byte slot l / 4; lane l gives the address of row l % 8 of block l / 8
__device__ __forceinline__ void stsm_x4_trans(uint32_t sa, uint32_t r0, uint32_t r1, uint32_t r2, uint32_t r3) {
  asm volatile("stmatrix.sync.aligned.m8n8.x4.trans.shared.b16 [%0], {%1, %2, %3, %4};" ::"r"(sa), "r"(r0), "r"(r1),
               "r"(r2), "r"(r3)
               : "memory");
}
// D[64 x 80] += A[64 x 16] (shared, bf16, K-major) . B[16 x 80] (shared, bf16, K-major)
__device__ __forceinline__ void mma_ss_bf16_n80(float* d, uint64_t a, uint64_t b) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %42, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n80k16.f32.bf16.bf16 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,"
      "%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39}, "
      "%40, %41, p, 1, 1, 0, 0;\n\t}\n"
      : L2O_ACC8(0), L2O_ACC8(8), L2O_ACC8(16), L2O_ACC8(24), L2O_ACC8(32)
      : "l"(a), "l"(b), "r"(1));
}
// named barrier over the 128 threads of warpgroup wg
__device__ __forceinline__ void wg_bar(int wg) { asm volatile("bar.sync %0, 128;" ::"r"(1 + wg) : "memory"); }
// L2 prefetch of `bytes` (multiple of 16, 16-byte aligned) with the TMA engine / of one element
__device__ __forceinline__ void prefetch_l2_bulk(const void* p, uint32_t bytes) {
  asm volatile("cp.async.bulk.prefetch.L2.global [%0], %1;" ::"l"(p), "r"(bytes) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }

// LSTM pointwise backward for one unit from the scaled pre-activations (i', j', f', o') of the forward image
// (gate_scale) -> overwritten with dz, the gradient with respect to the unscaled pre-activations; c: previous cell
// state; dh: gradient of h'; dc: carry in (gradient of c') / out (gradient of c).  hn: h' (the output layer needs it).
__device__ __forceinline__ void unit_bwd(float& zi, float& zj, float& zf, float& zo, float cprev, float dh, float& dc, float& hn) {
  const float i = sigmoid_scaled(zi), j = tanh_scaled(zj), f = sigmoid_scaled(zf), o = sigmoid_scaled(zo);
  const float cn = fmaf(f, cprev, i * j);
  const float tcn = tanh_fast(cn);
  hn = tcn * o;
  const float dho = dh * o;
  const float dcv = fmaf(dho, fmaf(-tcn, tcn, 1.0f), dc);
  zi = (dcv * j) * fmaf(-i, i, i);           // sigma' = i - i^2
  zj = (dcv * i) * fmaf(-j, j, 1.0f);        // tanh'  = 1 - j^2
  zf = (dcv * cprev) * fmaf(-f, f, f);
  zo = (dho * tcn) * (1.0f - o);             // dh tcn o (1 - o)
  dc = dcv * f;
}

// theta index of dW accumulator row m at reference gate column 0 (-1: padding row).  Row 8b + 2p + e holds slot 2b + e
// of quad thread p (stage_x): in blocks 0..4, slots 0..4 are units 5p + s of the first 20-vector, 5..9 of the second;
// in the layer-1 blocks 5..7 (MODE 0), slots 10..14 are units of h1p and slot 15 is column p of the feature chunk
// (feature p for p < F, the constant 1 at p = F).
template <class C, int MODE>
__device__ __forceinline__ int dw_row(int m) {
  const int p = (m & 7) >> 1, slot = 2 * (m >> 3) + (m & 1);
  if (m == kRowOne2) return MODE == 2 ? C::O_B1 : C::O_B2;
  if (slot < 2 * kBlkL1) {
    const int u = 5 * p + slot % kU;
    // MODE 2: fc nets, layer 1: h1p | e  (lstm_1/w_gates rows: the 20 fc outputs first, then h1)
    if (MODE == 2) return C::O_W1 + (slot < kU ? C::F + u : u) * C::G1;
    return C::O_W2 + (slot < kU ? u : kH + u) * C::G2;   // h1n | h2p rows of lstm_2/w_gates
  }
  if (MODE == 0) {
    const int s = slot - 2 * kBlkL1;
    if (s < kU) return C::O_W1 + (C::F + 5 * p + s) * C::G1;
    if (p < C::F) return C::O_W1 + p * C::G1;
    if (p == C::F) return C::O_B1;
  }
  return -1;
}

template <class C, int MODE>
struct SmemB {
  float img[Geo<C>::AllFloats];   // B1h|B1l|B2h|B2l|T1h|T1l|T2h|T2l; must stay first (TMA destination)
  float wo[kH + 4];
  float win[64];
  uint64_t wbar, pad;
};
template <class C, int MODE>
__host__ __device__ constexpr uint32_t stage_bytes() {   // per warpgroup: Xa (layer 2) [| Xa (layer 1)] | Xb, hi + lo each
  return (MODE == 0 ? 4 : 2) * kXaBytes + 2 * kXbBytes;
}
// Checkpoint ring of one warpgroup (MODE 0): the tile's checkpoint rows the next phase reads, copied in by TMA bulk
// copies.  The arena is [slot][h1 | c1 | h2 | c2][n][20] floats, so one block of a tile is 64 contiguous rows of 80 B,
// 16-byte aligned for every n.  `h` holds h2(t) for layer 2, then h1(t) for layer 1 (h2 is dead once it is in the
// operand row), so its barrier completes twice per step: parity 0 = h2, 1 = h1.
struct alignas(16) CkRing {   // 16: the bulk-copy destinations of the next warpgroup's ring
  float h[tc::kTile * kH], c2[tc::kTile * kH], c1[tc::kTile * kH];
  uint64_t barh, bar2, bar1;   // h | c2 | c1 landed
};
template <class C, int MODE>
__host__ __device__ constexpr size_t bwd_smem_bytes() {
  return ((sizeof(SmemB<C, MODE>) + 1023) & ~(size_t)1023) +
         (size_t)kBwdWG * (stage_bytes<C, MODE>() + (MODE == 0 ? sizeof(CkRing) : 0));
}

// Output-layer flags of an instantiation (FL), fixed at launch from the arguments: imitation mode (a.labels, the
// gradient of the output comes from delta_seq - labels) and a tanh output (rt.tanh_output, tanh' from delta_seq).  The
// plain instantiation (FL = 0) never reads delta_seq or labels.
constexpr int kFlImit = 1, kFlTanh = 2;

// MODE 0: both layers (DM nets); 1: layer 2 only, dX2[h1n] exported to a.scratch [T][n][20]; 2: layer 1 of an fc net,
// dX2[h1n] read from a.scratch.  CARRY: one segment of a longer unroll (l2o_unroll_bwd_carry); the pass's carries (layer 2
// and lambda, layer 1) start from cy and are written back there.  FULL (DM nets, n a multiple of 64): every tile is
// full, so the body tests no rows.
template <class C, int MODE, bool CARRY, int FL, bool FULL>
__global__ void __launch_bounds__(kBwdThreads, 1) unroll_bwd_kernel(l2o_bwd_args a, NetRt rt, const float* __restrict__ img,
                                                                    l2o_bwd_carry cy) {
  using G = Geo<C>;
  static_assert(MODE == 0 ? !C::FC : C::FC, "DM nets: one pass; fc nets: two passes");
  static_assert(MODE != 0 || C::F < 3, "the feature chunk leaves quad thread 3's slot of row 63 to layer 2's 1");
  static_assert(MODE != 2 || FL == 0, "the output-layer flags belong to the layer-2 passes");
  static_assert(MODE == 0 || !FULL, "the full-tile body is the DM nets'");
  constexpr bool kImit = (FL & kFlImit) != 0, kTanh = (FL & kFlTanh) != 0;
  extern __shared__ __align__(1024) unsigned char smem_raw[];
  SmemB<C, MODE>& S = *reinterpret_cast<SmemB<C, MODE>*>(smem_raw);
  // wg through a shuffle from lane 0: provably warp-uniform, so the staging descriptors built from it live in uniform
  // registers and feed the wgmma without a per-use copy
  const int wg = __shfl_sync(0xffffffffu, threadIdx.x >> 7, 0);
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const int g = lane >> 2, q = lane & 3;
  const uint32_t stage = smem_u32(smem_raw) + (uint32_t)((sizeof(SmemB<C, MODE>) + 1023) & ~(size_t)1023) +
                         (uint32_t)wg * stage_bytes<C, MODE>();
  constexpr uint32_t kXa2 = 0, kXa1 = 2 * kXaBytes;                          // MODE 0 only has kXa1
  constexpr uint32_t kXb = (MODE == 0 ? 4 : 2) * kXaBytes;
  constexpr bool kL2 = MODE != 2, kL1 = MODE != 1;
  // DM nets read the checkpoint rows from the ring, and h1n(t) from the operand row, which holds h1p(t + 1)
  constexpr bool kRing = MODE == 0;
  CkRing& R = *reinterpret_cast<CkRing*>(smem_raw + ((sizeof(SmemB<C, MODE>) + 1023) & ~(size_t)1023) +
                                         (size_t)kBwdWG * stage_bytes<C, MODE>() + (size_t)wg * sizeof(CkRing));
  const bool elected = (threadIdx.x & 127) == 0;

  // zero the staging (rows of the other layer stay zero for the whole kernel) but for the constant 1 of the blocks 0..4
  // operand: row kRowOne2 of its hi part, which no per-step store touches (bf16 1.0 = 0x3F80)
  for (uint32_t o = threadIdx.x * 4; o < kBwdWG * stage_bytes<C, MODE>(); o += blockDim.x * 4) {
    const uint32_t ow = o % stage_bytes<C, MODE>();
    const uint32_t v = (ow < kXaBytes && (ow % kXaLBO) >> 4 == (uint32_t)kRowOne2) ? 0x3F803F80u : 0u;
    asm volatile("st.shared.u32 [%0], %1;" ::"r"(stage - (uint32_t)wg * stage_bytes<C, MODE>() + o), "r"(v) : "memory");
  }
  if (threadIdx.x < kH) S.wo[threadIdx.x] = a.theta[C::O_WO + threadIdx.x];
  if constexpr (C::FC) {
    if (threadIdx.x >= 32 && threadIdx.x < 92) S.win[threadIdx.x - 32] = a.theta[C::O_WIN + threadIdx.x - 32];
  }
  if (threadIdx.x == 0) {
    mbar_init(&S.wbar, 1);
    if (!kRing) fence_barrier_init();
  }
  if (kRing && elected) {
    mbar_init(&R.barh, 1);
    mbar_init(&R.bar2, 1);
    mbar_init(&R.bar1, 1);
    fence_barrier_init();
  }
  fence_proxy_async();
  __syncthreads();
  stage_image(S.img, img, G::AllFloats * 4, &S.wbar);

  const uint64_t b1h = img_desc(S.img, kN), b1l = img_desc(S.img + G::B1Floats, kN);
  const uint64_t b2h = img_desc(S.img + 2 * G::B1Floats, kN), b2l = img_desc(S.img + 2 * G::B1Floats + G::B2Floats, kN);
  const float* tbase = S.img + G::FwdFloats;
  const uint64_t t1h = img_desc(tbase, G::N1), t1l = img_desc(tbase + G::T1Floats, G::N1);
  const uint64_t t2h = img_desc(tbase + 2 * G::T1Floats, G::N2), t2l = img_desc(tbase + 2 * G::T1Floats + G::T2Floats, G::N2);
  const uint64_t xbh = make_desc(stage + kXb, kXbLBO, 128), xbl = make_desc(stage + kXb + kXbBytes, kXbLBO, 128);
  const uint64_t xa2h = make_desc(stage + kXa2, kXaLBO, 128), xa2l = make_desc(stage + kXa2 + kXaBytes, kXaLBO, 128);
  const uint64_t xa1h = make_desc(stage + (MODE == 0 ? kXa1 : kXa2), kXaLBO, 128);
  const uint64_t xa1l = make_desc(stage + (MODE == 0 ? kXa1 : kXa2) + kXaBytes, kXaLBO, 128);

  const int T = a.T;
  const int64_t n = a.n, slot = n * C::SF;
  const int64_t ntiles = (n + tc::kTile - 1) / tc::kTile;
  const float inv_nt = kImit ? 1.0f / (float)a.n_total : 0.f;
  float wo[kU];
#pragma unroll
  for (int s = 0; s < kU; ++s) wo[s] = S.wo[5 * q + s];
  float acc_wo[kU] = {0.f, 0.f, 0.f, 0.f, 0.f}, acc_bo = 0.f;
  float aw0[kU] = {0.f, 0.f, 0.f, 0.f, 0.f}, aw1[kU] = {0.f, 0.f, 0.f, 0.f, 0.f}, ab[kU] = {0.f, 0.f, 0.f, 0.f, 0.f};
  float dw[kN / 2];
#pragma unroll
  for (int k = 0; k < kN / 2; ++k) dw[k] = 0.f;
  const int kx = warp * 16 + g;   // staged coordinate index of row rh = kx + 8 rh
  const int64_t tstride = (int64_t)gridDim.x * kBwdWG;
  // The time loop steps a pointer to the tile's block-0 checkpoint rows of slot t (a.ckpt + t slot + 64 tile kH) back
  // by one slot per step; from slot 0 of a tile, slot T - 1 of the warpgroup's next tile is ck_wrap ahead.
  const int64_t nkh = n * kH;
  const int64_t ck_wrap = (int64_t)(T - 1) * slot + tstride * tc::kTile * kH;

  // ---- checkpoint ring (kRing): each buffer is loaded one layer phase ahead of its reader.  The elected thread
  // re-arms a buffer once a warpgroup barrier has seen every thread's reads of it.  bar2 and bar1 complete once per
  // step, so both are waited with the parity `ph` of the step count; barh twice (CkRing).
  auto ck_block = [&](const float* ckt, int blk) {   // blk 0 h1 | 1 c1 | 2 h2 | 3 c2 of the tile's slot at ckt
    return ckt + blk * nkh;
  };
  auto tile_bytes = [&](int64_t tl) {   // the ragged last tile copies its n - 64 tl rows (a multiple of 16 bytes)
    const int64_t r = n - tl * tc::kTile;
    return (uint32_t)((r < tc::kTile ? r : tc::kTile) * kH * 4);
  };
  auto arm = [&](uint64_t* bar, float* dst, const float* ckt, int blk, uint32_t b) {
    mbar_expect_tx(bar, b);
    tma_bulk_g2s(dst, ck_block(ckt, blk), b, bar);
  };
  auto ring5 = [&](const float* buf, int rh, bool on, float* v) {   // this thread's 5 units of row rh of a ring buffer
    const float* p = buf + (kx + 8 * rh) * kH + 5 * q;
#pragma unroll
    for (int s = 0; s < kU; ++s) v[s] = on ? p[s] : 0.f;
  };
  if constexpr (kRing) {
    const int64_t tile0 = (int64_t)blockIdx.x * kBwdWG + wg;
    if (elected && tile0 < ntiles) {
      const float* ck0 = a.ckpt + (int64_t)(T - 1) * slot + tile0 * tc::kTile * kH;
      const uint32_t b = tile_bytes(tile0);
      arm(&R.barh, R.h, ck0, 2, b);
      arm(&R.bar2, R.c2, ck0, 3, b);
      arm(&R.bar1, R.c1, ck0, 1, b);
    }
  }
  uint32_t ph = 0;

  Frag<G::KB> A;
  // The staged operands are K-major core matrices (8 rows of 16 B = 8 coordinates), so an 8x8 block of (coordinate,
  // row) pairs in a thread's accumulator-style registers is one transposed stmatrix block.  Each x4 stores the blocks
  // (hi, rh 0) (hi, rh 1) (lo, rh 0) (lo, rh 1) of one 8-row group: lane l addresses row l % 8 of block l / 8.
  const int blk = lane >> 3;
  const uint32_t la = stage + (uint32_t)((2 * warp + (blk & 1)) * (int)kXaLBO + (blk >> 1) * (int)kXaBytes + (lane & 7) * 16);
  const uint32_t lb = stage + kXb + (uint32_t)((2 * warp + (blk & 1)) * (int)kXbLBO + (blk >> 1) * (int)kXbBytes + (lane & 7) * 16);
  // X^T blocks [b0, b0 + nb) of the operand at `buf`: slot i = 2 (b - b0) + e of this thread goes to row 8b + 2q + e;
  // slots 0..4 are its units of the 20-vector at operand column c0, slots 5.. those of the one at c1 (dw_row)
  auto stage_x = [&](uint32_t buf, int b0, int nb, int c0, int c1) {
    auto val = [&](int i, int rh) { return A.get_at(i < kU ? c0 + 4 * i : c1 + 4 * (i - kU), rh); };
#pragma unroll
    for (int b = 0; b < nb; ++b) {
      uint32_t h0, l0, h1, l1;
      split_bf16x2(val(2 * b, 0), val(2 * b + 1, 0), h0, l0);
      split_bf16x2(val(2 * b, 1), val(2 * b + 1, 1), h1, l1);
      stsm_x4_trans(la + buf + (uint32_t)(b0 + b) * 128, h0, h1, l0, l1);
    }
  };
  // dZ^T: accumulator registers z[4j + 2rh + {0, 1}] are gate columns 8j + 2q + {0, 1} of coordinate kx + 8 rh
  auto stage_dz = [&](const float* z) {
#pragma unroll
    for (int j = 0; j < kN / 8; ++j) {
      uint32_t h0, l0, h1, l1;
      split_bf16x2(z[4 * j], z[4 * j + 1], h0, l0);
      split_bf16x2(z[4 * j + 2], z[4 * j + 3], h1, l1);
      stsm_x4_trans(lb + (uint32_t)j * 128, h0, h1, l0, l1);
    }
  };
  // dX_l = dZ_l . W_l^T (3xTF32; the dZ accumulators as A fragments, cwlstm_tc.cuh dx_gate_col) then the dW batch
  auto dx_dw = [&](auto ncols, float* z, float* x, uint64_t th, uint64_t tl, uint64_t xah, uint64_t xal) {
    constexpr int NX = decltype(ncols)::value;
    uint32_t fh[kN / 8][4], fl[kN / 8][4];
#pragma unroll
    for (int j = 0; j < kN / 8; ++j) {
      split_tf32(z[4 * j + 0], fh[j][0], fl[j][0]);
      split_tf32(z[4 * j + 2], fh[j][1], fl[j][1]);
      split_tf32(z[4 * j + 1], fh[j][2], fl[j][2]);
      split_tf32(z[4 * j + 3], fh[j][3], fl[j][3]);
    }
    constexpr uint64_t step = img_kstep(NX);
    wg_fence();
#pragma unroll
    for (int j = 0; j < kN / 8; ++j) {
      mma_rs<NX>(x, fl[j], th + j * step, j > 0 ? 1u : 0u);
      mma_rs<NX>(x, fh[j], tl + j * step, 1u);
      mma_rs<NX>(x, fh[j], th + j * step, 1u);
    }
    wg_commit();
    constexpr uint64_t sa = (2 * kXaLBO) >> 4, sb = (2 * kXbLBO) >> 4;
#pragma unroll
    for (int kk = 0; kk < tc::kTile / 16; ++kk) {
      mma_ss_bf16_n80(dw, xal + kk * sa, xbh + kk * sb);
      mma_ss_bf16_n80(dw, xah + kk * sa, xbl + kk * sb);
      mma_ss_bf16_n80(dw, xah + kk * sa, xbh + kk * sb);
    }
    wg_commit();
    wg_wait<1>();   // dX done; the dW batch may still run (the next wait<0> retires it)
  };
  auto flush_dw = [&]() {
    wg_wait<0>();
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) {
      const int r = dw_row<C, MODE>(kx + 8 * rh);
#pragma unroll
      for (int j = 0; j < kN / 8; ++j)
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          float& v = dw[4 * j + 2 * rh + e];
          if (r >= 0 && v != 0.f) atomicAdd(&a.dtheta[r + gate_ref_col(8 * j + 2 * q + e)], (double)v);
          v = 0.f;
        }
    }
  };

  for (int64_t tile = (int64_t)blockIdx.x * kBwdWG + wg; tile < ntiles; tile += tstride) {
    const int64_t r0 = tile * tc::kTile + kx;
    const int64_t row[2] = {r0, r0 + 8};
    const bool act[2] = {FULL || row[0] < n, FULL || row[1] < n};
    // slot t, walked back one slot per step (see ck_wrap above): the tile's checkpoint rows and t n, the offset of
    // step t in the [T (+1)][n] per-coordinate sequences (both warp-uniform)
    const float* ckt = a.ckpt + (int64_t)(T - 1) * slot + tile * tc::kTile * kH;
    int64_t tn = (int64_t)(T - 1) * n;
    float dc2[2][kU], dh2c[2][kU], dc1[2][kU], dh1c[2][kU];
#pragma unroll
    for (int rh = 0; rh < 2; ++rh)
#pragma unroll
      for (int s = 0; s < kU; ++s) { dc2[rh][s] = 0.f; dh2c[rh][s] = 0.f; dc1[rh][s] = 0.f; dh1c[rh][s] = 0.f; }
    float lam[2];
#pragma unroll
    for (int rh = 0; rh < 2; ++rh) lam[rh] = (kL2 && act[rh] && !kImit) ? a.g_rec[tn + n + row[rh]] : 0.f;
    if constexpr (CARRY) {   // state arena [h1 | c1 | h2 | c2][n][20]; lambda = carry + g_t1 (the order of a whole sweep)
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        if (!act[rh]) continue;
        const int64_t i = row[rh];
        if constexpr (kL2) {
          load5(cy.d_state + (2 * n + i) * kH, q, dh2c[rh]);
          load5(cy.d_state + (3 * n + i) * kH, q, dc2[rh]);
          lam[rh] = cy.lam[i] + a.g_rec[tn + n + i];
        }
        if constexpr (kL1) {
          load5(cy.d_state + i * kH, q, dh1c[rh]);
          load5(cy.d_state + (n + i) * kH, q, dc1[rh]);
        }
      }
    }
    A.zero();
    A.template put<(G::ColOne & ~3)>(0, q == (G::ColOne & 3) ? 1.0f : 0.f);
    A.template put<(G::ColOne & ~3)>(1, q == (G::ColOne & 3) ? 1.0f : 0.f);

    for (int t = T - 1; t >= 0; --t) {
      const float* ckr = ckt + kx * kH;   // this thread's row r0 of slot t (row r0 + 8 at + 8 kH)
      float z[kN / 2];
      float dh1n[2][kU];
      // ================================= layer 2 =================================
      if constexpr (kL2) {
        float c2p[2][kU], dy[2];
        if constexpr (kRing) mbar_wait(&R.barh, 0);
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
          float h1n[kU] = {0.f, 0.f, 0.f, 0.f, 0.f}, h2p[kU] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int s = 0; s < kU; ++s) c2p[rh][s] = 0.f;
          float dtanh = 1.0f;
          if (act[rh]) {
            const float* cr = ckr + 8 * kH * rh;
            if constexpr (kRing) {
              if (t == T - 1) load5(cr + slot, q, h1n);
              ring5(R.h, rh, true, h2p);
            } else {
              load5(cr + slot, q, h1n);   // h1n(t) IS the checkpointed h1 of slot t+1
              load5(cr + 2 * nkh, q, h2p);
              load5(cr + 3 * nkh, q, c2p[rh]);
            }
            if constexpr (kImit) lam[rh] = (a.delta_seq[tn + row[rh]] - a.labels[tn + row[rh]]) * inv_nt;
            if constexpr (kTanh) {   // delta = scale tanh(y): the recorded delta gives tanh' without y
              const float th = a.delta_seq[tn + row[rh]] / rt.scale;
              dtanh = fmaf(-th, th, 1.0f);
            }
          }
          dy[rh] = rt.scale * lam[rh] * dtanh;
          // with the ring, layer 1 of step t + 1 left h1p(t + 1) = h1n(t) in the operand row (0 on inactive rows)
          if (!kRing || t == T - 1) A.template put_vec<G::ColH1>(rh, h1n);
          A.template put_vec<G::ColH2>(rh, h2p);
        }
        wg_fence();
        mma3<kN, G::KB, G::L2Lo, G::L2Hi>(z, A, b2h, b2l);
        wg_commit();
        wg_wait<0>();   // also retires every earlier dW batch of this warp
        if constexpr (kRing) {   // c2 is read only now, so it is not held in registers across the MMA
          mbar_wait(&R.bar2, ph);
#pragma unroll
          for (int rh = 0; rh < 2; ++rh) ring5(R.c2, rh, act[rh], c2p[rh]);
        }
        if (q == 0) acc_bo += dy[0] + dy[1];
#pragma unroll
        for (int rh = 0; rh < 2; ++rh)
#pragma unroll
          for (int s = 0; s < kU; ++s) {
            float hn;
            unit_bwd(z[acc_idx(s, 0, rh)], z[acc_idx(s, 1, rh)], z[acc_idx(s, 2, rh)], z[acc_idx(s, 3, rh)], c2p[rh][s],
                     fmaf(wo[s], dy[rh], dh2c[rh][s]), dc2[rh][s], hn);
            acc_wo[s] = fmaf(hn, dy[rh], acc_wo[s]);
          }
        wg_bar(wg);   // every warp has retired the previous dW batch: the staging may be overwritten
        if constexpr (kRing) {   // and every read of h2 / c2 is done: h1(t) for layer 1, c2 of the next slot
          if (elected) {
            // the slot the ring loads next: t - 1 of this tile, or T - 1 of the warpgroup's next tile
            const int64_t tl_next = t > 0 ? tile : tile + tstride;
            arm(&R.barh, R.h, ckt, 0, tile_bytes(tile));
            if (tl_next < ntiles) arm(&R.bar2, R.c2, t > 0 ? ckt - slot : ckt + ck_wrap, 3, tile_bytes(tl_next));
          }
        }
        stage_x(kXa2, 0, kBlkL1, G::ColH1, G::ColH2);   // h1n | h2p
        stage_dz(z);
        fence_proxy_async();
        wg_bar(wg);
        float x2[G::N2 / 2];
        dx_dw(IC<G::N2>{}, z, x2, t2h, t2l, xa2h, xa2l);
#pragma unroll
        for (int rh = 0; rh < 2; ++rh)
#pragma unroll
          for (int s = 0; s < kU; ++s) {
            // dX column of slot s: 8 (s / 2) + 2q + (s % 2) in group 0 (h1n), + 24 in group 1 (h2p)
            dh1n[rh][s] = x2[4 * (s >> 1) + 2 * rh + (s & 1)];
            dh2c[rh][s] = x2[4 * (3 + (s >> 1)) + 2 * rh + (s & 1)];
          }
        if constexpr (MODE == 1) {
#pragma unroll
          for (int rh = 0; rh < 2; ++rh)
            if (act[rh]) store5(a.scratch + (tn + row[rh]) * kH, q, dh1n[rh]);
        }
#pragma unroll
        for (int rh = 0; rh < 2; ++rh)
          if (!kImit && act[rh] && (!CARRY || t > 0)) lam[rh] += a.g_rec[tn + row[rh]];   // g_t0: the previous segment's
      }
      // ================================= layer 1 =================================
      if constexpr (kL1) {
        float c1p[2][kU];
        float r0v[2] = {0.f, 0.f};
        [[maybe_unused]] float r1v[2] = {0.f, 0.f};   // fc nets: the second input row
        [[maybe_unused]] float ep[2][kU];             // fc nets: elu'(a) of the thread's fc outputs
        if constexpr (kRing) mbar_wait(&R.barh, 1);
#pragma unroll
        for (int rh = 0; rh < 2; ++rh) {
          float h1p[kU] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
          for (int s = 0; s < kU; ++s) c1p[rh][s] = 0.f;
          if (act[rh]) {
            if constexpr (kRing) {
              ring5(R.h, rh, true, h1p);
            } else {
              load5(ckr + 8 * kH * rh, q, h1p);
              load5(ckr + nkh + 8 * kH * rh, q, c1p[rh]);
            }
            if constexpr (MODE == 2) {
              load5(a.scratch + (tn + row[rh]) * kH, q, dh1n[rh]);
              r0v[rh] = a.in_seq[2 * tn + row[rh]];
              r1v[rh] = a.in_seq[2 * tn + n + row[rh]];
            } else {
              r0v[rh] = a.in_seq[tn + row[rh]];
            }
          } else if constexpr (MODE == 2) {
#pragma unroll
            for (int s = 0; s < kU; ++s) dh1n[rh][s] = 0.f;
          }
          A.template put_vec<G::ColH1>(rh, h1p);
          if constexpr (MODE == 2) {
            // e = elu([m~, g~] Win + bin) for the thread's units, as the forward kernel computes it
            float e[kU];
#pragma unroll
            for (int s = 0; s < kU; ++s) {
              const int u = 5 * q + s;
              const float av = fmaf(r1v[rh], S.win[kH + u], fmaf(r0v[rh], S.win[u], S.win[2 * kH + u]));
              e[s] = elu_fast(av);
              ep[rh][s] = av > 0.f ? 1.0f : e[s] + 1.0f;   // elu' = exp(a) on the negative side
            }
            A.template put_vec<0>(rh, e);
          } else {
            float f[C::F];
            preprocess<C>(nullptr, rt, r0v[rh], 0.f, f);
            float v = q == C::F ? 1.0f : 0.f;
#pragma unroll
            for (int k = 0; k < C::F; ++k)
              if (q == k) v = f[k];
            A.template put<0>(rh, v);
          }
        }
        wg_fence();
        mma3<kN, G::KB, G::L1Lo, G::L1Hi>(z, A, b1h, b1l);
        wg_commit();
        wg_wait<0>();
        if constexpr (kRing) {
          mbar_wait(&R.bar1, ph);
#pragma unroll
          for (int rh = 0; rh < 2; ++rh) ring5(R.c1, rh, act[rh], c1p[rh]);
        }
#pragma unroll
        for (int rh = 0; rh < 2; ++rh)
#pragma unroll
          for (int s = 0; s < kU; ++s) {
            float hn;
            unit_bwd(z[acc_idx(s, 0, rh)], z[acc_idx(s, 1, rh)], z[acc_idx(s, 2, rh)], z[acc_idx(s, 3, rh)], c1p[rh][s],
                     dh1c[rh][s] + dh1n[rh][s], dc1[rh][s], hn);
          }
        wg_bar(wg);
        if constexpr (kRing) {   // every read of h1 / c1 is done: h2 and c1 of the next slot, its h1 and in_seq into L2
          const int64_t tl_next = t > 0 ? tile : tile + tstride;
          if (elected && tl_next < ntiles) {
            const float* ckn = t > 0 ? ckt - slot : ckt + ck_wrap;
            const uint32_t b = tile_bytes(tl_next);
            arm(&R.barh, R.h, ckn, 2, b);
            arm(&R.bar1, R.c1, ckn, 1, b);
            prefetch_l2_bulk(ck_block(ckn, 0), b);
          }
          // in_seq rows of the next slot: t - 1 of this tile, or T - 1 of the next tile
          const int64_t rn = t > 0 ? r0 : r0 + tstride * tc::kTile;
          const float* in_next = a.in_seq + (t > 0 ? tn - n : (int64_t)(T - 1) * n) + rn;
#pragma unroll
          for (int rh = 0; rh < 2; ++rh)
            if (q == 0 && ((FULL && t > 0) || rn + 8 * rh < n)) prefetch_l2(in_next + 8 * rh);
          ph ^= 1u;
        }
        if constexpr (MODE == 2) stage_x(kXa2, 0, kBlkL1, G::ColH1, 0);   // h1p | e
        else stage_x(kXa1, kBlkL1, 3, G::ColH1, 0);                     // h1p | column q of the feature chunk
        stage_dz(z);
        fence_proxy_async();
        wg_bar(wg);
        float x1[G::N1 / 2];
        dx_dw(IC<G::N1>{}, z, x1, t1h, t1l, xa1h, xa1l);
#pragma unroll
        for (int rh = 0; rh < 2; ++rh)
#pragma unroll
          for (int s = 0; s < kU; ++s) {
            dh1c[rh][s] = x1[4 * (s >> 1) + 2 * rh + (s & 1)];
            if constexpr (MODE == 2) {   // da = de * elu'(a);  dWin += [m~, g~]^T da, dbin += da
              const float da = x1[4 * (3 + (s >> 1)) + 2 * rh + (s & 1)] * ep[rh][s];
              aw0[s] = fmaf(r0v[rh], da, aw0[s]);
              aw1[s] = fmaf(r1v[rh], da, aw1[s]);
              ab[s] += da;
            }
          }
      }
      ckt -= slot;
      tn -= n;
    }
    if constexpr (CARRY) {
#pragma unroll
      for (int rh = 0; rh < 2; ++rh) {
        if (!act[rh]) continue;
        const int64_t i = row[rh];
        if constexpr (kL2) {
          store5(cy.d_state + (2 * n + i) * kH, q, dh2c[rh]);
          store5(cy.d_state + (3 * n + i) * kH, q, dc2[rh]);
          if (q == 0) cy.lam[i] = lam[rh];
        }
        if constexpr (kL1) {
          store5(cy.d_state + i * kH, q, dh1c[rh]);
          store5(cy.d_state + (n + i) * kH, q, dc1[rh]);
        }
      }
    }
    flush_dw();
  }
  wg_wait<0>();
  // ---- output layer (layer-2 passes) and fc layer (MODE 2) gradients: per-thread sums over the warp's rows -----------
  auto red8 = [&](float v) {   // sum over the 8 lanes with the same q
#pragma unroll
    for (int o = 4; o < 32; o <<= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
  };
#pragma unroll
  for (int s = 0; s < kU; ++s) {
    const int u = 5 * q + s;
    if constexpr (kL2) {
      const float v = red8(acc_wo[s]);
      if (lane < 4) atomicAdd(&a.dtheta[C::O_WO + u], (double)v);
    }
    if constexpr (MODE == 2) {
      const float v0 = red8(aw0[s]), v1 = red8(aw1[s]), vb = red8(ab[s]);
      if (lane < 4) {
        atomicAdd(&a.dtheta[C::O_WIN + u], (double)v0);
        atomicAdd(&a.dtheta[C::O_WIN + C::F + u], (double)v1);
        atomicAdd(&a.dtheta[C::O_BIN + u], (double)vb);
      }
    }
  }
  if constexpr (kL2) {
    const float v = red8(acc_bo);
    if (lane == 0) atomicAdd(&a.dtheta[C::O_BO], (double)v);
  }
}

}  // namespace tcb

template <class C, bool CARRY>
int tc_launch_bwd(const char* fn, const NetRt& rt, const l2o_bwd_args& a, float* img, cudaStream_t st, int sms,
                  const l2o_bwd_carry& cy) {
  tc::prep_weights_kernel<C><<<16, 256, 0, st>>>(a.theta, img, 1);
  if (int rc = after_launch(fn)) return rc;
  const int64_t ntiles = (a.n + tc::kTile - 1) / tc::kTile;
  const int64_t ctas = (ntiles + tcb::kBwdWG - 1) / tcb::kBwdWG;
  const int grid = (int)(ctas < sms ? ctas : sms);
  auto launch = [&](auto kern, size_t smem) {
    if (smem > 227 * 1024) return L2O_E_INVALID;
    if (int rc = raise_smem_limit(fn, kern, smem)) return rc;
    kern<<<grid, tcb::kBwdThreads, smem, st>>>(a, rt, img, cy);
    return after_launch(fn);
  };
  // the layer-2 pass's instantiation for the output-layer flags of these arguments
  const int fl = (a.labels != nullptr ? tcb::kFlImit : 0) | (rt.tanh_output ? tcb::kFlTanh : 0);
  // the layer-2 pass's instantiation for these flags, and for DM nets whether every tile is full
  auto launch_l2 = [&](auto mode, auto full) {
    constexpr int M = decltype(mode)::value;
    constexpr bool F = decltype(full)::value;
    constexpr size_t smem = tcb::bwd_smem_bytes<C, M>();
    switch (fl) {
      case 0: return launch(tcb::unroll_bwd_kernel<C, M, CARRY, 0, F>, smem);
      case tcb::kFlImit: return launch(tcb::unroll_bwd_kernel<C, M, CARRY, tcb::kFlImit, F>, smem);
      case tcb::kFlTanh: return launch(tcb::unroll_bwd_kernel<C, M, CARRY, tcb::kFlTanh, F>, smem);
      default: return launch(tcb::unroll_bwd_kernel<C, M, CARRY, tcb::kFlImit | tcb::kFlTanh, F>, smem);
    }
  };
  if constexpr (C::FC) {
    // two passes over time: layer 2 (exporting dX2[h1n] to a.scratch), then layer 1 fed by it
    int rc = launch_l2(tc::IC<1>{}, std::false_type{});
    if (rc != L2O_OK) return rc;
    return launch(tcb::unroll_bwd_kernel<C, 2, CARRY, 0, false>, tcb::bwd_smem_bytes<C, 2>());
  } else {
    if (a.n % tc::kTile == 0) return launch_l2(tc::IC<0>{}, std::true_type{});
    return launch_l2(tc::IC<0>{}, std::false_type{});
  }
}

}  // namespace l2o
