// HierarchicalRNN per-parameter level on the sm_90a tensor cores (included by l2o_hrnn.cu, inside namespace l2o::hrnn).
//
// The step of oracle/hrnn_oracle.py and of the exact-fp32 recompute in hrnn_bwd.cuh (HR:444-540 features,
// rnn_cells.py:46-68 BiasGRU(10), HR:606-706 readouts); the two GRU products run as error-compensated 3xTF32 wgmma with
// the per-coordinate operand rows staged in shared memory:
//   MMA 1  D[128 x 48] = A1[128 x 24] . B1[24 x 48]     A1 = [feat 0..11 | h 12..21 | 1 | 0]
//          D columns: r 0..9 | u 16..25 | candidate (feature part + bc) 32..41        (per 64-row half: 3 K-steps x 3)
//   MMA 2  D[:, 32..47] += A2[128 x 16] . B2[16 x 16]   A2 = [r*h 0..9 | 0]           (the same accumulator registers)
// A persistent CTA of 128 threads (one warpgroup; thread = coordinate) walks tiles of 128 coordinates: the 21 state
// planes and the gradient of the NEXT tile stream into a shared-memory ring with 4-byte cp.async (tensor boundaries are
// not 16-byte aligned, and every thread only ever reads what it copied itself, so no barrier guards the ring).  The
// accumulator fragments come back to their coordinate's thread through a padded shared-memory row buffer.  The
// per-tensor sums stay in registers across tiles and go through the warp butterfly + fp64 atomics every kFlushTiles
// tiles.
#pragma once

namespace tcg {
using namespace l2o::tc;

constexpr int kTile = 128;
constexpr int kKA = 24, kND = 48;      // MMA 1: K (A1 columns), N (D columns)
constexpr int kKA2 = 16, kND2 = 16;    // MMA 2
constexpr int kColU = 16, kColC = 32;  // D column groups (r at 0)
constexpr int kB1Floats = kKA * kND;
constexpr int kB2Floats = kKA2 * kND2;
constexpr int kPlanesIn = kPlanes + 1;  // + the gradient
constexpr int kStages = 2;
constexpr int kDStride = kND + 4;       // row stride of the accumulator buffer (conflict-free row reads)
constexpr uint32_t kALBO = (kTile / 8) * 128;   // K-major operand rows: 16 row groups of 128 B per 4 columns
constexpr int kFlushTiles = 8;
constexpr int kCtasPerSm = 2;

struct SmemG {
  float a1h[kKA * kTile], a1l[kKA * kTile];     // K-major core-matrix layout (first: 16-byte aligned)
  float a2h[kKA2 * kTile], a2l[kKA2 * kTile];
  float b1h[kB1Floats], b1l[kB1Floats], b2h[kB2Floats], b2l[kB2Floats];
  float dbuf[kTile * kDStride];
  float ring[kStages][kPlanesIn][kTile];
  float4 ro[H0];     // readout weights (Wu, Ws, Wi, Wl)[k]   (HR:609-611,645-651,663-666)
  float cst[12];     // bs | bi | bl | sigmoid(lr momentum) | offset | grad-shortcut weights 5..8
  double red[kTile / 32][kAcc];
};

__device__ __forceinline__ int b_index(int nn, int k, int n) { return ((k >> 2) * (nn / 8) + (n >> 3)) * 32 + (n & 7) * 4 + (k & 3); }
__device__ __forceinline__ void cp_async4(uint32_t saddr, const float* g) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(saddr), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }
__device__ __forceinline__ float lds(uint32_t saddr) {
  float v;
  asm volatile("ld.shared.f32 %0, [%1];" : "=f"(v) : "r"(saddr));
  return v;
}
// 4 operand columns [4c, 4c + 4) of this thread's row into the hi / lo images: hi = truncated tf32, lo = the remainder
__device__ __forceinline__ void st_split4(float* hi, float* lo, int c, int row, const float* v) {
  uint32_t h[4], l[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) split_tf32(v[k], h[k], l[k]);
  const int o = c * (int)(kALBO / 4) + row * 4;
  *reinterpret_cast<uint4*>(hi + o) = make_uint4(h[0], h[1], h[2], h[3]);
  *reinterpret_cast<uint4*>(lo + o) = make_uint4(l[0], l[1], l[2], l[3]);
}
// D[64 x N] (+)= A[64 x 8] (shared, tf32, K-major) . B[8 x N] (shared)
__device__ __forceinline__ void mma_ss_n48(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n48k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23}, "
      "%24, %25, p, 1, 1;\n\t}\n"
      : L2O_ACC8(0), L2O_ACC8(8), L2O_ACC8(16)
      : "l"(a), "l"(b), "r"(acc));
}
__device__ __forceinline__ void mma_ss_n16(float* d, uint64_t a, uint64_t b) {   // always accumulates
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
      "{%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1;\n\t}\n"
      : L2O_ACC8(0)
      : "l"(a), "l"(b), "r"(1));
}

// weight value of the extended matrices (theta layout: l2o_hrnn.cu O_* offsets)
__device__ __forceinline__ float b1_value(const float* __restrict__ theta, int k, int n) {
  int grp, j;
  if (n < H0) { grp = 0; j = n; }
  else if (n >= kColU && n < kColU + H0) { grp = 1; j = n - kColU; }
  else if (n >= kColC && n < kColC + H0) { grp = 2; j = n - kColC; }
  else return 0.f;
  if (k < F + H0) {
    if (grp < 2) return theta[O_WG0 + k * 2 * H0 + grp * H0 + j];
    return k < F ? theta[O_WC0 + k * H0 + j] : 0.f;   // the h rows of the candidate go through r*h (MMA 2)
  }
  if (k == F + H0) return grp < 2 ? theta[O_BG0 + grp * H0 + j] : theta[O_BC0 + j];
  return 0.f;
}
__device__ __forceinline__ float b2_value(const float* __restrict__ theta, int k, int n) {
  return (k < H0 && n < H0) ? theta[O_WC0 + (F + k) * H0 + n] : 0.f;
}

__global__ void __launch_bounds__(kTile, kCtasPerSm) coord_tc_kernel(const float* __restrict__ theta, const float* __restrict__ g,
                                                                     float* __restrict__ state, int64_t n,
                                                                     const BlockEnt* __restrict__ blocks, int ntiles,
                                                                     Workspace w) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  SmemG& S = *reinterpret_cast<SmemG*>(smem_raw);
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int gq = lane >> 2, q = lane & 3;

  // ---- one-time setup: weight images (hi/lo, K-major core-matrix layout), readout constants
  for (int e = tid; e < kB1Floats + kB2Floats; e += kTile) {
    const bool second = e >= kB1Floats;
    const int ee = second ? e - kB1Floats : e;
    const int nn = second ? kND2 : kND;
    const int k = ee / nn, c = ee % nn;
    const float wv = second ? b2_value(theta, k, c) : b1_value(theta, k, c);
    const float hi = to_tf32(wv);
    const int idx = b_index(nn, k, c);
    (second ? S.b2h : S.b1h)[idx] = hi;
    (second ? S.b2l : S.b1l)[idx] = to_tf32(wv - hi);
  }
  if (tid < H0) S.ro[tid] = make_float4(theta[O_WU + tid], theta[O_WS + tid], theta[O_WI + tid], theta[O_WL + tid]);
  if (tid == 32) {
    S.cst[0] = theta[O_BS];
    S.cst[1] = theta[O_BI];
    S.cst[2] = theta[O_BL];
    S.cst[3] = sigmoid_fast(theta[O_LRM]);
    S.cst[4] = theta[O_OFF];
#pragma unroll
    for (int s = 0; s < NS; ++s) S.cst[5 + s] = theta[O_G2D + s];
  }
  fence_proxy_async();   // the images are written with generic stores; the MMA reads them through the async proxy
  __syncthreads();
  const uint64_t d1h = make_desc(smem_u32(S.b1h), (kND / 8) * 128, 128), d1l = make_desc(smem_u32(S.b1l), (kND / 8) * 128, 128);
  const uint64_t d2h = make_desc(smem_u32(S.b2h), (kND2 / 8) * 128, 128), d2l = make_desc(smem_u32(S.b2l), (kND2 / 8) * 128, 128);
  const uint64_t a1h = make_desc(smem_u32(S.a1h), kALBO, 128), a1l = make_desc(smem_u32(S.a1l), kALBO, 128);
  const uint64_t a2h = make_desc(smem_u32(S.a2h), kALBO, 128), a2l = make_desc(smem_u32(S.a2l), kALBO, 128);
  constexpr uint64_t kStepA = (2 * kALBO) >> 4, kHalfA = (8 * 128) >> 4;    // per K = 8 / per 64-row half
  constexpr uint64_t kStep1 = (2 * (kND / 8) * 128) >> 4, kStep2 = (2 * (kND2 / 8) * 128) >> 4;
  const uint32_t ring_s = smem_u32(&S.ring[0][0][0]) + tid * 4;
  constexpr uint32_t kStageBytes = kPlanesIn * kTile * 4;

  auto prefetch = [&](int tile, int stage) {
    const BlockEnt be = blocks[tile];
    if (tid < be.count) {
      const int64_t i = be.start + tid;
      const uint32_t dst = ring_s + stage * kStageBytes;
#pragma unroll
      for (int p = 0; p < kPlanes; ++p) cp_async4(dst + p * kTile * 4, state + (int64_t)p * n + i);
      cp_async4(dst + kPlanes * kTile * 4, g + i);
    }
    cp_async_commit();
  };

  float vals[kAcc];
#pragma unroll
  for (int k = 0; k < kAcc; ++k) vals[k] = 0.f;
  int nz_mask = 0;
  auto flush = [&](int tensor) {
#pragma unroll
    for (int k = 0; k < kAcc; ++k) {
      float v = vals[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) S.red[warp][k] = (double)v;
      vals[k] = 0.f;
    }
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      const unsigned any = __ballot_sync(0xffffffffu, nz_mask & (1 << s));
      if (lane == 0 && any) atomicOr(&w.any_nz[tensor * NS + s], 1);
    }
    nz_mask = 0;
    __syncthreads();
    if (tid < kAcc) atomicAdd(&w.acc[tensor * kAcc + tid], ((S.red[0][tid] + S.red[1][tid]) + S.red[2][tid]) + S.red[3][tid]);
    __syncthreads();
  };
  // accumulator fragments of both 64-row halves -> the row buffer, columns [8 J0, 8 J1)
  auto put_acc = [&](const float (&d)[2][kND / 2], int j0, int j1) {
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
#pragma unroll
      for (int j = 0; j < kND / 8; ++j)
        if (j >= j0 && j < j1)
#pragma unroll
          for (int rh = 0; rh < 2; ++rh) {
            const int r = 64 * hf + 16 * warp + gq + 8 * rh;
            *reinterpret_cast<float2*>(&S.dbuf[r * kDStride + 8 * j + 2 * q]) = make_float2(d[hf][4 * j + 2 * rh], d[hf][4 * j + 2 * rh + 1]);
          }
  };
  auto get10 = [&](int col, float* z) {   // columns [col, col + 10) of this thread's row
    const float* p = &S.dbuf[tid * kDStride + col];
    const float4 x0 = *reinterpret_cast<const float4*>(p), x1 = *reinterpret_cast<const float4*>(p + 4);
    const float2 x2 = *reinterpret_cast<const float2*>(p + 8);
    z[0] = x0.x; z[1] = x0.y; z[2] = x0.z; z[3] = x0.w; z[4] = x1.x; z[5] = x1.y; z[6] = x1.z; z[7] = x1.w; z[8] = x2.x; z[9] = x2.y;
  };

  const float mean_llr = *w.mean_log_lr;
  float d[2][kND / 2];
#pragma unroll
  for (int hf = 0; hf < 2; ++hf)
#pragma unroll
    for (int k = 0; k < kND / 2; ++k) d[hf][k] = 0.f;
  int cur_tensor = -1, since = 0, it = 0;
  if ((int)blockIdx.x < ntiles) prefetch(blockIdx.x, 0);
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x, ++it) {
    const BlockEnt be = blocks[tile];
    if (be.tensor != cur_tensor || since == kFlushTiles) {
      if (cur_tensor >= 0) flush(cur_tensor);
      cur_tensor = be.tensor;
      since = 0;
    }
    ++since;
    const int stage = it & 1;
    if (tile + (int)gridDim.x < ntiles) {
      prefetch(tile + gridDim.x, stage ^ 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    const bool act = tid < be.count;
    const int64_t i = be.start + (act ? tid : 0);
    const uint32_t src = ring_s + stage * kStageBytes;
    auto in_plane = [&](int p) { return act ? lds(src + p * kTile * 4) : 0.f; };

    // ---- features (HR:458-531) -> A1 = [feat | h | 1 | 0]
    float a[kKA];
    float sc[NS];
    const float sd = in_plane(P_SCL);
    const float llr = in_plane(P_LLR);
    const float gi = in_plane(kPlanes);
    {
      const int4 zf = __ldg(reinterpret_cast<const int4*>(w.zero_flag + be.tensor * NS));
      const int zfl[NS] = {zf.x, zf.y, zf.z, zf.w};
      float dec = in_plane(P_INP);
      float lm[NS];
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        if (s > 0) dec = sqrt_approx(dec);  // each accumulator on twice the timescale (HR:466-470)
        const float acc_old = in_plane(P_ACC + s);
        const float ms_old = in_plane(P_MS + s);
        const float acc = gi * (1.0f - dec) + acc_old * dec;                  // HR:483-484
        const float dk = zfl[s] ? 0.f : sd;                                   // utils.py:128-130
        const float ms = (1.0f - dk) * (acc * acc + 1e-12f) + dk * ms_old;    // utils.py:133-134
        const float r = acc * rsqrt_approx(ms + 1e-16f);
        sc[s] = log_fast(r + sqrt_approx(fmaf(r, r, 1.0f)));                  // utils.asinh as written (utils.py:36-38)
        lm[s] = log_fast(ms + 1e-16f);
        if (act) {
          state[(int64_t)(P_ACC + s) * n + i] = acc;
          state[(int64_t)(P_MS + s) * n + i] = ms;
          if (ms != 0.f) nz_mask |= 1 << s;
        }
      }
#pragma unroll
      for (int s = 0; s < NS; ++s) a[s] = sc[s];
#pragma unroll
      for (int s = 0; s < NS - 1; ++s) a[NS + s] = sc[s] * sc[s + 1];
      const float avg = (((lm[0] + lm[1]) + lm[2]) + lm[3]) / 4.0f;
#pragma unroll
      for (int s = 0; s < NS; ++s) a[2 * NS - 1 + s] = lm[s] - avg;
      a[F - 1] = llr - mean_llr;
    }
    float h[H0];
#pragma unroll
    for (int k = 0; k < H0; ++k) {
      h[k] = in_plane(P_H + k);
      a[F + k] = h[k];
    }
    a[F + H0] = 1.0f;
    a[F + H0 + 1] = 0.f;
#pragma unroll
    for (int c = 0; c < kKA / 4; ++c) st_split4(S.a1h, S.a1l, c, tid, a + 4 * c);
    if (act) {
#pragma unroll
      for (int k = 0; k < F; ++k) vals[H0 + k] += a[k];   // features as fed to the gates (HR:582-587 mean of [h' | feat])
    }
    fence_proxy_async();
    __syncthreads();   // A1 complete; the previous tile's reads of the row buffer are done
    wg_fence();
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
#pragma unroll
      for (int kc = 0; kc < kKA / 8; ++kc) {
        const uint64_t oa = hf * kHalfA + kc * kStepA;
        mma_ss_n48(d[hf], a1l + oa, d1h + kc * kStep1, kc > 0 ? 1u : 0u);
        mma_ss_n48(d[hf], a1h + oa, d1l + kc * kStep1, 1u);
        mma_ss_n48(d[hf], a1h + oa, d1h + kc * kStep1, 1u);
      }
    wg_commit();
    const float4* b0 = reinterpret_cast<const float4*>(w.bias0 + be.tensor * kB0Stride);
    float bq[12];
    {
      const float4 q0 = __ldg(b0), q1 = __ldg(b0 + 1), q2 = __ldg(b0 + 2);
      bq[0] = q0.x; bq[1] = q0.y; bq[2] = q0.z; bq[3] = q0.w; bq[4] = q1.x; bq[5] = q1.y; bq[6] = q1.z; bq[7] = q1.w;
      bq[8] = q2.x; bq[9] = q2.y; bq[10] = q2.z; bq[11] = q2.w;
    }
    wg_wait<0>();
    put_acc(d, 0, 4);   // r | u (columns 0..31)
    __syncthreads();
    // ---- reset gate, A2 = [r*h | 0]
    {
      float z[16];
      get10(0, z);
#pragma unroll
      for (int k = 0; k < H0; ++k) z[k] = sigmoid_fast(z[k] + bq[k]) * h[k];
#pragma unroll
      for (int k = H0; k < 16; ++k) z[k] = 0.f;
#pragma unroll
      for (int c = 0; c < kKA2 / 4; ++c) st_split4(S.a2h, S.a2l, c, tid, z + 4 * c);
    }
    fence_proxy_async();
    __syncthreads();
    wg_fence();
#pragma unroll
    for (int hf = 0; hf < 2; ++hf)
#pragma unroll
      for (int kc = 0; kc < kKA2 / 8; ++kc) {
        const uint64_t oa = hf * kHalfA + kc * kStepA;
        mma_ss_n16(d[hf] + 16, a2l + oa, d2h + kc * kStep2);
        mma_ss_n16(d[hf] + 16, a2h + oa, d2l + kc * kStep2);
        mma_ss_n16(d[hf] + 16, a2h + oa, d2h + kc * kStep2);
      }
    wg_commit();
    // ---- update gate while MMA 2 runs (columns 16..25 are not touched by it)
    float u[H0];
    {
      const float4 q3 = __ldg(b0 + 3), q4 = __ldg(b0 + 4);
      const float bu[H0] = {bq[10], bq[11], q3.x, q3.y, q3.z, q3.w, q4.x, q4.y, q4.z, q4.w};
      float z[H0];
      get10(kColU, z);
#pragma unroll
      for (int k = 0; k < H0; ++k) u[k] = sigmoid_fast(z[k] + bu[k]);
    }
    float bc[H0];
    {
      const float4 q5 = __ldg(b0 + 5), q6 = __ldg(b0 + 6), q7 = __ldg(b0 + 7);
      bc[0] = q5.x; bc[1] = q5.y; bc[2] = q5.z; bc[3] = q5.w; bc[4] = q6.x; bc[5] = q6.y; bc[6] = q6.z; bc[7] = q6.w;
      bc[8] = q7.x; bc[9] = q7.y;
    }
    wg_wait<0>();
    put_acc(d, 4, 6);   // candidate (columns 32..47)
    __syncthreads();
    float delta = 0.f, zs = 0.f, zi = 0.f, zl = 0.f;
    {
      float z[H0];
      get10(kColC, z);
#pragma unroll
      for (int k = 0; k < H0; ++k) {
        const float c = tanh_fast(z[k] + bc[k]);
        const float hn = u[k] * h[k] + (1.0f - u[k]) * c;      // rnn_cells.py:66-68
        if (act) {
          state[(int64_t)(P_H + k) * n + i] = hn;
          vals[k] += hn;
        }
        const float4 ro = S.ro[k];
        delta = fmaf(hn, ro.x, delta);                        // update direction (HR:609-611)
        zs = fmaf(hn, ro.y, zs);
        zi = fmaf(hn, ro.z, zi);
        zl = fmaf(hn, ro.w, zl);
      }
    }
    float short_cut = 0.f;                                      // gradient shortcut (HR:612-620), no bias
#pragma unroll
    for (int s = 0; s < NS; ++s) short_cut = fmaf(sc[s], S.cst[5 + s], short_cut);
    delta += short_cut;
    const float scl_new = sigmoid_fast(zs + S.cst[0]);          // HR:645-651
    const float inp_new = sigmoid_fast(zi + S.cst[1]);
    const float step_llr = fminf(fmaxf(llr + (zl + S.cst[2]), -33.0f), 33.0f);   // HR:667-683
    const float lrm = S.cst[3];
    const float llr_new = lrm * llr + (1.0f - lrm) * step_llr;  // HR:688-689
    const float lr_param = exp_fast(step_llr + S.cst[4]);       // HR:692
    if (act) {
      state[(int64_t)P_SCL * n + i] = scl_new;
      state[(int64_t)P_INP * n + i] = inp_new;
      state[(int64_t)P_LLR * n + i] = llr_new;
      w.upd[i] = lr_param * delta;   // the per-tensor 1/RMS(delta) is applied by apply_kernel
      vals[H0 + F] += delta * delta;
      vals[H0 + F + 1] += llr_new;
    }
  }
  if (cur_tensor >= 0) flush(cur_tensor);
}

}  // namespace tcg
