// HierarchicalRNN per-parameter level, BACKWARD (meta-training: BPTT through l2o_hrnn_step; included by l2o_hrnn.cu
// inside namespace l2o::hrnn).  Reference: the TF autodiff of HR:444-540 (features), rnn_cells.py:46-68 (BiasGRU),
// HR:606-706 (readouts) as driven by SC/optimizer/trainable_optimizer.py:200-470.  The reference stop_gradient's the
// optimizee's gradients only when use_second_derivatives is off (:330-338; its default is on): with a null d_g, g is a
// constant here; otherwise the kernel also writes d g, the per-coordinate part of the second-order term (the optimizee's
// Hessian-vector product that carries it on to x belongs to the caller).
//
// One thread = one coordinate: recompute the forward step from the planes BEFORE the step (exact-fp32 FFMA, the same
// MUFU forms as the forward kernels), then walk it backwards.  Inputs: adjoints of the 21 new planes, of the raw update
// lr*delta (w.upd, before the per-tensor 1/RMS) and of the 24 per-tensor sums (broadcast to the tensor's coordinates).
// Outputs: adjoints of the 21 old planes; d theta of the 739 per-parameter-level weights; per-tensor d bias0 (the
// injected gate bias) and d mean_log_lr; optionally d g.  g enters only through the four accumulators
// acc'_s = g (1 - d_s) + acc_s d_s, so d g = sum_s d acc'_s (1 - d_s); the tensor-wide ALL(ms == 0) first-step predicate
// is piecewise constant and has no derivative.  The cross-coordinate pieces (per-tensor / global GRUs, 1/RMS(delta), the
// problem-wide mean log-lr, the objective) are tiny and live on the host side as torch autograd (hrnn_train.py).
//
// Reductions: every per-coordinate contribution is summed over the warp with a shuffle butterfly and added to a
// per-CTA shared-memory image of d theta; persistent CTAs flush the image into the fp64 accumulators when they are done
// (d bias0 / d mean_log_lr: whenever the tensor changes).  Correctness first: ~8 K instructions per warp-tile, meant for
// the problem sizes L2O-Scale meta-trains on (BASELINE config #4: 354 K coordinates x 20 steps = 2 ms of this kernel).
#pragma once

namespace bwd {

constexpr int kBwdBlock = 128;
constexpr int kImg = 768;   // shared d-theta image: Wg 440 | bg 20 | Wc 220 | bc 10 | Wu Ws Wi Wl 40 | bs bi bl 3 | g2d 4 | lrm off 2
constexpr int I_WG = 0, I_BG = 440, I_WC = 460, I_BC = 680, I_WU = 690, I_WS = 700, I_WI = 710, I_WL = 720;
constexpr int I_BS = 730, I_BI = 731, I_BL = 732, I_G2D = 733, I_LRM = 737, I_OFF = 738, I_N = 739;
constexpr int kTen = 32;    // per-tensor image: d bias0 [30] | d mean_log_lr [1]

struct Args {
  const float* theta;
  const float* state_old;   // [21][n]
  const float* g;           // [n]
  const float* bias0;       // [nt][kB0Stride]
  const int* zero_flag;     // [nt][NS]
  const float* mean_log_lr; // [1]
  const float* d_state_new; // [21][n]
  const float* d_upd;       // [n]
  const float* d_sums;      // [nt][kAcc]
  float* d_state_old;       // [21][n]
  double* d_theta;          // [kTheta] +=
  double* d_bias0;          // [nt][kB0Stride] +=
  double* d_mean_log_lr;    // [1] +=
  float* d_g;               // [n] or null
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ int theta_index(int k) {   // shared image slot -> flat theta offset
  if (k < I_BG) return O_WG0 + k;
  if (k < I_WC) return O_BG0 + (k - I_BG);
  if (k < I_BC) return O_WC0 + (k - I_WC);
  if (k < I_WU) return O_BC0 + (k - I_BC);
  if (k < I_WS) return O_WU + (k - I_WU);
  if (k < I_WI) return O_WS + (k - I_WS);
  if (k < I_WL) return O_WI + (k - I_WI);
  if (k < I_BS) return O_WL + (k - I_WL);
  if (k == I_BS) return O_BS;
  if (k == I_BI) return O_BI;
  if (k == I_BL) return O_BL;
  if (k < I_LRM) return O_G2D + (k - I_G2D);
  if (k == I_LRM) return O_LRM;
  return O_OFF;
}

__global__ void __launch_bounds__(kBwdBlock) coord_bwd_kernel(Args a, int64_t n, const BlockEnt* __restrict__ blocks, int ntiles) {
  __shared__ float sWg[(F + H0) * 2 * H0];
  __shared__ float sWc[(F + H0) * H0];
  __shared__ float sRo[4 * H0];        // Wu | Ws | Wi | Wl
  __shared__ float sC[40];             // bg 20 | bc 10 | bs bi bl | lrm(sigmoid) | off | g2d 4
  __shared__ float sImg[kImg];
  __shared__ float sTen[kTen];
  const int tid = threadIdx.x, lane = tid & 31;
  for (int k = tid; k < (F + H0) * 2 * H0; k += kBwdBlock) sWg[k] = a.theta[O_WG0 + k];
  for (int k = tid; k < (F + H0) * H0; k += kBwdBlock) sWc[k] = a.theta[O_WC0 + k];
  if (tid < H0) {
    sRo[tid] = a.theta[O_WU + tid];
    sRo[H0 + tid] = a.theta[O_WS + tid];
    sRo[2 * H0 + tid] = a.theta[O_WI + tid];
    sRo[3 * H0 + tid] = a.theta[O_WL + tid];
  }
  if (tid < 2 * H0) sC[tid] = a.theta[O_BG0 + tid];
  if (tid < H0) sC[20 + tid] = a.theta[O_BC0 + tid];
  if (tid == 0) {
    sC[30] = a.theta[O_BS];
    sC[31] = a.theta[O_BI];
    sC[32] = a.theta[O_BL];
    sC[33] = sigmoid_fast(a.theta[O_LRM]);
    sC[34] = a.theta[O_OFF];
    for (int s = 0; s < NS; ++s) sC[35 + s] = a.theta[O_G2D + s];
  }
  for (int k = tid; k < kImg; k += kBwdBlock) sImg[k] = 0.f;
  if (tid < kTen) sTen[tid] = 0.f;
  __syncthreads();
  auto add_img = [&](int slot, float v) {   // warp sum -> one shared atomic
    v = warp_sum(v);
    if (lane == 0) atomicAdd(&sImg[slot], v);
  };
  auto add_ten = [&](int slot, float v) {
    v = warp_sum(v);
    if (lane == 0) atomicAdd(&sTen[slot], v);
  };
  auto flush_ten = [&](int tensor) {
    __syncthreads();
    if (tid < 3 * H0) atomicAdd(&a.d_bias0[tensor * kB0Stride + tid], (double)sTen[tid]);
    if (tid == 3 * H0) atomicAdd(a.d_mean_log_lr, (double)sTen[tid]);
    __syncthreads();
    if (tid < kTen) sTen[tid] = 0.f;
    __syncthreads();
  };
  const float mean_llr = *a.mean_log_lr;
  int cur_tensor = -1;
  for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const BlockEnt be = blocks[tile];
    if (be.tensor != cur_tensor) {
      if (cur_tensor >= 0) flush_ten(cur_tensor);
      cur_tensor = be.tensor;
    }
    const bool act = tid < be.count;
    const int64_t i = be.start + (act ? tid : 0);
    // ------------------------------------------------------------------ forward recompute
    float h[H0], in[F], sc[NS], accv[NS], acc_old[NS], ms_old[NS], dec[NS], rs[NS], wv[NS], tt[NS], dk[NS], q[NS];
    int zf[NS];
#pragma unroll
    for (int k = 0; k < H0; ++k) h[k] = act ? a.state_old[(int64_t)(P_H + k) * n + i] : 0.f;
    const float sd = act ? a.state_old[(int64_t)P_SCL * n + i] : 0.f;
    const float d0 = act ? a.state_old[(int64_t)P_INP * n + i] : 0.f;
    const float llr = act ? a.state_old[(int64_t)P_LLR * n + i] : 0.f;
    const float gi = act ? a.g[i] : 0.f;
    dec[0] = d0;
#pragma unroll
    for (int s = 1; s < NS; ++s) dec[s] = sqrt_approx(dec[s - 1]);
    float lm[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      zf[s] = a.zero_flag[be.tensor * NS + s];
      acc_old[s] = act ? a.state_old[(int64_t)(P_ACC + s) * n + i] : 0.f;
      ms_old[s] = act ? a.state_old[(int64_t)(P_MS + s) * n + i] : 0.f;
      accv[s] = gi * (1.0f - dec[s]) + acc_old[s] * dec[s];
      dk[s] = zf[s] ? 0.f : sd;
      q[s] = accv[s] * accv[s] + 1e-12f;
      const float ms = (1.0f - dk[s]) * q[s] + dk[s] * ms_old[s];
      wv[s] = ms + 1e-16f;
      rs[s] = rsqrt_approx(wv[s]);
      const float r = accv[s] * rs[s];
      tt[s] = sqrt_approx(fmaf(r, r, 1.0f));
      sc[s] = log_fast(r + tt[s]);
      lm[s] = log_fast(wv[s]);
    }
#pragma unroll
    for (int s = 0; s < NS; ++s) in[s] = sc[s];
#pragma unroll
    for (int s = 0; s < NS - 1; ++s) in[NS + s] = sc[s] * sc[s + 1];
    const float avg = (((lm[0] + lm[1]) + lm[2]) + lm[3]) / 4.0f;
#pragma unroll
    for (int s = 0; s < NS; ++s) in[2 * NS - 1 + s] = lm[s] - avg;
    in[F - 1] = llr - mean_llr;
    const float* b0 = a.bias0 + be.tensor * kB0Stride;
    float rg[H0], ug[H0], cg[H0], hn[H0];
    {
      float pg[2 * H0];
#pragma unroll
      for (int o = 0; o < 2 * H0; ++o) pg[o] = 0.f;
#pragma unroll
      for (int k = 0; k < F + H0; ++k) {
        const float v = k < F ? in[k] : h[k - F];
#pragma unroll
        for (int o = 0; o < 2 * H0; ++o) pg[o] = fmaf(v, sWg[k * 2 * H0 + o], pg[o]);
      }
#pragma unroll
      for (int k = 0; k < H0; ++k) {
        rg[k] = sigmoid_fast((pg[k] + sC[k]) + b0[k]);
        ug[k] = sigmoid_fast((pg[H0 + k] + sC[H0 + k]) + b0[H0 + k]);
      }
      float pc[H0];
#pragma unroll
      for (int o = 0; o < H0; ++o) pc[o] = 0.f;
#pragma unroll
      for (int k = 0; k < F + H0; ++k) {
        const float v = k < F ? in[k] : rg[k - F] * h[k - F];
#pragma unroll
        for (int o = 0; o < H0; ++o) pc[o] = fmaf(v, sWc[k * H0 + o], pc[o]);
      }
#pragma unroll
      for (int k = 0; k < H0; ++k) {
        cg[k] = tanh_fast((pc[k] + sC[20 + k]) + b0[2 * H0 + k]);
        hn[k] = ug[k] * h[k] + (1.0f - ug[k]) * cg[k];
      }
    }
    float delta = 0.f, zs = 0.f, zi = 0.f, zl = 0.f;
#pragma unroll
    for (int k = 0; k < H0; ++k) {
      delta = fmaf(hn[k], sRo[k], delta);
      zs = fmaf(hn[k], sRo[H0 + k], zs);
      zi = fmaf(hn[k], sRo[2 * H0 + k], zi);
      zl = fmaf(hn[k], sRo[3 * H0 + k], zl);
    }
#pragma unroll
    for (int s = 0; s < NS; ++s) delta = fmaf(sc[s], sC[35 + s], delta);
    const float scl_n = sigmoid_fast(zs + sC[30]);
    const float inp_n = sigmoid_fast(zi + sC[31]);
    const float step = fminf(fmaxf(llr + (zl + sC[32]), -33.0f), 33.0f);
    const float m = sC[33];
    const float lr = exp_fast(step + sC[34]);
    // ------------------------------------------------------------------ backward
    const float* ds = a.d_sums + be.tensor * kAcc;
    float dhn[H0], din[F];
#pragma unroll
    for (int k = 0; k < H0; ++k) dhn[k] = act ? a.d_state_new[(int64_t)(P_H + k) * n + i] + ds[k] : 0.f;
#pragma unroll
    for (int k = 0; k < F; ++k) din[k] = act ? ds[H0 + k] : 0.f;
    const float D_upd = act ? a.d_upd[i] : 0.f;
    const float ddelta = act ? D_upd * lr + 2.0f * delta * ds[H0 + F] : 0.f;
    const float dlr = D_upd * delta;
    const float dllrn = act ? a.d_state_new[(int64_t)P_LLR * n + i] + ds[H0 + F + 1] : 0.f;
    const float dstep = dlr * lr + (1.0f - m) * dllrn;
    float dllr = m * dllrn + dstep;                         // straight-through clip (HR:678-686): d pre = d step
    const float dzl = dstep;
    const float dzs = act ? a.d_state_new[(int64_t)P_SCL * n + i] * scl_n * (1.0f - scl_n) : 0.f;
    const float dzi = act ? a.d_state_new[(int64_t)P_INP * n + i] * inp_n * (1.0f - inp_n) : 0.f;
    add_img(I_OFF, dlr * lr);
    add_img(I_LRM, (llr - step) * dllrn * m * (1.0f - m));
    add_img(I_BL, dzl);
    add_img(I_BS, dzs);
    add_img(I_BI, dzi);
#pragma unroll
    for (int k = 0; k < H0; ++k) {
      add_img(I_WU + k, ddelta * hn[k]);
      add_img(I_WS + k, dzs * hn[k]);
      add_img(I_WI + k, dzi * hn[k]);
      add_img(I_WL + k, dzl * hn[k]);
      dhn[k] += ddelta * sRo[k] + dzs * sRo[H0 + k] + dzi * sRo[2 * H0 + k] + dzl * sRo[3 * H0 + k];
    }
    float dsc[NS];
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      dsc[s] = ddelta * sC[35 + s];
      add_img(I_G2D + s, ddelta * sc[s]);
    }
    // BiasGRU backward
    float dh[H0], dpc[H0], dpg[2 * H0];
#pragma unroll
    for (int k = 0; k < H0; ++k) {
      dpg[H0 + k] = dhn[k] * (h[k] - cg[k]) * ug[k] * (1.0f - ug[k]);
      dpc[k] = dhn[k] * (1.0f - ug[k]) * (1.0f - cg[k] * cg[k]);
      dh[k] = dhn[k] * ug[k];
    }
#pragma unroll
    for (int k = 0; k < F + H0; ++k) {   // candidate affine: input [in | r*h]
      const float v = k < F ? in[k] : rg[k - F] * h[k - F];
      float dv = 0.f;
#pragma unroll
      for (int o = 0; o < H0; ++o) {
        dv = fmaf(dpc[o], sWc[k * H0 + o], dv);
        add_img(I_WC + k * H0 + o, v * dpc[o]);
      }
      if (k < F) din[k] += dv;
      else {
        const int j = k - F;
        dpg[j] = dv * h[j] * rg[j] * (1.0f - rg[j]);
        dh[j] += dv * rg[j];
      }
    }
#pragma unroll
    for (int o = 0; o < H0; ++o) {
      add_img(I_BC + o, dpc[o]);
      add_ten(2 * H0 + o, dpc[o]);
    }
#pragma unroll
    for (int k = 0; k < F + H0; ++k) {   // gate affine: input [in | h]
      const float v = k < F ? in[k] : h[k - F];
      float dv = 0.f;
#pragma unroll
      for (int o = 0; o < 2 * H0; ++o) {
        dv = fmaf(dpg[o], sWg[k * 2 * H0 + o], dv);
        add_img(I_WG + k * 2 * H0 + o, v * dpg[o]);
      }
      if (k < F) din[k] += dv;
      else dh[k - F] += dv;
    }
#pragma unroll
    for (int o = 0; o < 2 * H0; ++o) {
      add_img(I_BG + o, dpg[o]);
      add_ten(o, dpg[o]);
    }
    // features backward
    dllr += din[F - 1];
    add_ten(3 * H0, -din[F - 1]);
    const float dlm_mean = (((din[2 * NS - 1] + din[2 * NS]) + din[2 * NS + 1]) + din[2 * NS + 2]) / 4.0f;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      dsc[s] += din[s];
      if (s < NS - 1) dsc[s] += din[NS + s] * sc[s + 1];
      if (s > 0) dsc[s] += din[NS + s - 1] * sc[s - 1];
    }
    const bool want_dg = a.d_g != nullptr;
    float dsd = 0.f, ddec[NS], dacc_old[NS], dms_old[NS], dg = 0.f;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      const float dr = dsc[s] / tt[s];
      float dacc = (act ? a.d_state_new[(int64_t)(P_ACC + s) * n + i] : 0.f) + dr * rs[s];
      const float dlm = din[2 * NS - 1 + s] - dlm_mean;
      const float dw = dr * accv[s] * (-0.5f * rs[s] * rs[s] * rs[s]) + dlm / wv[s];
      const float dms = (act ? a.d_state_new[(int64_t)(P_MS + s) * n + i] : 0.f) + dw;
      dacc += dms * (1.0f - dk[s]) * 2.0f * accv[s];
      dms_old[s] = dms * dk[s];
      if (!zf[s]) dsd += dms * (ms_old[s] - q[s]);
      dacc_old[s] = dacc * dec[s];
      ddec[s] = dacc * (acc_old[s] - gi);
      if (want_dg) dg += dacc * (1.0f - dec[s]);
    }
#pragma unroll
    for (int s = NS - 1; s > 0; --s) ddec[s - 1] += dec[s] > 0.f ? ddec[s] * 0.5f / dec[s] : 0.f;
    if (act) {
#pragma unroll
      for (int k = 0; k < H0; ++k) a.d_state_old[(int64_t)(P_H + k) * n + i] = dh[k];
      a.d_state_old[(int64_t)P_SCL * n + i] = dsd;
      a.d_state_old[(int64_t)P_INP * n + i] = ddec[0];
      a.d_state_old[(int64_t)P_LLR * n + i] = dllr;
#pragma unroll
      for (int s = 0; s < NS; ++s) {
        a.d_state_old[(int64_t)(P_ACC + s) * n + i] = dacc_old[s];
        a.d_state_old[(int64_t)(P_MS + s) * n + i] = dms_old[s];
      }
      if (want_dg) a.d_g[i] = dg;
    }
  }
  if (cur_tensor >= 0) flush_ten(cur_tensor);
  __syncthreads();
  for (int k = tid; k < I_N; k += kBwdBlock) atomicAdd(&a.d_theta[theta_index(k)], (double)sImg[k]);
}

}  // namespace bwd
