// MNIST ConvNet producer (DM/problems.py:291-347 `mnist_conv`, batch_norm=True, + tf.gradients at DM/meta.py:322-329):
// f and df/dx of
//   f = mean_b xent(ReLU(fc(pool(ReLU(BN(conv2(pool(ReLU(BN(conv1(images[idx_b] / 255))))))))), labels[idx_b])
// in ONE launch, with idx_b drawn afresh at every evaluation by l2o_philox.cuh's draw, as l2o_mnist_grad draws it.
//
// Spec points (each restated from the reference):
//   - the variables, in creation order (DM/problems.py:312-318,330-337): conv_layer1/weights1 [3][3][1][16] (HWIO),
//     conv_layer1/biases1 [16], conv_layer2/weights1 [5][5][16][32], conv_layer2/biases1 [32], fc_weights [512][10],
//     fc_bias [10];
//   - batch norm (DM/problems.py:321-322) is tf.layers.batch_normalization in training mode: per channel, the mean and
//     the biased variance over all B*H*W positions, eps 1e-3.  Its gamma and beta are NOT optimizee variables
//     (DM/meta.py:88-99 patches tf.get_variable only; tf.layers creates them through variable_scope.get_variable), so
//     inside every evaluation gamma = 1 and beta = 0;
//   - the conv biases go through the chain rule like every other entry: BN removes the per-channel mean, so their true
//     gradient is zero and what this kernel writes is fp32 rounding noise;
//   - max-pool 2x2 stride 2 VALID (DM/problems.py:305-308): [26,26] -> [13,13] and [9,9] -> [4,4] (row and column 8
//     dropped); the gradient goes to the first maximum in row-major window order (ties only occur between ReLU zeros,
//     whose gradient ReLU' = 0 removes);
//   - the flatten is tf.reshape([B, -1]) of NHWC (DM/problems.py:328): feature (h * 4 + w) * 32 + c;
//   - the logits pass through a ReLU (DM/problems.py:338) before the mean sparse softmax cross entropy.
//
// Design.  A cooperative launch over at most the resident CTAs (one per SM at this shared-memory size).  Images are
// striped over the CTAs, b = blockIdx.x + k * gridDim.x, so every stage of image b runs on the same CTA.  Five grid-wide
// barriers separate the stages at the batch-wide points:
//   1  conv1 -> z1 (workspace), per-image BN1 statistics (mean, M2) in fp64
//   -- sync: BN1 statistics --
//   2  BN1, ReLU, pool -> p1 (shared), conv2 (W2 staged once per CTA in shared memory) -> z2, per-image BN2 statistics
//   -- sync: BN2 statistics --
//   3  BN2, ReLU, pool -> p2, fc, ReLU, cross entropy, dlogits; dp2 routed back to dy2; per-image BN2 backward sums
//   -- sync: BN2 backward sums --
//   4  dz2 = BN2 backward; dW2 and db2 of the image; dp1 = conv2 transposed; routed to the pool1 maxima; per-image
//      BN1 backward sums
//   -- sync: BN1 backward sums --
//   5  dz1 = BN1 backward; dW1 and db1 of the image
//   -- sync: the final reduction --
// Each image writes its partials to the workspace (the statistics, the backward sums and its dW / db slices), and every
// batch-wide quantity is a sum over b = 0..B-1 in a fixed order that depends on B only: the same inputs give bitwise
// identical f and g on any number of SMs, with no atomics.  The BN statistics of equal-count groups merge with Chan's
// formula in fp64 (mu = sum mean_b / B, M2 = sum_b M2_b + n (mean_b - mu)^2), never E[z^2] - E[z]^2, which cancels
// when |mu| >> sigma.  fc's weight gradient is sum_b p2_b (x) dlogits_b, formed in the final reduction from the
// per-image p2 and dlogits.
// Random scaling (DM/meta_dm_train.py:336-338,384-385) as l2o_lasso_grad: the loss at x (.) scale, g multiplied by scale.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include "l2o_bn.cuh"
#include "l2o_internal.h"
#include "l2o_philox.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr int kIn = 28, kH1 = 26, kP1 = 13, kH2 = 9, kP2 = 4;
constexpr int kC1 = 16, kC2 = 32, kCls = L2O_MNIST_CLASSES, kFc = kP2 * kP2 * kC2;   // 512
constexpr int kZ1 = kH1 * kH1 * kC1;      // 10816
constexpr int kQ1 = kP1 * kP1 * kC1;      // 2704 pooled conv1 cells
constexpr int kZ2 = kH2 * kH2 * kC2;      // 2592
constexpr int kW2 = 5 * 5 * kC1 * kC2;    // 12800
// arena offsets (creation order)
constexpr int oW1 = 0, oB1 = oW1 + 9 * kC1, oW2 = oB1 + kC1, oB2 = oW2 + kW2, oWf = oB2 + kC2, oBf = oWf + kFc * kCls;
constexpr int kCoords = oBf + kCls;
static_assert(kCoords == L2O_MNIST_CONV_COORDS, "arena size");
constexpr int kPart = oWf;                // per-image partial gradient: W1, b1, W2, b2 (fc from p2 and dlogits)
constexpr int kP1S = 17;                  // shared p1 position stride (16 channels + 1: conflict-free column reads)
constexpr int kPad = kH2 + 8;             // dz2 zero-padded by 4 on each side for the transposed conv
constexpr int kPadS = 33;                 // its position stride
constexpr float kEps = 1e-3f;             // tf.layers.batch_normalization's default epsilon

__host__ __device__ inline size_t up16(size_t v) { return (v + 15) & ~(size_t)15; }

// the workspace: per-image statistics and backward sums (fp64), the activations that cross a grid barrier, and each
// image's partial gradient
struct Ws {
  double2 *st1, *st2, *bk2, *bk1;   // [B][C]: (mean, M2) / (sum dy, sum dy * yhat)
  double* loss;                     // [B]
  float *z1, *z2, *dy2, *dyc;       // [B][kZ1], [B][kZ2], [B][kZ2], [B][kQ1] (dp1 routed to the pool1 maximum)
  float *part, *p2, *dl;            // [B][kPart], [B][kFc], [B][16]
  float* bn;                        // [96]: mu1 [16], rstd1 [16], mu2 [32], rstd2 [32] as the kernel applies them
  uint8_t* code;                    // [B][kQ1]: the pool1 maximum's place in its window
};

size_t ws_layout(int B, char* base, Ws* w) {
  size_t off = 0;
  auto take = [&](size_t bytes) {
    char* p = (char*)((uintptr_t)base + off);   // a null base gives the byte offsets
    off = up16(off + bytes);
    return p;
  };
  const size_t b = (size_t)B;
  Ws t;
  t.st1 = (double2*)take(b * kC1 * sizeof(double2));
  t.st2 = (double2*)take(b * kC2 * sizeof(double2));
  t.bk2 = (double2*)take(b * kC2 * sizeof(double2));
  t.bk1 = (double2*)take(b * kC1 * sizeof(double2));
  t.loss = (double*)take(b * sizeof(double));
  t.z1 = (float*)take(b * kZ1 * sizeof(float));
  t.z2 = (float*)take(b * kZ2 * sizeof(float));
  t.dy2 = (float*)take(b * kZ2 * sizeof(float));
  t.dyc = (float*)take(b * kQ1 * sizeof(float));
  t.part = (float*)take(b * kPart * sizeof(float));
  t.p2 = (float*)take(b * kFc * sizeof(float));
  t.dl = (float*)take(b * 16 * sizeof(float));
  t.code = (uint8_t*)take(b * kQ1);
  t.bn = (float*)take(2 * (kC1 + kC2) * sizeof(float));
  if (w) *w = t;
  return off;
}

// shared memory (floats)
constexpr int sW2 = 0;                          // [kW2] conv2 weights (scaled), HWIO
constexpr int sU = sW2 + kW2;                   // union: z1 [kZ1] | padded dz2 [kPad^2][kPadS] | dz1 [kZ1]
constexpr int sP1 = sU + kZ1;                   // [169][kP1S] pooled conv1 activations
constexpr int sZ2 = sP1 + 169 * kP1S + 3;       // [kZ2] z2 / dy2 / dz2
constexpr int sX = sZ2 + kZ2;                   // [784] the image
constexpr int sP2 = sX + kIn * kIn;             // [kFc]
constexpr int sDyc = sP2 + kFc;                 // [kQ1] routed dp1 | stage-5 dW1 partials
constexpr int sYs = sDyc + kQ1;                 // [kQ1] yhat1 at the pool1 maximum
constexpr int sCode = sYs + kQ1;                // [kQ1] bytes
constexpr int sW1 = sCode + kQ1 / 4;            // [144]
constexpr int sPc = sW1 + 9 * kC1;              // per-channel: mu1, rs1, ma1, mb1 [16 each]; mu2, rs2, ma2, mb2 [32 each]
constexpr int sLog = sPc + 4 * kC1 + 4 * kC2;   // [16] logits, then [16] dlogits
constexpr int kSmemFloats = sLog + 32;
static_assert(kPad * kPad * kPadS <= kZ1, "padded dz2 fits the union");
static_assert(sZ2 % 4 == 0 && sU % 4 == 0 && sW2 % 4 == 0, "float4 alignment");
constexpr size_t kSmem = (size_t)kSmemFloats * sizeof(float) + kThreads * sizeof(double);

struct Args {
  l2o_mnist_conv_args a;
  Ws w;
};

// BN1, ReLU and max-pool of image b from its z1 in the workspace: p1 and the maxima's window places in shared memory
__device__ void pool1(const float* z1, float* sm) {
  const float* mu = sm + sPc;
  const float* rs = mu + kC1;
  uint8_t* code = reinterpret_cast<uint8_t*>(sm + sCode);
  for (int e = threadIdx.x; e < kQ1; e += kThreads) {
    const int c = e & (kC1 - 1), q = e >> 4, pi = q / kP1, pj = q - pi * kP1;
    float best = 0.f;
    int arg = 0;
#pragma unroll
    for (int w = 0; w < 4; ++w) {
      const int p = (2 * pi + (w >> 1)) * kH1 + 2 * pj + (w & 1);
      const float a = fmaxf((z1[p * kC1 + c] - mu[c]) * rs[c], 0.f);
      if (w == 0 || a > best) {   // the first maximum in row-major window order
        best = a;
        arg = w;
      }
    }
    sm[sP1 + q * kP1S + c] = best;
    code[e] = (uint8_t)arg;
  }
}

__global__ void __launch_bounds__(kThreads, 1) mnist_conv_kernel(const Args args) {
  extern __shared__ __align__(16) float sm[];
  double* red = reinterpret_cast<double*>(sm + kSmemFloats);
  __shared__ double mu_tmp[kC2];
  const l2o_mnist_conv_args& a = args.a;
  const Ws& w = args.w;
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int B = a.batch, G = gridDim.x;
  const float* __restrict__ x = a.x;
  const float* __restrict__ sc = a.scale;
  auto wv = [&](int o) { return sc ? x[o] * sc[o] : x[o]; };
  float* mu1 = sm + sPc;
  float* rs1 = mu1 + kC1;
  float* ma1 = rs1 + kC1;
  float* mb1 = ma1 + kC1;
  float* mu2 = mb1 + kC1;
  float* rs2 = mu2 + kC2;
  float* ma2 = rs2 + kC2;
  float* mb2 = ma2 + kC2;
  const uint64_t ctr = (uint64_t)*a.counter;
  auto load_image = [&](int b) {
    const int idx = l2o::batch_index(a.seed, ctr, b, a.num_examples);
    for (int e = tid; e < kIn * kIn; e += kThreads) sm[sX + e] = l2o::mnist_pixel(a.images[(size_t)idx * 784 + e]);
    return idx;
  };

  for (int e = tid; e < kW2 / 4; e += kThreads) {
    float4 v = reinterpret_cast<const float4*>(x + oW2)[e];
    if (sc) {
      const float4 s = reinterpret_cast<const float4*>(sc + oW2)[e];
      v.x *= s.x, v.y *= s.y, v.z *= s.z, v.w *= s.w;
    }
    reinterpret_cast<float4*>(sm + sW2)[e] = v;
  }
  for (int e = tid; e < 9 * kC1; e += kThreads) sm[sW1 + e] = wv(oW1 + e);

  // ---- 1: conv1 + b1 -> z1; the image's BN1 statistics ------------------------------------------------------------
  for (int b = blockIdx.x; b < B; b += G) {
    const int idx = load_image(b);
    if (tid == 0 && a.idx_out) a.idx_out[b] = idx;
    __syncthreads();
    const int c = tid & (kC1 - 1), q = tid >> 4;
    float wk[9];
#pragma unroll
    for (int k = 0; k < 9; ++k) wk[k] = sm[sW1 + k * kC1 + c];
    const float bias = wv(oB1 + c);
    float* z1 = w.z1 + (size_t)b * kZ1;
    double s = 0.0;
    for (int p = q; p < kH1 * kH1; p += kThreads / kC1) {
      const int i = p / kH1, j = p - i * kH1;
      float acc = 0.f;
#pragma unroll
      for (int kh = 0; kh < 3; ++kh)
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) acc = fmaf(sm[sX + (i + kh) * kIn + j + kw], wk[kh * 3 + kw], acc);
      const float z = acc + bias;
      sm[sU + p * kC1 + c] = z;
      z1[p * kC1 + c] = z;
      s += (double)z;
    }
    s = l2o::chan_sum<kThreads>(red, s, kC1);
    if (tid < kC1) mu_tmp[tid] = s / (double)(kH1 * kH1);
    __syncthreads();
    const double m = mu_tmp[c];
    double m2 = 0.0;
    for (int p = q; p < kH1 * kH1; p += kThreads / kC1) {
      const double d = (double)sm[sU + p * kC1 + c] - m;
      m2 += d * d;
    }
    m2 = l2o::chan_sum<kThreads>(red, m2, kC1);
    if (tid < kC1) w.st1[(size_t)b * kC1 + tid] = make_double2(mu_tmp[tid], m2);
  }
  grid.sync();
  l2o::merge_stats<kThreads>(w.st1, B, kC1, kH1 * kH1, kEps, red, mu1, rs1, mu_tmp);
  if (blockIdx.x == 0 && tid < kC1) {   // every CTA holds the same values; CTA 0 records them for the caller
    w.bn[tid] = mu1[tid];
    w.bn[kC1 + tid] = rs1[tid];
  }

  // ---- 2: BN1, ReLU, pool -> p1; conv2 + b2 -> z2; the image's BN2 statistics --------------------------------------
  for (int b = blockIdx.x; b < B; b += G) {
    pool1(w.z1 + (size_t)b * kZ1, sm);
    __syncthreads();
    {   // warp = 4 output channels, lane = positions lane, lane + 32, lane + 64
      const int og = warp;
      int base[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int pos = min(lane + 32 * k, kH2 * kH2 - 1), i = pos / kH2, j = pos - i * kH2;
        base[k] = (i * kP1 + j) * kP1S;
      }
      float acc[3][4] = {};
      for (int kh = 0; kh < 5; ++kh)
        for (int kw = 0; kw < 5; ++kw) {
          const int roff = (kh * kP1 + kw) * kP1S;
          const float* wr = sm + sW2 + (kh * 5 + kw) * kC1 * kC2 + og * 4;
#pragma unroll 4
          for (int c = 0; c < kC1; ++c) {
            const float4 wq = *reinterpret_cast<const float4*>(wr + c * kC2);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
              const float v = sm[sP1 + base[k] + roff + c];
              acc[k][0] = fmaf(v, wq.x, acc[k][0]);
              acc[k][1] = fmaf(v, wq.y, acc[k][1]);
              acc[k][2] = fmaf(v, wq.z, acc[k][2]);
              acc[k][3] = fmaf(v, wq.w, acc[k][3]);
            }
          }
        }
      float* z2 = w.z2 + (size_t)b * kZ2;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int pos = lane + 32 * k;
        if (pos < kH2 * kH2) {
          float4 z;
          z.x = acc[k][0] + wv(oB2 + og * 4 + 0);
          z.y = acc[k][1] + wv(oB2 + og * 4 + 1);
          z.z = acc[k][2] + wv(oB2 + og * 4 + 2);
          z.w = acc[k][3] + wv(oB2 + og * 4 + 3);
          *reinterpret_cast<float4*>(sm + sZ2 + pos * kC2 + og * 4) = z;
          *reinterpret_cast<float4*>(z2 + pos * kC2 + og * 4) = z;
        }
      }
    }
    __syncthreads();
    const int c = tid & (kC2 - 1), q = tid >> 5;
    double s = 0.0;
    for (int p = q; p < kH2 * kH2; p += kThreads / kC2) s += (double)sm[sZ2 + p * kC2 + c];
    s = l2o::chan_sum<kThreads>(red, s, kC2);
    if (tid < kC2) mu_tmp[tid] = s / (double)(kH2 * kH2);
    __syncthreads();
    const double m = mu_tmp[c];
    double m2 = 0.0;
    for (int p = q; p < kH2 * kH2; p += kThreads / kC2) {
      const double d = (double)sm[sZ2 + p * kC2 + c] - m;
      m2 += d * d;
    }
    m2 = l2o::chan_sum<kThreads>(red, m2, kC2);
    if (tid < kC2) w.st2[(size_t)b * kC2 + tid] = make_double2(mu_tmp[tid], m2);
  }
  grid.sync();
  l2o::merge_stats<kThreads>(w.st2, B, kC2, kH2 * kH2, kEps, red, mu2, rs2, mu_tmp);
  if (blockIdx.x == 0 && tid < kC2) {
    w.bn[2 * kC1 + tid] = mu2[tid];
    w.bn[2 * kC1 + kC2 + tid] = rs2[tid];
  }

  // ---- 3: BN2, ReLU, pool -> p2; fc, ReLU, cross entropy; dlogits -> dp2 -> dy2; the BN2 backward sums -----------
  for (int b = blockIdx.x; b < B; b += G) {
    const int idx = l2o::batch_index(a.seed, ctr, b, a.num_examples);
    const int y = a.labels[idx];
    const float* z2 = w.z2 + (size_t)b * kZ2;
    int cpos[2];
    float cy[2];
#pragma unroll
    for (int k = 0; k < 2; ++k) {   // feature e = (h * 4 + w) * 32 + c, the NHWC flatten
      const int e = tid + kThreads * k, c = e & (kC2 - 1), q = e >> 5, pi = q >> 2, pj = q & 3;
      float best = 0.f, ybest = 0.f;
      int arg = 0;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const int p = (2 * pi + (t >> 1)) * kH2 + 2 * pj + (t & 1);
        const float yh = (z2[p * kC2 + c] - mu2[c]) * rs2[c];
        const float av = fmaxf(yh, 0.f);
        if (t == 0 || av > best) {
          best = av;
          ybest = yh;
          arg = p;
        }
      }
      cpos[k] = arg * kC2 + c;
      cy[k] = ybest;
      sm[sP2 + e] = best;
      w.p2[(size_t)b * kFc + e] = best;
    }
    __syncthreads();
    for (int j = warp; j < kCls; j += kWarps) {
      float s = 0.f;
      for (int k = lane; k < kFc; k += 32) s = fmaf(sm[sP2 + k], wv(oWf + k * kCls + j), s);
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
      if (lane == 0) sm[sLog + j] = s + wv(oBf + j);
    }
    __syncthreads();
    if (warp == 0) {
      const float l = lane < kCls ? sm[sLog + lane] : 0.f;
      const float o = fmaxf(l, 0.f);   // the ReLU on the logits, DM/problems.py:338
      const float zj = lane < kCls ? o : -INFINITY;
      float m = zj;
#pragma unroll
      for (int s = 16; s > 0; s >>= 1) m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, s));
      const float e = lane < kCls ? expf(zj - m) : 0.f;
      float s = e;
#pragma unroll
      for (int t = 16; t > 0; t >>= 1) s += __shfl_xor_sync(0xffffffffu, s, t);
      const float zy = __shfl_sync(0xffffffffu, zj, y);
      if (lane < kCls) {
        const float d = l > 0.f ? (e / s - (lane == y ? 1.f : 0.f)) / (float)B : 0.f;
        sm[sLog + 16 + lane] = d;
        w.dl[(size_t)b * 16 + lane] = d;
      }
      if (lane == 0) w.loss[b] = (double)m + (double)logf(s) - (double)zy;
    }
    for (int e = tid; e < kZ2; e += kThreads) sm[sZ2 + e] = 0.f;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < 2; ++k) {   // dp2 = Wfc dlogits, routed to the pool maximum through ReLU'
      const int e = tid + kThreads * k;
      float d = 0.f;
#pragma unroll
      for (int j = 0; j < kCls; ++j) d = fmaf(wv(oWf + e * kCls + j), sm[sLog + 16 + j], d);
      sm[sZ2 + cpos[k]] = cy[k] > 0.f ? d : 0.f;
    }
    __syncthreads();
    float* dy2 = w.dy2 + (size_t)b * kZ2;
    const int c = tid & (kC2 - 1), q = tid >> 5;
    double s1 = 0.0, s2 = 0.0;
    for (int p = q; p < kH2 * kH2; p += kThreads / kC2) {
      const float d = sm[sZ2 + p * kC2 + c];
      dy2[p * kC2 + c] = d;
      s1 += (double)d;
      s2 += (double)d * (double)((z2[p * kC2 + c] - mu2[c]) * rs2[c]);
    }
    s1 = l2o::chan_sum<kThreads>(red, s1, kC2);
    s2 = l2o::chan_sum<kThreads>(red, s2, kC2);
    if (tid < kC2) w.bk2[(size_t)b * kC2 + tid] = make_double2(s1, s2);
  }
  grid.sync();
  l2o::merge_back<kThreads>(w.bk2, B, kC2, kH2 * kH2, red, ma2, mb2);

  // ---- 4: dz2; dW2 and db2 of the image; dp1 = conv2 transposed, routed to the pool1 maxima; BN1 backward sums ---
  for (int b = blockIdx.x; b < B; b += G) {
    const float* z1 = w.z1 + (size_t)b * kZ1;
    const float* z2 = w.z2 + (size_t)b * kZ2;
    const float* dy2 = w.dy2 + (size_t)b * kZ2;
    float* part = w.part + (size_t)b * kPart;
    pool1(z1, sm);
    for (int e = tid; e < kPad * kPad * kPadS; e += kThreads) sm[sU + e] = 0.f;
    __syncthreads();
    for (int e = tid; e < kZ2; e += kThreads) {
      const int c = e & (kC2 - 1), p = e >> 5, i = p / kH2, j = p - i * kH2;
      const float yh = (z2[e] - mu2[c]) * rs2[c];
      const float dz = rs2[c] * (dy2[e] - ma2[c] - yh * mb2[c]);
      sm[sZ2 + e] = dz;
      sm[sU + ((i + 4) * kPad + j + 4) * kPadS + c] = dz;
    }
    __syncthreads();
    {   // db2
      const int c = tid & (kC2 - 1), q = tid >> 5;
      float s = 0.f;
      for (int p = q; p < kH2 * kH2; p += kThreads / kC2) s += sm[sZ2 + p * kC2 + c];
      const double t = l2o::chan_sum<kThreads>(red, (double)s, kC2);
      if (tid < kC2) part[oB2 + tid] = (float)t;
    }
    {   // dW2[r][o], r = (kh * 5 + kw) * 16 + c: warp = 4 output channels, lane = rows lane + 32 k
      const int og = warp;
      constexpr int kR = 13;   // ceil(400 / 32)
      int roff[kR];
#pragma unroll
      for (int k = 0; k < kR; ++k) {
        const int r = min(lane + 32 * k, 399), c = r & (kC1 - 1), t = r >> 4, kh = t / 5, kw = t - kh * 5;
        roff[k] = (kh * kP1 + kw) * kP1S + c;
      }
      float acc[kR][4] = {};
      for (int i = 0; i < kH2; ++i)
        for (int j = 0; j < kH2; ++j) {
          const float4 d = *reinterpret_cast<const float4*>(sm + sZ2 + (i * kH2 + j) * kC2 + og * 4);
          const float* pr = sm + sP1 + (i * kP1 + j) * kP1S;
#pragma unroll
          for (int k = 0; k < kR; ++k) {
            const float v = pr[roff[k]];
            acc[k][0] = fmaf(v, d.x, acc[k][0]);
            acc[k][1] = fmaf(v, d.y, acc[k][1]);
            acc[k][2] = fmaf(v, d.z, acc[k][2]);
            acc[k][3] = fmaf(v, d.w, acc[k][3]);
          }
        }
#pragma unroll
      for (int k = 0; k < kR; ++k) {
        const int r = lane + 32 * k;
        if (r < 400)
          *reinterpret_cast<float4*>(part + oW2 + r * kC2 + og * 4) =
              make_float4(acc[k][0], acc[k][1], acc[k][2], acc[k][3]);
      }
    }
    {   // dp1[q][c] = sum_{kh,kw,o} dz2pad[q - (kh,kw) + 4][o] W2[kh][kw][c][o]: warp pair = 4 channels, 3 cells each
      const int cg4 = warp >> 1, l64 = (warp & 1) * 32 + lane;
      int dbase[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int q = min(l64 + 64 * k, 168), pi = q / kP1, pj = q - pi * kP1;
        dbase[k] = ((pi + 4) * kPad + pj + 4) * kPadS;
      }
      float acc[3][4] = {};
      for (int kh = 0; kh < 5; ++kh)
        for (int kw = 0; kw < 5; ++kw) {
          const float* wr = sm + sW2 + ((kh * 5 + kw) * kC1 + cg4 * 4) * kC2;
          const int doff = sU - (kh * kPad + kw) * kPadS;
#pragma unroll 4
          for (int o = 0; o < kC2; ++o) {
            const float w0 = wr[o], w1 = wr[kC2 + o], w2 = wr[2 * kC2 + o], w3 = wr[3 * kC2 + o];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
              const float d = sm[doff + dbase[k] + o];
              acc[k][0] = fmaf(d, w0, acc[k][0]);
              acc[k][1] = fmaf(d, w1, acc[k][1]);
              acc[k][2] = fmaf(d, w2, acc[k][2]);
              acc[k][3] = fmaf(d, w3, acc[k][3]);
            }
          }
        }
      const uint8_t* code = reinterpret_cast<const uint8_t*>(sm + sCode);
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        const int q = l64 + 64 * k;
        if (q < kP1 * kP1) {
          const int pi = q / kP1, pj = q - pi * kP1;
#pragma unroll
          for (int t = 0; t < 4; ++t) {
            const int c = cg4 * 4 + t, e = q * kC1 + c, arg = code[e];
            const int p = (2 * pi + (arg >> 1)) * kH1 + 2 * pj + (arg & 1);
            const float yh = (z1[p * kC1 + c] - mu1[c]) * rs1[c];
            const float d = yh > 0.f ? acc[k][t] : 0.f;
            sm[sDyc + e] = d;
            sm[sYs + e] = yh;
            w.dyc[(size_t)b * kQ1 + e] = d;
            w.code[(size_t)b * kQ1 + e] = (uint8_t)arg;
          }
        }
      }
    }
    __syncthreads();
    const int c = tid & (kC1 - 1), q = tid >> 4;
    double s1 = 0.0, s2 = 0.0;
    for (int e = q * kC1 + c; e < kQ1; e += kThreads) {
      s1 += (double)sm[sDyc + e];
      s2 += (double)sm[sDyc + e] * (double)sm[sYs + e];
    }
    s1 = l2o::chan_sum<kThreads>(red, s1, kC1);
    s2 = l2o::chan_sum<kThreads>(red, s2, kC1);
    if (tid < kC1) w.bk1[(size_t)b * kC1 + tid] = make_double2(s1, s2);
  }
  grid.sync();
  l2o::merge_back<kThreads>(w.bk1, B, kC1, kH1 * kH1, red, ma1, mb1);

  // ---- 5: dz1; dW1 and db1 of the image -------------------------------------------------------------------------
  for (int b = blockIdx.x; b < B; b += G) {
    load_image(b);
    const float* z1 = w.z1 + (size_t)b * kZ1;
    const float* dyc = w.dyc + (size_t)b * kQ1;
    const uint8_t* code = w.code + (size_t)b * kQ1;
    for (int e = tid; e < kZ1; e += kThreads) {
      const int c = e & (kC1 - 1), p = e >> 4, i = p / kH1, j = p - i * kH1;
      const int cell = ((i >> 1) * kP1 + (j >> 1)) * kC1 + c;
      const float dy = code[cell] == ((i & 1) * 2 + (j & 1)) ? dyc[cell] : 0.f;
      const float yh = (z1[e] - mu1[c]) * rs1[c];
      sm[sU + e] = rs1[c] * (dy - ma1[c] - yh * mb1[c]);
    }
    __syncthreads();
    const int c = tid & (kC1 - 1), q = tid >> 4;
    float acc[10] = {};
    for (int p = q; p < kH1 * kH1; p += kThreads / kC1) {
      const int i = p / kH1, j = p - i * kH1;
      const float d = sm[sU + p * kC1 + c];
#pragma unroll
      for (int kh = 0; kh < 3; ++kh)
#pragma unroll
        for (int kw = 0; kw < 3; ++kw) acc[kh * 3 + kw] = fmaf(sm[sX + (i + kh) * kIn + j + kw], d, acc[kh * 3 + kw]);
      acc[9] += d;
    }
#pragma unroll
    for (int t = 0; t < 10; ++t) sm[sDyc + t * kThreads + tid] = acc[t];
    __syncthreads();
    if (tid < 10 * kC1) {   // (t, c): the 16 position groups in order
      const int t = tid / kC1, cc = tid - t * kC1;
      float s = 0.f;
      for (int qq = 0; qq < kThreads / kC1; ++qq) s += sm[sDyc + t * kThreads + qq * kC1 + cc];
      w.part[(size_t)b * kPart + (t < 9 ? oW1 + t * kC1 + cc : oB1 + cc)] = s;
    }
    __syncthreads();
  }
  grid.sync();

  // ---- the final reduction: every coordinate summed over b = 0..B-1 in order ---------------------------------------
  for (int n = blockIdx.x * kThreads + tid; n < kCoords; n += G * kThreads) {
    double s = 0.0;
    if (n < kPart) {
      for (int b = 0; b < B; ++b) s += (double)__ldcg(&w.part[(size_t)b * kPart + n]);
    } else if (n < oBf) {
      const int k = (n - oWf) / kCls, j = n - oWf - k * kCls;
      for (int b = 0; b < B; ++b)
        s = fma((double)__ldcg(&w.p2[(size_t)b * kFc + k]), (double)__ldcg(&w.dl[(size_t)b * 16 + j]), s);
    } else {
      for (int b = 0; b < B; ++b) s += (double)__ldcg(&w.dl[(size_t)b * 16 + n - oBf]);
    }
    const float gv = (float)s;
    a.g[n] = sc ? gv * sc[n] : gv;
  }
  if (blockIdx.x == 0 && tid == 0) {
    double t = 0.0;
    for (int b = 0; b < B; ++b) t += __ldcg(&w.loss[b]);
    if (a.f) *a.f = t / (double)B;
    *a.counter = (int64_t)(ctr + 1);
  }
}

}  // namespace

extern "C" int64_t l2o_mnist_conv_workspace_bytes(int32_t batch) {
  if (batch < 1 || batch > L2O_MNIST_CONV_MAX_BATCH) return L2O_E_INVALID;
  return (int64_t)ws_layout(batch, nullptr, nullptr);
}

extern "C" int l2o_mnist_conv_workspace_layout(int32_t batch, int64_t* off) {
  if (batch < 1 || batch > L2O_MNIST_CONV_MAX_BATCH || !off) return L2O_E_INVALID;
  Ws w;
  ws_layout(batch, nullptr, &w);   // a null base: the pointers are the byte offsets
  off[0] = (int64_t)(uintptr_t)w.z1;
  off[1] = (int64_t)(uintptr_t)w.z2;
  off[2] = (int64_t)(uintptr_t)w.bn;
  off[3] = (int64_t)(uintptr_t)w.dl;
  return L2O_OK;
}

extern "C" int l2o_mnist_conv_grad(const l2o_mnist_conv_args* a, void* stream) {
  if (!a || !a->images || !a->labels || !a->x || !a->g || !a->counter || !a->workspace) return L2O_E_INVALID;
  if (a->batch < 1 || a->batch > L2O_MNIST_CONV_MAX_BATCH || a->num_examples < 1) return L2O_E_INVALID;
  // W2 is staged as float4 and the workspace holds fp64 / float4 regions
  if (l2o::misaligned(a->x, 16) || l2o::misaligned(a->scale, 16) || l2o::misaligned(a->g, 4) ||
      l2o::misaligned(a->counter, 8) || l2o::misaligned(a->f, 8) || l2o::misaligned(a->idx_out, 4) ||
      l2o::misaligned(a->workspace, 16))
    return L2O_E_INVALID;
  if (a->workspace_bytes < ws_layout(a->batch, nullptr, nullptr)) return L2O_E_INVALID;
  Args args;
  args.a = *a;
  ws_layout(a->batch, (char*)a->workspace, &args.w);
  return l2o::cooperative_launch("l2o_mnist_conv_grad", mnist_conv_kernel, kThreads, kSmem,
                                 (int64_t)a->batch * kThreads, (cudaStream_t)stream, args);
}
