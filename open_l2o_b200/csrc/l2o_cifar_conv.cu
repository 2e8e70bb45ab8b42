// CIFAR-10 ConvNet producer (DM/problems.py:369-458 `cifar10`, batch_norm=True, + tf.gradients at DM/meta.py:322-329):
// f and df/dx of
//   f = mean_b xent(ReLU(fc(pool(ReLU(BN(conv2(pool(ReLU(BN(conv1(images[idx_b] / 255))))))))), labels[idx_b])
// in ONE launch, with idx_b drawn afresh at every evaluation by l2o_philox.cuh's draw, as l2o_mnist_grad draws it.
//
// Spec points (each restated from the reference; DESIGN §3.18):
//   - the input is the record's [3][32][32] planes, read NHWC (DM/problems.py:398-400), at fp32(p) / fp32(255)
//     (tf.math.divide(image, 255), a correctly rounded division, not a product with 1/255);
//   - the variables, in creation order (DM/problems.py:421-427,439-446): conv_layer1/weights1 [3][3][3][16] (HWIO),
//     conv_layer1/biases1 [16], conv_layer2/weights1 [5][5][16][32], conv_layer2/biases1 [32], fc_weights [32][10],
//     fc_bias [10];
//   - both convs are stride 2 VALID: [32,32] -> [15,15] and, after the pool, [7,7] -> [2,2];
//   - batch norm is tf.layers.batch_normalization in training mode: per channel, the mean and the biased variance over
//     all B*H*W positions, eps 1e-3, gamma = 1 and beta = 0 (not optimizee variables, as for mnist_conv, §3.17); the
//     conv biases' true gradient is therefore zero and what this kernel writes for them is fp32 rounding noise;
//   - max-pool 2x2 stride 2 VALID: [15,15] -> [7,7] (row and column 14 dropped) and [2,2] -> [1,1]; the gradient goes
//     to the first maximum in row-major window order;
//   - the flatten of [1][1][32] is the 32 channels; the logits pass through a ReLU before the cross entropy.
//
// Design.  As l2o_mnist_conv_grad (§3.17): a cooperative launch over at most the resident CTAs, images striped over the
// CTAs (b = blockIdx.x + k * gridDim.x), and five grid-wide barriers at the batch-wide points:
//   1  conv1 -> z1 (workspace), per-image BN1 statistics (mean, M2) in fp64
//   -- sync: BN1 statistics --
//   2  BN1, ReLU, pool -> p1 (shared), conv2 (W2 staged once per CTA in shared memory) -> z2, per-image BN2 statistics
//   -- sync: BN2 statistics --
//   3  BN2, ReLU, pool -> p2, fc, ReLU, cross entropy, dlogits; dp2 routed back to dy2; per-image BN2 backward sums
//   -- sync: BN2 backward sums --
//   4  dz2 = BN2 backward; dW2 and db2 of the image; dp1 = conv2 transposed (stride 2: output cell (r, s) gathers the
//      dz2 cells (i, j) with r - 2i and s - 2j inside the 5x5 kernel); routed to the pool1 maxima; BN1 backward sums
//   -- sync: BN1 backward sums --
//   5  dz1 = BN1 backward, at every conv1 position (row and column 14 too: the BN backward reaches them through the
//      batch means); dW1 and db1 of the image
//   -- sync: the final reduction --
// Every batch-wide quantity is a sum over b = 0..B-1 in a fixed order that depends on B only (l2o_bn.cuh for the batch
// norm), so the same inputs give bitwise identical f and g on any number of SMs, with no atomics.
// Random scaling (DM/meta_dm_train.py:336-338,384-385) as l2o_lasso_grad: the loss at x (.) scale, g times scale.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include "l2o_bn.cuh"
#include "l2o_internal.h"
#include "l2o_philox.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 256;
constexpr int kIn = 32, kCin = 3, kH1 = 15, kP1 = 7, kH2 = 2;
constexpr int kC1 = 16, kC2 = 32, kCls = 10, kFc = kC2;   // the pooled [1][1][32]
constexpr int kPix = kCin * kIn * kIn;    // 3072
constexpr int kK1 = 3 * 3 * kCin;         // 27 conv1 taps per output channel
constexpr int kZ1 = kH1 * kH1 * kC1;      // 3600
constexpr int kQ1 = kP1 * kP1 * kC1;      // 784 pooled conv1 cells
constexpr int kZ2 = kH2 * kH2 * kC2;      // 128
constexpr int kR2 = 5 * 5 * kC1;          // 400 conv2 weight rows (kh, kw, ci)
constexpr int kW2 = kR2 * kC2;            // 12800
// arena offsets (creation order)
constexpr int oW1 = 0, oB1 = oW1 + kK1 * kC1, oW2 = oB1 + kC1, oB2 = oW2 + kW2, oWf = oB2 + kC2, oBf = oWf + kFc * kCls;
constexpr int kCoords = oBf + kCls;
static_assert(kCoords == L2O_CIFAR_CONV_COORDS, "arena size");
constexpr int kPart = oWf;                // per-image partial gradient: W1, b1, W2, b2 (fc from p2 and dlogits)
constexpr int kP1S = 17;                  // shared p1 position stride (16 channels + 1)
constexpr int kW2S = 33;                  // shared W2 row stride (32 output channels + 1: conflict-free in dp1)
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
constexpr int sW2 = 0;                          // [kR2][kW2S] conv2 weights (scaled), HWIO rows
constexpr int sU = sW2 + kR2 * kW2S;            // [kZ1] z1 | dz1
constexpr int sAcc = sU + kZ1;                  // [28][kThreads] stage-5 dW1 / db1 partials
constexpr int sX = sAcc + (kK1 + 1) * kThreads; // [3][32][32] the image, planes as in the file
constexpr int sP1 = sX + kPix;                  // [49][kP1S] pooled conv1 activations
constexpr int sZ2 = sP1 + kP1 * kP1 * kP1S + 3; // [kZ2] z2 | dz2
constexpr int sP2 = sZ2 + kZ2;                  // [kFc]
constexpr int sDyc = sP2 + kFc;                 // [kQ1] routed dp1
constexpr int sYs = sDyc + kQ1;                 // [kQ1] yhat1 at the pool1 maximum
constexpr int sCode = sYs + kQ1;                // [kQ1] bytes
constexpr int sW1 = sCode + kQ1 / 4;            // [432]
constexpr int sPc = sW1 + kK1 * kC1;            // per channel: mu1, rs1, ma1, mb1 [16]; mu2, rs2, ma2, mb2 [32]
constexpr int sLog = sPc + 4 * kC1 + 4 * kC2;   // [16] logits, then [16] dlogits
constexpr int kSmemFloats = sLog + 32;
static_assert(kSmemFloats % 2 == 0, "the fp64 reduction buffer follows, 8-byte aligned");
constexpr size_t kSmem = (size_t)kSmemFloats * sizeof(float) + kThreads * sizeof(double);

struct Args {
  l2o_cifar_conv_args a;
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

__global__ void __launch_bounds__(kThreads, 1) cifar_conv_kernel(const Args args) {
  extern __shared__ __align__(16) float sm[];
  double* red = reinterpret_cast<double*>(sm + kSmemFloats);
  __shared__ double mu_tmp[kC2];
  const l2o_cifar_conv_args& a = args.a;
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
    for (int e = tid; e < kPix; e += kThreads) sm[sX + e] = l2o::cifar_pixel(a.images[(size_t)idx * kPix + e]);
    return idx;
  };
  // the pixel at (row, column, channel) of the NHWC image
  auto px = [&](int r, int s, int ci) { return sm[sX + (ci * kIn + r) * kIn + s]; };

  for (int e = tid; e < kW2; e += kThreads) sm[sW2 + (e >> 5) * kW2S + (e & (kC2 - 1))] = wv(oW2 + e);
  for (int e = tid; e < kK1 * kC1; e += kThreads) sm[sW1 + e] = wv(oW1 + e);

  // ---- 1: conv1 + b1 -> z1; the image's BN1 statistics ------------------------------------------------------------
  for (int b = blockIdx.x; b < B; b += G) {
    const int idx = load_image(b);
    if (tid == 0 && a.idx_out) a.idx_out[b] = idx;
    __syncthreads();
    const int c = tid & (kC1 - 1), q = tid >> 4;
    float wk[kK1];
#pragma unroll
    for (int k = 0; k < kK1; ++k) wk[k] = sm[sW1 + k * kC1 + c];
    const float bias = wv(oB1 + c);
    float* z1 = w.z1 + (size_t)b * kZ1;
    double s = 0.0;
    for (int p = q; p < kH1 * kH1; p += kThreads / kC1) {
      const int i = p / kH1, j = p - i * kH1;
      float acc = 0.f;
#pragma unroll
      for (int kh = 0; kh < 3; ++kh)
#pragma unroll
        for (int kw = 0; kw < 3; ++kw)
#pragma unroll
          for (int ci = 0; ci < kCin; ++ci)
            acc = fmaf(px(2 * i + kh, 2 * j + kw, ci), wk[(kh * 3 + kw) * kCin + ci], acc);
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
    if (tid < kZ2) {   // output (pos, o), pos = i * 2 + j: a warp reads one p1 cell (broadcast) and one W2 row
      const int o = tid & (kC2 - 1), pos = tid >> 5, i = pos >> 1, j = pos & 1;
      float acc = 0.f;
      for (int kh = 0; kh < 5; ++kh)
        for (int kw = 0; kw < 5; ++kw) {
          const float* pr = sm + sP1 + ((2 * i + kh) * kP1 + 2 * j + kw) * kP1S;
          const float* wr = sm + sW2 + (kh * 5 + kw) * kC1 * kW2S + o;
#pragma unroll
          for (int ci = 0; ci < kC1; ++ci) acc = fmaf(pr[ci], wr[ci * kW2S], acc);
        }
      const float z = acc + wv(oB2 + o);
      sm[sZ2 + tid] = z;
      w.z2[(size_t)b * kZ2 + tid] = z;
    }
    __syncthreads();
    if (tid < kC2) {   // the 4 positions of channel tid
      double s = 0.0;
      for (int p = 0; p < kH2 * kH2; ++p) s += (double)sm[sZ2 + p * kC2 + tid];
      const double m = s / (double)(kH2 * kH2);
      double m2 = 0.0;
      for (int p = 0; p < kH2 * kH2; ++p) {
        const double d = (double)sm[sZ2 + p * kC2 + tid] - m;
        m2 += d * d;
      }
      w.st2[(size_t)b * kC2 + tid] = make_double2(m, m2);
    }
    __syncthreads();
  }
  grid.sync();
  l2o::merge_stats<kThreads>(w.st2, B, kC2, kH2 * kH2, kEps, red, mu2, rs2, mu_tmp);
  if (blockIdx.x == 0 && tid < kC2) {
    w.bn[2 * kC1 + tid] = mu2[tid];
    w.bn[2 * kC1 + kC2 + tid] = rs2[tid];
  }

  // ---- 3: BN2, ReLU, pool -> p2; fc, ReLU, cross entropy; dlogits -> dp2 -> dy2; the BN2 backward sums -----------
  for (int b = blockIdx.x; b < B; b += G) {
    const float* z2 = w.z2 + (size_t)b * kZ2;
    int arg = 0;
    float ybest = 0.f, yh[4];
    if (tid < kC2) {   // feature c: the maximum over the one 2x2 window
      const int c = tid;
      float best = 0.f;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        yh[t] = (z2[t * kC2 + c] - mu2[c]) * rs2[c];
        const float av = fmaxf(yh[t], 0.f);
        if (t == 0 || av > best) {
          best = av;
          ybest = yh[t];
          arg = t;
        }
      }
      sm[sP2 + c] = best;
      w.p2[(size_t)b * kFc + c] = best;
    }
    __syncthreads();
    if (warp == 0) {
      const int y = a.labels[l2o::batch_index(a.seed, ctr, b, a.num_examples)];
      float l = 0.f;
      if (lane < kCls) {
        for (int k = 0; k < kFc; ++k) l = fmaf(sm[sP2 + k], wv(oWf + k * kCls + lane), l);
        l += wv(oBf + lane);
      }
      const float o = fmaxf(l, 0.f);   // the ReLU on the logits, DM/problems.py:448
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
    __syncthreads();
    if (tid < kC2) {   // dp2 = Wfc dlogits, routed to the pool maximum through ReLU'; the BN2 backward sums
      const int c = tid;
      float d = 0.f;
#pragma unroll
      for (int j = 0; j < kCls; ++j) d = fmaf(wv(oWf + c * kCls + j), sm[sLog + 16 + j], d);
      d = ybest > 0.f ? d : 0.f;
      double s1 = 0.0, s2 = 0.0;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float dy = t == arg ? d : 0.f;
        w.dy2[(size_t)b * kZ2 + t * kC2 + c] = dy;
        s1 += (double)dy;
        s2 += (double)dy * (double)yh[t];
      }
      w.bk2[(size_t)b * kC2 + c] = make_double2(s1, s2);
    }
    __syncthreads();
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
    if (tid < kZ2) {
      const int c = tid & (kC2 - 1);
      const float yh = (z2[tid] - mu2[c]) * rs2[c];
      sm[sZ2 + tid] = rs2[c] * (dy2[tid] - ma2[c] - yh * mb2[c]);
    }
    __syncthreads();
    if (tid < kC2) {   // db2
      float s = 0.f;
      for (int p = 0; p < kH2 * kH2; ++p) s += sm[sZ2 + p * kC2 + tid];
      part[oB2 + tid] = s;
    }
    // dW2[r][o], r = (kh * 5 + kw) * 16 + ci: sum over the 2x2 outputs of p1[2i + kh][2j + kw][ci] dz2[i][j][o]
    for (int e = tid; e < kW2; e += kThreads) {
      const int o = e & (kC2 - 1), r = e >> 5, ci = r & (kC1 - 1), t = r >> 4, kh = t / 5, kw = t - kh * 5;
      float acc = 0.f;
#pragma unroll
      for (int p = 0; p < kH2 * kH2; ++p)
        acc = fmaf(sm[sP1 + ((2 * (p >> 1) + kh) * kP1 + 2 * (p & 1) + kw) * kP1S + ci], sm[sZ2 + p * kC2 + o], acc);
      part[oW2 + e] = acc;
    }
    // dp1[r][s][ci] = sum over o and the outputs (i, j) whose window covers (r, s) of dz2[i][j][o] W2[r-2i][s-2j][ci][o]
    const uint8_t* code = reinterpret_cast<const uint8_t*>(sm + sCode);
    for (int e = tid; e < kQ1; e += kThreads) {
      const int ci = e & (kC1 - 1), q = e >> 4, r = q / kP1, s = q - r * kP1;
      float acc = 0.f;
      for (int i = 0; i < kH2; ++i)
        for (int j = 0; j < kH2; ++j) {
          const int kh = r - 2 * i, kw = s - 2 * j;
          if (kh < 0 || kh >= 5 || kw < 0 || kw >= 5) continue;
          const float* wr = sm + sW2 + ((kh * 5 + kw) * kC1 + ci) * kW2S;
          const float* dz = sm + sZ2 + (i * kH2 + j) * kC2;
#pragma unroll 8
          for (int o = 0; o < kC2; ++o) acc = fmaf(dz[o], wr[o], acc);
        }
      const int arg = code[e];
      const int p = (2 * r + (arg >> 1)) * kH1 + 2 * s + (arg & 1);
      const float yh = (z1[p * kC1 + ci] - mu1[ci]) * rs1[ci];
      const float d = yh > 0.f ? acc : 0.f;
      sm[sDyc + e] = d;
      sm[sYs + e] = yh;
      w.dyc[(size_t)b * kQ1 + e] = d;
      w.code[(size_t)b * kQ1 + e] = (uint8_t)arg;
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
      float dy = 0.f;
      if (i < 2 * kP1 && j < 2 * kP1) {   // row and column 14 lie outside every pool window
        const int cell = ((i >> 1) * kP1 + (j >> 1)) * kC1 + c;
        dy = code[cell] == ((i & 1) * 2 + (j & 1)) ? dyc[cell] : 0.f;
      }
      const float yh = (z1[e] - mu1[c]) * rs1[c];
      sm[sU + e] = rs1[c] * (dy - ma1[c] - yh * mb1[c]);
    }
    __syncthreads();
    const int c = tid & (kC1 - 1), q = tid >> 4;
    float acc[kK1 + 1] = {};
    for (int p = q; p < kH1 * kH1; p += kThreads / kC1) {
      const int i = p / kH1, j = p - i * kH1;
      const float d = sm[sU + p * kC1 + c];
#pragma unroll
      for (int kh = 0; kh < 3; ++kh)
#pragma unroll
        for (int kw = 0; kw < 3; ++kw)
#pragma unroll
          for (int ci = 0; ci < kCin; ++ci) {
            const int t = (kh * 3 + kw) * kCin + ci;
            acc[t] = fmaf(px(2 * i + kh, 2 * j + kw, ci), d, acc[t]);
          }
      acc[kK1] += d;
    }
#pragma unroll
    for (int t = 0; t <= kK1; ++t) sm[sAcc + t * kThreads + tid] = acc[t];
    __syncthreads();
    for (int e = tid; e < (kK1 + 1) * kC1; e += kThreads) {   // (t, c): the 16 position groups in order
      const int t = e / kC1, cc = e - t * kC1;
      float s = 0.f;
      for (int qq = 0; qq < kThreads / kC1; ++qq) s += sm[sAcc + t * kThreads + qq * kC1 + cc];
      w.part[(size_t)b * kPart + (t < kK1 ? oW1 + t * kC1 + cc : oB1 + cc)] = s;
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

extern "C" int64_t l2o_cifar_conv_workspace_bytes(int32_t batch) {
  if (batch < 1 || batch > L2O_CIFAR_CONV_MAX_BATCH) return L2O_E_INVALID;
  return (int64_t)ws_layout(batch, nullptr, nullptr);
}

extern "C" int l2o_cifar_conv_workspace_layout(int32_t batch, int64_t* off) {
  if (batch < 1 || batch > L2O_CIFAR_CONV_MAX_BATCH || !off) return L2O_E_INVALID;
  Ws w;
  ws_layout(batch, nullptr, &w);   // a null base: the pointers are the byte offsets
  off[0] = (int64_t)(uintptr_t)w.z1;
  off[1] = (int64_t)(uintptr_t)w.z2;
  off[2] = (int64_t)(uintptr_t)w.bn;
  off[3] = (int64_t)(uintptr_t)w.dl;
  return L2O_OK;
}

extern "C" int l2o_cifar_conv_grad(const l2o_cifar_conv_args* a, void* stream) {
  if (!a || !a->images || !a->labels || !a->x || !a->g || !a->counter || !a->workspace) return L2O_E_INVALID;
  if (a->batch < 1 || a->batch > L2O_CIFAR_CONV_MAX_BATCH || a->num_examples < 1) return L2O_E_INVALID;
  // the same alignment contract as l2o_mnist_conv_grad; the workspace holds fp64 regions
  if (l2o::misaligned(a->x, 16) || l2o::misaligned(a->scale, 16) || l2o::misaligned(a->g, 4) ||
      l2o::misaligned(a->counter, 8) || l2o::misaligned(a->f, 8) || l2o::misaligned(a->idx_out, 4) ||
      l2o::misaligned(a->workspace, 16))
    return L2O_E_INVALID;
  if (a->workspace_bytes < ws_layout(a->batch, nullptr, nullptr)) return L2O_E_INVALID;
  Args args;
  args.a = *a;
  ws_layout(a->batch, (char*)a->workspace, &args.w);
  return l2o::cooperative_launch("l2o_cifar_conv_grad", cifar_conv_kernel, kThreads, kSmem,
                                 (int64_t)a->batch * kThreads, (cudaStream_t)stream, args);
}
