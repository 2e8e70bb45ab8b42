// CIFAR-10 NAS-cell producer (DM/problems.py:540-634 `NAS`, batch_norm=True, + tf.gradients at DM/meta.py:322-329):
// f and df/dx of the cell network at a fresh batch in ONE launch, the batch drawn by l2o_philox.cuh's draw.
//
// Spec points (each restated from the reference; DESIGN §3.18):
//   - every conv is 3x3 SAME stride 1 + bias, batch norm, ReLU (DM/problems.py:585-600); batch norm as in
//     l2o_cifar_conv.cu: training mode, eps 1e-3, gamma = 1, beta = 0, so the conv biases' true gradient is zero;
//   - node0 = conv(x, 3->16); n0o2 = conv(node0); node1 = conv(node0); n1o3 = conv(node1) (each 16->16);
//     node2 = avgpool3x3/1 SAME(node1) + n0o2, where TF's SAME average divides by the in-image cells of the window
//     (4 at a corner, 6 on an edge, 9 inside); node3 = node2 + n1o3 + node0;
//   - the head: the mean of node3 over the 1024 positions per channel, fc 16->10 + bias, ReLU, cross entropy;
//   - the variables in creation order: node0/weights1 [3][3][3][16], node0/biases1 [16], node0_onto_node2/...,
//     node1/..., node1_onto_node3/... (each [3][3][16][16] + [16]), fc_weights [16][10], fc_bias [10].
//
// Design.  A cooperative launch over at most the resident CTAs (one per SM), images striped over the CTAs, and seven
// grid-wide barriers at the batch-wide points:
//   1  conv node0 -> z0 (workspace); per-image BN statistics of node0
//   2  node0 -> conv n0o2 -> za, conv node1 -> z1; their statistics
//   3  node1 -> conv n1o3 -> zb; its statistics
//   4  the forward tail and the loss; the BN backward sums of n0o2 and n1o3, whose upstream gradient is the spatially
//      uniform dnode3 = dfeat / 1024
//   5  dz of n1o3; its dW / db; dnode1 = conv^T(dz_b) + avgpool^T(dnode3) through node1's ReLU -> dy1; its sums
//   6  dz of node1 and of n0o2; their dW / db; dnode0 = dnode3 + conv^T(dz_1) + conv^T(dz_a) through node0's ReLU
//      -> dy0; its sums
//   7  dz of node0; its dW / db
//   -- then the final reduction over b = 0..B-1 in order.
// Per image the padded 34x34x16 maps live in shared memory (two of them, position stride 17 so that the 32 lanes of a
// warp, 32 consecutive columns of one row, hit 32 banks), the weights for the whole launch too.  Each thread owns 4
// positions x 16 channels of a conv output (register-tiled FFMA); the conv^T is the same loop over the padded dz with
// the kernel flipped and its channel axes swapped.  Every per-image channel sum is a fixed-order reduction, and every
// batch-wide one a sum over b in order (l2o_bn.cuh), so f and g are bitwise identical on any SM count, with no atomics.
// Random scaling as l2o_lasso_grad: the loss at x (.) scale, g times scale.
#include <cooperative_groups.h>
#include <cuda_runtime.h>

#include "l2o_bn.cuh"
#include "l2o_internal.h"
#include "l2o_philox.cuh"

namespace cg = cooperative_groups;

namespace {

constexpr int kThreads = 256;
constexpr int kN = 32, kHW = kN * kN, kC = 16, kCls = 10, kPixels = 3 * kHW;
constexpr int kPS = 17;                       // padded-map position stride (16 channels + 1)
constexpr int kPad = kN + 2;                  // 34
constexpr int kMap = kPad * kPad * kPS;       // one padded map in floats
constexpr int kZ = kHW * kC;                  // one unpadded map: [1024][16]
constexpr int kW0 = 9 * 3 * kC, kW = 9 * kC * kC;
// arena offsets (creation order): node0, node0_onto_node2 (a), node1, node1_onto_node3 (b), fc
constexpr int o0w = 0, o0b = o0w + kW0, oaw = o0b + kC, oab = oaw + kW, o1w = oab + kC, o1b = o1w + kW, obw = o1b + kC,
              obb = obw + kW, ofw = obb + kC, ofb = ofw + kC * kCls;
constexpr int kCoords = ofb + kCls;
static_assert(kCoords == L2O_NAS_COORDS, "arena size");
constexpr int kPart = ofw;                    // per-image partial gradient of the convs (fc from feat and dlogits)
constexpr float kEps = 1e-3f;
enum { L0 = 0, LA = 1, L1 = 2, LB = 3 };      // the four batch-normed layers

__host__ __device__ inline size_t up16(size_t v) { return (v + 15) & ~(size_t)15; }

struct Ws {
  double2* st;                 // [4][B][16] per-image (mean, M2)
  double2* bk;                 // [4][B][16] per-image (sum dy, sum dy * yhat)
  double* loss;                // [B]
  float *z0, *za, *z1, *zb;    // [B][1024][16] pre-BN maps
  float *dy1, *dy0;            // [B][1024][16] the ReLU-masked upstream gradients of node1 and node0
  float *part, *feat, *dl;     // [B][kPart], [B][16], [B][16]
  float* bn;                   // [4][2][16]: mu, rstd of node0, n0o2, node1, n1o3 as the kernel applies them
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
  t.st = (double2*)take(4 * b * kC * sizeof(double2));
  t.bk = (double2*)take(4 * b * kC * sizeof(double2));
  t.loss = (double*)take(b * sizeof(double));
  t.z0 = (float*)take(b * kZ * sizeof(float));
  t.za = (float*)take(b * kZ * sizeof(float));
  t.z1 = (float*)take(b * kZ * sizeof(float));
  t.zb = (float*)take(b * kZ * sizeof(float));
  t.dy1 = (float*)take(b * kZ * sizeof(float));
  t.dy0 = (float*)take(b * kZ * sizeof(float));
  t.part = (float*)take(b * kPart * sizeof(float));
  t.feat = (float*)take(b * 16 * sizeof(float));
  t.dl = (float*)take(b * 16 * sizeof(float));
  t.bn = (float*)take(4 * 2 * kC * sizeof(float));
  if (w) *w = t;
  return off;
}

// shared memory (floats)
constexpr int sP = 0;                       // padded map P
constexpr int sQ = sP + kMap;               // padded map Q
constexpr int sW = sQ + kMap;               // weights (scaled): W0 [9][3][16], Wa, W1, Wb [9][16][16]
constexpr int sBn = sW + kW0 + 3 * kW;      // [4 layers][mu, rs, ma, mb][16]
constexpr int sBias = sBn + 4 * 4 * kC;     // [4 layers][16] conv biases (scaled)
constexpr int sMisc = sBias + 4 * kC;       // feat [16], dlogits [16], dnode3 [16]
constexpr int kSmemFloats = sMisc + 48;
static_assert(kSmemFloats % 2 == 0, "the fp64 buffers follow, 8-byte aligned");
constexpr size_t kSmem = (size_t)kSmemFloats * sizeof(float) + (kThreads + 8 * kC) * sizeof(double);

struct Args {
  l2o_nas_args a;
  Ws w;
};

__device__ __forceinline__ int pad_at(int i, int j) { return ((i + 1) * kPad + j + 1) * kPS; }   // interior (i, j)

// conv 3x3 SAME over a padded map into acc[k][o], k over the thread's positions p = tid + 256 k.  Forward: weights
// w[tap][ci][o].  Transposed (T): the gradient of the input of a conv with weights w from the padded dz of its
// output, i.e. the flipped kernel with the channel axes swapped: w[8 - tap][o][ci].
template <int CIN, bool T>
__device__ __forceinline__ void conv3(const float* in, const float* w, float (&acc)[4][kC]) {
  int base[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int p = threadIdx.x + kThreads * k;
    base[k] = ((p >> 5) * kPad + (p & 31)) * kPS;
  }
  for (int tap = 0; tap < 9; ++tap) {
    const int roff = ((tap / 3) * kPad + tap % 3) * kPS;
    for (int ci = 0; ci < CIN; ++ci) {
      float v[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = in[base[k] + roff + ci];
#pragma unroll
      for (int o = 0; o < kC; ++o) {
        const float wt = T ? w[(8 - tap) * kC * kC + o * kC + ci] : w[(tap * CIN + ci) * kC + o];
#pragma unroll
        for (int k = 0; k < 4; ++k) acc[k][o] = fmaf(v[k], wt, acc[k][o]);
      }
    }
  }
}

// dW[tap][ci][o] = sum_p in[p + tap][ci] dz[p][o] and db[o] = sum_p dz[p][o] of one image: thread (ci, o).  The sums
// run in fp64: batch norm makes dz zero-mean over the 1024 positions, so the terms cancel, and a serial fp32 sum loses
// about 1e-5 of node0's dW.
template <int CIN>
__device__ void conv_dw(const float* in, const float* dz, float* part_w, float* part_b) {
  const int tid = threadIdx.x;
  if (tid >= CIN * kC) return;
  const int ci = tid >> 4, o = tid & (kC - 1);
  double acc[9] = {}, db = 0.0;
  for (int p = 0; p < kHW; ++p) {
    const int i = p >> 5, j = p & 31;
    const double d = dz[pad_at(i, j) + o];
    const float* r = in + (i * kPad + j) * kPS + ci;
#pragma unroll
    for (int tap = 0; tap < 9; ++tap) acc[tap] = fma((double)r[((tap / 3) * kPad + tap % 3) * kPS], d, acc[tap]);
    db += d;
  }
#pragma unroll
  for (int tap = 0; tap < 9; ++tap) part_w[(tap * CIN + ci) * kC + o] = (float)acc[tap];
  if (ci == 0) part_b[o] = (float)db;
}

// the per-channel sums over the CTA of v[16] held by every thread: a fixed butterfly per warp, then warps in order;
// the result in out[0..15] (shared), valid after the call
__device__ void chan16(double (&v)[kC], double* red16, double* out) {
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
#pragma unroll
  for (int c = 0; c < kC; ++c)
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) v[c] += __shfl_xor_sync(0xffffffffu, v[c], s);
  if (lane == 0)
#pragma unroll
    for (int c = 0; c < kC; ++c) red16[warp * kC + c] = v[c];
  __syncthreads();
  if (tid < kC) {
    double s = 0.0;
    for (int w8 = 0; w8 < kThreads / 32; ++w8) s += red16[w8 * kC + tid];
    out[tid] = s;
  }
  __syncthreads();
}

// the image's BN statistics (mean, M2) of the conv output in acc
__device__ void stats(const float (&acc)[4][kC], double* red16, double* tmp, double2* st) {
  double v[kC];
#pragma unroll
  for (int c = 0; c < kC; ++c) v[c] = (double)acc[0][c] + (double)acc[1][c] + (double)acc[2][c] + (double)acc[3][c];
  chan16(v, red16, tmp);
#pragma unroll
  for (int c = 0; c < kC; ++c) {
    const double m = tmp[c] / (double)kHW;
    v[c] = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const double d = (double)acc[k][c] - m;
      v[c] += d * d;
    }
  }
  chan16(v, red16, tmp + kC);
  if (threadIdx.x < kC) st[threadIdx.x] = make_double2(tmp[threadIdx.x] / (double)kHW, tmp[kC + threadIdx.x]);
  __syncthreads();
}

// conv output + bias -> the workspace map z (position-major) and the image's statistics
__device__ void finish_conv(float (&acc)[4][kC], const float* bias, float* z, double* red16, double* tmp,
                            double2* st) {
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int p = threadIdx.x + kThreads * k;
#pragma unroll
    for (int c = 0; c < kC; ++c) acc[k][c] += bias[c];
#pragma unroll
    for (int c = 0; c < kC; c += 4)
      *reinterpret_cast<float4*>(z + p * kC + c) = make_float4(acc[k][c], acc[k][c + 1], acc[k][c + 2], acc[k][c + 3]);
  }
  stats(acc, red16, tmp, st);
}

__device__ __forceinline__ void zero(float (&acc)[4][kC]) {
#pragma unroll
  for (int k = 0; k < 4; ++k)
#pragma unroll
    for (int c = 0; c < kC; ++c) acc[k][c] = 0.f;
}

// the in-image cells of the SAME 3x3 window centred on row (or column) i
__device__ __forceinline__ int span(int i) { return (i == 0 || i == kN - 1) ? 2 : 3; }

__global__ void __launch_bounds__(kThreads, 1) nas_kernel(const Args args) {
  extern __shared__ __align__(16) float sm[];
  double* red = reinterpret_cast<double*>(sm + kSmemFloats);   // [kThreads]
  double* red16 = red + kThreads;                               // [8][16]
  __shared__ double tmp[2 * kC];
  const l2o_nas_args& a = args.a;
  const Ws& w = args.w;
  cg::grid_group grid = cg::this_grid();
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int B = a.batch, G = gridDim.x;
  const float* __restrict__ x = a.x;
  const float* __restrict__ sc = a.scale;
  auto wv = [&](int o) { return sc ? x[o] * sc[o] : x[o]; };
  float* P = sm + sP;
  float* Q = sm + sQ;
  const float* W0 = sm + sW;
  const float* Wa = W0 + kW0;
  const float* W1 = Wa + kW;
  const float* Wb = W1 + kW;
  auto mu = [&](int l) { return sm + sBn + l * 4 * kC; };
  auto rs = [&](int l) { return sm + sBn + l * 4 * kC + kC; };
  auto ma = [&](int l) { return sm + sBn + l * 4 * kC + 2 * kC; };
  auto mb = [&](int l) { return sm + sBn + l * 4 * kC + 3 * kC; };
  auto bias = [&](int l) { return sm + sBias + l * kC; };
  float* feat = sm + sMisc;
  float* dlog = feat + 16;
  float* dn3 = feat + 32;
  const uint64_t ctr = (uint64_t)*a.counter;
  auto st = [&](int l, int b) { return w.st + ((size_t)l * B + b) * kC; };
  auto bk = [&](int l, int b) { return w.bk + ((size_t)l * B + b) * kC; };
  auto img = [&](const float* z, int b) { return z + (size_t)b * kZ; };
  // normalised value and ReLU of layer l at element e = p * 16 + c of map z
  auto yhat = [&](int l, const float* z, int e) { return (z[e] - mu(l)[e & (kC - 1)]) * rs(l)[e & (kC - 1)]; };
  // padded map M <- ReLU(BN_l(z)) of image b
  auto relu_map = [&](float* M, int l, const float* z) {
    for (int e = tid; e < kZ; e += kThreads) {
      const int p = e >> 4, c = e & (kC - 1);
      M[pad_at(p >> 5, p & 31) + c] = fmaxf(yhat(l, z, e), 0.f);
    }
  };
  // padded map M <- dz = rstd (dy - mean dy - yhat mean(dy yhat)) of layer l
  auto dz_map = [&](float* M, int l, const float* z, const float* dy) {
    for (int e = tid; e < kZ; e += kThreads) {
      const int p = e >> 4, c = e & (kC - 1);
      M[pad_at(p >> 5, p & 31) + c] = rs(l)[c] * (dy[e] - ma(l)[c] - yhat(l, z, e) * mb(l)[c]);
    }
  };
  // dnode3 of one image from its dlogits: dfeat = Wfc dlogits, and node3's mean is over 1024 positions
  auto load_dn3 = [&](const float* dl) {
    if (tid < kC) {
      float d = 0.f;
#pragma unroll
      for (int j = 0; j < kCls; ++j) d = fmaf(wv(ofw + tid * kCls + j), dl[j], d);
      dn3[tid] = d / (float)kHW;
    }
    __syncthreads();
  };
  auto load_image = [&](int b) {
    const int idx = l2o::batch_index(a.seed, ctr, b, a.num_examples);
    for (int e = tid; e < kPixels; e += kThreads) {
      const int c = e >> 10, p = e & (kHW - 1);
      Q[pad_at(p >> 5, p & 31) + c] = l2o::cifar_pixel(a.images[(size_t)idx * kPixels + e]);
    }
    return idx;
  };
  // the BN constants of layer l from the per-image statistics; CTA 0 records them for the caller
  auto merge = [&](int l) {
    l2o::merge_stats<kThreads>(st(l, 0), B, kC, kHW, kEps, red, mu(l), rs(l), tmp);
    if (blockIdx.x == 0 && tid < kC) {
      w.bn[l * 2 * kC + tid] = mu(l)[tid];
      w.bn[l * 2 * kC + kC + tid] = rs(l)[tid];
    }
  };

  for (int e = tid; e < 2 * kMap; e += kThreads) sm[e] = 0.f;   // the zero borders stay zero for the whole launch
  for (int e = tid; e < kW0; e += kThreads) sm[sW + e] = wv(o0w + e);
  if (tid < 4 * kC) {
    const int off[4] = {o0b, oab, o1b, obb};
    sm[sBias + tid] = wv(off[tid >> 4] + (tid & (kC - 1)));
  }
  for (int e = tid; e < kW; e += kThreads) {
    sm[sW + kW0 + e] = wv(oaw + e);
    sm[sW + kW0 + kW + e] = wv(o1w + e);
    sm[sW + kW0 + 2 * kW + e] = wv(obw + e);
  }
  __syncthreads();
  float acc[4][kC];

  // ---- 1: conv node0 -> z0; statistics ----------------------------------------------------------------------------
  for (int b = blockIdx.x; b < B; b += G) {
    const int idx = load_image(b);
    if (tid == 0 && a.idx_out) a.idx_out[b] = idx;
    __syncthreads();
    zero(acc);
    conv3<3, false>(Q, W0, acc);
    finish_conv(acc, bias(L0), w.z0 + (size_t)b * kZ, red16, tmp, st(L0, b));
  }
  grid.sync();
  merge(L0);

  // ---- 2: node0 -> conv n0o2 -> za, conv node1 -> z1; statistics -------------------------------------------------
  for (int b = blockIdx.x; b < B; b += G) {
    relu_map(P, L0, img(w.z0, b));
    __syncthreads();
    zero(acc);
    conv3<kC, false>(P, Wa, acc);
    finish_conv(acc, bias(LA), w.za + (size_t)b * kZ, red16, tmp, st(LA, b));
    zero(acc);
    conv3<kC, false>(P, W1, acc);
    finish_conv(acc, bias(L1), w.z1 + (size_t)b * kZ, red16, tmp, st(L1, b));
  }
  grid.sync();
  merge(LA);
  merge(L1);

  // ---- 3: node1 -> conv n1o3 -> zb; statistics --------------------------------------------------------------------
  for (int b = blockIdx.x; b < B; b += G) {
    relu_map(P, L1, img(w.z1, b));
    __syncthreads();
    zero(acc);
    conv3<kC, false>(P, Wb, acc);
    finish_conv(acc, bias(LB), w.zb + (size_t)b * kZ, red16, tmp, st(LB, b));
  }
  grid.sync();
  merge(LB);

  // ---- 4: node2, node3, the mean, fc, ReLU, cross entropy; dnode3; the BN backward sums of n0o2 and n1o3 -----------
  for (int b = blockIdx.x; b < B; b += G) {
    const float *z0 = img(w.z0, b), *za = img(w.za, b), *z1 = img(w.z1, b), *zb = img(w.zb, b);
    relu_map(P, L1, z1);
    __syncthreads();
    double s = 0.0;
    for (int e = tid; e < kZ; e += kThreads) {   // every e of this thread has channel tid & 15
      const int p = e >> 4, c = e & (kC - 1), i = p >> 5, j = p & 31;
      float pool = 0.f;
      for (int di = -1; di <= 1; ++di)
        for (int dj = -1; dj <= 1; ++dj) pool += P[pad_at(i + di, j + dj) + c];   // the zero border adds nothing
      const float node2 = pool / (float)(span(i) * span(j)) + fmaxf(yhat(LA, za, e), 0.f);
      const float node3 = node2 + fmaxf(yhat(LB, zb, e), 0.f) + fmaxf(yhat(L0, z0, e), 0.f);
      s += (double)node3;
    }
    s = l2o::chan_sum<kThreads>(red, s, kC);
    if (tid < kC) {
      feat[tid] = (float)(s / (double)kHW);
      w.feat[(size_t)b * 16 + tid] = feat[tid];
    }
    __syncthreads();
    if (warp == 0) {
      const int y = a.labels[l2o::batch_index(a.seed, ctr, b, a.num_examples)];
      float l = 0.f;
      if (lane < kCls) {
        for (int k = 0; k < kC; ++k) l = fmaf(feat[k], wv(ofw + k * kCls + lane), l);
        l += wv(ofb + lane);
      }
      // the softmax in fp64 from the fp32 logits: a confident correct prediction makes the loss and the label's
      // dlogit differences of numbers near 1, which fp32 would cancel
      const double zj = lane < kCls ? (double)fmaxf(l, 0.f) : -INFINITY;   // the ReLU on the logits, DM/problems.py:625
      double m = zj;
#pragma unroll
      for (int t = 16; t > 0; t >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, t));
      const double ex = lane < kCls ? exp(zj - m) : 0.0;
      double se = ex;
#pragma unroll
      for (int t = 16; t > 0; t >>= 1) se += __shfl_xor_sync(0xffffffffu, se, t);
      const double zy = __shfl_sync(0xffffffffu, zj, y);
      if (lane < kCls) {   // softmax - onehot; at the label, -(the other lanes' share)
        const double p = lane == y ? -(se - ex) / se : ex / se;
        const float d = l > 0.f ? (float)(p / (double)B) : 0.f;
        dlog[lane] = d;
        w.dl[(size_t)b * 16 + lane] = d;
      }
      if (lane == 0) w.loss[b] = m + log(se) - zy;
    }
    __syncthreads();
    load_dn3(dlog);
    // n0o2 and n1o3 both receive dnode3 (node2 = ... + n0o2, node3 = node2 + n1o3 + ...), through their ReLUs
    for (int l = LA; l <= LB; l += LB - LA) {
      const float* z = l == LA ? za : zb;
      double s1 = 0.0, s2 = 0.0;
      for (int e = tid; e < kZ; e += kThreads) {
        const float yh = yhat(l, z, e), dy = yh > 0.f ? dn3[e & (kC - 1)] : 0.f;
        s1 += (double)dy;
        s2 += (double)dy * (double)yh;
      }
      s1 = l2o::chan_sum<kThreads>(red, s1, kC);
      s2 = l2o::chan_sum<kThreads>(red, s2, kC);
      if (tid < kC) bk(l, b)[tid] = make_double2(s1, s2);
    }
  }
  grid.sync();
  l2o::merge_back<kThreads>(bk(LA, 0), B, kC, kHW, red, ma(LA), mb(LA));
  l2o::merge_back<kThreads>(bk(LB, 0), B, kC, kHW, red, ma(LB), mb(LB));

  // dy of n0o2 (and of n1o3) from dnode3: a layer-l dy map without storing it
  auto dy_uniform = [&](float* M, int l, const float* z) {
    for (int e = tid; e < kZ; e += kThreads) {
      const int p = e >> 4, c = e & (kC - 1);
      const float yh = yhat(l, z, e), dy = yh > 0.f ? dn3[c] : 0.f;
      M[pad_at(p >> 5, p & 31) + c] = rs(l)[c] * (dy - ma(l)[c] - yh * mb(l)[c]);
    }
  };
  // the ReLU-masked gradient in acc of layer l's output at the thread's positions -> dy (workspace) and its sums
  auto masked = [&](int l, const float* z, float* dy, double2* bk_out) {
    double v[kC];
#pragma unroll
    for (int c = 0; c < kC; ++c) v[c] = 0.0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const int p = tid + kThreads * k;
#pragma unroll
      for (int c = 0; c < kC; ++c) {
        acc[k][c] = yhat(l, z, p * kC + c) > 0.f ? acc[k][c] : 0.f;
        v[c] += (double)acc[k][c];
      }
#pragma unroll
      for (int c = 0; c < kC; c += 4)
        *reinterpret_cast<float4*>(dy + p * kC + c) = make_float4(acc[k][c], acc[k][c + 1], acc[k][c + 2],
                                                                  acc[k][c + 3]);
    }
    chan16(v, red16, tmp);
#pragma unroll
    for (int c = 0; c < kC; ++c) {
      v[c] = 0.0;
#pragma unroll
      for (int k = 0; k < 4; ++k)
        v[c] += (double)acc[k][c] * (double)yhat(l, z, (tid + kThreads * k) * kC + c);
    }
    chan16(v, red16, tmp + kC);
    if (tid < kC) bk_out[tid] = make_double2(tmp[tid], tmp[kC + tid]);
    __syncthreads();
  };

  // ---- 5: dz_b; dWb, dbb; dnode1 = conv^T(dz_b) + avgpool^T(dnode3), through node1's ReLU -> dy1; its sums --------
  for (int b = blockIdx.x; b < B; b += G) {
    const float *z1 = img(w.z1, b), *zb = img(w.zb, b);
    float* part = w.part + (size_t)b * kPart;
    load_dn3(w.dl + (size_t)b * 16);
    relu_map(P, L1, z1);
    dy_uniform(Q, LB, zb);
    __syncthreads();
    conv_dw<kC>(P, Q, part + obw, part + obb);
    zero(acc);
    conv3<kC, true>(Q, Wb, acc);
#pragma unroll
    for (int k = 0; k < 4; ++k) {   // avgpool^T of the uniform dnode3: sum over the windows covering (i, j) of 1 / cells
      const int p = tid + kThreads * k, i = p >> 5, j = p & 31;
      float r = 0.f;
      for (int di = -1; di <= 1; ++di)
        for (int dj = -1; dj <= 1; ++dj) {
          const int pi = i + di, pj = j + dj;
          if (pi >= 0 && pi < kN && pj >= 0 && pj < kN) r += 1.f / (float)(span(pi) * span(pj));
        }
#pragma unroll
      for (int c = 0; c < kC; ++c) acc[k][c] = fmaf(dn3[c], r, acc[k][c]);
    }
    masked(L1, z1, w.dy1 + (size_t)b * kZ, bk(L1, b));
  }
  grid.sync();
  l2o::merge_back<kThreads>(bk(L1, 0), B, kC, kHW, red, ma(L1), mb(L1));

  // ---- 6: dz_1, dz_a; their dW / db; dnode0 = dnode3 + conv^T(dz_1) + conv^T(dz_a) through node0's ReLU -> dy0 -----
  for (int b = blockIdx.x; b < B; b += G) {
    const float *z0 = img(w.z0, b), *za = img(w.za, b), *z1 = img(w.z1, b);
    float* part = w.part + (size_t)b * kPart;
    load_dn3(w.dl + (size_t)b * 16);
    relu_map(P, L0, z0);
    dz_map(Q, L1, z1, w.dy1 + (size_t)b * kZ);
    __syncthreads();
    conv_dw<kC>(P, Q, part + o1w, part + o1b);
    zero(acc);
    conv3<kC, true>(Q, W1, acc);
    __syncthreads();
    dy_uniform(Q, LA, za);
    __syncthreads();
    conv_dw<kC>(P, Q, part + oaw, part + oab);
    conv3<kC, true>(Q, Wa, acc);
#pragma unroll
    for (int k = 0; k < 4; ++k)
#pragma unroll
      for (int c = 0; c < kC; ++c) acc[k][c] += dn3[c];
    masked(L0, z0, w.dy0 + (size_t)b * kZ, bk(L0, b));
  }
  grid.sync();
  l2o::merge_back<kThreads>(bk(L0, 0), B, kC, kHW, red, ma(L0), mb(L0));

  // ---- 7: dz_0; dW0, db0 ---------------------------------------------------------------------------------------------
  for (int b = blockIdx.x; b < B; b += G) {
    float* part = w.part + (size_t)b * kPart;
    load_image(b);
    dz_map(P, L0, img(w.z0, b), w.dy0 + (size_t)b * kZ);
    __syncthreads();
    conv_dw<3>(Q, P, part + o0w, part + o0b);
    __syncthreads();
  }
  grid.sync();

  // ---- the final reduction: every coordinate summed over b = 0..B-1 in order ---------------------------------------
  for (int n = blockIdx.x * kThreads + tid; n < kCoords; n += G * kThreads) {
    double s = 0.0;
    if (n < kPart) {
      for (int b = 0; b < B; ++b) s += (double)__ldcg(&w.part[(size_t)b * kPart + n]);
    } else if (n < ofb) {
      const int k = (n - ofw) / kCls, j = n - ofw - k * kCls;
      for (int b = 0; b < B; ++b)
        s = fma((double)__ldcg(&w.feat[(size_t)b * 16 + k]), (double)__ldcg(&w.dl[(size_t)b * 16 + j]), s);
    } else {
      for (int b = 0; b < B; ++b) s += (double)__ldcg(&w.dl[(size_t)b * 16 + n - ofb]);
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

extern "C" int64_t l2o_nas_workspace_bytes(int32_t batch) {
  if (batch < 1 || batch > L2O_NAS_MAX_BATCH) return L2O_E_INVALID;
  return (int64_t)ws_layout(batch, nullptr, nullptr);
}

extern "C" int l2o_nas_workspace_layout(int32_t batch, int64_t* off) {
  if (batch < 1 || batch > L2O_NAS_MAX_BATCH || !off) return L2O_E_INVALID;
  Ws w;
  ws_layout(batch, nullptr, &w);   // a null base: the pointers are the byte offsets
  off[0] = (int64_t)(uintptr_t)w.z0;
  off[1] = (int64_t)(uintptr_t)w.za;
  off[2] = (int64_t)(uintptr_t)w.z1;
  off[3] = (int64_t)(uintptr_t)w.zb;
  off[4] = (int64_t)(uintptr_t)w.bn;
  off[5] = (int64_t)(uintptr_t)w.dl;
  return L2O_OK;
}

extern "C" int l2o_nas_grad(const l2o_nas_args* a, void* stream) {
  if (!a || !a->images || !a->labels || !a->x || !a->g || !a->counter || !a->workspace) return L2O_E_INVALID;
  if (a->batch < 1 || a->batch > L2O_NAS_MAX_BATCH || a->num_examples < 1) return L2O_E_INVALID;
  // the same alignment contract as l2o_mnist_conv_grad; the workspace holds fp64 and float4 regions
  if (l2o::misaligned(a->x, 16) || l2o::misaligned(a->scale, 16) || l2o::misaligned(a->g, 4) ||
      l2o::misaligned(a->counter, 8) || l2o::misaligned(a->f, 8) || l2o::misaligned(a->idx_out, 4) ||
      l2o::misaligned(a->workspace, 16))
    return L2O_E_INVALID;
  if (a->workspace_bytes < ws_layout(a->batch, nullptr, nullptr)) return L2O_E_INVALID;
  Args args;
  args.a = *a;
  ws_layout(a->batch, (char*)a->workspace, &args.w);
  return l2o::cooperative_launch("l2o_nas_grad", nas_kernel, kThreads, kSmem, (int64_t)a->batch * kThreads,
                                 (cudaStream_t)stream, args);
}
