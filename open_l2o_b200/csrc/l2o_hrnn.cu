// L2O-Scale HierarchicalRNN update step (SURVEY.md 8(f) row 1, BASELINE config #4) — sm_90a CUDA kernels + C-ABI.
// SC/ = Model_Free_L2O/L2O-Scale/L2O-Scale-Training/ of the reference; HR = SC/optimizer/hierarchical_rnn.py.
//
// One optimizer step over ALL optimizee tensors is three launches, with no host synchronisation (graph-capturable):
//   1. coord_tc_kernel (hrnn_tc.cuh) — thread = coordinate (HBM-bound: 88 B read + 88 B written per coordinate-step):
//                      gradient accumulators at 4 timescales, RMS scaling, the 12 input features, the per-parameter
//                      BiasGRU(10) on the tensor cores, the readouts (update direction, decays, log learning rate), and
//                      the per-tensor sums the upper levels need (fp64 atomics: mean of [h' | features], mean delta^2,
//                      sum log-lr).  Its reference is the fp64 oracle (oracle/hrnn_oracle.py); the backward
//                      (hrnn_bwd.cuh) recomputes the same step in exact fp32.
//   2. tensor_kernel — one CTA: per-tensor BiasGRU(20), the global BiasGRU(20) (fed by the LAST tensor's layer
//                      state only, HR:426-427), 1/RMS(delta) per tensor, and the NEXT step's per-tensor gate bias,
//                      problem-wide mean log-lr and first-step flags.
//   3. apply_kernel  — x -= lr * delta / RMS_tensor(delta)        (HR:621-626,652-653,404)
// State layout: 21 fp32 planes of [N] (N = all coordinates of all tensors, tensors contiguous):
//   0..9 parameter (BiasGRU hidden), 10 scl_decay, 11 inp_decay, 12 log_learning_rate, 13..16 grad_accum1..4,
//   17..20 ms1..4  (HR:303-343; "true_param" duplicates x when use_attention=False and is not stored).
#include <cstdint>
#include <new>
#include <mutex>
#include <vector>

#include "l2o_internal.h"
#include "cwlstm_ffma.cuh"   // helpers cwlstm_tc.cuh expects
#include "cwlstm_tc.cuh"     // wgmma / mbarrier wrappers, tf32 split

namespace l2o {
namespace hrnn {

constexpr int H0 = 10, H1 = 20, H2 = 20, F = 12, NS = 4;
constexpr int kPlanes = 21;
constexpr int P_H = 0, P_SCL = 10, P_INP = 11, P_LLR = 12, P_ACC = 13, P_MS = 17;
// flat theta offsets (order = oracle/hrnn_oracle.py theta_spec = TF variable creation order of HR:176-204,232-245)
constexpr int O_INIT0 = 0, O_INIT1 = 10, O_INIT2 = 30;
constexpr int O_WU = 50, O_WS = 60, O_BS = 70, O_WI = 71, O_BI = 81, O_WL = 82, O_BL = 92;
constexpr int O_PM = 93, O_PB = 693, O_GM = 723, O_GB = 1323;
constexpr int O_WG0 = 1353, O_BG0 = 1793, O_WC0 = 1813, O_BC0 = 2033;
constexpr int O_L1M = 2043, O_L1B = 3243;
constexpr int O_WG1 = 3303, O_BG1 = 4983, O_WC1 = 5023, O_BC1 = 5863;
constexpr int O_G2D = 5883, O_LRM = 5887, O_OFF = 5888;
constexpr int O_WG2 = 5889, O_BG2 = 7489, O_WC2 = 7529, O_BC2 = 8329;
constexpr int kTheta = 8349;
constexpr int kAcc = 24;  // per-tensor fp64 sums: [h'(10) | feat(12)], delta^2, log-lr'
constexpr int kBlock = 128;     // coordinates per block-table entry (= one tensor-core tile)
constexpr int kB0Stride = 32;   // floats per tensor in Workspace::bias0: r 0..9 | u 10..19 | c 20..29 | pad (16-byte rows)

struct BlockEnt {
  int64_t start;  // first coordinate of the block (global index)
  int32_t count;  // coordinates in the block (<= kBlock)
  int32_t tensor;
};

// caller-owned workspace, carved up by the library
struct Workspace {
  double* acc;        // [nt][kAcc]
  int* any_nz;        // [nt][NS]   any(ms_i' != 0) seen this step
  int* zero_flag;     // [nt][NS]   all(ms_i == 0) for the step about to run (utils.py:128-130)
  float* bias0;       // [nt][kB0Stride] per-tensor gate bias of the per-parameter GRU (HR:561-575)
  float* inv_denom;   // [nt]
  float* mean_log_lr; // [1]
  float* upd;         // [N]
};
__host__ __device__ inline size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }
inline size_t carve(Workspace& w, void* base, int nt, int64_t n) {
  size_t off = 0;
  char* b = (char*)base;
  auto take = [&](size_t bytes) { char* p = b ? b + off : nullptr; off = align_up(off + bytes, 256); return p; };
  w.acc = (double*)take(sizeof(double) * nt * kAcc);
  w.any_nz = (int*)take(sizeof(int) * nt * NS);
  w.zero_flag = (int*)take(sizeof(int) * nt * NS);
  w.bias0 = (float*)take(sizeof(float) * nt * kB0Stride);
  w.inv_denom = (float*)take(sizeof(float) * nt);
  w.mean_log_lr = (float*)take(sizeof(float));
  w.upd = (float*)take(sizeof(float) * (size_t)n);
  return off;
}

// Per-coordinate transcendental work (34 sigmoid/tanh, 8 log, 11 sqrt, 4 divisions per coordinate-step) would cost
// ~900 instructions in libdevice precision and make the step instruction-bound; the MUFU forms below (ex2 / lg2 /
// rsq / rcp .approx, ~1e-7 relative) cut that to ~200.  The tiny upper-level kernel keeps libdevice math.
__device__ __forceinline__ float sigmoidf_(float x) { return 1.0f / (1.0f + expf(-x)); }
__device__ __forceinline__ float lg2_approx(float x) {
  float y;
  asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float rsqrt_approx(float x) {
  float y;
  asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float sqrt_approx(float x) {
  float y;
  asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ float log_fast(float x) { return 0.6931471805599453f * lg2_approx(x); }
__device__ __forceinline__ float exp_fast(float x) { return ex2_approx(1.4426950408889634f * x); }

#include "hrnn_tc.cuh"
#include "hrnn_bwd.cuh"

// state scan used by l2o_hrnn_prepare: per-tensor sum of log-lr and any(ms_i != 0)
__global__ void __launch_bounds__(kBlock) scan_kernel(const float* __restrict__ state, int64_t n,
                                                      const BlockEnt* __restrict__ blocks, Workspace w) {
  __shared__ double sRed[kBlock / 32];
  const BlockEnt be = blocks[blockIdx.x];
  const int tid = threadIdx.x;
  const bool act = tid < be.count;
  const int64_t i = be.start + (act ? tid : 0);
  double v = act ? (double)state[(int64_t)P_LLR * n + i] : 0.0;
  int nz = 0;
  if (act)
#pragma unroll
    for (int s = 0; s < NS; ++s)
      if (state[(int64_t)(P_MS + s) * n + i] != 0.f) nz |= 1 << s;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = tid & 31, wid = tid >> 5;
  if (lane == 0) sRed[wid] = v;
#pragma unroll
  for (int s = 0; s < NS; ++s) {
    const unsigned any = __ballot_sync(0xffffffffu, nz & (1 << s));
    if (lane == 0 && any) atomicOr(&w.any_nz[be.tensor * NS + s], 1);
  }
  __syncthreads();
  if (tid == 0) {
    double t = 0.0;
    for (int q = 0; q < kBlock / 32; ++q) t += sRed[q];
    atomicAdd(&w.acc[be.tensor * kAcc + H0 + F + 1], t);
  }
}

// BiasGRU cell on one row held in shared memory (rnn_cells.py:46-68).  in[NI], h[NH] -> hn[NH]; bias[3*NH] (r|u|c).
// Threads 0..NH-1 each own one unit.  Wg: [NI+NH][2NH], Wc: [NI+NH][NH] (global memory, read once per call).
template <int NI, int NH>
__device__ void bias_gru(const float* __restrict__ Wg, const float* __restrict__ bg, const float* __restrict__ Wc,
                         const float* __restrict__ bc, const float* in, const float* h, const float* bias,
                         float* rh /*[NH] scratch*/, float* hn, int tid) {
  float r = 0.f, u = 0.f;
  if (tid < NH) {
    float pr = 0.f, pu = 0.f;
    for (int k = 0; k < NI; ++k) {
      pr = fmaf(in[k], Wg[k * 2 * NH + tid], pr);
      pu = fmaf(in[k], Wg[k * 2 * NH + NH + tid], pu);
    }
    for (int k = 0; k < NH; ++k) {
      pr = fmaf(h[k], Wg[(NI + k) * 2 * NH + tid], pr);
      pu = fmaf(h[k], Wg[(NI + k) * 2 * NH + NH + tid], pu);
    }
    r = sigmoidf_((pr + bg[tid]) + (bias ? bias[tid] : 0.f));
    u = sigmoidf_((pu + bg[NH + tid]) + (bias ? bias[NH + tid] : 0.f));
    rh[tid] = r * h[tid];
  }
  __syncthreads();
  if (tid < NH) {
    float pc = 0.f;
    for (int k = 0; k < NI; ++k) pc = fmaf(in[k], Wc[k * NH + tid], pc);
    for (int k = 0; k < NH; ++k) pc = fmaf(rh[k], Wc[(NI + k) * NH + tid], pc);
    const float c = tanhf((pc + bc[tid]) + (bias ? bias[2 * NH + tid] : 0.f));
    hn[tid] = u * h[tid] + (1.0f - u) * c;
  }
  __syncthreads();
}

// upper levels + bookkeeping for the next step.  mode 0 = after coord_tc_kernel (full step), 1 = prepare only.
__global__ void __launch_bounds__(64) tensor_kernel(const float* __restrict__ theta, float* __restrict__ layer,
                                                    float* __restrict__ global, int nt, const int64_t* __restrict__ sizes,
                                                    int64_t n_total, Workspace w, int mode) {
  __shared__ float sIn[H0 + F], sH[H1], sHn[H1], sRh[H1], sBias[3 * H1], sG[H2], sGn[H2];
  __shared__ double sSum;
  const int tid = threadIdx.x;
  if (tid < H2) sG[tid] = global[tid];
  if (tid == 0) sSum = 0.0;
  __syncthreads();
  if (mode == 0) {
    // bias injected into every per-tensor GRU: affine of the (old) global state (HR:588-594)
    for (int o = tid; o < 3 * H1; o += blockDim.x) {
      float v = 0.f;
      for (int k = 0; k < H2; ++k) v = fmaf(sG[k], theta[O_L1M + k * 3 * H1 + o], v);
      sBias[o] = v + theta[O_L1B + o];
    }
    __syncthreads();
    for (int j = 0; j < nt; ++j) {
      const double cnt = (double)sizes[j];
      if (tid < H0 + F) sIn[tid] = (float)(w.acc[j * kAcc + tid] / cnt);   // mean_coords([h' | feat]) (HR:582-587)
      if (tid < H1) sH[tid] = layer[j * H1 + tid];
      __syncthreads();
      bias_gru<H0 + F, H1>(theta + O_WG1, theta + O_BG1, theta + O_WC1, theta + O_BC1, sIn, sH, sBias, sRh, sHn, tid);
      if (tid < H1) layer[j * H1 + tid] = sHn[tid];
      if (tid == 0) {
        w.inv_denom[j] = 1.0f / sqrtf((float)(w.acc[j * kAcc + H0 + F] / cnt) + 1e-16f);   // HR:621-626
        sSum += w.acc[j * kAcc + H0 + F + 1];
      }
      __syncthreads();
    }
    // global GRU: input = the LAST tensor's new layer state (HR:426-427,720-727), no injected bias
    bias_gru<H1, H2>(theta + O_WG2, theta + O_BG2, theta + O_WC2, theta + O_BC2, sHn, sG, nullptr, sRh, sGn, tid);
    if (tid < H2) { global[tid] = sGn[tid]; sG[tid] = sGn[tid]; }
    __syncthreads();
  } else {
    if (tid == 0)
      for (int j = 0; j < nt; ++j) sSum += w.acc[j * kAcc + H0 + F + 1];
    __syncthreads();
  }
  // next step's inputs: per-tensor gate bias (HR:561-575), problem-wide mean log-lr (HR:432-442), first-step flags
  for (int j = 0; j < nt; ++j) {
    for (int o = tid; o < 3 * H0; o += blockDim.x) {
      float a = 0.f, b = 0.f;
      for (int k = 0; k < H1; ++k) a = fmaf(layer[j * H1 + k], theta[O_PM + k * 3 * H0 + o], a);
      for (int k = 0; k < H2; ++k) b = fmaf(sG[k], theta[O_GM + k * 3 * H0 + o], b);
      w.bias0[j * kB0Stride + o] = (a + theta[O_PB + o]) + (b + theta[O_GB + o]);
    }
  }
  if (tid == 0) *w.mean_log_lr = (float)(sSum / (double)n_total);
  for (int k = tid; k < nt * NS; k += blockDim.x) {
    w.zero_flag[k] = w.any_nz[k] ? 0 : 1;
    w.any_nz[k] = 0;
  }
  __syncthreads();
  for (int k = tid; k < nt * kAcc; k += blockDim.x) w.acc[k] = 0.0;
}

__global__ void __launch_bounds__(kBlock) apply_kernel(float* __restrict__ x, float* __restrict__ update_out,
                                                       const BlockEnt* __restrict__ blocks, int nblocks, Workspace w) {
  for (int b = blockIdx.x; b < nblocks; b += gridDim.x) {   // a few entries per CTA: independent 128-byte rows in flight
    const BlockEnt be = blocks[b];
    if ((int)threadIdx.x >= be.count) continue;
    const int64_t i = be.start + threadIdx.x;
    const float u = w.upd[i] * w.inv_denom[be.tensor];
    x[i] -= u;
    if (update_out) update_out[i] = u;
  }
}

__global__ void init_state_kernel(const float* __restrict__ theta, float* __restrict__ state, int64_t n,
                                  float* __restrict__ layer, float* __restrict__ global, int nt) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) {
#pragma unroll
    for (int k = 0; k < H0; ++k) state[(int64_t)(P_H + k) * n + i] = theta[O_INIT0 + k];   // HR:310
    state[(int64_t)P_SCL * n + i] = 0.f;
    state[(int64_t)P_INP * n + i] = 0.f;
#pragma unroll
    for (int s = 0; s < NS; ++s) {
      state[(int64_t)(P_ACC + s) * n + i] = 0.f;
      state[(int64_t)(P_MS + s) * n + i] = 0.f;
    }
  }
  if (i < (int64_t)nt * H1) layer[i] = theta[O_INIT1 + (int)(i % H1)];                     // HR:318
  if (i < H2) global[i] = theta[O_INIT2 + (int)i];                                        // HR:345-350
}

}  // namespace hrnn
}  // namespace l2o

using namespace l2o::hrnn;

struct l2o_hrnn {
  int nt;
  int64_t n;         // local coordinates
  int64_t n_global;  // problem-wide coordinate count the mean log-lr divides by (== n unless sharded)
  int nblocks;
  BlockEnt* d_blocks;
  int64_t* d_sizes;  // per-tensor counts the per-tensor means divide by (global sizes when sharded)
};

// A handle may be destroyed (Python GC) while another program is capturing a CUDA graph, and cudaFree during a capture
// invalidates it: destroy parks the device buffers and the next l2o_hrnn_create (never inside a capture) frees them.
namespace {
struct Graveyard {
  std::mutex mu;
  std::vector<void*> ptrs;
};
Graveyard& graveyard() {
  static Graveyard* g = new Graveyard();
  return *g;
}
void bury(void* p) {
  if (!p) return;
  Graveyard& g = graveyard();
  std::lock_guard<std::mutex> lk(g.mu);
  g.ptrs.push_back(p);
}
void free_buried() {
  Graveyard& g = graveyard();
  std::vector<void*> take;
  {
    std::lock_guard<std::mutex> lk(g.mu);
    take.swap(g.ptrs);
  }
  for (void* p : take) cudaFree(p);
}
}  // namespace

extern "C" {

int l2o_hrnn_create(l2o_hrnn_handle* out, const int64_t* tensor_sizes, int32_t n_tensors) {
  if (!out || !tensor_sizes || n_tensors <= 0) return L2O_E_INVALID;
  int64_t n = 0;
  int64_t nb = 0;
  for (int j = 0; j < n_tensors; ++j) {
    if (tensor_sizes[j] < 0) return L2O_E_INVALID;   // 0 = this rank holds no coordinate of tensor j (sharded use)
    n += tensor_sizes[j];
    nb += (tensor_sizes[j] + kBlock - 1) / kBlock;
  }
  if (nb > 0x7fffffff || n <= 0) return L2O_E_INVALID;
  BlockEnt* hb = new (std::nothrow) BlockEnt[nb];
  if (!hb) return L2O_E_NOMEM;
  int64_t b = 0, start = 0;
  for (int j = 0; j < n_tensors; ++j) {
    for (int64_t o = 0; o < tensor_sizes[j]; o += kBlock) {
      hb[b].start = start + o;
      hb[b].count = (int32_t)((tensor_sizes[j] - o) < kBlock ? (tensor_sizes[j] - o) : kBlock);
      hb[b].tensor = j;
      ++b;
    }
    start += tensor_sizes[j];
  }
  free_buried();
  l2o_hrnn* h = new (std::nothrow) l2o_hrnn();
  if (!h) { delete[] hb; return L2O_E_NOMEM; }
  h->nt = n_tensors;
  h->n = n;
  h->n_global = n;
  h->nblocks = (int)nb;
  h->d_blocks = nullptr;
  h->d_sizes = nullptr;
  cudaError_t e = cudaMalloc(&h->d_blocks, sizeof(BlockEnt) * nb);
  if (e == cudaSuccess) e = cudaMalloc(&h->d_sizes, sizeof(int64_t) * n_tensors);
  if (e == cudaSuccess) e = cudaMemcpy(h->d_blocks, hb, sizeof(BlockEnt) * nb, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(h->d_sizes, tensor_sizes, sizeof(int64_t) * n_tensors, cudaMemcpyHostToDevice);
  delete[] hb;
  if (e != cudaSuccess) {
    if (h->d_blocks) cudaFree(h->d_blocks);
    if (h->d_sizes) cudaFree(h->d_sizes);
    delete h;
    return l2o::set_cuda_error(e, "l2o_hrnn_create", "cudaMalloc / cudaMemcpy");
  }
  *out = h;
  return L2O_OK;
}

void l2o_hrnn_destroy(l2o_hrnn_handle h) {
  if (!h) return;
  bury(h->d_blocks);
  bury(h->d_sizes);
  delete h;
}

int64_t l2o_hrnn_theta_count(void) { return kTheta; }
int64_t l2o_hrnn_state_floats(void) { return kPlanes; }
int64_t l2o_hrnn_coords(l2o_hrnn_handle h) { return h ? h->n : L2O_E_INVALID; }

int64_t l2o_hrnn_workspace_bytes(l2o_hrnn_handle h) {
  if (!h) return L2O_E_INVALID;
  Workspace w;
  return (int64_t)carve(w, nullptr, h->nt, h->n);
}

static int check_args(l2o_hrnn_handle h, const l2o_hrnn_args* a, bool need_xg) {
  if (!h || !a || !a->theta || !a->state || !a->layer || !a->global || !a->workspace) return L2O_E_INVALID;
  if (need_xg && (!a->x || !a->g)) return L2O_E_INVALID;
  if (l2o::misaligned(a->workspace, 256)) return L2O_E_INVALID;
  return L2O_OK;
}

int l2o_hrnn_init_state(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream) {
  int rc = check_args(h, a, false);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  const int64_t work = h->n > (int64_t)h->nt * H1 ? h->n : (int64_t)h->nt * H1;
  init_state_kernel<<<(unsigned)((work + 255) / 256), 256, 0, st>>>(a->theta, a->state, h->n, a->layer, a->global, h->nt);
  return l2o::after_launch("l2o_hrnn_init_state");
}

// ---- phases.  Single-GPU: prepare = prepare_local + prepare_finish, step = step_local + step_finish.  Sharded: the
// caller all-reduces the per-tensor sums and flags (l2o_hrnn_workspace_layout offsets 0 and 1) between the two phases.
int l2o_hrnn_prepare_local(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream) {
  int rc = check_args(h, a, false);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Workspace w;
  const size_t bytes = carve(w, a->workspace, h->nt, h->n);
  L2O_CUDA_TRY("l2o_hrnn_prepare_local",
               cudaMemsetAsync(a->workspace, 0, bytes - align_up(sizeof(float) * (size_t)h->n, 256), st));
  scan_kernel<<<h->nblocks, kBlock, 0, st>>>(a->state, h->n, h->d_blocks, w);
  return l2o::after_launch("l2o_hrnn_prepare_local");
}

int l2o_hrnn_prepare_finish(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream) {
  int rc = check_args(h, a, false);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Workspace w;
  carve(w, a->workspace, h->nt, h->n);
  tensor_kernel<<<1, 64, 0, st>>>(a->theta, a->layer, a->global, h->nt, h->d_sizes, h->n_global, w, 1);
  return l2o::after_launch("l2o_hrnn_prepare_finish");
}

int l2o_hrnn_prepare(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream) {
  int rc = l2o_hrnn_prepare_local(h, a, stream);
  return rc ? rc : l2o_hrnn_prepare_finish(h, a, stream);
}

int l2o_hrnn_step_local(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream) {
  int rc = check_args(h, a, true);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Workspace w;
  carve(w, a->workspace, h->nt, h->n);
  const char* fn = "l2o_hrnn_step_local";
  rc = l2o::raise_smem_limit(fn, tcg::coord_tc_kernel, sizeof(tcg::SmemG));
  if (rc) return rc;
  const int sms = l2o::device_sms(fn);
  if (sms <= 0) return L2O_E_CUDA;
  const int cap = sms * tcg::kCtasPerSm;   // persistent CTAs
  const int grid = h->nblocks < cap ? h->nblocks : cap;
  tcg::coord_tc_kernel<<<grid, tcg::kTile, sizeof(tcg::SmemG), st>>>(a->theta, a->g, a->state, h->n, h->d_blocks, h->nblocks,
                                                                     w);
  return l2o::after_launch(fn);
}

int l2o_hrnn_step_finish(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream) {
  int rc = check_args(h, a, true);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  Workspace w;
  carve(w, a->workspace, h->nt, h->n);
  tensor_kernel<<<1, 64, 0, st>>>(a->theta, a->layer, a->global, h->nt, h->d_sizes, h->n_global, w, 0);
  rc = l2o::after_launch("l2o_hrnn_step_finish");
  if (rc) return rc;
  apply_kernel<<<(h->nblocks + 3) / 4, kBlock, 0, st>>>(a->x, a->update, h->d_blocks, h->nblocks, w);
  return l2o::after_launch("l2o_hrnn_step_finish");
}

int l2o_hrnn_step(l2o_hrnn_handle h, const l2o_hrnn_args* a, void* stream) {
  int rc = l2o_hrnn_step_local(h, a, stream);
  return rc ? rc : l2o_hrnn_step_finish(h, a, stream);
}

int l2o_hrnn_coord_bwd(l2o_hrnn_handle h, const l2o_hrnn_bwd_args* a, void* stream) {
  if (!h || !a || !a->theta || !a->state_old || !a->g || !a->bias0 || !a->zero_flag || !a->mean_log_lr ||
      !a->d_state_new || !a->d_upd || !a->d_sums || !a->d_state_old || !a->d_theta || !a->d_bias0 || !a->d_mean_log_lr)
    return L2O_E_INVALID;
  if (a->d_g) {
    if (l2o::misaligned(a->d_g, alignof(float))) return L2O_E_INVALID;
    const size_t n = (size_t)h->n, nt = (size_t)h->nt, f = sizeof(float), d = sizeof(double);
    const void* other[] = {a->theta, a->state_old, a->g, a->bias0, a->zero_flag, a->mean_log_lr, a->d_state_new,
                           a->d_upd, a->d_sums, a->d_state_old, a->d_theta, a->d_bias0, a->d_mean_log_lr};
    const size_t bytes[] = {kTheta * f, kPlanes * n * f, n * f, nt * kB0Stride * f, nt * NS * sizeof(int32_t), f,
                            kPlanes * n * f, n * f, nt * kAcc * f, kPlanes * n * f, kTheta * d, nt * kB0Stride * d, d};
    if (l2o::overlaps_any(a->d_g, n * f, other, bytes, 13)) return L2O_E_INVALID;
  }
  bwd::Args k{a->theta, a->state_old, a->g, a->bias0, a->zero_flag, a->mean_log_lr, a->d_state_new, a->d_upd, a->d_sums,
              a->d_state_old, a->d_theta, a->d_bias0, a->d_mean_log_lr, a->d_g};
  const int sms = l2o::device_sms("l2o_hrnn_coord_bwd");
  if (sms <= 0) return L2O_E_CUDA;
  const int grid = h->nblocks < 2 * sms ? h->nblocks : 2 * sms;
  bwd::coord_bwd_kernel<<<grid, bwd::kBwdBlock, 0, (cudaStream_t)stream>>>(k, h->n, h->d_blocks, h->nblocks);
  return l2o::after_launch("l2o_hrnn_coord_bwd");
}

int l2o_hrnn_workspace_layout(l2o_hrnn_handle h, int64_t offsets[7]) {
  if (!h || !offsets) return L2O_E_INVALID;
  Workspace w;
  char* base = (char*)256;   // offsets relative to a dummy non-null base
  carve(w, base, h->nt, h->n);
  offsets[0] = (char*)w.acc - base;
  offsets[1] = (char*)w.any_nz - base;
  offsets[2] = (char*)w.zero_flag - base;
  offsets[3] = (char*)w.bias0 - base;
  offsets[4] = (char*)w.inv_denom - base;
  offsets[5] = (char*)w.mean_log_lr - base;
  offsets[6] = (char*)w.upd - base;
  return L2O_OK;
}

int l2o_hrnn_set_global_sizes(l2o_hrnn_handle h, const int64_t* global_sizes) {
  if (!h || !global_sizes) return L2O_E_INVALID;
  int64_t tot = 0;
  for (int j = 0; j < h->nt; ++j) {
    if (global_sizes[j] <= 0) return L2O_E_INVALID;
    tot += global_sizes[j];
  }
  L2O_CUDA_TRY("l2o_hrnn_set_global_sizes",
               cudaMemcpy(h->d_sizes, global_sizes, sizeof(int64_t) * h->nt, cudaMemcpyHostToDevice));
  h->n_global = tot;
  return L2O_OK;
}

}  // extern "C"
