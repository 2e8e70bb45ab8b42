// C-ABI of the engine (include/l2o_b200.h): argument validation and engine dispatch.
#include <cuda_runtime.h>

#include <atomic>
#include <cmath>
#include <cstdio>
#include <map>
#include <new>
#include <tuple>
#include <utility>

#include "l2o_internal.h"

namespace {
std::atomic<int64_t> g_launches{0};
thread_local char g_cuda_err[256] = "";

int find_cfg(const l2o_net_desc& d) {
  const int h1 = d.n_layers >= 1 ? d.hidden[0] : 0;
  const int h2 = d.n_layers >= 2 ? d.hidden[1] : 0;
  const int f = d.preprocess == L2O_PRE_FC ? d.fc_dim : (d.preprocess == L2O_PRE_LOGSIGN ? 2 * d.n_in : d.n_in);
#define X(id, PRE, NIN, F, H1, H2) \
  if (d.preprocess == PRE && d.n_in == NIN && f == F && h1 == H1 && h2 == H2) return id;
  L2O_FOR_EACH_CFG(X)
#undef X
  return -1;
}

__global__ void adam_kernel(float* __restrict__ theta, const double* __restrict__ dtheta, float* __restrict__ m,
                            float* __restrict__ v, int64_t n, float lr_t, float b1, float b2, float eps) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float g = (float)dtheta[i];
  const float mi = b1 * m[i] + (1.0f - b1) * g;
  const float vi = b2 * v[i] + (1.0f - b2) * g * g;
  m[i] = mi;
  v[i] = vi;
  theta[i] -= lr_t * mi / (sqrtf(vi) + eps);
}

__global__ void log_and_sign_kernel(const float* __restrict__ g, float* __restrict__ out, int64_t n, float k, float ek) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float lo, sg;
  l2o::log_and_sign(g[i], k, ek, lo, sg);
  out[i] = lo;
  out[n + i] = sg;
}
}  // namespace

namespace l2o {
int set_cuda_error(cudaError_t e, const char* fn, const char* call) {
  snprintf(g_cuda_err, sizeof(g_cuda_err), "%s: %s: %s", fn, call, cudaGetErrorString(e));
  return L2O_E_CUDA;
}

static int current_device(const char* fn, int& dev) {
  L2O_CUDA_TRY(fn, cudaGetDevice(&dev));
  return L2O_OK;
}

int device_sms(const char* fn) {
  static thread_local int cached_dev = -1, sms = 0;
  int dev = 0;
  if (current_device(fn, dev)) return 0;
  if (dev != cached_dev) {
    int v = 0;
    const cudaError_t e = cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    if (e != cudaSuccess) {
      set_cuda_error(e, fn, "cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev)");
      return 0;
    }
    sms = v;
    cached_dev = dev;
  }
  return sms;
}

static int raise_smem_limit_on(const char* fn, int dev, const void* kernel, size_t smem) {
  static thread_local std::map<std::pair<const void*, int>, size_t> limit;
  size_t& lim = limit[{kernel, dev}];
  if (smem <= lim) return L2O_OK;
  L2O_CUDA_TRY(fn, cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  lim = smem;
  return L2O_OK;
}

int raise_smem_limit(const char* fn, const void* kernel, size_t smem) {
  int dev = 0;
  if (int rc = current_device(fn, dev)) return rc;
  return raise_smem_limit_on(fn, dev, kernel, smem);
}

int occupancy_grid(const char* fn, const void* kernel, int block, size_t smem, int64_t n, int& grid) {
  static thread_local std::map<std::tuple<const void*, int, int, size_t>, int> resident;
  int dev = 0;
  if (int rc = current_device(fn, dev)) return rc;
  const auto key = std::make_tuple(kernel, dev, block, smem);
  auto it = resident.find(key);
  if (it == resident.end()) {
    if (int rc = raise_smem_limit_on(fn, dev, kernel, smem)) return rc;
    int occ = 0;
    L2O_CUDA_TRY(fn, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, block, smem));
    if (occ < 1) return L2O_E_UNSUPPORTED;
    const int sms = device_sms(fn);
    if (sms <= 0) return L2O_E_CUDA;
    it = resident.emplace(key, occ * sms).first;
  }
  const int64_t blocks = (n + block - 1) / block;
  grid = (int)(blocks < it->second ? blocks : it->second);
  return L2O_OK;
}

int after_launch(const char* fn) {
  const cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return set_cuda_error(e, fn, "kernel launch");
  ++g_launches;
  return L2O_OK;
}
}  // namespace l2o

extern "C" {

int l2o_net_create(l2o_handle* out, const l2o_net_desc* d) {
  if (!out || !d) return L2O_E_INVALID;
  if (d->n_layers < 0 || d->n_layers > 2 || (d->n_in != 1 && d->n_in != 2)) return L2O_E_INVALID;
  const int cfg = find_cfg(*d);
  if (cfg < 0) return L2O_E_UNSUPPORTED;
  l2o_net* h = new (std::nothrow) l2o_net();
  if (!h) return L2O_E_NOMEM;
  h->desc = *d;
  h->cfg = cfg;
  h->engine = L2O_ENGINE_AUTO;
  h->tc_img = nullptr;
  h->tc_img_dev = -1;
  h->tc_img_mode = -1;
  h->rt.scale = d->scale;
  h->rt.logsign_k = d->logsign_k;
  h->rt.logsign_ek = (float)std::exp((double)d->logsign_k);
  h->rt.tanh_output = d->tanh_output;
#define X(id, PRE, NIN, F, H1, H2)                               \
  if (cfg == id) {                                               \
    h->n_theta = l2o::Cfg<PRE, NIN, F, H1, H2>::P;               \
    h->state_floats = l2o::Cfg<PRE, NIN, F, H1, H2>::SF;         \
  }
  L2O_FOR_EACH_CFG(X)
#undef X
  *out = h;
  return L2O_OK;
}

void l2o_net_destroy(l2o_handle h) {
  if (!h) return;
  l2o::tc_release_image(h);
  delete h;
}

int l2o_net_set_engine(l2o_handle h, int32_t engine) {
  if (!h || engine < L2O_ENGINE_AUTO || engine > L2O_ENGINE_TC) return L2O_E_INVALID;
  if (engine == L2O_ENGINE_TC && !l2o::tc_supported(h->cfg)) return L2O_E_UNSUPPORTED;
  h->engine = engine;
  return L2O_OK;
}

int64_t l2o_theta_count(l2o_handle h) { return h ? h->n_theta : L2O_E_INVALID; }
int64_t l2o_state_floats(l2o_handle h) { return h ? h->state_floats : L2O_E_INVALID; }

int l2o_workspace_bytes(l2o_handle h, int64_t n, int32_t T, size_t* fwd_bytes, size_t* bwd_bytes) {
  if (!h || n < 0 || T < 0) return L2O_E_INVALID;
  const size_t arena = (size_t)h->state_floats * (size_t)n * sizeof(float);
  const size_t ckpt = arena * ((size_t)T + 1);
  const size_t grec = (size_t)(T + 1) * (size_t)n * sizeof(float);
  const size_t feat = h->desc.n_in == 2 ? (size_t)T * 2 * (size_t)n * sizeof(float) : 0;
  if (fwd_bytes) *fwd_bytes = arena + ckpt + grec + feat;
  // fc(20) nets: + the recorded deltas and the [T][n][20] hand-over buffer of the two-pass tensor-core BPTT (both optional)
  const size_t fc_extra = h->cfg == 2 ? (size_t)T * (size_t)n * (1 + 20) * sizeof(float) : 0;
  if (bwd_bytes) *bwd_bytes = ckpt + grec + feat + fc_extra + (size_t)h->n_theta * sizeof(double);
  return L2O_OK;
}

int l2o_step(l2o_handle h, const l2o_step_args* a, void* stream) {
  if (!h || !a || a->n < 0 || !a->theta || !a->in0) return L2O_E_INVALID;
  if (h->state_floats > 0 && (!a->state_in || !a->state_out)) return L2O_E_INVALID;
  if (h->desc.n_in == 2 && !a->m && !a->in1) return L2O_E_INVALID;
  if ((a->m == nullptr) != (a->v == nullptr)) return L2O_E_INVALID;
  if (a->m && h->desc.n_in != 2) return L2O_E_INVALID;
  if (a->n == 0) return L2O_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const bool tc_can = l2o::tc_step_ok(h, *a);
  if (h->engine == L2O_ENGINE_TC) return tc_can ? l2o::tc_step(h, *a, st) : L2O_E_UNSUPPORTED;
  // AUTO: the tensor-core path pays a fixed cost (weight image prep + staging) per launch; use it for real sizes
  if (h->engine == L2O_ENGINE_AUTO && tc_can && a->n >= 16384) return l2o::tc_step(h, *a, st);
  return l2o::ffma_step(h, *a, st);
}

int l2o_unroll_fwd(l2o_handle h, const l2o_unroll_args* a, void* stream) {
  if (!h || !a || a->n < 0 || a->T < 0 || !a->theta) return L2O_E_INVALID;
  if (a->opt_kind == L2O_OPT_NONE && !a->in_seq && a->T > 0) return L2O_E_INVALID;
  if (a->opt_kind < L2O_OPT_NONE || a->opt_kind > L2O_OPT_QUADRATIC_BATCH) return L2O_E_INVALID;
  if (a->opt_kind == L2O_OPT_QUADRATIC_BATCH &&
      (a->opt_group < 1 || a->opt_group > 128 || a->n % a->opt_group != 0)) return L2O_E_INVALID;
  if (a->opt_kind != L2O_OPT_NONE && (!a->x || !a->opt_a || !a->opt_b)) return L2O_E_INVALID;
  if (a->opt_kind != L2O_OPT_NONE && h->desc.n_in == 2 && !a->m) return L2O_E_INVALID;
  if (h->state_floats > 0 && !a->state) return L2O_E_INVALID;
  if ((a->m == nullptr) != (a->v == nullptr)) return L2O_E_INVALID;
  if (a->m && h->desc.n_in != 2) return L2O_E_INVALID;
  if (a->labels && (!a->imit_loss || a->n_total <= 0)) return L2O_E_INVALID;
  if (a->n == 0) return L2O_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const bool tc_can = l2o::tc_supported(h->cfg) && l2o::tc_fwd_ok(h, *a);
  if (h->engine == L2O_ENGINE_TC) return tc_can ? l2o::tc_unroll_fwd(h, *a, st) : L2O_E_UNSUPPORTED;
  if (h->engine == L2O_ENGINE_AUTO && tc_can) return l2o::tc_unroll_fwd(h, *a, st);
  return l2o::ffma_unroll_fwd(h, *a, st);
}

int l2o_tc_fwd_variant(l2o_handle h, const l2o_unroll_args* a) {
  if (!h || !a) return L2O_E_INVALID;
  return l2o::tc_fwd_variant(h, *a);
}

int64_t l2o_tc_weight_image(l2o_handle h, const float* theta, float* img, int32_t with_transposed, void* stream) {
  if (!h || (img && !theta) || l2o::misaligned(img, 16)) return L2O_E_INVALID;
  return l2o::tc_weight_image(h, theta, img, with_transposed != 0, (cudaStream_t)stream);
}

int l2o_unroll_bwd(l2o_handle h, const l2o_bwd_args* a, void* stream) {
  if (!h || !a || a->n < 0 || a->T < 0 || !a->theta || !a->dtheta) return L2O_E_INVALID;
  if (a->T > 0 && !a->in_seq) return L2O_E_INVALID;
  if (h->state_floats > 0 && !a->ckpt) return L2O_E_INVALID;
  // both engines read checkpoint rows 16 bytes at a time (FFMA: float4 loads; tensor cores: TMA bulk copies)
  if (l2o::misaligned(a->ckpt, 16)) return L2O_E_INVALID;
  if (!a->g_rec && (!a->labels || a->n_total <= 0)) return L2O_E_INVALID;
  if (a->n == 0 || a->T == 0) return L2O_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const bool tc_can = l2o::tc_bwd_ok(h, *a);
  if (h->engine == L2O_ENGINE_TC) return tc_can ? l2o::tc_unroll_bwd(h, *a, st) : L2O_E_UNSUPPORTED;
  if (h->engine == L2O_ENGINE_AUTO && tc_can) return l2o::tc_unroll_bwd(h, *a, st);
  return l2o::ffma_unroll_bwd(h, *a, st);
}

int l2o_unroll_bwd_carry(l2o_handle h, const l2o_bwd_args* a, const l2o_bwd_carry* c, void* stream) {
  if (!h || !a || !c || a->n < 0 || a->T < 0 || !a->theta || !a->dtheta) return L2O_E_INVALID;
  if (a->T > 0 && !a->in_seq) return L2O_E_INVALID;
  if (h->state_floats > 0 && (!a->ckpt || !c->d_state)) return L2O_E_INVALID;
  // the FFMA engine moves checkpoint and adjoint-state rows as float4, the tensor-core engine copies checkpoints by TMA
  if (l2o::misaligned(a->ckpt, 16) || l2o::misaligned(c->d_state, 16)) return L2O_E_INVALID;
  if (!c->lam) return L2O_E_INVALID;
  if (!a->g_rec && (!a->labels || a->n_total <= 0)) return L2O_E_INVALID;
  if (a->labels) return L2O_E_UNSUPPORTED;   // imitation losses have no lambda to carry
  if (a->n == 0 || a->T == 0) return L2O_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const bool tc_can = l2o::tc_bwd_ok(h, *a);
  if (h->engine == L2O_ENGINE_TC) return tc_can ? l2o::tc_unroll_bwd(h, *a, st, c) : L2O_E_UNSUPPORTED;
  if (h->engine == L2O_ENGINE_AUTO && tc_can) return l2o::tc_unroll_bwd(h, *a, st, c);
  return l2o::ffma_unroll_bwd(h, *a, st, c);
}

int l2o_adam_step(float* theta, const double* dtheta, float* m, float* v, int64_t n, int32_t k, float lr, float beta1,
                  float beta2, float eps, void* stream) {
  if (!theta || !dtheta || !m || !v || n < 0 || k < 1) return L2O_E_INVALID;
  if (n == 0) return L2O_OK;
  // tf.train.AdamOptimizer (TF 1.14): lr_t = lr * sqrt(1 - b2^k) / (1 - b1^k)
  const double lr_t = (double)lr * std::sqrt(1.0 - std::pow((double)beta2, k)) / (1.0 - std::pow((double)beta1, k));
  const int block = 256;
  adam_kernel<<<(int)((n + block - 1) / block), block, 0, (cudaStream_t)stream>>>(theta, dtheta, m, v, n, (float)lr_t,
                                                                                 beta1, beta2, eps);
  return l2o::after_launch("l2o_adam_step");
}

int l2o_log_and_sign(const float* g, float* out, int64_t n, float k, void* stream) {
  if (!g || !out || n < 0) return L2O_E_INVALID;
  if (n == 0) return L2O_OK;
  const int block = 256;
  log_and_sign_kernel<<<(int)((n + block - 1) / block), block, 0, (cudaStream_t)stream>>>(g, out, n, k,
                                                                                         (float)std::exp((double)k));
  return l2o::after_launch("l2o_log_and_sign");
}

int64_t l2o_launch_count(void) { return g_launches.load(); }

const char* l2o_status_string(int s) {
  switch (s) {
    case L2O_OK: return "ok";
    case L2O_E_INVALID: return "invalid argument";
    case L2O_E_UNSUPPORTED: return "net shape or mode not supported by this build";
    case L2O_E_CUDA: return "CUDA error";
    case L2O_E_NOMEM: return "out of memory";
    default: return "unknown status";
  }
}

const char* l2o_last_cuda_error(void) { return g_cuda_err; }
const char* l2o_version(void) { return "l2o_b200 0.3 (sm_90a; engines: ffma, wgmma)"; }

}  // extern "C"
