// Tensor-core (wgmma) engine translation unit.
#include "cwlstm_ffma.cuh"   // load_vec / store_vec / preprocess helpers
#include "cwlstm_tc.cuh"
#include "cwlstm_tc_bwd.cuh"
#include <mutex>
#include <utility>
#include <vector>
#include "l2o_internal.h"

namespace l2o {
// forward / step / BPTT: LSTM-20x2 with identity / LogAndSign preprocessing (cfg 0, 1) and RNNProp's fc(2->20)+ELU net
// (cfg 2).  The BPTT of cfg 2 runs as two passes over time (layer 2, then layer 1) with a caller-provided hand-over buffer.
bool tc_supported(int cfg) { return cfg == 0 || cfg == 1 || cfg == 2; }
bool tc_fwd_ok(const l2o_net* h, const l2o_unroll_args& a) {
  if (a.opt_kind == L2O_OPT_QUADRATIC_BATCH) return false;  // grouped optimizees exchange x: exact-fp32 engine only
  if (h->cfg == 2) return true;                             // fused Adam-feature mode (m, v) or given (m~, g~) rows
  return a.m == nullptr && a.feat_rec == nullptr;
}
// Weight-image buffers are recycled through a process-wide free list and never cudaFree'd: a handle may be destroyed
// (Python GC) while ANOTHER program is capturing a CUDA graph, and cudaFree during a capture invalidates it.
namespace {
struct ImgPool {
  std::mutex mu;
  std::vector<std::pair<int, float*>> free_list;   // (device, pointer)
};
ImgPool& img_pool() {
  static ImgPool* p = new ImgPool();   // intentionally leaked: outlives every handle
  return *p;
}
}  // namespace

void tc_release_image(l2o_net* h) {
  if (!h->tc_img) return;
  ImgPool& P = img_pool();
  std::lock_guard<std::mutex> g(P.mu);
  P.free_list.emplace_back(h->tc_img_dev, h->tc_img);
  h->tc_img = nullptr;
}

static int ensure_image(l2o_net* h, const char* fn) {
  int dev = 0;
  L2O_CUDA_TRY(fn, cudaGetDevice(&dev));
  if (h->tc_img == nullptr || h->tc_img_dev != dev) {
    tc_release_image(h);
    {
      ImgPool& P = img_pool();
      std::lock_guard<std::mutex> g(P.mu);
      for (size_t k = 0; k < P.free_list.size(); ++k)
        if (P.free_list[k].first == dev) {
          h->tc_img = P.free_list[k].second;
          P.free_list.erase(P.free_list.begin() + k);
          break;
        }
    }
    if (h->tc_img == nullptr) L2O_CUDA_TRY(fn, cudaMalloc(&h->tc_img, tc::kImgMaxFloats * sizeof(float)));
    h->tc_img_dev = dev;
    h->tc_img_mode = -1;
  }
  return L2O_OK;
}

bool tc_bwd_ok(const l2o_net* h, const l2o_bwd_args& a) {
  // meta-loss mode (lambda suffix sums of g_rec) or imitation mode with the forward pass's recorded deltas
  const bool mode_ok = a.labels ? (a.delta_seq != nullptr && a.n_total > 0) : a.g_rec != nullptr;
  if (h->cfg == 2 && a.scratch == nullptr) return false;   // fc nets: two passes with a caller-provided hand-over buffer
  if (h->rt.tanh_output && a.delta_seq == nullptr) return false;   // tanh' comes from the recorded deltas
  return tc_supported(h->cfg) && mode_ok;
}

template <class C>
static int tc_launch_bwd_any(const char* fn, const l2o_net* h, const l2o_bwd_args& a, cudaStream_t st, int sms,
                             const l2o_bwd_carry* c) {
  return c ? tc_launch_bwd<C, true>(fn, h->rt, a, h->tc_img, st, sms, *c)
           : tc_launch_bwd<C, false>(fn, h->rt, a, h->tc_img, st, sms, l2o_bwd_carry{});
}

int tc_unroll_bwd(l2o_net* h, const l2o_bwd_args& a, cudaStream_t st, const l2o_bwd_carry* c) {
  if (!tc_bwd_ok(h, a)) return L2O_E_UNSUPPORTED;
  const char* fn = c ? "l2o_unroll_bwd_carry" : "l2o_unroll_bwd";
  int rc = ensure_image(h, fn);
  if (rc) return rc;
  const int sms = device_sms(fn);
  if (sms <= 0) return L2O_E_CUDA;
  rc = L2O_E_UNSUPPORTED;
  if (h->cfg == 0) rc = tc_launch_bwd_any<Cfg<L2O_PRE_IDENTITY, 1, 1, 20, 20>>(fn, h, a, st, sms, c);
  if (h->cfg == 1) rc = tc_launch_bwd_any<Cfg<L2O_PRE_LOGSIGN, 1, 2, 20, 20>>(fn, h, a, st, sms, c);
  if (h->cfg == 2) rc = tc_launch_bwd_any<Cfg<L2O_PRE_FC, 2, 20, 20, 20>>(fn, h, a, st, sms, c);
  h->tc_img_mode = rc == L2O_OK ? 1 : -1;   // after a failed call the image may hold either layout, or a partial one
  return rc;
}

bool tc_step_ok(const l2o_net* h, const l2o_step_args& a) {
  if (h->cfg == 2) return a.m != nullptr;   // fused RNNProp features; precomputed (m~, g~) pairs stay on the FFMA engine
  return tc_supported(h->cfg) && a.m == nullptr && a.in1 == nullptr && a.feat_out == nullptr;
}

// One time step with the state in HBM (external-gradient regime) = the forward unroll with T = 1 and an
// out-of-place final-state write.
int tc_step(l2o_net* h, const l2o_step_args& s, cudaStream_t st) {
  if (!tc_step_ok(h, s)) return L2O_E_UNSUPPORTED;
  const char* fn = "l2o_step";
  int rc = ensure_image(h, fn);
  if (rc) return rc;
  const int sms = device_sms(fn);
  if (sms <= 0) return L2O_E_CUDA;
  l2o_unroll_args a{};
  a.n = s.n;
  a.T = 1;
  a.theta = s.theta;
  a.in_seq = s.in0;
  a.opt_kind = L2O_OPT_NONE;
  a.x = s.x;
  a.state = const_cast<float*>(s.state_in);
  a.delta_seq = s.delta;
  a.m = s.m;
  a.v = s.v;
  a.beta1 = s.beta1;
  a.beta2 = s.beta2;
  a.step0 = 1;
  a.feat_rec = s.feat_out;
  const tc::FwdExtra ex{s.step_ptr, s.t_offset, s.step_ptr ? 0.f : s.p};
  rc = L2O_E_UNSUPPORTED;
  const bool prep = !(s.reuse_weights && h->tc_img_mode == 0);   // forward image of this theta already in place
  if (h->cfg == 0)
    rc = tc_launch_fwd<Cfg<L2O_PRE_IDENTITY, 1, 1, 20, 20>>(fn, h->rt, a, h->tc_img, st, sms, s.state_out, ex, prep);
  if (h->cfg == 1)
    rc = tc_launch_fwd<Cfg<L2O_PRE_LOGSIGN, 1, 2, 20, 20>>(fn, h->rt, a, h->tc_img, st, sms, s.state_out, ex, prep);
  if (h->cfg == 2)
    rc = tc_launch_fwd<Cfg<L2O_PRE_FC, 2, 20, 20, 20>>(fn, h->rt, a, h->tc_img, st, sms, s.state_out, ex, prep);
  h->tc_img_mode = rc == L2O_OK ? 0 : -1;
  return rc;
}

int tc_unroll_fwd(l2o_net* h, const l2o_unroll_args& a, cudaStream_t st) {
  if (!tc_supported(h->cfg) || !tc_fwd_ok(h, a)) return L2O_E_UNSUPPORTED;
  const char* fn = "l2o_unroll_fwd";
  int rc = ensure_image(h, fn);
  if (rc) return rc;
  const int sms = device_sms(fn);
  if (sms <= 0) return L2O_E_CUDA;
  rc = L2O_E_UNSUPPORTED;
  if (h->cfg == 0) rc = tc_launch_fwd<Cfg<L2O_PRE_IDENTITY, 1, 1, 20, 20>>(fn, h->rt, a, h->tc_img, st, sms);
  if (h->cfg == 1) rc = tc_launch_fwd<Cfg<L2O_PRE_LOGSIGN, 1, 2, 20, 20>>(fn, h->rt, a, h->tc_img, st, sms);
  if (h->cfg == 2) rc = tc_launch_fwd<Cfg<L2O_PRE_FC, 2, 20, 20, 20>>(fn, h->rt, a, h->tc_img, st, sms);
  h->tc_img_mode = rc == L2O_OK ? 0 : -1;
  return rc;
}

template <class C>
static int64_t tc_image(const float* theta, float* img, bool with_transposed, cudaStream_t st) {
  using G = tc::Geo<C>;
  const int64_t floats = with_transposed ? G::AllFloats : G::FwdFloats;
  if (img == nullptr) return floats;
  tc::prep_weights_kernel<C><<<16, 256, 0, st>>>(theta, img, with_transposed ? 1 : 0);
  if (int rc = after_launch("l2o_tc_weight_image")) return rc;
  return floats;
}

int64_t tc_weight_image(const l2o_net* h, const float* theta, float* img, bool with_transposed, cudaStream_t st) {
  if (h->cfg == 0) return tc_image<Cfg<L2O_PRE_IDENTITY, 1, 1, 20, 20>>(theta, img, with_transposed, st);
  if (h->cfg == 1) return tc_image<Cfg<L2O_PRE_LOGSIGN, 1, 2, 20, 20>>(theta, img, with_transposed, st);
  if (h->cfg == 2) return tc_image<Cfg<L2O_PRE_FC, 2, 20, 20, 20>>(theta, img, with_transposed, st);
  return L2O_E_UNSUPPORTED;
}

int tc_fwd_variant(const l2o_net* h, const l2o_unroll_args& a) {
  if (!tc_supported(h->cfg) || !tc_fwd_ok(h, a)) return L2O_E_UNSUPPORTED;
  return tc_fwd_fast(h->cfg == 2, h->rt, a, nullptr) ? 1 : 0;
}
}  // namespace l2o
