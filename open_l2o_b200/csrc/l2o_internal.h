// Internal (non-ABI) declarations shared by the translation units of libl2o_b200.so.
#pragma once
#include <cuda_runtime.h>

#include "cwlstm_common.cuh"
#include "l2o_b200.h"

// Net shapes compiled into this build.  (id, PRE, NIN, F, H1, H2)
#define L2O_FOR_EACH_CFG(X)               \
  X(0, L2O_PRE_IDENTITY, 1, 1, 20, 20)    \
  X(1, L2O_PRE_LOGSIGN, 1, 2, 20, 20)     \
  X(2, L2O_PRE_FC, 2, 20, 20, 20)         \
  X(3, L2O_PRE_IDENTITY, 1, 1, 0, 0)      \
  X(4, L2O_PRE_IDENTITY, 1, 1, 1, 0)      \
  X(5, L2O_PRE_IDENTITY, 1, 1, 1, 1)      \
  X(6, L2O_PRE_IDENTITY, 1, 1, 2, 3)

struct l2o_net {
  l2o_net_desc desc;
  int cfg;
  int engine;
  int64_t n_theta;
  int64_t state_floats;
  l2o::NetRt rt;
  float* tc_img;   // device-side weight image of the tensor-core engine, then its BPTT dW partials (owned; lazy)
  int tc_img_dev;
  int tc_img_mode; // what the image currently holds: -1 nothing, 0 forward layout, 1 BPTT layout
};

namespace l2o {
// Host side of every launch.  `fn` names the C entry point being served: a failure is recorded for
// l2o_last_cuda_error as "<fn>: <CUDA call>: <error string>" and returns L2O_E_CUDA.
int set_cuda_error(cudaError_t e, const char* fn, const char* call);
int device_sms(const char* fn);   // SM count of the current device (cached), 0 on failure
// Raises kernel's dynamic shared-memory limit on the current device to at least smem.  The process remembers the
// highest limit set per kernel and device, whichever thread set it, so the limit is only ever raised: a lower one
// would break the launches another thread sized for a higher one.
int raise_smem_limit(const char* fn, const void* kernel, size_t smem);
// raise_smem_limit, then grid = min(ceil(n / block), occupancy x SMs) for (kernel, block, smem), the resident CTAs
// cached per kernel, device, block and smem on each thread.  L2O_E_UNSUPPORTED when not one CTA fits on an SM.
int occupancy_grid(const char* fn, const void* kernel, int block, size_t smem, int64_t n, int& grid);
// Checks the launch just issued with one cudaGetLastError and counts it in l2o_launch_count if it succeeded.
int after_launch(const char* fn);

template <class K>
int raise_smem_limit(const char* fn, K* kernel, size_t smem) {
  return raise_smem_limit(fn, (const void*)kernel, smem);
}

// Launches kernel(args...) over n items, `block` per CTA, with at most as many CTAs as are resident at once (the
// kernels loop over the remaining blocks).
template <class K, class... Args>
int occupancy_launch(const char* fn, K* kernel, int block, size_t smem, int64_t n, cudaStream_t st, const Args&... args) {
  int grid = 0;
  if (int rc = occupancy_grid(fn, (const void*)kernel, block, smem, n, grid)) return rc;
  kernel<<<grid, block, smem, st>>>(args...);
  return after_launch(fn);
}

// occupancy_launch as a cooperative launch (cudaLaunchAttributeCooperative, also valid for captured graph nodes): the
// grid is at most the resident CTAs, so every CTA is running at once and the kernel may use cg::this_grid().sync().
template <class... KArgs, class... Args>
int cooperative_launch(const char* fn, void (*kernel)(KArgs...), int block, size_t smem, int64_t n, cudaStream_t st,
                       const Args&... args) {
  int grid = 0;
  if (int rc = occupancy_grid(fn, (const void*)kernel, block, smem, n, grid)) return rc;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeCooperative;
  attr[0].val.cooperative = 1;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)grid);
  cfg.blockDim = dim3((unsigned)block);
  cfg.dynamicSmemBytes = smem;
  cfg.stream = st;
  cfg.attrs = attr;
  cfg.numAttrs = 1;
  const cudaError_t e = cudaLaunchKernelEx(&cfg, kernel, args...);
  if (e != cudaSuccess) return set_cuda_error(e, fn, "cudaLaunchKernelEx (cooperative)");
  return after_launch(fn);
}

inline bool misaligned(const void* p, uintptr_t align) { return ((uintptr_t)p & (align - 1)) != 0; }

// Does the byte range [p, p + bytes) share a byte with any of the ranges (q[k], qbytes[k])?  Null q[k] are skipped.
inline bool overlaps_any(const void* p, size_t bytes, const void* const* q, const size_t* qbytes, int nq) {
  const uintptr_t a = (uintptr_t)p;
  for (int k = 0; k < nq; ++k) {
    const uintptr_t b = (uintptr_t)q[k];
    if (b && a < b + qbytes[k] && b < a + bytes) return true;
  }
  return false;
}

int ffma_step(const l2o_net* h, const l2o_step_args& a, cudaStream_t st);
int ffma_unroll_fwd(const l2o_net* h, const l2o_unroll_args& a, cudaStream_t st);
// c: the boundary conditions of a segmented sweep (l2o_unroll_bwd_carry), null for a whole unroll
int ffma_unroll_bwd(const l2o_net* h, const l2o_bwd_args& a, cudaStream_t st, const l2o_bwd_carry* c = nullptr);

bool tc_supported(int cfg);
void tc_release_image(l2o_net* h);   // hand the weight image back to the process-wide pool (never cudaFree)
bool tc_fwd_ok(const l2o_net* h, const l2o_unroll_args& a);
int tc_unroll_fwd(l2o_net* h, const l2o_unroll_args& a, cudaStream_t st);
int tc_fwd_variant(const l2o_net* h, const l2o_unroll_args& a);   // l2o_tc_fwd_variant
int64_t tc_weight_image(const l2o_net* h, const float* theta, float* img, bool with_transposed,
                        cudaStream_t st);   // l2o_tc_weight_image
bool tc_step_ok(const l2o_net* h, const l2o_step_args& a);
int tc_step(l2o_net* h, const l2o_step_args& a, cudaStream_t st);
bool tc_bwd_ok(const l2o_net* h, const l2o_bwd_args& a);
int tc_unroll_bwd(l2o_net* h, const l2o_bwd_args& a, cudaStream_t st, const l2o_bwd_carry* c = nullptr);
}  // namespace l2o

#define L2O_CUDA_TRY(fn, expr)                                            \
  do {                                                                    \
    cudaError_t e__ = (expr);                                             \
    if (e__ != cudaSuccess) return l2o::set_cuda_error(e__, fn, #expr);   \
  } while (0)
