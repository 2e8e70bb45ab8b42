// FFMA engine, BPTT kernel instantiations.
#include "l2o_ffma_launch.cuh"

namespace l2o {
template <class C, bool CARRY>
static int do_unroll_bwd(const l2o_net* h, const l2o_bwd_args& a, cudaStream_t st, const l2o_bwd_carry& c) {
  auto k = unroll_bwd_kernel<C, CARRY>;
  const size_t smem = BwdGeom<C>::BYTES;
  int grid = 1;
  int rc = ffma_launch_cfg(k, smem, a.n, grid);
  if (rc) return rc;
  k<<<grid, kTile, smem, st>>>(a, h->rt, c);
  count_launch();
  L2O_CUDA_TRY(cudaGetLastError());
  return L2O_OK;
}

int ffma_unroll_bwd(const l2o_net* h, const l2o_bwd_args& a, cudaStream_t st, const l2o_bwd_carry* c) {
#define X(id, PRE, NIN, F, H1, H2)                                                             \
  if (h->cfg == id) return c ? do_unroll_bwd<Cfg<PRE, NIN, F, H1, H2>, true>(h, a, st, *c)     \
                             : do_unroll_bwd<Cfg<PRE, NIN, F, H1, H2>, false>(h, a, st, l2o_bwd_carry{});
  L2O_FOR_EACH_CFG(X)
#undef X
  return L2O_E_UNSUPPORTED;
}
}  // namespace l2o
