// FFMA engine, BPTT kernel instantiations.
#include "cwlstm_ffma.cuh"
#include "l2o_internal.h"

namespace l2o {
int ffma_unroll_bwd(const l2o_net* h, const l2o_bwd_args& a, cudaStream_t st, const l2o_bwd_carry* c) {
#define X(id, PRE, NIN, F, H1, H2)                                                                             \
  if (h->cfg == id) {                                                                                          \
    using C = Cfg<PRE, NIN, F, H1, H2>;                                                                        \
    const size_t smem = BwdGeom<C>::BYTES;                                                                     \
    return c ? occupancy_launch("l2o_unroll_bwd_carry", unroll_bwd_kernel<C, true>, kTile, smem, a.n, st, a,   \
                                h->rt, *c)                                                                     \
             : occupancy_launch("l2o_unroll_bwd", unroll_bwd_kernel<C, false>, kTile, smem, a.n, st, a, h->rt, \
                                l2o_bwd_carry{});                                                              \
  }
  L2O_FOR_EACH_CFG(X)
#undef X
  return L2O_E_UNSUPPORTED;
}
}  // namespace l2o
