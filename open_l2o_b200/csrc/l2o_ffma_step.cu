// FFMA engine, single-step kernel instantiations.
#include "cwlstm_ffma.cuh"
#include "l2o_internal.h"

namespace l2o {
int ffma_step(const l2o_net* h, const l2o_step_args& a, cudaStream_t st) {
#define X(id, PRE, NIN, F, H1, H2)                                                                  \
  if (h->cfg == id) {                                                                               \
    using C = Cfg<PRE, NIN, F, H1, H2>;                                                             \
    const size_t smem = (size_t)(round4(C::P) + 4) * sizeof(float);                                 \
    return occupancy_launch("l2o_step", step_kernel<C>, kTile, smem, a.n, st, a, h->rt);            \
  }
  L2O_FOR_EACH_CFG(X)
#undef X
  return L2O_E_UNSUPPORTED;
}
}  // namespace l2o
