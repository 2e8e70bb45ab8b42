"""Tensor-core BPTT, block by block: every theta block of the meta-gradient against the fp64 oracle on its own scale.

The BPTT kernel maps its dW accumulator rows to theta through a row permutation (cwlstm_tc_bwd.cuh dw_row); a block
of small magnitude (a bias, the LogAndSign feature rows, the fc layer) that went to the wrong rows would still pass a
whole-vector relative error."""
import numpy as np
import pytest
import torch

from oracle import l2o_oracle as orc
from tests.helpers import SPECS, make_handle, rel_err
from tests.test_kernels_gpu import _fused_problem, _theta

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
# Floor of the per-block tolerance.  Block by block, the engine's fast activations and 3xTF32 recompute reach 2.4e-5 of
# a block's max-norm (the identity net's recurrent lstm_2 rows; measured on an H100 over seeds, unroll lengths and
# output gains), above the 1e-5 that holds for the whole vector.  A row sent to the wrong theta entries, or a block left
# at zero, is off by O(1).
BLOCK_TOL = 5e-5


def theta_blocks(spec):
    """(name, offset, count) of each theta block; a gate matrix splits into its input rows and its recurrent rows."""
    off, out = 0, []
    for mod, var, shape in spec.shapes():
        cnt = int(np.prod(shape))
        if var == "w_gates":
            k_in = shape[0] - shape[1] // 4
            out.append((f"{mod}/w_gates[inputs]", off, k_in * shape[1]))
            out.append((f"{mod}/w_gates[h]", off + k_in * shape[1], cnt - k_in * shape[1]))
        else:
            out.append((f"{mod}/{var}", off, cnt))
        off += cnt
    assert off == spec.n_theta()
    return out


@pytest.mark.parametrize("name", ["dm_identity", "dm_logsign", "rnnprop"])
def test_tc_bptt_every_theta_block_matches_oracle(name):
    """Fused Rastrigin unroll on the tensor-core engine, then its BPTT; a ragged n (not a multiple of 64 or of 4)."""
    from open_l2o_b200.engine import ENGINE_TC, OPT_KINDS
    spec = SPECS[name]
    n, T = 2037, 5
    gen = torch.Generator().manual_seed(23)
    theta = _theta(spec, gain=0.3)
    prob, x0 = _fused_problem("rastrigin_sep", n, gen)
    prob64 = orc.FusedProblem("rastrigin_sep", prob.a.double(), prob.b.double(), prob.alpha, prob.fscale)
    kw32, kw64 = {}, {}
    if spec.rnnprop:
        kw32 = dict(mv0=(torch.zeros(n), torch.zeros(n)), step0=1, beta1=0.95, beta2=0.95)
        kw64 = dict(mv0=(torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)), step0=1,
                    beta1=0.95, beta2=0.95)
    g64, _ = orc.meta_grad(spec, theta.double(), x0.double(), orc.initial_state(spec, n, torch.float64), None, T,
                           grad_of=prob64.f_and_g, **kw64)
    g32, _ = orc.meta_grad(spec, theta, x0, orc.initial_state(spec, n), None, T, grad_of=prob.f_and_g, **kw32)

    h = make_handle(spec)
    h.set_engine(ENGINE_TC)
    th = theta.to(DEV)
    arena = h.new_state(n, DEV)
    ckpt = torch.zeros((T + 1) * h.state_floats * n, device=DEV)
    x = x0.to(DEV).clone()
    g_rec = torch.empty(T + 1, n, device=DEV)
    fwd, bwd = {}, {}
    if spec.rnnprop:
        feat = torch.empty(T, 2, n, device=DEV)
        dseq = torch.empty(T, n, device=DEV)
        fwd = dict(m=torch.zeros(n, device=DEV), v=torch.zeros(n, device=DEV), beta1=0.95, beta2=0.95, step0=1,
                   feat_rec=feat, delta_seq=dseq)
        bwd = dict(delta_seq=dseq, scratch=torch.empty(T, n, 20, device=DEV))
    h.unroll_fwd(th, n, T, arena, opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=prob.a.to(DEV), opt_b=prob.b.to(DEV),
                 opt_alpha=prob.alpha, opt_fscale=prob.fscale, x=x, ckpt=ckpt, g_rec=g_rec, **fwd)
    dtheta = torch.zeros(h.n_theta, dtype=torch.float64, device=DEV)
    h.unroll_bwd(th, n, T, feat if spec.rnnprop else g_rec[:T].contiguous(), ckpt, dtheta, g_rec=g_rec, **bwd)
    torch.cuda.synchronize()
    dtheta = dtheta.cpu()

    for block, off, cnt in theta_blocks(spec):
        ref = g64[off:off + cnt]
        assert float(ref.abs().max()) > 0, block
        slack = max(BLOCK_TOL, 3.0 * rel_err(g32[off:off + cnt], ref))
        err = rel_err(dtheta[off:off + cnt], ref)
        assert err <= slack, (block, err, slack)
