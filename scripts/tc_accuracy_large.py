"""d-theta accuracy of the BPTT kernels at a size where the per-CTA accumulation is long (test infrastructure; GPU box).
Reference = the exact-fp32 engine run over 1024-coordinate chunks whose results are summed in fp64 (each chunk: one tile
per CTA, T steps in fp32, then fp64 atomics), i.e. no long fp32 accumulation anywhere.  Reports the max-norm relative
error of (a) the tensor-core BPTT and (b) the exact-fp32 engine in ONE launch, both on the same checkpoints / recorded
gradients.

    python scripts/tc_accuracy_large.py [n] [T]"""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import l2o_oracle as orc  # noqa: E402
from tests.helpers import SPECS, make_handle, rel_err  # noqa: E402
from open_l2o_b200.engine import ENGINE_TC, ENGINE_FFMA, OPT_KINDS  # noqa: E402

DEV = "cuda:0"


def main():
    n = int(sys.argv[1]) if len(sys.argv) > 1 else 65536
    T = int(sys.argv[2]) if len(sys.argv) > 2 else 100
    spec = SPECS["dm_identity"]
    gen = torch.Generator().manual_seed(5)
    theta = orc.init_theta(spec, seed=0, out_gain=0.05).to(DEV)
    a, b, x0 = (torch.randn(n, generator=gen).to(DEV) for _ in range(3))
    h = make_handle(spec)
    sf = h.state_floats
    h.set_engine(ENGINE_TC)
    arena = h.new_state(n, DEV)
    ckpt = torch.zeros((T + 1) * sf * n, device=DEV)
    x = x0.clone()
    g_rec = torch.empty(T + 1, n, device=DEV)
    fx = torch.zeros(T + 1, dtype=torch.float64, device=DEV)
    h.unroll_fwd(theta, n, T, arena, opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=a, opt_b=b, opt_alpha=10.0,
                 opt_fscale=1.0 / n, x=x, ckpt=ckpt, g_rec=g_rec, fx=fx)

    def bwd(engine, g, ck, nn):
        h.set_engine(engine)
        d = torch.zeros(h.n_theta, dtype=torch.float64, device=DEV)
        h.unroll_bwd(theta, nn, T, g, ck, d, g_rec=g)
        torch.cuda.synchronize()
        return d
    d_tc = bwd(ENGINE_TC, g_rec, ckpt, n)
    d_ff = bwd(ENGINE_FFMA, g_rec, ckpt, n)
    ck4 = ckpt.view(T + 1, 4, n, 20)
    ref = torch.zeros(h.n_theta, dtype=torch.float64, device=DEV)
    C = 1024
    for lo in range(0, n, C):
        hi = min(n, lo + C)
        ref += bwd(ENGINE_FFMA, g_rec[:, lo:hi].contiguous(), ck4[:, :, lo:hi, :].contiguous().view(-1), hi - lo)
    print("n=%d T=%d  tensor-core BPTT vs chunked-fp64 reference: %.3e   exact-fp32 engine, one launch: %.3e   "
          "(tc vs ffma: %.3e)" % (n, T, rel_err(d_tc, ref), rel_err(d_ff, ref), rel_err(d_tc, d_ff)), flush=True)


if __name__ == "__main__":
    main()
