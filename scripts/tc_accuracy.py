"""Accuracy report of the tensor-core engine against the fp64 oracle (test infrastructure; run on the GPU box):
pre-recorded-gradient unroll (state / deltas) and fused Rastrigin forward + BPTT (x_T, fx, dtheta), next to the
error the fp32 oracle itself has against fp64 on the same inputs.  Used to A/B numerics-affecting kernel variants
(L2O_LIB=<variant .so> python scripts/tc_accuracy.py)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from oracle import l2o_oracle as orc  # noqa: E402
from tests.helpers import SPECS, make_handle, rel_err  # noqa: E402
from open_l2o_b200.engine import ENGINE_TC, ENGINE_FFMA, OPT_KINDS  # noqa: E402

DEV = "cuda:0"


def fused(spec_name, T, n=2000, engine=ENGINE_TC):
    spec = SPECS[spec_name]
    gen = torch.Generator().manual_seed(5)
    theta = orc.init_theta(spec, seed=0, out_gain=0.05)
    a = torch.randn(n, generator=gen)
    b = torch.randn(n, generator=gen)
    x0 = torch.randn(n, generator=gen)
    prob = orc.FusedProblem("rastrigin_sep", a, b, 10.0, 1.0 / n)
    prob64 = orc.FusedProblem("rastrigin_sep", a.double(), b.double(), 10.0, 1.0 / n)
    g64, r64 = orc.meta_grad(spec, theta.double(), x0.double(), orc.initial_state(spec, n, torch.float64), None, T,
                             grad_of=prob64.f_and_g)
    g32, r32 = orc.meta_grad(spec, theta, x0, orc.initial_state(spec, n), None, T, grad_of=prob.f_and_g)
    h = make_handle(spec)
    h.set_engine(engine)
    sf = h.state_floats
    th = theta.to(DEV)
    arena = h.new_state(n, DEV)
    ckpt = torch.zeros((T + 1) * sf * n, device=DEV)
    x = x0.to(DEV).clone()
    g_rec = torch.empty(T + 1, n, device=DEV)
    fx = torch.zeros(T + 1, dtype=torch.float64, device=DEV)
    h.unroll_fwd(th, n, T, arena, opt_kind=OPT_KINDS["rastrigin_sep"], opt_a=a.to(DEV), opt_b=b.to(DEV),
                 opt_alpha=10.0, opt_fscale=1.0 / n, x=x, ckpt=ckpt, g_rec=g_rec, fx=fx)
    d = torch.zeros(h.n_theta, dtype=torch.float64, device=DEV)
    h.unroll_bwd(th, n, T, g_rec, ckpt, d, g_rec=g_rec)
    torch.cuda.synchronize()
    return {"x": rel_err(x, r64.x_final), "x_o32": rel_err(r32.x_final, r64.x_final), "fx": rel_err(fx, r64.fx),
            "dtheta": rel_err(d, g64), "dtheta_o32": rel_err(g32, g64)}


if __name__ == "__main__":
    print("lib:", os.environ.get("L2O_LIB", "(default)"))
    for name, eng in (("tc", ENGINE_TC), ("ffma", ENGINE_FFMA)):
        for T in (20, 100):
            r = fused("dm_identity", T, engine=eng)
            print(f"  {name:4s} T={T:3d}  " + "  ".join(f"{k}={v:.2e}" for k, v in r.items()), flush=True)
