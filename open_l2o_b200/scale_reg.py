"""The Hessian and Jacobian regularisers of L2O-Scale meta-training (``--reg_optimizer`` / ``--reg_optimizee``,
SC/problems/problem_generator.py:128-368, SC/optimizer/trainable_optimizer.py:307-360 and SC/metaopt.py:458-475; SC/ =
Model_Free_L2O/L2O-Scale/L2O-Scale-Training/).

``Regularizer(option, hessian_itrs, seed)(objective, x, split, gen)`` is reg(x) of one step, with its graph to x:

* ``jacob``: the mean over all coordinates of g^2;
* ``hessian``: Hutchinson, the mean over ``hessian_itrs`` Rademacher probes of p^T H p.  The probes are drawn once per
  objective (problem) from the regulariser's seeded generator and reused at every step;
* ``hessian-ev``: power iteration (top_n = 1) from v0 ~ N(0, I) drawn from ``gen`` at every evaluation: each iteration
  normalises v by ||v|| + 1e-6, takes lambda = (H v).v and v <- H v / (||H v|| + 1e-6); reg is the last lambda;
* ``hessian-esd``: ``hessian_itrs`` Lanczos steps with full re-orthogonalisation from one fixed normalised Rademacher
  vector; reg = the sum of the tridiagonal's eigenvalues = its trace = sum alpha_i.

g is the noise-free gradient of the step's objective on the batch that objective saw: for a ``scale_zoo
.training_objective`` the problem's own objective at ``objective.batch()`` (no gradient noise, no dropout); any other
callable is differentiated as it is.  On a bare analytic family ``hessian`` is ONE ``l2o_zoo_hess_form`` launch that
gives the value and its gradient (saved for the backward); everything else is double or triple autograd, which
reaches the zoo kernels through ``scale_zoo``'s Functions.
"""
from __future__ import annotations

import weakref

import torch

OPTIONS = ("hessian", "jacob", "hessian-ev", "hessian-esd")


def check_options(reg_option, reg_optimizee, use_second_derivatives):
    """The constructor checks of the trainers' regulariser arguments."""
    if reg_option not in OPTIONS:
        raise ValueError("unknown reg_option %r (one of %s)" % (reg_option, ", ".join(OPTIONS)))
    if reg_optimizee and use_second_derivatives and reg_option != "jacob":
        raise NotImplementedError("reg_optimizee with reg_option=%r and use_second_derivatives needs fourth derivatives "
                                  "of the objective; use --nouse_second_derivatives or reg_option='jacob'" % reg_option)


def reg_switch(regularize_time: str, i: int, num_unrolls: int, reg_scale: float) -> bool:
    """Whether partial unroll ``i`` of ``num_unrolls`` adds the regulariser to the meta objective (SC/metaopt.py:458-475):
    ``posterior``: i > int(N reg_scale + 1); ``prior``: i < int(N reg_scale + 1); ``none``: never; anything else: always."""
    b = int(num_unrolls * reg_scale + 1)
    if regularize_time == "posterior":
        return i > b
    if regularize_time == "prior":
        return i < b
    return regularize_time != "none"


class _HutchForm(torch.autograd.Function):
    """mean_k p_k^T H(x) p_k of the probes P [k, n] from one ``l2o_zoo_hess_form`` launch; backward: the saved
    gradient, no launch."""

    @staticmethod
    def forward(ctx, x, P, z):
        q, dq = z.hess_form(x.detach().contiguous(), P)
        ctx.save_for_backward(dq)
        ctx.k = int(P.shape[0])
        return q / ctx.k

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, dr):
        (dq,) = ctx.saved_tensors
        return dr * dq / ctx.k, None, None


def _normalize(v):
    return v / (torch.sqrt((v * v).sum()) + 1e-6)


class Regularizer(object):
    def __init__(self, option="hessian", hessian_itrs=10, seed=None):
        check_options(option, False, False)
        if int(hessian_itrs) < 1:
            raise ValueError("hessian_itrs must be >= 1")
        self.option, self.itrs = option, int(hessian_itrs)
        self._gen = torch.Generator()
        self._gen.manual_seed(0 if seed is None else int(seed))
        self._fixed = weakref.WeakKeyDictionary()

    def probes(self, objective, n: int, device, dtype=torch.float32) -> torch.Tensor:
        """The fixed vectors of ``objective``: ``hessian_itrs`` Rademacher probes [itrs, n] (``hessian``) or the
        normalised Rademacher start [1, n] (``hessian-esd``), drawn on first use."""
        if objective not in self._fixed:
            k = self.itrs if self.option == "hessian" else 1
            p = torch.randint(0, 2, (k, n), generator=self._gen).to(torch.float64) * 2.0 - 1.0
            self._fixed[objective] = _normalize(p) if self.option == "hessian-esd" else p
        return self._fixed[objective].to(device=device, dtype=dtype)

    def __call__(self, objective, x: torch.Tensor, split, gen: torch.Generator) -> torch.Tensor:
        """reg at the flat optimizee vector ``x`` (a tensor that requires grad); ``split(x)`` gives the objective's
        tensors; ``gen`` draws ``hessian-ev``'s start vectors."""
        problem = getattr(objective, "problem", None)
        if problem is not None:
            data, labels = objective.batch()

            def f(ps):
                return problem.objective(ps, data, labels)
            if self.option == "hessian" and problem.family is not None:
                return _HutchForm.apply(x, self.probes(objective, x.numel(), x.device, x.dtype).contiguous(),
                                        problem.kernel(x, data))
        else:
            f = objective
        with torch.enable_grad():
            (g,) = torch.autograd.grad(f(split(x)), x, create_graph=True)
            if self.option == "jacob":
                return (g * g).mean()

            def hv(v):
                return torch.autograd.grad(g, x, grad_outputs=v, create_graph=True, retain_graph=True)[0]
            if self.option == "hessian":
                P = self.probes(objective, x.numel(), x.device, x.dtype)
                return sum((hv(p) * p).sum() for p in P) / P.shape[0]
            if self.option == "hessian-ev":
                v = _normalize(torch.randn(x.numel(), generator=gen).to(device=x.device, dtype=x.dtype))
                for _ in range(self.itrs):
                    v = _normalize(v)
                    w = hv(v)
                    lam = (w * v).sum()
                    v = _normalize(w)
                return lam
            # hessian-esd: Lanczos with full re-orthogonalisation
            v = self.probes(objective, x.numel(), x.device, x.dtype)[0]
            vs, total = [v], 0.0
            w = hv(v)
            a = (w * v).sum()
            total = total + a
            w = w - a * v
            for _ in range(1, self.itrs):
                b = torch.sqrt((w * w).sum())
                v = w
                for u in vs:
                    v = v - (v * u).sum() * u
                v = _normalize(v)
                vs.append(v)
                w = hv(v)
                a = (w * v).sum()
                total = total + a
                w = w - a * v - b * vs[-2]
            return total
