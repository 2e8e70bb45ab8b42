"""CPU oracle for the confocal_microscopy_3d and square_cos optimizees (test infrastructure, like ``oracle/``; the
product path never imports it).

Op-for-op torch restatements of DM/problems.py:799-956 (confocal_microscopy_3d, ``inference=False``) in the reference's
dense ``[B, nx*ny*nz]`` tf.meshgrid form, and of DM/problems.py:959-995 (square_cos), in the dtype of their inputs
(fp32 or fp64).  ``DM/`` is the reference's ``Model_Free_L2O/L2O-DM and L2O-RNNProp/``.

PARITY PINNING.  TensorFlow and TensorFlow Probability are not installed, so two points are **parity unpinned**: the op
order of ``tfd.Uniform.quantile`` (taken here as ``low + p (high - low)``) and TF's fp32 ``erf`` (torch's ``erf``
here, CUDA's ``erff`` in the kernel)."""
import torch


def square_cos_f(x, w, y, wcos):
    """DM/problems.py:959-995. x [B,d], w / wcos [B,d,d], y [B,d]; the angle constant is fp32(2 * 3.1415926)."""
    c = torch.tensor(2 * 3.1415926, dtype=torch.float32).to(x.dtype)
    product = torch.bmm(w, x.unsqueeze(-1)).squeeze(-1)
    product2 = torch.bmm(wcos, (10 * torch.cos(c * x)).unsqueeze(-1)).squeeze(-1)
    return torch.mean(torch.sum((product - y) ** 2, 1) - torch.sum(product2, 1) + 10 * x.shape[1])


def confocal_psf(theta, roi):
    """point_spread_function_3d (DM/problems.py:899-932) in the dense [B, nx*ny*nz] tf.meshgrid form: theta = six [B]
    tensors (I0, x0, y0, z0, sigmaxy, sigmaz quantiles); tfd.Uniform(lo, hi).quantile(p) = lo + p (hi - lo)."""
    dt = theta[0].dtype
    lows = (0.5, 0.5, 0.5, 0.5, 2.0, 2.0)
    highs = (2.0, roi[0] - 1, roi[1] - 1, roi[2] - 1, 4.0, 4.0)
    X, Y, Z = torch.meshgrid(*[torch.linspace(0.0, float(n - 1), n, dtype=dt) for n in roi], indexing="xy")
    I0, x0, y0, z0, sxy, sz = (lo + t.reshape(-1, 1) * (hi - lo) for t, lo, hi in zip(theta, lows, highs))
    xk, yk, zk = X.reshape(1, -1), Y.reshape(1, -1), Z.reshape(1, -1)
    r2 = torch.sqrt(torch.tensor(2.0, dtype=dt))
    ex = -torch.erf((-0.5 - x0 + xk) / (r2 * sxy)) + torch.erf((0.5 - x0 + xk) / (r2 * sxy))
    ey = -torch.erf((-0.5 - y0 + yk) / (r2 * sxy)) + torch.erf((0.5 - y0 + yk) / (r2 * sxy))
    ez = -torch.erf((-0.5 - z0 + zk) / (r2 * sz)) + torch.erf((0.5 - z0 + zk) / (r2 * sz))
    return I0 * (ex * ey * ez) / 8.0


def confocal_f(x, sim, B, P, roi):
    """DM/problems.py:799-956 (inference=False): x and sim are [6P+1][B] (flat or 2-D; rows I, x0, y0, z0, sigmaxy,
    sigmaz of each point, then the background), in the dtype of x.
    f = mean_b sum_v (sum_p psf(x_p) + bg - l2_normalize(sum_p psf(sim_p) + bg_sim))^2."""
    x = x.reshape(6 * P + 1, B)
    sim = sim.reshape(6 * P + 1, B).to(x.dtype)
    y_pred = sum(confocal_psf(x[6 * p:6 * p + 6], roi) for p in range(P))
    y_sim = sum(confocal_psf(sim[6 * p:6 * p + 6], roi) for p in range(P))
    t = y_sim + sim[6 * P].reshape(B, 1)
    t = t * torch.rsqrt(torch.clamp_min(torch.sum(t * t, dim=1, keepdim=True), 1e-12))
    return torch.mean(torch.sum((y_pred + x[6 * P].reshape(B, 1) - t) ** 2, dim=1))
