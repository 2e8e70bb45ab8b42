"""Shared helpers for the parity tests: spec <-> handle construction, error metric."""
import math

import torch

from oracle import l2o_oracle as orc

REL_TOL = 1e-5  # north_star: "within 1e-5 relative fp32"

SPECS = {
    "dm_identity": orc.NetSpec(layers=(20, 20)),
    "dm_logsign": orc.NetSpec(layers=(20, 20), preprocess_name="LogAndSign", preprocess_options={"k": 5}, scale=0.01),
    "rnnprop": orc.NetSpec(layers=(20, 20), preprocess_name="fc", preprocess_options={"dim": 20}, scale=0.01,
                           tanh_output=True, rnnprop=True),
    "empty": orc.NetSpec(layers=()),
    "one": orc.NetSpec(layers=(1,)),
    "one_one": orc.NetSpec(layers=(1, 1)),
    "two_three": orc.NetSpec(layers=(2, 3)),
}


def make_handle(spec):
    from open_l2o_b200.engine import NetHandle
    return NetHandle(layers=spec.layers, preprocess_name=spec.preprocess_name,
                     preprocess_options=spec.preprocess_options, scale=spec.scale, tanh_output=spec.tanh_output,
                     n_in=spec.n_in)


def rel_err(a, b):
    """max-norm relative error of a against reference b."""
    a = torch.as_tensor(a).detach().double().cpu().reshape(-1)
    b = torch.as_tensor(b).detach().double().cpu().reshape(-1)
    den = max(float(b.abs().max()), 1e-30)
    return float((a - b).abs().max()) / den


def state_to_arena(state, n):
    """tuple over layers of (h, c) [n, H] -> flat arena (include/l2o_b200.h layout)."""
    parts = []
    for h, c in state:
        parts += [h.reshape(-1), c.reshape(-1)]
    if not parts:
        return torch.zeros(1)
    return torch.cat(parts).contiguous()


def arena_to_state(arena, layers, n):
    out, off = [], 0
    for h in layers:
        hh = arena[off:off + n * h].view(n, h)
        cc = arena[off + n * h:off + 2 * n * h].view(n, h)
        out.append((hh, cc))
        off += 2 * n * h
    return tuple(out)


def random_state(spec, n, gen, amp=0.5, dtype=torch.float32):
    return tuple(((torch.rand(n, h, generator=gen, dtype=torch.float64) * 2 - 1).mul(amp).to(dtype),
                  (torch.rand(n, h, generator=gen, dtype=torch.float64) * 2 - 1).mul(amp).to(dtype))
                 for h in spec.layers)


def wild_gradients(n, gen):
    """Gradients spanning many magnitudes, with exact zeros and both signs (LogAndSign edge cases)."""
    e = torch.randint(-12, 4, (n,), generator=gen).double()
    g = torch.randn(n, generator=gen, dtype=torch.float64) * (10.0 ** e)
    g[::17] = 0.0
    g[1::29] = 1.0
    g[2::31] = -1e-3
    return g.float()


HRNN_CONVNET = ((3, 32, 32), 10, [(3, 3, 32), (5, 5, 32)])   # optimizee of BASELINE config #4: 354,218 coordinates
HRNN_TILE = 128   # coordinates per tile of the HierarchicalRNN coordinate kernels (l2o_hrnn.cu kBlock)


def hrnn_ragged_shapes(n_small=300, big=20011, seed=0):
    """n_small tensors at the sizes around a 128-coordinate tile (a lone coordinate, one short, exactly full, one over,
    two tiles, two tiles plus one) in a seeded order, plus one tensor of 157 tiles in the middle.  More than 16
    tensors make the HierarchicalRNN tensor_kernel's strided loops wrap."""
    sizes = [1, 37, 127, 128, 129, 200, 255, 257]
    perm = torch.randperm(n_small, generator=torch.Generator().manual_seed(seed))
    shapes = [(sizes[int(k) % len(sizes)],) for k in perm]
    shapes.insert(n_small // 2, (big,))
    return shapes


def hrnn_generic_theta(seed, dtype=torch.float32):
    """HierarchicalRNN weights with no symmetry left to hide an indexing slip.  The reference's initial distribution
    (oracle/hrnn_oracle.init_theta) zeroes whole paths and repeats constants, so a kernel that drops a term or permutes
    entries of a constant vector computes the same numbers there.  Starting from init_theta(seed), every such block is
    redrawn at about init scale:
      - learning_rate_weights N(0, 0.3), and learning_rate_bias = -(init vector . Wl) + N(0, 0.05): lr_change =
        h' . Wl + bl starts near zero and drifts by O(0.1 - 0.4) as h' moves away from the shared init vector, with a
        sign that differs between coordinates for suitable seeds (seed 5: -0.3 .. +0.2 within 4 steps, checked in
        tests/test_hrnn_oracle.py).  So the log-lr path is live, and a log-lr at -33 is pushed below the clip for
        some coordinates and stays inside it for others;
      - every gate bias 2.2 + N(0, 0.5): distinct entries, so a permuted or misplaced gate-bias row shows;
      - candidate biases and the Param / Global / Layer1 affine biases N(0, 0.3): they are zero at init;
      - scl / inp decay biases and the param stepsize offset shifted by N(0, 0.3);
      - the lr-momentum logit at 2.0 + N(0, 0.3) instead of 3.2: (1 - lrm) grows from 0.04 to about 0.12, so the
        step log-lr (and its clip) weighs more in the new log-lr.
    The affine matrices, readouts, GradsToDelta and init vectors are already distinct random draws and are kept."""
    from oracle import hrnn_oracle as H
    base = H.init_theta(seed, dtype=torch.float64)
    g = torch.Generator().manual_seed(1000 + int(seed))
    P = H.unpack_theta(base)
    out = []
    for name, shape in H.theta_spec():
        v = P[name].reshape(-1).clone()
        n = v.numel()
        noise = lambda s: torch.randn(n, generator=g, dtype=torch.float64) * s
        if name == "learning_rate_weights":
            v = noise(0.3)
            wl = v
        elif name == "learning_rate_bias":   # centres lr_change at the initial hidden state (see the docstring)
            v = -(P["Level0_RNN/init_vector"].reshape(-1) @ wl).reshape(1) + noise(0.05)
        elif name.endswith("gates/Affine/Bias"):
            v = 2.2 + noise(0.5)
        elif name.endswith("Bias"):   # candidate and affine biases (the gate biases are matched above)
            v = noise(0.3)
        elif name in ("scl_decay_bias", "inp_decay_bias") or name.endswith("param_stepsize_offset"):
            v = v + noise(0.3)
        elif name.endswith("learning_rate_momentum_logit"):
            v = 2.0 + noise(0.3)
        out.append(v)
    return torch.cat(out).to(dtype)


def assert_theta_close(theta_gpu, trainer, tag=None, tol=REL_TOL, tol_all=5e-5):
    """theta after TF-Adam against the oracle trainer.  Adam's update is ~ lr * sign(g) in its first steps, so entries
    whose meta-gradient sits at round-off level (|g| <= 1e-5 max|g|) may legitimately differ by a fraction of lr; every
    other entry must agree to `tol` (max-norm relative), and all entries to `tol_all`."""
    th = torch.as_tensor(theta_gpu).detach().cpu()
    g = trainer.last_grad.detach().abs()
    big = g > 1e-5 * float(g.max())
    assert rel_err(th[big], trainer.theta[big]) <= tol, (tag, rel_err(th[big], trainer.theta[big]))
    assert rel_err(th, trainer.theta) <= tol_all, (tag, rel_err(th, trainer.theta))
