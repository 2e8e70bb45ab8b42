"""The chunked fp64 reference of tests/dm_scale_reference.py against one unchunked oracle unroll, without a GPU.

n = 300 in chunks of 64 leaves a short last chunk (44), so a chunk dropped, overlapped or given its own fscale shows in
every output.  A random initial state and, for RNNProp, random m, v and a later step0 make every chunk's slices of the
inputs matter."""
import pytest
import torch

from oracle import l2o_oracle as orc
from tests.dm_scale_reference import chunked_meta_grad
from tests.helpers import SPECS, random_state, rel_err

N, T, CHUNK = 300, 6, 64
TOL = 1e-12


def _problem(kind, gen):
    if kind == "rastrigin_sep":
        a, b, x0 = (torch.randn(N, generator=gen, dtype=torch.float64) for _ in range(3))
        return orc.FusedProblem(kind, a, b, alpha=10.0, fscale=1.0 / N), x0
    a = torch.rand(N, generator=gen, dtype=torch.float64) + 0.5
    b = torch.rand(N, generator=gen, dtype=torch.float64)
    return orc.FusedProblem(kind, a, b, fscale=1.0 / N), torch.randn(N, generator=gen, dtype=torch.float64) * 0.01


@pytest.mark.parametrize("kind", ["rastrigin_sep", "quadratic_diag"])
@pytest.mark.parametrize("name", ["dm_identity", "dm_logsign", "rnnprop"])
def test_chunked_reference_matches_one_unroll(name, kind):
    spec = SPECS[name]
    gen = torch.Generator().manual_seed(11)
    theta = orc.init_theta(spec, seed=3, out_gain=0.3, dtype=torch.float64)
    prob, x0 = _problem(kind, gen)
    state0 = random_state(spec, N, gen, dtype=torch.float64)
    kw = {}
    if spec.rnnprop:
        mv0 = (torch.randn(N, generator=gen, dtype=torch.float64) * 1e-3,
               torch.rand(N, generator=gen, dtype=torch.float64) * 1e-6)
        kw = dict(mv0=mv0, step0=4)
    g, res = orc.meta_grad(spec, theta, x0, state0, None, T, grad_of=prob.f_and_g, **kw)
    out = chunked_meta_grad(spec, theta, prob, x0, T, torch.float64, state0=state0, chunk=CHUNK, **kw)

    assert rel_err(out.dtheta, g) <= TOL
    assert rel_err(out.fx, res.fx) <= TOL
    assert rel_err(out.x, res.x_final) <= TOL
    for (h, c), (hr, cr) in zip(out.state, res.state_final):
        assert rel_err(h, hr) <= TOL and rel_err(c, cr) <= TOL
    g_rows = torch.stack(res.grads + [prob.f_and_g(res.x_final)[1]])
    assert rel_err(out.g_rec, g_rows) <= TOL
    if spec.rnnprop:
        assert rel_err(out.mv[0], res.mv_final[0]) <= TOL and rel_err(out.mv[1], res.mv_final[1]) <= TOL
    else:
        assert out.mv is None


def test_chunks_cover_every_coordinate():
    """A chunk that does not divide n, a chunk of one coordinate and a chunk larger than n give the same result."""
    spec = SPECS["dm_identity"]
    gen = torch.Generator().manual_seed(12)
    theta = orc.init_theta(spec, seed=4, out_gain=0.3, dtype=torch.float64)
    prob, x0 = _problem("rastrigin_sep", gen)
    ref = chunked_meta_grad(spec, theta, prob, x0, 3, torch.float64, chunk=N + 1)
    for chunk in (1, 7, N - 1):
        out = chunked_meta_grad(spec, theta, prob, x0, 3, torch.float64, chunk=chunk)
        assert rel_err(out.dtheta, ref.dtheta) <= TOL and rel_err(out.fx, ref.fx) <= TOL, chunk
        assert rel_err(out.x, ref.x) <= TOL and rel_err(out.g_rec, ref.g_rec) <= TOL, chunk
