"""Debug helper (not a test): prints tensor-core-engine error statistics against the oracle."""
import sys, torch
sys.path.insert(0, ".")
from oracle import l2o_oracle as orc
from tests.helpers import SPECS, make_handle, rel_err, arena_to_state
from tests.test_kernels_gpu import _run_prerecorded
from open_l2o_b200.engine import ENGINE_TC, ENGINE_FFMA

for name in ["dm_identity", "dm_logsign"]:
    for (n, T) in [(256, 1), (300, 2), (777, 20)]:
        try:
            r = _run_prerecorded(SPECS[name], n=n, T=T, seed=7, engine=ENGINE_TC)
        except Exception as e:
            print(name, n, T, "EXC", repr(e)[:300]); continue
        d = rel_err(r["dseq"], torch.stack(r["deltas"]))
        xs = rel_err(r["xg"], r["x_ref"])
        sf = r["sf"]
        st1 = arena_to_state(r["ckpt"][1 * sf * n:2 * sf * n].cpu(), SPECS[name].layers, n)
        e1 = [(rel_err(hg, hr), rel_err(cg, cr)) for (hg, cg), (hr, cr) in zip(st1, r["states"][1])]
        print(name, n, T, "delta", d, "x", xs, "state@1", e1)
        if d > 1e-3:
            print("  dseq[0,:8]", r["dseq"][0, :8].cpu().tolist()); print("  ref      ", r["deltas"][0][:8].tolist())
            print("  h1@1[0]", st1[0][0][0, :8].tolist()); print("  ref    ", r["states"][1][0][0][0, :8].tolist())
