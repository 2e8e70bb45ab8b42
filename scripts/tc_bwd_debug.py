"""Debug helper: tensor-core BPTT vs FFMA BPTT, block-wise error report."""
import sys, torch
sys.path.insert(0, ".")
from oracle import l2o_oracle as orc
from tests.helpers import SPECS, make_handle, rel_err
from open_l2o_b200.engine import ENGINE_TC, ENGINE_FFMA
DEV = "cuda:0"
spec = SPECS["dm_identity"]
for (n, T) in [(128, 1), (128, 2), (300, 3), (19021, 4)]:
    gen = torch.Generator().manual_seed(21)
    theta = orc.init_theta(spec, seed=0, out_gain=0.05).to(DEV)
    g_rec = (torch.randn(T + 1, n, generator=gen) * 0.5).to(DEV)
    h = make_handle(spec); h.set_engine(ENGINE_FFMA)
    sf = h.state_floats
    arena = h.new_state(n, DEV)
    ckpt = torch.zeros((T + 1) * sf * n, device=DEV)
    h.unroll_fwd(theta, n, T, arena, in_seq=g_rec[:T].contiguous(), ckpt=ckpt)
    outs = {}
    for eng in (ENGINE_FFMA, ENGINE_TC):
        h.set_engine(eng)
        d = torch.zeros(h.n_theta, dtype=torch.float64, device=DEV)
        try:
            h.unroll_bwd(theta, n, T, g_rec[:T].contiguous(), ckpt, d, g_rec=g_rec)
            torch.cuda.synchronize()
        except Exception as e:
            print("EXC", eng, repr(e)[:300]); raise
        outs[eng] = d.cpu()
    a, b = outs[ENGINE_TC], outs[ENGINE_FFMA]
    print(f"n={n} T={T} total rel err {rel_err(a, b):.3e}")
    off = 0
    for mod, var, shp in spec.shapes():
        k = 1
        for s_ in shp: k *= s_
        ea, eb = a[off:off + k], b[off:off + k]
        print(f"   {mod}/{var:8s} {str(shp):10s} rel {rel_err(ea, eb):.3e}  |ref|max {float(eb.abs().max()):.3e}")
        if rel_err(ea, eb) > 1e-3 and len(shp) == 2:
            A, B = ea.reshape(shp), eb.reshape(shp)
            rows = ((A - B).abs().max(dim=1).values / (B.abs().max() + 1e-30))
            print("      worst rows:", [(int(r), float(rows[r])) for r in rows.argsort(descending=True)[:6]])
            print("      tc row0[:8] ", A[0, :8].tolist()); print("      ref row0[:8]", B[0, :8].tolist())
        off += k
