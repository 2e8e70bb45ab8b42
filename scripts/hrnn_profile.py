"""Profiling driver (run under a profiler): a few l2o_hrnn_step calls on a state larger than L2 (16 tensors x 2M)."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from open_l2o_b200 import hierarchical_rnn as hr  # noqa: E402

dev = "cuda:0"
sizes = [2_000_000] * 16
big = [torch.zeros(sz, device=dev).requires_grad_(True) for sz in sizes]
opt = hr.HierarchicalRNN(random_seed=0, **hr.metarun_flags())
opt.apply_gradients(zip([torch.randn(sz, device=dev) * 0.1 for sz in sizes], big))
for _ in range(3):
    opt.step_flat()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(10):
    opt.step_flat()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / 10
print("hrnn step: %.3f ms for %d coords -> %.1f GB/s algorithmic (192 B/coord-step)" % (ms, opt.N, 192.0 * opt.N / ms / 1e6),
      "| lib", os.environ.get("L2O_LIB", "default"))
