"""CPU-only: the flat coordinate arena MetaOptimizer lays out (meta.plan_arena) and the initial theta of the optimizer
nets (networks.factory), which the meta-optimizer's results depend on bit for bit."""
import hashlib

import numpy as np
import pytest

from open_l2o_b200 import meta, networks


def _plan(shapes, config, net_assignments=None):
    variables = [dict(name=name, shape=shape) for name, shape in shapes]
    config = {k: dict(v, net_options=dict(v["net_options"], device="cpu")) for k, v in config.items()}
    nets, keys, subsets = meta._make_nets(variables, config, net_assignments)
    slices, N, runs = meta.plan_arena(variables, subsets, keys, nets)
    for r in runs:
        assert r.net is nets[r.key]
    return [(s.start, s.stop) for s in slices], N, [(r.key, r.off, r.n) for r in runs]


CW1 = {"net": "CoordinateWiseDeepLSTM", "net_options": {"layers": (1,)}}


def test_one_net_over_all_variables():
    assert _plan([("a", [3, 4]), ("b", [5]), ("c", [])], {"net": CW1}) == (
        [(0, 12), (12, 17), (17, 18)], 18, [("net", 0, 18)])


@pytest.mark.parametrize("net_assignments,config,runs", [
    (None, {"net": CW1}, [("net", 0, 2)]),
    ([("net", ["x_0", "x_1"])], {"net": CW1}, [("net", 0, 2)]),
    ([("net1", ["x_0"]), ("net2", ["x_0"])], {"net1": CW1, "net2": CW1}, [("net1", 0, 1), ("net2", 0, 1)]),
])
def test_multi_optimizer_assignments(net_assignments, config, runs):
    """The three assignments of test_meta_gpu.test_multi_optimizer (two scalars x_0, x_1); in the last, two nets serve
    x_0 and x_1 is served by none."""
    assert _plan([("x_0", []), ("x_1", [])], config, net_assignments) == ([(0, 1), (1, 2)], 2, runs)


def test_kernel_net_gets_one_run_per_variable():
    """The two-filter-bank config of test_dense_engine_gpu: the filter banks are adjacent in the arena but are served
    by a per-variable KernelDeepLSTM, so each is its own run; the biases merge into one coordinate-wise run."""
    config = {"conv": {"net": "KernelDeepLSTM", "net_options": {"kernel_shape": [3, 3], "layers": (32, 32)}},
              "cw": {"net": "CoordinateWiseDeepLSTM", "net_options": {"layers": (20, 20)}}}
    shapes = [("c1/w", [3, 3, 4, 40]), ("c1/b", [40]), ("c2/w", [3, 3, 40, 8]), ("c2/b", [8])]
    assert _plan(shapes, config, [("conv", ["c1/w", "c2/w"]), ("cw", ["c1/b", "c2/b"])]) == (
        [(0, 1440), (4320, 4360), (1440, 4320), (4360, 4368)], 4368,
        [("conv", 0, 1440), ("conv", 1440, 2880), ("cw", 4320, 48)])


def test_subset_not_contiguous_in_creation_order():
    """a, c are placed first (the first subset names them), then b; d belongs to no subset and goes last.  The second
    subset (b, c) is not contiguous in the arena and is cut into two runs."""
    shapes = [("a", [2]), ("b", [3]), ("c", [2, 2]), ("d", [5])]
    assert _plan(shapes, {"k0": CW1, "k1": CW1}, [("k0", ["a", "c"]), ("k1", ["b", "c"])]) == (
        [(0, 2), (6, 9), (2, 6), (9, 14)], 14, [("k0", 0, 6), ("k1", 6, 3), ("k1", 2, 4)])


# SHA-256 of the initial theta's float32 bytes, recorded on CPU at the commit that introduced this file
THETA_SHA256 = {
    "cw_empty": (("CoordinateWiseDeepLSTM", {"layers": ()}),
                 "2c2731fc2f0a489a99bb647dcba535eb1ea238d52afce4984ef5bd119d1b1811"),
    "cw_1_1": (("CoordinateWiseDeepLSTM", {"layers": (1, 1), "seed": 3}),
               "2375638b9daf1cc20e1a074b4c6bf108718328758bcf1bcf52e15593f4877389"),
    "cw_20_20_logsign": (("CoordinateWiseDeepLSTM", {"layers": (20, 20), "preprocess_name": "LogAndSign",
                                                     "preprocess_options": {"k": 5}, "scale": 0.01}),
                         "c8d5b1c4da4d61848798acd034cf11d3a6ea90c98aebcf3d646e1908a439d8f9"),
    "cw_zeros": (("CoordinateWiseDeepLSTM", {"layers": (2, 3), "initializer": "zeros"}),
                 "1fe2373734955e60c172999142934b52e69ba7ab9039b3c18ea54082ba32afcd"),
    "cw_dict": (("CoordinateWiseDeepLSTM", {"layers": (2, 3), "initializer": {
        "lstm_1": {"b_gates": "ones"}, "linear": {"b": np.array([0.25], np.float32)}}}),
                "5cc21b5927727870877ebae282a8500558ecbed5bb2561dc2aa7e3e1fcbc0699"),
    "rnnprop_fc20_tanh": (("RNNprop", {"layers": (20, 20), "preprocess_name": "fc", "preprocess_options": {"dim": 20},
                                       "scale": 0.01, "tanh_output": True}),
                          "45d801b0de7868378dee329a68dd71e44c14103a6e52d4263ccc6463f02d74b7"),
    "kernel_32_32_logsign": (("KernelDeepLSTM", {"kernel_shape": [3, 3], "layers": (32, 32),
                                                 "preprocess_name": "LogAndSign", "preprocess_options": {"k": 5},
                                                 "scale": 0.1}),
                             "922bc53fcdd4edf8dacc23f07781ec8ab83172832e0ac5060b0e97d33d65b10f"),
}


@pytest.mark.parametrize("case", sorted(THETA_SHA256))
def test_factory_theta_is_unchanged(case):
    (net, opts), digest = THETA_SHA256[case]
    theta = networks.factory(net, dict(opts, device="cpu")).theta
    assert hashlib.sha256(theta.numpy().tobytes()).hexdigest() == digest
