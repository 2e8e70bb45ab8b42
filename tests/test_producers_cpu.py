"""CPU-only: which arenas and shapes each gradient producer (producers.py) takes, on the variables, arena slices and
constants MetaOptimizer hands it, and the in-kernel kinds of the FusedSpecs the problems attach."""
import pytest
import torch

from open_l2o_b200 import engine, meta, problems, util
from tests.mnist_fixture import write_mnist


def _layout(build, reverse=False):
    """What _Program passes to ``accepts``: the variables and constants build() creates, and the slices plan_arena lays
    out for one net over the variables in creation order, or in reverse (net_assignments naming them backwards)."""
    variables, constants = meta._get_variables(build, torch.Generator().manual_seed(0), "cpu")
    order = list(range(len(variables)))[::-1 if reverse else 1]
    slices, _, _ = meta.plan_arena(variables, [order], ["cw"], {"cw": None})
    return variables, slices, constants


def _renamed(layout, j=0):
    variables, slices, constants = layout
    return [dict(v, name=v["name"] + "_other") if i == j else v for i, v in enumerate(variables)], slices, constants


@pytest.fixture(scope="module")
def data_dir(tmp_path_factory):
    d = str(tmp_path_factory.mktemp("mnist"))
    write_mnist(d)
    return d


@pytest.mark.parametrize("build", [problems.lasso(batch_size=4, num_dims=3),
                                   problems.lasso_fixed(torch.rand(4, 5, 3), torch.rand(4, 5, 1))],
                         ids=["lasso", "lasso_fixed"])
def test_lasso_takes_its_one_variable(build):
    p = build.producer
    assert p.kind == "lasso_batch"
    layout = _layout(build)
    assert p.accepts(*layout)
    assert not p.accepts(*_renamed(layout))
    variables, slices, constants = layout
    two = variables + [dict(variables[0], name="x2")]
    assert not p.accepts(two, slices + [slice(slices[0].stop, 2 * slices[0].stop)], constants)


def test_mlp_xent_takes_its_layers_in_any_arena_order():
    build = problems.mlp(layers=(3, 4), in_dim=5, batch_size=2)
    p = build.producer
    assert p.kind == "mlp_xent" and p.n_layers == 3
    assert p.accepts(*_layout(build))
    assert p.accepts(*_layout(build, reverse=True))   # it reads and writes through each variable's view
    assert not p.accepts(*_renamed(_layout(build), 2))
    assert not problems.mlp(layers=(3,), in_dim=5, batch_size=2).producer.accepts(*_layout(build))


def test_confocal_takes_its_rows_within_the_shared_memory_limit():
    build = problems.confocal_microscopy_3d(batch_size=3, num_points=2, ROI=(5, 6, 7))
    p = build.producer
    assert p.kind == "confocal_psf" and p.num_points == 2 and p.roi == (5, 6, 7)
    layout = _layout(build)
    assert p.accepts(*layout)
    assert not p.accepts(*_layout(build, reverse=True))
    assert not p.accepts(*_renamed(layout, 4))
    variables, slices, constants = layout
    assert not p.accepts(variables, slices, constants[::-1])
    for P, roi, fits in [(5, (64, 64, 64), False), (1, (38, 38, 38), False), (48, (32, 32, 32), False),
                         (1, (1 << 20, 1, 1), False), (47, (32, 32, 32), True), (5, (28, 28, 28), True)]:
        assert engine.confocal_fits(P, roi) == fits
        build = problems.confocal_microscopy_3d(batch_size=1, num_points=P, ROI=roi)
        assert build.producer.accepts(*_layout(build)) == fits, (P, roi)


def test_mnist_mlp_takes_the_kernels_shapes_in_creation_order(data_dir):
    for layers, fits in [((20,), True), ((64,) * 4, True), ((65,), False), ((64,) * 5, False), ((1, 64, 3), True)]:
        build = problems.mnist(layers, batch_size=4, data_dir=data_dir)
        assert build.producer.kind == "mnist_mlp"
        assert build.producer.accepts(*_layout(build)) == fits, layers
    build = problems.mnist((20,), data_dir=data_dir)
    layout = _layout(build)
    assert build.producer.accepts(*layout)
    assert not build.producer.accepts(*_layout(build, reverse=True))
    assert not build.producer.accepts(*_renamed(layout, 1))
    for batch, fits in [(1, True), (1024, True), (1025, False)]:
        assert problems.mnist((20,), batch_size=batch, data_dir=data_dir).producer.accepts(*layout) == fits, batch


def test_mnist_conv_takes_batch_norm_and_the_kernels_batches_in_creation_order(data_dir):
    build = problems.mnist_conv(batch_size=4, data_dir=data_dir)
    p = build.producer
    assert p.kind == "mnist_conv"
    layout = _layout(build)
    assert p.accepts(*layout)
    assert not p.accepts(*_layout(build, reverse=True))
    assert not p.accepts(*_renamed(layout, 5))
    assert not problems.mnist_conv(batch_norm=False, batch_size=4, data_dir=data_dir).producer.accepts(*layout)
    for batch, fits in [(1, True), (1024, True), (1025, False)]:
        assert problems.mnist_conv(batch_size=batch, data_dir=data_dir).producer.accepts(*layout) == fits, batch


def test_fused_specs_are_in_kernel_kinds(data_dir):
    names = ["simple", "quadratic", "rastrigin", "lasso", "confocal_microscopy_3d", "square_cos", "mnist", "mnist_relu",
             "mnist_deeper", "mnist_conv", "rastrigin_separable", "mlp"]
    builds = [util.get_config(n, data_dir=data_dir)[0] for n in names]
    builds += [problems.quadratic(batch_size=256, num_dims=64), problems.quadratic_diag(),
               problems.rastrigin_separable(num_dims=10)]
    specs = [b.fused for b in builds if getattr(b, "fused", None) is not None]
    assert sorted(s.kind for s in specs) == ["quadratic_batch", "quadratic_diag", "rastrigin_sep", "rastrigin_sep"]
    assert all(s.kind in engine.OPT_KINDS for s in specs)
    assert not any(hasattr(b, "fused") and hasattr(b, "producer") for b in builds)
