"""Synthetic optimizees (the callers that feed the hot path).  Each ``problem()`` returns a zero-arg
``build()`` that creates its tensors through ``get_variable`` and returns a scalar loss, exactly like
DM/problems.py; gradients come from torch autograd on the device (the "external-gradient" regime) unless
the builder carries a ``fused`` spec, in which case the unroll kernel evaluates the separable gradient
in-kernel (the "fused" regime), or a ``producer`` (producers.py) that makes f and df/dx in one call."""
from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np
import torch

from . import producers
from .variables import (constant_initializer, get_variable, ones_initializer, random_normal_initializer,
                        random_uniform_initializer)


@dataclass
class FusedSpec:
    """An optimizee the unroll kernel evaluates in-kernel: one launch for all T steps of its one variable."""
    kind: str        # a key of engine.OPT_KINDS: "rastrigin_sep" | "quadratic_diag" | "quadratic_batch"
    a: str           # constant names
    b: str
    alpha: float = 10.0
    fscale: float = 1.0
    group: int = 0   # "quadratic_batch": coordinates per dense group


def simple():
    """f(x) = x^2 (DM/problems.py:41-53)."""
    def build():
        x = get_variable("x", shape=[], initializer=ones_initializer())
        return torch.square(x)
    return build


def simple_multi_optimizer(num_dims=2):
    """DM/problems.py:56-70."""
    def build():
        coords = [get_variable("x_{}".format(i), shape=[], initializer=ones_initializer()) for i in range(num_dims)]
        x = torch.stack([c.reshape(()) for c in coords])
        return torch.sum(torch.square(x))
    return build


def quadratic(batch_size=128, num_dims=10, stddev=0.01):
    """f(x) = mean_b ||W_b x_b - y_b||^2 (DM/problems.py:73-101)."""
    def build():
        x = get_variable("x", shape=[batch_size, num_dims], initializer=random_normal_initializer(stddev=stddev))
        w = get_variable("w", shape=[batch_size, num_dims, num_dims], initializer=random_uniform_initializer(),
                         trainable=False)
        y = get_variable("y", shape=[batch_size, num_dims], initializer=random_uniform_initializer(), trainable=False)
        product = torch.bmm(w, x.unsqueeze(-1)).squeeze(-1)
        return torch.mean(torch.sum((product - y) ** 2, dim=1))
    # dense W_b x_b evaluated in-kernel: the whole unroll is one launch (SURVEY.md 8(f) row 4).  Only where the
    # kernels are throughput-bound: at BASELINE config #1's 1,280 coordinates a thread walks the whole LSTM serially
    # either way, and the graph-captured step-at-a-time path is measured faster (1.29 vs 1.63 ms per unroll).
    if num_dims <= 128 and batch_size * num_dims >= 16384:
        build.fused = FusedSpec("quadratic_batch", "w", "y", fscale=1.0 / batch_size, group=num_dims)
    return build


def _lasso_loss(x, w, y, l):
    product = torch.bmm(w, x.unsqueeze(-1))
    left = 0.5 * torch.sum((product - y) ** 2, dim=1)
    other = l * torch.sum(torch.abs(x), dim=1, keepdim=True)
    return torch.mean(left + other)


def lasso(batch_size=128, num_dims=10, stddev=0.01, l=0.005):
    """DM/problems.py:103-135."""
    def build():
        x = get_variable("x", shape=[batch_size, num_dims], initializer=random_normal_initializer(stddev=stddev))
        w = get_variable("w", shape=[batch_size, num_dims, num_dims], initializer=random_uniform_initializer(),
                         trainable=False)
        y = get_variable("y", shape=[batch_size, num_dims, 1], initializer=random_uniform_initializer(),
                         trainable=False)
        return _lasso_loss(x, w, y, l)
    build.producer = producers.Lasso("x", "w", "y", alpha=float(l))
    return build


def lasso_fixed(data_A, data_b, stddev=0.01, l=0.005):
    """DM/problems.py:137-175: A [B, m, n], b [B, m, 1]."""
    a = torch.as_tensor(data_A, dtype=torch.float32)
    b = torch.as_tensor(data_b, dtype=torch.float32)

    def build():
        x = get_variable("x", shape=[a.shape[0], a.shape[2]], initializer=random_normal_initializer(stddev=stddev))
        w = get_variable("w", shape=list(a.shape), initializer=constant_initializer(a), trainable=False)
        y = get_variable("y", shape=list(b.shape), initializer=constant_initializer(b), trainable=False)
        return _lasso_loss(x, w, y, l)
    build.producer = producers.Lasso("x", "w", "y", alpha=float(l))
    return build


def rastrigin(batch_size=128, num_dims=10, alpha=10, stddev=1):
    """Dense Rastrigin family (DM/problems.py:177-213)."""
    def build():
        x = get_variable("x", shape=[batch_size, num_dims, 1], initializer=random_normal_initializer(stddev=stddev))
        A = get_variable("A", shape=[batch_size, num_dims, num_dims],
                         initializer=random_normal_initializer(stddev=stddev), trainable=False)
        B = get_variable("B", shape=[batch_size, num_dims, 1], initializer=random_normal_initializer(stddev=stddev),
                         trainable=False)
        Cc = get_variable("C", shape=[batch_size, num_dims, 1], initializer=random_normal_initializer(stddev=stddev),
                          trainable=False)
        product = torch.bmm(A, x)
        ras_norm2 = torch.sum((product - B) ** 2, dim=(-2, -1))
        cq = torch.bmm(Cc.transpose(1, 2), torch.cos(2 * math.pi * x)).reshape(-1)
        return torch.mean(0.5 * ras_norm2 - alpha * cq + alpha * num_dims)
    return build


def rastrigin_separable(num_dims=1000000, alpha=10.0, stddev=1.0, normalize=True, shard=None):
    """The A = I member of DM/problems.py:177-213 with batch 1 - the only member that exists at d = 1e6
    (a dense A would be 4 TB).  f = fscale * sum_i (0.5 (x_i-b_i)^2 - alpha c_i cos(2 pi x_i) + alpha).

    ``shard=(lo, hi)``: this rank's contiguous slice of the ``num_dims`` coordinates (SURVEY.md 8(e), strong scaling of
    BASELINE config #5).  The initializers draw the full tensors and keep [lo, hi), so the union over the ranks is
    exactly the single-GPU problem for the same seed; ``fscale`` stays 1/num_dims (the GLOBAL count) and the ranks'
    partial f values are summed by the meta-step's all-reduce."""
    fscale = 1.0 / num_dims if normalize else 1.0
    two_pi = 6.2831855  # fp32(2 pi), the constant the kernel uses
    lo, hi = shard if shard is not None else (0, num_dims)
    n_loc = hi - lo

    def sliced(init):
        if shard is None:
            return init
        return lambda shape, gen: init((num_dims,), gen)[lo:hi].clone()

    def build():
        normal = sliced(random_normal_initializer(stddev=stddev))
        x = get_variable("x", shape=[n_loc], initializer=normal)
        b = get_variable("b", shape=[n_loc], initializer=normal, trainable=False)
        c = get_variable("c", shape=[n_loc], initializer=normal, trainable=False)
        fi = 0.5 * (x - b) ** 2 - alpha * c * torch.cos(two_pi * x) + alpha
        return fscale * torch.sum(fi)
    build.fused = FusedSpec("rastrigin_sep", "b", "c", alpha=float(alpha), fscale=fscale)
    return build


def quadratic_diag(num_dims=1280, stddev=0.01, normalize=True):
    """DM/problems.py:73-101 with diagonal W: f = fscale * sum_i (w_i x_i - y_i)^2."""
    fscale = 1.0 / num_dims if normalize else 1.0

    def build():
        x = get_variable("x", shape=[num_dims], initializer=random_normal_initializer(stddev=stddev))
        w = get_variable("w", shape=[num_dims], initializer=random_uniform_initializer(0.5, 1.5), trainable=False)
        y = get_variable("y", shape=[num_dims], initializer=random_uniform_initializer(), trainable=False)
        return fscale * torch.sum((w * x - y) ** 2)
    build.fused = FusedSpec("quadratic_diag", "w", "y", fscale=fscale)
    return build


def mlp(layers=(100,), in_dim=784, n_classes=10, batch_size=128, activation="sigmoid", init_stddev=0.01):
    """Sigmoid/ReLU MLP with softmax cross-entropy on a fixed synthetic batch (shape of DM/problems.py:254-288;
    the data is synthetic because MNIST cannot be downloaded here)."""
    act = {"sigmoid": torch.sigmoid, "relu": torch.relu}[activation]

    def build():
        data = get_variable("data", shape=[batch_size, in_dim], initializer=random_uniform_initializer(),
                            trainable=False)
        labels = get_variable("labels", shape=[batch_size],
                              initializer=lambda shape, gen: torch.randint(0, n_classes, shape, generator=gen).float(),
                              trainable=False)
        h, k = data, in_dim
        for i, width in enumerate(tuple(layers) + (n_classes,)):
            w = get_variable("mlp/linear_{}/w".format(i), shape=[k, width],
                             initializer=random_normal_initializer(stddev=init_stddev))
            b = get_variable("mlp/linear_{}/b".format(i), shape=[width],
                             initializer=random_normal_initializer(stddev=init_stddev))
            h = h @ w + b
            if i < len(layers):
                h = act(h)
            k = width
        return torch.nn.functional.cross_entropy(h, labels.long())
    # analytic producer: f and df/dx without the autograd engine (mlp_value_and_grad below)
    build.producer = producers.MlpXent(activation, n_layers=len(tuple(layers)) + 1)
    return build


def mlp_value_and_grad(params, data, labels, activation, grads_out):
    """Loss and gradient of the `mlp` optimizee written out by hand (the optimizee step feeding the hot path, SURVEY.md
    8(f) row 4): the forward pass keeps the activations, the backward pass writes every dW = h^T dz / db = sum(dz)
    STRAIGHT INTO the caller's gradient views - about a dozen launches (3 GEMMs per layer, fused elementwise) instead of
    the ~30 of the autograd engine with its per-variable copies.  params / grads_out: [w0, b0, w1, b1, ...]."""
    n_layers = len(params) // 2
    hs, h = [data], data
    for i in range(n_layers):
        z = torch.addmm(params[2 * i + 1], h, params[2 * i])
        if i < n_layers - 1:
            h = torch.sigmoid(z) if activation == "sigmoid" else torch.relu(z)
            hs.append(h)
    lab = labels.long()
    logp = torch.log_softmax(z, dim=1)
    loss = -logp.gather(1, lab.unsqueeze(1)).mean()
    dz = torch.exp(logp)
    dz.scatter_add_(1, lab.unsqueeze(1), torch.full((lab.numel(), 1), -1.0, device=dz.device, dtype=dz.dtype))
    dz.mul_(1.0 / lab.numel())
    for i in reversed(range(n_layers)):
        torch.mm(hs[i].t(), dz, out=grads_out[2 * i])
        torch.sum(dz, dim=0, out=grads_out[2 * i + 1])
        if i > 0:
            dh = dz @ params[2 * i].t()
            dz = dh * hs[i] * (1.0 - hs[i]) if activation == "sigmoid" else dh * (hs[i] > 0).to(dh.dtype)
    return loss


def mnist(layers, activation="sigmoid", batch_size=128, mode="train", data_dir="MNIST-data"):
    """MNIST classification with a multi-layer perceptron (DM/problems.py:254-288): Sonnet's ``mlp/linear_{i}/w|b``,
    both N(0, 0.01) (``_nn_initializers``), sigmoid or ReLU between layers, the mean sparse softmax cross entropy of a
    fresh batch of ``batch_size`` examples drawn uniformly with replacement at EVERY evaluation.  The data is read from
    ``data_dir`` (mnist_data; never downloaded) when the problem is made, and is not an optimizee variable: a reset
    re-initialises the weights only, as the reference's ``tf.constant`` images are untouched by its reset."""
    from . import mnist_data
    if activation not in ("sigmoid", "relu"):
        raise ValueError("{} activation not supported".format(activation))
    if mode not in ("train", "validation", "test"):
        raise ValueError("{} is not an MNIST split".format(mode))
    layers = tuple(int(w) for w in layers)
    num_examples = mnist_data.load_mnist(data_dir)[mode].num_examples
    act = {"sigmoid": torch.sigmoid, "relu": torch.relu}[activation]

    def build():
        params, k = [], 784
        for i, width in enumerate(layers + (10,)):
            params.append(get_variable("mlp/linear_{}/w".format(i), shape=[k, width],
                                       initializer=random_normal_initializer(stddev=0.01)))
            params.append(get_variable("mlp/linear_{}/b".format(i), shape=[width],
                                       initializer=random_normal_initializer(stddev=0.01)))
            k = width
        images, labels = mnist_data.device_split(data_dir, mode, params[0].device)
        idx = torch.randint(0, num_examples, (batch_size,), device=images.device)
        h = images.index_select(0, idx).float() * float(mnist_data.SCALE)
        for i in range(len(params) // 2):
            h = h @ params[2 * i] + params[2 * i + 1]
            if i < len(layers):
                h = act(h)
        return torch.nn.functional.cross_entropy(h, labels.index_select(0, idx).long())
    build.producer = producers.MnistMlp(batch_size=int(batch_size), mode=mode, data_dir=data_dir, layers=layers,
                                        activation=activation)
    return build


MNIST_CONV_VARIABLES = (("conv_layer1/weights1", (3, 3, 1, 16)), ("conv_layer1/biases1", (16,)),
                        ("conv_layer2/weights1", (5, 5, 16, 32)), ("conv_layer2/biases1", (32,)),
                        ("fc_weights", (512, 10)), ("fc_bias", (10,)))


def mnist_conv_forward(params, pixels, labels, batch_norm=True):
    """The ConvNet of DM/problems.py:302-338 on a batch of fp32 pixels [B, 784]: NHWC semantics on torch's NCHW ops.
    ``params`` are the six variables in creation order (HWIO conv weights)."""
    w1, b1, w2, b2, wf, bf = params
    F = torch.nn.functional
    h = pixels.to(w1.dtype).reshape(-1, 1, 28, 28)
    for w, b in ((w1, b1), (w2, b2)):
        h = F.conv2d(h, w.permute(3, 2, 0, 1)) + b.reshape(1, -1, 1, 1)   # VALID, stride 1, then bias_add
        if batch_norm:
            # tf.layers.batch_normalization(training=True): batch mean and biased variance, eps 1e-3; its gamma / beta
            # are not optimizee variables (DM/meta.py:88-99 patches tf.get_variable only), so they stay 1 and 0
            h = F.batch_norm(h, None, None, training=True, eps=1e-3)
        h = F.max_pool2d(F.relu(h), 2, 2)                   # VALID: 26 -> 13, 9 -> 4 (row and column 8 dropped)
    h = h.permute(0, 2, 3, 1).reshape(h.shape[0], -1)     # tf.reshape([B, -1]) of NHWC: (h, w, c)
    logits = F.relu(h @ wf + bf)                          # DM/problems.py:338: a ReLU on the logits
    return F.cross_entropy(logits, labels.long())


def mnist_conv(batch_norm=True, batch_size=128, mode="train", data_dir="MNIST-data"):
    """MNIST classification with the batch-normalised ConvNet of DM/problems.py:291-347: conv 3x3 1->16 and conv 5x5
    16->32 (VALID, each + bias, batch norm, ReLU, max-pool 2x2/2), fc 512->10 with a ReLU on the logits, the mean sparse
    softmax cross entropy of a fresh batch of ``batch_size`` drawn uniformly with replacement at EVERY evaluation.  The
    variables are the six of MNIST_CONV_VARIABLES (18,122 coordinates): weights N(0, 0.01), biases zero; batch norm's
    gamma and beta are not among them.  The data come from ``data_dir`` as for ``mnist``."""
    from . import mnist_data
    if mode not in ("train", "validation", "test"):
        raise ValueError("{} is not an MNIST split".format(mode))
    num_examples = mnist_data.load_mnist(data_dir)[mode].num_examples

    def build():
        params = [get_variable(name, shape=list(shape),
                               initializer=(random_normal_initializer(stddev=0.01) if len(shape) > 1 else
                                            constant_initializer(0.0)))
                  for name, shape in MNIST_CONV_VARIABLES]
        images, labels = mnist_data.device_split(data_dir, mode, params[0].device)
        idx = torch.randint(0, num_examples, (batch_size,), device=images.device)
        pixels = images.index_select(0, idx).float() * float(mnist_data.SCALE)
        return mnist_conv_forward(params, pixels, labels.index_select(0, idx), batch_norm)
    build.producer = producers.MnistConv(batch_size=int(batch_size), mode=mode, data_dir=data_dir,
                                         batch_norm=bool(batch_norm), variables=MNIST_CONV_VARIABLES)
    return build


CIFAR10_VARIABLES = (("conv_layer1/weights1", (3, 3, 3, 16)), ("conv_layer1/biases1", (16,)),
                     ("conv_layer2/weights1", (5, 5, 16, 32)), ("conv_layer2/biases1", (32,)),
                     ("fc_weights", (32, 10)), ("fc_bias", (10,)))


def cifar10_forward(params, pixels, labels, batch_norm=True):
    """The ConvNet of DM/problems.py:410-448 on a batch of fp32 NHWC pixels [B, 32, 32, 3]: NHWC semantics on torch's
    NCHW ops.  ``params`` are the six variables in creation order (HWIO conv weights)."""
    w1, b1, w2, b2, wf, bf = params
    F = torch.nn.functional
    h = pixels.to(w1.dtype).reshape(-1, 32, 32, 3).permute(0, 3, 1, 2)
    for w, b in ((w1, b1), (w2, b2)):
        h = F.conv2d(h, w.permute(3, 2, 0, 1), stride=2) + b.reshape(1, -1, 1, 1)   # VALID, stride 2, then bias_add
        if batch_norm:   # training mode, gamma = 1, beta = 0, as mnist_conv_forward (DESIGN §3.18)
            h = F.batch_norm(h, None, None, training=True, eps=1e-3)
        h = F.max_pool2d(F.relu(h), 2, 2)                   # VALID: 15 -> 7 (row and column 14 dropped), 2 -> 1
    h = h.permute(0, 2, 3, 1).reshape(h.shape[0], -1)     # tf.reshape([B, -1]) of NHWC: (h, w, c)
    logits = F.relu(h @ wf + bf)                          # DM/problems.py:448: a ReLU on the logits
    return F.cross_entropy(logits, labels.long())


def cifar10(batch_norm=True, batch_size=128, mode="train", data_dir="cifar10"):
    """CIFAR-10 classification with the batch-normalised ConvNet of DM/problems.py:369-458: conv 3x3 3->16 and conv
    5x5 16->32 (stride 2, VALID, each + bias, batch norm, ReLU, max-pool 2x2/2), fc 32->10 with a ReLU on the logits,
    the mean sparse softmax cross entropy of a fresh batch of ``batch_size`` drawn uniformly with replacement at EVERY
    evaluation (the reference dequeues from a shuffling queue instead; DESIGN §3.18).  The variables are the six of
    CIFAR10_VARIABLES (13,610 coordinates): weights N(0, 0.01), biases zero; batch norm's gamma and beta are not among
    them.  The data come from the CIFAR-10 binary files in ``data_dir`` (cifar_data; never downloaded)."""
    from . import cifar_data
    num_examples = cifar_data.load_cifar10(data_dir, mode).num_examples

    def build():
        params = [get_variable(name, shape=list(shape),
                               initializer=(random_normal_initializer(stddev=0.01) if len(shape) > 1 else
                                            constant_initializer(0.0)))
                  for name, shape in CIFAR10_VARIABLES]
        images, labels = cifar_data.device_split(data_dir, mode, params[0].device)
        idx = torch.randint(0, num_examples, (batch_size,), device=images.device)
        pixels = cifar_data.device_values(images.device)[images.index_select(0, idx).long()]   # fp32(p) / fp32(255)
        pixels = pixels.reshape(-1, 3, 32, 32).permute(0, 2, 3, 1)                            # the planes, NHWC
        return cifar10_forward(params, pixels, labels.index_select(0, idx), batch_norm)
    build.producer = producers.CifarConv(batch_size=int(batch_size), mode=mode, data_dir=data_dir,
                                         batch_norm=bool(batch_norm), variables=CIFAR10_VARIABLES)
    return build


NAS_VARIABLES = tuple((scope + suffix, shape) for scope, cin in (("node0", 3), ("node0_onto_node2", 16), ("node1", 16),
                                                                  ("node1_onto_node3", 16))
                      for suffix, shape in (("/weights1", (3, 3, cin, 16)), ("/biases1", (16,)))) + \
    (("fc_weights", (16, 10)), ("fc_bias", (10,)))


def nas_forward(params, pixels, labels, batch_norm=True):
    """The NAS cell network of DM/problems.py:584-625 on a batch of fp32 NHWC pixels [B, 32, 32, 3]: NHWC semantics on
    torch's NCHW ops.  ``params`` are the ten variables in creation order (HWIO conv weights)."""
    w0, b0, wa, ba, w1, b1, wb, bb, wf, bf = params
    F = torch.nn.functional

    def conv(h, w, b):   # 3x3 SAME stride 1 (pad 1), bias_add, batch norm as cifar10_forward, ReLU
        h = F.conv2d(h, w.permute(3, 2, 0, 1), padding=1) + b.reshape(1, -1, 1, 1)
        if batch_norm:
            h = F.batch_norm(h, None, None, training=True, eps=1e-3)
        return F.relu(h)
    node0 = conv(pixels.to(w0.dtype).reshape(-1, 32, 32, 3).permute(0, 3, 1, 2), w0, b0)
    node0_onto_node2 = conv(node0, wa, ba)
    node1 = conv(node0, w1, b1)
    node1_onto_node3 = conv(node1, wb, bb)
    # tf.nn.avg_pool SAME divides by the in-image cells of each window (4 at a corner, 6 on an edge, 9 inside)
    node2 = F.avg_pool2d(node1, 3, 1, padding=1, count_include_pad=False) + node0_onto_node2
    node3 = node2 + node1_onto_node3 + node0
    logits = F.relu(node3.mean(dim=(2, 3)) @ wf + bf)   # the mean over the 1024 positions per channel
    return F.cross_entropy(logits, labels.long())


def nas(batch_norm=True, batch_size=128, mode="train", data_dir="cifar10"):
    """CIFAR-10 classification with the NAS cell of DM/problems.py:540-634: four 3x3 SAME convs (each + bias, batch
    norm, ReLU) wired node0 -> {n0o2, node1}, node1 -> n1o3, node2 = avgpool3x3(node1) + n0o2, node3 = node2 + n1o3 +
    node0, the mean over positions, fc 16->10 with a ReLU on the logits.  The variables are the ten of NAS_VARIABLES
    (7,578 coordinates): weights N(0, 0.01), biases zero.  Data and batch draw as ``cifar10``."""
    from . import cifar_data
    num_examples = cifar_data.load_cifar10(data_dir, mode).num_examples

    def build():
        params = [get_variable(name, shape=list(shape),
                               initializer=(random_normal_initializer(stddev=0.01) if len(shape) > 1 else
                                            constant_initializer(0.0)))
                  for name, shape in NAS_VARIABLES]
        images, labels = cifar_data.device_split(data_dir, mode, params[0].device)
        idx = torch.randint(0, num_examples, (batch_size,), device=images.device)
        pixels = cifar_data.device_values(images.device)[images.index_select(0, idx).long()]   # fp32(p) / fp32(255)
        pixels = pixels.reshape(-1, 3, 32, 32).permute(0, 2, 3, 1)                            # the planes, NHWC
        return nas_forward(params, pixels, labels.index_select(0, idx), batch_norm)
    build.producer = producers.Nas(batch_size=int(batch_size), mode=mode, data_dir=data_dir,
                                   batch_norm=bool(batch_norm), variables=NAS_VARIABLES)
    return build


_PSF_PARAMS = ("I", "x", "y", "z", "sigmaxy", "sigmaz")


def _psf_3d(theta, ROI):
    """point_spread_function_3d (DM/problems.py:899-932): theta = [I0, x0, y0, z0, sigmaxy, sigmaz] as [B, 1] quantiles
    of their tfd.Uniform priors (quantile(p) = low + p (high - low)); returns the image [B, nx*ny*nz] on the reference's
    tf.meshgrid ('xy' indexing) voxel order."""
    dt, dev = theta[0].dtype, theta[0].device
    lows = (0.5, 0.5, 0.5, 0.5, 2.0, 2.0)
    highs = (2.0, ROI[0] - 1, ROI[1] - 1, ROI[2] - 1, 4.0, 4.0)
    xs, ys, zs = (torch.linspace(0.0, float(n - 1), n, dtype=dt, device=dev) for n in ROI)
    X, Y, Z = torch.meshgrid(xs, ys, zs, indexing="xy")
    I0, x0, y0, z0, sigmaxy, sigmaz = (lo + t.reshape(t.shape[0], 1) * (hi - lo)
                                       for t, lo, hi in zip(theta, lows, highs))
    xk, yk, zk = X.reshape(1, -1), Y.reshape(1, -1), Z.reshape(1, -1)
    sqrt2 = float(np.sqrt(np.float32(2.0), dtype=np.float32))   # tf.math.sqrt(2.0); a Python scalar keeps graph capture free
                                                                # of host-to-device copies
    return I0 * ((-torch.erf((-0.5 - x0 + xk) / (sqrt2 * sigmaxy)) + torch.erf((0.5 - x0 + xk) / (sqrt2 * sigmaxy)))
                 * (-torch.erf((-0.5 - y0 + yk) / (sqrt2 * sigmaxy)) + torch.erf((0.5 - y0 + yk) / (sqrt2 * sigmaxy)))
                 * (-torch.erf((-0.5 - z0 + zk) / (sqrt2 * sigmaz)) + torch.erf((0.5 - z0 + zk) / (sqrt2 * sigmaz)))) / 8.0


def _l2_normalize(v):
    """tf.math.l2_normalize(v, axis=1): v * rsqrt(max(sum v^2, 1e-12))."""
    return v * torch.rsqrt(torch.clamp_min(torch.sum(v * v, dim=1, keepdim=True), 1e-12))


def confocal_microscopy_3d(batch_size=128, num_points=5, ROI=(28, 28, 28), stddev=0.01):
    """Fit num_points Gaussian point-spread functions and a background to a simulated confocal image (DM/problems.py:
    701-956, the ``inference=False`` branch :799-956).  Trainables [batch, 1]: I_var_p, x_var_p, y_var_p, z_var_p,
    sigmaxy_var_p, sigmaz_var_p per point, then bg_var; the simulated constants likewise (``y_sim%d`` has no underscore
    in the reference, :871), then bg_sim."""
    ROI = tuple(int(n) for n in ROI)

    def build():
        var = [[get_variable("%s_var_%d" % (name, i), shape=[batch_size, 1], initializer=random_uniform_initializer())
                for name in _PSF_PARAMS] for i in range(num_points)]
        sim = [[get_variable(("y_sim%d" if name == "y" else name + "_sim_%d") % i, shape=[batch_size, 1],
                             initializer=random_uniform_initializer(), trainable=False)
                for name in _PSF_PARAMS] for i in range(num_points)]
        y_pred = _psf_3d(var[0], ROI)
        for i in range(1, num_points):
            y_pred = y_pred + _psf_3d(var[i], ROI)
        y_sim = _psf_3d(sim[0], ROI)
        for i in range(1, num_points):
            y_sim = y_sim + _psf_3d(sim[i], ROI)
        bg_var = get_variable("bg_var", shape=[batch_size, 1], initializer=random_normal_initializer(stddev=stddev))
        bg_sim = get_variable("bg_sim", shape=[batch_size, 1], initializer=random_uniform_initializer(), trainable=False)
        return torch.mean(torch.sum((y_pred + bg_var - _l2_normalize(y_sim + bg_sim)) ** 2, dim=1))
    # the separable PSF lets one kernel launch produce f and df/dx without forming the [batch, voxels] image in HBM
    names = ["%s_var_%d" % (n, i) for i in range(num_points) for n in _PSF_PARAMS] + ["bg_var"]
    sims = [("y_sim%d" if n == "y" else n + "_sim_%d") % i for i in range(num_points) for n in _PSF_PARAMS]
    build.producer = producers.Confocal(num_points, ROI, variables=names, constants=sims + ["bg_sim"])
    return build


def square_cos(batch_size=128, num_dims=10, stddev=0.01):
    """f = mean_b( ||W_b x_b - y_b||^2 - sum(Wcos_b 10 cos(c x_b)) + 10 num_dims ), c = fp32(2 * 3.1415926)
    (DM/problems.py:959-995).  At the registry's 256 coordinates the graph-captured autograd step is the fast path
    (see ``quadratic``), so it has no kernel."""
    c = float(np.float32(2 * 3.1415926))

    def build():
        x = get_variable("x", shape=[batch_size, num_dims], initializer=random_normal_initializer(stddev=stddev))
        w = get_variable("w", shape=[batch_size, num_dims, num_dims], initializer=random_uniform_initializer(),
                         trainable=False)
        y = get_variable("y", shape=[batch_size, num_dims], initializer=random_uniform_initializer(), trainable=False)
        wcos = get_variable("wcos", shape=[batch_size, num_dims, num_dims], initializer=random_uniform_initializer(),
                            trainable=False)
        product = torch.bmm(w, x.unsqueeze(-1)).squeeze(-1)
        product2 = torch.bmm(wcos, (10 * torch.cos(c * x)).unsqueeze(-1)).squeeze(-1)
        product3 = torch.sum((product - y) ** 2, 1) - torch.sum(product2, 1) + 10 * num_dims
        return torch.mean(product3)
    return build
