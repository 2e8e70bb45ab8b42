"""Optimizer networks behind the reference's ``networks`` surface (DM/networks.py).

``factory`` / ``save`` / ``Network.__call__(inputs, prev_state) -> (delta, next_state)`` /
``initial_state_for_inputs`` keep the reference's names, argument meaning and error behaviour;
the arithmetic runs in the CUDA library (one fused kernel per call instead of ~40 TF ops).
"""
from __future__ import annotations

import collections
import math
import pickle
import sys
from typing import Optional

import numpy as np
import torch

from . import engine as _engine
from ._lib import L2OError

try:  # the reference pickles with dill (DM/networks.py:25); the wire format is plain pickle-compatible
    import dill as _pickle
except Exception:  # pragma: no cover
    _pickle = pickle


def factory(net, net_options=(), net_path=None):
    """Network factory (DM/networks.py:34-44)."""
    net_class = getattr(sys.modules[__name__], net)
    net_options = dict(net_options)
    if net_path:
        with open(net_path, "rb") as f:
            net_options["initializer"] = _pickle.load(f)
    return net_class(**net_options)


def save(network, sess=None, filename=None):
    """Save the variables of a network: ``{module_name: {variable_name: ndarray}}`` (DM/networks.py:47-62)."""
    to_save = collections.defaultdict(dict)
    for (mod, var, shp), arr in zip(network.variable_shapes(), network.get_variables()):
        to_save[mod][var] = arr
    if filename:
        with open(filename, "wb") as f:
            _pickle.dump(dict(to_save), f)
    return dict(to_save)


class State(tuple):
    """Tuple over layers of (hidden, cell) views [N, H] that remembers its backing arena."""
    arena: Optional[torch.Tensor] = None


def _trunc_normal(shape, std, gen):
    t = torch.empty(shape, dtype=torch.float64)
    torch.nn.init.trunc_normal_(t, mean=0.0, std=std, a=-2 * std, b=2 * std, generator=gen)
    return t.float()


def _convert_initializer(init, shape, gen):
    """DM/networks.py:75-95: string -> tf.<name>_initializer, ndarray -> constant, else callable."""
    if isinstance(init, str):
        if init == "zeros":
            return torch.zeros(shape)
        if init == "ones":
            return torch.ones(shape)
        raise ValueError("unsupported initializer string {!r}".format(init))
    if isinstance(init, (np.ndarray, torch.Tensor)):
        return torch.as_tensor(np.asarray(init), dtype=torch.float32).reshape(shape).clone()
    if callable(init):
        return torch.as_tensor(init(shape, gen), dtype=torch.float32).reshape(shape)
    raise ValueError("unsupported initializer {!r}".format(type(init)))


def _lookup_initializer(initializers, layer_name, field):
    """DM/networks.py:98-151 (_get_initializers / _get_layer_initializers)."""
    if initializers is None:
        return None
    if isinstance(initializers, dict) and layer_name in initializers:
        initializers = initializers[layer_name]
    if isinstance(initializers, dict):
        return initializers.get(field)
    return initializers


class Network(object):
    """Base class for meta-optimizer networks (DM/networks.py:65-72)."""

    def initial_state_for_inputs(self, inputs, **kwargs):
        raise NotImplementedError


class _LSTMNet(Network):
    """What StandardDeepLSTM and KernelDeepLSTM share: theta in Sonnet creation order, the state arena, and one step
    call.  Subclasses create ``_handle`` and define ``variable_shapes`` before they call ``_init_theta``."""

    def _init_theta(self, initializer, seed, device):
        self.device = torch.device(device) if device is not None else (
            torch.device("cuda", torch.cuda.current_device()) if torch.cuda.is_available() else torch.device("cpu"))
        gen = torch.Generator().manual_seed(seed)
        parts = []
        for mod, var, shp in self.variable_shapes():
            init = _lookup_initializer(initializer, mod, var)
            if init is not None:
                t = _convert_initializer(init, shp, gen)
            elif mod.startswith("lstm"):     # Sonnet 1.x LSTM default: TruncatedNormal(1/sqrt(fan_in)) for w and b
                fan_in = [s for m, v, s in self.variable_shapes() if m == mod and v == "w_gates"][0][0]
                t = _trunc_normal(shp, 1.0 / math.sqrt(fan_in), gen)
            elif var == "w":                 # Sonnet Linear default
                t = _trunc_normal(shp, 1.0 / math.sqrt(shp[0]), gen)
            else:
                t = torch.zeros(shp)
            parts.append(t.reshape(-1))
        self.theta = torch.cat(parts).to(self.device).contiguous()
        assert self.theta.numel() == self._handle.n_theta

    @property
    def handle(self):
        return self._handle

    def get_variables(self):
        th = self.theta.detach().cpu().numpy()
        out, off = [], 0
        for _, _, shp in self.variable_shapes():
            n = int(np.prod(shp))
            out.append(th[off:off + n].reshape(shp).copy())
            off += n
        return out

    def set_variables(self, data):
        """``data``: {module: {var: ndarray}} (the .l2l format)."""
        parts = [torch.as_tensor(np.asarray(data[m][v]), dtype=torch.float32).reshape(-1)
                 for m, v, _ in self.variable_shapes()]
        self.theta.copy_(torch.cat(parts).to(self.theta.device))

    # ---- operator surface --------------------------------------------------------------------
    def _state_arena(self, prev_state):
        arena = getattr(prev_state, "arena", None)
        if arena is not None:
            return arena
        parts = []
        for h, c in prev_state:
            parts += [h.reshape(-1), c.reshape(-1)]
        return torch.cat(parts).contiguous() if parts else torch.zeros(1, device=self.theta.device)

    def _wrap_state(self, arena, n):
        st = State(self._handle.state_views(arena, n))
        st.arena = arena
        return st

    def _step(self, g, prev_state, m=None):
        """delta, next_state for the gradients ``g`` (RNNProp: and the moments ``m``, stacked as (m~, g~)).  Elements
        are taken in memory order; delta has the shape of ``g``."""
        gf = g.reshape(-1).contiguous()
        n = gf.numel()
        in0, in1 = (gf, None) if m is None else (m.reshape(-1).contiguous(), gf)
        arena_in = self._state_arena(prev_state)
        arena_out = torch.empty_like(arena_in)
        delta = torch.empty(n, dtype=torch.float32, device=gf.device)
        self._handle.step(self.theta, in0, arena_in, arena_out, in1=in1, delta=delta)
        return delta.reshape(g.shape), self._wrap_state(arena_out, n)

    def initial_state_for_inputs(self, inputs, **kwargs):
        """Zero (hidden, cell) per layer, one state row per coordinate (DM/networks.py:234-236, 273-276)."""
        n = int(np.prod(inputs.shape))
        return self._wrap_state(self._handle.new_state(n, self.theta.device), n)


class StandardDeepLSTM(_LSTMNet):
    """LSTM layers with a Linear layer on top (DM/networks.py:154-236).  Only the coordinate-wise uses
    (output_size == 1) are on the accelerated path."""

    _n_in = 1

    def __init__(self, output_size, layers, preprocess_name="identity", preprocess_options=None, scale=1.0,
                 initializer=None, name="deep_lstm", tanh_output=False, seed=0, device=None):
        if output_size != 1:
            raise NotImplementedError("only coordinate-wise nets (output_size=1) are accelerated")
        self.name = name
        self._layers = tuple(int(h) for h in layers)
        self._preprocess_name = preprocess_name
        self._preprocess_options = dict(preprocess_options or {})
        self._scale = scale
        self.tanh_output = tanh_output
        self._handle = _engine.NetHandle(layers=self._layers, preprocess_name=preprocess_name,
                                         preprocess_options=self._preprocess_options, scale=scale,
                                         tanh_output=tanh_output, n_in=self._n_in)
        self._init_theta(initializer, seed, device)

    @property
    def feat(self):
        if self._preprocess_name == "fc":
            return int(self._preprocess_options["dim"])
        if self._preprocess_name == "LogAndSign":
            return 2 * self._n_in
        return self._n_in

    def variable_shapes(self):
        """(module, variable, shape) in Sonnet creation order == flat theta order."""
        out = []
        if self._preprocess_name == "fc":
            out += [("input_projection", "w", (self._n_in, self.feat)), ("input_projection", "b", (self.feat,))]
        k = self.feat
        for i, h in enumerate(self._layers, start=1):
            out += [("lstm_{}".format(i), "w_gates", (k + h, 4 * h)), ("lstm_{}".format(i), "b_gates", (4 * h,))]
            k = h
        out += [("linear", "w", (k, 1)), ("linear", "b", (1,))]
        return out

    def __call__(self, inputs, prev_state):
        """delta, next_state = net(gradients, prev_state) (DM/networks.py:207-232, 254-271)."""
        return self._step(inputs, prev_state)


class CoordinateWiseDeepLSTM(StandardDeepLSTM):
    """Coordinate-wise ``DeepLSTM`` (DM/networks.py:239-276)."""

    def __init__(self, name="cw_deep_lstm", **kwargs):
        super(CoordinateWiseDeepLSTM, self).__init__(1, name=name, **kwargs)


class RNNprop(StandardDeepLSTM):
    """DM/networks.py:279-300: net(m, g, prev_state), inputs stacked in the order (m~, g~)."""

    _n_in = 2

    def __init__(self, name="RNNprop", **kwargs):
        super(RNNprop, self).__init__(1, name=name, **kwargs)

    def __call__(self, m, g, prev_state):
        return self._step(g, prev_state, m)


class KernelDeepLSTM(_LSTMNet):
    """``DeepLSTM`` for convolutional filters (DM/networks.py:303-351): the input is a filter bank
    [kernel_w, kernel_h, n_input_channels, n_output_channels]; every (input, output) channel pair is one ROW whose
    kernel_w*kernel_h entries are the LSTM's inputs, and the output Linear produces the row's kernel_w*kernel_h updates.
    Runs on the run-time-shaped dense engine (``l2o_dense_*``)."""

    per_variable = True   # one run per optimizee variable (rows differ per filter bank)

    def __init__(self, kernel_shape, layers, preprocess_name="identity", preprocess_options=None, scale=1.0,
                 initializer=None, name="kernel_deep_lstm", tanh_output=False, seed=0, device=None):
        self.name = name
        self._kernel_shape = list(kernel_shape)
        self._k = int(np.prod(kernel_shape))
        self._layers = tuple(int(h) for h in layers)
        self._preprocess_name = preprocess_name
        self._preprocess_options = dict(preprocess_options or {})
        self._handle = _engine.DenseNetHandle(self._layers, self._k, self._k, preprocess_name=preprocess_name,
                                              preprocess_options=self._preprocess_options, scale=scale,
                                              tanh_output=tanh_output)
        self._init_theta(initializer, seed, device)

    @property
    def feat(self):
        return 2 * self._k if self._preprocess_name == "LogAndSign" else self._k

    def variable_shapes(self):
        out, k = [], self.feat
        for i, h in enumerate(self._layers, start=1):
            out += [("lstm_{}".format(i), "w_gates", (k + h, 4 * h)), ("lstm_{}".format(i), "b_gates", (4 * h,))]
            k = h
        out += [("linear", "w", (k, self._k)), ("linear", "b", (self._k,))]
        return out

    def _check(self, inputs):
        if inputs.dim() != 4 or list(inputs.shape[:2]) != self._kernel_shape:
            raise ValueError("KernelDeepLSTM expects a [kw, kh, cin, cout] tensor with kernel shape {}; got {}".format(
                self._kernel_shape, list(inputs.shape)))

    def initial_state_for_inputs(self, inputs, **kwargs):
        """Batch size = n_input_channels * n_output_channels (DM/networks.py:347-351)."""
        self._check(inputs)
        return super(KernelDeepLSTM, self).initial_state_for_inputs(inputs)

    def __call__(self, inputs, prev_state):
        """update, next_state = net(filter_gradient, prev_state) (DM/networks.py:329-346): element (k, r) of the flat
        input is at k * R + r, so the reference's transposes are index arithmetic."""
        self._check(inputs)
        return self._step(inputs, prev_state)


class Sgd(Network):
    def __init__(self, *a, **k):
        raise NotImplementedError("Sgd baseline net is outside the accelerated hot path (SURVEY.md section 2)")


class Adam(Network):
    def __init__(self, *a, **k):
        raise NotImplementedError("Adam baseline net is outside the accelerated hot path (SURVEY.md section 2)")
