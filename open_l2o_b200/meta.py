"""Learning-to-learn (meta) optimizer behind the reference's ``MetaOptimizer`` surface (DM/meta.py).

The reference builds a TF graph and crosses the device boundary once per unroll with
``sess.run([cost, update, step])``.  Here ``meta_loss`` / ``meta_minimize`` return lightweight op
handles and ``Session.run`` executes one fused unroll (forward T steps [+ BPTT + Adam] + carry-over)
with the same fetch semantics:

  * all fetches of one ``run`` are evaluated from the same pre-update theta / x / state
    (TF evaluates ``update`` and ``step`` in the same step as ``cost``);
  * ``update`` commits x <- x_T, state <- s_T (truncated-BPTT carry-over, DM/meta.py:385-389);
  * ``step`` applies TF-Adam to the optimizer nets' variables (DM/meta.py:411-413);
  * ``reset`` re-runs the initializers of state + x + constants (DM/meta.py:378-383).

Two regimes (DESIGN.md): *fused* (separable optimizee evaluated in-kernel, one launch for all T steps) and
*external-gradient* (torch autograd, or a gradient producer of producers.py, between single-step launches, state
checkpointed in HBM).
"""
from __future__ import annotations

import collections
import os

import numpy as np
import torch

from . import engine as _engine
from . import networks
from .variables import variable_getter

MetaLoss = collections.namedtuple("MetaLoss", "loss, update, reset, fx, x")
MetaStep = collections.namedtuple("MetaStep", "step, update, reset, fx, x")


class Op(object):
    """Handle returned in MetaLoss / MetaStep; evaluated by Session.run."""

    def __init__(self, kind, program):
        self.kind, self.program = kind, program

    def __repr__(self):
        return "<l2o op {}>".format(self.kind)


class Placeholder(object):
    def __init__(self, name):
        self.name = name


class Session(object):
    """Minimal stand-in for tf.Session: ``run(fetches, feed_dict)``."""

    def run(self, fetches, feed_dict=None):
        flat = []

        def walk(f):
            if isinstance(f, (list, tuple)):
                for g in f:
                    walk(g)
            elif isinstance(f, Op):
                flat.append(f)
            elif f is not None:
                raise TypeError("cannot fetch {!r}".format(f))
        walk(fetches)
        results = {}
        for prog in {id(op.program): op.program for op in flat}.values():
            kinds = set(op.kind for op in flat if op.program is prog)
            results[id(prog)] = prog.execute(kinds, feed_dict or {})

        def build(f):
            if isinstance(f, list):
                return [build(g) for g in f]
            if isinstance(f, tuple):
                return tuple(build(g) for g in f)
            if f is None:
                return None
            return results[id(f.program)].get(f.kind)
        return build(fetches)

    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


# ------------------------------------------------------------------------------------------------
def _get_variables(func, gen, device):
    """Call ``func`` once, capturing the tensors it creates (DM/meta.py:102-128).
    Returns (variables, constants): lists of dicts {name, shape, init}."""
    variables, constants = [], []

    def getter(name, shape, dtype, initializer, trainable):
        if initializer is None:
            raise ValueError("variable {!r} needs an initializer".format(name))
        rec = dict(name=name, shape=shape, init=initializer)
        (variables if trainable else constants).append(rec)
        return initializer(shape, gen).to(device=device, dtype=torch.float32)

    with variable_getter(getter), torch.no_grad():
        func()
    return variables, constants


def _make_nets(variables, config, net_assignments):
    """DM/meta.py:162-216, same errors."""
    name_to_index = dict((v["name"], i) for i, v in enumerate(variables))
    if net_assignments is None:
        if len(config) != 1:
            raise ValueError("Default net_assignments can only be used if there is a single net config.")
        key = next(iter(config))
        nets = {key: networks.factory(**config[key])}
        keys, subsets = [key], [list(range(len(variables)))]
    else:
        nets, keys, subsets = {}, [], []
        for key, names in net_assignments:
            if key in nets:
                raise ValueError("Repeated netid in net_assigments.")
            nets[key] = networks.factory(**config[key])
            subsets.append([name_to_index[name] for name in names])
            keys.append(key)
    return nets, keys, subsets


class _Run(object):
    """A maximal contiguous slice of the flat coordinate arena served by one net."""

    def __init__(self, key, net, off, n):
        self.key, self.net, self.off, self.n = key, net, off, n


def plan_arena(variables, subsets, net_keys, nets):
    """Lay out the flat coordinate arena: variables in the order the subsets name them (so that each net's subset is
    contiguous where possible), unassigned ones last.  Each subset is then cut into maximal contiguous runs; a
    ``per_variable`` net gets one run per variable.  Returns ([slice of variable j in creation order], N, runs)."""
    sizes = [int(np.prod(v["shape"])) for v in variables]
    order = dict.fromkeys([j for subset in subsets for j in subset] + list(range(len(variables))))
    off, N = {}, 0
    for j in order:
        off[j], N = N, N + sizes[j]
    runs = []
    for key, subset in zip(net_keys, subsets):
        cur = None
        for j in subset:
            if cur is not None and cur.off + cur.n == off[j] and not getattr(nets[key], "per_variable", False):
                cur.n += sizes[j]
            else:
                cur = _Run(key, nets[key], off[j], sizes[j])
                runs.append(cur)
    return [slice(off[j], off[j] + sizes[j]) for j in range(len(variables))], N, runs


SegmentPlan = collections.namedtuple("SegmentPlan", "S bounds bytes")


def plan_segments(T, slot_floats, n, free_bytes=None, *, S=None, boundary_floats=0, step_floats=0, fixed_bytes=0,
                  headroom=0.9):
    """How the BPTT of a T-step unroll keeps the states it differentiates through.  ``slot_floats``: one checkpoint slot
    (every segmented run's state arena); ``n``: their coordinates (the carried lambda); ``boundary_floats``: what a
    segment start saves besides the state (the fused regime's x, RNNProp's m and v); ``step_floats``: floats per step of
    the buffers the backward sizes by its sweep length (RNNProp's tensor-core hand-over buffer); ``fixed_bytes``: what
    the program allocates either way.

    Full checkpoints (S = T) when they fit in ``headroom`` of ``free_bytes`` (None: always); otherwise segments of the
    S that minimises ceil(T/S) + S, and L2OError when even those do not fit.  ``S`` forces the segment length.  Returns
    SegmentPlan(S, bounds [0, S, 2S, ..., T], bytes per buffer): "ckpt" (S + 1 slots: the whole unroll's, or the one
    segment the backward recomputes), "handover" (S steps), and when segmented "boundary" (the state at every bound and
    the extras at every segment start) and "recompute" (the scratch copies a recompute runs on, and the carry)."""
    T = int(T)

    def plan(s):
        s = min(max(int(s), 1), max(T, 1))
        bounds = list(range(0, T, s)) + [T]
        b = {"ckpt": 4 * (s + 1) * slot_floats, "handover": 4 * s * step_floats}
        if s < T:
            nseg = len(bounds) - 1
            b["boundary"] = 4 * ((nseg + 1) * slot_floats + nseg * boundary_floats)
            b["recompute"] = 4 * (2 * slot_floats + boundary_floats + n)
        return SegmentPlan(s, bounds, b)

    if S is not None:
        return plan(S)
    full = plan(T)
    if free_bytes is None or fixed_bytes + sum(full.bytes.values()) <= headroom * free_bytes:
        return full
    seg = plan(min(range(1, T + 1), key=lambda s: (-(-T // s) + s, s)))
    need = fixed_bytes + sum(seg.bytes.values())
    if need > headroom * free_bytes:
        raise _engine.L2OError("the unroll needs {:.3g} GB even with BPTT segments of {} steps ({}), {:.3g} GB of {:.3g} GB "
                               "free may be used".format(need / 1e9, seg.S, seg.bytes, headroom * free_bytes / 1e9,
                                                         free_bytes / 1e9))
    return seg


def bptt_buffers(plan, runs, N, fused):
    """The BPTT buffers _Program allocates for ``plan``, under the plan's byte keys: {key: [(owner, name, shape)]},
    owner a run index or None (the program).  ``runs``: (slot floats, n, RNNProp moments, hand-over buffer) per
    segmented run; ``N``: the arena the fused regime saves x of."""
    S, nseg = plan.S, len(plan.bounds) - 1
    out = collections.defaultdict(list)
    for i, (slot, n, moments, handover) in enumerate(runs):
        out["ckpt"].append((i, "ckpt", ((S + 1) * slot,)))
        if handover:
            out["handover"].append((i, "bwd_scratch", (S, n, 20)))
        if nseg > 1:
            out["boundary"].append((i, "bstate", (nseg + 1, slot)))
            out["recompute"] += [(i, "rstate", (slot,)), (i, "d_state", (slot,)), (i, "lam", (n,))]
            if moments:
                out["boundary"].append((i, "bmv", (nseg, 2, n)))
                out["recompute"].append((i, "mv", (2, n)))
    if nseg > 1 and fused:
        out["boundary"].append((None, "bx", (nseg, N)))
        out["recompute"].append((None, "x_scr", (N,)))
    return dict(out)


def _adam_slots(nets):
    return {k: dict(m=torch.zeros_like(net.theta), v=torch.zeros_like(net.theta), k=0) for k, net in nets.items()}


def _adam_step(nets, dtheta, slots, lr):
    """TF-Adam on every net's theta from its meta-gradient, with the Adam slots ``slots`` (DM/meta.py:411-413)."""
    for k, net in nets.items():
        ad = slots[k]
        ad["k"] += 1
        _engine.adam_step(net.theta, dtheta[k], ad["m"], ad["v"], ad["k"], lr=lr)


class _Program(object):
    """One meta_loss graph: variables, nets, state, workspaces and the unroll executor."""

    def __init__(self, optimizer, make_loss, len_unroll, net_assignments, second_derivatives, learning_rate=None):
        if second_derivatives:
            raise NotImplementedError("second_derivatives=True needs optimizee Hessian-vector products "
                                      "(out of scope, SURVEY.md Appendix B)")
        if not torch.cuda.is_available():
            raise _engine.L2OError("MetaOptimizer needs a CUDA device (no CPU path)")
        self.opt = optimizer
        self.make_loss = make_loss
        self.T = int(len_unroll)
        self.device = torch.device("cuda", torch.cuda.current_device())
        self.gen = torch.Generator().manual_seed(optimizer.seed)
        self.learning_rate = learning_rate
        self.variables, self.constants = _get_variables(make_loss, torch.Generator().manual_seed(optimizer.seed),
                                                        self.device)
        print("Optimizee variables")
        print([v["name"] for v in self.variables])
        print("Problem variables")
        print([c["name"] for c in self.constants])
        self.nets, self.net_keys, self.subsets = _make_nets(self.variables, optimizer._config, net_assignments)
        optimizer._nets = self.nets
        self.var_slices, self.N, self.runs = plan_arena(self.variables, self.subsets, self.net_keys, self.nets)
        self.X = torch.zeros(self.N, device=self.device)
        self.const_vals = {}
        # both kernel regimes run one net over the whole arena; L2O_DISABLE_FUSED=1 turns both off (autograd, the
        # reference the profile scripts and parity tests compare against)
        enabled = os.environ.get("L2O_DISABLE_FUSED") != "1" and len(self.runs) == 1 and self.runs[0].n == self.N
        fused, producer = getattr(make_loss, "fused", None), getattr(make_loss, "producer", None)
        self.fused = fused if enabled and fused is not None and len(self.variables) == 1 else None
        # a gradient producer (producers.py): f and df/dx from ONE library call per step instead of torch autograd
        self.producer = (producer.bind(self) if enabled and producer is not None and
                         producer.accepts(self.variables, self.var_slices, self.constants) else None)
        self.adam = _adam_slots(self.nets)
        self.dtheta = {k: torch.zeros(net.theta.numel(), dtype=torch.float64, device=self.device)
                       for k, net in self.nets.items()}
        self.step_placeholder = Placeholder("step")
        # per-variable scale placeholders (random-scaling trick, DM/meta_dm_train.py:336-338,384-385): fx = f(x * scale)
        self.scale_placeholders = [Placeholder(v["name"] + "_scale") for v in self.variables]
        self.scale_flat = torch.ones(self.N, device=self.device)
        self.step_dev = torch.ones(1, dtype=torch.int32, device=self.device)  # step0 of the current unroll (RNNProp)
        self.scale_active = False
        self.mt_tasks = []
        self.unroll_idx = 0
        self._graphs, self._eager_calls, self._graph_failed, self._graph_kernels = {}, {}, False, {}
        self._alloc_workspaces(optimizer.bptt_segment)
        self.reset()

    # ---- memory ---------------------------------------------------------------------------------
    def _alloc_workspaces(self, segment=None):
        """``segment``: force BPTT segments of that many steps (tests); otherwise full checkpoints when they fit in the
        free device memory, segments otherwise (plan_segments)."""
        T = self.T
        fixed = 0
        for r in self.runs:
            h = r.net.handle
            r.slot = max(h.state_size(r.n), 1)   # floats of one checkpoint slot
            r.state = h.new_state(r.n, self.device)
            r.g_rec = torch.zeros(T + 1, r.n, device=self.device)
            if h.n_in == 2:
                r.m = torch.zeros(r.n, device=self.device)
                r.v = torch.zeros(r.n, device=self.device)
                r.m_work, r.v_work = torch.zeros_like(r.m), torch.zeros_like(r.v)
                r.feat_rec = torch.zeros(T, 2, r.n, device=self.device)
            # what the tensor-core BPTT of a tanh-output / fc(20) net (RNNProp) needs on top: the recorded deltas
            # (tanh' of the output layer) and the hand-over buffer between its layer-2 and layer-1 pass
            r.delta_rec = r.bwd_scratch = None
            if getattr(r.net, "tanh_output", False) and isinstance(h, _engine.NetHandle):
                r.delta_rec = torch.zeros(T, r.n, device=self.device)
            r.handover = h.n_in == 2 and isinstance(h, _engine.NetHandle) and tuple(h.layers) == (20, 20)
            # the dense engine (KernelDeepLSTM) has no segmented BPTT: its runs keep full checkpoints
            r.seg_ok = isinstance(h, _engine.NetHandle)
            fixed += 4 * (r.state.numel() + r.g_rec.numel() + (5 * r.n + 2 * T * r.n if h.n_in == 2 else 0) +
                          (T * r.n if r.delta_rec is not None else 0))
            if not r.seg_ok:
                r.ckpt = torch.zeros((T + 1) * r.slot, device=self.device)
                fixed += 4 * r.ckpt.numel()
        seg_runs = [r for r in self.runs if r.seg_ok]
        fused_N = self.N if self.fused is not None else 0
        free = None if segment is not None else torch.cuda.mem_get_info(self.device)[0]
        self.plan = plan_segments(T, sum(r.slot for r in seg_runs), sum(r.n for r in seg_runs), free, S=segment,
                                  boundary_floats=fused_N + sum(2 * r.n for r in seg_runs if r.net.handle.n_in == 2),
                                  step_floats=sum(20 * r.n for r in seg_runs if r.handover),
                                  fixed_bytes=fixed + 4 * 3 * self.N)
        self.segmented = len(self.plan.bounds) > 2
        self._bound_index = {t: k for k, t in enumerate(self.plan.bounds)}
        spec = [(r.slot, r.n, r.net.handle.n_in == 2, r.handover) for r in seg_runs]
        for bufs in bptt_buffers(self.plan, spec, self.N, self.fused is not None).values():
            for owner, name, shape in bufs:
                setattr(self if owner is None else seg_runs[owner], name, torch.zeros(shape, device=self.device))
        for r in self.runs:
            r.seg = self.segmented and r.seg_ok
        self._Xw = torch.zeros(self.N, device=self.device)   # x after the last unroll, committed by `update`
        self.fx_buf = torch.zeros(T + 1, dtype=torch.float64, device=self.device)

    def reset_x(self):
        """Re-run the initializers of x + constants only (``reset_x`` of DM/data_generator.py:50,80).  The tensors are
        refilled IN PLACE: captured CUDA graphs and views handed out earlier keep pointing at live, current data."""
        for v, xv in zip(self.variables, self._var_views(self.X)):
            xv.view(-1).copy_(v["init"](v["shape"], self.gen).reshape(-1).to(self.device))
        for c in self.constants:
            new = c["init"](c["shape"], self.gen).to(torch.float32).contiguous()
            cur = self.const_vals.get(c["name"])
            if cur is None or cur.shape != new.shape:
                self.const_vals[c["name"]] = new.to(self.device)
            else:
                cur.copy_(new)

    def reset(self):
        """variables_initializer(state + x + constants) (DM/meta.py:378-383)."""
        self.reset_x()
        for r in self.runs:
            r.state.zero_()
            if r.net.handle.n_in == 2:
                r.m.zero_()
                r.v.zero_()
        self.unroll_idx = 0

    # ---- optimizee evaluation --------------------------------------------------------------------
    @property
    def var_off(self):
        """Offset of each variable in the flat arena (creation order)."""
        return [s.start for s in self.var_slices]

    def _var_views(self, Xflat):
        """The optimizee variables as views of the flat arena (creation order)."""
        return [Xflat[s].view(v["shape"]) for s, v in zip(self.var_slices, self.variables)]

    @staticmethod
    def _fill(view, value):
        """Copy a host array (any shape with the view's element count) into a variable's view of the arena."""
        view.view(-1).copy_(torch.as_tensor(np.asarray(value, dtype=np.float32)).reshape(-1))

    def _loss_from_vars(self, var_list):
        """_make_with_custom_variables (DM/meta.py:131-155): trainables popped in creation order."""
        queue = collections.deque(range(len(self.variables)))

        def getter(name, shape, dtype, initializer, trainable):
            if trainable:
                return var_list[queue.popleft()]
            return self.const_vals[name]

        if self.scale_active:   # x (.) scale of the enhanced recipe (DM/meta_dm_train.py:336-338,384-385)
            var_list = [v * sc for v, sc in zip(var_list, self._var_views(self.scale_flat))]
        with variable_getter(getter):
            return self.make_loss()

    def _loss_at(self, Xflat):
        return self._loss_from_vars(self._var_views(Xflat))

    def _apply_scale_feed(self, feed):
        fed = [p for p in self.scale_placeholders if p in feed]
        if not fed:
            if self.scale_active:
                self.scale_flat.fill_(1.0)
                self.scale_active = False
            return
        self.scale_flat.fill_(1.0)
        for p, sv in zip(self.scale_placeholders, self._var_views(self.scale_flat)):
            if p in feed:
                self._fill(sv, feed[p])
        self.scale_active = True

    def assign_x(self, values):
        """assign_func of DM/train_dm.py:101-113: overwrite the optimizee variables (list in creation order)."""
        for xv, val in zip(self._var_views(self.X), values):
            self._fill(xv, val)

    def x_values(self, Xflat=None):
        """The optimizee variables of ``Xflat`` (default: the committed x) as host arrays in creation order."""
        return [v.cpu().numpy() for v in self._var_views(self.X if Xflat is None else Xflat)]

    def _value_and_grad(self, Xflat, t=None):
        """f(x) and df/dx as a flat [N] tensor at evaluation ``t`` of the unroll (0..T-1 the steps, T or None the final
        loss).  A producer makes them in one call; otherwise each variable is its own autograd leaf (a view of the
        arena), so the backward pass produces one gradient per variable and never materialises zero-filled [N]
        tensors."""
        if self.producer is not None:
            return self.producer(Xflat, self.scale_flat if self.scale_active else None, self.T if t is None else t)
        leaves = [v.detach().requires_grad_(True) for v in self._var_views(Xflat)]
        with torch.enable_grad():
            fx = self._loss_from_vars(leaves)
            grads = torch.autograd.grad(fx, leaves, allow_unused=True)
        g = torch.empty_like(Xflat)
        for gv, gj in zip(self._var_views(g), grads):
            if gj is None:
                gv.zero_()
            else:
                gv.copy_(gj)
        return fx.detach(), g

    # ---- the unroll --------------------------------------------------------------------------------
    def _step0(self, feed):
        if self.step_placeholder in feed:
            return int(feed[self.step_placeholder])
        return self.unroll_idx * self.T + 1

    def _moments(self, m, v, **kw):
        """RNNProp's Adam-moment arguments: the net's (m~, g~) input is formed in-kernel from (m, v)."""
        return dict(m=m, v=v, beta1=self.opt.beta1, beta2=self.opt.beta2, **kw)

    def _load_moments(self, r):
        """RNNProp: the unroll advances copies of the committed moments (committed by `update`)."""
        if r.net.handle.n_in == 2:
            r.m_work.copy_(r.m)
            r.v_work.copy_(r.v)

    def _fused_unroll(self, r, t0, t1, state, x, m, v, ckpt, fx, train):
        """The fused forward kernel over steps t0..t1 from (state, x, m, v), updated in place; records rows t0.. of
        g_rec (and RNNProp's features, the deltas) and adds f(x_t) to fx[t - t0]."""
        f, h = self.fused, r.net.handle
        kw = self._moments(m, v, step0=self._fused_step0 + t0, feat_rec=r.feat_rec[t0:]) if h.n_in == 2 else {}
        if train and r.delta_rec is not None:
            kw["delta_seq"] = r.delta_rec[t0:]
        h.unroll_fwd(r.net.theta, r.n, t1 - t0, state, opt_kind=_engine.OPT_KINDS[f.kind],
                     opt_a=self.const_vals[f.a].reshape(-1), opt_b=self.const_vals[f.b].reshape(-1),
                     opt_alpha=f.alpha, opt_fscale=f.fscale, x=x, ckpt=ckpt, g_rec=r.g_rec[t0:], fx=fx,
                     opt_group=getattr(f, "group", 0), **kw)

    def _forward_fused(self, train, step0):
        r, T = self.runs[0], self.T
        self._fused_regime, self._fused_step0 = True, step0
        self._Xw.copy_(self.X)
        work_state = r.state.clone()
        self.fx_buf.zero_()
        self._load_moments(r)
        m, v = (r.m_work, r.v_work) if r.net.handle.n_in == 2 else (None, None)
        if train and r.seg:
            # one launch per segment, the state, x (and m, v) carried through HBM between them and saved at each
            # segment start; f(x_t0) of a later segment replaces the earlier segment's last row
            for k, (t0, t1) in enumerate(zip(self.plan.bounds[:-1], self.plan.bounds[1:])):
                r.bstate[k].copy_(work_state)
                self.bx[k].copy_(self._Xw)
                if m is not None:
                    r.bmv[k, 0].copy_(m)
                    r.bmv[k, 1].copy_(v)
                if k > 0:
                    self.fx_buf[t0].zero_()
                self._fused_unroll(r, t0, t1, work_state, self._Xw, m, v, None, self.fx_buf[t0:], train)
        else:
            self._fused_unroll(r, 0, T, work_state, self._Xw, m, v, r.ckpt if train else None, self.fx_buf, train)
        r.state_final = work_state
        return self.fx_buf

    def _recompute(self, r, k):
        """Checkpoint slots 0..t1-t0 of segment k into r.ckpt, with the kernel and mode of the forward that ran, from
        scratch copies of what it saved at t0 (the boundary store and the committed x stay untouched)."""
        t0, t1 = self.plan.bounds[k], self.plan.bounds[k + 1]
        h, slot = r.net.handle, r.slot
        m = v = None
        if h.n_in == 2:
            r.mv.copy_(r.bmv[k])
            m, v = r.mv[0], r.mv[1]
        if self._fused_regime:
            r.rstate.copy_(r.bstate[k])
            self.x_scr.copy_(self.bx[k])
            self._fused_unroll(r, t0, t1, r.rstate, self.x_scr, m, v, r.ckpt, None, True)
            return
        r.ckpt[:slot].copy_(r.bstate[k])
        for t in range(t0, t1):
            kw = self._moments(m, v, step_ptr=self.step_dev, t_offset=t) if h.n_in == 2 else {}
            j = t - t0
            h.step(r.net.theta, r.g_rec[t], r.ckpt[j * slot:(j + 1) * slot], r.ckpt[(j + 1) * slot:(j + 2) * slot],
                   reuse_weights=(j > 0), **kw)

    def _state_slot(self, r, t):
        """Where the external-gradient forward keeps run r's state before step t: its checkpoint slot; segmented, the
        boundary store at a segment start and otherwise one of two rolling slots (the recompute scratch)."""
        slot = r.slot
        if not r.seg:
            return r.ckpt[t * slot:(t + 1) * slot]
        k = self._bound_index.get(t)
        if k is not None:
            return r.bstate[k]
        return r.ckpt[(t % 2) * slot:(t % 2 + 1) * slot]

    def _forward_external(self, train, step0):
        T, Xw = self.T, self._Xw
        self._fused_regime = False
        Xw.copy_(self.X)
        fxs = []
        for r in self.runs:
            self._state_slot(r, 0).copy_(r.state)
            self._load_moments(r)
        for t in range(T):
            fx, g = self._value_and_grad(Xw, t)
            fxs.append(fx)
            for r in self.runs:
                h = r.net.handle
                r.g_rec[t].copy_(g[r.off:r.off + r.n])
                kw = {}
                if h.n_in == 2:
                    if r.seg and t in self._bound_index:   # the moments a recompute of this segment starts from
                        r.bmv[self._bound_index[t], 0].copy_(r.m_work)
                        r.bmv[self._bound_index[t], 1].copy_(r.v_work)
                    kw = self._moments(r.m_work, r.v_work, step_ptr=self.step_dev, t_offset=t, feat_out=r.feat_rec[t])
                if train and r.delta_rec is not None:
                    kw["delta"] = r.delta_rec[t]
                # theta is constant inside an unroll: the weight image built at t = 0 serves every later step (runs that
                # share a net share its handle, so only the first run of step 0 rebuilds)
                h.step(r.net.theta, r.g_rec[t], self._state_slot(r, t), self._state_slot(r, t + 1),
                       x=Xw[r.off:r.off + r.n], reuse_weights=(t > 0), **kw)
        if train:
            fx, g = self._value_and_grad(Xw, T)
            for r in self.runs:
                r.g_rec[T].copy_(g[r.off:r.off + r.n])
        elif self.producer is not None:
            fx = self._value_and_grad(Xw, T)[0]
        else:
            with torch.no_grad():
                fx = self._loss_at(Xw)
        fxs.append(fx)
        for r in self.runs:
            r.state_final = self._state_slot(r, T)
        return torch.stack([f.reshape(()).double() for f in fxs])

    # ---- CUDA-graph path of the external-gradient regime ------------------------------------------------
    def _graph_body(self, train, step0):
        """Everything of one unroll that is launch-bound and shape-static: T x (autograd + step kernel) [+ BPTT]."""
        fx = self._forward_external(train, step0)
        if train:
            self._bptt()
        return fx

    def _bptt(self):
        """The meta-gradient of the unroll just run: dtheta zeroed, then one BPTT launch per run."""
        for d in self.dtheta.values():
            d.zero_()
        for r in self.runs:
            h = r.net.handle
            in_seq = r.feat_rec if h.n_in == 2 else r.g_rec
            if not r.seg:
                h.unroll_bwd(r.net.theta, r.n, self.T, in_seq, r.ckpt, self.dtheta[r.key], g_rec=r.g_rec,
                             **self._bwd_extra(r))
                continue
            # last segment first: recompute its checkpoints, then BPTT over them from the carried adjoint state and
            # lambda suffix sum (zero after the last step)
            r.d_state.zero_()
            r.lam.zero_()
            for k in reversed(range(len(self.plan.bounds) - 1)):
                t0, t1 = self.plan.bounds[k], self.plan.bounds[k + 1]
                self._recompute(r, k)
                kw = {} if r.delta_rec is None else {"delta_seq": r.delta_rec[t0:]}
                h.unroll_bwd_carry(r.net.theta, r.n, t1 - t0, in_seq[t0:], r.ckpt, self.dtheta[r.key], r.d_state, r.lam,
                                   g_rec=r.g_rec[t0:], scratch=r.bwd_scratch, **kw)

    @staticmethod
    def _bwd_extra(r):
        kw = {}
        if r.delta_rec is not None:
            kw["delta_seq"] = r.delta_rec
        if r.bwd_scratch is not None:
            kw["scratch"] = r.bwd_scratch
        return kw

    def _graph_eligible(self):
        # RNNProp's bias-correction exponent p = step0 + t is read from a device scalar (self.step_dev), so the graph
        # stays valid from unroll to unroll
        return os.environ.get("L2O_CUDA_GRAPH", "1") != "0" and self.fused is None and not self.scale_active

    def _run_external(self, train, step0):
        """Eager on the first two calls (warm-up: lazy allocations, autograd caches), then capture once per mode and
        replay: the per-step launches (~15 tiny kernels) collapse into one graph launch."""
        self.step_dev.fill_(int(step0))
        key = bool(train)
        if not self._graph_eligible() or self._graph_failed:
            return self._graph_body(train, step0)
        self._eager_calls[key] = self._eager_calls.get(key, 0) + 1
        if self._eager_calls[key] <= 2:
            return self._graph_body(train, step0)
        if key not in self._graphs:
            try:
                # garbage from earlier programs (their CUDAGraph objects free device memory when collected) must not be
                # finalised in the middle of this capture: a cudaFree during capture invalidates it
                import gc
                gc.collect()
                torch.cuda.synchronize()
                g = torch.cuda.CUDAGraph()
                n0 = _engine.launch_count()
                with torch.cuda.graph(g):
                    fx = self._graph_body(train, step0)
                self._graph_kernels[key] = _engine.launch_count() - n0   # library kernels recorded in this graph
                self._graphs[key] = (g, fx, [r.state_final for r in self.runs])
            except Exception as e:  # capture not possible for this optimizee: keep running the same kernels eagerly
                import warnings
                warnings.warn("CUDA-graph capture of the unroll failed (%r); staying eager" % (e,))
                self._graph_failed = True
                torch.cuda.synchronize()
                return self._graph_body(train, step0)
        g, fx, finals = self._graphs[key]
        g.replay()
        _engine.note_graph_replay(self._graph_kernels[key])
        for r, f in zip(self.runs, finals):
            r.state_final = f
        return fx

    def execute(self, kinds, feed):
        if kinds == {"reset"}:
            self.reset()
            return {}
        if "reset" in kinds:
            raise ValueError("fetch `reset` on its own (the reference runs it separately, DM/util.py:37)")
        out, mt = {}, collections.defaultdict(set)   # imitation fetches are "<kind>:<task index>"
        for k in kinds:
            if ":" in k:
                kind, ti = k.split(":")
                mt[int(ti)].add(kind)
        for ti in sorted(mt):
            out.update(self.mt_tasks[ti].execute(mt[ti], feed))
        kinds = set(k for k in kinds if ":" not in k)
        if mt and not kinds:
            return out
        train = "step" in kinds
        step0 = self._step0(feed)
        self._apply_scale_feed(feed)
        if self.fused is not None and not self.scale_active:
            fx = self._forward_fused(train, step0)
            if train:
                self._bptt()
        else:
            fx = self._run_external(train, step0)
        if train:
            if self.opt.distributed:
                from .dist import allreduce_meta_grad
                fx = allreduce_meta_grad(self.dtheta, fx)
        elif self.opt.distributed:
            import torch.distributed as dist
            fx = fx.clone()
            dist.all_reduce(fx)
        if "loss" in kinds:
            out["loss"] = float(fx.sum().item())
        if "fx" in kinds:
            out["fx"] = float(fx[self.T].item())
        if "x" in kinds:
            out["x"] = self.x_values(self._Xw)
        self.last_fx = fx
        if train:
            _adam_step(self.nets, self.dtheta, self.adam, self.learning_rate)
            out["step"] = None
        if "update" in kinds:
            self.X.copy_(self._Xw)
            for r in self.runs:
                r.state.copy_(r.state_final)
                if r.net.handle.n_in == 2:
                    r.m.copy_(r.m_work)
                    r.v.copy_(r.v_work)
            self.unroll_idx += 1
            out["update"] = None
        return out


class _MtTask(object):
    """One imitation-learning ("mt") task (DM/meta_dm_train.py:421-499): the optimizer nets run over PRE-RECORDED
    gradient sequences [T, N] with their own LSTM state; loss = sum_t 0.5 ||label_t - delta_t||^2 / N_total; its own
    Adam slots on the shared theta (DM/meta_dm_train.py:549-553).  This is the fully fused regime: one forward-unroll
    launch + one BPTT launch per subset, no optimizee in the loop."""

    def __init__(self, prog, index):
        self.prog, self.index = prog, index
        T = prog.T
        self.subsets = []
        for key, subset in zip(prog.net_keys, prog.subsets):
            runs = [r for r in prog.runs if r.key == key]
            if len(runs) != 1:
                raise NotImplementedError("imitation tasks need each net's variables contiguous in the arena")
            r = runs[0]
            h = r.net.handle
            if getattr(r.net, "per_variable", False):
                raise NotImplementedError("imitation tasks are implemented for the coordinate-wise nets")
            sb = dict(run=r, n=r.n, state=h.new_state(r.n, prog.device),
                      ckpt=torch.zeros((T + 1) * r.slot, device=prog.device),
                      dseq=torch.zeros(T * r.n, device=prog.device),
                      inp=Placeholder("mt{}_input_subset{}".format(index, len(self.subsets))),
                      lab=Placeholder("mt{}_label_subset{}".format(index, len(self.subsets))))
            if h.n_in == 2:   # RNNProp: the task carries its own Adam moments (DM/meta_rnnprop_train.py:469-486)
                sb.update(m=torch.zeros(r.n, device=prog.device), v=torch.zeros(r.n, device=prog.device),
                          feat=torch.zeros(T, 2, r.n, device=prog.device))
            if r.bwd_scratch is not None and prog.segmented:   # imitation keeps whole-unroll BPTT: a T-step hand-over
                sb["scratch"] = torch.zeros(T, r.n, 20, device=prog.device)
            self.subsets.append(sb)
        self.n_total = sum(sb["n"] for sb in self.subsets)
        self.adam = _adam_slots(prog.nets)
        self.il = torch.zeros(1, dtype=torch.float64, device=prog.device)

    def _dev(self, arr, T, n):
        t = torch.as_tensor(np.asarray(arr, dtype=np.float32)) if not torch.is_tensor(arr) else arr.float()
        return t.reshape(T, n).to(self.prog.device).contiguous()

    def execute(self, kinds, feed):
        prog, T = self.prog, self.prog.T
        if kinds == {"reset_mt"}:
            for sb in self.subsets:
                sb["state"].zero_()
                if "m" in sb:
                    sb["m"].zero_()
                    sb["v"].zero_()
            return {}
        train, commit = "step_mt" in kinds, "update_mt" in kinds
        self.il.zero_()
        if train:
            for d in prog.dtheta.values():
                d.zero_()
        finals = []
        step0 = prog._step0(feed)
        for sb in self.subsets:
            r, n = sb["run"], sb["n"]
            h = r.net.handle
            inp, lab = self._dev(feed[sb["inp"]], T, n), self._dev(feed[sb["lab"]], T, n)
            work, moments, kw, in_seq = sb["state"].clone(), None, {}, inp
            if h.n_in == 2:
                # RNNProp imitation unroll (DM/meta_rnnprop_train.py:505-534): raw gradients in, Adam features formed
                # in-kernel from the task's own (m, v) with p = float(step + t), recorded for the BPTT to read
                moments = (sb["m"].clone(), sb["v"].clone())
                kw, in_seq = prog._moments(*moments, step0=step0, feat_rec=sb["feat"]), sb["feat"]
            h.unroll_fwd(r.net.theta, n, T, work, in_seq=inp, ckpt=sb["ckpt"] if train else None, labels=lab,
                         imit_loss=self.il, n_total=self.n_total, delta_seq=sb["dseq"] if train else None, **kw)
            if train:  # the recorded deltas let the tensor-core BPTT run in imitation mode too
                bwd_kw = dict(prog._bwd_extra(r), delta_seq=sb["dseq"])
                if "scratch" in sb:
                    bwd_kw["scratch"] = sb["scratch"]
                h.unroll_bwd(r.net.theta, n, T, in_seq, sb["ckpt"], prog.dtheta[r.key], labels=lab, n_total=self.n_total,
                             **bwd_kw)
            finals.append((work, moments))
        out = {}
        if "loss_mt" in kinds:
            out["loss_mt:%d" % self.index] = float(self.il.item())
        if train:
            _adam_step(prog.nets, prog.dtheta, self.adam, prog.learning_rate)
            out["step_mt:%d" % self.index] = None
        if commit:
            for sb, (w, moments) in zip(self.subsets, finals):
                sb["state"].copy_(w)
                if moments is not None:
                    sb["m"].copy_(moments[0])
                    sb["v"].copy_(moments[1])
            out["update_mt:%d" % self.index] = None
        return out


class MetaOptimizer(object):
    """Learning to learn (meta) optimizer (DM/meta.py:219-414)."""

    beta1 = 0.95
    beta2 = 0.95

    def __init__(self, **kwargs):
        """``MetaOptimizer(**net_config)`` exactly as the reference (DM/meta.py:228): every keyword is a net id.  The
        two engine-side knobs ride on underscore-prefixed names that cannot collide with a net id the reference's
        drivers use: ``_seed`` (generator seed of the optimizee initializers, default 0) and ``_distributed``
        (coordinates sharded over torch.distributed ranks, one all-reduce of [dtheta | fx] per meta-step)."""
        self._nets = None
        self.seed = int(kwargs.pop("_seed", 0))
        self.distributed = bool(kwargs.pop("_distributed", False))
        # BPTT segment length (steps); None: full checkpoints whenever they fit in device memory (plan_segments)
        self.bptt_segment = kwargs.pop("_bptt_segment", None)
        if not kwargs:
            # default coordinatewise network (DM/meta.py:244-255)
            self._config = {
                "coordinatewise": {
                    "net": "CoordinateWiseDeepLSTM",
                    "net_options": {
                        "layers": (20, 20),
                        "preprocess_name": "LogAndSign",
                        "preprocess_options": {"k": 5},
                        "scale": 0.01,
                    }}}
        else:
            self._config = kwargs

    def save(self, sess=None, path=None, index=None):
        """Save meta-optimizer (DM/meta.py:255-267; ``index`` as in DM/meta_dm_train.py:257-272)."""
        result = {}
        for k, net in self._nets.items():
            if path is None:
                filename, key = None, k
            elif index is not None:
                filename = os.path.join(path, "{}.l2l-{}".format(k, index))
                key = filename
            else:
                filename = os.path.join(path, "{}.l2l".format(k))
                key = filename
            result[key] = networks.save(net, sess, filename=filename)
        return result

    def restore(self, sess, path, index):
        """DM/meta_dm_train.py:290-302: load ``<net id>.l2l-<index>`` into the live nets (Adam slots are untouched,
        exactly as the reference's assign ops leave them)."""
        for k, net in self._nets.items():
            with open(os.path.join(path, "{}.l2l-{}".format(k, index)), "rb") as f:
                data = networks._pickle.load(f)
            for m, v, shp in net.variable_shapes():
                if m not in data or v not in data[m] or tuple(np.shape(data[m][v])) != tuple(shp):
                    raise ValueError("{}.l2l-{}: variable {}/{} missing or of the wrong shape".format(k, index, m, v))
            net.set_variables(data)

    def meta_loss(self, make_loss, len_unroll, net_assignments=None, second_derivatives=False):
        """Returns ops computing the meta-loss (DM/meta.py:269-396)."""
        prog = _Program(self, make_loss, len_unroll, net_assignments, second_derivatives)
        self.program = prog
        self.step_placeholder = prog.step_placeholder
        return MetaLoss(Op("loss", prog), Op("update", prog), Op("reset", prog), Op("fx", prog), Op("x", prog))

    def meta_minimize(self, make_loss, len_unroll, learning_rate=0.01, **kwargs):
        """Returns ops minimizing the meta-loss with Adam (DM/meta.py:398-414)."""
        info = self.meta_loss(make_loss, len_unroll, **kwargs)
        self.program.learning_rate = learning_rate
        return MetaStep(Op("step", self.program), *info[1:])


class RNNpropMetaOptimizer(MetaOptimizer):
    """DM/meta_rnnprop_train.py / meta_rnnprop_eval.py: per-coordinate Adam moments feed the net."""

    def __init__(self, beta1=0.95, beta2=0.95, **kwargs):
        super(RNNpropMetaOptimizer, self).__init__(**kwargs)
        self.beta1, self.beta2 = beta1, beta2
