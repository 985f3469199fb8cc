"""Data-parallel training step around the matcher (one process per GPU).

Restates the per-iteration body of the reference trainer
(/root/reference/gluefactory/train.py:456-517: zero_grad -> forward -> loss ->
mean -> backward -> gradient exchange -> Adam) with the two H100-specific
changes SURVEY.md section 2.2 (C1) calls for:

  * every parameter lives in ONE flat fp32 buffer and every gradient in one flat
    gradient buffer (the nn.Parameters are views), so the gradient exchange is a
    single `all_reduce` over NVLink per optimiser step instead of DDP's bucketed
    hooks plus the extra scalar all-reduce of train.py:483-488;
  * the optimiser (Adam, AdamW, SGD or RMSprop: train.optimizer) runs as one kernel
    over the flat buffers (`lgb200_<rule>_flat`), with the 1/world averaging folded
    into it.

Frozen parameters (train.opt_regexp, or requires_grad=False) stay in the flat
parameter buffer, behind the trainable ones, but are outside the gradient buffer,
the all-reduce and the optimiser; the backward skips their gradients.

The matcher is per-pair, so image pairs shard across ranks with no other
collective (SURVEY.md section 8e).
"""
import re

import torch
import torch.distributed as dist

from . import ops
from .synthetic import to_device

_ALIGN = 64  # elements; keeps every parameter view 256-byte aligned


class FlatParams:
    """Re-homes the parameters of `module` into one flat buffer (+ flat grad buffer).

    The trainable parameters (`params`) come first and occupy flat[:numel]; the frozen ones (requires_grad=False,
    `frozen`) follow, so that the one cast kernel of shadow_bf16 keeps refreshing their bf16 views too, while the
    gradient buffer, the all-reduce and the optimiser cover the trainable range only."""

    def __init__(self, module):
        self.params = [p for p in module.parameters() if p.requires_grad]
        self.frozen = [p for p in module.parameters() if not p.requires_grad]
        assert self.params, "no trainable parameters"
        dev, dt = self.params[0].device, torch.float32
        self.offsets, n = [], 0
        for p in self.params + self.frozen:
            assert p.dtype == dt and p.device == dev
            self.offsets.append(n)
            n += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
            if len(self.offsets) == len(self.params):
                self.numel = n  # the trainable range
        self.frozen_offsets = self.offsets[len(self.params):]
        del self.offsets[len(self.params):]
        self.numel_all = n
        self.flat = torch.zeros(n, device=dev, dtype=dt)
        # one extra aligned slot behind the gradients carries the step's loss through the SAME all-reduce, so that
        # every rank sees a non-finite loss of any rank and skips the update together (train.py:477-488)
        n = self.numel
        self.grad_ext = torch.zeros(n + _ALIGN, device=dev, dtype=dt)
        self.grad = self.grad_ext[:n]
        self.loss_slot = self.grad_ext[n:n + 1]
        for p, off in zip(self.params + self.frozen, self.offsets + self.frozen_offsets):
            self.flat[off:off + p.numel()].copy_(p.data.reshape(-1))
            p.data = self.flat[off:off + p.numel()].view_as(p)
        for p, off in zip(self.params, self.offsets):
            p.grad = self.grad[off:off + p.numel()].view_as(p)
        # bf16 shadow of the whole buffer (one cast kernel per step) for the tensor-core GEMMs
        self._names = {id(p): n for n, p in module.named_parameters()}
        self.flat16 = None
        self._views16 = None
        self.grad_views = [self.grad[off:off + p.numel()].view_as(p) for p, off in zip(self.params, self.offsets)]
        # "direct" parameter groups: their gradients are written into the flat buffer by the backward kernels themselves
        # (engine.LayerFn), so their .grad views stay attached (see enable_direct)
        self.direct_groups = []
        self._direct_ids = set()
        module._b200_flat = self

    def enable_direct(self, groups):
        """groups: lists of parameters (e.g. one transformer layer) whose backward writes the flat gradient buffer.
        A frozen parameter has no gradient slot: its entry in the group's view list is None."""
        index = {id(p): i for i, p in enumerate(self.params)}
        for params in groups:
            self.direct_groups.append([self.grad_views[index[id(p)]] if id(p) in index else None for p in params])
            self._direct_ids.update(id(p) for p in params if id(p) in index)
        for p, v in zip(self.params, self.grad_views):
            if id(p) in self._direct_ids:
                p.grad = v

    def direct_views(self, gi):
        return self.direct_groups[gi]

    def shadow_bf16(self):
        """name -> bf16 view of the parameter, refreshed from the fp32 master copy by ONE cast kernel."""
        if self.flat16 is None:
            self.flat16 = torch.empty(self.numel_all, device=self.flat.device, dtype=torch.bfloat16)
            self._views16 = {self._names[id(p)]: self.flat16[off:off + p.numel()].view_as(p)
                             for p, off in zip(self.params + self.frozen, self.offsets + self.frozen_offsets)}
        ops.call("lgb200_cast_bf16", ops.ptr(self.flat), ops.ptr(self.flat16), self.numel_all, ops.stream_ptr())
        return self._views16

    def lr_factors(self, lr_scaling):
        """The reference's LR groups (train.py:177-196 pack_lr_parameters, :353-361): `lr_scaling` is a list of
        (factor, [name substrings]); a parameter whose name contains one of the substrings trains at factor x lr
        (first matching group wins, as the reference's filter loop).  Returns one factor per parameter."""
        factors = []
        for p in self.params:
            name = self._names[id(p)]
            factors.append(next((factor for factor, filters in lr_scaling or () if any(f in name for f in filters)), 1))
        return factors

    def lr_scale_per_elem(self, lr_scaling):
        """The per-element multiplier vector of `lr_factors` for lgb200_adam_flat, or None when every factor is 1."""
        factors = self.lr_factors(lr_scaling)
        if all(f == 1 for f in factors):
            return None
        scale = torch.ones(self.numel, device=self.flat.device, dtype=torch.float32)
        for p, off, factor in zip(self.params, self.offsets, factors):
            if factor != 1:
                scale[off:off + p.numel()] = float(factor)
        return scale

    def lr_groups(self, lr_scaling):
        """[(factor, [parameter index])]: the optimiser groups pack_lr_parameters builds, one per distinct factor in
        order of first appearance, parameters in module order."""
        groups = {}
        for i, factor in enumerate(self.lr_factors(lr_scaling)):
            groups.setdefault(factor, []).append(i)
        return list(groups.items())

    def zero_grad(self):
        """Detach the .grad views: autograd then hands each freshly computed gradient over by reference
        (no per-parameter accumulate kernel); `gather_grads` packs them into the flat buffer."""
        for p, v in zip(self.params, self.grad_views):
            p.grad = v if id(p) in self._direct_ids else None  # direct groups are overwritten in place by backward

    def gather_grads(self):
        rest = [(v, p) for v, p in zip(self.grad_views, self.params) if id(p) not in self._direct_ids]
        have = [(v, p.grad) for v, p in rest if p.grad is not None]
        missing = [v for v, p in rest if p.grad is None]
        if have:
            torch._foreach_copy_([v for v, _ in have], [g for _, g in have])
        if missing:
            torch._foreach_zero_(missing)
        for p, v in zip(self.params, self.grad_views):
            p.grad = v


# train.optimizer (train.py:347-352) -> the torch.optim class whose options, state layout and arithmetic the flat
# kernel restates
OPTIMIZERS = {"sgd": torch.optim.SGD, "adam": torch.optim.Adam, "adamw": torch.optim.AdamW, "rmsprop": torch.optim.RMSprop}
# options that only choose among torch's own implementations of the same arithmetic: accepted and ignored
_IMPLEMENTATION_OPTIONS = ("foreach", "fused", "capturable", "differentiable")


def _resolve_optimizer(optimizer, lr, options):
    """-> (rule, torch's full option dict for one group without params / lr, per-parameter state keys in torch's order,
    whether that state holds a step count).  rule: the flat kernel ("adam", "adamw", "sgd", "rmsprop")."""
    if optimizer not in OPTIMIZERS:
        raise ValueError(f"optimizer {optimizer!r} is not one of {sorted(OPTIMIZERS)}")
    for key in ("maximize", "amsgrad"):
        if options.get(key):
            raise ValueError(f"optimizer option {key}=True is not supported by the flat-buffer trainer")
    # torch validates the values and fills in its defaults
    probe = {k: v for k, v in options.items() if k not in _IMPLEMENTATION_OPTIONS}
    group = OPTIMIZERS[optimizer]([torch.zeros(1, requires_grad=True)], lr=lr, **probe).param_groups[0]
    opts = {k: v for k, v in group.items() if k not in ("params", "lr")}
    if optimizer in ("adam", "adamw"):
        rule = "adamw" if optimizer == "adamw" or opts.get("decoupled_weight_decay") else "adam"
        return rule, opts, ["exp_avg", "exp_avg_sq"], True
    if optimizer == "sgd":
        return "sgd", opts, ["momentum_buffer"] if opts["momentum"] != 0 else [], False
    keys = ["square_avg"] + (["momentum_buffer"] if opts["momentum"] > 0 else []) + (["grad_avg"] if opts["centered"] else [])
    return "rmsprop", opts, keys, True


def select_parameters(model, opt_regexp):
    """train.py:125-141 filter_parameters over the model's own parameter names: every trainable parameter whose name
    `re.search(opt_regexp, name)` does not match is frozen (requires_grad_(False)).  Returns the selected names;
    raises ValueError, changing nothing, when no trainable parameter matches."""
    named = [(n, p) for n, p in model.named_parameters() if p.requires_grad]
    keep = [n for n, _ in named if re.search(opt_regexp, n)]
    if not keep:
        raise ValueError(f"opt_regexp {opt_regexp!r} matches no trainable parameter")
    for n, p in named:
        if not re.search(opt_regexp, n):
            p.requires_grad_(False)
    return keep


class MatcherTrainer:
    """model: a matcher with forward(data)->pred and loss(pred, data)->(losses, metrics).

    Every per-step control lives in device memory, so the eager step and the CUDA-graph replay run the SAME
    sequence with no host synchronisation:
        loss -> backward -> flat gradients (+ the loss in the extra slot) -> ONE all-reduce
             -> lgb200_flat_grad_check (any non-finite value on any rank?) -> lgb200_amp_update (step count)
             -> lgb200_<optimizer>_flat (skipped on the device when the check fired: train.py:477-480, 503-512).
    `loss_scale`: None (default; bf16 needs no loss scaling) or an initial GradScaler scale (train.py:456, 490):
    the loss is multiplied by the device-resident scale, the gradients are un-scaled inside the Adam kernel and the
    scale follows torch.amp.GradScaler.update.  `lr_scaling`: the reference's LR groups (train.py:353-361).
    `ground_truth`: device label generator (SURVEY 8f row 1), so a batch needs only keypoints, descriptors and H.
    `sync_batchnorm`: at world size > 1, convert the model's BatchNorms to nn.SyncBatchNorm over `process_group` (as
    train.py:337-339 does before the DDP wrap), so that they normalise with the statistics of the global batch;
    `self.model` is the converted module.
    `clip_grad`: the reference's train.clip_grad (train.py:501-512), fixed at construction; falsy disables it.  The
    check is then lgb200_flat_grad_norm: the norm of the averaged, unscaled gradient is taken on the device after the
    all-reduce (so every rank computes the same coefficient), a non-finite norm skips the step like
    clip_grad_norm_(error_if_nonfinite=True), and Adam receives the coefficient through its loss-scale divisor.
    `optimizer`: the reference's train.optimizer (train.py:347-361): "adam" (default), "adamw", "sgd" or "rmsprop", and
    `optimizer_options` its train.optimizer_options: torch's option names and defaults for that class (weight_decay 0.01
    for adamw; Adam with decoupled_weight_decay=True runs as AdamW).  `betas` / `eps` / `weight_decay` are Adam's and
    are overridden by optimizer_options.  maximize=True and amsgrad=True raise ValueError; foreach, fused, capturable
    and differentiable only choose among torch's implementations and are ignored.  Each rule is one kernel over the
    flat buffers (lgb200_{adam,adamw,sgd,rmsprop}_flat) with the same device-side controls; state buffers exist only
    where torch keeps that state (none for SGD without momentum).
    `opt_regexp`: the reference's train.opt_regexp (train.py:125-141, 353-356): trainable parameters whose name
    re.search does not match are frozen (requires_grad_(False)); ValueError when none matches.  Names are the model's
    own (the name space of `lr_scaling`), so a glue-factory pattern that includes the pipeline's `matcher.` prefix needs
    that prefix dropped.  Frozen parameters, whether frozen here or by the caller, stay in the flat parameter buffer
    but have no gradient, optimiser state or place in the all-reduce, and their weight gradients are never computed.
    `state_dict()` / `load_state_dict()` carry the optimiser state in the formats of torch.optim.<X> and
    torch.amp.GradScaler; the weights go through `model.state_dict()`, whose tensors are views of the flat buffer."""

    def __init__(self, model, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, process_group=None,
                 loss_scale=None, growth_factor=2.0, backoff_factor=0.5, growth_interval=2000, lr_scaling=None,
                 ground_truth=None, sync_batchnorm=False, clip_grad=None, optimizer="adam", optimizer_options=None,
                 opt_regexp=None):
        if optimizer == "adam":
            options = {"betas": betas, "eps": eps, "weight_decay": weight_decay, **(optimizer_options or {})}
        elif (tuple(betas), eps, weight_decay) != ((0.9, 0.999), 1e-8, 0.0):
            raise ValueError(f"the betas / eps / weight_decay keywords are Adam's: give {optimizer!r} its options "
                             "through optimizer_options")
        else:
            options = dict(optimizer_options or {})
        self.optimizer = optimizer
        self._rule, self._opt, self._state_keys, self._state_has_step = _resolve_optimizer(optimizer, float(lr), options)
        self._opt_given = options  # what a torch.optim.<X> over the same groups is built with (state_dict layout)
        if opt_regexp:
            select_parameters(model, opt_regexp)
        self.group = process_group
        self.world = dist.get_world_size(process_group) if dist.is_available() and dist.is_initialized() else 1
        if sync_batchnorm and self.world > 1:  # before FlatParams: the converted modules keep the same Parameters
            model = torch.nn.SyncBatchNorm.convert_sync_batchnorm(model, process_group)
        self.model = model.train()
        # optional label generator run at the top of every step on the device (two_view_pipeline.py:98-100 runs the
        # `ground_truth` component inside loss()): a module data -> {matches0, matches1, assignment, ...}, e.g.
        # gluefactory_b200.matchers.homography_matcher; its outputs are merged into the batch under the `gt_` prefix
        self.ground_truth = ground_truth
        self.fp = FlatParams(model)
        dev = self.fp.flat.device
        # optimiser state: one flat buffer per torch state key, over the trainable range
        self.state_buffers = {k: torch.zeros(self.fp.numel, device=dev) for k in self._state_keys}
        self.m, self.v = self.state_buffers.get("exp_avg"), self.state_buffers.get("exp_avg_sq")  # Adam / AdamW only
        layers = getattr(model, "transformers", None)
        if layers is not None:
            self.fp.enable_direct([list(layer.parameters()) for layer in layers])
        self._lr_dev = torch.full((1,), float(lr), device=dev, dtype=torch.float32)
        self._t_dev = torch.zeros(1, device=dev, dtype=torch.int32)
        self._found_inf = torch.zeros(1, device=dev, dtype=torch.float32)
        self._scale_dev = None if loss_scale is None else torch.full((1,), float(loss_scale), device=dev)
        self._growth = None if loss_scale is None else torch.zeros(1, device=dev, dtype=torch.int32)
        self._amp = (growth_factor, backoff_factor, growth_interval)
        self._lr_scale = self.fp.lr_scale_per_elem(lr_scaling) if lr_scaling else None
        self._groups = self.fp.lr_groups(lr_scaling)
        self._lr_host = float(lr)
        self._max_norm = float(clip_grad) if clip_grad else None
        if self._max_norm:
            self._grad_norm = torch.zeros(1, device=dev, dtype=torch.float32)
            self._adam_div = torch.ones(1, device=dev, dtype=torch.float32)
            self._norm_ws = None  # sized by the library at the first step: construction makes no library call
        self.calls = 0  # optimiser-step attempts (skipped steps included)

    # ---- controls (device scalars: changing them never invalidates a captured graph)
    @property
    def lr(self):
        return self._lr_host

    @lr.setter
    def lr(self, value):
        """Scheduler hook (train.py `lr_scheduler.step()`): takes effect on the next step, eager or replayed."""
        self._lr_host = float(value)
        self._lr_dev.fill_(float(value))

    @property
    def t(self):
        """Number of optimiser updates actually applied (reads the device counter: synchronises)."""
        return int(self._t_dev.item())

    def skipped_last_step(self):
        return bool(self._found_inf.item() != 0)

    def loss_scale(self):
        return None if self._scale_dev is None else float(self._scale_dev.item())

    # ---- checkpoints (utils/experiments.py:113-118 saves optimizer.state_dict(); train.py:379-382 restores it)
    def state_dict(self):
        """{"optimizer": the state_dict of a torch.optim.<optimizer> over pack_lr_parameters' groups (train.py:177-196),
        "grad_scaler": torch.amp.GradScaler.state_dict() (only with loss_scale)}, holding copies of the device state.
        SGD keeps no step count: as torch, it has no state before its first step and none at all without momentum."""
        fp, t = self.fp, float(self.t)
        layout = OPTIMIZERS[self.optimizer]([{"params": [fp.params[i] for i in ids], "lr": factor * self._lr_host}
                                             for factor, ids in self._groups],
                                            lr=self._lr_host, **self._opt_given).state_dict()
        state = {}
        if self._state_has_step or (self._state_keys and t >= 1):
            for k, i in enumerate(i for _, ids in self._groups for i in ids):
                p, off = fp.params[i], fp.offsets[i]
                st = {"step": torch.tensor(t, dtype=torch.float32)} if self._state_has_step else {}
                for key, buf in self.state_buffers.items():
                    st[key] = buf[off:off + p.numel()].view_as(p).clone()
                state[k] = st
        out = {"optimizer": {"state": state, "param_groups": layout["param_groups"]}}
        if self._scale_dev is not None:
            g, b, i = self._amp
            out["grad_scaler"] = {"scale": self.loss_scale(), "growth_factor": g, "backoff_factor": b,
                                  "growth_interval": i, "_growth_tracker": int(self._growth.item())}
        return out

    def load_state_dict(self, state_dict):
        """Load `state_dict()` output, or the state of a torch.optim.<optimizer> built over the same groups, in place: a
        captured graph stays valid.  Sets lr from the groups.  Raises ValueError, naming the first offending parameter,
        when the groups, shapes or states do not fit this trainer (it keeps one step count for every parameter), e.g.
        the state of another optimiser.  An SGD state carries no step count: the count becomes 1 when momentum buffers
        are loaded (the next step is not the first) and 0 when the state is empty.
        A "grad_scaler" entry is ignored without loss_scale, as by a disabled GradScaler."""
        fp, opt = self.fp, state_dict["optimizer"]
        groups, state = opt["param_groups"], opt["state"]

        def name(i):
            return fp._names[id(fp.params[i])]

        # group of each parameter in group order, on both sides: a differing group count or size shows as a difference
        order = [i for _, ids in self._groups for i in ids]
        mine = [gi for gi, (_, ids) in enumerate(self._groups) for _ in ids]
        theirs = [gi for gi, g in enumerate(groups) for _ in g["params"]]
        if mine != theirs:
            k = next((k for k, (a, b) in enumerate(zip(mine, theirs)) if a != b), min(len(mine), len(theirs)))
            raise ValueError(f"optimizer state has parameter groups of sizes {[len(g['params']) for g in groups]}, the "
                             f"trainer {[len(ids) for _, ids in self._groups]}: they first differ at parameter "
                             f"{name(order[min(k, len(order) - 1)])!r}")
        want = (["step"] if self._state_has_step else []) + self._state_keys
        label = OPTIMIZERS[self.optimizer].__name__
        # SGD before its first step, or without momentum, has no state at all
        fresh = not self._state_has_step and not any(state.get(key) for g in groups for key in g["params"])
        pairs, steps = [], []  # (trainer parameter index, source state), in group order
        for src, (_, ids) in zip(groups, self._groups):
            for i, key in zip(ids, src["params"]):
                if fresh:
                    continue
                st = state.get(key) or {}
                if any(k not in st for k in want):
                    raise ValueError(f"no {label} state for parameter {name(i)!r}: it holds {sorted(st)}, the trainer "
                                     f"needs {want}")
                if set(st) != set(want):
                    raise ValueError(f"parameter {name(i)!r}: state {sorted(st)} is not the {label} state {want}")
                shape = fp.params[i].shape
                for k in self._state_keys:
                    if st[k].shape != shape:
                        raise ValueError(f"parameter {name(i)!r}: state shape {tuple(st[k].shape)}, "
                                         f"parameter shape {tuple(shape)}")
                steps.append(float(st["step"]) if self._state_has_step else 1.0)
                if steps[-1] != steps[0]:
                    raise ValueError(f"parameter {name(i)!r} is at step {steps[-1]:g}, the first at {steps[0]:g}: the "
                                     "trainer keeps one step count")
                pairs.append((i, st))
        sc = state_dict.get("grad_scaler")
        if self._scale_dev is not None and sc:
            if (sc["growth_factor"], sc["backoff_factor"], sc["growth_interval"]) != self._amp:
                raise ValueError(f"GradScaler growth_factor / backoff_factor / growth_interval "
                                 f"{(sc['growth_factor'], sc['backoff_factor'], sc['growth_interval'])} differ from the "
                                 f"trainer's {self._amp}, which are fixed at construction")
        for i, st in pairs:
            off, n = fp.offsets[i], fp.params[i].numel()
            for k, buf in self.state_buffers.items():
                buf[off:off + n].copy_(st[k].reshape(-1))
        if fresh:
            for buf in self.state_buffers.values():
                buf.zero_()
        self._t_dev.fill_(int(steps[0]) if steps else 0)
        # base lr from a group of factor 1 when there is one (exact), else from the first group with a factor != 0
        lrs = [(f, g["lr"]) for (f, _), g in zip(self._groups, groups) if f != 0]
        if lrs:
            factor, lr = next((c for c in lrs if c[0] == 1), lrs[0])
            self.lr = lr / factor
        if self._scale_dev is not None and sc:
            self._scale_dev.fill_(float(sc["scale"]))
            self._growth.fill_(int(sc["_growth_tracker"]))

    def exchange_gradients(self):
        """The step's one exchange: ONE sum-all-reduce of the whole flat gradient buffer (+ the loss slot), behind
        backward.  Issued in its synchronous form, so the collective runs on the current stream and a captured step
        stays one linear chain of graph nodes."""
        if self.world > 1:
            dist.all_reduce(self.fp.grad_ext, op=dist.ReduceOp.SUM, group=self.group)

    # ---- CUDA-graph replay of the whole step (removes the ~2500 per-step launch calls from the host)
    def capture(self, example, device, warmup=3):
        """Capture forward + loss + backward + all-reduce + optimiser step into one CUDA graph.  `example` fixes the
        shapes; later batches are copied into the captured static input buffers.  The warm-up steps run on the
        example batch but leave no trace: parameters, optimiser state, step count and loss scale are restored."""
        # private static inputs: to_device() returns device tensors as they are, and step_graphed() overwrites these
        self._static = _clone(to_device(example, device))
        keep = [t.clone() for t in self._state_tensors()]
        side = torch.cuda.Stream(device=device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(warmup):
                self._step_impl(self._static)
        torch.cuda.current_stream().wait_stream(side)
        for t, k in zip(self._state_tensors(), keep):
            t.copy_(k)
        self.calls -= warmup
        self._graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(self._graph):
            self._static_loss, self._static_losses = self._step_impl(self._static)
        self.calls -= 1  # the capture itself executes nothing
        return self

    def _state_tensors(self):
        ts = [self.fp.flat, *self.state_buffers.values(), self._t_dev]
        if self._scale_dev is not None:
            ts += [self._scale_dev, self._growth]
        return ts

    def step_graphed(self, data, prefetch=None):
        """Replay the captured step on a new batch (host or device tensors of the captured shapes).

        `prefetch`: the batch of the NEXT call (pinned host memory).  Its host-to-device copy is queued on a side
        stream into a staging set right after this step's graph launch, so it overlaps this step's compute; the next
        call (which must pass that same object as `data`) then only does a device-to-device copy into the captured
        static inputs."""
        cur = torch.cuda.current_stream()
        if getattr(self, "_staged_src", None) is data and data is not None:
            cur.wait_event(self._staged_ready)
            _copy_into(self._static, self._staged)
            self._staged_src = None
            self._staged_free.record(cur)
        else:
            _copy_into(self._static, data)
        self._graph.replay()
        if prefetch is not None:
            if getattr(self, "_staged", None) is None:
                self._staged = _empty_like(self._static)
                self._copy_stream = torch.cuda.Stream(device=self.fp.flat.device)
                self._staged_ready, self._staged_free = torch.cuda.Event(), torch.cuda.Event()
                self._staged_free.record(cur)
            self._copy_stream.wait_event(self._staged_free)  # the last D2D out of the staging set has finished
            with torch.cuda.stream(self._copy_stream):
                _copy_into(self._staged, prefetch)
                self._staged_ready.record(self._copy_stream)
            self._staged_src = prefetch
        self.calls += 1
        return self._static_loss, self._static_losses

    def step(self, data, device=None):
        """One optimiser step on one batch; `data` may live in (pinned) host memory."""
        if device is not None:
            data = to_device(data, device, non_blocking=True)
        return self._step_impl(data)

    def _step_impl(self, data):
        self.fp.zero_grad()
        if self.ground_truth is not None:
            data = {**data, **{f"gt_{k}": v for k, v in self.ground_truth(data).items()}}
        pred = self.model(data)
        losses, _ = self.model.loss(pred, data)
        loss = losses["total"].mean()
        (loss if self._scale_dev is None else loss * self._scale_dev[0]).backward()
        self.fp.gather_grads()
        self.fp.loss_slot.copy_(loss.detach().reshape(1))
        self.exchange_gradients()
        # non-finite loss or gradient on ANY rank -> every rank skips this update (and backs the loss scale off)
        checked = self.fp.grad_ext[:self.fp.numel + 4]
        if self._max_norm:  # the same check, plus the clip coefficient folded into Adam's loss-scale divisor
            if self._norm_ws is None:
                self._norm_ws = ops.flat_grad_norm_ws(self.fp.numel, self.fp.flat.device)
            ops.flat_grad_norm(checked, self.fp.numel, 1.0 / self.world, self._scale_dev, self._max_norm,
                               self._found_inf, self._grad_norm, self._adam_div, self._norm_ws)
            divisor = self._adam_div
        else:
            ops.flat_grad_check(checked, self._found_inf)
            divisor = self._scale_dev
        ops.amp_update(self._found_inf, step_dev=self._t_dev)  # ++step unless skipped (Adam's bias correction reads it)
        self._optimizer_step(divisor)
        if self._scale_dev is not None:  # GradScaler.update AFTER the step: the gradients carry the old scale
            g, b, i = self._amp
            ops.amp_update(self._found_inf, None, self._scale_dev, self._growth, g, b, i)
        self.calls += 1
        return loss.detach(), losses


    def _optimizer_step(self, divisor):
        """The update rule's one kernel over the trainable range of the flat buffers, skipped on the device when the
        check fired; `divisor`: the loss scale, or the clip coefficient's divisor."""
        fp, o, b = self.fp, self._opt, self.state_buffers
        p = fp.flat[:fp.numel]
        common = dict(grad_scale=1.0 / self.world, lr_scale_per_elem=self._lr_scale, lr_dev=self._lr_dev,
                      loss_scale_dev=divisor, found_inf_dev=self._found_inf)
        if self._rule in ("adam", "adamw"):
            update = ops.adam_flat_ if self._rule == "adam" else ops.adamw_flat_
            update(p, fp.grad, b["exp_avg"], b["exp_avg_sq"], 0, self._lr_host, o["betas"], o["eps"],
                   o["weight_decay"], step_dev=self._t_dev, **common)
        elif self._rule == "sgd":
            ops.sgd_flat_(p, fp.grad, b.get("momentum_buffer"), 0, self._lr_host, o["momentum"], o["dampening"],
                          o["nesterov"], o["weight_decay"], step_dev=self._t_dev, **common)
        else:
            ops.rmsprop_flat_(p, fp.grad, b["square_avg"], b.get("momentum_buffer"), b.get("grad_avg"), self._lr_host,
                              o["alpha"], o["eps"], o["weight_decay"], o["momentum"], **common)


def _clone(tree):
    return {k: (_clone(v) if isinstance(v, dict) else v.clone() if torch.is_tensor(v) else v) for k, v in tree.items()}


def _empty_like(tree):
    return {k: (_empty_like(v) if isinstance(v, dict) else torch.empty_like(v) if torch.is_tensor(v) else v)
            for k, v in tree.items()}


def _copy_into(dst, src):
    for k, v in dst.items():
        if isinstance(v, dict):
            _copy_into(v, src[k])
        elif torch.is_tensor(v):
            v.copy_(src[k], non_blocking=True)
