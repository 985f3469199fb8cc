"""Data-parallel training step around the matcher (one process per GPU).

Restates the per-iteration body of the reference trainer
(/root/reference/gluefactory/train.py:456-517: zero_grad -> forward -> loss ->
mean -> backward -> gradient exchange -> Adam) with the two H100-specific
changes SURVEY.md section 2.2 (C1) calls for:

  * every parameter lives in ONE flat fp32 buffer and every gradient in one flat
    gradient buffer (the nn.Parameters are views), so the gradient exchange is a
    single `all_reduce` over NVLink per optimiser step instead of DDP's bucketed
    hooks plus the extra scalar all-reduce of train.py:483-488;
  * Adam runs as one kernel over the flat buffers (`lgb200_adam_flat`), with the
    1/world averaging folded into it.

The matcher is per-pair, so image pairs shard across ranks with no other
collective (SURVEY.md section 8e).
"""
import torch
import torch.distributed as dist

from . import ops
from .synthetic import to_device

_ALIGN = 64  # elements; keeps every parameter view 256-byte aligned


class FlatParams:
    """Re-homes the trainable parameters of `module` into one flat buffer (+ flat grad buffer)."""

    def __init__(self, module):
        self.params = [p for p in module.parameters() if p.requires_grad]
        assert self.params, "no trainable parameters"
        dev, dt = self.params[0].device, torch.float32
        self.offsets, n = [], 0
        for p in self.params:
            assert p.dtype == dt and p.device == dev
            self.offsets.append(n)
            n += (p.numel() + _ALIGN - 1) // _ALIGN * _ALIGN
        self.numel = n
        self.flat = torch.zeros(n, device=dev, dtype=dt)
        # one extra aligned slot behind the gradients carries the step's loss through the SAME all-reduce, so that
        # every rank sees a non-finite loss of any rank and skips the update together (train.py:477-488)
        self.grad_ext = torch.zeros(n + _ALIGN, device=dev, dtype=dt)
        self.grad = self.grad_ext[:n]
        self.loss_slot = self.grad_ext[n:n + 1]
        for p, off in zip(self.params, self.offsets):
            self.flat[off:off + p.numel()].copy_(p.data.reshape(-1))
            p.data = self.flat[off:off + p.numel()].view_as(p)
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
        """groups: lists of parameters (e.g. one transformer layer) whose backward writes the flat gradient buffer."""
        index = {id(p): i for i, p in enumerate(self.params)}
        for params in groups:
            self.direct_groups.append([self.grad_views[index[id(p)]] for p in params])
            self._direct_ids.update(id(p) for p in params)
        for p, v in zip(self.params, self.grad_views):
            if id(p) in self._direct_ids:
                p.grad = v

    def direct_views(self, gi):
        return self.direct_groups[gi]

    def shadow_bf16(self):
        """name -> bf16 view of the parameter, refreshed from the fp32 master copy by ONE cast kernel."""
        if self.flat16 is None:
            self.flat16 = torch.empty(self.numel, device=self.flat.device, dtype=torch.bfloat16)
            self._views16 = {self._names[id(p)]: self.flat16[off:off + p.numel()].view_as(p)
                             for p, off in zip(self.params, self.offsets)}
        ops.call("lgb200_cast_bf16", ops.ptr(self.flat), ops.ptr(self.flat16), self.numel, ops.stream_ptr())
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


class MatcherTrainer:
    """model: a matcher with forward(data)->pred and loss(pred, data)->(losses, metrics).

    Every per-step control lives in device memory, so the eager step and the CUDA-graph replay run the SAME
    sequence with no host synchronisation:
        loss -> backward -> flat gradients (+ the loss in the extra slot) -> ONE all-reduce
             -> lgb200_flat_grad_check (any non-finite value on any rank?) -> lgb200_amp_update (step count)
             -> lgb200_adam_flat (skipped on the device when the check fired: train.py:477-480, 503-512).
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
    `state_dict()` / `load_state_dict()` carry the optimiser state in the formats of torch.optim.Adam and
    torch.amp.GradScaler; the weights go through `model.state_dict()`, whose tensors are views of the flat buffer."""

    def __init__(self, model, lr=1e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, process_group=None,
                 loss_scale=None, growth_factor=2.0, backoff_factor=0.5, growth_interval=2000, lr_scaling=None,
                 ground_truth=None, sync_batchnorm=False, clip_grad=None):
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
        self.m = torch.zeros_like(self.fp.flat)
        self.v = torch.zeros_like(self.fp.flat)
        self.betas, self.eps, self.wd = betas, eps, weight_decay
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
        """{"optimizer": the state_dict of a torch.optim.Adam over pack_lr_parameters' groups (train.py:177-196),
        "grad_scaler": torch.amp.GradScaler.state_dict() (only with loss_scale)}, holding copies of the device state."""
        fp, t = self.fp, float(self.t)
        layout = torch.optim.Adam([{"params": [fp.params[i] for i in ids], "lr": factor * self._lr_host}
                                   for factor, ids in self._groups],
                                  lr=self._lr_host, betas=self.betas, eps=self.eps, weight_decay=self.wd).state_dict()
        state = {}
        for k, i in enumerate(i for _, ids in self._groups for i in ids):
            p, off = fp.params[i], fp.offsets[i]
            state[k] = {"step": torch.tensor(t, dtype=torch.float32),
                        "exp_avg": self.m[off:off + p.numel()].view_as(p).clone(),
                        "exp_avg_sq": self.v[off:off + p.numel()].view_as(p).clone()}
        out = {"optimizer": {"state": state, "param_groups": layout["param_groups"]}}
        if self._scale_dev is not None:
            g, b, i = self._amp
            out["grad_scaler"] = {"scale": self.loss_scale(), "growth_factor": g, "backoff_factor": b,
                                  "growth_interval": i, "_growth_tracker": int(self._growth.item())}
        return out

    def load_state_dict(self, state_dict):
        """Load `state_dict()` output, or the state of a torch.optim.Adam built over the same groups, in place: a
        captured graph stays valid.  Sets lr from the groups.  Raises ValueError, naming the first offending parameter,
        when the groups, shapes or states do not fit this trainer (it keeps one step count for every parameter).
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
        pairs, steps = [], []  # (trainer parameter index, source state), in group order
        for src, (_, ids) in zip(groups, self._groups):
            for i, key in zip(ids, src["params"]):
                st = state.get(key)
                if st is None or not all(k in st for k in ("step", "exp_avg", "exp_avg_sq")):
                    raise ValueError(f"no Adam state for parameter {name(i)!r}")
                shape = fp.params[i].shape
                if st["exp_avg"].shape != shape or st["exp_avg_sq"].shape != shape:
                    raise ValueError(f"parameter {name(i)!r}: state shape {tuple(st['exp_avg'].shape)}, "
                                     f"parameter shape {tuple(shape)}")
                steps.append(float(st["step"]))
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
            self.m[off:off + n].copy_(st["exp_avg"].reshape(-1))
            self.v[off:off + n].copy_(st["exp_avg_sq"].reshape(-1))
        self._t_dev.fill_(int(steps[0]))
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
        """Capture forward + loss + backward + all-reduce + Adam into one CUDA graph.  `example` fixes the
        shapes; later batches are copied into the captured static input buffers.  The warm-up steps run on the
        example batch but leave no trace: parameters, Adam moments, step count and loss scale are restored."""
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
        ts = [self.fp.flat, self.m, self.v, self._t_dev]
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
        ops.adam_flat_(self.fp.flat, self.fp.grad, self.m, self.v, 0, self._lr_host, self.betas, self.eps, self.wd,
                       grad_scale=1.0 / self.world, lr_scale_per_elem=self._lr_scale, step_dev=self._t_dev,
                       lr_dev=self._lr_dev, loss_scale_dev=divisor, found_inf_dev=self._found_inf)
        if self._scale_dev is not None:  # GradScaler.update AFTER the step: the gradients carry the old scale
            g, b, i = self._amp
            ops.amp_update(self._found_inf, None, self._scale_dev, self._growth, g, b, i)
        self.calls += 1
        return loss.detach(), losses


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
