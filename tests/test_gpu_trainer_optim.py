"""GPU: the flat SGD / AdamW / RMSprop kernels against torch.optim.<X>(foreach=False) with LR groups, GradScaler, an
overflow step and clipping; MatcherTrainer(optimizer=X) against plain autograd + torch.optim.X; and fine-tuning runs
(opt_regexp) that must leave frozen parameters bit-unchanged, match a plain autograd loop over the same frozen model and
launch no weight-gradient GEMM for a frozen layer."""
import pytest
import torch

from gluefactory_b200 import ops, synthetic
from gluefactory_b200.matchers.gluestick import GlueStick
from gluefactory_b200.matchers.lightglue import LightGlue
from gluefactory_b200.matchers.superglue import SuperGlue
from gluefactory_b200.trainer import OPTIMIZERS, MatcherTrainer, _resolve_optimizer, select_parameters
from tests.util import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"

RULES = [
    ("adamw", {"weight_decay": 0.05}),
    ("sgd", {}),
    ("sgd", {"momentum": 0.9, "dampening": 0.1, "weight_decay": 1e-3}),
    ("sgd", {"momentum": 0.9, "nesterov": True}),
    ("rmsprop", {}),
    ("rmsprop", {"momentum": 0.5, "centered": True, "weight_decay": 1e-3}),
]


def _rand(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, generator=g).to(DEV)


class _Flat:
    """One flat rule with the trainer's device controls: check (or clip) -> step count -> update -> GradScaler."""

    def __init__(self, name, options, p0, k, lr, clip):
        self.rule, self.o, keys, _ = _resolve_optimizer(name, lr, options)
        n = p0.numel()
        self.p, self.g = p0.clone(), torch.zeros(n, device=DEV)
        self.bufs = {key: torch.zeros(n, device=DEV) for key in keys}
        self.lr_scale = torch.ones(n, device=DEV)
        self.lr_scale[k:] = 10.0
        self.step = torch.zeros(1, device=DEV, dtype=torch.int32)
        self.scale = torch.full((1,), 1024.0, device=DEV)
        self.growth = torch.zeros(1, device=DEV, dtype=torch.int32)
        self.found, self.norm, self.div = (torch.zeros(1, device=DEV) for _ in range(3))
        self.lr_dev = torch.full((1,), lr, device=DEV)
        self.clip = clip
        self.ws = ops.flat_grad_norm_ws(n, DEV) if clip else None

    def run(self):
        if self.clip:
            ops.flat_grad_norm(self.g, self.g.numel(), 1.0, self.scale, self.clip, self.found, self.norm, self.div,
                               self.ws)
            divisor = self.div
        else:
            ops.flat_grad_check(self.g, self.found)
            divisor = self.scale
        ops.amp_update(self.found, step_dev=self.step)
        o, b = self.o, self.bufs
        common = dict(lr_scale_per_elem=self.lr_scale, lr_dev=self.lr_dev, loss_scale_dev=divisor,
                      found_inf_dev=self.found)
        if self.rule == "adamw":
            ops.adamw_flat_(self.p, self.g, b["exp_avg"], b["exp_avg_sq"], 0, 0.0, o["betas"], o["eps"],
                            o["weight_decay"], step_dev=self.step, **common)
        elif self.rule == "sgd":
            ops.sgd_flat_(self.p, self.g, b.get("momentum_buffer"), 0, 0.0, o["momentum"], o["dampening"],
                          o["nesterov"], o["weight_decay"], step_dev=self.step, **common)
        else:
            ops.rmsprop_flat_(self.p, self.g, b["square_avg"], b.get("momentum_buffer"), b.get("grad_avg"), 0.0,
                              o["alpha"], o["eps"], o["weight_decay"], o["momentum"], **common)
        ops.amp_update(self.found, None, self.scale, self.growth, 2.0, 0.5, 2)

    def state(self):
        return [self.p, self.step, self.scale, self.growth, *self.bufs.values()]


@pytest.mark.parametrize("clip", [None, 10.0])
@pytest.mark.parametrize("rule", range(len(RULES)))
def test_flat_rule_with_grad_scaler_matches_torch(rule, clip):
    """torch.optim.<X>(foreach=False) over two LR groups (factors 1 and 10) + GradScaler (+ unscale_ and
    clip_grad_norm_(error_if_nonfinite=True) with clipping), seven steps with one overflow, against the flat kernel with
    device-resident step / scale / skip flag; the same steps replayed from one captured graph give identical bits."""
    name, options = RULES[rule]
    n, k, lr = 50_003, 20_001, 2e-3
    p0 = _rand(n, 1)
    a, b = torch.nn.Parameter(p0[:k].clone()), torch.nn.Parameter(p0[k:].clone())
    opt = OPTIMIZERS[name]([{"params": [a], "lr": lr}, {"params": [b], "lr": 10 * lr}], lr=lr, foreach=False, **options)
    scaler = torch.amp.GradScaler("cuda", init_scale=1024.0, growth_factor=2.0, backoff_factor=0.5, growth_interval=2)
    scaler.scale(torch.ones(1, device=DEV))
    eager, graphed = _Flat(name, options, p0, k, lr, clip), _Flat(name, options, p0, k, lr, clip)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        graphed.run()
    mags = [1.0, 0.01, 1.0, 0.02, 1.0, 0.5, 0.01]
    for t, mag in enumerate(mags):
        g = _rand(n, 10 + t) * mag
        if t == 2:
            g[777] = float("inf")  # overflow: both skip and halve the scale
        cur = scaler.get_scale()
        a.grad, b.grad = g[:k] * cur, g[k:] * cur
        if clip:
            scaler.unscale_(opt)
            try:
                torch.nn.utils.clip_grad_norm_([a, b], max_norm=clip, error_if_nonfinite=True)
                scaler.step(opt)
            except RuntimeError:
                pass
        else:
            scaler.step(opt)
        scaler.update()
        gs = g * float(eager.scale.item())
        eager.g.copy_(gs)
        eager.run()
        graphed.g.copy_(gs)
        graph.replay()
        assert float(eager.scale.item()) == scaler.get_scale(), t
    assert int(eager.step.item()) == len(mags) - 1
    assert rel_err(eager.p, torch.cat([a.data, b.data])) < 1e-6
    # the state torch keeps, in the same layout.  The betas reach the kernel as fp32, so its 1 - beta2 is
    # 1 - fl(0.999), 1.3e-5 from torch's fl(1 - 0.999): exp_avg_sq carries that relative offset (as with Adam)
    for key, buf in eager.bufs.items():
        ref = torch.cat([opt.state[a][key].reshape(-1), opt.state[b][key].reshape(-1)])
        assert rel_err(buf, ref) < 5e-5, (key, rel_err(buf, ref))
    for x, y in zip(eager.state(), graphed.state()):
        assert torch.equal(x, y)


def _model(L=2, seed=51):
    conf = dict(synthetic.DEFAULT_CONF, n_layers=L)
    model = LightGlue(dict(conf, precision="bf16"))
    model.load_state_dict({k: v.float() for k, v in synthetic.make_weights(conf, seed=seed).items()}, strict=False)
    return model.to(DEV).train()


def _plain_step(model, opt, data):
    """Plain autograd + torch.optim; a trainable parameter autograd leaves without gradient gets zeros, as in the
    trainer's flat gradient buffer."""
    opt.zero_grad()
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    for p in model.parameters():
        if p.requires_grad and p.grad is None:
            p.grad = torch.zeros_like(p)
    opt.step()


def _assert_close(model, ref, tol):
    ps = [p for p in model.parameters() if p.requires_grad]
    rs = [r for r in ref.parameters() if r.requires_grad]
    err = rel_err(torch.cat([p.detach().reshape(-1) for p in ps]), torch.cat([r.detach().reshape(-1) for r in rs]))
    assert err < tol, err


TRAINER_RULES = [("sgd", {"momentum": 0.9}, 1e-2), ("adamw", {}, 1e-4), ("rmsprop", {"centered": True}, 1e-5)]


@pytest.mark.parametrize("rule", range(len(TRAINER_RULES)))
def test_trainer_optimizer_matches_plain_autograd(rule):
    name, options, lr = TRAINER_RULES[rule]
    data = [synthetic.to_device(synthetic.make_pairs(2, 256, seed=90 + i), DEV) for i in range(3)]
    tr = MatcherTrainer(_model(), lr=lr, optimizer=name, optimizer_options=options)
    ref = _model()
    opt = OPTIMIZERS[name](ref.parameters(), lr=lr, foreach=False, **options)
    for d in data:
        tr.step(d)
        _plain_step(ref, opt, d)
    assert tr.t == 3
    _assert_close(tr.model, ref, 1e-4)  # bf16 gradients of two schedules of the same kernels
    for key, buf in tr.state_buffers.items():
        mine = torch.cat([buf[o:o + p.numel()] for p, o in zip(tr.fp.params, tr.fp.offsets)])
        theirs = torch.cat([opt.state[p][key].reshape(-1) for p in ref.parameters()])
        assert rel_err(mine, theirs) < 1e-3, key


def _gluestick():
    model = GlueStick({"precision": "bf16"})
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=5), strict=True)
    return model.to(DEV).train()


def _superglue():
    model = SuperGlue({"weights": None, "GNN_layers": ["self", "cross"] * 2, "precision": "bf16"})
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=6), strict=True)
    return model.to(DEV).train()


FINETUNE = {
    "lightglue_heads": (lambda: _model(9), r"log_assignment|token_confidence",
                        lambda s: synthetic.make_pairs(2, 256, seed=s)),
    "lightglue_last": (lambda: _model(9), r"transformers\.[5-8]\.|log_assignment|token_confidence",
                       lambda s: synthetic.make_pairs(2, 256, seed=s)),
    "gluestick": (_gluestick, r"gnn\.layers\.1[0-7]|final", lambda s: synthetic.make_gluestick_batch(2, 256, 32, s)),
    "superglue": (_superglue, r"final_proj|bin_score", lambda s: synthetic.make_superglue_batch(2, 256, 256, s)),
}


@pytest.mark.parametrize("case", list(FINETUNE))
def test_finetune_matches_plain_autograd_and_keeps_frozen_bits(case):
    build, regexp, batch = FINETUNE[case]
    data = [synthetic.to_device(batch(100 + i), DEV) for i in range(3)]
    eager = MatcherTrainer(build(), lr=1e-4, opt_regexp=regexp)
    frozen = {n: p.detach().clone() for n, p in eager.model.named_parameters() if not p.requires_grad}
    assert frozen
    ref = build()
    select_parameters(ref, regexp)
    opt = torch.optim.Adam([p for p in ref.parameters() if p.requires_grad], lr=1e-4, foreach=False)
    graphed = MatcherTrainer(build(), lr=1e-4, opt_regexp=regexp).capture(data[0], DEV)
    for d in data:
        eager.step(d)
        graphed.step_graphed(d)
        _plain_step(ref, opt, d)
    for n, p in eager.model.named_parameters():
        if n in frozen:
            assert torch.equal(p.detach(), frozen[n]), n
    assert eager.t == 3
    _assert_close(eager.model, ref, 1e-4)
    assert torch.equal(eager.fp.flat, graphed.fp.flat) and torch.equal(eager.m, graphed.m)


def _kernels(tr, data):
    tr.step(data)  # warm-up outside the trace
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        tr.step(data)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    return sum("splitk_reduce" in n for n in names), sum("attn_bwd" in n for n in names)


def test_frozen_layers_launch_no_weight_gradient_gemm():
    """Kernel lists of one step (torch.profiler): each split-K weight-gradient GEMM ends in one splitk_reduce launch.
    Heads only: no layer's weight gradient and no attention backward.  Last four of nine layers: four ninths of the
    layers' weight-gradient GEMMs and attention backwards."""
    data = synthetic.to_device(synthetic.make_pairs(2, 256, seed=120), DEV)
    full = _kernels(MatcherTrainer(_model(9), lr=1e-4), data)
    heads = _kernels(MatcherTrainer(_model(9), lr=1e-4, opt_regexp=FINETUNE["lightglue_heads"][1]), data)
    last = _kernels(MatcherTrainer(_model(9), lr=1e-4, opt_regexp=FINETUNE["lightglue_last"][1]), data)
    assert full[0] > heads[0] > 0 and (full[0] - heads[0]) % 9 == 0, (full, heads)
    per_layer = (full[0] - heads[0]) // 9
    assert heads[1] == 0 and full[1] > 0 and full[1] % 9 == 0, (full, heads)
    assert last == (heads[0] + 4 * per_layer, 4 * full[1] // 9), (full, heads, last)
