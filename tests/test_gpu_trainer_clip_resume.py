"""GPU: gradient-norm clipping on the device (lgb200_flat_grad_norm; train.py:501-512 clip_grad with
clip_grad_norm_(error_if_nonfinite=True) after GradScaler.unscale_) and resuming the flat-buffer trainer from
checkpoints in torch's optimiser formats (utils/experiments.py:113-118, train.py:379-382)."""
import pytest
import torch

from gluefactory_b200 import ops, synthetic
from gluefactory_b200.matchers.lightglue import LightGlue
from gluefactory_b200.trainer import MatcherTrainer
from tests.util import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _model(seed=51):
    conf = dict(synthetic.DEFAULT_CONF, n_layers=2)
    model = LightGlue(dict(conf, precision="bf16"))
    model.load_state_dict({k: v.float() for k, v in synthetic.make_weights(conf, seed=seed).items()}, strict=False)
    return model.to(DEV).train()


def _rand(n, seed):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(n, generator=g).to(DEV)


class _Norm:
    """flat_grad_norm with its outputs, over g[:n] plus four checked-only slots (the trainer's loss slot)."""

    def __init__(self, n):
        self.n = n
        self.found, self.norm, self.div = (torch.full((1,), -1.0, device=DEV) for _ in range(3))
        self.ws = ops.flat_grad_norm_ws(n, DEV)

    def __call__(self, g, grad_scale, scale, max_norm):
        ops.flat_grad_norm(g, self.n, grad_scale, scale, max_norm, self.found, self.norm, self.div, self.ws)
        return self.found.clone(), self.norm.clone(), self.div.clone()


@pytest.mark.parametrize("n", [1, 3, 50_003, 12_000_003])
def test_grad_norm_kernel(n):
    g = torch.zeros(n + 4, device=DEV)
    g[:n] = _rand(n, n) * 300.0
    scale = torch.full((1,), 1024.0, device=DEV)
    gs, s = 0.5, 1024.0
    ref = (g[:n].double() * gs / s).norm().item()
    run = _Norm(n)
    for max_norm in (0.25 * ref, 4.0 * ref):  # clipping engages / the coefficient clamps to 1
        found, norm, div = run(g, gs, scale, max_norm)
        assert found.item() == 0.0
        assert abs(norm.item() - ref) <= 1e-6 * ref, (norm.item(), ref)
        coef = (torch.tensor(max_norm, dtype=torch.float32, device=DEV) / (norm + 1e-6)).clamp(max=1.0)
        assert torch.equal(div, scale / coef), (div.item(), (scale / coef).item())
        if max_norm > ref:
            assert div.item() == s
        # two calls and a graph replay: bit-identical
        again = run(g, gs, scale, max_norm)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            run(g, gs, scale, max_norm)
        graph.replay()
        replayed = (run.found.clone(), run.norm.clone(), run.div.clone())
        for other in (again, replayed):
            assert all(torch.equal(a, b) for a, b in zip((found, norm, div), other))
    # no device loss scale: s = 1
    _, norm, div = run(g, gs, None, 0.5 * ref * s)
    assert abs(norm.item() - ref * s) <= 1e-6 * ref * s and abs(div.item() - 2.0) < 1e-5
    # any non-finite value at the first element, the last normed element or the loss slot skips the step
    for i in (0, n - 1, n):
        for bad in (float("inf"), float("nan")):
            h = g.clone()
            h[i] = bad
            found, _, div = run(h, gs, scale, 0.25 * ref)
            assert found.item() == 1.0, (i, bad)
            assert div.item() == s
    # finite values whose norm overflows fp32
    h = torch.full((n + 4,), 3e38, device=DEV)
    h[n:] = 0.0
    found, norm, _ = run(h, 4.0, None, 1.0)
    assert found.item() == 1.0 and norm.item() == float("inf")


def test_clipped_adam_with_grad_scaler_matches_torch():
    """torch.optim.Adam + GradScaler + unscale_ + clip_grad_norm_(error_if_nonfinite=True), skipping on its error, as
    train.py:501-512, against flat_grad_norm -> amp_update -> adam_flat_ with the divisor: steps that clip, steps whose
    coefficient clamps to 1 and an overflowing step."""
    n, max_norm = 50_003, 10.0
    p = _rand(n, 1)
    ref = torch.nn.Parameter(p.clone())
    opt = torch.optim.Adam([ref], lr=2e-3, weight_decay=0.01)
    scaler = torch.amp.GradScaler("cuda", init_scale=1024.0, growth_factor=2.0, backoff_factor=0.5, growth_interval=2)
    m, v = torch.zeros_like(p), torch.zeros_like(p)
    step = torch.zeros(1, device=DEV, dtype=torch.int32)
    scale = torch.full((1,), 1024.0, device=DEV)
    growth = torch.zeros(1, device=DEV, dtype=torch.int32)
    lr_dev = torch.full((1,), 2e-3, device=DEV)
    run = _Norm(n)
    scaler.scale(torch.ones(1, device=DEV))
    kinds = []
    for t, mag in enumerate([1.0, 0.01, 1.0, 0.02, 1.0, 0.5, 0.01]):
        g = _rand(n, 10 + t) * mag  # |g| ~ 224 mag: clipped when mag = 1 or 0.5, coefficient 1 when small
        if t == 2:
            g[777] = float("inf")
        cur = scaler.get_scale()
        ref.grad = g.clone() * cur
        scaler.unscale_(opt)
        try:
            torch.nn.utils.clip_grad_norm_([ref], max_norm=max_norm, error_if_nonfinite=True)
            scaler.step(opt)
        except RuntimeError:
            pass
        scaler.update()
        gs = g * float(scale.item())
        found, norm, div = run(gs, 1.0, scale, max_norm)
        ops.amp_update(run.found, step_dev=step)
        ops.adam_flat_(p, gs, m, v, 0, 0.0, weight_decay=0.01, step_dev=step, lr_dev=lr_dev, loss_scale_dev=run.div,
                       found_inf_dev=run.found)
        ops.amp_update(run.found, None, scale, growth, 2.0, 0.5, 2)
        assert float(scale.item()) == scaler.get_scale(), (t, float(scale.item()), scaler.get_scale())
        kinds.append("inf" if found.item() else ("clip" if norm.item() > max_norm else "unclipped"))
    assert set(kinds) == {"inf", "clip", "unclipped"}, kinds
    assert int(step.item()) == 6
    assert rel_err(p, ref.data) < 1e-6


def _batches(k, seed=70):
    return [synthetic.to_device(synthetic.make_pairs(2, 256, seed=seed + i), DEV) for i in range(k)]


def _run(tr, data, graphed):
    if graphed and getattr(tr, "_graph", None) is None:
        tr.capture(data[0], DEV)
    for d in data:
        (tr.step_graphed if graphed else tr.step)(d)
    return tr


@pytest.mark.parametrize("graphed", [False, True])
def test_trainer_clip(graphed):
    data = _batches(2)
    # a max_norm no gradient reaches: the divisor is exactly 1 and the update is bit-identical to no clipping
    plain = _run(MatcherTrainer(_model(), lr=1e-3), data, graphed)
    wide = _run(MatcherTrainer(_model(), lr=1e-3, clip_grad=1e30), data, graphed)
    assert torch.equal(plain.fp.flat, wide.fp.flat) and torch.equal(plain.m, wide.m) and torch.equal(plain.v, wide.v)
    assert wide._adam_div.item() == 1.0
    # a small max_norm: torch Adam applied to clip_grad_norm_ of the same steps' flat gradients
    tr = MatcherTrainer(_model(), lr=1e-3, clip_grad=0.05)
    if graphed:
        tr.capture(data[0], DEV)
    ref = torch.nn.Parameter(tr.fp.flat.clone())
    opt = torch.optim.Adam([ref], lr=1e-3)
    for d in data:
        (tr.step_graphed if graphed else tr.step)(d)
        ref.grad = tr.fp.grad.clone()
        true = ref.grad.double().norm().item()
        assert abs(tr._grad_norm.item() - true) <= 1e-6 * true and true > 0.05
        torch.nn.utils.clip_grad_norm_([ref], max_norm=0.05, error_if_nonfinite=True)
        opt.step()
    assert tr.t == 2 and rel_err(tr.fp.flat, ref.data) < 1e-6
    # a NaN batch is skipped with clipping on (train.py:477-480)
    bad = dict(data[1], descriptors0=data[1]["descriptors0"].clone())
    bad["descriptors0"][1, 3, 5] = float("nan")
    before = (tr.fp.flat.clone(), tr.m.clone(), tr.v.clone())
    loss, _ = (tr.step_graphed if graphed else tr.step)(bad)
    assert not torch.isfinite(loss) and tr.skipped_last_step() and tr.t == 2
    assert torch.equal(tr.fp.flat, before[0]) and torch.equal(tr.m, before[1]) and torch.equal(tr.v, before[2])
    (tr.step_graphed if graphed else tr.step)(data[0])
    assert tr.t == 3 and not tr.skipped_last_step() and not torch.equal(tr.fp.flat, before[0])


CONF = dict(lr=1e-3, loss_scale=1024.0, growth_interval=3, lr_scaling=[(10.0, ["posenc"])], clip_grad=1.0)


@pytest.mark.parametrize("capture_first", [False, True])
def test_resume_is_bit_identical(tmp_path, capture_first):
    """A trains 4 steps; B trains 2, is saved and loaded into a fresh C that trains the other 2: C ends where A does."""
    data = _batches(4)
    a = _run(MatcherTrainer(_model(), **CONF), data, graphed=False)
    b = _run(MatcherTrainer(_model(), **CONF), data[:2], graphed=False)
    torch.save({"model": b.model.state_dict(), **b.state_dict()}, tmp_path / "checkpoint.tar")
    c = MatcherTrainer(_model(seed=99), **CONF)
    if capture_first:  # the load writes in place: the captured graph keeps running on the loaded state
        c.capture(data[0], DEV)
    ck = torch.load(tmp_path / "checkpoint.tar", weights_only=True)
    c.model.load_state_dict(ck["model"])
    c.load_state_dict(ck)
    assert torch.equal(c.fp.flat, b.fp.flat) and c.t == 2 and c.loss_scale() == b.loss_scale()
    for d in data[2:]:
        (c.step_graphed if capture_first else c.step)(d)
    assert a.t == c.t == 4
    assert a.loss_scale() == c.loss_scale() == 2048.0  # grew after 3 clean steps: the growth tracker was restored
    for x, y in [(a.fp.flat, c.fp.flat), (a.m, c.m), (a.v, c.v)]:
        assert torch.equal(x, y), rel_err(y, x)


def _lr_groups(model, lr, lr_scaling):
    rules = [(f, factor) for factor, filters in lr_scaling for f in filters]
    groups = {}
    for n, p in model.named_parameters():
        if p.requires_grad:
            groups.setdefault(next((factor for f, factor in rules if f in n), 1), []).append(p)
    return [{"lr": factor * lr, "params": ps} for factor, ps in groups.items()]


def _torch_step(model, opt, data):
    opt.zero_grad()
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    for p in model.parameters():  # the trainer's flat gradient holds zeros where autograd leaves None
        if p.grad is None:
            p.grad = torch.zeros_like(p)
    opt.step()


SCALING = [(10.0, ["posenc"])]


def test_cross_load_with_torch_adam():
    data = _batches(3, seed=80)
    # torch.optim.Adam -> trainer
    tm = _model()
    opt = torch.optim.Adam(_lr_groups(tm, 1e-4, SCALING), lr=1e-4)
    for d in data[:2]:
        _torch_step(tm, opt, d)
    tr = MatcherTrainer(_model(seed=99), lr=1.0, lr_scaling=SCALING)
    tr.model.load_state_dict(tm.state_dict())
    tr.load_state_dict({"optimizer": opt.state_dict()})
    assert tr.t == 2 and tr.lr == 1e-4
    _torch_step(tm, opt, data[2])
    tr.step(data[2])
    _assert_close(tr.model, tm)
    # trainer -> torch.optim.Adam
    tr = _run(MatcherTrainer(_model(), lr=1e-4, lr_scaling=SCALING), data[:2], graphed=False)
    tm = _model(seed=99)
    tm.load_state_dict(tr.model.state_dict())
    opt = torch.optim.Adam(_lr_groups(tm, 1.0, SCALING), lr=1.0)
    opt.load_state_dict(tr.state_dict()["optimizer"])
    assert [g["lr"] for g in opt.param_groups] == [g["lr"] for g in _lr_groups(tm, 1e-4, SCALING)]
    _torch_step(tm, opt, data[2])
    tr.step(data[2])
    _assert_close(tr.model, tm)


def _assert_close(model, ref):
    ps, rs = list(model.parameters()), list(ref.parameters())
    err = rel_err(torch.cat([p.detach().reshape(-1) for p in ps]), torch.cat([r.detach().reshape(-1) for r in rs]))
    worst = max((rel_err(p, r), n) for (n, r), p in zip(ref.named_parameters(), ps))
    assert err < 1e-5, (err, worst)
