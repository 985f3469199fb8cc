"""CPU: MatcherTrainer.state_dict() / load_state_dict() speak torch.optim.Adam's and torch.amp.GradScaler's formats
(utils/experiments.py:113-118 saves optimizer.state_dict(), train.py:379-382 restores it) over the optimiser groups of
train.py:177-196.  The trainer is built on a CPU module: it makes no library call before its first step."""
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.lightglue import LightGlue
from gluefactory_b200.trainer import MatcherTrainer

SCALINGS = [None, [(100, ["posenc"])], [(0.0, ["log_assignment"]), (10.0, ["posenc", "final_proj"])]]


def _model(seed=51):
    conf = dict(synthetic.DEFAULT_CONF, n_layers=2)
    model = LightGlue(dict(conf, precision="bf16"))
    model.load_state_dict({k: v.float() for k, v in synthetic.make_weights(conf, seed=seed).items()}, strict=False)
    return model.train()


def _lr_groups(model, lr, lr_scaling):
    """The groups train.py builds for its optimiser: one per distinct factor, in order of first appearance over the
    trainable parameters; a parameter takes the factor of the first filter its name contains."""
    rules = [(f, factor) for factor, filters in (lr_scaling or []) for f in filters]
    groups = {}
    for n, p in model.named_parameters():
        if p.requires_grad:
            factor = next((factor for f, factor in rules if f in n), 1)
            groups.setdefault(factor, []).append(p)
    return [{"lr": factor * lr, "params": ps} for factor, ps in groups.items()]


def _torch_adam(model, lr, lr_scaling, steps, seed=0):
    opt = torch.optim.Adam(_lr_groups(model, lr, lr_scaling), lr=lr, weight_decay=0.01)
    gen = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        for p in model.parameters():
            p.grad = torch.randn(p.shape, generator=gen)
        opt.step()
    return opt


def _assert_same(a, b, path="sd"):
    if isinstance(a, dict):
        assert isinstance(b, dict) and list(a) == list(b), (path, list(a), list(b))
        for k in a:
            _assert_same(a[k], b[k], f"{path}[{k!r}]")
    elif isinstance(a, (list, tuple)):
        assert type(a) is type(b) and len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _assert_same(x, y, f"{path}[{i}]")
    elif torch.is_tensor(a):
        assert torch.is_tensor(b) and a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), path
    else:
        assert type(a) is type(b) and a == b, (path, a, b)


@pytest.mark.parametrize("scaling", range(len(SCALINGS)))
def test_state_dict_has_the_layout_of_torch_adam(scaling):
    lr_scaling = SCALINGS[scaling]
    tr = MatcherTrainer(_model(), lr=1e-3, weight_decay=0.01, lr_scaling=lr_scaling)
    ref = _torch_adam(_model(), 1e-3, lr_scaling, steps=1).state_dict()
    sd = tr.state_dict()
    assert list(sd) == ["optimizer"]
    mine = sd["optimizer"]
    assert mine["param_groups"] == ref["param_groups"]
    assert list(mine["state"]) == list(ref["state"])
    for k, st in ref["state"].items():
        assert list(mine["state"][k]) == list(st)
        for key, t in st.items():
            assert mine["state"][k][key].shape == t.shape and mine["state"][k][key].dtype == t.dtype, (k, key)
    assert float(mine["state"][0]["step"]) == 0.0


@pytest.mark.parametrize("scaling", range(len(SCALINGS)))
def test_torch_adam_state_loads_and_exports_back_equal(scaling):
    lr_scaling = SCALINGS[scaling]
    model = _model()
    tr = MatcherTrainer(model, lr=5e-4, weight_decay=0.01, lr_scaling=lr_scaling)
    ref = _torch_adam(_model(), 2e-3, lr_scaling, steps=3).state_dict()
    tr.load_state_dict({"optimizer": ref})
    assert tr.t == 3 and tr.lr == 2e-3
    _assert_same(tr.state_dict()["optimizer"], ref)
    # the copies are not views of the trainer's buffers
    out = tr.state_dict()["optimizer"]["state"][0]["exp_avg"]
    out.add_(1.0)
    assert not torch.equal(tr.state_dict()["optimizer"]["state"][0]["exp_avg"], out)


def test_save_load_round_trip_is_exact(tmp_path):
    tr = MatcherTrainer(_model(), lr=1e-3, loss_scale=512.0, growth_interval=7, lr_scaling=SCALINGS[1])
    tr.load_state_dict({"optimizer": _torch_adam(_model(), 1e-3, SCALINGS[1], steps=2).state_dict()})
    tr._scale_dev.fill_(128.0)
    tr._growth.fill_(3)
    sd = tr.state_dict()
    assert sd["grad_scaler"] == {"scale": 128.0, "growth_factor": 2.0, "backoff_factor": 0.5, "growth_interval": 7,
                                 "_growth_tracker": 3}
    torch.save(sd, tmp_path / "opt.pt")
    back = torch.load(tmp_path / "opt.pt", weights_only=True)
    _assert_same(back, sd)
    fresh = MatcherTrainer(_model(), lr=1.0, loss_scale=512.0, growth_interval=7, lr_scaling=SCALINGS[1])
    fresh.load_state_dict(back)
    _assert_same(fresh.state_dict(), sd)
    assert fresh.loss_scale() == 128.0 and fresh.t == 2


def _names(model):
    return [n for n, p in model.named_parameters() if p.requires_grad]


def test_mismatches_raise_value_error_naming_the_parameter():
    model = _model()
    names = _names(model)
    tr = MatcherTrainer(model, lr=1e-3, lr_scaling=SCALINGS[1], loss_scale=64.0)
    good = _torch_adam(_model(), 1e-3, SCALINGS[1], steps=2).state_dict()
    before = (tr.m.clone(), tr.v.clone(), tr.t, tr.lr)

    def bad(edit):
        sd = _torch_adam(_model(), 1e-3, SCALINGS[1], steps=2).state_dict()
        edit(sd)
        return sd

    # group count: the state of a run without LR groups
    one_group = _torch_adam(_model(), 1e-3, None, steps=1).state_dict()
    with pytest.raises(ValueError, match="groups"):
        tr.load_state_dict({"optimizer": one_group})
    order = [names[i] for _, ids in tr._groups for i in ids]  # parameters in group order
    # group sizes: the first parameter of the second group moved into the first
    def move(sd):
        sd["param_groups"][0]["params"].append(sd["param_groups"][1]["params"].pop(0))
    with pytest.raises(ValueError, match=f"groups.*{order[len(tr._groups[0][1])]}"):
        tr.load_state_dict({"optimizer": bad(move)})
    k = 3
    def shape(sd):
        sd["state"][k]["exp_avg"] = sd["state"][k]["exp_avg"].reshape(-1)[:1]
    def missing(sd):
        del sd["state"][k]
    def steps(sd):
        sd["state"][k]["step"] = torch.tensor(7.0)
    for edit, what in [(shape, "shape"), (missing, "no Adam state"), (steps, "step")]:
        with pytest.raises(ValueError, match=f"{what}.*{order[k]}|{order[k]}.*{what}"):
            tr.load_state_dict({"optimizer": bad(edit)})
    with pytest.raises(ValueError, match="growth_factor"):
        tr.load_state_dict({"optimizer": good, "grad_scaler": {"scale": 8.0, "growth_factor": 4.0,
                                                               "backoff_factor": 0.5, "growth_interval": 2000,
                                                               "_growth_tracker": 0}})
    # a refused state changes nothing
    assert torch.equal(tr.m, before[0]) and torch.equal(tr.v, before[1]) and (tr.t, tr.lr) == before[2:]
    assert tr.loss_scale() == 64.0
    tr.load_state_dict({"optimizer": good})
    assert tr.t == 2


def test_clip_grad_falsy_disables_clipping():
    for off in (None, 0, 0.0):
        assert MatcherTrainer(_model(), clip_grad=off)._max_norm is None
    assert MatcherTrainer(_model(), clip_grad=10)._max_norm == 10.0
