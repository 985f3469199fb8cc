"""CPU: MatcherTrainer's optimiser choice (train.optimizer / train.optimizer_options, train.py:347-361) and parameter
selection (train.opt_regexp, train.py:125-141): state layouts equal torch.optim.<X>'s over the same groups, torch states
load and export back equal, mismatches raise, and the frozen parameters leave the gradient buffer.  The trainer is built
on a CPU module: it makes no library call before its first step."""
import re

import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.gluestick import GlueStick
from gluefactory_b200.matchers.lightglue import LightGlue
from gluefactory_b200.matchers.superglue import SuperGlue
from gluefactory_b200.trainer import _ALIGN, MatcherTrainer
from tests.test_trainer_state_cpu import _assert_same, _lr_groups

SCALINGS = [None, [(0.0, ["log_assignment"]), (10.0, ["posenc", "final_proj"])]]
CONFIGS = [
    ("sgd", {}),
    ("sgd", {"momentum": 0.9, "dampening": 0.1, "weight_decay": 1e-3}),
    ("sgd", {"momentum": 0.9, "nesterov": True, "foreach": False}),
    ("adamw", {}),
    ("adamw", {"betas": (0.8, 0.99), "eps": 1e-6, "weight_decay": 0.05, "capturable": False}),
    ("adam", {"decoupled_weight_decay": True, "weight_decay": 0.02}),
    ("rmsprop", {}),
    ("rmsprop", {"momentum": 0.5, "centered": True, "weight_decay": 1e-3, "differentiable": False}),
    ("rmsprop", {"centered": True, "alpha": 0.9}),
]
TORCH = {"sgd": torch.optim.SGD, "adam": torch.optim.Adam, "adamw": torch.optim.AdamW, "rmsprop": torch.optim.RMSprop}


def _model(n_layers=2, seed=51):
    conf = dict(synthetic.DEFAULT_CONF, n_layers=n_layers)
    model = LightGlue(dict(conf, precision="bf16"))
    model.load_state_dict({k: v.float() for k, v in synthetic.make_weights(conf, seed=seed).items()}, strict=False)
    return model.train()


def _torch_opt(name, options, lr, lr_scaling, steps, seed=0):
    model = _model()
    opt = TORCH[name](_lr_groups(model, lr, lr_scaling), lr=lr, **options)
    gen = torch.Generator().manual_seed(seed)
    for _ in range(steps):
        for p in model.parameters():
            p.grad = torch.randn(p.shape, generator=gen)
        opt.step()
    return opt


@pytest.mark.parametrize("scaling", range(len(SCALINGS)))
@pytest.mark.parametrize("config", range(len(CONFIGS)))
def test_state_layout_and_round_trip_equal_torch(config, scaling):
    name, options = CONFIGS[config]
    lr_scaling = SCALINGS[scaling]
    tr = MatcherTrainer(_model(), lr=1e-3, optimizer=name, optimizer_options=options, lr_scaling=lr_scaling)
    ref = _torch_opt(name, options, 1e-3, lr_scaling, steps=1).state_dict()
    mine = tr.state_dict()["optimizer"]
    assert mine["param_groups"] == ref["param_groups"]
    if name == "sgd":  # torch keeps no SGD state before the first step
        assert mine["state"] == {}
    else:
        assert list(mine["state"]) == list(ref["state"])
        for k, st in ref["state"].items():
            assert list(mine["state"][k]) == list(st), k
            for key, t in st.items():
                assert mine["state"][k][key].shape == t.shape and mine["state"][k][key].dtype == t.dtype, (k, key)
    # a torch state after three steps loads and exports back equal
    ref = _torch_opt(name, options, 2e-3, lr_scaling, steps=3).state_dict()
    tr.load_state_dict({"optimizer": ref})
    assert tr.lr == 2e-3
    assert tr.t == (3 if name != "sgd" else 1 if options.get("momentum") else 0)
    _assert_same(tr.state_dict()["optimizer"], ref)


def test_state_buffers_only_where_torch_keeps_state():
    def keys(name, options):
        return list(MatcherTrainer(_model(), optimizer=name, optimizer_options=options).state_buffers)

    assert keys("sgd", {}) == []
    assert keys("sgd", {"momentum": 0.5}) == ["momentum_buffer"]
    assert keys("rmsprop", {}) == ["square_avg"]
    assert keys("rmsprop", {"momentum": 0.5, "centered": True}) == ["square_avg", "momentum_buffer", "grad_avg"]
    assert keys("adamw", {}) == ["exp_avg", "exp_avg_sq"]
    tr = MatcherTrainer(_model(), optimizer="adamw")
    assert tr._opt["weight_decay"] == 0.01 and tr._rule == "adamw"  # torch's AdamW default
    assert MatcherTrainer(_model())._rule == "adam"


def test_mismatches_raise_value_error_naming_the_parameter():
    names = [n for n, _ in _model().named_parameters()]
    adam = _torch_opt("adam", {}, 1e-3, None, steps=2).state_dict()
    sgd = _torch_opt("sgd", {"momentum": 0.9}, 1e-3, None, steps=2).state_dict()
    centered = _torch_opt("rmsprop", {"centered": True}, 1e-3, None, steps=2).state_dict()
    for name, options, state in [("sgd", {"momentum": 0.9}, adam), ("sgd", {}, adam), ("rmsprop", {}, sgd),
                                 ("rmsprop", {}, centered), ("adam", {}, sgd), ("adamw", {}, centered)]:
        tr = MatcherTrainer(_model(), optimizer=name, optimizer_options=options)
        before = [b.clone() for b in tr.state_buffers.values()]
        with pytest.raises(ValueError, match=re.escape(names[0])):
            tr.load_state_dict({"optimizer": state})
        assert all(torch.equal(a, b) for a, b in zip(before, tr.state_buffers.values()))
    # SGD: a state in which only some parameters have a momentum buffer
    part = _torch_opt("sgd", {"momentum": 0.9}, 1e-3, None, steps=2).state_dict()
    del part["state"][3]
    tr = MatcherTrainer(_model(), optimizer="sgd", optimizer_options={"momentum": 0.9})
    with pytest.raises(ValueError, match=f"no SGD state.*{re.escape(names[3])}"):
        tr.load_state_dict({"optimizer": part})
    # shapes
    bad = _torch_opt("rmsprop", {}, 1e-3, None, steps=1).state_dict()
    bad["state"][2]["square_avg"] = bad["state"][2]["square_avg"].reshape(-1)[:1]
    with pytest.raises(ValueError, match=f"{re.escape(names[2])}.*shape"):
        MatcherTrainer(_model(), optimizer="rmsprop").load_state_dict({"optimizer": bad})


def test_unsupported_options_raise():
    for key in ("maximize", "amsgrad"):
        opt = "adamw" if key == "amsgrad" else "sgd"
        with pytest.raises(ValueError, match=key):
            MatcherTrainer(_model(), optimizer=opt, optimizer_options={key: True})
    with pytest.raises(ValueError, match="lbfgs"):
        MatcherTrainer(_model(), optimizer="lbfgs")
    with pytest.raises(ValueError, match="optimizer_options"):
        MatcherTrainer(_model(), optimizer="sgd", weight_decay=0.1)
    # torch's own validation of the values
    with pytest.raises(ValueError):
        MatcherTrainer(_model(), optimizer="sgd", optimizer_options={"nesterov": True})
    # explicit False is accepted, as are the implementation selectors
    MatcherTrainer(_model(), optimizer="adam", optimizer_options={"amsgrad": False, "maximize": False, "foreach": True,
                                                                  "fused": None, "capturable": True})


def _filter_parameters(model, regexp):
    """train.py:125-141 restated: the selected (name, parameter) pairs; the others are frozen."""
    params = [(n, p) for n, p in model.named_parameters() if p.requires_grad]

    def filter_fn(x):
        n, p = x
        match = re.search(regexp, n)
        if not match:
            p.requires_grad = False
        return match

    params = list(filter(filter_fn, params))
    assert len(params) > 0, regexp
    return [n for n, _ in params]


def _gluestick():
    return GlueStick({})


def _superglue():
    return SuperGlue({"weights": None, "GNN_layers": ["self", "cross"] * 2})


PATTERNS = [
    (lambda: _model(9), r"log_assignment|token_confidence"),
    (lambda: _model(9), r"transformers\.[5-8]\.|log_assignment|token_confidence"),
    (_gluestick, r"gnn\.layers\.1[0-7]|final"),
    (_superglue, r"final_proj|bin_score"),
]


@pytest.mark.parametrize("case", range(len(PATTERNS)))
def test_opt_regexp_selects_as_filter_parameters(case):
    build, regexp = PATTERNS[case]
    ref = build()
    selected = _filter_parameters(ref, regexp)
    model = build()
    frozen_by_caller = next(n for n, _ in model.named_parameters() if n not in selected)
    tr = MatcherTrainer(model, opt_regexp=regexp)
    assert [n for n, p in model.named_parameters() if p.requires_grad] == selected
    assert [tr.fp._names[id(p)] for p in tr.fp.params] == selected
    # the gradient buffer, the optimiser state and the lr vector cover the trainable elements only
    aligned = lambda k: (k + _ALIGN - 1) // _ALIGN * _ALIGN  # noqa: E731
    n_train = sum(aligned(p.numel()) for p in tr.fp.params)
    assert tr.fp.numel == n_train == tr.fp.grad.numel() == tr.m.numel()
    assert tr.fp.numel_all == n_train + sum(aligned(p.numel()) for p in tr.fp.frozen)
    assert all(p.grad is None for p in tr.fp.frozen)
    # frozen parameters are views of the flat buffer, behind the trainable ones
    for p, off in zip(tr.fp.frozen, tr.fp.frozen_offsets):
        assert off >= n_train and p.data_ptr() == tr.fp.flat.data_ptr() + 4 * off
    # optimiser groups hold the trainable parameters only (pack_lr_parameters over the filtered list)
    groups = tr.state_dict()["optimizer"]["param_groups"]
    assert sum(len(g["params"]) for g in groups) == len(selected)
    # a parameter frozen by the caller before construction is treated the same way
    model = build()
    dict(model.named_parameters())[frozen_by_caller].requires_grad_(False)
    tr = MatcherTrainer(model)
    assert frozen_by_caller not in [tr.fp._names[id(p)] for p in tr.fp.params]


def test_opt_regexp_without_match_raises_and_freezes_nothing():
    model = _model()
    with pytest.raises(ValueError, match="matches no"):
        MatcherTrainer(model, opt_regexp=r"^matcher\.")  # the pipeline's prefix is not part of the model's names
    assert all(p.requires_grad for p in model.parameters())
