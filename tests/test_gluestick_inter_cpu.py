"""CPU: GlueStick intermediate line supervision (`inter_supervision`).  The fp64 oracle (tests/gluestick_inter_oracle.py)
against the fixture produced by the unmodified reference (tests/golden/gluestick_inter_l8_n160.npz,
scripts/make_gluestick_inter_golden.py), the plugin's state_dict key order against the reference's recorded orders,
the configurations it refuses, and the unchanged layout without it.  The numerics run on the GPU
(tests/test_gpu_gluestick_inter.py)."""
import ast
import os

import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.gluestick import GlueStick
from tests.util import GOLDEN, check_grad_summary

NAME = "gluestick_inter_l8_n160"


def load_golden():
    g = dict(np.load(os.path.join(GOLDEN, NAME + ".npz"), allow_pickle=False))
    conf = ast.literal_eval(str(g["meta|conf"]))
    B, N, L, seed = (int(g["meta|" + k]) for k in ("B", "N", "L", "seed"))
    return g, conf, B, N, L, seed


def test_oracle_matches_reference_golden():
    from tests import gluestick_inter_oracle as O

    g, conf, B, N, L, seed = load_golden()
    assert conf["inter_supervision"] == [0, 2] and conf["loss"]["inter_supervision"] == [0.3, 0.6]
    w = {k: (v.double() if v.is_floating_point() else v)
         for k, v in synthetic.make_gluestick_weights(GlueStick(dict(conf)).state_dict(), seed=seed).items()}
    params = {k: v.requires_grad_(True) for k, v in w.items() if v.is_floating_point() and "running_" not in k}
    ww = {**w, **params}
    data = synthetic.make_gluestick_batch(B, N, L, seed + 1, dtype=torch.float64)
    stats = {}
    pred = O.gluestick_forward(ww, data, conf, bn_stats=stats)
    losses = O.gluestick_loss(ww, pred, data, conf)
    losses["total"].mean().backward()
    pred = {**pred, **O.point_log_assignment_summary(pred["log_assignment"])}
    assert {k[len("pred|"):] for k in g if k.startswith("pred|")} <= set(pred)
    for k in (k[len("pred|"):] for k in g if k.startswith("pred|")):
        if "matches" in k and "scores" not in k:
            assert np.array_equal(pred[k].numpy(), g["pred|" + k]), k
        else:
            np.testing.assert_allclose(pred[k].detach().numpy(), g["pred|" + k], rtol=1e-9, atol=1e-9, err_msg=k)
    assert set(losses) == {k[len("loss|"):] for k in g if k.startswith("loss|")}
    assert {"line_0_assignment_nll", "line_2_assignment_nll"} <= set(losses)
    for k, v in losses.items():
        np.testing.assert_allclose(v.detach().numpy(), g["loss|" + k], rtol=1e-9, atol=1e-12, err_msg=k)
    assert {k for k in params if k.startswith("inter_line_proj.")} == {
        f"inter_line_proj.{i}.{p}" for i in (0, 1) for p in ("weight", "bias")}
    for k, p in params.items():
        if float(g[f"grad|{k}|norm"]) < 1e-9:  # a conv bias in front of a BatchNorm: zero in theory, rounding noise
            assert p.grad.norm().item() < 1e-8, k
            continue
        check_grad_summary(g, k, p.grad, rtol=1e-9)
    # running statistics: momentum 0.1, one update per call (image 0 then image 1)
    assert {k[len("bn|"):].rsplit(".", 1)[0] for k in g if k.startswith("bn|")} == set(stats)
    for name, calls in stats.items():
        rm, rv = torch.zeros_like(calls[0][0]), torch.ones_like(calls[0][1])
        for mean, var_unbiased in calls:
            rm, rv = 0.9 * rm + 0.1 * mean, 0.9 * rv + 0.1 * var_unbiased
        np.testing.assert_allclose(rm.numpy(), g["bn|" + name + ".running_mean"], rtol=1e-9, atol=1e-12, err_msg=name)
        np.testing.assert_allclose(rv.numpy(), g["bn|" + name + ".running_var"], rtol=1e-9, atol=1e-12, err_msg=name)


def test_inter_weights_are_indexed_by_position_not_block():
    """The fixture's total is the sum of the five NLL terms with weights 1, 1, 0.3 (block 0) and 0.6 (block 2)."""
    g, *_ = load_golden()
    total = (g["loss|assignment_nll"] + g["loss|line_assignment_nll"] + 0.3 * g["loss|line_0_assignment_nll"]
             + 0.6 * g["loss|line_2_assignment_nll"])
    np.testing.assert_allclose(g["loss|total"], total, rtol=1e-12)


def test_state_dict_key_order_equals_reference():
    """The reference's key order (recorded in the fixture) for the fixture's configuration and for the matcher section of
    configs/superpoint+lsd+gluestick-homography.yaml; glue-factory's optimiser checkpoints index parameters in that
    order.  Shapes of the fixture's full-size gradients too."""
    g, conf, *_ = load_golden()
    sd = GlueStick(dict(conf)).state_dict()
    assert list(sd) == [str(k) for k in g["meta|ref_keys"]]
    for k in g:
        if k.startswith("grad|") and k.endswith("|full"):
            assert tuple(sd[k[len("grad|"):-len("|full")]].shape) == g[k].shape, k
    hconf = ast.literal_eval(str(g["meta|homography_conf"]))
    assert hconf["inter_supervision"] == [2, 5] and len(hconf["GNN_layers"]) == 18 and hconf["checkpointed"]
    model = GlueStick(dict(hconf))
    assert list(model.state_dict()) == [str(k) for k in g["meta|homography_ref_keys"]]
    assert model.layer2idx == {2: 0, 5: 1} and len(model.inter_line_proj) == 2
    assert tuple(model.inter_line_proj[1].weight.shape) == (256, 256, 1)


def test_without_inter_supervision_the_state_dict_is_unchanged():
    """inter_supervision None (the default) registers nothing new: the same keys, shapes and, from the same seed, the same
    initial values as the modules it shares with a model that has two intermediate heads."""
    _, conf, *_ = load_golden()
    plain = dict(conf, inter_supervision=None)
    torch.manual_seed(0)
    base = GlueStick(plain).state_dict()
    torch.manual_seed(0)
    inter = GlueStick(dict(conf)).state_dict()
    assert not hasattr(GlueStick(plain), "inter_line_proj")
    assert list(base) == [k for k in inter if not k.startswith("inter_line_proj.")]
    for k, v in base.items():
        assert torch.equal(v, inter[k]), k
    assert GlueStick.default_conf["inter_supervision"] is None


@pytest.mark.parametrize("layers,inter", [
    (["self", "cross"] * 4, [4]),          # past the last block
    (["self", "cross"] * 4, [-1]),
    (["self", "cross"] * 4, [0, 7]),       # 7 is a layer index, not a block index
    (["self", "cross"] * 4, ["2"]),
    (["self", "cross"] * 4, [True]),
    (["cross", "self", "self", "cross"], [2]),
    (["self", "self", "self", "cross"], [0]),  # block 0 holds two self layers
])
def test_inter_supervision_entry_that_is_not_a_cross_block_is_refused(layers, inter):
    with pytest.raises(ValueError, match="block index"):
        GlueStick({"GNN_layers": layers, "inter_supervision": inter})


def test_cross_blocks_are_accepted_in_any_layer_pattern():
    assert GlueStick({"GNN_layers": ["cross", "self", "self", "cross"], "inter_supervision": [0, 1]}).layer2idx == {0: 0, 1: 1}


@pytest.mark.parametrize("inter,weights", [([0, 1, 2], [0.3, 0.6]), ([1], []), ([1], None)])
def test_too_few_loss_weights_are_refused(inter, weights):
    with pytest.raises(ValueError, match="fewer weights"):
        GlueStick({"GNN_layers": ["self", "cross"] * 4, "inter_supervision": inter, "loss": {"inter_supervision": weights}})


@pytest.mark.parametrize("key", ["line_attention", "skip_init"])
def test_line_attention_and_skip_init_are_still_not_built(key):
    with pytest.raises(NotImplementedError, match=key):
        GlueStick({key: True, "inter_supervision": [2, 5]})
