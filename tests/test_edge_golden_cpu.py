"""CPU: the fp64 oracles against the loss-setting and label-extreme fixtures (tests/golden/edge_*.npz,
scripts/make_edge_golden.py: the unmodified reference matchers in fp64, training mode, with loss weights away from their
defaults and labels edited into empty classes).  This pins the oracles at those settings before
tests/test_gpu_pair_edges.py uses them at shapes no fixture has.  The fixtures are also checked for what that GPU file
relies on: every empty label class and every asymmetric loss weight is present."""
import ast
import os

import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.gluestick import GlueStick
from gluefactory_b200.matchers.superglue import SuperGlue
from oracle import lightglue_oracle as O
from tests import gluestick_inter_oracle as GO
from tests import superglue_oracle as SO
from tests.util import GOLDEN, check_grad_summary

LG = ["edge_lg_a_labels", "edge_lg_b_m1_n65", "edge_lg_c_m63_n130"]
RTOL, ATOL = 1e-11, 1e-12  # both sides are fp64 evaluations of the same sums, in other orders
# The reference's token-confidence BCE takes an fp32 target (`correct.float()`, lightglue.py:90-92) and so returns fp32:
# LightGlue's `confidence`, the `total` it is added to and the token heads' gradients carry fp32 rounding, a few units
# of 2^-24 relative.
RTOL_FP32_TERM = 4 * 2.0 ** -24


def load(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False))
    return g, ast.literal_eval(str(g["meta|conf"]))


def _labels(g, data, keys=("gt_assignment", "gt_matches0", "gt_matches1")):
    for k in keys:
        data[k] = torch.from_numpy(g["label|" + k])
    return data


def lightglue_case(name, dtype=torch.float64):
    """(golden, conf, weights, data) with the fixture's labels."""
    g, conf = load(name)
    B, M, N, seed = (int(g["meta|" + k]) for k in ("B", "M", "N", "seed"))
    w = {k: v.to(dtype) for k, v in synthetic.make_weights(conf, seed=seed).items()}
    data = synthetic.make_pairs(B, N, seed=seed + 1, D=conf["input_dim"], M=M, dtype=dtype)
    return g, conf, w, _labels(g, data)


def _close(got, g, key):
    np.testing.assert_allclose(got.detach().numpy(), g[key], rtol=RTOL, atol=ATOL, err_msg=key)


def _check_losses(losses, g, fp32_terms=()):
    assert set(losses) == {k[len("loss|"):] for k in g if k.startswith("loss|")}
    for k, v in losses.items():
        v = v if torch.is_tensor(v) else torch.tensor(v)
        if k in fp32_terms:
            np.testing.assert_allclose(v.detach().numpy(), g["loss|" + k], rtol=RTOL_FP32_TERM, err_msg=k)
        else:
            _close(v, g, "loss|" + k)


def _check_grads(g, params):
    for k, p in params.items():
        if float(g[f"grad|{k}|norm"]) < 1e-9:  # a conv bias in front of a BatchNorm: zero in theory, rounding noise
            assert p.grad.norm().item() < 1e-8, k
            continue
        check_grad_summary(g, k, p.grad, rtol=RTOL_FP32_TERM if k.startswith("token_confidence.") else RTOL)


@pytest.mark.parametrize("name", LG)
def test_lightglue_oracle_matches_edge_fixture(name):
    g, conf, w, data = lightglue_case(name)
    w = {k: v.requires_grad_(True) for k, v in w.items()}
    pred = O.lightglue_forward(w, data, conf)
    losses = O.lightglue_loss(w, pred, data, conf)
    losses["total"].mean().backward()
    for k in ("matches0", "matches1"):
        assert np.array_equal(pred[k].numpy(), g["pred|" + k]), k
    for k in ("matching_scores0", "matching_scores1", "log_assignment"):
        _close(pred[k], g, "pred|" + k)
    _check_losses(losses, g, fp32_terms=("confidence", "total"))
    _check_grads(g, w)


def test_superglue_oracle_matches_edge_fixture():
    g, conf = load("edge_sg_labels")
    B, M, N, seed = (int(g["meta|" + k]) for k in ("B", "M", "N", "seed"))
    w = {k: (v.double() if v.is_floating_point() else v)
         for k, v in synthetic.make_gluestick_weights(SuperGlue(dict(conf)).state_dict(), seed=seed).items()}
    params = {k: w[k].clone().requires_grad_(True) for k, _ in SuperGlue(dict(conf)).named_parameters()}
    data = _labels(g, synthetic.make_superglue_batch(B, M, N, seed + 1, dtype=torch.float64))
    stats = {}
    pred = SO.superglue_forward({**w, **params}, data, conf, stats)
    losses = SO.superglue_loss({**w, **params}, pred, data, conf)
    losses["total"].mean().backward()
    for k in ("matches0", "matches1"):
        assert np.array_equal(pred[k].numpy(), g["pred|" + k]), k
    for k in ("sinkhorn_cost", "log_assignment", "matching_scores0", "matching_scores1"):
        _close(pred[k], g, "pred|" + k)
    _check_losses(losses, g)
    _check_grads(g, params)
    for k, v in SO.running_stats(w, stats, conf).items():
        np.testing.assert_allclose(v.numpy(), g["bn|" + k], rtol=RTOL, atol=ATOL, err_msg=k)


def test_gluestick_oracle_matches_edge_fixture():
    g, conf = load("edge_gs_labels")
    B, N, L, seed = (int(g["meta|" + k]) for k in ("B", "N", "L", "seed"))
    w = {k: (v.double() if v.is_floating_point() else v)
         for k, v in synthetic.make_gluestick_weights(GlueStick(dict(conf)).state_dict(), seed=seed).items()}
    params = {k: v.requires_grad_(True) for k, v in w.items() if v.is_floating_point() and "running_" not in k}
    data = synthetic.make_gluestick_batch(B, N, L, seed + 1, dtype=torch.float64)
    data = _labels(g, data, ("gt_assignment", "gt_matches0", "gt_matches1", "gt_line_assignment", "gt_line_matches0",
                             "gt_line_matches1"))
    stats = {}
    pred = GO.gluestick_forward({**w, **params}, data, conf, bn_stats=stats)
    losses = GO.gluestick_loss({**w, **params}, pred, data, conf)
    losses["total"].mean().backward()
    for k in (k[len("pred|"):] for k in g if k.startswith("pred|")):
        if "matches" in k and "scores" not in k:
            assert np.array_equal(pred[k].numpy(), g["pred|" + k]), k
        else:
            _close(pred[k], g, "pred|" + k)
    _check_losses(losses, g)
    _check_grads(g, params)
    for name, calls in stats.items():
        rm, rv = torch.zeros_like(calls[0][0]), torch.ones_like(calls[0][1])
        for mean, var_unbiased in calls:
            rm, rv = 0.9 * rm + 0.1 * mean, 0.9 * rv + 0.1 * var_unbiased
        np.testing.assert_allclose(rm.numpy(), g["bn|" + name + ".running_mean"], rtol=RTOL, atol=ATOL, err_msg=name)
        np.testing.assert_allclose(rv.numpy(), g["bn|" + name + ".running_var"], rtol=RTOL, atol=ATOL, err_msg=name)


def _classes(asg, m0, m1):
    """Per pair: (positives, negatives in view 0, negatives in view 1, labelled points, largest row count)."""
    asg = asg.reshape(asg.shape[0], asg.shape[1], -1).astype(np.int64)
    return [(int(asg[b].sum()), int((m0[b] == -1).sum()), int((m1[b] == -1).sum()),
             int((m0[b] != -2).sum() + (m1[b] != -2).sum()), int(asg[b].sum(1).max())) for b in range(asg.shape[0])]


def test_fixtures_hold_the_empty_classes_and_asymmetric_weights():
    """What tests/test_gpu_pair_edges.py takes from these fixtures: each empty label class, and loss weights at which a
    swapped balance or a wrong layer weight changes the result."""
    seen = set()
    for name in LG + ["edge_sg_labels", "edge_gs_labels"]:
        g, conf = load(name)
        prefixes = ["", "line_"] if name == "edge_gs_labels" else [""]
        for p in prefixes:
            for pos, n0, n1, labelled, rowmax in _classes(g[f"label|gt_{p}assignment"], g[f"label|gt_{p}matches0"],
                                                          g[f"label|gt_{p}matches1"]):
                assert labelled == 0 or n0 + n1 > 0 or pos > 0
                if labelled == 0:
                    seen.add("all ignored")
                elif pos == 0:
                    seen.add("no positives")
                if pos > 0 and (n0 == 0) != (n1 == 0):
                    seen.add(f"{name[:7]} no negatives in one view")
                if pos > 1 and rowmax == pos:
                    seen.add("positives in one row")
                if name == "edge_lg_b_m1_n65" and pos > 0:
                    seen.add("one-point view positive")
    assert seen >= {"all ignored", "no positives", "positives in one row", "one-point view positive",
                    "edge_lg no negatives in one view", "edge_sg no negatives in one view",
                    "edge_gs no negatives in one view"}, seen
    # the loss weights: gamma 0 (linear layer weights) and gamma 0.7 (powers); balances away from 0.5
    confs = {name: load(name)[1] for name in LG + ["edge_sg_labels", "edge_gs_labels"]}
    assert {c["loss"]["gamma"] for n, c in confs.items() if n in LG} == {0.0, 0.7}
    assert all(c["loss"]["nll_balancing"] != 0.5 for c in confs.values())
    gs = confs["edge_gs_labels"]["loss"]
    assert gs["nll_weight"] == 2.0 and gs["inter_supervision"] != [0.3, 0.6]
    # the stored totals follow those weights: LightGlue's total is the weighted mean of the layer NLLs (checked on the
    # last layer's share) plus the confidence term, GlueStick's the weighted sum of its five NLL terms
    g, _ = load("edge_gs_labels")
    total = 2.0 * (g["loss|assignment_nll"] + g["loss|line_assignment_nll"] + 0.25 * g["loss|line_1_assignment_nll"]
                   + 0.9 * g["loss|line_0_assignment_nll"])
    np.testing.assert_allclose(g["loss|total"], total, rtol=1e-12)
    # a pair with every label ignored has zero NLL in every term; a pair without positives has nll_pos exactly 0
    g, _ = load("edge_lg_a_labels")
    assert g["loss|nll_pos"][1] == 0.0 and g["loss|nll_neg"][1] == 0.0 and g["loss|assignment_nll"][1] == 0.0
    assert (g["loss|nll_pos"][[0, 2]] != 0).all()
    g, _ = load("edge_lg_b_m1_n65")
    assert g["loss|nll_pos"][1] == 0.0 and g["loss|nll_pos"][0] != 0.0
    # LightGlue clamps the negative count per view, SuperGlue and GlueStick the sum: recorded in num_unmatchable
    g, _ = load("edge_lg_a_labels")
    m0, m1 = g["label|gt_matches0"], g["label|gt_matches1"]
    n0, n1 = (m0 == -1).sum(1), (m1 == -1).sum(1)
    np.testing.assert_array_equal(g["loss|num_unmatchable"], (np.maximum(n0, 1) + np.maximum(n1, 1)) / 2.0)
    assert n1[2] == 0
    g, _ = load("edge_sg_labels")
    n = (g["label|gt_matches0"] == -1).sum(1) + (g["label|gt_matches1"] == -1).sum(1)
    np.testing.assert_array_equal(g["loss|num_unmatchable"], np.maximum(n, 1))
