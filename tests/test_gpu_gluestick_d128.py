"""GPU: the GlueStick plugin at descriptor_dim = input_dim = 128 (the DISK variant of the shipped configs; attention at
head dim 32) against the fixture produced by the unmodified reference (tests/golden/gluestick_d128_l4_n160.npz: forward
+ loss + backward in fp64, training-mode BatchNorm) and, at a ragged size, against the fp64 CPU oracle.

precision="fp32" meets the same bar as at 256 channels: match indices bit-exact, log-scores / losses / gradients /
running statistics within 1e-3.  precision="bf16" tolerances come from the errors measured on an H100 80GB HBM3 (700 W) against this fixture
(profiles/gluestick_d128_h100.md), with about 2x headroom:
    log-assignment rel. L2 error 1.3e-3, line log-assignment 2.3e-3 (bound 5e-3); loss entries rel. 1.7e-3 (bound 5e-3);
    worst gradient-norm rel. error 0.060 (bound 0.12); running statistics 3.4e-3 of the largest entry (elementwise
    bound rtol 3e-2, atol 1e-3, as at 256 channels); ragged case log-assignment 6.6e-4 (bound 5e-3)."""
import ast
import os

import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.gluestick import GlueStick
from tests.util import GOLDEN, check_grad_summary, rel_err, report

pytestmark = pytest.mark.gpu
DEV = "cuda"
D = 128


def _case():
    g = dict(np.load(os.path.join(GOLDEN, "gluestick_d128_l4_n160.npz"), allow_pickle=False))
    conf = ast.literal_eval(str(g["meta|conf"]))
    B, N, L, seed = (int(g["meta|" + k]) for k in ("B", "N", "L", "seed"))
    return g, conf, B, N, L, seed


def _build(conf, seed, precision):
    model = GlueStick(dict(conf, precision=precision))
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=seed), strict=True)
    return model.to(DEV).train()


LOSS_KEYS = ["total", "assignment_nll", "line_assignment_nll", "num_matchable", "line_num_matchable", "num_unmatchable",
             "sinkhorn_norm", "line_sinkhorn_norm", "bin_score", "line_bin_score"]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_gluestick_d128_matches_reference_golden(precision):
    g, conf, B, N, L, seed = _case()
    model = _build(conf, seed, precision)
    data = synthetic.to_device(synthetic.make_gluestick_batch(B, N, L, seed + 1, D=D), DEV)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    tight = precision == "fp32"
    tag = f"gluestick d128 {precision}"
    if tight:
        for k in ["matches0", "matches1", "line_matches0", "line_matches1"]:
            assert np.array_equal(pred[k].cpu().numpy(), g["pred|" + k]), k
    for k in ["log_assignment", "line_log_assignment"]:
        e = rel_err(pred[k], torch.from_numpy(g["pred|" + k]))
        report(f"{tag} {k}", rel_l2=e)
        assert e < (1e-4 if tight else 5e-3), (k, e)
        if tight:
            np.testing.assert_allclose(pred[k].detach().cpu().numpy(), g["pred|" + k], rtol=1e-3, atol=1e-3)
    worst_loss = 0.0
    for k in LOSS_KEYS:
        got, ref = losses[k].detach().double().cpu().numpy(), g["loss|" + k]
        worst_loss = max(worst_loss, float(np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1e-12))))
        np.testing.assert_allclose(got, ref, rtol=1e-3 if tight else 5e-3, err_msg=k)
    worst = 0.0
    for k, p in model.named_parameters():
        ref_norm = float(g[f"grad|{k}|norm"])
        if ref_norm < 1e-9:  # conv bias in front of a BatchNorm: zero gradient in theory, rounding noise in practice
            assert p.grad.norm().item() < (1e-4 if tight else 2e-2), k
            continue
        if tight:
            check_grad_summary(g, k, p.grad, rtol=1e-3)
        worst = max(worst, abs(p.grad.double().norm().item() - ref_norm) / ref_norm)
    worst_bn = 0.0
    for k, v in model.state_dict().items():
        if "running_" in k:
            ref = g["bn|" + k]
            worst_bn = max(worst_bn, float(np.abs(v.cpu().numpy() - ref).max() / max(np.abs(ref).max(), 1e-12)))
            np.testing.assert_allclose(v.cpu().numpy(), ref, rtol=1e-3 if tight else 3e-2, atol=1e-5 if tight else 1e-3,
                                       err_msg=k)
    report(tag, worst_loss_rel=worst_loss, worst_grad_norm_rel=worst, worst_running_stat_rel=worst_bn)
    assert worst < (1e-3 if tight else 0.12), worst


def _ragged_batch():
    """M = 150 != N = 203 points, 17 lines in view 0 and 20 in view 1: no size is a multiple of a tile."""
    d = synthetic.make_gluestick_batch(2, 203, 20, 143, D=D)
    for k in ("keypoints0", "descriptors0", "keypoint_scores0"):
        d[k] = d[k][:, :150]
    d["gt_assignment"], d["gt_matches0"] = d["gt_assignment"][:, :150], d["gt_matches0"][:, :150]
    d["gt_matches1"] = torch.where(d["gt_matches1"] >= 150, torch.full_like(d["gt_matches1"], -1), d["gt_matches1"])
    L0 = 17
    d["lines0"], d["line_scores0"] = d["lines0"][:, :L0], d["line_scores0"][:, :L0]
    d["lines_junc_idx0"] = d["lines_junc_idx0"][:, :L0]
    d["gt_line_assignment"], d["gt_line_matches0"] = d["gt_line_assignment"][:, :L0], d["gt_line_matches0"][:, :L0]
    d["gt_line_matches1"] = torch.where(d["gt_line_matches1"] >= L0, torch.full_like(d["gt_line_matches1"], -1),
                                        d["gt_line_matches1"])
    return d


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_gluestick_d128_ragged_against_oracle(precision):
    """fp32: matches equal the fp64 oracle's and log-scores / loss / gradients within 1e-4 / 1e-4 / 2e-3; bf16 within
    the golden test's bounds."""
    from oracle import gluestick_oracle as G

    conf = {"GNN_layers": ["self", "cross"], "filter_threshold": 0.1, "input_dim": D, "descriptor_dim": D}
    model = _build(conf, 141, precision)
    d = _ragged_batch()
    data = synthetic.to_device(d, DEV)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    w = {k: (v.detach().double().cpu() if v.is_floating_point() else v.cpu()) for k, v in model.state_dict().items()}
    params = {k: w[k].requires_grad_(True) for k, _ in model.named_parameters()}
    ww = {**w, **params}
    d64 = {k: ({kk: vv.double() for kk, vv in v.items()} if isinstance(v, dict) else
               (v.double() if v.is_floating_point() else v)) for k, v in d.items()}
    rp = G.gluestick_forward(ww, d64, conf)
    rl = G.gluestick_loss(ww, rp, d64, conf)
    rl["total"].mean().backward()
    tight = precision == "fp32"
    if tight:
        assert torch.equal(pred["matches0"].cpu(), rp["matches0"]) and torch.equal(pred["line_matches0"].cpu(),
                                                                                   rp["line_matches0"])
    e = rel_err(pred["log_assignment"], rp["log_assignment"])
    report(f"gluestick d128 ragged {precision}", log_assignment_rel_l2=e)
    assert e < (1e-4 if tight else 5e-3), e
    assert rel_err(losses["total"], rl["total"]) < (1e-4 if tight else 2e-2)
    for k, p in model.named_parameters():
        if params[k].grad.norm().item() < 1e-9:
            continue
        if tight:
            assert rel_err(p.grad, params[k].grad) < 2e-3, k
        else:
            ref = params[k].grad.norm().item()
            assert abs(p.grad.double().norm().item() - ref) / ref < 0.1, k


def test_gluestick_d128_training_step_replays_bit_identical():
    """MatcherTrainer captures the bf16 training step at 128 channels as one CUDA graph; its replay computes what the
    eager step computes, bit for bit: the loss and every parameter after the Adam update."""
    from gluefactory_b200.trainer import MatcherTrainer

    g, conf, B, N, L, seed = _case()
    data = synthetic.to_device(synthetic.make_gluestick_batch(B, N, L, seed + 1, D=D), DEV)
    eager = MatcherTrainer(_build(conf, seed, "bf16"), lr=1e-4)
    graphed = MatcherTrainer(_build(conf, seed, "bf16"), lr=1e-4)
    graphed.capture(data, torch.device(DEV))
    assert torch.equal(eager.fp.flat, graphed.fp.flat)
    for it in range(2):
        le, _ = eager.step(data)
        lg, _ = graphed.step_graphed(data)
        torch.cuda.synchronize()
        assert torch.isfinite(lg).all()
        assert torch.equal(le, lg), (it, le.item(), lg.item())
        assert torch.equal(eager.fp.flat, graphed.fp.flat), it
