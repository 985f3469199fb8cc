"""GPU: GlueStick with intermediate line supervision (`inter_supervision`) against the fixture produced by the unmodified
reference (tests/golden/gluestick_inter_l8_n160.npz: 8 GNN layers, inter_supervision [0, 2], loss weights [0.3, 0.6];
forward + loss + backward in fp64, training-mode BatchNorm) and, at a ragged size, against the fp64 CPU oracle
(tests/gluestick_inter_oracle.py).

Measured on an H100 80GB HBM3 (700 W):
The fixture keeps the point head's log-assignment as a strided sample and its row / column maxima
(gluestick_inter_oracle.point_log_assignment_summary); the line heads' are compared whole.
  * precision="fp32": match indices bit-exact; log-assignments rel. L2 8.2e-7 (bound 1e-4), losses 1.3e-7 (1e-3),
    gradient norms 4.3e-4.  Gradients against the fixture's summaries (tests.util.check_grad_summary's rtol) 2.25e-3
    at worst, all in the line endpoint encoder, whose gradient sums the contributions of every line layer: bound 5e-3.
    That error is not the intermediate heads': the same 8-layer model without them is off by 2.5e-3 on the same
    parameters against the fp64 oracle.  The 4-layer fixture of tests/test_gpu_gluestick.py is held to 2e-3.
  * precision="bf16": the tolerances of tests/test_gpu_gluestick.py; log-assignments rel. L2 6.2e-3 at most, losses
    rel. 6.3e-3, gradient norms rel. 0.056.
Then the eval-mode metrics of the intermediate heads, the CUDA-graph replay of a MatcherTrainer step, and the matcher
section of configs/superpoint+lsd+gluestick-homography.yaml training on device line labels."""
import ast
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gluefactory_b200 import synthetic
from gluefactory_b200.geometry import warp_points
from gluefactory_b200.matchers.gluestick import GlueStick
from gluefactory_b200.matchers.lightglue import matcher_metrics
from tests.gluestick_inter_oracle import point_log_assignment_summary
from tests.util import GOLDEN, probe_index, probe_vector, rel_err, report

pytestmark = pytest.mark.gpu
DEV = "cuda"
GRAD_RTOL_FP32 = 5e-3


def _case():
    g = dict(np.load(os.path.join(GOLDEN, "gluestick_inter_l8_n160.npz"), allow_pickle=False))
    conf = ast.literal_eval(str(g["meta|conf"]))
    B, N, L, seed = (int(g["meta|" + k]) for k in ("B", "N", "L", "seed"))
    return g, conf, B, N, L, seed


def _build(conf, seed, precision):
    model = GlueStick(dict(conf, precision=precision))
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=seed), strict=True)
    return model.to(DEV).train()


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_gluestick_inter_matches_reference_golden(precision):
    g, conf, B, N, L, seed = _case()
    model = _build(conf, seed, precision)
    data = synthetic.to_device(synthetic.make_gluestick_batch(B, N, L, seed + 1), DEV)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    tight = precision == "fp32"
    tag = f"gluestick inter {precision}"
    heads = ["", "line_", "line_0_", "line_2_"]
    if tight:
        for h in heads:
            for k in (h + "matches0", h + "matches1"):
                assert np.array_equal(pred[k].cpu().numpy(), g["pred|" + k]), k
    tol = 1e-3 if tight else 4e-2
    got = {**pred, **point_log_assignment_summary(pred["log_assignment"].detach())}
    for k in ["log_assignment_sub", "log_assignment_rowmax", "log_assignment_colmax"] + [h + "log_assignment"
                                                                                         for h in heads[1:]]:
        e = rel_err(got[k], torch.from_numpy(g["pred|" + k]))
        report(f"{tag} {k}", rel_l2=e)
        assert e < (1e-4 if tight else 2e-2), (k, e)
        np.testing.assert_allclose(got[k].detach().cpu().numpy(), g["pred|" + k], rtol=tol, atol=tol if tight else 0.5,
                                   err_msg=k)
    loss_keys = [k[len("loss|"):] for k in g if k.startswith("loss|")]
    assert set(losses) == set(loss_keys)
    worst_loss = 0.0
    for k in loss_keys:
        got, ref = losses[k].detach().double().cpu().numpy(), g["loss|" + k]
        worst_loss = max(worst_loss, float(np.max(np.abs(got - ref) / np.maximum(np.abs(ref), 1e-12))))
        np.testing.assert_allclose(got, ref, rtol=1e-3 if tight else 3e-2, err_msg=k)
    worst, summary = 0.0, []
    for k, p in model.named_parameters():
        ref_norm = float(g[f"grad|{k}|norm"])
        if ref_norm < 1e-9:  # conv bias in front of a BatchNorm: zero gradient in theory, rounding noise in practice
            assert p.grad.norm().item() < (1e-4 if tight else 2e-2), k
            continue
        worst = max(worst, abs(p.grad.double().norm().item() - ref_norm) / ref_norm)
        summary.append((_summary_rtol(g, k, p.grad), k))
    for k, v in model.state_dict().items():
        if "running_" in k:
            np.testing.assert_allclose(v.cpu().numpy(), g["bn|" + k], rtol=1e-3 if tight else 3e-2,
                                       atol=1e-5 if tight else 1e-3, err_msg=k)
    summary.sort(reverse=True)
    report(tag, worst_loss_rel=worst_loss, worst_grad_norm_rel=worst,
           worst_grad_summary_rtol=" ".join(f"{k}:{e:.3g}" for e, k in summary[:4]))
    if tight:
        assert summary[0][0] < GRAD_RTOL_FP32, summary[:4]
    assert worst < (GRAD_RTOL_FP32 if tight else 0.15), worst


def _summary_rtol(g, name, grad):
    """The smallest rtol at which tests.util.check_grad_summary accepts `grad` against the fixture's summary."""
    grad = grad.detach().double().cpu()
    ref_norm = max(float(g[f"grad|{name}|norm"]), 1e-12)
    errs = [abs(grad.norm().item() - ref_norm) / ref_norm]
    if f"grad|{name}|full" in g:
        errs.append((grad - torch.from_numpy(g[f"grad|{name}|full"])).norm().item() / ref_norm)
    else:
        flat = grad.reshape(-1)
        scale = ref_norm * (512.0 / flat.numel()) ** 0.5
        errs.append((flat[probe_index(flat.numel())] - torch.from_numpy(g[f"grad|{name}|sample"])).norm().item() / (4 * scale))
        errs.append(abs((flat * probe_vector(flat.numel())).sum().item() - float(g[f"grad|{name}|proj"])) / (4 * ref_norm))
    return max(errs)


def _ragged_batch():
    """M = 150 != N = 203 points, 17 lines in view 0 and 20 in view 1: no size is a multiple of a tile."""
    d = synthetic.make_gluestick_batch(2, 203, 20, 163)
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
def test_gluestick_inter_ragged_against_oracle(precision):
    """Heads after blocks 1 and 0 (listed out of order) of a 3-block GNN, weights 0.7 and 0.2.  fp32: matches equal the
    fp64 oracle's and log-assignments / loss / gradients within 1e-4 / 1e-4 / 2e-3; bf16 within the golden test's
    bounds."""
    from tests import gluestick_inter_oracle as O

    conf = {"GNN_layers": ["self", "cross"] * 3, "filter_threshold": 0.1, "inter_supervision": [1, 0],
            "loss": {"inter_supervision": [0.7, 0.2]}}
    model = _build(conf, 161, precision)
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
    rp = O.gluestick_forward(ww, d64, dict(conf, descriptor_dim=256))
    rl = O.gluestick_loss(ww, rp, d64, conf)
    rl["total"].mean().backward()
    tight = precision == "fp32"
    for h in ["", "line_", "line_1_", "line_0_"]:
        if tight:
            assert torch.equal(pred[h + "matches0"].cpu(), rp[h + "matches0"]), h
            assert torch.equal(pred[h + "matches1"].cpu(), rp[h + "matches1"]), h
        e = rel_err(pred[h + "log_assignment"], rp[h + "log_assignment"])
        report(f"gluestick inter ragged {precision} {h}log_assignment", rel_l2=e)
        assert e < (1e-4 if tight else 2e-2), (h, e)
    for k in ("total", "line_0_assignment_nll", "line_1_assignment_nll"):
        assert rel_err(losses[k], rl[k]) < (1e-4 if tight else 3e-2), k
    for k, p in model.named_parameters():
        if params[k].grad.norm().item() < 1e-9:
            continue
        if tight:
            assert rel_err(p.grad, params[k].grad) < 2e-3, k
        else:
            ref = params[k].grad.norm().item()
            assert abs(p.grad.double().norm().item() - ref) / ref < 0.15, k


def test_gluestick_inter_eval_metrics():
    """In eval mode the intermediate heads still run, and loss() adds matcher_metrics of each under line_{l}_ against
    the final line head's ground truth (gluestick.py:455-460)."""
    g, conf, B, N, L, seed = _case()
    model = _build(conf, seed, "bf16").eval()
    data = synthetic.to_device(synthetic.make_gluestick_batch(B, N, L, seed + 1), DEV)
    with torch.no_grad():
        pred = model(data)
        losses, metrics = model.loss(pred, data)
    for block in (0, 2):
        h = f"line_{block}_"
        assert {h + k for k in ("log_assignment", "matches0", "matches1", "matching_scores0",
                                "matching_scores1")} <= set(pred)
        assert torch.isfinite(losses[h + "assignment_nll"]).all()
        ref = matcher_metrics({"matches0": pred[h + "matches0"], "matching_scores0": pred[h + "matching_scores0"]},
                              {"gt_matches0": data["gt_line_matches0"]})
        for k, v in ref.items():
            assert torch.equal(metrics[h + k], v), h + k
    assert {"match_recall", "line_match_recall", "line_0_match_recall", "line_2_average_precision"} <= set(metrics)


def test_gluestick_inter_training_step_replays_bit_identical():
    """MatcherTrainer captures the bf16 step with both intermediate heads and their loss terms as one CUDA graph; its
    replay computes what the eager step computes, bit for bit: the loss and every parameter after the Adam update."""
    from gluefactory_b200.trainer import MatcherTrainer

    g, conf, B, N, L, seed = _case()
    data = synthetic.to_device(synthetic.make_gluestick_batch(B, N, L, seed + 1), DEV)
    eager = MatcherTrainer(_build(conf, seed, "bf16"), lr=1e-4)
    graphed = MatcherTrainer(_build(conf, seed, "bf16"), lr=1e-4)
    graphed.capture(data, torch.device(DEV))
    assert {"line_0_assignment_nll", "line_2_assignment_nll"} <= set(graphed._static_losses)
    assert torch.equal(eager.fp.flat, graphed.fp.flat)
    for it in range(2):
        le, _ = eager.step(data)
        lg, _ = graphed.step_graphed(data)
        torch.cuda.synchronize()
        assert torch.isfinite(lg).all()
        assert torch.equal(le, lg), (it, le.item(), lg.item())
        assert torch.equal(eager.fp.flat, graphed.fp.flat), it


def test_homography_config_matcher_trains_with_device_line_labels():
    """The matcher section of configs/superpoint+lsd+gluestick-homography.yaml (18 layers, inter_supervision [2, 5],
    checkpointed) with its ground truth (homography_matcher, use_lines, th_positive 3, th_negative 5) on the device, at
    a small batch: the loss, with both intermediate terms, is finite and falls over a few Adam steps."""
    from gluefactory_b200.matchers.homography_matcher import HomographyMatcher
    from gluefactory_b200.trainer import MatcherTrainer

    g, *_ = _case()
    hconf = ast.literal_eval(str(g["meta|homography_conf"]))
    B, N, L = 2, 256, 32
    d = synthetic.make_gluestick_batch(B, N, L, 171)
    # view 1's lines: view 0's warped by H, shuffled and jittered by 0.5 px, so that the line labels have positives
    gen = torch.Generator().manual_seed(171)
    perm = torch.randperm(L, generator=gen)
    lines1 = warp_points(d["lines0"].reshape(B, 2 * L, 2), d["H_0to1"]).reshape(B, L, 2, 2)[:, perm]
    d["lines1"] = (lines1 + 0.5 * torch.randn(lines1.shape, generator=gen)).clamp(0.5, 1023.5)
    d["keypoints1"][:, :2 * L] = d["lines1"].reshape(B, 2 * L, 2)
    desc1 = d["descriptors0"][:, :2 * L].reshape(B, L, 2, -1)[:, perm].reshape(B, 2 * L, -1)
    d["descriptors1"][:, :2 * L] = F.normalize(desc1 + 0.02 * torch.randn(desc1.shape, generator=gen), dim=-1)
    for i in "01":
        d[f"valid_lines{i}"] = torch.ones(B, L, dtype=torch.bool)
        d[f"view{i}"]["image"] = torch.zeros(B, 1, 1024, 1024)
    data = synthetic.to_device({k: v for k, v in d.items() if not k.startswith("gt_")}, DEV)
    gt = HomographyMatcher({"use_points": True, "use_lines": True, "th_positive": 3.0, "th_negative": 5.0})
    labels = gt(data)
    assert (labels["line_matches0"] > -1).sum() > L and (labels["matches0"] > -1).any()
    model = _build(hconf, 173, "bf16")
    tr = MatcherTrainer(model, lr=1e-4, ground_truth=gt)
    history = []
    for _ in range(8):
        loss, losses = tr.step(data)
        assert torch.isfinite(losses["line_2_assignment_nll"]).all() and torch.isfinite(losses["line_5_assignment_nll"]).all()
        history.append(loss.item())
    assert all(np.isfinite(history)), history
    assert history[-1] < history[0], history
