"""GPU: the GlueStick plugin on wireframes against the fixtures the unmodified reference produced on inputs built by its
own `lines_to_wireframe` (tests/golden/gluestick_wireframe_*.npz, scripts/make_gluestick_wireframe_golden.py; the fp64
oracle that restates it is pinned to the same fixtures in tests/test_gluestick_wireframe_cpu.py):
  a_eval          shared junctions (some ending 3+ lines), nodes no line touches, eval-mode BatchNorm with non-default
                  running statistics, B = 1, M = 191 != N = 199;
  b_train         padded wireframes with shared junctions, training mode, B = 2, inter_supervision [1]: losses, every
                  parameter gradient, running statistics;
  c_no_lines      view 1 without lines: no LineLayer or line head runs, the line outputs are zero / -1;
  d_no_keypoints  view 0 without keypoints: the reference's early-exit pred;
  e_image_shape   views given with `image` and without `image_size`.
precision="fp32" is held to tests/test_gpu_gluestick.py's fp32 bounds (match indices exact, log-assignments rel. L2
1e-4 and elementwise 1e-3, losses 1e-3, gradients 2e-3 of their norm), precision="bf16" to that file's bf16 bounds."""
import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.gluestick import GlueStick
from tests import gluestick_wireframe_oracle as O
from tests.gluestick_inter_oracle import point_log_assignment_summary
from tests.util import GOLDEN, check_grad_summary, rel_err, report

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _load(name):
    g, conf, _, data = O.load_case(GOLDEN, name, dtype=torch.float32)
    return g, conf, synthetic.to_device(data, DEV)


def _build(g, conf, precision):
    model = GlueStick(dict(conf, precision=precision))
    model.load_state_dict(O.case_state_dict(g, model.state_dict()), strict=True)
    return model.to(DEV).train(bool(g["meta|training"]))


def _run(name, precision):
    g, conf, data = _load(name)
    model = _build(g, conf, precision)
    if bool(g["meta|training"]):
        pred = model(data)
        losses, _ = model.loss(pred, data)
        losses["total"].mean().backward()
    else:
        with torch.no_grad():
            pred = model(data)
        losses = None
    return g, model, pred, losses


def _check_pred(g, pred, tight, tag):
    stored = [k[len("pred|"):] for k in g if k.startswith("pred|")]
    if "log_assignment_sub" in stored:
        pred = {**pred, **point_log_assignment_summary(pred["log_assignment"].detach())}
    for k in stored:
        got, ref = pred[k], g["pred|" + k]
        assert tuple(got.shape) == ref.shape, k
        if "matches" in k and "scores" not in k:
            assert got.dtype == torch.int64, k
            if tight:
                assert np.array_equal(got.cpu().numpy(), ref), k
        elif "log_assignment" in k or k == "raw_line_scores":
            e = rel_err(got, torch.from_numpy(ref))
            report(f"{tag} {k}", rel_l2=e)
            assert e < (1e-4 if tight else 2e-2), (k, e)
            tol = 1e-3 if tight else 4e-2
            np.testing.assert_allclose(got.detach().cpu().numpy(), ref, rtol=tol, atol=tol if tight else 0.5, err_msg=k)


@pytest.mark.parametrize("name", ["a_eval", "b_train", "c_no_lines", "e_image_shape"])
def test_wireframe_fp32_matches_reference_golden(name):
    g, model, pred, losses = _run(name, "fp32")
    _check_pred(g, pred, True, f"gluestick wireframe {name} fp32")
    expected = {k[len("pred|"):] for k in g if k.startswith("pred|")}
    if "log_assignment_sub" in expected:  # b_train keeps the point log-assignment as a summary
        expected = expected - {"log_assignment_sub", "log_assignment_rowmax", "log_assignment_colmax"} | {"log_assignment"}
    assert set(pred) == expected, set(pred) ^ expected
    for k in pred:
        if "matching_scores" in k:
            np.testing.assert_allclose(pred[k].cpu().numpy(), g["pred|" + k], rtol=1e-3, atol=1e-4, err_msg=k)
    if losses is None:
        return
    assert set(losses) == {k[len("loss|"):] for k in g if k.startswith("loss|")}
    for k, v in losses.items():
        np.testing.assert_allclose(v.detach().cpu().numpy(), g["loss|" + k], rtol=1e-3, err_msg=k)
    for k, p in model.named_parameters():
        if float(g[f"grad|{k}|norm"]) < 1e-9:  # conv bias in front of a BatchNorm: zero in theory, rounding noise
            assert p.grad.norm().item() < 1e-4, k
            continue
        check_grad_summary(g, k, p.grad, rtol=2e-3)
    for k, v in model.state_dict().items():
        if "running_" in k:
            np.testing.assert_allclose(v.cpu().numpy(), g["bn|" + k], rtol=1e-3, atol=1e-5, err_msg=k)


@pytest.mark.parametrize("name", ["a_eval", "b_train"])
def test_wireframe_bf16_matches_reference_golden(name):
    g, model, pred, losses = _run(name, "bf16")
    _check_pred(g, pred, False, f"gluestick wireframe {name} bf16")
    if losses is None:
        return
    for k, v in losses.items():
        np.testing.assert_allclose(v.detach().cpu().numpy(), g["loss|" + k], rtol=3e-2, err_msg=k)
    worst = 0.0
    for k, p in model.named_parameters():
        ref_norm = float(g[f"grad|{k}|norm"])
        if ref_norm < 1e-9:
            assert p.grad.norm().item() < 2e-2, k
            continue
        worst = max(worst, abs(p.grad.double().norm().item() - ref_norm) / ref_norm)
    report(f"gluestick wireframe {name} bf16", worst_grad_norm_rel=worst)
    assert worst < 0.15, worst
    for k, v in model.state_dict().items():
        if "running_" in k:
            np.testing.assert_allclose(v.cpu().numpy(), g["bn|" + k], rtol=3e-2, atol=1e-3, err_msg=k)


def _line_free_outputs(B, L0, L1):
    z = dict(dtype=torch.float32, device=DEV)
    return {"line_log_assignment": torch.zeros(B, L0, L1, **z), "raw_line_scores": torch.zeros(B, L0, L1, **z),
            "line_matches0": torch.full((B, L0), -1, dtype=torch.int64, device=DEV),
            "line_matches1": torch.full((B, L1), -1, dtype=torch.int64, device=DEV),
            "line_matching_scores0": torch.zeros(B, L0, **z), "line_matching_scores1": torch.zeros(B, L1, **z)}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_view_without_lines_gives_the_reference_line_outputs(precision):
    """gluestick.py:293-312, key for key; with inter_supervision no intermediate head runs or appears (the reference
    only adds those keys with lines), and the point outputs do not change."""
    g, conf, data = _load("c_no_lines")
    L0, L1 = data["lines0"].shape[1], data["lines1"].shape[1]
    assert L0 > 0 and L1 == 0
    model = _build(g, conf, precision)
    inter_conf = dict(conf, inter_supervision=[1], loss={"inter_supervision": [0.3]})
    inter = GlueStick(dict(inter_conf, precision=precision))
    inter.load_state_dict({**model.state_dict(), **{k: v for k, v in inter.state_dict().items()
                                                    if k.startswith("inter_line_proj.")}}, strict=True)
    inter = inter.to(DEV).eval()
    with torch.no_grad():
        pred, pred_inter = model(data), inter(data)
    assert set(pred) == set(pred_inter) == {"log_assignment", "matches0", "matches1", "matching_scores0",
                                            "matching_scores1", *_line_free_outputs(1, L0, L1)}
    for k, ref in _line_free_outputs(1, L0, L1).items():
        for p in (pred, pred_inter):
            assert p[k].dtype == ref.dtype and p[k].shape == ref.shape and torch.equal(p[k], ref), k
    for k in ("log_assignment", "matches0", "matches1", "matching_scores0", "matching_scores1"):
        assert torch.equal(pred[k], pred_inter[k]), k
    assert tuple(pred["log_assignment"].shape) == (1, data["keypoints0"].shape[1] + 1, data["keypoints1"].shape[1] + 1)


def test_view_without_keypoints_gives_the_reference_early_exit_pred():
    """gluestick.py:163-195: exactly the reference's keys, shapes (log_assignment [B, M, N], line_matching_scores1
    [B, N]), dtypes and values, on the device of the inputs."""
    g, conf, data = _load("d_no_keypoints")
    model = _build(g, conf, "bf16")
    with torch.no_grad():
        pred = model(data)
    stored = {k[len("pred|"):] for k in g if k.startswith("pred|")}
    assert set(pred) == stored
    N, L1 = data["keypoints1"].shape[1], data["lines1"].shape[1]
    assert pred["log_assignment"].shape == (1, 0, N) and pred["line_matching_scores1"].shape == (1, N) and N != L1
    for k in stored:
        assert pred[k].device.type == "cuda", k
        assert pred[k].dtype == (torch.int64 if "matches" in k and "scores" not in k else torch.float32), k
        assert tuple(pred[k].shape) == g["pred|" + k].shape and np.array_equal(pred[k].cpu().numpy(), g["pred|" + k]), k


def test_loss_without_lines_raises():
    g, conf, data = _load("c_no_lines")
    model = _build(g, conf, "bf16").train()
    pred = model(data)
    with pytest.raises(ValueError, match="line loss needs lines in both views"):
        model.loss(pred, data)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_trainer_step_on_shared_junctions_gives_the_autograd_gradients(precision):
    """MatcherTrainer.step on b_train (shared junctions, padded, inter_supervision [1]) computes the gradients that
    forward + loss + backward on an identical model compute.  Measured on an H100 80GB HBM3 (700 W), conv biases in
    front of a BatchNorm aside (zero in theory): rel. L2 7.4e-9 in bf16 and 2.9e-6 in fp32 (cuBLAS linears) at worst.
    The scatter-mean over shared junctions and the backward of the gathers over repeated junction indices sum by atomic
    adds in no fixed order, so neither bound is zero."""
    from gluefactory_b200.trainer import MatcherTrainer

    g, conf, data = _load("b_train")
    ref = _build(g, conf, precision)
    pred = ref(data)
    losses, _ = ref.loss(pred, data)
    losses["total"].mean().backward()
    tr = MatcherTrainer(_build(g, conf, precision), lr=1e-4)
    loss, _ = tr.step(data)
    assert torch.isfinite(loss).all()
    assert rel_err(loss, losses["total"].mean()) < (1e-6 if precision == "fp32" else 1e-4)
    names = {id(p): n for n, p in tr.model.named_parameters()}
    grads = dict(ref.named_parameters())
    worst = 0.0
    for p, v in zip(tr.fp.params, tr.fp.grad_views):
        k = names[id(p)]
        if float(g[f"grad|{k}|norm"]) < 1e-9:  # conv bias in front of a BatchNorm: zero in theory, rounding noise
            bound = 1e-4 if precision == "fp32" else 2e-2
            assert v.norm().item() < bound and grads[k].grad.norm().item() < bound, k
            continue
        worst = max(worst, rel_err(v, grads[k].grad))
    report(f"gluestick wireframe trainer step {precision}", worst_grad_rel=worst)
    assert worst < (5e-4 if precision == "fp32" else 2e-3), worst
