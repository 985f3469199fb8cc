"""GPU: the GlueStick plugin (points + lines, BASELINE configs[4], SURVEY 8a row a15) against the fixture produced by the
unmodified reference (tests/golden/gluestick_l4_n160.npz: forward + loss + backward in fp64, training-mode BatchNorm)
and, at a larger ragged size, against the CPU oracle (oracle/gluestick_oracle.py, pinned to the same fixture).

precision="fp32" (fp32 cuBLAS linears, CUDA-core attention: the reference also forces its attention to fp32) meets the
north-star bar: match indices bit-exact, log-scores / losses / gradients within 1e-3.  precision="bf16" (wgmma
GEMMs and attention) is held to bf16-operand tolerances."""
import ast
import os

import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.gluestick import GlueStick
from tests.util import GOLDEN, check_grad_summary, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _case():
    g = dict(np.load(os.path.join(GOLDEN, "gluestick_l4_n160.npz"), allow_pickle=False))
    conf = ast.literal_eval(str(g["meta|conf"]))
    B, N, L, seed = (int(g["meta|" + k]) for k in ("B", "N", "L", "seed"))
    return g, conf, B, N, L, seed


def _build(conf, seed, precision):
    model = GlueStick(dict(conf, precision=precision))
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=seed), strict=True)
    return model.to(DEV).train()


def test_state_dict_layout_equals_reference_fixture():
    g, conf, *_ = _case()
    model = GlueStick(dict(conf))
    grads = {k[len("grad|"):].rsplit("|", 1)[0] for k in g if k.startswith("grad|")}
    assert grads == {n for n, _ in model.named_parameters()}
    assert {k[len("bn|"):] for k in g if k.startswith("bn|")} == {k for k in model.state_dict() if "running_" in k}


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_gluestick_matches_reference_golden(precision):
    g, conf, B, N, L, seed = _case()
    model = _build(conf, seed, precision)
    data = synthetic.to_device(synthetic.make_gluestick_batch(B, N, L, seed + 1), DEV)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    tight = precision == "fp32"
    if tight:
        for k in ["matches0", "matches1", "line_matches0", "line_matches1"]:
            assert np.array_equal(pred[k].cpu().numpy(), g["pred|" + k]), k
    tol = 1e-3 if tight else 4e-2
    for k in ["log_assignment", "line_log_assignment"]:
        assert rel_err(pred[k], torch.from_numpy(g["pred|" + k])) < (1e-4 if tight else 2e-2), k
        np.testing.assert_allclose(pred[k].detach().cpu().numpy(), g["pred|" + k], rtol=tol, atol=tol if tight else 0.5)
    for k in ["total", "assignment_nll", "line_assignment_nll", "num_matchable", "line_num_matchable", "num_unmatchable",
              "sinkhorn_norm", "line_sinkhorn_norm", "bin_score", "line_bin_score"]:
        np.testing.assert_allclose(losses[k].detach().cpu().numpy(), g["loss|" + k], rtol=1e-3 if tight else 3e-2, err_msg=k)
    worst = 0.0
    for k, p in model.named_parameters():
        ref_norm = float(g[f"grad|{k}|norm"])
        if ref_norm < 1e-9:  # conv bias in front of a BatchNorm: zero gradient in theory, rounding noise in practice
            assert p.grad.norm().item() < (1e-4 if tight else 2e-2), k
            continue
        if tight:
            check_grad_summary(g, k, p.grad, rtol=2e-3)
        else:
            worst = max(worst, abs(p.grad.double().norm().item() - ref_norm) / ref_norm)
    assert worst < 0.15, worst
    # BatchNorm running statistics were updated exactly like the reference's (two calls per layer)
    for k, v in model.state_dict().items():
        if "running_" in k:
            np.testing.assert_allclose(v.cpu().numpy(), g["bn|" + k], rtol=1e-3 if tight else 3e-2, atol=1e-5 if tight else 1e-3,
                                       err_msg=k)


def test_gluestick_ragged_against_oracle():
    """M != N, line counts differ, sizes not multiples of the tile sizes; fp32 mode vs the fp64 oracle."""
    from oracle import gluestick_oracle as G

    conf = {"GNN_layers": ["self", "cross"], "filter_threshold": 0.1}
    model = _build(conf, 41, "fp32")
    d = synthetic.make_gluestick_batch(2, 203, 20, 43)
    d0 = synthetic.make_gluestick_batch(2, 150, 20, 44)  # a second batch only to take a shorter view 0 from
    for k in ("keypoints0", "descriptors0", "keypoint_scores0"):
        d[k] = d[k][:, :150]
    d["gt_assignment"], d["gt_matches0"] = d["gt_assignment"][:, :150], d["gt_matches0"][:, :150]
    d["gt_matches1"] = torch.where(d["gt_matches1"] >= 150, torch.full_like(d["gt_matches1"], -1), d["gt_matches1"])
    del d0
    data = synthetic.to_device(d, DEV)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    w = {k: (v.detach().double().cpu() if v.is_floating_point() else v.cpu()) for k, v in model.state_dict().items()}
    # the oracle must see the weights BEFORE this forward's running-stat update; only parameters matter to it
    params = {k: w[k].requires_grad_(True) for k, _ in model.named_parameters()}
    ww = {**w, **params}
    d64 = {k: ({kk: vv.double() for kk, vv in v.items()} if isinstance(v, dict) else
               (v.double() if v.is_floating_point() else v)) for k, v in d.items()}
    rp = G.gluestick_forward(ww, d64, dict(conf, descriptor_dim=256))
    rl = G.gluestick_loss(ww, rp, d64, conf)
    rl["total"].mean().backward()
    assert torch.equal(pred["matches0"].cpu(), rp["matches0"]) and torch.equal(pred["line_matches0"].cpu(), rp["line_matches0"])
    assert rel_err(pred["log_assignment"], rp["log_assignment"]) < 1e-4
    assert rel_err(losses["total"], rl["total"]) < 1e-4
    for k, p in model.named_parameters():
        if params[k].grad.norm().item() < 1e-9:
            continue
        assert rel_err(p.grad, params[k].grad) < 2e-3, k


def test_gluestick_trains_and_evaluates():
    conf = {"GNN_layers": ["self", "cross"] * 2}
    model = _build(conf, 51, "bf16")
    data = synthetic.to_device(synthetic.make_gluestick_batch(2, 256, 32, 52), DEV)
    opt = torch.optim.Adam(model.parameters(), lr=3e-4)
    first = last = None
    for _ in range(8):
        opt.zero_grad()
        pred = model(data)
        losses, _ = model.loss(pred, data)
        loss = losses["total"].mean()
        loss.backward()
        opt.step()
        first = loss.item() if first is None else first
        last = loss.item()
    assert np.isfinite(last) and last < first, (first, last)
    model.eval()
    with torch.no_grad():
        pred = model(data)
        _, metrics = model.loss(pred, data)
    assert {"match_recall", "line_match_recall", "average_precision"} <= set(metrics)


def test_gluestick_training_step_replays_as_one_cuda_graph():
    """The whole GlueStick step (forward, both assignment losses, backward, flat Adam) holds no host read-back -- the
    learnt bin scores are read on the device -- so trainer.MatcherTrainer can capture it; replay == eager steps."""
    from gluefactory_b200.trainer import MatcherTrainer

    g, conf, B, N, L, seed = _case()
    data = synthetic.to_device(synthetic.make_gluestick_batch(B, N, L, seed + 1), DEV)
    eager = MatcherTrainer(_build(conf, seed, "bf16"), lr=1e-4)
    graphed = MatcherTrainer(_build(conf, seed, "bf16"), lr=1e-4)
    graphed.capture(data, torch.device(DEV))
    for it in range(3):
        le, _ = eager.step(data)
        lg, _ = graphed.step_graphed(data)
        assert torch.isfinite(lg).all()
        assert abs(le.item() - lg.item()) < (1e-5 if it == 0 else 2e-3) * abs(le.item()), (it, le.item(), lg.item())
