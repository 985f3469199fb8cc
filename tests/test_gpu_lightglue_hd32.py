"""GPU: the LightGlue plugin at head dimension 32 -- `descriptor_dim 128` / 4 heads and `descriptor_dim 256` / 8 heads --
against the fixtures produced by the unmodified reference (scripts/make_lightglue_hd32_golden.py): forward, loss and
backward in fp64 for M == N, M != N, 8 heads and `add_scale_ori`, and eval-mode point pruning in fp32.

The bars are those of the head-dim-64 fixtures (tests/test_gpu_matcher.py): `fp32` with match indices bit-exact and
log-assignment, matching scores, every loss entry and the gradient summaries within 1e-3; `bf16` with the
log-assignment within 0.15, the total loss within 2e-2, indices equal wherever the reference's top-2 margin exceeds
0.3, and every gradient norm within 10 %."""
import ast
import os

import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.lightglue import LightGlue
from gluefactory_b200.trainer import MatcherTrainer
from tests.util import GOLDEN, check_grad_summary, load_case, rel_err, report

pytestmark = pytest.mark.gpu
DEV = "cuda"
HD32_CASES = ["lg_hd32_d128_h4_l3_n128", "lg_hd32_d128_h4_l3_m80_n112", "lg_hd32_d256_h8_l2_n128",
              "lg_hd32_sift_d128_h4_l2_n96"]
LOSS_KEYS = ["total", "last", "assignment_nll", "nll_pos", "nll_neg", "num_matchable", "num_unmatchable", "confidence",
             "row_norm"]


def _build(conf, weights, precision):
    model = LightGlue(dict(conf, precision=precision))
    missing, unexpected = model.load_state_dict({k: v.float() for k, v in weights.items()}, strict=False)
    assert not unexpected and missing in ([], ["confidence_thresholds"])
    return model.to(DEV).train()


def _f32(data):
    return synthetic.to_device({k: ({kk: vv.float() for kk, vv in v.items()} if isinstance(v, dict) else
                                    (v.float() if v.is_floating_point() else v)) for k, v in data.items()}, DEV)


def _run(name, precision):
    g, conf, w, data = load_case(name)
    assert conf["descriptor_dim"] // conf["num_heads"] == 32
    model = _build(conf, w, precision)
    d = _f32(data)
    pred = model(d)
    losses, _ = model.loss(pred, d)
    losses["total"].mean().backward()
    return g, model, pred, losses


@pytest.mark.parametrize("name", HD32_CASES)
def test_fp32_matches_reference_golden(name):
    g, model, pred, losses = _run(name, "fp32")
    assert np.array_equal(pred["matches0"].cpu().numpy(), g["pred|matches0"])
    assert np.array_equal(pred["matches1"].cpu().numpy(), g["pred|matches1"])
    report(f"hd32 {name} fp32", la=rel_err(pred["log_assignment"], torch.from_numpy(g["pred|log_assignment"])))
    np.testing.assert_allclose(pred["log_assignment"].cpu().numpy(), g["pred|log_assignment"], rtol=1e-3, atol=1e-3)
    np.testing.assert_allclose(pred["matching_scores0"].cpu().numpy(), g["pred|matching_scores0"], rtol=1e-3, atol=1e-6)
    np.testing.assert_allclose(pred["matching_scores1"].cpu().numpy(), g["pred|matching_scores1"], rtol=1e-3, atol=1e-6)
    for k in LOSS_KEYS:
        np.testing.assert_allclose(losses[k].detach().cpu().numpy(), g["loss|" + k], rtol=1e-3, err_msg=k)
    assert model.posenc.Wr.weight.grad.shape[0] == 16
    for k, p in model.named_parameters():
        check_grad_summary(g, k, p.grad, rtol=1e-3)


@pytest.mark.parametrize("name", HD32_CASES)
def test_bf16_close_to_reference_golden(name):
    g, model, pred, losses = _run(name, "bf16")
    la = pred["log_assignment"].cpu().double().numpy()
    report(f"hd32 {name} bf16", la_max_abs=float(np.abs(la - g["pred|log_assignment"]).max()),
           total_rel=float(np.abs(losses["total"].detach().cpu().numpy() - g["loss|total"]).max() / np.abs(g["loss|total"]).max()))
    assert np.abs(la - g["pred|log_assignment"]).max() < 0.15
    np.testing.assert_allclose(losses["total"].detach().cpu().numpy(), g["loss|total"], rtol=2e-2)
    ref = torch.from_numpy(g["pred|log_assignment"])[:, :-1, :-1]
    top2 = ref.topk(2, dim=2).values
    safe = (top2[..., 0] - top2[..., 1]) > 0.3
    got = torch.from_numpy(la)[:, :-1, :-1].max(2).indices
    assert torch.equal(got[safe], ref.max(2).indices[safe])
    worst = 0.0
    for k, p in model.named_parameters():
        ref_norm = float(g[f"grad|{k}|norm"])
        worst = max(worst, abs(p.grad.double().norm().item() - ref_norm) / max(ref_norm, 1e-12))
    report(f"hd32 {name} bf16", worst_grad_norm_rel=worst)
    assert worst < 0.1, worst


def test_adaptive_point_pruning_matches_reference():
    """Eval-mode point pruning at 128 channels / 4 heads (every pruning decision of the fixture clears its threshold by
    more than 2e-4): the same points survive every layer, the same pruned log-assignment, the same matches scattered
    back to the full sets."""
    g = dict(np.load(os.path.join(GOLDEN, "lg_hd32_d128_h4_adaptive_prune.npz")))
    conf = ast.literal_eval(str(g["meta|conf"]))
    seed, M, N = int(g["meta|seed"]), int(g["meta|M"]), int(g["meta|N"])
    model = _build(conf, synthetic.make_weights(conf, seed=seed), "fp32").eval()
    d = synthetic.to_device(synthetic.make_pairs(1, N, seed=seed + 1, D=conf["input_dim"], M=M), DEV)
    with torch.no_grad():
        pred = model(d)
    assert np.array_equal(pred["prune0"].cpu().numpy(), g["pred|prune0"])
    assert np.array_equal(pred["prune1"].cpu().numpy(), g["pred|prune1"])
    assert pred["log_assignment"].shape == g["pred|log_assignment"].shape
    np.testing.assert_allclose(pred["log_assignment"].cpu().numpy(), g["pred|log_assignment"], rtol=1e-3, atol=1e-3)
    assert np.array_equal(pred["matches0"].cpu().numpy(), g["pred|matches0"])
    assert np.array_equal(pred["matches1"].cpu().numpy(), g["pred|matches1"])
    np.testing.assert_allclose(pred["matching_scores0"].cpu().numpy(), g["pred|matching_scores0"], rtol=1e-3, atol=1e-6)
    # early stopping on the same model runs and stops no later than the last layer
    stop = _build(dict(conf, depth_confidence=0.95), synthetic.make_weights(conf, seed=seed), "bf16").eval()
    with torch.no_grad():
        ps = stop(d)
    assert 0 <= ps["stop_layer"] <= conf["n_layers"] - 1 and torch.isfinite(ps["log_assignment"]).all()


@pytest.mark.parametrize("D,H", [(128, 4), (256, 8)])
def test_training_step_replays_bit_identical(D, H):
    """MatcherTrainer captures the bf16 training step at head dim 32 as one CUDA graph; its replay computes what the
    eager step computes, bit for bit: the loss and every parameter after the Adam update.  Both batches have
    M = 192 != N = 256 points."""
    conf = dict(synthetic.DEFAULT_CONF, descriptor_dim=D, input_dim=D, num_heads=H, n_layers=2)
    w = synthetic.make_weights(conf, seed=61)
    batches = [synthetic.to_device(synthetic.make_pairs(2, 256, seed=62 + i, D=D, M=192), DEV) for i in range(2)]
    eager = MatcherTrainer(_build(conf, w, "bf16"), lr=1e-4)
    graphed = MatcherTrainer(_build(conf, w, "bf16"), lr=1e-4)
    graphed.capture(batches[0], torch.device(DEV))
    assert torch.equal(eager.fp.flat, graphed.fp.flat)
    for it, b in enumerate(batches):
        le, _ = eager.step(b)
        lg, _ = graphed.step_graphed(b)
        torch.cuda.synchronize()
        assert torch.isfinite(lg).all()
        assert torch.equal(le, lg), (it, le.item(), lg.item())
        assert torch.equal(eager.fp.flat, graphed.fp.flat), it


@pytest.mark.parametrize("D,H", [(128, 4), (256, 8)])
def test_training_reduces_loss(D, H):
    conf = dict(synthetic.DEFAULT_CONF, descriptor_dim=D, input_dim=D, num_heads=H, n_layers=3)
    model = _build(conf, synthetic.make_weights(conf, seed=71), "bf16")
    trainer = MatcherTrainer(model, lr=3e-4)
    data = synthetic.to_device(synthetic.make_pairs(4, 256, seed=72, D=D), DEV)
    first = last = None
    for _ in range(12):
        loss, _ = trainer.step(data)
        first = loss.item() if first is None else first
        last = loss.item()
    report(f"hd32 train D{D} H{H}", first=first, last=last)
    assert np.isfinite(last) and last < first - 0.05, (first, last)
