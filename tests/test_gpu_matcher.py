"""GPU: the drop-in matcher (forward + loss + backward through the C ABI) against the golden
fixtures produced by the unmodified reference, and against the oracle at larger sizes.

precision="fp32" must meet the north-star bar on the fp32 reference: assignment indices bit-exact,
log-scores, losses and gradients within 1e-3 relative.  precision="bf16" (tensor-core operands) is
held to the same bar against an oracle evaluated on bf16-rounded GEMM operands at kernel level
(tests/test_gpu_kernels.py) and to 3e-2 here end to end (bf16 has 8 mantissa bits; nine residual
layers compound), with index agreement required wherever the reference's top-2 margin is > 0.05.
"""
import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.lightglue import LightGlue
from gluefactory_b200.trainer import MatcherTrainer
from oracle import lightglue_oracle as O
from tests.util import CASES, EXTRA_CASES, check_grad_summary, load_case, mirror_oracle, rel_err, report

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _build(conf, weights, precision):
    model = LightGlue(dict(conf, precision=precision))
    missing, unexpected = model.load_state_dict({k: v.float() for k, v in weights.items()}, strict=False)
    assert not unexpected and missing in ([], ["confidence_thresholds"])
    return model.to(DEV).train()


def _f32(data):
    return synthetic.to_device({k: ({kk: vv.float() for kk, vv in v.items()} if isinstance(v, dict) else
                                    (v.float() if v.is_floating_point() else v)) for k, v in data.items()}, DEV)


@pytest.mark.parametrize("name", CASES[:4] + EXTRA_CASES)
def test_fp32_path_matches_reference_golden(name):
    g, conf, w, data = load_case(name)
    model = _build(conf, w, "fp32")
    d = _f32(data)
    pred = model(d)
    losses, _ = model.loss(pred, d)
    losses["total"].mean().backward()
    assert np.array_equal(pred["matches0"].cpu().numpy(), g["pred|matches0"])
    assert np.array_equal(pred["matches1"].cpu().numpy(), g["pred|matches1"])
    np.testing.assert_allclose(pred["log_assignment"].cpu().numpy(), g["pred|log_assignment"], rtol=1e-3, atol=1e-3)
    np.testing.assert_allclose(pred["matching_scores0"].cpu().numpy(), g["pred|matching_scores0"], rtol=1e-3, atol=1e-6)
    for k in ["total", "last", "assignment_nll", "nll_pos", "nll_neg", "num_matchable", "num_unmatchable",
              "confidence", "row_norm"]:
        np.testing.assert_allclose(losses[k].detach().cpu().numpy(), g["loss|" + k], rtol=1e-3, err_msg=k)
    for k, p in model.named_parameters():
        check_grad_summary(g, k, p.grad, rtol=1e-3)


def test_fp32_path_full_size_forward():
    g, conf, w, data = load_case(CASES[4])
    model = _build(conf, w, "fp32").eval()
    with torch.no_grad():
        pred = model(_f32(data))
    assert np.array_equal(pred["matches0"].cpu().numpy(), g["pred|matches0"])
    assert np.array_equal(pred["matches1"].cpu().numpy(), g["pred|matches1"])
    np.testing.assert_allclose(pred["log_assignment"][:, ::8, ::8].cpu().numpy(), g["pred|log_assignment"],
                               rtol=1e-3, atol=1e-3)
    assert pred["ref_descriptors0"].shape[1] == 1  # eval keeps only the last layer (lightglue.py:485)


@pytest.mark.parametrize("name", CASES[2:4])
def test_bf16_path_close_to_reference_golden(name):
    g, conf, w, data = load_case(name)
    model = _build(conf, w, "bf16")
    d = _f32(data)
    pred = model(d)
    losses, _ = model.loss(pred, d)
    losses["total"].mean().backward()
    la = pred["log_assignment"].cpu().double().numpy()
    assert np.abs(la - g["pred|log_assignment"]).max() < 0.15
    np.testing.assert_allclose(losses["total"].detach().cpu().numpy(), g["loss|total"], rtol=2e-2)
    # indices: must agree wherever the reference's row top-2 margin is comfortably above bf16 noise
    ref = torch.from_numpy(g["pred|log_assignment"])[:, :-1, :-1]
    top2 = ref.topk(2, dim=2).values
    safe = (top2[..., 0] - top2[..., 1]) > 0.3
    got = torch.from_numpy(la)[:, :-1, :-1].max(2).indices
    assert torch.equal(got[safe], ref.max(2).indices[safe])
    worst = 0.0
    for k, p in model.named_parameters():
        ref_norm = float(g[f"grad|{k}|norm"])
        worst = max(worst, abs(p.grad.double().norm().item() - ref_norm) / max(ref_norm, 1e-12))
    assert worst < 0.1, worst


# fp32 path against fp64 at the two shapes below, bound on the log-assignment, each loss entry and each parameter
# gradient.  Measured on an H100 80GB HBM3 (400 W limit), worst of both shapes: log-assignment 9.8e-8, loss entries
# 7.3e-8, gradients 2.7e-6 (the shared cross-attention to_qk bias).
FP32_VS_FP64 = 2e-5


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("M,N", [(192, 192), (150, 203)])
def test_ragged_sizes_against_oracle(M, N, precision):
    """Forward, loss and backward against the fp64 oracle at M == N (both images in one launch) and at M != N, neither
    a multiple of the tile sizes (the reference supports any keypoint count).  bf16 is also held to the oracle evaluated
    with the CUDA path's bf16 rounding model (O.Bf16Mirror)."""
    conf = dict(synthetic.DEFAULT_CONF, n_layers=2)
    w = synthetic.make_weights(conf, seed=21)
    data = synthetic.make_pairs(2, N, seed=22, M=M)
    model = _build(conf, w, precision)
    d = synthetic.to_device(data, DEV)
    pred = model(d)
    losses, _ = model.loss(pred, d)
    losses["total"].mean().backward()
    w64 = {k: v.double().requires_grad_(True) for k, v in w.items()}
    d64 = {k: ({kk: vv.double() for kk, vv in v.items()} if isinstance(v, dict) else
               (v.double() if v.is_floating_point() else v)) for k, v in data.items()}
    rp = O.lightglue_forward(w64, d64, conf)
    rl = O.lightglue_loss(w64, rp, d64, conf)
    rl["total"].mean().backward()
    e_la = rel_err(pred["log_assignment"], rp["log_assignment"])
    e_loss = {k: rel_err(losses[k], rl[k]) for k in rl if torch.is_tensor(rl[k])}
    e_grad = {k: rel_err(p.grad, w64[k].grad) for k, p in model.named_parameters()}
    report(f"ragged:{precision}:M{M}:N{N}:fp64", la=e_la, loss_max=max(e_loss.values()),
           loss_max_key=max(e_loss, key=e_loss.get), grad_max=max(e_grad.values()), grad_max_key=max(e_grad, key=e_grad.get))
    if precision == "fp32":
        assert torch.equal(pred["matches0"].cpu(), rp["matches0"])
        assert e_la < FP32_VS_FP64, e_la
        for k, e in e_loss.items():
            assert e < FP32_VS_FP64, (k, e)
        for k, e in e_grad.items():
            assert e < FP32_VS_FP64, (k, e)
        return
    assert e_loss["total"] < 3e-2 and e_la < 3e-2, (e_loss["total"], e_la)
    for k, e in e_grad.items():
        assert e < 0.15, (k, e)
    mp, ml, mg = mirror_oracle(conf, w, data)
    m_la = rel_err(pred["log_assignment"], mp["log_assignment"])
    m_loss = {k: rel_err(losses[k], ml[k]) for k in ml if torch.is_tensor(ml[k])}
    m_grad = {k: rel_err(p.grad, mg[k]) for k, p in model.named_parameters()}
    report(f"ragged:bf16:M{M}:N{N}:mirror", la=m_la, loss_max=max(m_loss.values()),
           loss_max_key=max(m_loss, key=m_loss.get), grad_max=max(m_grad.values()), grad_max_key=max(m_grad, key=m_grad.get))
    assert m_la < 2e-2, m_la
    for k, e in m_loss.items():
        assert e < 2e-2, (k, e)
    for k, e in m_grad.items():
        assert e < 0.1, (k, e)


def test_training_reduces_loss_and_eval_metrics():
    conf = dict(synthetic.DEFAULT_CONF, n_layers=3)
    model = _build(conf, synthetic.make_weights(conf, seed=31), "bf16")
    trainer = MatcherTrainer(model, lr=3e-4)
    data = synthetic.to_device(synthetic.make_pairs(4, 256, seed=32), DEV)
    first = last = None
    for it in range(12):
        loss, _ = trainer.step(data)
        first = loss.item() if first is None else first
        last = loss.item()
    assert np.isfinite(last) and last < first - 0.05, (first, last)
    model.eval()
    with torch.no_grad():
        pred = model(data)
        losses, metrics = model.loss(pred, data)
    assert set(metrics) == {"match_recall", "match_precision", "accuracy", "average_precision"}
    assert "confidence" not in losses


def test_eval_mode_loss_uses_last_head():
    """Validation loss (train.py:92-93): in eval mode only the last layer's state is stacked (lightglue.py:485) and
    the loss must still apply the LAST assignment head (lightglue.py:588), not head 0.  Golden = the reference in
    eval mode (tests/golden/eval_loss.npz)."""
    import ast
    import os

    from tests.util import GOLDEN

    g = dict(np.load(os.path.join(GOLDEN, "eval_loss.npz")))
    conf = ast.literal_eval(str(g["meta|conf"]))
    B, N, seed = int(g["meta|B"]), int(g["meta|N"]), int(g["meta|seed"])
    model = _build(conf, synthetic.make_weights(conf, seed=seed), "fp32").eval()
    d = _f32(synthetic.make_pairs(B, N, seed=seed + 1, dtype=torch.float64))
    with torch.no_grad():
        pred = model(d)
        losses, metrics = model.loss(pred, d)
    for k in ["total", "last", "assignment_nll", "nll_pos", "nll_neg", "num_matchable", "num_unmatchable", "row_norm"]:
        np.testing.assert_allclose(losses[k].cpu().numpy(), g["loss|" + k], rtol=1e-3, err_msg=k)
    assert "confidence" not in losses
    for k in ["match_recall", "match_precision", "accuracy", "average_precision"]:
        np.testing.assert_allclose(metrics[k].cpu().numpy(), g["metric|" + k], rtol=1e-3, atol=1e-6, err_msg=k)


def test_adaptive_point_pruning_matches_reference():
    """SURVEY 8f row 4: inference-time point pruning (lightglue.py:461-526) against the reference in eval mode (fp32;
    tests/golden/adaptive_prune.npz, every pruning decision clears its threshold by > 2e-4): the same points survive
    every layer (prune0/1), the same pruned log-assignment, the same matches scattered back to the full sets."""
    import ast
    import os

    from tests.util import GOLDEN

    g = dict(np.load(os.path.join(GOLDEN, "adaptive_prune.npz")))
    conf = ast.literal_eval(str(g["meta|conf"]))
    seed, M, N = int(g["meta|seed"]), int(g["meta|M"]), int(g["meta|N"])
    model = _build(conf, synthetic.make_weights(conf, seed=seed), "fp32").eval()
    d = synthetic.to_device(synthetic.make_pairs(1, N, seed=seed + 1, M=M), DEV)
    with torch.no_grad():
        pred = model(d)
    assert np.array_equal(pred["prune0"].cpu().numpy(), g["pred|prune0"]) and np.array_equal(pred["prune1"].cpu().numpy(), g["pred|prune1"])
    assert pred["log_assignment"].shape == g["pred|log_assignment"].shape
    np.testing.assert_allclose(pred["log_assignment"].cpu().numpy(), g["pred|log_assignment"], rtol=1e-3, atol=1e-3)
    assert np.array_equal(pred["matches0"].cpu().numpy(), g["pred|matches0"])
    assert np.array_equal(pred["matches1"].cpu().numpy(), g["pred|matches1"])
    np.testing.assert_allclose(pred["matching_scores0"].cpu().numpy(), g["pred|matching_scores0"], rtol=1e-3, atol=1e-6)
    # the loss needs every point: a pruned pred, or one from elsewhere, is refused
    with pytest.raises(ValueError, match="pruning"):
        model.loss(pred, d)
    with pytest.raises(ValueError, match="own forward"):
        model.loss({k: v for k, v in pred.items() if not k.startswith("_b200")}, d)
    # bf16 path: same code, pruning counts within a few points of the fp32 path
    mb = _build(conf, synthetic.make_weights(conf, seed=seed), "bf16").eval()
    with torch.no_grad():
        pb = mb(d)
    assert abs(int((pb["prune0"] == conf["n_layers"]).sum()) - int((pred["prune0"] == conf["n_layers"]).sum())) <= 8


def test_adaptive_early_stop():
    """Early stopping (lightglue.py:486-490, 560-571): with confident token heads the matcher stops after the first
    layer and uses that layer's assignment head; with depth_confidence out of reach it runs all layers and equals the
    plain forward."""
    conf = dict(synthetic.DEFAULT_CONF, n_layers=4, depth_confidence=0.9)
    w = synthetic.make_weights(conf, seed=77)
    d = synthetic.to_device(synthetic.make_pairs(1, 192, seed=78), DEV)
    for i in range(3):
        w[f"token_confidence.{i}.token.0.bias"] = torch.tensor([6.0])  # sigmoid(6 +- small) > every threshold
        w[f"token_confidence.{i}.token.0.weight"] = w[f"token_confidence.{i}.token.0.weight"] * 0.01
    model = _build(conf, w, "fp32").eval()
    with torch.no_grad():
        pred = model(d)
        assert pred["stop_layer"] == 0
        # same result as a one-layer model that uses head 0
        w1 = {k: v for k, v in w.items() if k.startswith(("posenc", "transformers.0.", "log_assignment.0."))}
        x_ref = _build(dict(conf, n_layers=1, depth_confidence=-1), w1, "fp32").eval()(d)
    assert torch.equal(pred["matches0"], x_ref["matches0"])
    np.testing.assert_allclose(pred["log_assignment"].cpu().numpy(), x_ref["log_assignment"].cpu().numpy(), rtol=1e-5, atol=1e-5)
    model2 = _build(dict(conf, depth_confidence=1.5), w, "fp32").eval()
    plain = _build(dict(conf, depth_confidence=-1), w, "fp32").eval()
    with torch.no_grad():
        a, b = model2(d), plain(d)
        (la, ma), (lb, mb) = model2.loss(a, d), plain.loss(b, d)
    assert a["stop_layer"] == 3 and torch.equal(a["matches0"], b["matches0"])
    assert la.keys() == lb.keys() and ma.keys() == mb.keys()
    for k in lb:
        assert torch.equal(la[k], lb[k]), k
    for k in mb:
        assert torch.equal(ma[k], mb[k]), k


def test_nan_propagates_to_loss():
    """train.py:477-480 skips the step on a NaN loss; the kernels must not trap or hide it."""
    conf = dict(synthetic.DEFAULT_CONF, n_layers=1)
    model = _build(conf, synthetic.make_weights(conf, seed=41), "fp32")
    data = synthetic.to_device(synthetic.make_pairs(1, 128, seed=42), DEV)
    data["descriptors0"][0, 5, 7] = float("nan")
    pred = model(data)
    losses, _ = model.loss(pred, data)
    assert torch.isnan(losses["total"]).all()


def test_cuda_graph_step_matches_eager_step():
    """The captured-graph replay of the training step must produce the same parameters as eager steps."""
    conf = dict(synthetic.DEFAULT_CONF, n_layers=2)
    batches = [synthetic.to_device(synthetic.make_pairs(2, 256, seed=50 + i), DEV) for i in range(3)]

    host = [{k: (v.cpu().pin_memory() if torch.is_tensor(v) else {kk: vv.cpu().pin_memory() for kk, vv in v.items()})
             for k, v in b.items()} for b in batches]

    def run(graphed, prefetch=False):
        model = _build(conf, synthetic.make_weights(conf, seed=51), "bf16")
        tr = MatcherTrainer(model, lr=1e-3)
        tr.step(batches[0])  # one eager step in both runs (it is also the capture warm-up)
        if graphed:
            tr.capture(batches[0], DEV, warmup=0)
        losses = []
        for i, b in enumerate(batches):
            if prefetch:  # pinned host batches, the next one copied on the side stream during this step
                loss, _ = tr.step_graphed(host[i], prefetch=host[i + 1] if i + 1 < len(host) else None)
            else:
                loss, _ = tr.step_graphed(b) if graphed else tr.step(b)
            losses.append(loss.item())
        return tr.fp.flat.clone(), losses

    p_eager, l_eager = run(False)
    p_graph, l_graph = run(True)
    np.testing.assert_allclose(l_graph, l_eager, rtol=1e-5)
    assert rel_err(p_graph, p_eager) < 1e-5
    p_pre, l_pre = run(True, prefetch=True)
    np.testing.assert_allclose(l_pre, l_graph, rtol=1e-6)
    assert rel_err(p_pre, p_graph) < 1e-6
