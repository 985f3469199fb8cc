"""GPU: the SuperGlue plugin (matchers/superglue.py) and its head kernels.

  1. the device-resident bin score: lgb200_sinkhorn_{fwd,bwd}_dev equal the host-scalar entry points bit for bit,
     with the strip cache on (B=1, N=2048: one work item per CTA) and off (B=4, N=2048);
  2. the NLL head on the dense Sinkhorn output (lgb200_ot_nll_fwd / _bwd) against fp64 torch;
  3. the filter statistics (lgb200_ot_filter_stats) against CPU torch.max with planted ties;
  4. the plugin against the fixture produced by the unmodified reference (tests/golden/superglue_l4_m150_n160.npz:
     fp64, training mode, forward + loss + backward, BatchNorm running statistics after the backward);
  5. a ragged size against the fp64 CPU oracle (tests/superglue_oracle.py);
  6. training, evaluation and the empty-keypoint branch;
  7. the whole training step captured as one CUDA graph by trainer.MatcherTrainer.

precision="fp32" is held to the north-star bar (matches bit-exact, log_assignment / sinkhorn_cost within 1e-4
relative, losses within 1e-3, gradients within 2e-3).  precision="bf16" rounds the GNN's GEMM and attention operands
to bf16 (the Sinkhorn head stays fp32); its tolerances are about three times the errors measured at the golden's size
on an H100 80GB HBM3 (700 W power limit):
    mode  log_assignment  sinkhorn_cost  losses (worst)  gradient norms (worst)  matches0 agreeing
    fp32  1.9e-7          5.2e-7         9.4e-8          1.0e-6                  all (bit-exact)
    bf16  1.4e-3          4.7e-3         4.5e-4          3.0e-2                  all
(relative errors against the fp64 golden; the fp32 mode agrees with the golden to ~1e-6, so the bf16 row is also its
distance from fp32.)
"""
import ast
import os

import numpy as np
import pytest
import torch

from gluefactory_b200 import ops, synthetic
from gluefactory_b200.matchers.superglue import SuperGlue
from tests.util import GOLDEN, check_grad_summary, rel_err, report

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _case():
    g = dict(np.load(os.path.join(GOLDEN, "superglue_l4_m150_n160.npz"), allow_pickle=False))
    conf = ast.literal_eval(str(g["meta|conf"]))
    B, M, N, seed = (int(g["meta|" + k]) for k in ("B", "M", "N", "seed"))
    return g, conf, B, M, N, seed


def _build(conf, seed, precision):
    model = SuperGlue(dict(conf, weights=None, precision=precision))
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=seed), strict=True)
    return model.to(DEV).train()


# ------------------------------------------------------------------------------------------ 1. device-resident alpha
@pytest.mark.parametrize("B,M,N", [(1, 2048, 2048), (4, 2048, 2048), (3, 150, 203)])
def test_sinkhorn_dev_entry_points_equal_host_scalar(B, M, N):
    g = torch.Generator(device=DEV).manual_seed(B * 7 + N)
    sim = torch.randn(B, M, N, device=DEV, generator=g)
    alpha = torch.tensor(0.73, device=DEV)
    iters = 50
    out_h, uh_h, vh_h = ops._log_optimal_transport_fwd(sim, float(alpha), iters, keep_potentials=True)
    out_d, uh_d, vh_d = ops._log_optimal_transport_fwd(sim, alpha, iters, keep_potentials=True)
    assert torch.equal(out_h, out_d) and torch.equal(uh_h, uh_d) and torch.equal(vh_h, vh_d)
    assert torch.equal(ops._log_optimal_transport_fwd(sim, alpha, iters), out_h)
    grad = torch.randn(B, M + 1, N + 1, device=DEV, generator=g)
    ds_h, da_h = ops._log_optimal_transport_bwd(sim, float(alpha), iters, grad, uh_h, vh_h)
    ds_d, da_d = ops._log_optimal_transport_bwd(sim, alpha, iters, grad, uh_h, vh_h)
    assert torch.equal(ds_h, ds_d) and torch.equal(da_h, da_d)
    assert da_d.is_cuda
    # and through autograd: a CUDA alpha tensor takes the device path with the same result
    s, a = sim.clone().requires_grad_(True), alpha.clone().requires_grad_(True)
    out = ops.log_optimal_transport(s, a, iters)
    assert torch.equal(out, out_h)
    out.backward(grad)
    assert torch.equal(s.grad, ds_h) and torch.equal(a.grad, da_h)


# ------------------------------------------------------------------------------------------ 2. NLL head
def _nll_inputs(B, M, N, seed):
    g = torch.Generator().manual_seed(seed)
    Z = -torch.rand(B, M + 1, N + 1, generator=g, dtype=torch.float64) * 8
    mask = torch.rand(B, M, N, generator=g) < 3.0 / N
    m0 = torch.where(torch.rand(B, M, generator=g) < 0.4, -1, torch.randint(0, N, (B, M), generator=g))
    m1 = torch.where(torch.rand(B, N, generator=g) < 0.4, -1, torch.randint(0, M, (B, N), generator=g))
    m0[0, :3] = -2  # ignored points are neither positive nor negative
    return Z, mask, m0, m1


@pytest.mark.parametrize("B,M,N", [(2, 150, 203), (3, 1, 7), (1, 333, 64), (4, 2048, 2048)])
def test_ot_nll_against_fp64(B, M, N):
    Z64, mask, m0, m1 = _nll_inputs(B, M, N, 100 + M)
    Z = Z64.float().to(DEV).requires_grad_(True)
    nll_pos, nll_neg, num_pos, num_neg = ops.ot_nll(Z, mask.to(DEV), m0.to(DEV), m1.to(DEV))
    # fp64 restatement of superglue.py:325-336 on the same fp32 values
    Zr = Z64.float().double().requires_grad_(True)
    pos = mask.double()
    n_pos = pos.sum((1, 2)).clamp(min=1.0)
    neg0, neg1 = (m0 == -1).double(), (m1 == -1).double()
    n_neg = (neg0.sum(1) + neg1.sum(1)).clamp(min=1.0)
    r_pos = -(Zr[:, :-1, :-1] * pos).sum((1, 2)) / n_pos
    r_neg = (-(Zr[:, :-1, -1] * neg0).sum(1) - (Zr[:, -1, :-1] * neg1).sum(1)) / n_neg
    torch.testing.assert_close(num_pos.cpu().double(), n_pos)
    torch.testing.assert_close(num_neg.cpu().double(), n_neg)
    torch.testing.assert_close(nll_pos.detach().cpu().double(), r_pos, rtol=1e-5, atol=1e-6)
    torch.testing.assert_close(nll_neg.detach().cpu().double(), r_neg, rtol=1e-5, atol=1e-6)
    # two calls: bit-identical
    again = ops.ot_nll(Z, mask.to(DEV), m0.to(DEV), m1.to(DEV))
    assert torch.equal(again[0], nll_pos) and torch.equal(again[1], nll_neg)
    # backward against fp64 autograd, including the zero corner and the zeros off the positives
    gw = torch.rand(B, dtype=torch.float64) + 0.5
    (0.5 * r_pos * gw + 0.5 * r_neg * gw).sum().backward()
    (0.5 * nll_pos * gw.float().to(DEV) + 0.5 * nll_neg * gw.float().to(DEV)).sum().backward()
    torch.testing.assert_close(Z.grad.cpu().double(), Zr.grad, rtol=1e-5, atol=1e-9)
    assert not Z.grad[:, -1, -1].any()
    # linear in the incoming gradient (GradScaler multiplies it): exact scaling by a power of two
    mk, n0, n1 = mask.to(DEV).to(torch.uint8), (m0 == -1).float().to(DEV), (m1 == -1).float().to(DEV)
    gp, gn = torch.rand(B, device=DEV), torch.rand(B, device=DEV)
    d1 = ops.ot_nll_bwd(mk, n0, n1, num_pos, num_neg, gp, gn)
    d8 = ops.ot_nll_bwd(mk, n0, n1, num_pos, num_neg, gp * 8, gn * 8)
    assert torch.equal(d8, d1 * 8)


# ------------------------------------------------------------------------------------------ 3. filter statistics
@pytest.mark.parametrize("B,M,N", [(2, 150, 203), (1, 2048, 2048), (3, 5, 1)])
def test_ot_filter_stats_first_index_ties(B, M, N):
    g = torch.Generator().manual_seed(M + N)
    Z = torch.randint(-6, 1, (B, M + 1, N + 1), generator=g).float()  # small integer range: ties everywhere
    Z[0, :, :] = -3.0  # a pair where every entry ties
    if M > 3 and N > 3:
        Z[-1, 2, 1] = Z[-1, 2, 3] = 5.0
    Z[:, -1, :] = 10.0  # dustbins larger than everything: must be ignored
    Z[:, :, -1] = 10.0
    rowmax, rowarg, colarg = ops.ot_filter_stats(Z.to(DEV))
    inner = Z[:, :-1, :-1]
    mx0, mx1 = inner.max(2), inner.max(1)
    assert torch.equal(rowmax.cpu(), mx0.values)
    assert torch.equal(rowarg.cpu().long(), mx0.indices)
    assert torch.equal(colarg.cpu().long(), mx1.indices)


# ------------------------------------------------------------------------------------------ 4. golden parity
def _golden_run(precision):
    g, conf, B, M, N, seed = _case()
    model = _build(conf, seed, precision)
    data = synthetic.to_device(synthetic.make_superglue_batch(B, M, N, seed + 1), DEV)
    pred = model(data)
    losses, metrics = model.loss(pred, data)
    assert metrics == {}
    losses["total"].mean().backward()
    return g, model, pred, losses


def test_superglue_fp32_matches_reference_golden():
    g, model, pred, losses = _golden_run("fp32")
    for k in ("matches0", "matches1"):
        assert np.array_equal(pred[k].cpu().numpy(), g["pred|" + k]), k
    errs = {k: rel_err(pred[k], torch.from_numpy(g["pred|" + k])) for k in ("log_assignment", "sinkhorn_cost")}
    for k in ("total", "assignment_nll", "nll_pos", "nll_neg", "num_matchable", "num_unmatchable", "bin_score"):
        errs["loss_" + k] = rel_err(losses[k], torch.from_numpy(g["loss|" + k]))
    grad_worst = 0.0
    for k, p in model.named_parameters():
        ref_norm = float(g[f"grad|{k}|norm"])
        if ref_norm < 1e-9:  # conv bias in front of a BatchNorm: zero gradient in theory, rounding noise in practice
            assert p.grad.norm().item() < 1e-4, k
            continue
        grad_worst = max(grad_worst, abs(p.grad.double().norm().item() - ref_norm) / ref_norm)
        check_grad_summary(g, k, p.grad, rtol=2e-3)
    report("superglue_golden_fp32", grad_norm_worst=grad_worst, **errs)
    assert errs["log_assignment"] < 1e-4 and errs["sinkhorn_cost"] < 1e-4, errs
    for k in ("total", "assignment_nll", "nll_pos", "nll_neg", "num_matchable", "num_unmatchable", "bin_score"):
        np.testing.assert_allclose(losses[k].detach().cpu().numpy(), g["loss|" + k], rtol=1e-3, err_msg=k)
    assert p.grad is not None and model.bin_score.grad is not None
    # running statistics: kenc once per image, every GNN MLP BatchNorm twice per image (the reference's checkpoint
    # recomputation in the backward)
    for k, v in model.state_dict().items():
        if "num_batches_tracked" in k:
            assert int(v) == int(g["bn|" + k]), k
        elif "running_" in k:
            np.testing.assert_allclose(v.cpu().numpy(), g["bn|" + k], rtol=1e-3, atol=1e-5, err_msg=k)


def test_superglue_bf16_against_reference_golden():
    g, model, pred, losses = _golden_run("bf16")
    errs = {k: rel_err(pred[k], torch.from_numpy(g["pred|" + k])) for k in ("log_assignment", "sinkhorn_cost")}
    loss_worst = max(rel_err(losses[k], torch.from_numpy(g["loss|" + k])) for k in ("total", "nll_pos", "nll_neg"))
    grad_worst = 0.0
    for k, p in model.named_parameters():
        ref_norm = float(g[f"grad|{k}|norm"])
        if ref_norm < 1e-9:
            continue
        grad_worst = max(grad_worst, abs(p.grad.double().norm().item() - ref_norm) / ref_norm)
    agree = (pred["matches0"].cpu() == torch.from_numpy(g["pred|matches0"])).float().mean().item()
    report("superglue_golden_bf16", loss_worst=loss_worst, grad_norm_worst=grad_worst, matches0_agree=agree, **errs)
    assert errs["log_assignment"] < 5e-3 and errs["sinkhorn_cost"] < 1.5e-2, errs
    assert loss_worst < 2e-3, loss_worst
    assert grad_worst < 0.1, grad_worst
    assert agree > 0.9, agree
    for k, v in model.state_dict().items():
        if "num_batches_tracked" in k:
            assert int(v) == int(g["bn|" + k]), k
        elif "running_" in k:
            np.testing.assert_allclose(v.cpu().numpy(), g["bn|" + k], rtol=3e-2, atol=1e-3, err_msg=k)


# ------------------------------------------------------------------------------------------ 5. ragged sizes
def test_superglue_ragged_against_oracle():
    """M = 150, N = 203 (no tile multiple), fp32 mode against the fp64 CPU oracle."""
    from tests import superglue_oracle as SO

    conf = {"GNN_layers": ["self", "cross"], "filter_threshold": 0.1}
    model = _build(conf, 41, "fp32")
    d = synthetic.make_superglue_batch(2, 150, 203, 43)
    data = synthetic.to_device(d, DEV)
    w = {k: (v.detach().double().cpu() if v.is_floating_point() else v.cpu()) for k, v in model.state_dict().items()}
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    params = {k: w[k].clone().requires_grad_(True) for k, _ in model.named_parameters()}
    d64 = {k: ({kk: vv.double() for kk, vv in v.items()} if isinstance(v, dict) else
               (v.double() if v.is_floating_point() else v)) for k, v in d.items()}
    stats = {}
    rp = SO.superglue_forward({**w, **params}, d64, dict(conf), stats)
    rl = SO.superglue_loss({**w, **params}, rp, d64, conf)
    rl["total"].mean().backward()
    assert torch.equal(pred["matches0"].cpu(), rp["matches0"]) and torch.equal(pred["matches1"].cpu(), rp["matches1"])
    assert rel_err(pred["log_assignment"], rp["log_assignment"]) < 1e-4
    assert rel_err(pred["sinkhorn_cost"], rp["sinkhorn_cost"]) < 1e-4
    assert rel_err(losses["total"], rl["total"]) < 1e-4
    # element-wise gradient errors, measured on an H100: median 1.1e-3, worst 4.8e-3 (layer 0's attention projections,
    # small gradients formed by cancellation behind 50 fp32 Sinkhorn iterations)
    gerr = {k: rel_err(p.grad, params[k].grad) for k, p in model.named_parameters() if params[k].grad.norm().item() >= 1e-9}
    worst = max(gerr, key=gerr.get)
    report("superglue_ragged_fp32", grad_worst=gerr[worst], grad_worst_param=worst,
           grad_median=float(np.median(list(gerr.values()))))
    assert gerr[worst] < 1e-2, (worst, gerr[worst])
    for k, v in SO.running_stats(w, stats, conf).items():
        got = model.state_dict()[k].cpu()
        if "num_batches_tracked" in k:
            assert int(got) == int(v), k
        else:
            assert rel_err(got, v) < 1e-4, k


# ------------------------------------------------------------------------------------------ 6. training / evaluation
def test_superglue_trains_and_evaluates():
    model = _build({"GNN_layers": ["self", "cross"] * 2}, 51, "bf16")
    data = synthetic.to_device(synthetic.make_superglue_batch(2, 256, 320, 52), DEV)
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
        losses, metrics = model.loss(pred, data)
    assert {"match_recall", "match_precision", "average_precision"} <= set(metrics)
    assert set(losses) == {"total", "assignment_nll", "nll_pos", "nll_neg", "num_matchable", "num_unmatchable",
                           "bin_score"}
    # no keypoints in one view: the reference's four outputs
    empty = dict(data, keypoints1=data["keypoints1"][:, :0], descriptors1=data["descriptors1"][:, :0],
                 keypoint_scores1=data["keypoint_scores1"][:, :0])
    out = model(empty)
    assert set(out) == {"matches0", "matches1", "matching_scores0", "matching_scores1"}
    assert out["matches0"].dtype == torch.int32 and (out["matches0"] == -1).all() and out["matches1"].shape == (2, 0)
    assert not out["matching_scores0"].any()
    # image_size absent: the image shape is used instead
    no_size = {**data, "view0": {"image": torch.zeros(2, 1, 1024, 1024, device=DEV)},
               "view1": {"image": torch.zeros(2, 1, 1024, 1024, device=DEV)}}
    with torch.no_grad():
        assert torch.equal(model(no_size)["matches0"], pred["matches0"])


# ------------------------------------------------------------------------------------------ 7. CUDA graph
def test_superglue_training_step_replays_as_one_cuda_graph():
    """Forward, the Sinkhorn head (cooperative launches, bin score read on the device), the NLL, backward and flat Adam
    hold no host read-back, so trainer.MatcherTrainer captures the step; replay == eager steps."""
    from gluefactory_b200.trainer import MatcherTrainer

    g, conf, B, M, N, seed = _case()
    data = synthetic.to_device(synthetic.make_superglue_batch(B, 152, N, seed + 1), DEV)
    eager = MatcherTrainer(_build(conf, seed, "bf16"), lr=1e-4)
    graphed = MatcherTrainer(_build(conf, seed, "bf16"), lr=1e-4)
    graphed.capture(data, torch.device(DEV))
    for it in range(3):
        le, _ = eager.step(data)
        lg, _ = graphed.step_graphed(data)
        assert torch.isfinite(lg).all()
        assert abs(le.item() - lg.item()) < (1e-5 if it == 0 else 2e-3) * abs(le.item()), (it, le.item(), lg.item())


def test_two_view_pipeline_runs_superglue():
    """A glue-factory config selecting the plugin builds through TwoViewPipeline and runs forward and loss."""
    import sys

    saved = list(sys.path)
    try:
        from oracle import stage_reference

        if stage_reference.import_reference() is None:
            pytest.skip("reference not staged under oracle/_ref")
        from gluefactory.models.two_view_pipeline import TwoViewPipeline

        pipe = TwoViewPipeline({"matcher": {"name": "gluefactory_b200.matchers.superglue", "weights": None,
                                            "GNN_layers": ["self", "cross"]},
                                "extractor": {"name": None}, "allow_no_extract": True}).to(DEV).train()
        data = synthetic.to_device(synthetic.make_superglue_batch(2, 128, 160, 7), DEV)
        pred = pipe(data)
        losses, metrics = pipe.loss(pred, data)
        assert torch.isfinite(losses["total"]).all()
    finally:
        sys.path[:] = saved
