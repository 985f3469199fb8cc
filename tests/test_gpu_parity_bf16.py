"""GPU: parity of the MEASURED path (precision = bf16: wgmma attention / GEMM kernels) at the shapes it is
benchmarked on, under two contracts:

(A) "same autocast dtype" contract (SURVEY.md section 7, hard part 1b).  tests/golden/ac_*.npz hold, per output /
    loss entry / parameter gradient, how far the UNMODIFIED reference moves from its own fp64 result when it is
    run the way `train.py --mp bfloat16` runs it (fp32 module under torch.autocast(bfloat16), train.py:468-472).
    The CUDA bf16 path must be at least that close to the same fp64 golden.

(B) rounding-model contract.  The oracle evaluated with `rnd=O.Bf16Mirror()` rounds to bf16 exactly where the CUDA
    path stores / reads bf16 (operands, Linear outputs, gradients of bf16-stored tensors).  Against that oracle the
    kernels are held to tight tolerances at N = 2048 / L = 9 (BASELINE configs[2], the bench shape: 32 key tiles
    per query tile, the 4-stage TMA ring wraps 8 times, two CTAs per SM) and N = 1024 / L = 9 (configs[1]) to the
    bf16 noise floor (measured in the test: two valid rounding models differ by ~1.5e-3 rel. on the log-scores), losses
    2e-3 rel (measured 5e-5), row / column argmax equal wherever the model's top-2 margin exceeds 0.6.

(C) attention kernels alone at the bench shape (B=2 pairs -> 4 sequences x 4 heads x N=2048, self and kv_shift) against
    an fp64 evaluation of the same bf16 operands.
"""
import os

import numpy as np
import pytest
import torch

from gluefactory_b200 import ops, synthetic
from gluefactory_b200.matchers.lightglue import LightGlue
from oracle import lightglue_oracle as O
from tests.util import GOLDEN, load_case, mirror_oracle, probe_index, rel_err, report

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _build(conf, weights, precision="bf16"):
    model = LightGlue(dict(conf, precision=precision))
    missing, unexpected = model.load_state_dict({k: v.float() for k, v in weights.items()}, strict=False)
    assert not unexpected and missing in ([], ["confidence_thresholds"])
    return model.to(DEV).train()


def _cast(data, dtype):
    return {k: ({kk: vv.to(dtype) for kk, vv in v.items()} if isinstance(v, dict) else
                (v.to(dtype) if v.is_floating_point() else v)) for k, v in data.items()}


def _run_gpu(conf, w, data):
    model = _build(conf, w)
    d = synthetic.to_device(_cast(data, torch.float32), DEV)
    pred = model(d)
    losses, _ = model.loss(pred, d)
    losses["total"].mean().backward()
    return model, pred, losses


# ------------------------------------------------------------------------------------------------ (A)
AC_CASES = ["lg_d256_l3_n160", "lg_disk_d256_l2_n128", "lg_full_l9_n512"]


def _oracle_fp64(conf, w, data):
    w64 = {k: v.double().clone().requires_grad_(True) for k, v in w.items()}
    d64 = _cast(data, torch.float64)
    pred = O.lightglue_forward(w64, d64, conf)
    losses = O.lightglue_loss(w64, pred, d64, conf, training=True)
    losses["total"].mean().backward()
    return pred, losses, {k: p.grad for k, p in w64.items()}


@pytest.mark.parametrize("name", AC_CASES)
def test_bf16_path_at_least_as_close_as_reference_autocast(name):
    """Single scalars are one draw of the rounding noise each, so the comparison is made on aggregates: the whole
    log-assignment matrix, the loss entries as a vector, the parameter gradients as a population."""
    g, conf, w, data = load_case(name)
    ac = dict(np.load(os.path.join(GOLDEN, "ac_" + name + ".npz")))
    # fp64 truth: the oracle, pinned to the reference at 1e-9 on this very case (tests/test_oracle_golden.py)
    p64, l64, g64 = _oracle_fp64(conf, w, data)
    model, pred, losses = _run_gpu(conf, w, data)
    e_la = rel_err(pred["log_assignment"], p64["log_assignment"])
    maxabs = (pred["log_assignment"].double().cpu() - p64["log_assignment"]).abs().max().item()
    keys = ["total", "assignment_nll", "nll_pos", "nll_neg", "row_norm", "confidence"]
    e_loss = np.array([rel_err(losses[k], l64[k]) for k in keys])
    a_loss = np.array([float(ac["err|loss|" + k]) for k in keys])
    inner64 = p64["log_assignment"][:, :-1, :-1]
    top2 = inner64.topk(2, dim=2).values
    safe = (top2[..., 0] - top2[..., 1]) > float(ac["idx|row_safe_margin"])
    got = pred["log_assignment"][:, :-1, :-1].max(2).indices.cpu()
    agree = (got == inner64.max(2).indices).double().mean().item()
    errs_ac = {k[len("err|grad|"):]: float(v) for k, v in ac.items() if k.startswith("err|grad|")}
    ours = {}
    for k, p in model.named_parameters():
        r = g64[k]
        if r.numel() <= 4096:
            ours[k] = rel_err(p.grad, r)
        else:
            idx = probe_index(r.numel())
            ours[k] = rel_err(p.grad.reshape(-1).cpu()[idx], r.reshape(-1)[idx])
    names = sorted(ours)
    eo, ea = np.array([ours[k] for k in names]), np.array([errs_ac[k] for k in names])
    ratio = eo / np.maximum(ea, 1e-30)
    report("A:" + name, la_rel=e_la, la_rel_ac=float(ac["err|log_assignment"]), la_maxabs=maxabs,
           la_maxabs_ac=float(ac["err|log_assignment_maxabs"]), loss_rms=float(np.sqrt((e_loss ** 2).mean())),
           loss_rms_ac=float(np.sqrt((a_loss ** 2).mean())), loss_total=float(e_loss[0]), loss_total_ac=float(a_loss[0]),
           grad_median=float(np.median(eo)), grad_median_ac=float(np.median(ea)), grad_max=float(eo.max()),
           grad_max_ac=float(ea.max()), grad_ratio_median=float(np.median(ratio)), grad_ratio_max=float(ratio.max()),
           grad_ratio_max_key=names[int(ratio.argmax())], frac_params_better=float((ratio <= 1).mean()), agree=agree,
           agree_ac=float(ac["idx|row_agree_frac"]))
    # outputs
    assert e_la <= float(ac["err|log_assignment"]), (e_la, float(ac["err|log_assignment"]))
    assert maxabs <= float(ac["err|log_assignment_maxabs"]), (maxabs, float(ac["err|log_assignment_maxabs"]))
    # losses: the headline entry on its own, the rest as a vector
    assert e_loss[0] <= a_loss[0], (e_loss[0], a_loss[0])
    assert np.sqrt((e_loss ** 2).mean()) <= np.sqrt((a_loss ** 2).mean()), (e_loss, a_loss)
    # indices: every row argmax the autocast reference keeps by margin, and at least its overall agreement
    assert torch.equal(got[safe], inner64.max(2).indices[safe])
    assert agree >= float(ac["idx|row_agree_frac"]), (agree, float(ac["idx|row_agree_frac"]))
    # gradients as a population: typical (median) and mean error no larger than the autocast reference's, a clear
    # majority of the parameters individually closer.  Single parameters are one noise draw each
    # (the worst ratio is always the shared to_qk bias, whose gradient is a near-cancellation of the two attention
    # directions summed over all tokens), so the worst one is only held to twice the reference's worst.
    assert np.median(eo) <= np.median(ea), (np.median(eo), np.median(ea))
    assert eo.mean() <= ea.mean(), (eo.mean(), ea.mean())
    assert (ratio <= 1).mean() >= 0.75, float((ratio <= 1).mean())
    assert eo.max() <= 2.0 * ea.max(), (names[int(eo.argmax())], eo.max(), ea.max())


# ------------------------------------------------------------------------------------------------ (B)
def _margin_safe(la, dim, margin):
    inner = la[:, :-1, :-1]
    top2 = inner.topk(2, dim=dim).values
    t0, t1 = top2.select(dim, 0), top2.select(dim, 1)
    return (t0 - t1) > margin


@pytest.mark.parametrize("N,seed", [(2048, 71), (1024, 72)])
def test_bf16_path_at_bench_shape_against_rounding_model(N, seed):
    """Full matcher at the benchmark shapes.  bf16 rounding noise is amplified by nine residual layers to a floor of
    ~1.5e-3 relative on the log-scores REGARDLESS of which (valid) set of rounding points is used -- two CPU rounding
    models differ from each other by as much as each differs from fp64 -- so the tolerances below
    are that floor with ~2x head-room; an indexing / pipeline bug at N = 2048 shows up as O(1) errors.  At N = 1024 the
    floor is measured in the test itself and the CUDA path must be no further from the model than a second model is."""
    conf = dict(synthetic.DEFAULT_CONF)  # L = 9, H = 4, d = 256
    w = synthetic.make_weights(conf, seed=seed)
    data = synthetic.make_pairs(1, N, seed=seed + 1)
    model, pred, losses = _run_gpu(conf, w, data)
    rp, rl, rg = mirror_oracle(conf, w, data)
    la, rla = pred["log_assignment"].float().cpu(), rp["log_assignment"]
    d_la = (la - rla).abs()
    la_rel = (d_la.norm() / rla.norm()).item()
    gerr = {k: rel_err(p.grad, rg[k]) for k, p in model.named_parameters()}
    m0_agree = (pred["matches0"].cpu() == rp["matches0"]).double().mean().item()
    report(f"B:N{N}", la_maxabs=d_la.max().item(), la_rel=la_rel,
           loss_rel=rel_err(losses["total"], rl["total"]), conf_rel=rel_err(losses["confidence"], rl["confidence"]),
           grad_max=max(gerr.values()), grad_max_key=max(gerr, key=gerr.get),
           grad_median=float(np.median(list(gerr.values()))), m0_agree=m0_agree)
    assert d_la.max().item() < 0.3 and la_rel < 3e-3, (d_la.max().item(), la_rel)
    for k in ["total", "assignment_nll", "nll_pos", "nll_neg", "confidence", "row_norm"]:
        assert rel_err(losses[k], rl[k]) < 2e-3, (k, rel_err(losses[k], rl[k]))
    # indices: identical wherever the model's own top-2 margin is above twice the score tolerance
    for dim in (2, 1):
        safe = _margin_safe(rla, dim, 0.6)
        got = la[:, :-1, :-1].max(dim).indices
        want = rla[:, :-1, :-1].max(dim).indices
        assert torch.equal(got[safe], want[safe])
    assert m0_agree > 0.98, m0_agree
    assert max(gerr.values()) < 5e-2 and np.median(list(gerr.values())) < 6e-3, (max(gerr, key=gerr.get), max(gerr.values()))
    if N == 1024:  # the floor, measured: a second valid rounding model (operand rounding only) against the first
        rp2, _, rg2 = mirror_oracle(conf, w, data, rnd=O.bf16_round)
        floor_la = ((rp2["log_assignment"] - rla).norm() / rla.norm()).item()
        floor_g = float(np.median([rel_err(rg2[k], rg[k]) for k in rg]))
        report(f"B:N{N}:floor", la_rel_between_models=floor_la, grad_median_between_models=floor_g)
        assert la_rel <= 1.5 * floor_la, (la_rel, floor_la)
        assert np.median(list(gerr.values())) <= 1.5 * floor_g, (np.median(list(gerr.values())), floor_g)
    # batch invariance: the same pair inside a batch of 3 (several waves of CTAs) gives the same prediction
    more = synthetic.make_pairs(3, N, seed=seed + 1)
    d3 = synthetic.to_device(_cast(more, torch.float32), DEV)
    with torch.no_grad():
        pred3 = model(d3)
    assert torch.equal(pred3["matches0"][0], pred["matches0"][0])
    assert (pred3["log_assignment"][0] - pred["log_assignment"][0]).abs().max().item() < 1e-5


# ------------------------------------------------------------------------------------------------ (C)
def _attn_ref64(q, k, v, shift):
    q, k, v = (t.double().permute(0, 2, 1, 3) for t in (q, k, v))
    B = q.shape[0]
    idx = (torch.arange(B, device=q.device) + shift) % B
    s = q @ k[idx].transpose(-1, -2) / 8.0
    return (torch.softmax(s, -1) @ v[idx]).permute(0, 2, 1, 3), torch.logsumexp(s, -1)


@pytest.mark.parametrize("shift", [0, 2])
def test_attention_kernels_at_bench_shape(shift):
    """4 sequences (2 pairs) x 4 heads x N = 2048: forward, lse, dQ, dK, dV of the wgmma kernels against fp64 on the
    same bf16 operands (self attention: shift 0; cross attention: keys of sequence (b + 2) % 4)."""
    B, N, H = 4, 2048, 4
    g = torch.Generator().manual_seed(5 + shift)
    mk = lambda s: (torch.randn(B, N, H, 64, generator=g) * s).to(torch.bfloat16).to(DEV)  # noqa: E731
    q, k, v, go = mk(1.5).requires_grad_(True), mk(1.5).requires_grad_(True), mk(1.0).requires_grad_(True), mk(1.0)
    out, lse = ops.attn_fwd(q.detach(), k.detach(), v.detach(), shift, 0.125)
    dq, dk, dv = ops.attn_bwd(q.detach(), k.detach(), v.detach(), out, lse, go, shift, 0.125)
    qr, kr, vr = (t.detach().double().requires_grad_(True) for t in (q, k, v))
    ref, ref_lse = _attn_ref64(qr, kr, vr, shift)
    ref.backward(go.double())
    report(f"C:shift{shift}", out=rel_err(out, ref), lse=(lse.double() - ref_lse).abs().max().item(),
           dq=rel_err(dq, qr.grad), dk=rel_err(dk, kr.grad), dv=rel_err(dv, vr.grad))
    assert rel_err(out, ref) < 4e-3
    assert (lse.double() - ref_lse).abs().max().item() < 1e-3
    assert rel_err(dq, qr.grad) < 6e-3
    assert rel_err(dk, kr.grad) < 6e-3
    assert rel_err(dv, vr.grad) < 6e-3
    # every query / key tile boundary, not just the average: worst 128-row block
    def worst_block(a, b):
        a, b = a.double(), b.double()
        e = (a - b).reshape(B, N // 128, 128, -1).norm(dim=(2, 3)) / b.reshape(B, N // 128, 128, -1).norm(dim=(2, 3))
        return e.max().item()
    assert worst_block(out, ref) < 6e-3
    assert worst_block(dq, qr.grad) < 1e-2 and worst_block(dk, kr.grad) < 1e-2 and worst_block(dv, vr.grad) < 1e-2
