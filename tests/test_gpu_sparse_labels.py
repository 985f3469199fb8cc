"""GPU: training from match lists (gt_matches0/1 without the [B, M, N] gt_assignment mask).

1. The positive-term kernels (lgb200_assign_pos_fwd / _bwd, lgb200_assign_bwd_sparse) against fp64 at D 128 / 256 and
   at M, N off the tile multiples, with -1 / -2 labels and an inconsistent pair (NaN).
2. The matchers' reference-golden tests, rerun with every gt_*assignment key removed from the batch the loss sees, at
   the tolerances those tests hold the mask path to.
3. SuperGlue's sparse NLL: loss and dZ bit-identical to the mask's.
4. MatcherTrainer with a dense_assignment: False ground-truth component: eager and replayed steps give the same bits,
   and so do two replays; an inconsistent pair gives a NaN loss and the step is skipped.
5. At the benchmark shape the captured step's peak memory falls by at least B M N bytes.
"""
import pytest
import torch

import tests.test_gpu_gluestick as tgs
import tests.test_gpu_matcher as tgm
import tests.test_gpu_pair_edges as tpe
import tests.test_gpu_superglue as tsg
from gluefactory_b200 import ops, synthetic
from gluefactory_b200.matchers.gluestick import GlueStick
from gluefactory_b200.matchers.homography_matcher import HomographyMatcher
from gluefactory_b200.matchers.lightglue import LightGlue
from gluefactory_b200.matchers.superglue import SuperGlue
from gluefactory_b200.trainer import MatcherTrainer

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24


def _lists(B, M, N, seed, frac=0.5):
    """Random one-to-one match lists with -1 / -2 labels; pair 0 keeps no positive."""
    g = torch.Generator().manual_seed(seed)
    m0 = torch.full((B, M), -1, dtype=torch.long)
    m1 = torch.full((B, N), -1, dtype=torch.long)
    for b in range(1, B):
        k = max(1, int(min(M, N) * frac))
        i, j = torch.randperm(M, generator=g)[:k], torch.randperm(N, generator=g)[:k]
        m0[b, i], m1[b, j] = j, i
    m0[torch.rand(B, M, generator=g) < 0.1] = -2
    # an ignored row keeps no positive, so its partner column is ignored too
    m1[(m1 >= 0) & (m0.gather(1, m1.clamp(min=0)) < 0)] = -2
    return m0, m1


def _dense(m0, N):
    B, M = m0.shape
    gt = torch.zeros(B, M, N, dtype=torch.bool)
    b, i = torch.nonzero(m0 >= 0, as_tuple=True)
    gt[b, i, m0[b, i]] = True
    return gt


@pytest.mark.parametrize("D", [128, 256])
@pytest.mark.parametrize("B,M,N", [(3, 200, 333), (2, 129, 64), (1, 1, 65)])
def test_positive_term_kernels_against_fp64(B, M, N, D):
    g = torch.Generator().manual_seed(B * M + N + D)
    md0 = torch.randn(B, M, D, generator=g).bfloat16()
    md1 = torch.randn(B, N, D, generator=g).bfloat16()
    lr, lc = torch.randn(B, M, generator=g), torch.randn(B, N, generator=g)
    gc = torch.randn(B, generator=g)
    m0, m1 = _lists(max(B, 2), M, N, D)
    m0, m1 = m0[-B:].contiguous(), m1[-B:].contiguous()
    alpha = D ** -0.5
    dv = lambda t: t.to(DEV).contiguous()  # noqa: E731
    # forward from the descriptors, against fp64 of the same bf16 operands
    got = ops.assign_pos_fwd(dv(m0), dv(m1), dv(lr), dv(lc), alpha, dv(md0), dv(md1)).cpu().double()
    a, c = md0.double(), md1.double()
    pos = m0 >= 0
    j = m0.clamp(min=0)
    S = (a * c.gather(1, j[..., None].expand(-1, -1, D))).sum(-1)
    want = torch.where(pos, 2 * alpha * S - lr.double() - lc.double().gather(1, j), torch.zeros_like(S))
    bound = (2 * D + 8) * U * torch.where(pos, 2 * alpha * (a.abs() * c.gather(1, j[..., None].expand(-1, -1, D)).abs()).sum(-1)
                                           + lr.double().abs() + lc.double().gather(1, j).abs(), torch.zeros_like(S))
    assert ((got - want).abs() <= bound).all()
    # forward from a stored sim: the mask path's arithmetic, bit for bit
    sim = torch.randn(B, M, N, generator=g)
    got_s = ops.assign_pos_fwd(dv(m0), dv(m1), dv(lr), dv(lc), alpha, sim=dv(sim)).cpu()
    ref = ops.assign_stats(dv(sim), dv(torch.zeros(B, M)), dv(torch.zeros(B, N)), dv(torch.zeros(B, M)),
                           dv(torch.zeros(B, N)), gt_u8=dv(_dense(m0, N).to(torch.uint8)))
    got_l = ops.assign_pos_fwd(dv(m0), dv(m1), ref["lse_row"], ref["lse_col"], alpha, sim=dv(sim)).cpu()
    assert torch.equal(got_l, ref["pos_row_sum"].cpu())
    xs = sim.gather(2, j[..., None])[..., 0]
    assert torch.equal(got_s, torch.where(pos, (xs - lr) + (xs - lc.gather(1, j)), torch.zeros_like(xs)))
    # backward: dmd += 2 gc md_other[partner], one rounding to bf16
    d0, d1 = torch.randn(B * M, D, generator=g).bfloat16(), torch.randn(B * N, D, generator=g).bfloat16()
    o0, o1 = dv(d0), dv(d1)
    ops.assign_pos_bwd(dv(md0), dv(md1), dv(gc), dv(m0), dv(m1), o0, o1)
    for o, d, src, mm, other in ((o0, d0, c, m0, N), (o1, d1, a, m1, M)):
        k = mm.clamp(min=0)
        w = d.double().view(B, -1, D) + torch.where((mm >= 0)[..., None], 2 * gc.double()[:, None, None]
                                                    * src.gather(1, k[..., None].expand(-1, -1, D)), torch.zeros(1))
        err = (o.cpu().double().view(B, -1, D) - w).abs()
        assert (err <= 2 ** -8 * w.abs() + 4 * U * (d.double().abs().view(B, -1, D) + 1)).all()
    # unfused backward from the list: the mask's dsim, bit for bit
    rc, cc = (m0 >= 0).float(), (m1 >= 0).float()
    for dt in (torch.float32, torch.bfloat16):
        outs = []
        for name, gt in (("lgb200_assign_bwd", dv(_dense(m0, N).to(torch.uint8))), ("lgb200_assign_bwd_sparse", dv(m0))):
            ds = torch.empty(B, M, N, device=DEV, dtype=dt)
            ops.call(name, ops.ptr(dv(sim)), ops.ptr(ref["lse_row"]), ops.ptr(ref["lse_col"]), ops.ptr(gt),
                     ops.ptr(dv(gc)), ops.ptr(dv(rc)), ops.ptr(dv(cc)), ops.ptr(ds), ops._code(dt), B, M, N,
                     ops.stream_ptr())
            outs.append(ds.cpu())
        assert torch.equal(outs[0], outs[1])
    # inconsistent lists: the pair's positive entry is NaN, the others untouched
    if not pos.any():
        return
    bad = m1.clone()
    b, i = (t[0].item() for t in torch.nonzero(pos, as_tuple=True))
    bad[b, m0[b, i]] = (i + 1) % M if M > 1 else -1
    got_bad = ops.assign_pos_fwd(dv(m0), dv(bad), dv(lr), dv(lc), alpha, dv(md0), dv(md1)).cpu()
    assert torch.isnan(got_bad[b, i]) and torch.isnan(got_bad).sum() == 1


# ------------------------------------------------------------------------------------------------
# reference goldens with the mask removed
# ------------------------------------------------------------------------------------------------
@pytest.fixture
def lists_only(monkeypatch):
    """Every matcher's loss sees the batch without its gt_*assignment keys (so the mask path cannot run)."""
    for cls in (LightGlue, SuperGlue, GlueStick):
        orig = cls.loss

        def loss(self, pred, data, _orig=orig):
            return _orig(self, pred, {k: v for k, v in data.items() if "assignment" not in k})
        monkeypatch.setattr(cls, "loss", loss)


@pytest.mark.parametrize("name", tgm.CASES[:4] + tgm.EXTRA_CASES)
def test_lightglue_fp32_golden_from_lists(lists_only, name):
    tgm.test_fp32_path_matches_reference_golden(name)


@pytest.mark.parametrize("name", tgm.CASES[2:4])
def test_lightglue_bf16_golden_from_lists(lists_only, name):
    tgm.test_bf16_path_close_to_reference_golden(name)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", ["edge_lg_a_labels", "edge_lg_b_m1_n65"])
def test_lightglue_edge_fixtures_from_lists(lists_only, name, precision):
    """edge_lg_c_m63_n130 is left out: its pair 1 puts four positives in one row, which match lists cannot express."""
    tpe.test_lightglue_edge_fixtures(name, precision)


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
def test_gluestick_golden_from_lists(lists_only, precision):
    tgs.test_gluestick_matches_reference_golden(precision)


def test_superglue_goldens_from_lists(lists_only):
    tsg.test_superglue_fp32_matches_reference_golden()
    tsg.test_superglue_bf16_against_reference_golden()
    tpe.test_superglue_gluestick_edge_fixtures("edge_sg_labels")
    tpe.test_superglue_gluestick_edge_fixtures("edge_gs_labels")


@pytest.mark.parametrize("B,M,N", [(2, 150, 203), (3, 1, 7), (4, 2048, 2048)])
def test_superglue_sparse_nll_bit_identical(B, M, N):
    g = torch.Generator().manual_seed(M + N)
    Z = torch.randn(B, M + 1, N + 1, generator=g).to(DEV)
    m0, m1 = _lists(B, M, N, M * N)
    m0, m1 = m0.to(DEV), m1.to(DEV)
    gt = _dense(m0.cpu(), N).to(DEV)
    outs = []
    for mask in (gt, None):
        z = Z.clone().requires_grad_(True)
        nll_pos, nll_neg, num_pos, num_neg = ops.ot_nll(z, mask, m0, m1)
        (0.3 * nll_pos + 0.7 * nll_neg).sum().backward()
        outs.append([t.detach().cpu() for t in (nll_pos, nll_neg, num_pos, num_neg, z.grad)])
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    bad = m1.clone()
    b, i = torch.nonzero(m0[1:] >= 0, as_tuple=True)
    bad[1 + b[0], m0[1 + b[0], i[0]]] = -1  # the column loses its partner: counts differ and the row check fails
    nll_pos, _, _, _ = ops.ot_nll(Z, None, m0, bad)
    assert torch.isnan(nll_pos[1 + b[0]]) and torch.isfinite(nll_pos[torch.arange(B, device=DEV) != 1 + b[0]]).all()


# ------------------------------------------------------------------------------------------------
# training with a dense_assignment: False ground-truth component
# ------------------------------------------------------------------------------------------------
def _lg(conf, seed, precision="bf16"):
    model = LightGlue(dict(conf, precision=precision))
    model.load_state_dict(synthetic.make_weights(conf, seed=seed), strict=False)
    return model.to(DEV).train()


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_trainer_from_lists_replays_bit_for_bit(precision):
    conf = dict(synthetic.DEFAULT_CONF, n_layers=2)
    data = {k: v for k, v in synthetic.to_device(synthetic.make_pairs(2, 256, seed=70), DEV).items()
            if not k.startswith("gt_")}
    gt = HomographyMatcher({"dense_assignment": False})
    labels = gt(data)
    assert "assignment" not in labels and {"matches0", "matches1"} <= set(labels)
    assert (labels["matches0"] >= 0).sum() > 0
    trs = [MatcherTrainer(_lg(conf, 71, precision), lr=1e-3, ground_truth=gt) for _ in range(3)]
    for tr in trs:
        tr.step(data)  # one eager step each (also the capture warm-up)
    for tr in trs[1:]:
        tr.capture(data, torch.device(DEV), warmup=0)
    for _ in range(2):
        le, _ = trs[0].step(data)
        l1, _ = trs[1].step_graphed(data)
        l2, _ = trs[2].step_graphed(data)
        assert torch.isfinite(le).all() and torch.equal(le, l1) and torch.equal(l1, l2)
        assert torch.equal(trs[0].fp.flat, trs[1].fp.flat) and torch.equal(trs[1].fp.flat, trs[2].fp.flat)


def test_trainer_skips_step_on_inconsistent_lists():
    conf = dict(synthetic.DEFAULT_CONF, n_layers=2)
    data = synthetic.to_device(synthetic.make_pairs(2, 256, seed=80), DEV)
    data = {k: v for k, v in data.items() if k != "gt_assignment"}
    m1 = data["gt_matches1"].clone()
    j = torch.nonzero(m1[1] >= 0)[0, 0]
    m1[1, j] = (m1[1, j] + 1) % 256  # points at a row that names another column
    data["gt_matches1"] = m1
    tr = MatcherTrainer(_lg(conf, 81), lr=1e-3)
    before = tr.fp.flat.clone()
    loss, losses = tr.step(data)
    assert torch.isnan(losses["total"][1]) and torch.isfinite(losses["total"][0])
    assert tr.skipped_last_step() and torch.equal(tr.fp.flat, before)


def test_captured_step_peak_memory_falls_by_the_mask():
    """Benchmark shape (32 pairs, 2048 points): the captured step with match lists needs at least B M N bytes less."""
    B, N = 32, 2048
    conf = dict(synthetic.DEFAULT_CONF)
    batch = synthetic.to_device(synthetic.make_pairs(B, N, seed=90), DEV)
    peaks = {}
    for kind in ("dense", "lists"):
        data = batch if kind == "dense" else {k: v for k, v in batch.items() if k != "gt_assignment"}
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()  # the batch (with or without its mask) is resident in both runs
        tr = MatcherTrainer(_lg(conf, 91), lr=1e-4)
        tr.step(data)
        tr.capture(data, torch.device(DEV), warmup=0)
        tr.step_graphed(data)
        torch.cuda.synchronize()
        peaks[kind] = torch.cuda.max_memory_allocated() - base
        del tr
        torch.cuda.empty_cache()
    assert peaks["dense"] - peaks["lists"] >= B * N * N, peaks
