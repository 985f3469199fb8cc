"""GPU: the matchers' training and evaluation steps at the pair shapes and labels where the plugins switch paths, against
fp64 oracles, pair by pair and entry by entry.

Each kernel has its own fp64 tests at its tile edges; this file checks how the matchers compose them.  The LightGlue
plugin takes different routes by pair shape: one attention launch over [2B] when M == N, two per block otherwise; the
one-pass shared-qk backward only when M == N at head dim 64; the fused GEMM + assignment head only for bf16 descriptors
of width 64..256, else the unfused head, whose backward uses the tensor cores only when M and N are multiples of 8;
`ops.mask_counts` falls back to torch when N % 16 != 0 or N > 4096.  `test_launch_census` shows that the cases below take
every one of these branches.  The shapes: one-point views (1 x 1, 1 x 2048, 2048 x 1), views smaller than a tile (7 x 9),
counts on and one past a 64-row tile, 130 x 130 (N % 16 != 0), 33 x 4100 (past the mask_counts limit), B = 1, B = 3 and
300 pairs of 5 x 9.  The labels: pairs without positives, with every label ignored, without negatives in one view and
with all positives in one row.  The loss weights are never the symmetric defaults (gamma 0 or 0.7, nll_balancing 0.2 or
0.85), so that a swapped balance or a wrong layer weight shows.  The loss-setting fixtures tests/golden/edge_*.npz
(scripts/make_edge_golden.py, pinned to the oracles by tests/test_edge_golden_cpu.py) are run here as well.

References: the fp64 oracles (oracle/lightglue_oracle.py, tests/superglue_oracle.py, tests/gluestick_inter_oracle.py) on
the same inputs and weights; bf16 LightGlue also against the oracle with the CUDA path's bf16 rounding model
(tests.util.mirror_oracle, O.Bf16Mirror).  Comparisons are per pair: every loss entry of every pair, the log-assignment of
each pair element by element, every parameter's gradient as its own tensor.

Every bound names the error it allows for:
  U32  = 2^-24  fp32 unit round-off;  UBF = 2^-8  bf16 rounding of one stored value
  TOL32 = 2e-5 (336 U32)  fp32 path against fp64.  A log-assignment entry is the end of at most 3 layers x 6 rounded
        contractions plus the 3 of the head, 21 stages; each adds at most 16 U32 relative to the scale of its operands
        (the kernels accumulate in fp32 over blocks of at most 256 terms, whose rounding grows like sqrt(256) U32).
        21 x 16 = 336 U32.  This is also the bar of tests/test_gpu_matcher.py's whole-batch comparison.
  TOLM = 2e-2 (~5 UBF)  bf16 path against the bf16 mirror.  The mirror makes every bf16 rounding the kernels make; what it
        does not model (P rounded before normalisation in the kernels, the shared to_qk gradient rounded per direction,
        an operand rounded the other way because its fp32 sum was ordered differently) is a few bf16 roundings, 5 UBF.
  TOLB = 3e-2 (~8 UBF)  bf16 path against fp64: the rounding of the bf16 operands themselves, 2 per product, through the
        same stages as TOL32, accumulating like a random walk, at most 8 UBF.
  The gradient bars are the end-to-end ones of tests/test_gpu_matcher.py, per tensor: TOL32 fp32, 0.1 (25 UBF) against
  the mirror and 0.15 (38 UBF) against fp64 in bf16: a gradient runs the chain twice and multiplies two rounded factors.
Each tolerance t is applied relative to the pair's scale S: every log-assignment entry is a sum of the similarity, two
log-sum-exps and two log-sigmoids, none larger in size than S = 1 + max|sim| + max|finite log-assignment| over the
pair's heads, so |err| <= t (|ref| + S) elementwise; an NLL entry is a weighted mean of such entries, so |err| <= 2 t S,
also where the reference is exactly 0 (a pair without positives has nll_pos 0).  A gradient tensor is held to
t max(|ref|, 1e-3 G), G the model's largest gradient norm: a tensor whose gradient cancels to 1e-3 of the largest one
carries rounding from that largest one.  Counts are exact.
Indices: matches, and the token-confidence targets (the final layer's argmax over [scores | dustbin]), must equal the
fp64 ones wherever the fp64 top-2 margin exceeds 1e-4 (fp32) or 0.3 (bf16, the rule of tests/test_gpu_matcher.py); for
matches the margins that count are the row's, the matched column's and the distance to the filter threshold.  A target
that may flip moves the pair's confidence term by at most |logit| / (2 n (L - 1)), which the confidence bound adds.
"""
import ast
import math
import os
import time

import numpy as np
import pytest
import torch

from gluefactory_b200 import ops, synthetic
from gluefactory_b200.matchers.gluestick import GlueStick
from gluefactory_b200.matchers.lightglue import LightGlue, matcher_metrics
from gluefactory_b200.matchers.superglue import SuperGlue
from oracle import lightglue_oracle as O
from tests import gluestick_inter_oracle as GO
from tests import superglue_oracle as SO
from tests.util import GOLDEN, mirror_oracle, report

pytestmark = pytest.mark.gpu
DEV = "cuda"
U32, UBF = 2.0 ** -24, 2.0 ** -8
TOL32, TOLM, TOLB = 2e-5, 2e-2, 3e-2
GRAD_TOL = {"fp32": TOL32, "mirror": 0.1, "bf16": 0.15}
MARGIN = {"fp32": 1e-4, "bf16": 0.3}
GRAD_FLOOR = 1e-3

# loss settings away from the defaults (those of the edge fixtures)
LOSS_A = {"gamma": 0.0, "fn": "nll", "nll_balancing": 0.2}
LOSS_B = {"gamma": 0.7, "fn": "nll", "nll_balancing": 0.85}
D256 = dict(synthetic.DEFAULT_CONF, n_layers=3)
D128 = dict(synthetic.DEFAULT_CONF, descriptor_dim=128, input_dim=128, num_heads=4, n_layers=2)  # head dim 32
D512 = dict(synthetic.DEFAULT_CONF, descriptor_dim=512, input_dim=256, num_heads=8, n_layers=2)  # unfused head in bf16
MODELS = {"d256": D256, "d128": D128, "d512": D512}
SMALLEST_MARGIN = {}


@pytest.fixture(scope="module", autouse=True)
def _file_budget():
    """Wall time and peak device memory of this file, and the smallest index margin that was held to equality."""
    torch.cuda.reset_peak_memory_stats()
    t = time.time()
    yield
    torch.cuda.synchronize()
    report("test_gpu_pair_edges", seconds=time.time() - t, peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30,
           **{f"smallest_margin_{k}": v for k, v in SMALLEST_MARGIN.items()})


def _ratio(tag, err, bound):
    """err <= bound elementwise (NaN fails); records the worst err / bound of the check `tag`."""
    err, bound = torch.as_tensor(err).double().reshape(-1), torch.as_tensor(bound).double().reshape(-1).expand_as(
        torch.as_tensor(err).double().reshape(-1))
    ratio = (err / bound.clamp(min=1e-300)).max().item() if err.numel() else 0.0
    key = tag.split(":")[0]
    if ratio >= WORST.get(key, (0.0, ""))[0]:
        WORST[key] = (ratio, tag[len(key) + 1:])
    bad = ~(err <= bound)
    assert not bad.any(), (tag, int(bad.sum()), ratio, err[bad][:4].tolist(), bound[bad][:4].tolist())


WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _worst_ratios():
    yield
    for key, (ratio, where) in sorted(WORST.items()):
        report(f"test_gpu_pair_edges worst err/bound {key}", ratio=ratio, at=where)


# ================================================================================================
# inputs
# ================================================================================================
def ignore_all(d, b, p=""):
    d[f"gt_{p}assignment"][b] = False
    d[f"gt_{p}matches0"][b] = -2
    d[f"gt_{p}matches1"][b] = -2


def no_negatives(d, b, view, p=""):
    m = d[f"gt_{p}matches{view}"]
    m[b] = torch.where(m[b] == -1, torch.full_like(m[b], -2), m[b])


def no_positives(d, b, p=""):
    asg, m0, m1 = d[f"gt_{p}assignment"], d[f"gt_{p}matches0"], d[f"gt_{p}matches1"]
    asg[b] = False
    m0[b] = torch.where(m0[b] >= 0, torch.full_like(m0[b], -1), m0[b])
    m1[b] = torch.where(m1[b] >= 0, torch.full_like(m1[b], -1), m1[b])


def one_row(d, b, i, cols):
    """Pair b: view-0 point i positive with every view-1 point in `cols`, no other positive."""
    no_positives(d, b)
    for j in cols:
        d["gt_assignment"][b, i, j] = True
        d["gt_matches1"][b, j] = i
    d["gt_matches0"][b, i] = cols[0]


def degenerate_inputs(d, b):
    """Pair b: every keypoint of a view at one place with one descriptor (uniform attention, tied scores)."""
    for i in "01":
        d[f"keypoints{i}"][b] = d[f"keypoints{i}"][b, :1]
        d[f"descriptors{i}"][b] = d[f"descriptors{i}"][b, :1]


def edit_labels(d, kinds):
    """kinds[b]: what pair b's labels become (None: as the homography labels them)."""
    M, N = d["gt_assignment"].shape[1:]
    for b, kind in enumerate(kinds):
        if kind == "ignored":
            ignore_all(d, b)
        elif kind == "no_neg1":
            no_negatives(d, b, 1)
        elif kind == "no_neg0":
            no_negatives(d, b, 0)
        elif kind == "no_pos":
            no_positives(d, b)
        elif kind == "one_row":
            one_row(d, b, M // 2, sorted({0, N // 3, N - 1, (2 * N) // 3})[:max(1, min(4, N))])
        elif kind == "one_pos":  # the one positive every 1-point view can have
            no_positives(d, b)
            d["gt_assignment"][b, 0, N - 1] = True
            d["gt_matches0"][b, 0], d["gt_matches1"][b, N - 1] = N - 1, 0
    return d


def lg_data(conf, B, M, N, seed, kinds):
    d = synthetic.make_pairs(B, N, seed=seed, D=conf["input_dim"], M=M)
    return edit_labels(d, kinds)


def _double(d):
    return {k: ({kk: vv.double() for kk, vv in v.items()} if isinstance(v, dict) else
                (v.double() if v.is_floating_point() else v)) for k, v in d.items()}


def _pair(d, b):
    return {k: ({kk: vv[b:b + 1] for kk, vv in v.items()} if isinstance(v, dict) else v[b:b + 1]) for k, v in d.items()}


# ================================================================================================
# LightGlue: runs
# ================================================================================================
def build_lg(conf, w, precision, training=True):
    model = LightGlue(dict(conf, precision=precision))
    missing, unexpected = model.load_state_dict({k: v.float() for k, v in w.items()}, strict=False)
    assert not unexpected and missing in ([], ["confidence_thresholds"])
    return model.to(DEV).train(training)


def run_lg(model, data, training=True):
    d = synthetic.to_device(data, DEV)
    if training:
        pred = model(d)
        losses, metrics = model.loss(pred, d)
        losses["total"].mean().backward()
        grads = {k: p.grad.detach().double().cpu() for k, p in model.named_parameters()}
    else:
        with torch.no_grad():
            pred = model(d)
            losses, metrics = model.loss(pred, d)
        grads = None
    cpu = lambda v: v.detach().cpu() if torch.is_tensor(v) else v  # noqa: E731
    pred = {k: cpu(v) for k, v in pred.items() if not k.startswith("_b200") or k == "_b200_final_arg"}
    pred["_b200_final_arg"] = tuple(t.cpu() for t in pred["_b200_final_arg"])
    return pred, {k: cpu(v) for k, v in losses.items()}, grads, {k: cpu(v) for k, v in metrics.items()}


def oracle_lg(conf, w, data, training=True):
    """fp64 oracle: pred, losses, gradients and, per head, (log-assignment, sim, token logits)."""
    w64 = {k: v.double().requires_grad_(training) for k, v in w.items()}
    d64 = _double(data)
    L = conf["n_layers"]
    rp = O.lightglue_forward(w64, d64, conf)
    if training:
        rl = O.lightglue_loss(w64, rp, d64, conf)
        rl["total"].mean().backward()
    else:  # eval: the last layer's head only (lightglue.py:485, 588)
        bal = conf["loss"]["nll_balancing"]
        nll, nll_pos, nll_neg, num_pos, num_neg = O.nll_terms(rp["log_assignment"], d64["gt_assignment"],
                                                              d64["gt_matches0"], d64["gt_matches1"], balancing=bal)
        rl = {"total": nll, "last": nll, "assignment_nll": nll, "nll_pos": nll_pos, "nll_neg": nll_neg,
              "num_matchable": num_pos, "num_unmatchable": num_neg,
              "row_norm": rp["log_assignment"].exp()[:, :-1].sum(2).mean(1)}
    heads = []
    with torch.no_grad():
        for i in range(L):
            d0, d1 = rp["ref_descriptors0"][:, i], rp["ref_descriptors1"][:, i]
            la, sim = O.match_assignment(d0, d1, w64, i)
            z = None
            if i < L - 1:
                pre = f"token_confidence.{i}.token.0"
                z = [(d @ w64[pre + ".weight"].t() + w64[pre + ".bias"]).squeeze(-1) for d in (d0, d1)]
            heads.append((la, sim, z))
    det = lambda v: v.detach() if torch.is_tensor(v) else torch.tensor(v)  # noqa: E731
    grads = {k: v.grad for k, v in w64.items()} if training else None
    return {k: det(v) for k, v in rp.items()}, {k: det(v) for k, v in rl.items()}, grads, heads


def pair_scale(heads, b):
    s = 0.0
    for la, sim, _ in heads:
        fin = la[b][torch.isfinite(la[b])]
        s = max(s, sim[b].abs().max().item() + (fin.abs().max().item() if fin.numel() else 0.0))
    return 1.0 + s


def _top2_margin(x, dim):
    if x.shape[dim] < 2:
        return torch.full(x.select(dim, 0).shape, math.inf, dtype=x.dtype)
    t = x.topk(2, dim=dim).values
    return t.select(dim, 0) - t.select(dim, 1)


def match_margins(la, th):
    """fp64 margins that decide matches0 / matches1 (row and matched column top-2, distance to the threshold)."""
    inner = la[:, :-1, :-1]
    rm, cm = _top2_margin(inner, 2), _top2_margin(inner, 1)
    m0, m1 = inner.max(2).indices, inner.max(1).indices
    thm = (inner.max(2).values - math.log(th)).abs() if th > 0 else torch.full_like(rm, math.inf)
    s0 = torch.minimum(torch.minimum(rm, cm.gather(1, m0)), thm)
    s1 = torch.minimum(torch.minimum(cm, rm.gather(1, m1)), thm.gather(1, m1))
    return s0, s1


def check_matches(tag, pred, rp, th, thr):
    s0, s1 = match_margins(rp["log_assignment"], th)
    for key, s in (("matches0", s0), ("matches1", s1)):
        safe = s > thr
        SMALLEST_MARGIN[tag.split(":")[0]] = min(SMALLEST_MARGIN.get(tag.split(":")[0], math.inf),
                                                 s[safe].min().item() if safe.any() else math.inf)
        assert torch.equal(pred[key][safe], rp[key][safe]), (tag, key)
    return s0, s1


def check_lg(tag, conf, pred, losses, grads, ref, precision, kind, training=True, bars=None):
    """One run against one reference: kind 'fp64' or 'mirror'.  ref = (pred, losses, grads, heads) of the fp64 oracle;
    for 'mirror' the mirror's (pred, losses, grads) with the fp64 heads for the scales and margins.
    bars: {"tol", "gtol", "thr"} in place of this file's bars (derived for at most 3 layers), for deeper models."""
    rp, rl, rg, heads = ref
    B = pred["log_assignment"].shape[0]
    L = len(heads)
    tol = TOL32 if precision == "fp32" else (TOLM if kind == "mirror" else TOLB)
    gtol = GRAD_TOL["fp32" if precision == "fp32" else kind if kind == "mirror" else "bf16"]
    thr = MARGIN[precision]
    if bars is not None:
        tol, gtol, thr = bars["tol"], bars["gtol"], bars["thr"]
    if kind == "fp64":
        check_matches(tag, pred, rp, conf.get("filter_threshold", 0.0), thr)
    th = conf.get("filter_threshold", 0.0)
    s0, s1 = match_margins(heads[-1][0], th)
    la, rla = pred["log_assignment"].double(), rp["log_assignment"].double()
    for b in range(B):
        S = pair_scale(heads, b)
        fin = torch.isfinite(rla[b])
        assert torch.equal(fin, torch.isfinite(la[b])), (tag, b)
        _ratio(f"log_assignment {precision} {kind}:{tag}:pair{b}", (la[b] - rla[b])[fin].abs(),
               tol * (rla[b][fin].abs() + S))
        for key, s in (("matching_scores0", s0[b]), ("matching_scores1", s1[b])):
            safe = s > thr
            got, want = pred[key][b].double()[safe], rp[key][b].double()[safe]
            _ratio(f"matching_scores {precision} {kind}:{tag}:pair{b}", (got - want).abs(), tol * want * (2 * S) + 1e-30)
        for k in ("num_matchable", "num_unmatchable"):
            assert losses[k][b].item() == rl[k][b].item(), (tag, k, b)
        for k in ("last", "assignment_nll", "nll_pos", "nll_neg"):
            _ratio(f"loss {precision} {kind}:{tag}:pair{b}:{k}", abs(losses[k][b].item() - rl[k][b].item()), 2 * tol * S)
        rn = rl["row_norm"][b].item()
        _ratio(f"row_norm {precision} {kind}:{tag}:pair{b}", abs(losses["row_norm"][b].item() - rn), 2 * tol * S * max(rn, 1.0))
        conf_bound = 0.0
        if training and L > 1:
            conf_bound = conf_term_bound(heads, b, tol, thr)
            _ratio(f"confidence {precision} {kind}:{tag}:pair{b}",
                   abs(losses["confidence"][b].item() - rl["confidence"][b].item()), conf_bound)
        _ratio(f"loss {precision} {kind}:{tag}:pair{b}:total", abs(losses["total"][b].item() - rl["total"][b].item()),
               2 * tol * S + conf_bound)
    if training and kind == "fp64":
        check_final_targets(tag, pred, heads, thr)
    if grads is not None:
        check_grads(tag, grads, rg, gtol, precision, kind)


def check_grads(tag, grads, rg, gtol, precision, kind):
    """Every parameter's gradient as its own tensor: ||g - ref|| <= gtol max(||ref||, GRAD_FLOOR G)."""
    G = max(v.double().norm().item() for v in rg.values())
    for k, g in grads.items():
        r = rg[k].double()
        _ratio(f"grad {precision} {kind}:{tag}:{k}", (g.double() - r).norm().item(),
               gtol * max(r.norm().item(), GRAD_FLOOR * G))


def conf_term_bound(heads, b, tol, thr):
    """Bound of one pair's token-confidence term: the logits' rounding (the BCE is 1-Lipschitz in its logit) plus, for
    every token whose target may flip (a top-2 margin over [scores | dustbin] <= thr in its layer's head or in the final
    head), |logit| / (2 n (L - 1))."""
    L = len(heads)
    fin = heads[-1][0][b]
    fr, fc = _top2_margin(fin[:-1, :], 1), _top2_margin(fin[:, :-1], 0)
    out = 0.0
    for la, _, z in heads[:-1]:
        r, c = _top2_margin(la[b][:-1, :], 1), _top2_margin(la[b][:, :-1], 0)
        for zz, m_now, m_fin in ((z[0][b], r, fr), (z[1][b], c, fc)):
            n = zz.numel()
            unsafe = (m_now <= thr) | (m_fin <= thr)
            out += (tol * (zz.abs() + 1).max().item() + zz[unsafe].abs().sum().item() / n) / (2 * (L - 1))
    return out + 1e-12


def check_final_targets(tag, pred, heads, thr):
    """The token-confidence targets: the final head's argmax over [scores | dustbin], per row and per column."""
    fin = heads[-1][0]
    rows, cols = fin[:, :-1, :], fin[:, :, :-1]
    for got, x, dim in ((pred["_b200_final_arg"][0], rows, 2), (pred["_b200_final_arg"][1], cols, 1)):
        safe = _top2_margin(x, dim) > thr
        assert torch.equal(got.long()[safe], x.max(dim).indices[safe]), tag


def mirror_ref(conf, w, data, heads):
    mp, ml, mg = mirror_oracle(conf, w, data)
    return mp, ml, mg, heads


# ================================================================================================
# LightGlue training: edge shapes x precision x model
# ================================================================================================
# (model, M, N, B, label kinds of the pairs); the loss settings alternate between LOSS_A and LOSS_B
SHAPES = [
    ("d256", 1, 1, 2, ("one_pos", "no_pos")),
    ("d256", 1, 2048, 1, ("one_pos",)),
    ("d256", 2048, 1, 1, ("no_neg1",)),
    ("d256", 7, 9, 3, (None, "ignored", "no_neg1")),
    ("d256", 63, 63, 2, (None, "no_neg0")),
    ("d256", 64, 64, 2, (None, "one_row")),
    ("d256", 65, 65, 2, ("no_pos", None)),
    ("d256", 64, 65, 2, (None, "no_neg1")),
    ("d256", 65, 64, 2, ("one_row", None)),
    ("d256", 8, 16, 2, (None, "no_pos")),
    ("d256", 130, 130, 2, (None, "ignored")),
    ("d256", 33, 4100, 1, (None,)),
    ("d128", 1, 1, 2, ("one_pos", "ignored")),
    ("d128", 7, 9, 3, (None, "no_pos", "no_neg0")),
    ("d128", 64, 65, 2, ("one_row", None)),
    ("d128", 8, 16, 2, (None, "no_neg1")),
    ("d128", 130, 130, 1, (None,)),
    ("d128", 1, 2048, 1, ("one_pos",)),
    ("d512", 8, 16, 2, (None, "no_neg0")),
    ("d512", 7, 9, 2, ("no_pos", None)),
]


def _shape_id(s):
    return f"{s[0]}-{s[1]}x{s[2]}-B{s[3]}"


def _lg_case(i, model, M, N, B, kinds):
    conf = dict(MODELS[model], loss=LOSS_A if i % 2 == 0 else LOSS_B)
    w = synthetic.make_weights(conf, seed=500 + i)
    data = lg_data(conf, B, M, N, 600 + i, kinds)
    return conf, w, data


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("i", range(len(SHAPES)), ids=[_shape_id(s) for s in SHAPES])
def test_lightglue_training_at_edge_shapes(i, precision):
    model, M, N, B, kinds = SHAPES[i]
    conf, w, data = _lg_case(i, model, M, N, B, kinds)
    got = run_lg(build_lg(conf, w, precision), data)
    ref = oracle_lg(conf, w, data)
    tag = f"train:{_shape_id(SHAPES[i])}"
    check_lg(tag, conf, got[0], got[1], got[2], ref, precision, "fp64")
    if precision == "bf16":
        check_lg(tag, conf, got[0], got[1], got[2], mirror_ref(conf, w, data, ref[3]), precision, "mirror")


def test_lightglue_training_300_tiny_pairs():
    """300 pairs of 5 x 9 in one batch (the head-terms kernel's per-pair reduction and counters, 600 attention segments):
    every pair's loss entries and log-assignment against fp64; fp32 and bf16."""
    conf = dict(D256, n_layers=2, loss=LOSS_B)
    w = synthetic.make_weights(conf, seed=531)
    kinds = [(None, "no_pos", "ignored", "no_neg1", "one_row")[b % 5] for b in range(300)]
    data = lg_data(conf, 300, 5, 9, 631, kinds)
    ref = oracle_lg(conf, w, data)
    for precision in ("fp32", "bf16"):
        got = run_lg(build_lg(conf, w, precision), data)
        check_lg("train:300x5x9", conf, got[0], got[1], got[2], ref, precision, "fp64")


# ================================================================================================
# LightGlue training: the loss-setting fixtures
# ================================================================================================
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name", ["edge_lg_a_labels", "edge_lg_b_m1_n65", "edge_lg_c_m63_n130"])
def test_lightglue_edge_fixtures(name, precision):
    """The reference's own loss entries at gamma 0 / 0.7 and nll_balancing 0.2 / 0.85 with empty label classes: per pair
    against the fixture (fp32 within TOL32 of the pair's scale), and everything against the fp64 oracle on the same
    inputs."""
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False))
    conf = ast.literal_eval(str(g["meta|conf"]))
    B, M, N, seed = (int(g["meta|" + k]) for k in ("B", "M", "N", "seed"))
    w = synthetic.make_weights(conf, seed=seed)
    data = synthetic.make_pairs(B, N, seed=seed + 1, D=conf["input_dim"], M=M)
    for k in ("gt_assignment", "gt_matches0", "gt_matches1"):
        data[k] = torch.from_numpy(g["label|" + k])
    model = build_lg(conf, w, precision)
    pred, losses, grads, _ = run_lg(model, data)
    ref = oracle_lg(conf, w, data)
    check_lg(f"fixture:{name}", conf, pred, losses, grads, ref, precision, "fp64")
    tol = TOL32 if precision == "fp32" else TOLB
    for b in range(B):
        S = pair_scale(ref[3], b)
        for k in ("total", "assignment_nll", "nll_pos", "nll_neg", "num_matchable", "num_unmatchable"):
            _ratio(f"fixture loss {precision}:{name}:pair{b}:{k}", abs(losses[k][b].item() - float(g["loss|" + k][b])),
                   2 * tol * S + conf_term_bound(ref[3], b, tol, MARGIN[precision]) + 1e-300)


# ================================================================================================
# LightGlue: batch isolation
# ================================================================================================
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("M,N", [(65, 65), (63, 130)])
def test_lightglue_degenerate_pair_does_not_touch_its_neighbours(M, N, precision):
    """B = 3: an ordinary pair, a pair with every keypoint at one place with one descriptor and every label ignored, and a
    pair without negatives in view 1.  Each pair's forward outputs and its own loss entries equal those of the same pair
    run alone: bit for bit in bf16 (every kernel of the step works per pair or per token; only parameter gradients sum
    over the batch, and they are not compared), within TOL32 of the pair's scale in fp32 (cuBLAS may pick another
    kernel for another row count)."""
    conf = dict(D256, n_layers=2, loss=LOSS_A)
    w = synthetic.make_weights(conf, seed=541)
    data = lg_data(conf, 3, M, N, 641, (None, "ignored", "no_neg1"))
    degenerate_inputs(data, 1)
    model = build_lg(conf, w, precision)
    whole = run_lg(model, data)
    heads = oracle_lg(conf, w, data, training=False)[3] if precision == "fp32" else None
    keys = ["log_assignment", "matches0", "matches1", "matching_scores0", "matching_scores1"]
    margins = match_margins(heads[-1][0], 0.0) if heads is not None else None
    for b in range(3):
        model.zero_grad(set_to_none=True)
        alone = run_lg(model, _pair(data, b))
        for k in keys:
            a, w_ = alone[0][k][0], whole[0][k][b]
            if precision == "bf16":
                assert torch.equal(a, w_), (k, b)
            elif k.startswith("matches"):  # the degenerate pair's scores tie: compared where fp64 decides by margin
                safe = margins[int(k[-1])][b] > MARGIN["fp32"]
                assert torch.equal(a[safe], w_[safe]), (k, b)
            else:
                S = pair_scale(heads, b)
                _ratio(f"isolation fp32:{M}x{N}:pair{b}:{k}", (a.double() - w_.double()).abs(), TOL32 * S)
        for k in ("total", "last", "assignment_nll", "nll_pos", "nll_neg", "num_matchable", "num_unmatchable",
                  "confidence", "row_norm"):
            a, w_ = alone[1][k][0], whole[1][k][b]
            if precision == "bf16":
                assert torch.equal(a, w_), (k, b, a.item(), w_.item())
            else:
                _ratio(f"isolation fp32:{M}x{N}:pair{b}:{k}", abs(a.item() - w_.item()), 2 * TOL32 * pair_scale(heads, b))


# ================================================================================================
# LightGlue: evaluation
# ================================================================================================
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("i", range(12), ids=[_shape_id(s) for s in SHAPES[:12]])
def test_lightglue_eval_at_edge_shapes(i, precision):
    """Eval mode: the dense assign_stats + filter_matches with filter_threshold 0.1, the loss of the last head alone
    (L == 1) and matcher_metrics, per pair against fp64.  The metrics of a pair are compared where all its matches are
    decided by margins above the threshold (they depend on the matches exactly); they are the plugin's restatement of
    glue-factory's metrics (pinned by tests/golden/eval_loss.npz) applied to the fp64 matches and scores."""
    model_name, M, N, B, kinds = SHAPES[i]
    conf = dict(MODELS[model_name], loss=LOSS_B if i % 2 == 0 else LOSS_A, filter_threshold=0.1)
    w = synthetic.make_weights(conf, seed=700 + i)
    data = lg_data(conf, B, M, N, 800 + i, kinds)
    pred, losses, _, metrics = run_lg(build_lg(conf, w, precision, training=False), data, training=False)
    ref = oracle_lg(conf, w, data, training=False)
    assert pred["ref_descriptors0"].shape[1] == 1 and "confidence" not in losses
    check_lg(f"eval:{_shape_id(SHAPES[i])}", conf, pred, losses, None, ref, precision, "fp64", training=False)
    rp = ref[0]
    ref_metrics = matcher_metrics({"matches0": rp["matches0"], "matching_scores0": rp["matching_scores0"]},
                                  {"gt_matches0": data["gt_matches0"]})
    s0, s1 = match_margins(rp["log_assignment"], 0.1)
    for b in range(B):
        if (s0[b] > MARGIN[precision]).all() and (s1[b] > MARGIN[precision]).all():
            for k, v in ref_metrics.items():
                _ratio(f"metrics {precision}:eval:{i}:pair{b}:{k}", abs(metrics[k][b].item() - v[b].item()),
                       1e-6 + 1e-5 * abs(v[b].item()))


def test_lightglue_refuses_empty_keypoint_sets():
    """An empty view is refused (the reference's loss would divide by an empty mean); it never reaches a kernel."""
    conf = dict(D256, n_layers=1)
    model = build_lg(conf, synthetic.make_weights(conf, seed=1), "bf16")
    data = synthetic.to_device(synthetic.make_pairs(1, 16, seed=2, M=16), DEV)
    for k, n in (("0", 0), ("1", 0)):
        d = dict(data)
        d["keypoints" + k] = d["keypoints" + k][:, :n]
        d["descriptors" + k] = d["descriptors" + k][:, :n]
        with pytest.raises(AssertionError, match="empty keypoint sets"):
            model(d)


# ================================================================================================
# launch census: the cases above take every branch
# ================================================================================================
def test_launch_census(monkeypatch):
    """Records which engine and ops branch each training / eval case takes (shims around the ops functions and the C
    calls the engine makes) and checks that every branch is taken: one attention launch over [2B] with kv_shift B and
    two per block; the one-pass shared-qk backward and its dq + dk fallback; the fused head, the unfused head with the
    tensor-core and with the fp32 dsim backward; the mask_counts kernel and its torch fallback; the dense eval head."""
    seen = set()
    real = {n: getattr(ops, n) for n in ("attn_fwd", "attn_bwd", "attn_bwd_shared_qk", "assign_fused_stats",
                                         "assign_stats", "mask_counts", "call")}

    def shim(name):
        def f(*a, **k):
            if name == "attn_fwd":
                seen.add(("attn_fwd", "shift" if a[3] else "no_shift"))
            elif name == "attn_bwd":
                seen.add(("attn_bwd", "shift" if a[6] else "no_shift"))
            elif name == "assign_stats":
                seen.add(("assign_stats", "dense" if k.get("dense") else "sparse"))
            elif name == "mask_counts":
                n = a[0].shape[2]
                seen.add(("mask_counts", "torch" if n % 16 or n > 4096 else "kernel"))
            elif name == "call":
                if a[0] == "lgb200_assign_bwd":
                    seen.add(("assign_unfused_bwd", "tc" if a[9] == ops._code(torch.bfloat16) else "fp32_dsim"))
                if a[0] == "lgb200_mask_counts":
                    seen.add(("mask_counts_kernel_launch",))
            else:
                seen.add((name,))
            return real[name](*a, **k)
        return f

    for n in real:
        monkeypatch.setattr(ops, n, shim(n))
    cases = {("d256", 64, 64), ("d256", 64, 65), ("d128", 64, 65), ("d256", 130, 130), ("d256", 33, 4100),
             ("d512", 8, 16), ("d512", 7, 9)}
    for model_name, M, N in sorted(cases):
        conf = dict(MODELS[model_name], n_layers=1)
        w = synthetic.make_weights(conf, seed=3)
        data = lg_data(conf, 1, M, N, 4, (None,))
        for precision in ("fp32", "bf16"):
            run_lg(build_lg(conf, w, precision), data)
        run_lg(build_lg(conf, w, "bf16", training=False), data, training=False)
    report("census test_gpu_pair_edges", **{f"s{i}": "/".join(s) for i, s in enumerate(sorted(seen))})
    want = {("attn_fwd", "shift"), ("attn_fwd", "no_shift"), ("attn_bwd", "shift"), ("attn_bwd", "no_shift"),
            ("attn_bwd_shared_qk",), ("assign_fused_stats",), ("assign_stats", "sparse"), ("assign_stats", "dense"),
            ("assign_unfused_bwd", "tc"), ("assign_unfused_bwd", "fp32_dsim"), ("mask_counts", "kernel"),
            ("mask_counts", "torch"), ("mask_counts_kernel_launch",)}
    assert want <= seen, want - seen


# ================================================================================================
# SuperGlue and GlueStick
# ================================================================================================
def _per_pair_la(tag, la, rla, tol):
    for b in range(la.shape[0]):
        S = 1.0 + rla[b].abs().max().item()
        _ratio(f"{tag}:pair{b}", (la[b].double() - rla[b]).abs(), tol * (rla[b].abs() + S))


def _per_pair_losses(tag, losses, rl, keys, scale, tol):
    for k in keys:
        for b in range(rl[k].shape[0]):
            if k.startswith(("num_", "line_num_")):
                assert losses[k][b].item() == rl[k][b].item(), (tag, k, b)
            else:
                _ratio(f"{tag}:pair{b}:{k}", abs(losses[k][b].item() - rl[k][b].item()), 2 * tol * scale[b])


def _grads(tag, model, params, precision, few_samples=()):
    """fp32: each tensor within 2e-3 relative L2 (the bar of tests/test_gpu_gluestick_inter.py's fp32 comparison with
    the fp64 oracle: the GNN's BatchNorms divide by batch deviations, which amplifies rounding); bf16: each tensor's norm
    within 0.15 (that file's bf16 bar).  A conv bias in front of a BatchNorm has zero gradient in theory: its rounding
    noise is held to those files' absolute bars.
    few_samples: parameter-name prefixes ("" for all) behind a BatchNorm that sees fewer than 16 samples in one view (B
    times a view's point or line count; the point MLPs of every GNN layer normalise each view on its own).  Over two
    samples a BatchNorm maps its input to +-1 whatever it is, so the gradient it passes back is zero up to the eps term,
    and what comes back is the rounding of the cancellation g - mean(g) - x_hat mean(g x_hat), amplified by 1 / sigma;
    over a few samples it is nearly so.  In bf16, where that BatchNorm reads a bf16-rounded input, the rounding is as
    large as the gradient itself (the reference under bf16 autocast has the same conditioning), so those gradients are
    held to the bound in fp32 only."""
    G = max(p.grad.norm().item() for p in params.values())
    for k, p in model.named_parameters():
        r, got = params[k].grad.double(), p.grad.double().cpu()
        if precision == "bf16" and k.startswith(tuple(few_samples)):
            continue
        if r.norm().item() < 1e-9:
            assert got.norm().item() < (1e-4 if precision == "fp32" else 2e-2), (tag, k)
            continue
        if precision == "fp32":
            _ratio(f"{tag}:{k}", (got - r).norm().item(), 2e-3 * max(r.norm().item(), GRAD_FLOOR * G))
        else:
            _ratio(f"{tag}:{k}", abs(got.norm().item() - r.norm().item()), 0.15 * max(r.norm().item(), GRAD_FLOOR * G))


SG_SHAPES = [(1, 65), (64, 65), (1, 2048), (2048, 1)]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("M,N", SG_SHAPES)
def test_superglue_at_edge_shapes(M, N, precision):
    """nll_balancing 0.3; pair 0 without negatives in view 1, pair 1 without positives.  SuperGlue clamps the negative
    count as a sum (superglue.py:329).  The Sinkhorn log-assignment per pair element-wise, every loss entry per pair,
    every gradient per tensor, against fp64; fp32 matches where decided by margin."""
    conf = {"GNN_layers": ["self", "cross"], "filter_threshold": 0.2, "loss": {"nll_balancing": 0.3}}
    model = SuperGlue(dict(conf, weights=None, precision=precision))
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=M + N), strict=True)
    model = model.to(DEV).train()
    d = synthetic.make_superglue_batch(2, M, N, 900 + M)
    no_negatives(d, 0, 1)
    no_positives(d, 1)
    pred = model(synthetic.to_device(d, DEV))
    losses, _ = model.loss(pred, synthetic.to_device(d, DEV))
    losses["total"].mean().backward()
    w = {k: (v.detach().double().cpu() if v.is_floating_point() else v.cpu()) for k, v in model.state_dict().items()}
    params = {k: w[k].clone().requires_grad_(True) for k, _ in model.named_parameters()}
    rp = SO.superglue_forward({**w, **params}, _double(d), conf)
    rl = SO.superglue_loss({**w, **params}, rp, _double(d), conf)
    rl["total"].mean().backward()
    tol = TOL32 if precision == "fp32" else TOLB
    tag = f"superglue {precision}:{M}x{N}"
    la, rla = pred["log_assignment"].detach().cpu(), rp["log_assignment"].detach()
    _per_pair_la(tag, la, rla, tol * 5)  # 50 Sinkhorn iterations: five times the stages of one head
    scale = [1.0 + rla[b].abs().max().item() for b in range(2)]
    _per_pair_losses(tag, {k: v.detach().cpu() for k, v in losses.items()}, {k: v.detach() for k, v in rl.items()},
                     ["total", "nll_pos", "nll_neg", "num_matchable", "num_unmatchable"], scale, tol * 5)
    if precision == "fp32":
        s0, s1 = match_margins(rla, 0.2)
        for key, s in (("matches0", s0), ("matches1", s1)):
            safe = s > MARGIN["fp32"]
            assert torch.equal(pred[key].cpu()[safe], rp[key][safe]), key
    _grads(f"superglue grad {precision}:{M}x{N}", model, params, precision, [""] if 2 * min(M, N) < 16 else [])


def gluestick_batch(B, M, N, L0, L1, seed):
    """make_gluestick_batch with view 0 cut to M points / L0 lines and view 1 to N points / L1 lines (lines are made of
    the first 2 L keypoints, so M >= 2 L0 and N >= 2 L1 keep them), labels cut the same way."""
    d = synthetic.make_gluestick_batch(B, max(M, N), max(L0, L1), seed)
    cut = {"0": (M, L0), "1": (N, L1)}
    for i, (n, l) in cut.items():
        j = "1" if i == "0" else "0"
        for k in ("keypoints", "descriptors", "keypoint_scores"):
            d[k + i] = d[k + i][:, :n]
        d["lines" + i], d["line_scores" + i], d["lines_junc_idx" + i] = (d["lines" + i][:, :l], d["line_scores" + i][:, :l],
                                                                         d["lines_junc_idx" + i][:, :l])
        for p, cnt, other in (("", n, cut[j][0]), ("line_", l, cut[j][1])):
            m = d[f"gt_{p}matches{i}"][:, :cnt]
            d[f"gt_{p}matches{i}"] = torch.where(m >= other, torch.full_like(m, -1), m)
    for p, (a, b) in (("", (M, N)), ("line_", (L0, L1))):
        d[f"gt_{p}assignment"] = d[f"gt_{p}assignment"][:, :a, :b].contiguous()
    return d


GS_SHAPES = [(2, 65, 1, 8), (64, 65, 8, 8), (2, 1100, 1, 16), (1100, 4, 16, 2)]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("M,N,L0,L1", GS_SHAPES)
def test_gluestick_at_edge_shapes(M, N, L0, L1, precision):
    """nll_balancing 0.8, nll_weight 2, intermediate heads after blocks 1 and 0 weighted 0.25 and 0.9; a view with one
    line, lopsided point counts; pair 0 without point and line negatives in view 1, pair 1 without positives.  GlueStick
    clamps the negative count as a sum (gluestick.py:313).  Against fp64, per pair and per tensor."""
    conf = {"GNN_layers": ["self", "cross"] * 2, "filter_threshold": 0.2, "inter_supervision": [1, 0],
            "loss": {"nll_weight": 2.0, "nll_balancing": 0.8, "inter_supervision": [0.25, 0.9]}}
    model = GlueStick(dict(conf, precision=precision))
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=M + N + L0), strict=True)
    model = model.to(DEV).train()
    d = gluestick_batch(2, M, N, L0, L1, 950 + M)
    for p in ("", "line_"):
        no_negatives(d, 0, 1, p)
        no_positives(d, 1, p)
    data = synthetic.to_device(d, DEV)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    w = {k: (v.detach().double().cpu() if v.is_floating_point() else v.cpu()) for k, v in model.state_dict().items()}
    params = {k: w[k].requires_grad_(True) for k, _ in model.named_parameters()}
    rp = GO.gluestick_forward({**w, **params}, _double(d), dict(conf, descriptor_dim=256))
    rl = GO.gluestick_loss({**w, **params}, rp, _double(d), conf)
    rl["total"].mean().backward()
    tol = 5 * TOL32 if precision == "fp32" else TOLB  # fp32: the GNN stacks 8 attention / line layers, 5x the stages
    tag = f"gluestick {precision}:{M}x{N}:L{L0}x{L1}"
    scale = [1.0] * 2
    for h in ("", "line_", "line_1_", "line_0_"):
        la, rla = pred[h + "log_assignment"].detach().cpu(), rp[h + "log_assignment"].detach()
        _per_pair_la(f"{tag}:{h}log_assignment", la, rla, tol)
        scale = [max(scale[b], 1.0 + rla[b].abs().max().item()) for b in range(2)]
        if precision == "fp32":
            s0, s1 = match_margins(rla, 0.2)
            for key, s in ((h + "matches0", s0), (h + "matches1", s1)):
                safe = s > MARGIN["fp32"]
                assert torch.equal(pred[key].cpu()[safe], rp[key][safe]), key
    keys = ["total", "assignment_nll", "line_assignment_nll", "line_0_assignment_nll", "line_1_assignment_nll",
            "num_matchable", "num_unmatchable", "line_num_matchable", "line_num_unmatchable"]
    _per_pair_losses(tag, {k: v.detach().cpu() for k, v in losses.items()}, {k: v.detach() for k, v in rl.items()}, keys,
                     [6 * s for s in scale], tol)  # total: 2 x (1 + 1 + 0.25 + 0.9) < 6 NLL terms
    few = ([""] if 2 * min(M, N) < 16 else []) + (["lenc."] if 2 * min(L0, L1) < 16 else [])
    _grads(f"gluestick grad {precision}:{M}x{N}", model, params, precision, few)


@pytest.mark.parametrize("name", ["edge_sg_labels", "edge_gs_labels"])
def test_superglue_gluestick_edge_fixtures(name):
    """The reference's loss entries at the fixtures' settings, per pair, fp32 path (relative 5 TOL32 per entry: each
    is one NLL over a head that is at most 8 GNN layers deep; counts exact)."""
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False))
    conf = ast.literal_eval(str(g["meta|conf"]))
    if name == "edge_sg_labels":
        B, M, N, seed = (int(g["meta|" + k]) for k in ("B", "M", "N", "seed"))
        model = SuperGlue(dict(conf, precision="fp32"))
        d = synthetic.make_superglue_batch(B, M, N, seed + 1)
        labels = ("gt_assignment", "gt_matches0", "gt_matches1")
    else:
        B, N, L, seed = (int(g["meta|" + k]) for k in ("B", "N", "L", "seed"))
        model = GlueStick(dict(conf, precision="fp32"))
        d = synthetic.make_gluestick_batch(B, N, L, seed + 1)
        labels = ("gt_assignment", "gt_matches0", "gt_matches1", "gt_line_assignment", "gt_line_matches0",
                  "gt_line_matches1")
    for k in labels:
        d[k] = torch.from_numpy(g["label|" + k])
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=seed), strict=True)
    model = model.to(DEV).train()
    data = synthetic.to_device(d, DEV)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    for k in (k[len("loss|"):] for k in g if k.startswith("loss|")):
        got, ref = losses[k].detach().double().cpu().numpy().reshape(-1), g["loss|" + k].reshape(-1)
        if "num_" in k:
            assert np.array_equal(got, ref), k
            continue
        _ratio(f"fixture {name}:{k}", np.abs(got - ref), 5 * TOL32 * (np.abs(ref) + 1.0))
    for k in ("matches0", "matches1"):
        assert np.array_equal(pred[k].cpu().numpy(), g["pred|" + k]), k
