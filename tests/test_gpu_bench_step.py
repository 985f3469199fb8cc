"""GPU: the benchmark's training step at its own shape against fp64.

bench.py times one configuration: LightGlue with 9 layers, d 256 and 4 heads, on 32 pairs of 2048 + 2048 points, run
by MatcherTrainer with device labels from HomographyMatcher (th_positive = th_negative = 3, transposed mask).  Each
kernel of that step has its own fp64 tests; this file checks the step they make up.  Only this step has a batch of 32
(64 attention sequences with kv_shift 32, 32 pairs of counters in head_terms_fwd), split-K weight gradients over 131072
tokens written straight into the flat gradient buffer (FlatParams.enable_direct, which only MatcherTrainer turns on),
the transposed mask of the device labels and the captured replay.

Cases (all with the benchmark's Adam at lr 1e-4 and DEFAULT_CONF's loss, gamma 1 and nll_balancing 0.5):
  bench       bf16  32 x 2048 x 2048  mask + transposed mask (the benchmark's labels)
  bench_fp32  fp32  32 x 2048 x 2048  mask (the fp32 parity path, whose nine-layer backward nothing else compares)
  lists       bf16  32 x 2048 x 2048  match lists (dense_assignment: False): the fused head without masks, then
                                      assign_pos_bwd
  ragged      bf16   8 x 2048 x 1536  mask + transposed mask (two attention launches per block)
  d128        bf16   8 x 2048 x 2048  descriptor_dim = input_dim = 128, 4 heads (head dim 32)

What is compared, all from one eager trainer step: the flat gradient buffer trainer.fp.grad, cut into parameters at
FlatParams's offsets (the loss slot behind it is not a gradient; the trainer has no loss scale here, so nothing is
undone); the per-pair loss entries the step returns; the final log-assignment, matches, matching scores and token-
confidence targets of the forward pass the step ran (read by a forward hook, which also sees the labels the step
stored; those must equal what the same ground-truth component gives for the batch).  In the bench case the captured
step (trainer.capture + step_graphed) from the same saved state must give the eager step's loss, gradient and updated
parameters bit for bit, and two replays must agree bit for bit.

The reference is the fp64 oracle (oracle/lightglue_oracle.py) on the device, CHUNK pairs at a time, each layer under
torch.utils.checkpoint.  The step's loss is losses["total"].mean() over the B pairs (trainer.py: _step_impl), so each
chunk contributes d(sum of its pairs' totals) / B and the chunks' gradients are summed.  For bf16 the oracle with the
CUDA path's rounding model (O.Bf16Mirror) runs the same chunks in fp32.  TF32 is off for the whole file (fixture).

Bars.  tests/test_gpu_pair_edges.py derives TOL32, TOLM and TOLB for at most 3 layers (21 rounded stages, sums of at most
256 terms); the same derivation for this step:
  stages   9 layers x 6 rounded contractions + the 3 of the head = 57.
  TOL32 = 57 x 46 U32 = 2622 U32 = 1.56e-4   fp32 path against fp64.  Each stage adds at most sqrt(n) U32 relative to
           its operands' scale, n its longest fp32 sum; here the softmax and log-sum-exp sums and P V run over 2048 keys
           and the head's LSEs over 2048 rows or columns: sqrt(2048) < 46.
  TOLM  = 9 UBF = 3.5e-2   bf16 against the bf16 mirror.  What the mirror does not model is a few bf16 roundings per
           layer (P rounded before normalisation, to_qk's gradient per direction, an operand rounded the other way);
           test_gpu_pair_edges allows 5 UBF for 21 stages, and a random walk over 57 grows that by sqrt(57 / 21) = 1.65.
  TOLB  = 11 UBF = 4.3e-2  bf16 against fp64: two operand roundings per product through 57 stages as a random walk,
           sqrt(2 x 57) = 10.7.
  Gradients run the chain twice and end in one weight-gradient sum over 131072 tokens (sqrt(131072) U32 = 2.2e-5):
  GTOL32 = 2 TOL32 + 2.2e-5 = 3.34e-4 (inside the 1e-3 of DESIGN.md section 1), GTOLM = 41 UBF = 0.16 and GTOLB = 63
  UBF = 0.25 (test_gpu_pair_edges's 25 and 38 UBF grown by 1.65).
Each bar t is applied as in test_gpu_pair_edges.check_lg, against the pair's scale S (1 + max|sim| + max|finite
log-assignment| over its nine heads): every log-assignment entry |err| <= t (|ref| + S), every loss entry of every pair
|err| <= 2 t S (confidence: plus the flips below), each gradient tensor ||err|| <= t max(||ref||, 1e-3 G).  An index
(matches, matched column, the token-confidence targets = the argmax over [scores | dustbin]) must equal fp64's wherever
the fp64 top-2 margin exceeds THR = 4 t S_max, S_max the largest S of the chunk: two entries of a row each move by at
most t (|ref| + S) <= 2 t S, so a margin above 4 t S cannot flip.  A target that may flip moves the confidence term by
at most |logit| / (2 n (L - 1)), which its bound adds.  Counts are exact.
At B = 32 one pair's share of a gradient is 1/32, below the bf16 gradient bars: that the pairs are summed with the right
weights is held by bench_fp32, whose bar is 100 times smaller, and by the negative controls.

Negative controls (CPU, toy sizes, no library call): the gradient check rejects one pair's gradient left out of the sum,
the mean taken over B - 1 pairs, and one chunk's gradient weighted as if it were the whole batch; the log-assignment
check rejects the cross-attention partner shifted by one pair.  Each wrong answer is built from the reference itself.
The gradient controls and the partner control use the fp32 bars: in the two-layer toy model a shifted partner moves the
log-assignment by 0.5 % of the pair's scale, which the bf16 bars (3.5e-2, 4.3e-2) do not resolve.
"""
import gc
import math
import time

import pytest
import torch
from torch.utils.checkpoint import checkpoint

import tests.test_gpu_pair_edges as tpe
from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.homography_matcher import HomographyMatcher
from gluefactory_b200.matchers.lightglue import LightGlue
from gluefactory_b200.trainer import MatcherTrainer
from oracle import lightglue_oracle as O
from tests.util import report

DEV = "cuda"
U32, UBF = 2.0 ** -24, 2.0 ** -8
STAGES = 9 * 6 + 3
TOL32 = STAGES * 46 * U32
TOLM, TOLB = 9 * UBF, 11 * UBF
GTOL32, GTOLM, GTOLB = 2 * TOL32 + math.sqrt(131072) * U32, 41 * UBF, 63 * UBF
CHUNK = 2  # pairs per reference chunk
PEAK_GIB = 24.0  # bound of the reference's peak device memory (the step's own peak is the trainer's, reported apart)
GT_BENCH = {"th_positive": 3.0, "th_negative": 3.0, "transposed_assignment": True}
D128 = dict(synthetic.DEFAULT_CONF, descriptor_dim=128, input_dim=128, num_heads=4)

CASES = {
    "bench": ("bf16", 32, 2048, 2048, synthetic.DEFAULT_CONF, GT_BENCH),
    "bench_fp32": ("fp32", 32, 2048, 2048, synthetic.DEFAULT_CONF, {"th_positive": 3.0, "th_negative": 3.0}),
    "lists": ("bf16", 32, 2048, 2048, synthetic.DEFAULT_CONF, dict(GT_BENCH, transposed_assignment=False,
                                                                  dense_assignment=False)),
    "ragged": ("bf16", 8, 2048, 1536, synthetic.DEFAULT_CONF, GT_BENCH),
    "d128": ("bf16", 8, 2048, 2048, D128, GT_BENCH),
}


@pytest.fixture(scope="module", autouse=True)
def _no_tf32():
    """fp32 products in true fp32, for the fp32 path and for the mirror (restored after this file)."""
    saved = torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False
    yield
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = saved


def bars(precision, kind, tol_scale):
    """check_lg's bars for this step; tol_scale = the largest pair scale S of the chunk."""
    tol, gtol = {("fp32", "fp64"): (TOL32, GTOL32), ("bf16", "fp64"): (TOLB, GTOLB),
                 ("bf16", "mirror"): (TOLM, GTOLM)}[(precision, kind)]
    return {"tol": tol, "gtol": gtol, "thr": 4 * (TOL32 if precision == "fp32" else TOLB) * tol_scale}


# ================================================================================================
# the reference, chunk by chunk
# ================================================================================================
def _ckpt_layer(*args):
    return checkpoint(O.transformer_layer, *args, use_reentrant=False)


def _shifted_partner_layer(d0, d1, th0, th1, w, i, H, rnd):
    """transformer_layer with each pair's cross-attention partner taken from the next pair (negative control)."""
    d0 = O.self_block(d0, th0, w, f"transformers.{i}.self_attn", H, rnd)
    d1 = O.self_block(d1, th1, w, f"transformers.{i}.self_attn", H, rnd)
    pre = f"transformers.{i}.cross_attn"
    y0, _ = O.cross_block(d0, d1.roll(-1, 0), w, pre, H, rnd)
    _, y1 = O.cross_block(d0.roll(-1, 0), d1, w, pre, H, rnd)
    return y0, y1


def _slice(d, lo, hi, dtype):
    out = {}
    for k, v in d.items():
        if isinstance(v, dict):
            out[k] = _slice(v, lo, hi, dtype)
        else:
            out[k] = v[lo:hi].to(dtype) if v.is_floating_point() else v[lo:hi]
    return out


def dense_labels(labels, N):
    """gt_assignment from the match lists when the step trained without the mask (one-to-one lists: the same mask)."""
    if "gt_assignment" in labels:
        return labels["gt_assignment"]
    m0 = labels["gt_matches0"]
    return torch.zeros(*m0.shape, N, dtype=torch.bool, device=m0.device).scatter_(
        2, m0.clamp(min=0)[..., None], (m0 >= 0)[..., None])


def ref_chunk(conf, w, data, dtype, rnd=None, layer=_ckpt_layer, heads=True):
    """Oracle on one chunk of pairs: (pred, losses, heads, d(sum of the chunk's totals) / d(weights)).  heads: per
    layer (log-assignment, sim, token logits), for the pair scales and index margins."""
    wr = {k: v.to(dtype).requires_grad_(True) for k, v in w.items()}
    rnd = O._id if rnd is None else rnd
    rp = O.lightglue_forward(wr, data, conf, rnd=rnd, layer=layer)
    rl = O.lightglue_loss(wr, rp, data, conf, training=True, rnd=rnd)
    names = list(wr)
    gs = torch.autograd.grad(rl["total"].sum(), [wr[k] for k in names], allow_unused=True)
    grads = {k: (g if g is not None else torch.zeros_like(wr[k])) for k, g in zip(names, gs)}
    hs = []
    if heads:
        with torch.no_grad():
            for i in range(conf["n_layers"]):
                d0, d1 = rp["ref_descriptors0"][:, i], rp["ref_descriptors1"][:, i]
                la, sim = O.match_assignment(d0, d1, wr, i)
                z = None
                if i < conf["n_layers"] - 1:
                    pre = f"token_confidence.{i}.token.0"
                    z = [(d @ wr[pre + ".weight"].t() + wr[pre + ".bias"]).squeeze(-1) for d in (d0, d1)]
                hs.append((la, sim, z))
    det = lambda v: v.detach() if torch.is_tensor(v) else torch.tensor(v)  # noqa: E731
    pred = {k: det(v) for k, v in rp.items() if not k.startswith("ref_descriptors")}
    return pred, {k: det(v) for k, v in rl.items()}, hs, grads


def combine(pieces, B):
    """The gradient of mean over B pairs from per-chunk gradients of the chunk's sum."""
    return {k: sum(p[k] for p in pieces) / B for k in pieces[0]}


def with_final_arg(pred):
    """A reference pred with the token-confidence targets the plugin's pred carries (argmax over [scores | dustbin])."""
    la = pred["log_assignment"]
    return dict(pred, _b200_final_arg=(la[:, :-1, :].argmax(2), la[:, :, :-1].argmax(1)))


# ================================================================================================
# the step under test
# ================================================================================================
def run_step(name):
    """One eager step of the benchmark's trainer on the case's batch -> what it computed, and (bench) the replay."""
    precision, B, M, N, conf, gt_conf = CASES[name]
    model = LightGlue(dict(conf, precision=precision))
    model.load_state_dict(synthetic.make_weights(conf, seed=0), strict=False)
    model = model.to(DEV)
    gt = HomographyMatcher(gt_conf)
    trainer = MatcherTrainer(model, lr=1e-4, ground_truth=gt)
    data = synthetic.to_device(synthetic.make_pairs(B, N, seed=1234, D=conf["input_dim"], M=M, with_gt=False), DEV)
    fp = trainer.fp
    names = [fp._names[id(p)] for p in fp.params]
    saved = [t.clone() for t in trainer._state_tensors()]
    weights = {n: fp.flat[off:off + p.numel()].view_as(p).clone() for n, p, off in zip(names, fp.params, fp.offsets)}
    seen = {}
    hook = model.register_forward_hook(lambda mod, args, out: seen.update(data=args[0], pred=out))
    loss, losses = trainer.step(data)
    hook.remove()
    torch.cuda.synchronize()
    grads = {n: fp.grad[off:off + p.numel()].view_as(p).clone() for n, p, off in zip(names, fp.params, fp.offsets)}
    keep = ("log_assignment", "matches0", "matches1", "matching_scores0", "matching_scores1")
    pred = {k: seen["pred"][k].detach() for k in keep}
    pred["_b200_final_arg"] = tuple(t.detach() for t in seen["pred"]["_b200_final_arg"])
    labels = {k: v for k, v in seen["data"].items() if k.startswith("gt_")}
    out = dict(weights=weights, grads=grads, pred=pred, losses={k: v.detach() for k, v in losses.items()
                                                                  if torch.is_tensor(v)},
               labels=labels, data=data, gt=gt)
    eager = (loss.clone(), fp.grad.clone(), fp.flat.clone())
    del seen, losses, loss  # nothing may keep the eager step's autograd graph alive into a capture
    if name == "bench":
        def restore():
            for t, s in zip(trainer._state_tensors(), saved):
                t.copy_(s)
        restore()
        trainer.capture(data, torch.device(DEV))
        replays = []
        for _ in range(2):
            restore()
            l, _ = trainer.step_graphed(data)
            torch.cuda.synchronize()
            replays.append((l.clone(), fp.grad.clone(), fp.flat.clone()))
        out["replay"] = (eager, replays)
    del trainer, model, eager
    gc.collect()
    torch.cuda.empty_cache()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", list(CASES))
def test_bench_step_against_fp64(name):
    precision, B, M, N, conf, _ = CASES[name]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.time()
    step = run_step(name)
    if name == "bench":
        (le, ge, fe), ((l1, g1, f1), (l2, g2, f2)) = step["replay"]
        assert torch.equal(l1, le) and torch.equal(g1, ge) and torch.equal(f1, fe), "replay differs from the eager step"
        assert torch.equal(l2, l1) and torch.equal(g2, g1) and torch.equal(f2, f1), "two replays differ"
        del step["replay"]
    # the labels the step trained on are the ground-truth component's for this batch
    again = step["gt"](step["data"])
    assert set(step["labels"]) == {"gt_" + k for k in again}, (sorted(step["labels"]), sorted(again))
    for k, v in again.items():
        assert torch.equal(step["labels"]["gt_" + k], v), k
    assert ("gt_assignment" in step["labels"]) == (name != "lists")
    assert ("gt_assignment_t" in step["labels"]) == (CASES[name][5].get("transposed_assignment", False))
    t_step = time.time() - t0
    torch.cuda.synchronize()
    peak_step = torch.cuda.max_memory_allocated() / 2 ** 30  # the trainer's own (fp32 at B = 32: about 31 GiB)
    torch.cuda.reset_peak_memory_stats()
    tpe.WORST.clear()
    w = step["weights"]
    lab = dict(step["labels"], gt_assignment=dense_labels(step["labels"], N))
    pieces, mirror_pieces = [], []
    for lo in range(0, B, CHUNK):
        hi = min(B, lo + CHUNK)
        d64 = dict(_slice(step["data"], lo, hi, torch.float64), **_slice(lab, lo, hi, torch.float64))
        rp, rl, heads, g64 = ref_chunk(conf, w, d64, torch.float64)
        pieces.append(g64)
        S = max(tpe.pair_scale(heads, b) for b in range(hi - lo))
        pred = {k: (tuple(t[lo:hi] for t in v) if isinstance(v, tuple) else v[lo:hi]) for k, v in step["pred"].items()}
        losses = {k: v[lo:hi] for k, v in step["losses"].items() if v.dim() == 1 and v.shape[0] == B}
        tag = f"{name}:pairs{lo}-{hi - 1}"
        tpe.check_lg(tag, conf, pred, losses, None, (rp, rl, None, heads), precision, "fp64",
                     bars=bars(precision, "fp64", S))
        del d64, rp, rl
        if precision == "bf16":
            d32 = dict(_slice(step["data"], lo, hi, torch.float32), **_slice(lab, lo, hi, torch.float32))
            mp, ml, _, g32 = ref_chunk(conf, w, d32, torch.float32, rnd=O.Bf16Mirror(), heads=False)
            mirror_pieces.append(g32)
            tpe.check_lg(tag, conf, pred, losses, None, (mp, ml, None, heads), precision, "mirror",
                         bars=bars(precision, "mirror", S))
            del d32, mp, ml
        del heads
    tpe.check_grads(name, step["grads"], combine(pieces, B), bars(precision, "fp64", 1.0)["gtol"], precision, "fp64")
    if mirror_pieces:
        tpe.check_grads(name, step["grads"], combine(mirror_pieces, B), GTOLM, precision, "mirror")
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 2 ** 30  # the reference and the checks, the step's outputs resident
    report(f"test_gpu_bench_step {name}", seconds=time.time() - t0, step_seconds=t_step, step_peak_gib=peak_step,
           reference_peak_gib=peak)
    for key, (ratio, where) in sorted(tpe.WORST.items()):
        report(f"test_gpu_bench_step worst err/bound {name} {key}", ratio=ratio, at=where)
    assert peak < PEAK_GIB, peak


# ================================================================================================
# negative controls: each check rejects a wrong answer built from its own reference (CPU, no library call)
# ================================================================================================
TOY = dict(synthetic.DEFAULT_CONF, n_layers=2, descriptor_dim=64, input_dim=64, num_heads=2)


def _toy(B=4, N=24):
    w = {k: v.double() for k, v in synthetic.make_weights(TOY, seed=11).items()}
    data = synthetic.make_pairs(B, N, seed=12, D=64, dtype=torch.float64)
    return w, data


def _toy_pieces(w, data, chunk):
    B = data["keypoints0"].shape[0]
    return [ref_chunk(TOY, w, _slice(data, lo, lo + chunk, torch.float64), torch.float64)
            for lo in range(0, B, chunk)]


def _reject_grads(wrong, ref):
    with pytest.raises(AssertionError):
        tpe.check_grads("control", wrong, ref, GTOL32, "fp32", "fp64")


def test_gradient_check_rejects_wrong_pair_sums():
    w, data = _toy()
    B = 4
    per_pair = [p[3] for p in _toy_pieces(w, data, 1)]
    ref = combine(per_pair, B)
    tpe.check_grads("control", ref, ref, GTOL32, "fp32", "fp64")  # the right answer passes
    # the same reference in chunks of two pairs is the same sum
    tpe.check_grads("control", combine([p[3] for p in _toy_pieces(w, data, 2)], B), ref, GTOL32, "fp32", "fp64")
    # one pair's gradient missing from the sum
    _reject_grads(combine(per_pair[:2] + per_pair[3:], B), ref)
    # the mean taken over B - 1 pairs
    _reject_grads(combine(per_pair, B - 1), ref)
    # a chunk's gradient weighted as if it were the whole batch (its own mean: 1 / 2 in place of 1 / B)
    chunks = [p[3] for p in _toy_pieces(w, data, 2)]
    wrong = {k: chunks[0][k] / 2 + chunks[1][k] / B for k in ref}
    _reject_grads(wrong, ref)


def test_log_assignment_check_rejects_a_shifted_cross_attention_partner():
    w, data = _toy()
    rp, rl, heads, _ = ref_chunk(TOY, w, data, torch.float64)
    S = max(tpe.pair_scale(heads, b) for b in range(4))
    for precision, kind in (("fp32", "fp64"), ("bf16", "fp64"), ("bf16", "mirror")):
        tpe.check_lg("control", TOY, with_final_arg(rp), rl, None, (rp, rl, None, heads), precision, kind,
                     bars=bars(precision, kind, S))  # the right answer passes every bar
    sp, sl, _, _ = ref_chunk(TOY, w, data, torch.float64, layer=_shifted_partner_layer, heads=False)
    with pytest.raises(AssertionError):
        tpe.check_lg("control", TOY, with_final_arg(sp), sl, None, (rp, rl, None, heads), "fp32", "fp64",
                     bars=bars("fp32", "fp64", S))
