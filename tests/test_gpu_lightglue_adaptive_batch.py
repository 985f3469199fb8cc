"""GPU: LightGlue's adaptive depth / width (eval mode, `depth_confidence` / `width_confidence` > 0) on batches of pairs.

Contract: for each pair of a batch, the outputs equal what a one-pair call returns for that pair alone -- the same
matches0/1, prune0/1 and stop layer, matching scores and log-assignment within the bars of the one-pair adaptive
tests (tests/test_gpu_matcher.py, tests/test_gpu_lightglue_hd32.py: 1e-3 relative / 1e-3 absolute on the
log-assignment, 1e-3 / 1e-6 on the scores).  The batch's log-assignment is [B, M+1, N+1] in the original indexing
with -inf rows / columns at pruned points, so each pair's one-pair matrix is its survivors' rows and columns plus the
dustbins.

Batches of 3-5 synthetic pairs with different planted-match fractions.  The thresholds are picked from the pairs'
own token statistics (a training-mode forward exposes every layer's state) so that the pairs stop at different
layers and prune by different amounts: token-confidence biases that make the confident share rise with depth,
depth_confidence halfway between two pairs' confidence ratios, and
1 - width_confidence at the lowest 30th percentile of the layers' matchabilities (with early stopping as well: at
the median of layer 0's).  The golden pairs of the one-pair pruning tests
are also run inside a batch and held to those tests' bars, and the compaction kernel is checked against a torch
restatement (torch.where per pair).

Budget: under a minute and under 4 GiB of device memory on one H100, recorded by the module fixture."""
import ast
import math
import os
import time

import numpy as np
import pytest
import torch

from gluefactory_b200 import ops, synthetic
from gluefactory_b200.matchers.lightglue import LightGlue
from tests.util import GOLDEN, report

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _file_budget():
    """Wall time and peak device memory of this file (the machines running it are shared)."""
    torch.cuda.reset_peak_memory_stats()
    t = time.time()
    yield
    torch.cuda.synchronize()
    report("test_gpu_lightglue_adaptive_batch", seconds=time.time() - t,
           peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)


def _build(conf, weights, precision):
    model = LightGlue(dict(conf, precision=precision))
    missing, unexpected = model.load_state_dict({k: v.float() for k, v in weights.items()}, strict=False)
    assert not unexpected and missing in ([], ["confidence_thresholds"])
    return model.to(DEV).eval()


def _pair_inputs(p):
    return {"keypoints0": p["keypoints0"], "keypoints1": p["keypoints1"], "descriptors0": p["descriptors0"],
            "descriptors1": p["descriptors1"], "view0": {"image_size": p["view0"]["image_size"]},
            "view1": {"image_size": p["view1"]["image_size"]}}


def _cat(pairs):
    c = lambda key: torch.cat([p[key] for p in pairs])  # noqa: E731
    return synthetic.to_device({"keypoints0": c("keypoints0"), "keypoints1": c("keypoints1"),
                                "descriptors0": c("descriptors0"), "descriptors1": c("descriptors1"),
                                "view0": {"image_size": torch.cat([p["view0"]["image_size"] for p in pairs])},
                                "view1": {"image_size": torch.cat([p["view1"]["image_size"] for p in pairs])}}, DEV)


def _pairs(n_pairs, N, M, D, seed):
    fracs = np.linspace(0.1, 0.8, n_pairs)
    return [_pair_inputs(synthetic.make_pairs(1, N, seed=seed + i, D=D, M=M, frac=float(f)))
            for i, f in enumerate(fracs)]


def _token_stats(conf, w, precision, pairs):
    """Per pair and layer i < L-1: the confidence ratio 1 - #(token < thr_i) / (M + N); per layer: the matchabilities and
    the token-confidence pre-activations x . w_i of the un-pruned states (a training-mode forward keeps every layer's
    output)."""
    model = _build(dict(conf, depth_confidence=-1, width_confidence=-1), w, precision).train()
    L = conf["n_layers"]
    ratios, match, pre = [], [[] for _ in range(L - 1)], [[] for _ in range(L - 1)]
    with torch.no_grad():
        for p in pairs:
            pred = model(synthetic.to_device(p, DEV))
            r = []
            for i in range(L - 1):
                x = pred["_b200_layers"][i]
                tk, la = model.token_confidence[i].token[0], model.log_assignment[i].matchability
                tok = torch.sigmoid(x @ tk.weight.view(-1) + tk.bias)
                r.append(1.0 - float((tok < model.confidence_thresholds[i]).float().sum()) / x.shape[0])
                match[i].append(torch.sigmoid(x @ la.weight.view(-1) + la.bias))
                pre[i].append(x @ tk.weight.view(-1))
            ratios.append(r)
    return ratios, [torch.cat(m) for m in match], [torch.cat(a) for a in pre], model.confidence_thresholds


def _calibrate_confidence(w, pre, thr):
    """Token-confidence biases under which about 50, 60, 70, ... % of the points are confident after layer 0, 1, 2, ...
    (synthetic weights can leave every point below its threshold), so that the pairs' ratios rise with depth and
    differ from pair to pair."""
    w = dict(w)
    for i, a in enumerate(pre):
        t = float(thr[i])
        w[f"token_confidence.{i}.token.0.bias"] = torch.tensor([math.log(t / (1 - t)) -
                                                               float(a.float().quantile(0.5 - 0.1 * i))])
    return w


def _pick_depth(ratios, L):
    """A depth_confidence, clear of every ratio by > 1e-3, under which the most distinct stop layers occur."""
    vals = sorted({v for r in ratios for v in r})
    best, best_n = None, 0
    for a, b in zip(vals, vals[1:]):
        if b - a < 2e-3:
            continue
        dc = 0.5 * (a + b)
        stops = {next((i for i, v in enumerate(r) if v > dc), L - 1) for r in ratios}
        if len(stops) > best_n:
            best, best_n = dc, len(stops)
    return best, best_n


def _check_pair_against_single(pb, ps, b, M, N, tag):
    """Pair b of the batched pred pb against the one-pair pred ps."""
    for k in ("matches0", "matches1", "prune0", "prune1"):
        assert torch.equal(pb[k][b], ps[k][0]), (tag, k)
    assert int(pb["stop_layer"][b]) == ps["stop_layer"], tag
    for k in ("matching_scores0", "matching_scores1"):
        np.testing.assert_allclose(pb[k][b].cpu().numpy(), ps[k][0].cpu().numpy(), rtol=1e-3, atol=1e-6, err_msg=tag)
    la_b = pb["log_assignment"][b]
    m, n = ps["log_assignment"].shape[1] - 1, ps["log_assignment"].shape[2] - 1
    s0 = torch.isfinite(la_b[:M, N])  # a survivor's row and column hold finite scores, a pruned point's are -inf
    s1 = torch.isfinite(la_b[M, :N])
    assert int(s0.sum()) == m and int(s1.sum()) == n, tag
    rows = torch.cat([torch.where(s0)[0], torch.tensor([M], device=DEV)])
    cols = torch.cat([torch.where(s1)[0], torch.tensor([N], device=DEV)])
    got = la_b[rows][:, cols]
    np.testing.assert_allclose(got.cpu().numpy(), ps["log_assignment"][0].cpu().numpy(), rtol=1e-3, atol=1e-3,
                               err_msg=tag)
    pruned = torch.ones(M + 1, dtype=torch.bool, device=DEV)
    pruned[rows] = False
    assert torch.isneginf(la_b[pruned]).all(), tag
    return float((got - ps["log_assignment"][0]).abs().max())


MODES = {"depth": (True, False), "width": (False, True), "both": (True, True)}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("D,H", [(256, 4), (128, 4)])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_batch_equals_one_pair_calls(precision, D, H, mode):
    n_pairs = {"depth": 4, "width": 3, "both": 5}[mode]
    M, N, L = 224, 256, 5
    conf = dict(synthetic.DEFAULT_CONF, descriptor_dim=D, input_dim=D, num_heads=H, n_layers=L)
    w = synthetic.make_weights(conf, seed=300 + D)
    pairs = _pairs(n_pairs, N, M, D, seed=400 + D + 10 * len(mode))
    use_depth, use_width = MODES[mode]
    ratios, match, pre, thr = _token_stats(conf, w, precision, pairs)
    if use_depth:
        w = _calibrate_confidence(w, pre, thr)
        ratios, match, _, _ = _token_stats(conf, w, precision, pairs)
    dc, n_stops = _pick_depth(ratios, L) if use_depth else (-1, 1)
    # width only: no layer prunes more than about 30 % of its points, so no view runs empty over the four pruning
    # steps; with early stopping the pairs stop within the first layers and half of the points are exempt as
    # low-confidence ones, so the threshold is layer 0's median
    if use_width:
        wc = 1.0 - (float(match[0].median()) if use_depth else min(float(m.quantile(0.3)) for m in match))
    else:
        wc = -1
    if use_depth:
        assert dc is not None and n_stops >= 2, ratios
    conf = dict(conf, depth_confidence=dc, width_confidence=wc)
    model = _build(conf, w, precision)
    with torch.no_grad():
        pb = model(_cat(pairs))
        singles = [model(synthetic.to_device(p, DEV)) for p in pairs]
    worst = 0.0
    for b, ps in enumerate(singles):
        worst = max(worst, _check_pair_against_single(pb, ps, b, M, N, f"{precision} D{D} {mode} pair {b}"))
    stops = pb["stop_layer"].tolist()
    kept = [int((pb["prune0"][b] == pb["prune0"][b].max()).sum()) for b in range(n_pairs)]
    report(f"adaptive batch {precision} D{D} H{H} {mode}", la_max_abs=worst, stops=str(stops), kept0=str(kept))
    if mode == "depth":  # with pruning as well, the stop layers follow from the pruned states
        assert len(set(stops)) >= 2, stops
    if use_width:
        assert len(set(kept)) >= 2, kept
    assert pb["log_assignment"].shape == (n_pairs, M + 1, N + 1)
    assert pb["ref_descriptors0"].shape == (n_pairs, 1, M, D)
    with pytest.raises(ValueError, match="several pairs"):
        model.loss(pb, {})


@pytest.mark.parametrize("golden", ["adaptive_prune", "lg_hd32_d128_h4_adaptive_prune"])
def test_golden_pair_inside_a_batch(golden):
    """The one-pair pruning fixtures (fp32, produced by the unmodified reference), with the golden pair in the middle
    of a batch of three: the bars of their one-pair tests."""
    g = dict(np.load(os.path.join(GOLDEN, golden + ".npz")))
    conf = ast.literal_eval(str(g["meta|conf"]))
    seed, M, N = int(g["meta|seed"]), int(g["meta|M"]), int(g["meta|N"])
    D = conf["input_dim"]
    model = _build(conf, synthetic.make_weights(conf, seed=seed), "fp32")
    gold = _pair_inputs(synthetic.make_pairs(1, N, seed=seed + 1, D=D, M=M))
    others = [_pair_inputs(synthetic.make_pairs(1, N, seed=seed + 50 + i, D=D, M=M, frac=f))
              for i, f in enumerate((0.1, 0.7))]
    with torch.no_grad():
        pred = model(_cat([others[0], gold, others[1]]))
    b = 1
    p0, p1 = pred["prune0"][b].cpu().numpy(), pred["prune1"][b].cpu().numpy()
    assert np.array_equal(p0, g["pred|prune0"][0]) and np.array_equal(p1, g["pred|prune1"][0])
    assert np.array_equal(pred["matches0"][b].cpu().numpy(), g["pred|matches0"][0])
    assert np.array_equal(pred["matches1"][b].cpu().numpy(), g["pred|matches1"][0])
    np.testing.assert_allclose(pred["matching_scores0"][b].cpu().numpy(), g["pred|matching_scores0"][0], rtol=1e-3,
                               atol=1e-6)
    rows = np.concatenate([np.where(p0 == p0.max())[0], [M]])
    cols = np.concatenate([np.where(p1 == p1.max())[0], [N]])
    la = pred["log_assignment"][b].cpu().numpy()[np.ix_(rows, cols)]
    assert la.shape == g["pred|log_assignment"].shape[1:]
    np.testing.assert_allclose(la, g["pred|log_assignment"][0], rtol=1e-3, atol=1e-3)
    report(f"adaptive batch golden {golden}", la_max_abs=float(np.abs(la - g["pred|log_assignment"][0]).max()))


def _compact_reference(x, theta, ind, zt, seg, B, M, N, thr, dc, wc, layer):
    """torch restatement of one lgb200_adaptive_compact step, pair by pair with torch.where."""
    off, ln = seg[0].tolist(), seg[1].tolist()
    xs, ts, js, new_len = [], [], [], []
    stop = {}
    prune0, prune1 = torch.zeros(B, M, dtype=torch.int64), torch.zeros(B, N, dtype=torch.int64)
    for b in range(B):
        sl = [slice(off[2 * b + j], off[2 * b + j] + ln[2 * b + j]) for j in range(2)]
        if ln[2 * b] == 0 and ln[2 * b + 1] == 0:
            new_len += [0, 0]
            continue
        tok = [torch.sigmoid(zt[s, 1]) for s in sl]
        if dc > 0 and 1.0 - float(sum((t < thr).float().sum() for t in tok)) / (M + N) > dc:
            stop[b] = sl
            new_len += [0, 0]
            continue
        for j, s in enumerate(sl):
            keep = torch.sigmoid(zt[s, 0]) > (1 - wc)
            if dc > 0:
                keep = keep | (tok[j] <= thr)
            k = torch.where(keep)[0]
            xs.append(x[s][k]), ts.append(theta[s][k]), js.append(ind[s][k])
            new_len.append(int(k.numel()))
            (prune0 if j == 0 else prune1)[b, ind[s][k].long()] += 1
    return torch.cat(xs), torch.cat(ts), torch.cat(js), new_len, stop, prune0, prune1


def test_compaction_kernel_against_torch_where():
    """One stop / prune step on a packed state of four pairs in the pair-major layout, one pair already stopped: the
    packed outputs, the new segments, the prune counters, the final buffer of the pair that stops and the status."""
    torch.manual_seed(0)
    B, M, N, D, R = 4, 300, 260, 256, 32
    lens = [300, 260, 0, 0, 17, 250, 129, 1]   # pair 1 stopped earlier
    offs = np.concatenate([[0], np.cumsum(lens)[:-1]]).tolist()
    T = sum(lens)
    x = torch.randn(T, D)
    theta = torch.randn(T, R)
    ind = torch.cat([torch.randperm(M if s % 2 == 0 else N)[:n].sort().values for s, n in enumerate(lens)]).int()
    zt = torch.randn(T, 2) * 3
    # pair 2's tokens confident (it stops at the ratio test), the others' not
    zt[offs[4]:offs[4] + 17 + 250, 1] = 8.0
    zt[offs[6]:, 1] = -8.0 * (torch.rand(T - offs[6]) < 0.6) + 4.0
    thr, dc, wc, layer = 0.85, 0.9, 0.5, 3
    # keep every decision clear of its threshold (the restatement is not the kernel's arithmetic)
    zt[:, 0] = torch.where(zt[:, 0].abs() < 1e-3, torch.full_like(zt[:, 0], 0.5), zt[:, 0])
    off_p = [offs[s ^ 1] for s in range(2 * B)]
    len_p = [lens[s ^ 1] for s in range(2 * B)]
    seg = torch.tensor([offs, lens, off_p, len_p], dtype=torch.int32)
    ref = _compact_reference(x, theta, ind, zt, seg, B, M, N, torch.tensor(thr), dc, wc, layer)
    i32 = dict(device=DEV, dtype=torch.int32)
    fin = {"x": torch.zeros(B * (M + N), D, device=DEV), "ind": torch.full((B * (M + N),), -7, **i32),
           "len": torch.zeros(2 * B, **i32), "stop": torch.full((B,), 9, **i32),
           "prune0": torch.zeros(B, M, device=DEV, dtype=torch.int64),
           "prune1": torch.zeros(B, N, device=DEV, dtype=torch.int64)}
    xo, to, io, so, status = ops.adaptive_compact(x.to(DEV), theta.to(DEV), ind.to(DEV), zt.to(DEV), seg.to(DEV), fin,
                                                  layer, (B, M, N), conf_thr=torch.tensor([thr], device=DEV),
                                                  depth_conf=dc, width_conf=wc)
    kept, emptied = status.tolist()
    rx, rt, ri, new_len, stop, rp0, rp1 = ref
    assert kept == rx.shape[0] and emptied == 0
    assert torch.equal(xo[:kept].cpu(), rx) and torch.equal(to[:kept].cpu(), rt) and torch.equal(io[:kept].cpu(), ri)
    new_off = np.concatenate([[0], np.cumsum(new_len)[:-1]]).tolist()
    assert so.cpu().tolist() == [new_off, new_len, [new_off[s ^ 1] for s in range(2 * B)],
                                 [new_len[s ^ 1] for s in range(2 * B)]]
    assert torch.equal(fin["prune0"].cpu(), rp0) and torch.equal(fin["prune1"].cpu(), rp1)
    assert list(stop) == [2] and fin["stop"].cpu().tolist() == [9, 9, layer, 9]
    assert fin["len"].cpu().tolist() == [0, 0, 0, 0, 17, 250, 0, 0]
    base = 2 * (M + N)
    s0, s1 = stop[2]
    assert torch.equal(fin["x"][base:base + 17].cpu(), x[s0]) and torch.equal(fin["x"][base + M:base + M + 250].cpu(), x[s1])
    assert torch.equal(fin["ind"][base:base + 17].cpu(), ind[s0])
    assert torch.equal(fin["ind"][base + M:base + M + 250].cpu(), ind[s1])
    # a step that empties a view is reported, not packed silently
    zt2 = zt.clone()
    zt2[offs[7], :] = -20.0  # pair 3's only image-1 token: unmatchable and confident
    *_, status2 = ops.adaptive_compact(x.to(DEV), theta.to(DEV), ind.to(DEV), zt2.to(DEV), seg.to(DEV), fin, layer,
                                       (B, M, N), conf_thr=torch.tensor([thr], device=DEV), depth_conf=-1, width_conf=wc)
    assert status2.tolist()[1] == 1


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_outputs_keep_the_plain_forwards_dtypes(precision):
    """The adaptive forward returns every key it shares with the plain eval forward in that forward's dtype, for one
    pair and for a batch: prune0/1 stay fp32 n_layers without point pruning (lightglue.py:528-529), and are int64
    layer counts with it."""
    conf = dict(synthetic.DEFAULT_CONF, n_layers=3)
    w = synthetic.make_weights(conf, seed=31)
    pairs = _pairs(3, 192, 160, 256, seed=32)
    plain = _build(conf, w, precision)
    with torch.no_grad():
        ref = plain(synthetic.to_device(pairs[0], DEV))
        for depth, width in ((0.99, -1), (-1, 0.99), (0.99, 0.99)):
            model = _build(dict(conf, depth_confidence=depth, width_confidence=width), w, precision)
            for data in (synthetic.to_device(pairs[0], DEV), _cat(pairs)):
                pred = model(data)
                for k in ("matches0", "matches1", "matching_scores0", "matching_scores1", "log_assignment"):
                    assert pred[k].dtype == ref[k].dtype, (k, depth, width)
                want = torch.int64 if width > 0 else ref["prune0"].dtype
                assert pred["prune0"].dtype == pred["prune1"].dtype == want, (depth, width, pred["prune0"].dtype)
                if width <= 0:
                    assert (pred["prune0"] == conf["n_layers"]).all() and (pred["prune1"] == conf["n_layers"]).all()
    assert ref["prune0"].dtype == torch.float32


def test_compaction_rejects_a_non_fp32_threshold():
    """The per-layer confidence threshold is read on the device as one fp32: another dtype is refused, not
    reinterpreted."""
    x, theta = torch.zeros(8, 256, device=DEV), torch.zeros(8, 32, device=DEV)
    ind, zt = torch.arange(8, device=DEV, dtype=torch.int32) % 4, torch.zeros(8, 2, device=DEV)
    seg = torch.tensor([[0, 4], [4, 4], [4, 0], [4, 4]], device=DEV, dtype=torch.int32)
    i32 = dict(device=DEV, dtype=torch.int32)
    fin = {"x": torch.zeros(8, 256, device=DEV), "ind": torch.zeros(8, **i32), "len": torch.zeros(2, **i32),
           "stop": torch.zeros(1, **i32), "prune0": torch.ones(1, 4, device=DEV, dtype=torch.int64),
           "prune1": torch.ones(1, 4, device=DEV, dtype=torch.int64)}
    with pytest.raises(AssertionError):
        ops.adaptive_compact(x, theta, ind, zt, seg, fin, 0, (1, 4, 4), conf_thr=torch.tensor([0.9], device=DEV,
                             dtype=torch.float64), depth_conf=0.5, width_conf=0.5)
