"""Generate the early-stopping LightGlue fixtures tests/golden/lg_adaptive_*.npz by running the UNMODIFIED reference
LightGlue (gluefactory/models/matchers/lightglue.py) on the CPU in eval mode, fp32, with `depth_confidence` > 0 (and
`width_confidence` > 0 in cases b-d).  Test infrastructure only; it needs the reference tree ($GLUEFACTORY_REFERENCE)
and the omegaconf stand-in of oracle/_shim, like oracle/make_golden.py, whose helpers it uses.  It writes no other
fixture.

    python scripts/make_lightglue_adaptive_golden.py

The reference takes the early-stopping branch (lightglue.py:491-495) but then fails at `torch.stack(all_desc0, 1)`
(lightglue.py:536): after the `break` the list of per-layer states is empty.  Everything recorded here is computed
before that line (lightglue.py:513-526: the stop layer's assignment head, `filter_matches` and the scatter to the
original keypoint indices), so during the forward call `torch.stack` is replaced by a stand-in that returns an empty
tensor for an empty list and calls the original otherwise; the stand-in is removed in a `finally`.

`check_if_stop` and `get_pruning_mask` are observed (not changed) to record each pair's stop layer, which the reference
does not return, its count of low-confidence tokens at every layer it checked, and the distance of every decision from
its threshold.  A case is kept only if no recorded decision depends on fp32 rounding:
  - every stop test's ratio 1 - low / (M + N) is at least 3 tokens, 3 / (M + N), away from depth_confidence;
  - every matchability clears 1 - width_confidence by more than 2e-4;
  - every token confidence that decides the low-confidence exemption (the points whose matchability is not above the
    width threshold) clears its layer's threshold by more than 2e-4.

Weights come from `synthetic.make_weights(conf, seed)` with the token-confidence biases replaced by calibrated ones
(stored in the fixture): as in tests/test_gpu_lightglue_adaptive_batch.py `_calibrate_confidence`, about 50, 60, 70,
80 % of the un-pruned points are confident after layer 0, 1, 2, 3, so the pairs stop at different layers.  Pairs come
from `synthetic.make_pairs(1, N, seed=pair_seed, D, M, frac)`; every seed and frac is stored.  depth_confidence is
the midpoint of the widest gap between the pairs' un-pruned confidence ratios that gives the most distinct stop
layers; the recorded decisions of the pruned forward are then checked against the rules above.

Stored per pair j (`p{j}|...`): stop layer, per-layer low counts (-1 after the stop layer), prune0/1, matches0/1,
matching_scores0/1 and log_assignment [1, m+1, n+1] over the survivors, as the reference returns it.  Case d (views
of more than 1024 tokens) stores log_assignment as a fixed subset of survivor rows and columns (`la_rows` /
`la_cols` in the survivors' indexing), the dustbin row and column in full and the logsumexp of every row.
"""
import math
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden  # noqa: E402  (puts the reference and oracle/_shim on sys.path)
from gluefactory_b200 import synthetic  # noqa: E402

D256 = dict(synthetic.DEFAULT_CONF)
D128 = dict(synthetic.DEFAULT_CONF, descriptor_dim=128, input_dim=128, num_heads=4)
RATIO_TOKENS, SIG_MARGIN = 3, 2e-4
# The synthetic heads' logits spread by about 0.2-0.4, so among a few thousand sigmoids some land within 2e-4 of any
# threshold.  Scaling the matchability and token-confidence weights spreads them by 32x (the heads of a trained model
# are confident too), so that cases whose every decision clears its threshold exist.
HEAD_SCALE = 32.0

# name -> (model conf, pairs, M, N, width pruning, first weight seed, subset of log_assignment)
CASES = {
    "lg_adaptive_a_depth": (D256, 4, 200, 224, False, 500, False),
    "lg_adaptive_b_both": (D256, 4, 200, 224, True, 520, False),
    "lg_adaptive_c_d128_both": (D128, 4, 200, 224, True, 540, False),
    "lg_adaptive_d_long": (D256, 2, 1100, 1300, True, 560, True),
}
L = 5


def _model(conf, w):
    from gluefactory.models import get_model

    model = get_model("matchers.lightglue")(dict(conf, name="matchers.lightglue"))
    missing, unexpected = model.load_state_dict(w, strict=False)
    assert not unexpected and missing in ([], ["confidence_thresholds"]), (missing, unexpected)
    return model


def head_weights(w, n_layers, scale, token_bias):
    """make_weights' dict with the matchability and token-confidence weights scaled by `scale` and the calibrated
    token-confidence biases (the GPU test rebuilds the fixture's weights with this)."""
    w = dict(w)
    for i in range(n_layers):
        for k in (f"log_assignment.{i}.matchability.weight", f"log_assignment.{i}.matchability.bias",
                  f"token_confidence.{i}.token.0.weight"):
            if k in w:
                w[k] = w[k] * scale
    for i, b in enumerate(token_bias):
        w[f"token_confidence.{i}.token.0.bias"] = torch.tensor([float(b)], dtype=torch.float32)
    return w


def _pairs(n_pairs, M, N, D, seed):
    seeds = [seed + 1 + j for j in range(n_pairs)]
    fracs = [float(f) for f in np.linspace(0.1, 0.8, n_pairs)]
    return seeds, fracs, [synthetic.make_pairs(1, N, seed=s, D=D, M=M, frac=f) for s, f in zip(seeds, fracs)]


def _calibrate(conf, w, pairs):
    """Token-confidence biases from the un-pruned states of a training-mode forward (every layer's state is kept), and
    each pair's confidence ratio per layer under them."""
    model = _model(dict(conf, depth_confidence=-1, width_confidence=-1), w).train()
    thr = model.confidence_thresholds
    states = []
    with torch.no_grad():
        for p in pairs:
            pred = model(p)
            states.append([torch.cat([pred["ref_descriptors0"][0, i], pred["ref_descriptors1"][0, i]])
                           for i in range(L - 1)])
    bias, match = {}, []
    for i in range(L - 1):
        tk = model.token_confidence[i].token[0]
        pre = torch.cat([s[i] for s in states]) @ tk.weight.detach().view(-1)
        t = float(thr[i])
        bias[i] = math.log(t / (1 - t)) - float(pre.quantile(0.5 - 0.1 * i))
        la = model.log_assignment[i].matchability
        match.append(torch.sigmoid(torch.cat([s[i] for s in states]) @ la.weight.detach().view(-1) + la.bias.detach()))
    ratios = []
    for s in states:
        r = []
        for i in range(L - 1):
            tk = model.token_confidence[i].token[0]
            tok = torch.sigmoid(s[i] @ tk.weight.detach().view(-1) + torch.tensor(bias[i], dtype=torch.float32))
            r.append(1.0 - float((tok < thr[i]).float().sum()) / s[i].shape[0])
        ratios.append(r)
    return bias, ratios, match


def _depth_candidates(ratios, tokens):
    """depth_confidence values at the midpoints of the gaps between the pairs' ratios that are wide enough for the
    margin rule: most distinct stop layers first, then the latest stops."""
    vals = sorted({v for r in ratios for v in r})
    cands = []
    for a, b in zip(vals, vals[1:]):
        if (b - a) * tokens < 2 * RATIO_TOKENS + 2:
            continue
        dc = round(0.5 * (a + b), 6)
        stops = [next((i for i, v in enumerate(r) if v > dc), L - 1) for r in ratios]
        cands.append((-len(set(stops)), -sum(stops), -(b - a), dc))
    return [dc for *_, dc in sorted(cands)]


def _run_pair(model, data, conf):
    """One eval-mode forward of the reference with the stop / prune decisions observed."""
    M, N = data["keypoints0"].shape[1], data["keypoints1"].shape[1]
    rec = {"low": [], "stops": [], "ratio_margin": math.inf, "sig_margin": math.inf, "kept": []}
    orig_stop, orig_mask, orig_stack = model.check_if_stop, model.get_pruning_mask, torch.stack
    wthr = 1 - conf["width_confidence"]

    def check_if_stop(c0, c1, layer_index, num_points):
        c = torch.cat([c0, c1], -1)
        low = int((c < model.confidence_thresholds[layer_index]).sum())
        rec["low"].append(low)
        rec["ratio_margin"] = min(rec["ratio_margin"], abs((1 - conf["depth_confidence"]) * num_points - low))
        out = orig_stop(c0, c1, layer_index, num_points)
        rec["stops"].append(bool(out))
        return out

    def get_pruning_mask(confidences, scores, layer_index):
        rec["sig_margin"] = min(rec["sig_margin"], float((scores - wthr).abs().min()))
        if confidences is not None:
            undecided = scores <= wthr  # only these points' exemption depends on their confidence
            if undecided.any():
                thr = model.confidence_thresholds[layer_index]
                rec["sig_margin"] = min(rec["sig_margin"], float((confidences[undecided] - thr).abs().min()))
        keep = orig_mask(confidences, scores, layer_index)
        rec["kept"].append(int(keep.sum()))
        return keep

    def stack(tensors, *args, **kwargs):
        if len(tensors) == 0:
            return torch.empty(0)
        return orig_stack(tensors, *args, **kwargs)

    model.check_if_stop, model.get_pruning_mask = check_if_stop, get_pruning_mask
    torch.stack = stack
    try:
        with torch.no_grad():
            pred = model(data)
    finally:
        torch.stack = orig_stack
        del model.check_if_stop, model.get_pruning_mask
    stop = rec["stops"].index(True) if True in rec["stops"] else L - 1
    rec["stop"] = stop
    return pred, rec


def run_case(name, base, n_pairs, M, N, width, seed0, subset, tries=20):
    t0 = time.time()
    D = base["input_dim"]
    for seed in range(seed0, seed0 + tries):
        conf = dict(base, n_layers=L, filter_threshold=0.0)
        w = head_weights(synthetic.make_weights(conf, seed=seed), L, HEAD_SCALE, [])
        pair_seeds, fracs, pairs = _pairs(n_pairs, M, N, D, seed)
        bias, ratios, match = _calibrate(conf, w, pairs)
        bias = np.array([bias[i] for i in range(L - 1)], np.float32)
        w = head_weights(w, L, 1.0, bias)
        # with pruning as well: layer 0's median matchability, so about a quarter of the points go per layer (the
        # other low-matchability half is exempt as low-confidence)
        wc = round(1.0 - float(match[0].median()), 6) if width else -1
        for dc in _depth_candidates(ratios, M + N)[:8]:
            conf = dict(base, n_layers=L, filter_threshold=0.0, depth_confidence=dc, width_confidence=wc)
            model = _model(conf, w).eval()
            runs = [_run_pair(model, p, conf) for p in pairs]
            recs = [r for _, r in runs]
            stops = [r["stop"] for r in recs]
            kept0 = [int(p["log_assignment"].shape[1] - 1) for p, _ in runs]
            ok = min(r["ratio_margin"] for r in recs) >= RATIO_TOKENS
            ok &= not width or min(r["sig_margin"] for r in recs) > SIG_MARGIN
            ok &= len(set(stops)) >= 2 and min(stops) < L - 1
            if width:
                ok &= len(set(kept0)) >= 2 and min(kept0) > 0 and sum(s > 0 for s in stops) >= min(2, n_pairs - 1)
            else:
                ok &= len(set(stops)) < len(stops)  # two pairs share a stop layer: one batched head
            if ok:
                break
        else:
            continue
        break
    else:
        raise RuntimeError(f"{name}: no seed whose decisions all clear their thresholds")
    out = {"meta|conf": np.array(repr(conf)), "meta|seed": np.array(seed), "meta|M": np.array(M),
           "meta|N": np.array(N), "meta|pairs": np.array(n_pairs), "meta|pair_seeds": np.array(pair_seeds),
           "meta|fracs": np.array(fracs), "meta|token_bias": bias,
           "meta|head_scale": np.array(HEAD_SCALE),
           "meta|min_ratio_margin_tokens": np.array(min(r["ratio_margin"] for r in recs)),
           "meta|min_sig_margin": np.array(min(r["sig_margin"] for r in recs))}
    for j, (pred, rec) in enumerate(runs):
        p = f"p{j}|"
        out[p + "stop_layer"] = np.array(rec["stop"])
        out[p + "low"] = np.array(rec["low"] + [-1] * (L - 1 - len(rec["low"])))
        for k in ["matches0", "matches1", "matching_scores0", "matching_scores1", "prune0", "prune1"]:
            out[p + k] = pred[k].numpy()
        la = pred["log_assignment"]
        if subset:
            m, n = la.shape[1] - 1, la.shape[2] - 1
            rs = np.random.RandomState(seed + j)
            rows = np.sort(rs.choice(m, size=min(m, 96), replace=False))
            cols = np.sort(rs.choice(n, size=min(n, 96), replace=False))
            out[p + "la_shape"] = np.array(la.shape)
            out[p + "la_rows"], out[p + "la_cols"] = rows, cols
            out[p + "la_sub"] = la[0][np.ix_(rows, cols)].numpy()
            out[p + "la_dust_row"] = la[0, m].numpy()
            out[p + "la_dust_col"] = la[0, :, n].numpy()
            out[p + "la_row_lse"] = torch.logsumexp(la[0, :m].double(), -1).numpy()
        else:
            out[p + "log_assignment"] = la.numpy()
    path = os.path.join(make_golden.OUT, name + ".npz")
    np.savez_compressed(path, **out)
    kept = [(int((r["prune0"] == r["prune0"].max()).sum()), int((r["prune1"] == r["prune1"].max()).sum()))
            if width else (M, N) for r in (p for p, _ in runs)]
    print(f"{name}: seed={seed} depth_confidence={conf['depth_confidence']} width_confidence={wc} "
          f"stop layers={[r['stop'] for r in recs]} kept={kept} "
          f"min ratio margin={out['meta|min_ratio_margin_tokens']:.2f} tokens "
          f"min sigmoid margin={float(out['meta|min_sig_margin']):.2e} -> {path} "
          f"({os.path.getsize(path) / 1e6:.2f} MB, {time.time() - t0:.0f} s)")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    only = sys.argv[1:]
    for name, args in CASES.items():
        if not only or name in only:
            run_case(name, *args)
