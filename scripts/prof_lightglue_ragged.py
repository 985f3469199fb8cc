"""Eval-mode LightGlue on pairs with their own keypoint counts, on one GPU: NP pairs (default 32) whose images keep
between 1024 and 2048 points each, matched one call per pair (each pair's own truncated inputs) against one ragged call
of all NP pairs (`num_keypoints0/1`, padded to 2048), and the assignment head alone: the packed varlen head
(ops.assign_varlen, one launch per kernel for all pairs) against a per-pair loop over ops.assign_stats +
ops.filter_matches at the same per-pair sizes.

    python scripts/prof_lightglue_ragged.py [--out FILE]     # prints the results; --out also writes them to FILE

The benchmark's model shape (256 channels, 4 heads, 9 layers, bf16) with synthetic weights and pairs
(gluefactory_b200.synthetic; planted-match fractions spread over 0.1-0.8), two ways:
  off       adaptive depth / width off;
  adaptive  depth_confidence 0.95 / width_confidence 0.99, with the token-confidence biases calibrated the way
            tests/test_gpu_lightglue_adaptive_batch.py's _calibrate_confidence does (on a schedule for 9 layers) and
            the matchability biases shifted, so that pairs stop and prune differently (calibrate_confidence below).
The per-pair head sizes are the points each pair has left at its stop layer in that mode.  The ways of calling
alternate, ROUNDS rounds (default 7); each round times REPS passes (default 4) over all NP pairs with a host clock
ending in a device synchronise; the heads alone are timed with CUDA events over HEAD_REPS passes (default 20).  Medians
and ranges over the rounds, per pass.  The card's name, power limit, maximum SM clock and the SM clock sampled right
after each timed window are read in the same run.
"""
import argparse
import math
import os
import statistics
import subprocess
import sys
import time

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gluefactory_b200 import ops, synthetic  # noqa: E402
from gluefactory_b200.matchers.lightglue import LightGlue  # noqa: E402
from tests.test_gpu_lightglue_adaptive_batch import _token_stats  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", help="also write the results to this file")
args = ap.parse_args()
NP, NMAX = int(os.environ.get("NP", "32")), 2048
ROUNDS = int(os.environ.get("ROUNDS", "7"))
REPS = int(os.environ.get("REPS", "4"))
HEAD_REPS = int(os.environ.get("HEAD_REPS", "20"))
KEYS = ("keypoints0", "keypoints1", "descriptors0", "descriptors1")


def smi(q):
    r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return [s.strip() for s in r.stdout.strip().split(",")]


def make_pairs():
    g = torch.Generator().manual_seed(17)
    counts = torch.randint(1024, NMAX + 1, (NP, 2), generator=g).tolist()
    fracs = torch.linspace(0.1, 0.8, NP).tolist()
    pairs = []
    for i, ((m, n), f) in enumerate(zip(counts, fracs)):
        p = synthetic.make_pairs(1, n, seed=900 + i, M=m, frac=f)
        pairs.append({k: p[k] for k in KEYS} | {"view0": {"image_size": p["view0"]["image_size"]},
                                                "view1": {"image_size": p["view1"]["image_size"]}})
    return pairs, counts


def calibrate_confidence(w, pre, thr, match):
    """Token-confidence biases as tests/test_gpu_lightglue_adaptive_batch.py's _calibrate_confidence sets them, on a
    schedule that suits 0.95 / 0.99 over 9 layers: about 86, 88, 90, ... % of the points are confident after layer 0,
    1, 2, ..., so the share crosses depth_confidence 0.95 around layer 4 and each pair crosses it at its own layer;
    and matchability biases under which a fifth of the points score at most 1 - width_confidence = 0.01 (synthetic
    weights alone leave every point below its confidence threshold and above 0.01)."""
    w = dict(w)
    for i, a in enumerate(pre):
        t = float(thr[i])
        w[f"token_confidence.{i}.token.0.bias"] = torch.tensor([math.log(t / (1 - t)) -
                                                               float(a.float().quantile(max(0.14 - 0.02 * i, 0.0)))])
        q = float(match[i].float().quantile(0.2))
        key = f"log_assignment.{i}.matchability.bias"
        w[key] = w[key] - math.log(q / (1 - q)) + math.log(0.01 / 0.99)
    return w


def ragged_batch(pairs, dev):
    d = {}
    for k, L in zip(KEYS, (NMAX, NMAX, NMAX, NMAX)):
        t = torch.zeros(len(pairs), L, pairs[0][k].shape[-1])
        for b, p in enumerate(pairs):
            t[b, :p[k].shape[1]] = p[k][0]
        d[k] = t
    for j in (0, 1):
        d[f"view{j}"] = {"image_size": torch.cat([p[f"view{j}"]["image_size"] for p in pairs])}
        d[f"num_keypoints{j}"] = torch.tensor([p[f"keypoints{j}"].shape[1] for p in pairs])
    return synthetic.to_device(d, dev)


def head_timings(sizes, dev):
    """(packed ms, per-pair loop ms) for heads of the given (m, n) per pair, random similarities."""
    g = torch.Generator(device=dev).manual_seed(3)
    G, Mg, Ng = len(sizes), max(m for m, _ in sizes), max(n for _, n in sizes)
    sim = torch.randn(G, Mg, Ng, device=dev, generator=g) * 3
    z0, z1 = torch.randn(G, Mg, device=dev, generator=g), torch.randn(G, Ng, device=dev, generator=g)
    ls0, ls1, du0, du1 = F.logsigmoid(z0), F.logsigmoid(z1), F.logsigmoid(-z0), F.logsigmoid(-z1)
    pairs = torch.tensor([[m for m, _ in sizes], [n for _, n in sizes], list(range(G))], dtype=torch.int32, device=dev)
    ind0 = torch.arange(Mg, device=dev, dtype=torch.int32).repeat(G, 1)
    ind1 = torch.arange(Ng, device=dev, dtype=torch.int32).repeat(G, 1)
    per = [(sim[k, :m, :n].contiguous()[None], ls0[k:k + 1, :m], ls1[k:k + 1, :n], du0[k:k + 1, :m], du1[k:k + 1, :n])
           for k, (m, n) in enumerate(sizes)]

    def packed():
        out = {"scores": torch.full((G, Mg + 1, Ng + 1), -float("inf"), device=dev),
               "m0": torch.full((G, Mg), -1, device=dev, dtype=torch.int64),
               "m1": torch.full((G, Ng), -1, device=dev, dtype=torch.int64),
               "ms0": torch.zeros(G, Mg, device=dev), "ms1": torch.zeros(G, Ng, device=dev)}
        ops.assign_varlen(sim, ls0, ls1, du0, du1, pairs, ind0, ind1, 0.0, out)

    def loop():
        for s, a, b, c, d in per:
            st = ops.assign_stats(s, a, b, c, d, dense=True)
            ops.filter_matches(st["rowmax"], st["rowarg"], st["colarg"], 0.0)

    res = {}
    for name, fn in (("packed", packed), ("loop", loop)):
        fn()
    for r in range(ROUNDS):
        for name, fn in ((("packed", packed), ("loop", loop)) if r % 2 == 0 else (("loop", loop), ("packed", packed))):
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            s.record()
            for _ in range(HEAD_REPS):
                fn()
            e.record()
            torch.cuda.synchronize()
            res.setdefault(name, []).append(s.elapsed_time(e) / HEAD_REPS)
    return res


def main():
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    dev = torch.device("cuda")
    pairs, counts = make_pairs()
    base = dict(synthetic.DEFAULT_CONF, n_layers=9)
    w0 = synthetic.make_weights(base, seed=5)
    lines = []
    clocks = []
    for mode in ("off", "adaptive"):
        conf, w = dict(base), w0
        if mode == "adaptive":
            conf = dict(base, depth_confidence=0.95, width_confidence=0.99)
            _, match, pre, thr = _token_stats(base, w0, "bf16", pairs)
            w = calibrate_confidence(w0, pre, thr, match)
        model = LightGlue(dict(conf, precision="bf16"))
        model.load_state_dict({k: v.float() for k, v in w.items()}, strict=False)
        model = model.to(dev).eval()
        singles = [synthetic.to_device(p, dev) for p in pairs]
        ragged = ragged_batch(pairs, dev)

        def run_single():
            with torch.no_grad():
                return [model(d) for d in singles]

        def run_ragged():
            with torch.no_grad():
                return model(ragged)

        run_single(), run_ragged()  # warm-up: module loads, allocator, every shape the timed windows use
        pr = run_ragged()
        torch.cuda.synchronize()
        la = pr["log_assignment"]
        sizes = [(int(torch.isfinite(la[b, :NMAX, NMAX]).sum()), int(torch.isfinite(la[b, NMAX, :NMAX]).sum()))
                 for b in range(NP)]
        stops = pr["stop_layer"].tolist()
        times = {"one call per pair": [], f"one ragged call of {NP}": []}
        for r in range(ROUNDS):
            ways = list(zip(times, (run_single, run_ragged)))
            for name, fn in (ways if r % 2 == 0 else ways[::-1]):
                torch.cuda.synchronize()
                t = time.perf_counter()
                for _ in range(REPS):
                    fn()
                torch.cuda.synchronize()
                times[name].append((time.perf_counter() - t) / REPS)
                clocks.append(smi("clocks.sm")[0])
        heads = head_timings(sizes, dev)
        lines += [f"## {mode}" + (" (depth_confidence 0.95, width_confidence 0.99, calibrated token biases)"
                                  if mode == "adaptive" else " (adaptive depth / width off)"),
                  f"stop layers: {stops}",
                  f"points left at the stop layer (m, n): {sizes}",
                  "| way | time for all pairs (median of the rounds, ms) | range (ms) | pairs/s |",
                  "|---|---|---|---|"]
        for name, ts in times.items():
            med = statistics.median(ts)
            lines.append(f"| {name} | {med * 1e3:.1f} | {min(ts) * 1e3:.1f}-{max(ts) * 1e3:.1f} | {NP / med:.1f} |")
        one, rag = (statistics.median(v) for v in times.values())
        lines += [f"ragged / one call per pair: {one / rag:.2f}x", "",
                  "| assignment head alone | median (ms) | range (ms) |", "|---|---|---|"]
        for name, ts in heads.items():
            label = "packed varlen head, one pass" if name == "packed" else "per-pair assign_stats + filter_matches"
            lines.append(f"| {label} | {statistics.median(ts):.3f} | {min(ts):.3f}-{max(ts):.3f} |")
        lines += [f"packed head / per-pair loop: {statistics.median(heads['loop']) / statistics.median(heads['packed']):.2f}x",
                  ""]
        del model, singles, ragged, pr
        torch.cuda.empty_cache()
    name, power, maxclk = smi("name,power.limit,clocks.max.sm")
    head = [f"card: {name}, power limit {power}, max SM clock {maxclk}; SM clock after the timed windows: "
            f"{', '.join(sorted(set(clocks)))}",
            f"{NP} pairs, per-image counts drawn from [1024, {NMAX}] (padded to {NMAX}): {counts}",
            f"9 layers, 256 channels / 4 heads, bf16, {ROUNDS} alternating rounds of {REPS} passes "
            f"(heads: {HEAD_REPS} passes per round)", ""]
    text = "\n".join(head + lines)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
