"""Eval-mode LightGlue with adaptive depth and width (depth_confidence 0.95, width_confidence 0.99) on one GPU: pairs per
second when NP pairs (default 32) of N = 2048 points per image are matched one call per pair (B = 1 in a loop) against
B = 8 and B = 32 pairs per call.

    python scripts/prof_lightglue_adaptive_batch.py [--out FILE]     # prints the results; --out also writes them to FILE

The benchmark's model shape (256 channels, 4 heads, 9 layers, bf16) with synthetic weights and pairs
(gluefactory_b200.synthetic; planted-match fractions spread over 0.1-0.8).  With synthetic weights the stop layers and
pruning are whatever the token heads give; they are printed with the timings.  The three ways of calling alternate,
ROUNDS rounds (default 7); each round times REPS passes (default 6) over all NP pairs with a host clock ending in a
device synchronise, so that every timed window lasts a quarter of a second or more.  Medians and ranges over the
rounds, per pass.  The card's name, power limit, maximum SM clock and the SM clock sampled right after each timed
window are read in the same run.
"""
import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gluefactory_b200 import synthetic  # noqa: E402
from gluefactory_b200.matchers.lightglue import LightGlue  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", help="also write the results to this file")
args = ap.parse_args()
NP, N = int(os.environ.get("NP", "32")), 2048
ROUNDS = int(os.environ.get("ROUNDS", "7"))
REPS = int(os.environ.get("REPS", "6"))
BATCHES = [1, 8, 32]


def smi(q):
    r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return [s.strip() for s in r.stdout.strip().split(",")]


def main():
    assert torch.cuda.is_available(), "this measurement needs the GPU"
    dev = torch.device("cuda")
    conf = dict(synthetic.DEFAULT_CONF, n_layers=9, depth_confidence=0.95, width_confidence=0.99)
    model = LightGlue(dict(conf, precision="bf16"))
    model.load_state_dict({k: v.float() for k, v in synthetic.make_weights(conf, seed=5).items()}, strict=False)
    model = model.to(dev).eval()
    fracs = torch.linspace(0.1, 0.8, NP).tolist()
    pairs = [synthetic.make_pairs(1, N, seed=900 + i, frac=f) for i, f in enumerate(fracs)]
    keys = ("keypoints0", "keypoints1", "descriptors0", "descriptors1")

    def batch(lo, hi):
        d = {k: torch.cat([p[k] for p in pairs[lo:hi]]) for k in keys}
        d["view0"] = {"image_size": torch.cat([p["view0"]["image_size"] for p in pairs[lo:hi]])}
        d["view1"] = {"image_size": torch.cat([p["view1"]["image_size"] for p in pairs[lo:hi]])}
        return synthetic.to_device(d, dev)

    inputs = {B: [batch(i, i + B) for i in range(0, NP, B)] for B in BATCHES}

    def run(B):
        with torch.no_grad():
            return [model(d) for d in inputs[B]]

    for B in BATCHES:  # warm-up: module loads, allocator, every shape the timed window uses
        run(B)
    torch.cuda.synchronize()
    stops = [p["stop_layer"] for p in run(1)]
    kept0 = [int((p["prune0"] == p["prune0"].max()).sum()) for p in run(1)]
    times = {B: [] for B in BATCHES}
    clocks = []
    for r in range(ROUNDS):
        for B in (BATCHES if r % 2 == 0 else BATCHES[::-1]):
            torch.cuda.synchronize()
            t = time.perf_counter()
            for _ in range(REPS):
                run(B)
            torch.cuda.synchronize()
            times[B].append((time.perf_counter() - t) / REPS)
            clocks.append(smi("clocks.sm")[0])
    name, power, maxclk = smi("name,power.limit,clocks.max.sm")
    lines = [f"card: {name}, power limit {power}, max SM clock {maxclk}; SM clock after the timed windows: "
             f"{', '.join(sorted(set(clocks)))}",
             f"{NP} pairs of {N} + {N} points, 9 layers, 256 channels / 4 heads, bf16, depth_confidence 0.95, "
             f"width_confidence 0.99, {ROUNDS} rounds of {REPS} passes",
             f"stop layers (one-pair calls): {stops}",
             f"points of image 0 left at the end (one-pair calls): {kept0}",
             "| pairs per call | calls | time for all pairs (median of the rounds, ms) | range (ms) | pairs/s | vs B = 1 |",
             "|---|---|---|---|---|---|"]
    base = statistics.median(times[1])
    for B in BATCHES:
        med = statistics.median(times[B])
        lines.append(f"| {B} | {NP // B} | {med * 1e3:.1f} | {min(times[B]) * 1e3:.1f}-{max(times[B]) * 1e3:.1f} | "
                     f"{NP / med:.1f} | {base / med:.2f}x |")
    text = "\n".join(lines)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text + "\n")


if __name__ == "__main__":
    main()
