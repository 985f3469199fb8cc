"""LightGlue's graph-replayed bf16 training step with device ground truth, dense labels (the [B, M, N] mask and its
transpose) against match lists (`dense_assignment: False`), in alternating rounds.  Prints one JSON line per shape
with the card, its power limit and max SM clock, the median step time of each arm and each arm's peak memory.

    python scripts/prof_sparse_labels.py [--shapes 32x2048,8x4096] [--steps 20] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gluefactory_b200 import synthetic  # noqa: E402
from gluefactory_b200.matchers.homography_matcher import HomographyMatcher  # noqa: E402
from gluefactory_b200.matchers.lightglue import LightGlue  # noqa: E402
from gluefactory_b200.trainer import MatcherTrainer  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def arm(B, N, dense, steps):
    conf = dict(synthetic.DEFAULT_CONF, precision="bf16")
    model = LightGlue(conf)
    model.load_state_dict(synthetic.make_weights(conf, seed=5), strict=False)
    model = model.cuda().train()
    data = {k: v for k, v in synthetic.to_device(synthetic.make_pairs(B, N, seed=6, with_gt=False), "cuda").items()}
    gt = HomographyMatcher({"dense_assignment": dense, "transposed_assignment": dense})
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    tr = MatcherTrainer(model, lr=1e-5, ground_truth=gt)
    tr.step(data)
    tr.capture(data, torch.device("cuda"), warmup=0)
    tr.step_graphed(data)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base

    def timed():
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        for _ in range(steps):
            tr.step_graphed(data)
        e.record()
        e.synchronize()
        return s.elapsed_time(e) / steps
    return tr, timed, peak


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="32x2048,8x4096")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    name = card()
    for shp in a.shapes.split(","):
        B, N = (int(v) for v in shp.split("x"))
        arms = {k: arm(B, N, k == "dense", a.steps) for k in ("dense", "lists")}
        times = {k: [] for k in arms}
        for _ in range(a.rounds):
            for k, (_, timed, _) in arms.items():
                times[k].append(timed())
        med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
        print(json.dumps({"card": name, "B": B, "M": N, "N": N, "steps": a.steps, "rounds": a.rounds,
                          "dense_ms": round(med["dense"], 3), "lists_ms": round(med["lists"], 3),
                          "speedup": round(med["dense"] / med["lists"], 4),
                          "dense_peak_GiB": round(arms["dense"][2] / 2 ** 30, 3),
                          "lists_peak_GiB": round(arms["lists"][2] / 2 ** 30, 3),
                          "mask_bytes": B * N * N, "all_ms": times}), flush=True)
        del arms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
