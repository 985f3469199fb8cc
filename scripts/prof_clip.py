"""Cost of gradient-norm clipping (MatcherTrainer(clip_grad=...), lgb200_flat_grad_norm) in the graph-replayed
training step at the benchmark's shape: two captured trainers, clipping off and on, timed in alternating rounds with
CUDA events; then the norm kernel against the check it replaces, on the step's flat gradient.  Prints the card's name,
power limit and max SM clock read in the same run.

    python scripts/prof_clip.py [--batch 32] [--rounds 10] [--steps 20]
"""
import argparse
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gluefactory_b200 import ops, synthetic  # noqa: E402
from gluefactory_b200.matchers.homography_matcher import HomographyMatcher  # noqa: E402
from gluefactory_b200.matchers.lightglue import LightGlue  # noqa: E402
from gluefactory_b200.trainer import MatcherTrainer  # noqa: E402


def card(dev):
    q = "name,power.limit,clocks.max.sm"
    out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(dev.index)],
                         capture_output=True, text=True)
    return out.stdout.strip() or torch.cuda.get_device_name(dev)


def trainer(dev, clip_grad, example):
    conf = dict(synthetic.DEFAULT_CONF, precision="bf16")
    model = LightGlue(conf)
    model.load_state_dict(synthetic.make_weights(conf, seed=0), strict=False)
    gt = HomographyMatcher({"th_positive": 3.0, "th_negative": 3.0, "transposed_assignment": True})
    return MatcherTrainer(model.to(dev), lr=1e-4, ground_truth=gt, clip_grad=clip_grad).capture(example, dev, warmup=2)


def timed(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / reps  # ms per call


def spread(xs):
    xs = sorted(xs)
    return f"median {statistics.median(xs):.3f}, min {xs[0]:.3f}, max {xs[-1]:.3f}"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32, help="pairs per step (the benchmark's default)")
    ap.add_argument("--kpts", type=int, default=2048)
    ap.add_argument("--clip", type=float, default=10.0, help="max_norm (the GlueStick homography config's clip_grad)")
    ap.add_argument("--rounds", type=int, default=10)
    ap.add_argument("--steps", type=int, default=20, help="graph replays per arm and round")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    print("card:", card(dev))
    batches = [synthetic.to_device(synthetic.make_pairs(args.batch, args.kpts, seed=1234 + i, with_gt=False), dev)
               for i in range(2)]
    arms = {"off": trainer(dev, None, batches[0]), "on": trainer(dev, args.clip, batches[0])}
    print(f"B={args.batch} pairs x {args.kpts} keypoints, 9 layers, bf16; peak memory "
          f"{torch.cuda.max_memory_allocated(dev) / 2**30:.1f} GiB for both captured steps")
    it = {k: 0 for k in arms}

    def step(k):
        arms[k].step_graphed(batches[it[k] % 2])
        it[k] += 1

    for k in arms:  # warm replays
        for _ in range(3):
            step(k)
    ms = {k: [] for k in arms}
    for r in range(args.rounds):
        for k in (("off", "on") if r % 2 == 0 else ("on", "off")):
            ms[k].append(timed(lambda: step(k), args.steps))
    diff_us = [1e3 * (a - b) for a, b in zip(ms["on"], ms["off"])]
    print(f"step, clipping off (ms): {spread(ms['off'])}")
    print(f"step, clipping on  (ms): {spread(ms['on'])}")
    print(f"on - off per round (us): {spread(diff_us)}")
    print(f"clip_grad={args.clip}: last step's gradient norm {arms['on']._grad_norm.item():.4g}, "
          f"{arms['on'].t} updates applied")

    # the kernels alone on the step's flat gradient (+ its loss slot), alternating
    tr = arms["on"]
    g = tr.fp.grad_ext[:tr.fp.numel + 4]
    found, norm, div = (torch.zeros(1, device=dev) for _ in range(3))
    ws = ops.flat_grad_norm_ws(tr.fp.numel, dev)
    calls = {"flat_grad_check": lambda: ops.flat_grad_check(g, found),
             "flat_grad_norm": lambda: ops.flat_grad_norm(g, tr.fp.numel, 1.0, None, args.clip, found, norm, div, ws)}
    us = {k: [] for k in calls}
    for r in range(args.rounds):
        for k, fn in (calls.items() if r % 2 == 0 else reversed(calls.items())):
            us[k].append(1e3 * timed(fn, 200))
    mb = g.numel() * 4 / 1e6
    for k in calls:
        print(f"{k} over {mb:.1f} MB (us/call, back to back): {spread(us[k])}; "
              f"{mb / 1e3 / (statistics.median(us[k]) * 1e-6):.0f} GB/s at the median")


if __name__ == "__main__":
    main()
