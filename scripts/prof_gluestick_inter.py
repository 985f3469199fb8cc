"""Cost of GlueStick's intermediate line supervision on one GPU.

    python scripts/prof_gluestick_inter.py [--out FILE]     # prints the results; --out also writes them to FILE

The bf16 training step (forward + loss + backward + Adam) as a CUDA-graph replay of MatcherTrainer, at the C5 shape:
PB pairs (default 8) of 2048 points + 512 lines per image, 18 GNN layers, 256 channels, with `inter_supervision` None
and [2, 5] (configs/superpoint+lsd+gluestick-homography.yaml).  The two are alternated, ROUNDS (default 3) rounds each,
in one process; each round builds the model, captures the step and times REPS (default 20) replays after 3 untimed
ones.  Also the peak device memory of each step.  The card's name, power limit and maximum SM clock are read in the
same run.
"""
import argparse
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gluefactory_b200 import synthetic  # noqa: E402
from gluefactory_b200.matchers.gluestick import GlueStick  # noqa: E402
from gluefactory_b200.trainer import MatcherTrainer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", help="also write the results to this file")
args = ap.parse_args()
B, N, L = int(os.environ.get("PB", "8")), 2048, 512
ROUNDS = int(os.environ.get("ROUNDS", "3"))
REPS = int(os.environ.get("REPS", "20"))
dev = torch.device("cuda", 0)
lines = []


def out(s=""):
    print(s, flush=True)
    lines.append(s)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clk = (x.strip() for x in r.stdout.splitlines()[0].split(","))
    return name, power, clk


def replay_time(inter):
    """ms per graph-replayed step and peak MiB of the captured step."""
    data = synthetic.to_device(synthetic.make_gluestick_batch(B, N, L, 5), dev)
    m = GlueStick(dict(GlueStick.default_conf, inter_supervision=inter))
    m.load_state_dict(synthetic.make_gluestick_weights(m.state_dict(), seed=3), strict=True)
    tr = MatcherTrainer(m.to(dev).train(), lr=1e-5)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    tr.capture(data, dev)
    for _ in range(3):
        tr.step_graphed(data)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(REPS):
        tr.step_graphed(data)
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) / REPS * 1e3
    peak = torch.cuda.max_memory_allocated(dev) / 2**20
    del tr, m, data
    torch.cuda.empty_cache()
    return ms, peak


name, power, clk = gpu_info()
out(f"GPU: {name}, power limit {power}, max SM clock {clk}")
out(f"GlueStick bf16 training step (CUDA-graph replay of MatcherTrainer), {B} pairs, {N} points + {L} lines per image, "
    f"18 GNN layers, D=256; {ROUNDS} alternating rounds of {REPS} replays")
arms = {"None": None, "[2, 5]": [2, 5]}
res = {k: [] for k in arms}
for r in range(ROUNDS):
    for tag, inter in arms.items():
        res[tag].append(replay_time(inter))
        out(f"  round {r} inter_supervision {tag}: {res[tag][-1][0]:.2f} ms/step, peak {res[tag][-1][1]:.0f} MiB")
med = {}
for tag in arms:
    t = sorted(x[0] for x in res[tag])
    med[tag] = t[len(t) // 2]
    out(f"inter_supervision {tag}: median {med[tag]:.2f} ms/step (range {t[0]:.2f}-{t[-1]:.2f}) = "
        f"{B / med[tag] * 1e3:.1f} pairs/s; peak {max(x[1] for x in res[tag]):.0f} MiB")
diffs = sorted(b[0] - a[0] for a, b in zip(res["None"], res["[2, 5]"]))
out(f"two intermediate heads: median {med['[2, 5]'] - med['None']:+.2f} ms/step "
    f"({100 * (med['[2, 5]'] / med['None'] - 1):+.1f} %); per-round differences {diffs[0]:+.2f} to {diffs[-1]:+.2f} ms")

if args.out:
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")
