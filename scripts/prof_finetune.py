"""Optimiser choice and fine-tuning on the flat-buffer trainer, on one GPU.

    python scripts/prof_finetune.py [--out FILE]     # prints the results; --out also writes them to FILE

1. The bf16 LightGlue training step at the benchmark shape: PB pairs per step (default 32) of 2048 points per image,
   9 layers, ground-truth labels on the device (HomographyMatcher), CUDA-graph replay of the whole step (MatcherTrainer).
   Arms: full training with Adam (the benchmark's), AdamW, SGD with momentum 0.9 and centered RMSprop with momentum 0.9;
   Adam fine-tuning of the heads only (opt_regexp `log_assignment|token_confidence`) and of the last four layers and
   the heads (`transformers\\.[5-8]\\.|log_assignment|token_confidence`).  The arms run in alternating order, ROUNDS
   rounds (default 3); each round times STEPS replays with CUDA events.  Medians and ranges over the rounds; the SM
   clock is sampled right after each timed window.
2. Each optimiser kernel over the full model's flat buffers (n trainable elements, no LR groups), CUDA events over
   REPS launches, against the HBM bound (3.35 TB/s, data sheet).  Algorithmic bytes: 4 n times the fp32 words read plus
   written per element: Adam / AdamW 7, SGD with momentum 5, centered RMSprop with momentum 9.
The card's name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gluefactory_b200 import ops, synthetic  # noqa: E402
from gluefactory_b200.matchers.homography_matcher import HomographyMatcher  # noqa: E402
from gluefactory_b200.matchers.lightglue import LightGlue  # noqa: E402
from gluefactory_b200.trainer import MatcherTrainer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", help="also write the results to this file")
args = ap.parse_args()
B, N = int(os.environ.get("PB", "32")), 2048
ROUNDS = int(os.environ.get("ROUNDS", "3"))
STEPS = int(os.environ.get("STEPS", "10"))
REPS = 50
HBM = 3.35e12
ARMS = {
    "adam": dict(),
    "adamw": dict(optimizer="adamw"),
    "sgd momentum": dict(optimizer="sgd", optimizer_options={"momentum": 0.9}),
    "rmsprop centered momentum": dict(optimizer="rmsprop", optimizer_options={"momentum": 0.9, "centered": True}),
    "adam, heads only": dict(opt_regexp=r"log_assignment|token_confidence"),
    "adam, last 4 layers + heads": dict(opt_regexp=r"transformers\.[5-8]\.|log_assignment|token_confidence"),
}
dev = torch.device("cuda", 0)
lines = []


def out(s=""):
    print(s, flush=True)
    lines.append(s)


def smi(q):
    r = subprocess.run(["nvidia-smi", "-i", "0", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return [x.strip() for x in r.stdout.splitlines()[0].split(",")]


def events(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def trainer(**kw):
    conf = dict(synthetic.DEFAULT_CONF, precision="bf16")
    model = LightGlue(conf)
    model.load_state_dict(synthetic.make_weights(conf, seed=0), strict=False)
    return MatcherTrainer(model.to(dev), lr=1e-4, ground_truth=HomographyMatcher(
        {"th_positive": 3.0, "th_negative": 3.0, "transposed_assignment": True}), **kw)


def step_time(kw):
    tr = trainer(**kw)
    pool = [synthetic.to_device(synthetic.make_pairs(B, N, seed=1234 + i, with_gt=False), dev) for i in range(2)]
    tr.step(pool[0])
    tr.capture(pool[0], dev, warmup=2)
    for i in range(3):
        tr.step_graphed(pool[i % 2])
    it = iter(range(10 ** 9))
    ms = events(lambda: tr.step_graphed(pool[next(it) % 2]), STEPS)
    clk = smi("clocks.sm")[0]
    trainable = tr.fp.numel
    del tr, pool
    torch.cuda.empty_cache()
    return ms, clk, trainable


def med(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2], xs[0], xs[-1]


name, power, maxclk = smi("name,power.limit,clocks.max.sm")
out(f"GPU: {name}, power limit {power}, max SM clock {maxclk}")
out(f"LightGlue bf16 training step, {B} pairs x {N} points per image, 9 layers, device ground truth, CUDA-graph replay, "
    f"{STEPS} replays per window, {ROUNDS} alternating rounds")
res, sizes = {a: [] for a in ARMS}, {}
for r in range(ROUNDS):
    order = list(ARMS) if r % 2 == 0 else list(ARMS)[::-1]
    for arm in order:
        ms, clk, sizes[arm] = step_time(ARMS[arm])
        res[arm].append(ms)
        out(f"  round {r} {arm}: {ms:.2f} ms/step, SM clock after the window {clk}")
base = med(res["adam"])[0]
out("| arm | trainable elements | ms/step median (range) | pairs/s | vs full Adam |")
out("|---|---|---|---|---|")
for arm in ARMS:
    m, lo, hi = med(res[arm])
    out(f"| {arm} | {sizes[arm]:,} | {m:.2f} ({lo:.2f}-{hi:.2f}) | {B / m * 1e3:.1f} | {base / m:.3f}x |")

# ---- optimiser kernels over the full model's flat buffers
n = sizes["adam"]
g = torch.Generator(device=dev).manual_seed(0)
p, grad = torch.randn(n, device=dev, generator=g), torch.randn(n, device=dev, generator=g) * 1e-3
s = [torch.zeros(n, device=dev) for _ in range(3)]
step = torch.ones(1, device=dev, dtype=torch.int32)
lr = torch.full((1,), 1e-6, device=dev)
found = torch.zeros(1, device=dev)
dv = dict(lr_dev=lr, found_inf_dev=found)
KERNELS = [
    ("lgb200_adam_flat", 7, lambda: ops.adam_flat_(p, grad, s[0], s[1], 0, 0.0, step_dev=step, **dv)),
    ("lgb200_adamw_flat", 7, lambda: ops.adamw_flat_(p, grad, s[0], s[1], 0, 0.0, step_dev=step, **dv)),
    ("lgb200_sgd_flat (momentum)", 5, lambda: ops.sgd_flat_(p, grad, s[0], 0, 0.0, momentum=0.9, step_dev=step, **dv)),
    ("lgb200_rmsprop_flat (centered, momentum)", 9,
     lambda: ops.rmsprop_flat_(p, grad, s[0], s[1], s[2], 0.0, momentum=0.9, **dv)),
]
out(f"\nOptimiser kernels, n = {n:,} fp32 elements (the full model's trainable range), {REPS} launches per timing")
out("| kernel | words / element | ms | algorithmic MB | GB/s | HBM bound ms | share of HBM bound |")
out("|---|---|---|---|---|---|---|")
for tag, words, fn in KERNELS:
    fn()
    ms = events(fn, REPS)
    nbytes = 4 * words * n
    t_hbm = nbytes / HBM * 1e3
    out(f"| {tag} | {words} | {ms:.4f} | {nbytes / 1e6:.1f} | {nbytes / ms / 1e6:.0f} | {t_hbm:.4f} | "
        f"{100 * t_hbm / ms:.0f}% |")

if args.out:
    with open(args.out, "w") as fh:
        fh.write("\n".join(lines) + "\n")
