"""LightGlue at head dimension 32 (descriptor_dim 128 / 4 heads, 256 / 8 heads) against the benchmark's 256 / 4 heads on
one GPU.

    python scripts/prof_lightglue_hd32.py [--out FILE]     # prints the results; --out also writes them to FILE

1. The bf16 training step at the benchmark shape: PB pairs per step (default 32) of 2048 points per image, 9 layers,
   ground-truth labels on the device (HomographyMatcher), CUDA-graph replay of the whole step (MatcherTrainer).  The
   three configurations run in alternating order, ROUNDS rounds (default 3); each round times STEPS replays with CUDA
   events.  Medians and ranges over the rounds; the SM clock is sampled right after each timed window.
2. Per kernel, with CUDA events over many launches at the benchmark's token count T = 2 PB 2048:
   - the rotary split forward and backward at head dims 32 and 64 against the HBM bound (3.35 TB/s, data sheet).
     Algorithmic bytes: forward 2 T 3 D 2 (qkv in, q / k / v out, bf16) + T hd/2 4 (theta); backward (3 + 2 + 3) T D 2
     (dq, dk, dv, q, k in, dqkv out) + 3 T hd/2 4 (theta in, dtheta read and written);
   - the self-attention forward and backward of each configuration (2 PB sequences of 2048 tokens);
   - the cross-attention backward as the layer runs it: at head dim 32 both directions into separate dq / dk buffers
     and one add; at head dim 64 the one-sweep shared-qk kernel, and for comparison the same two-direction path.
The card's name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gluefactory_b200 import engine, ops, synthetic  # noqa: E402
from gluefactory_b200.matchers.homography_matcher import HomographyMatcher  # noqa: E402
from gluefactory_b200.matchers.lightglue import LightGlue  # noqa: E402
from gluefactory_b200.trainer import MatcherTrainer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", help="also write the results to this file")
args = ap.parse_args()
B, N = int(os.environ.get("PB", "32")), 2048
ROUNDS = int(os.environ.get("ROUNDS", "3"))
STEPS = int(os.environ.get("STEPS", "10"))
CONFIGS = [(128, 4), (256, 8), (256, 4)]  # (descriptor_dim, num_heads); the last is the benchmark's
HBM = 3.35e12
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


def step_time(D, H):
    conf = dict(synthetic.DEFAULT_CONF, descriptor_dim=D, input_dim=D, num_heads=H, precision="bf16")
    model = LightGlue(conf)
    model.load_state_dict(synthetic.make_weights(conf, seed=0), strict=False)
    tr = MatcherTrainer(model.to(dev), lr=1e-4, ground_truth=HomographyMatcher(
        {"th_positive": 3.0, "th_negative": 3.0, "transposed_assignment": True}))
    pool = [synthetic.to_device(synthetic.make_pairs(B, N, seed=1234 + i, D=D, with_gt=False), dev) for i in range(2)]
    tr.step(pool[0])
    tr.capture(pool[0], dev, warmup=2)
    for i in range(3):
        tr.step_graphed(pool[i % 2])
    it = iter(range(10 ** 9))
    ms = events(lambda: tr.step_graphed(pool[next(it) % 2]), STEPS)
    clk = smi("clocks.sm")[0]
    del tr, model, pool
    torch.cuda.empty_cache()
    return ms, clk


def med(xs):
    xs = sorted(xs)
    return xs[len(xs) // 2], xs[0], xs[-1]


name, power, maxclk = smi("name,power.limit,clocks.max.sm")
out(f"GPU: {name}, power limit {power}, max SM clock {maxclk}")
out(f"LightGlue bf16 training step, {B} pairs x {N} points per image, 9 layers, device ground truth, CUDA-graph replay, "
    f"{STEPS} replays per window, {ROUNDS} alternating rounds")
res = {c: [] for c in CONFIGS}
for r in range(ROUNDS):
    order = CONFIGS if r % 2 == 0 else CONFIGS[::-1]
    for D, H in order:
        ms, clk = step_time(D, H)
        res[(D, H)].append(ms)
        out(f"  round {r} D={D} H={H} (hd {D // H}): {ms:.2f} ms/step, SM clock after the window {clk}")
base = med(res[(256, 4)])[0]
out("| descriptor_dim / heads | head dim | ms/step median (range) | pairs/s | vs 256 / 4 |")
out("|---|---|---|---|---|")
for D, H in CONFIGS:
    m, lo, hi = med(res[(D, H)])
    out(f"| {D} / {H} | {D // H} | {m:.2f} ({lo:.2f}-{hi:.2f}) | {B / m * 1e3:.1f} | {base / m:.2f}x |")

# ---- kernels
T = 2 * B * N
REPS = 50
g = torch.Generator(device=dev).manual_seed(0)
out(f"\nRotary split, T = {T} tokens, bf16, {REPS} launches per timing")
out("| D / heads | head dim | call | ms | algorithmic MB | GB/s | HBM bound ms | share of HBM bound |")
out("|---|---|---|---|---|---|---|---|")
for D, H in CONFIGS:
    hd = D // H
    qkv = torch.randn(T, 3 * D, device=dev, generator=g).to(torch.bfloat16)
    theta = torch.randn(T, hd // 2, device=dev, generator=g)
    q, k, v = ops.rope_fwd(qkv, theta, H)
    dq, dk, dv = (torch.randn(T, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(3))
    dtheta = torch.zeros_like(theta)
    ops.rope_bwd(dq, dk, dv, q, k, theta, H, dtheta=dtheta)
    f = events(lambda: ops.rope_fwd(qkv, theta, H), REPS)
    b = events(lambda: ops.rope_bwd(dq, dk, dv, q, k, theta, H, dtheta=dtheta), REPS)
    for tag, ms, nbytes in (("fwd", f, 2 * T * 3 * D * 2 + T * (hd // 2) * 4),
                            ("bwd", b, 8 * T * D * 2 + 3 * T * (hd // 2) * 4)):
        t_hbm = nbytes / HBM * 1e3
        out(f"| {D} / {H} | {hd} | {tag} | {ms:.4f} | {nbytes / 1e6:.1f} | {nbytes / ms / 1e6:.0f} | {t_hbm:.4f} | "
            f"{100 * t_hbm / ms:.0f}% |")
    del qkv, theta, q, k, v, dq, dk, dv, dtheta

out(f"\nAttention, bf16, {2 * B} sequences x {N} tokens (self: each image attends to itself; cross: image 0 <-> 1), "
    f"{REPS // 5} launches per timing")
out("| D / heads | head dim | self fwd ms | self bwd ms | cross bwd as run ms | cross bwd two-direction ms |")
out("|---|---|---|---|---|---|")
sizes = (B, N, N)
for D, H in CONFIGS:
    hd = D // H
    q, k, v, do = (torch.randn(T, D, device=dev, generator=g).to(torch.bfloat16) for _ in range(4))
    o, lse = engine._attend_fwd(q, k, v, sizes, H, cross=False)
    oc, lsec = engine._attend_fwd(q, q, v, sizes, H, cross=True)
    r = REPS // 5
    sf = events(lambda: engine._attend_fwd(q, k, v, sizes, H, cross=False), r)
    sb = events(lambda: engine._attend_bwd(q, k, v, o, lse, do, sizes, H, cross=False), r)
    cb = events(lambda: engine._attend_bwd_shared_qk(q, v, oc, lsec, do, sizes, H), r)

    def two_dir():
        dq, dk, dv = engine._attend_bwd(q, q, v, oc, lsec, do, sizes, H, cross=True)
        dq.add_(dk)
    c2 = events(two_dir, r)
    out(f"| {D} / {H} | {hd} | {sf:.3f} | {sb:.3f} | {cb:.3f} | {c2:.3f} |")
    del q, k, v, do, o, oc
    torch.cuda.empty_cache()

if args.out:
    with open(args.out, "w") as fh:
        fh.write("\n".join(lines) + "\n")
