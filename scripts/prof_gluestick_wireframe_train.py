"""Cost of GlueStick's fixed-order LineLayer and line-head kernels in training, on wireframes with shared junctions.

    python scripts/prof_gluestick_wireframe_train.py [--out FILE]   # prints the results; --out also writes them to FILE

The bf16 training step (forward + loss + backward + Adam) as a CUDA-graph replay of MatcherTrainer at the C5 shape:
PB pairs (default 8) of 2048 points + 512 lines per image, 18 GNN layers, 256 channels, on wireframes whose junctions
each end about 2.5 lines (hubs of 9 and 5, degenerate lines).  Two arms alternate, ROUNDS (default 5) rounds each, in
one process; each round builds the model, captures the step and times REPS (default 20) replays after 3 untimed ones:
  fixed   this tree: ops.JunctionGather / JunctionMean / LineScores (fixed-order kernels in both directions);
  torch   the same model with the LineLayer and line head restated on the torch ops they replace (index_select + flip
          + scatter_reduce(mean); two gathers + maximum), whose backward sums by atomics.
Then one torch.profiler pass of three eager steps per arm: device time per step of the kernels of the junction and
line-score work, by kernel name.  Also whether each arm repeats its loss and parameters bit for bit over two replays
from one saved state.  The card's name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import os
import subprocess
import sys
import time
from collections import defaultdict

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
ROUNDS = int(os.environ.get("ROUNDS", "5"))
REPS = int(os.environ.get("REPS", "20"))
dev = torch.device("cuda", 0)
lines = []


def out(s=""):
    print(s, flush=True)
    lines.append(s)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    return tuple(x.strip() for x in r.stdout.splitlines()[0].split(","))


class TorchLineOps(GlueStick):
    """The LineLayer and line head on torch's gather / scatter ops (atomic backward), on the same layouts."""

    def _line_layer(self, x, enc, lay, layer):
        D = x.shape[1]
        flat = lay.tgt.long()
        ld = x.index_select(0, flat)
        other = ld.view(-1, 2, D).flip(1).reshape(-1, D)
        upd = self._mlp(torch.cat([ld, other, enc], 1), layer.mlp)
        acc = torch.zeros_like(x).scatter_reduce(0, flat[:, None].expand(-1, D), upd.to(x.dtype), reduce="mean",
                                                 include_self=False)
        return x + acc

    def _line_head(self, d0, d1, lay0, lay1, L0, L1, proj, B):
        D = d0.shape[1]
        idx0, idx1 = lay0.junc.long(), lay1.junc.long()
        ld0 = d0.view(B, -1, D)[:, :2 * L0].reshape(-1, D)
        ld1 = d1.view(B, -1, D)[:, :2 * L1].reshape(-1, D)
        s = self._similarity(self._conv(ld0, proj), self._conv(ld1, proj), B)
        n20, n21 = idx0.shape[1], idx1.shape[1]
        s = torch.gather(s, 2, idx1[:, None, :].expand(B, s.shape[1], n21))
        s = torch.gather(s, 1, idx0[:, :, None].expand(B, n20, n21)).reshape(B, n20 // 2, 2, n21 // 2, 2)
        raw = 0.5 * torch.maximum(s[:, :, 0, :, 0] + s[:, :, 1, :, 1], s[:, :, 0, :, 1] + s[:, :, 1, :, 0])
        from gluefactory_b200 import ops

        lscores = ops.log_double_softmax(raw.contiguous(), self.line_bin_score)
        return (lscores, *self._matches(lscores.detach()), raw)


def wireframe_batch(seed=5):
    d = synthetic.make_gluestick_batch(B, N, L, seed)
    gen = torch.Generator().manual_seed(seed)
    for i in "01":
        idx = torch.randint(0, int(2 * L / 2.5), (B, L, 2), generator=gen)
        idx[:, :9, 0] = 3
        idx[:, 9:14, 1] = 7
        idx[:, 14:17, 1] = idx[:, 14:17, 0]
        d[f"lines_junc_idx{i}"] = idx
        kp = d[f"keypoints{i}"]
        d[f"lines{i}"] = torch.stack([kp[b][idx[b].reshape(-1)] for b in range(B)]).view(B, L, 2, 2)
    return synthetic.to_device(d, dev)


def build(cls):
    m = cls(dict(GlueStick.default_conf))
    m.load_state_dict(synthetic.make_gluestick_weights(m.state_dict(), seed=3), strict=True)
    return m.to(dev).train()


def replay_round(cls, data):
    """ms per graph-replayed step, peak MiB, and whether two replays from one saved state give the same bits."""
    m = build(cls)
    start = {k: v.clone() for k, v in m.state_dict().items()}
    tr = MatcherTrainer(m, lr=1e-5)
    opt = tr.state_dict()
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
    res = []
    for _ in range(2):
        m.load_state_dict(start)
        tr.load_state_dict(opt)
        loss, _ = tr.step_graphed(data)
        res.append((loss.clone(), tr.fp.flat.clone()))
    same = torch.equal(res[0][0], res[1][0]) and torch.equal(res[0][1], res[1][1])
    del tr, m, res
    torch.cuda.empty_cache()
    return ms, peak, same


KEYS = ("junction", "line_scores", "scatter", "gather", "index", "sort", "searchsorted", "radix", "max")


def kernel_times(cls, data, steps=3):
    """Device ms per eager step of the kernels whose names contain one of KEYS (the junction and line-score work and
    the generic torch kernels it shares names with)."""
    m = build(cls)
    tr = MatcherTrainer(m, lr=1e-5)
    tr.step(data)
    torch.cuda.synchronize()
    acts = [torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts) as prof:
        for _ in range(steps):
            tr.step(data)
        torch.cuda.synchronize()
    tot = defaultdict(float)
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name
            if any(k in name.lower() for k in KEYS):
                tot[name[:110]] += e.device_time_total / 1e3 / steps
    del tr, m
    torch.cuda.empty_cache()
    return tot


name, power, clk = gpu_info()
out(f"GPU: {name}, power limit {power}, max SM clock {clk}")
out(f"GlueStick bf16 training step (CUDA-graph replay of MatcherTrainer), {B} pairs, {N} points + {L} lines per image, "
    f"wireframes with shared junctions, 18 GNN layers, D=256; {ROUNDS} alternating rounds of {REPS} replays")
data = wireframe_batch()
arms = {"fixed": GlueStick, "torch": TorchLineOps}
res = {k: [] for k in arms}
for r in range(ROUNDS):
    for tag, cls in arms.items():
        res[tag].append(replay_round(cls, data))
        ms, peak, same = res[tag][-1]
        out(f"  round {r} {tag}: {ms:.2f} ms/step, peak {peak:.0f} MiB, two replays bit-identical: {same}")
med = {}
for tag in arms:
    t = sorted(x[0] for x in res[tag])
    med[tag] = t[len(t) // 2]
    out(f"{tag}: median {med[tag]:.2f} ms/step (range {t[0]:.2f}-{t[-1]:.2f}) = {B / med[tag] * 1e3:.1f} pairs/s; "
        f"peak {max(x[1] for x in res[tag]):.0f} MiB; bit-identical replays in {sum(x[2] for x in res[tag])} of "
        f"{ROUNDS} rounds")
diffs = sorted(a[0] - b[0] for a, b in zip(res["fixed"], res["torch"]))
out(f"fixed - torch: median {med['fixed'] - med['torch']:+.2f} ms/step ({100 * (med['fixed'] / med['torch'] - 1):+.1f} %); "
    f"per-round differences {diffs[0]:+.2f} to {diffs[-1]:+.2f} ms")
for tag, cls in arms.items():
    tot = kernel_times(cls, data)
    out(f"\n{tag}: device ms per step of the kernels named like {', '.join(KEYS)} (torch.profiler, eager steps)")
    for k, v in sorted(tot.items(), key=lambda kv: -kv[1]):
        if v >= 0.005:
            out(f"  {v:8.3f}  {k}")
    out(f"  {sum(tot.values()):8.3f}  total")

if args.out:
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")
