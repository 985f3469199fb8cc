"""Multi-GPU diagnosis (torchrun, one rank per GPU): (1) the flat-gradient all-reduce alone (47.4 MB fp32 + loss slot),
eager and inside a CUDA graph; (2) per-rank step time of the captured training step, which ends in that one all-reduce
(rank skew / jitter)."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
torch.cuda.set_device(dev)
dist.init_process_group("nccl", device_id=dev)
buf = torch.randn(11_850_000 + 64, device=dev)


def ev():
    return torch.cuda.Event(enable_timing=True)


def timed(fn, n=20):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(n):
        dist.barrier()
        torch.cuda.synchronize()
        a, b = ev(), ev()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    t = torch.tensor(ts, device=dev)
    return t.median().item(), t.max().item()


med, mx = timed(lambda: dist.all_reduce(buf))
if rank == 0:
    print(f"all_reduce 47.4 MB fp32, eager: median {med:.3f} ms, max {mx:.3f} ms  ({buf.numel() * 4 / med / 1e6:.0f} GB/s algbw)")
g = torch.cuda.CUDAGraph()
s = torch.cuda.Stream()
s.wait_stream(torch.cuda.current_stream())
with torch.cuda.stream(s):
    dist.all_reduce(buf)
torch.cuda.current_stream().wait_stream(s)
with torch.cuda.graph(g):
    dist.all_reduce(buf)
med, mx = timed(g.replay)
if rank == 0:
    print(f"all_reduce inside a CUDA graph: median {med:.3f} ms, max {mx:.3f} ms")

# (2): the training step, per-rank timing
from gluefactory_b200 import synthetic  # noqa: E402
from gluefactory_b200.matchers.homography_matcher import HomographyMatcher  # noqa: E402
from gluefactory_b200.matchers.lightglue import LightGlue  # noqa: E402
from gluefactory_b200.trainer import MatcherTrainer  # noqa: E402

B = 32
conf = dict(synthetic.DEFAULT_CONF, precision="bf16")
model = LightGlue(conf)
model.load_state_dict(synthetic.make_weights(conf, seed=0), strict=False)
gt = HomographyMatcher({"th_positive": 3.0, "th_negative": 3.0, "transposed_assignment": True})
trainer = MatcherTrainer(model.to(dev), lr=1e-4, ground_truth=gt)
data = synthetic.to_device(synthetic.make_pairs(B, 2048, seed=1 + rank, with_gt=False), dev)
trainer.capture(data, dev)
for _ in range(3):
    trainer.step_graphed(data)
torch.cuda.synchronize()
ts = []
for _ in range(20):
    a, b = ev(), ev()
    a.record()
    trainer.step_graphed(data)
    b.record()
    torch.cuda.synchronize()
    ts.append(a.elapsed_time(b))
t = torch.tensor(ts, device=dev)
stats = torch.stack([t.mean(), t.std(), t.min(), t.max()])
allst = [torch.zeros_like(stats) for _ in range(world)]
dist.all_gather(allst, stats)
if rank == 0:
    print("captured step, per rank mean/std/min/max ms: "
          + " | ".join("/".join(f"{x:.2f}" for x in s_.tolist()) for s_ in allst))
dist.destroy_process_group()
