"""2-GPU diagnosis (torchrun): where does the synchronous step lose time against two free-running ranks?
Eager steps with CUDA events around the gradient exchange: [forward + backward] | [exchange incl. waiting for the peer] |
[check + Adam], per rank.  The exchange is the trainer's one all-reduce of the flat gradient buffer."""
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
torch.cuda.set_device(dev)
dist.init_process_group("nccl", device_id=dev)
from gluefactory_b200 import synthetic  # noqa: E402
from gluefactory_b200.matchers.homography_matcher import HomographyMatcher  # noqa: E402
from gluefactory_b200.matchers.lightglue import LightGlue  # noqa: E402
from gluefactory_b200.trainer import MatcherTrainer  # noqa: E402

conf = dict(synthetic.DEFAULT_CONF, precision="bf16")
model = LightGlue(conf)
model.load_state_dict(synthetic.make_weights(conf, seed=0), strict=False)
gt = HomographyMatcher({"th_positive": 3.0, "th_negative": 3.0, "transposed_assignment": True})
trainer = MatcherTrainer(model.to(dev), lr=1e-4, ground_truth=gt)
data = synthetic.to_device(synthetic.make_pairs(32, 2048, seed=1 + rank, with_gt=False), dev)
E = lambda: torch.cuda.Event(enable_timing=True)  # noqa: E731
e = [E() for _ in range(4)]
orig = trainer.exchange_gradients


def patched():
    e[1].record()
    orig()
    e[2].record()


trainer.exchange_gradients = patched
rows = []
for it in range(14):
    e[0].record()
    trainer.step(data)
    e[3].record()
    torch.cuda.synchronize()
    if it >= 4:
        rows.append([e[0].elapsed_time(e[1]), e[1].elapsed_time(e[2]), e[2].elapsed_time(e[3]), e[0].elapsed_time(e[3])])
t = torch.tensor(rows, device=dev)
st = torch.cat([t.mean(0), t.std(0)])
allst = [torch.zeros_like(st) for _ in range(world)]
dist.all_gather(allst, st)
if rank == 0:
    print("eager steps, per rank mean ms "
          "[fwd+bwd | exchange | check+adam | total] (std):", flush=True)
    for r, s_ in enumerate(allst):
        v = s_.tolist()
        print(f"  rank {r}: " + " | ".join(f"{v[i]:.2f} ({v[4 + i]:.2f})" for i in range(4)), flush=True)
sys.stdout.flush()
os._exit(0)
