"""Generate tests/golden/gluestick_d128_l4_n160.npz by running the UNMODIFIED reference GlueStick
(gluefactory/models/matchers/gluestick.py) at input_dim = descriptor_dim = 128 -- the DISK variant of the shipped
GlueStick configs, 4 heads of 32 channels -- on the CPU in fp64.  Test infrastructure only; it needs the reference tree
($GLUEFACTORY_REFERENCE) and the omegaconf stand-in of oracle/_shim, like oracle/make_golden.py, whose helpers it uses.
It writes no other fixture.

    python scripts/make_gluestick_d128_golden.py

Training mode (BatchNorm batch statistics), forward + loss + backward, B=2, N=160 points, L=24 lines, 4 GNN layers.
Weights come from synthetic.make_gluestick_weights over the PLUGIN's state_dict and are loaded strictly into the
reference (which also proves the two module trees carry identical names and shapes); inputs from
synthetic.make_gluestick_batch with 128-channel descriptors.  Stored: predictions, every loss entry, summarised
parameter gradients and the updated BatchNorm running statistics -- the same keys as oracle/make_golden.py `gluestick`.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden  # noqa: E402  (puts the reference and oracle/_shim on sys.path)
from gluefactory_b200 import synthetic  # noqa: E402


def run_gluestick_d128(name="gluestick_d128_l4_n160", n_gnn=4, B=2, N=160, L=24, seed=131, D=128):
    from gluefactory.models import get_model
    from gluefactory_b200.matchers.gluestick import GlueStick as Plugin

    conf = {"GNN_layers": ["self", "cross"] * (n_gnn // 2), "filter_threshold": 0.2, "input_dim": D,
            "descriptor_dim": D}
    sd = synthetic.make_gluestick_weights(Plugin(dict(conf)).state_dict(), seed=seed)
    model = get_model("matchers.gluestick")(dict(conf, name="matchers.gluestick")).double()
    assert list(model.state_dict().keys()) == list(sd.keys())
    model.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}, strict=True)
    model = model.train()
    data = synthetic.make_gluestick_batch(B, N, L, seed + 1, D=D, dtype=torch.float64)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    out = {"meta|conf": np.array(repr(conf)), "meta|B": np.array(B), "meta|N": np.array(N), "meta|L": np.array(L),
           "meta|seed": np.array(seed)}
    for k in ["matches0", "matches1", "matching_scores0", "matching_scores1", "log_assignment", "line_matches0",
              "line_matches1", "line_matching_scores0", "line_log_assignment", "raw_line_scores"]:
        out["pred|" + k] = pred[k].detach().numpy()
    for k, v in losses.items():
        out["loss|" + k] = v.detach().numpy() if torch.is_tensor(v) else np.array(v)
    for k, p in model.named_parameters():
        assert p.grad is not None, k
        out.update(make_golden.summarise("grad|" + k, p.grad))
    for k, v in model.state_dict().items():
        if "running_" in k:
            out["bn|" + k] = v.numpy()
    path = os.path.join(make_golden.OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name}: loss={losses['total'].mean().item():.6f} point matches={int((pred['matches0'] > -1).sum())} "
          f"line matches={int((pred['line_matches0'] > -1).sum())} params={sum(p.numel() for p in model.parameters())} "
          f"-> {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    torch.set_num_threads(8)
    run_gluestick_d128()
