"""Generate tests/golden/superglue_l4_m150_n160.npz by running the UNMODIFIED reference SuperGlue
(gluefactory_nonfree/superglue.py) on the CPU in fp64 -- test infrastructure only; it needs the reference tree
($GLUEFACTORY_REFERENCE) and the omegaconf stand-in of oracle/_shim, like oracle/make_golden.py, whose helpers it uses.

    python scripts/make_superglue_golden.py

Training mode, forward + loss + backward, B=2, M=150, N=160, 4 GNN layers, 50 Sinkhorn iterations, threshold 0.2.
Weights come from synthetic.make_gluestick_weights over the PLUGIN's state_dict and are loaded strictly into the
reference (which also proves the two module trees carry identical names and shapes); inputs from
synthetic.make_superglue_batch.  Stored: predictions (sinkhorn_cost included), every loss entry, summarised parameter
gradients and the BatchNorm running statistics after the backward -- which carry the second update the reference's
checkpointed GNN layers make when the backward recomputes them.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden  # noqa: E402  (puts the reference and oracle/_shim on sys.path)
from gluefactory_b200 import synthetic  # noqa: E402


def run_superglue(name="superglue_l4_m150_n160", n_gnn=4, B=2, M=150, N=160, seed=91):
    from gluefactory_nonfree.superglue import SuperGlue as Reference
    from gluefactory_b200.matchers.superglue import SuperGlue as Plugin

    conf = {"GNN_layers": ["self", "cross"] * (n_gnn // 2), "filter_threshold": 0.2, "weights": None}
    sd = synthetic.make_gluestick_weights(Plugin(dict(conf)).state_dict(), seed=seed)
    model = Reference(dict(conf)).double()
    assert list(model.state_dict().keys()) == list(sd.keys())
    model.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}, strict=True)
    model = model.train()
    data = synthetic.make_superglue_batch(B, M, N, seed + 1, dtype=torch.float64)
    for i, n in (("0", M), ("1", N)):  # the reference reads view["image"].shape even when image_size is given
        data["view" + i]["image"] = torch.zeros(()).expand(B, 1, 1024, 1024)
    pred = model(data)
    losses = model.loss(pred, data)  # the reference's loss returns the losses dict alone
    losses["total"].mean().backward()
    out = {"meta|conf": np.array(repr(conf)), "meta|B": np.array(B), "meta|M": np.array(M), "meta|N": np.array(N),
           "meta|seed": np.array(seed)}
    for k in ["sinkhorn_cost", "log_assignment", "matches0", "matches1", "matching_scores0", "matching_scores1"]:
        out["pred|" + k] = pred[k].detach().numpy()
    for k, v in losses.items():
        out["loss|" + k] = v.detach().numpy() if torch.is_tensor(v) else np.array(v)
    for k, p in model.named_parameters():
        assert p.grad is not None, k
        out.update(make_golden.summarise("grad|" + k, p.grad))
    for k, v in model.state_dict().items():
        if "running_" in k or "num_batches_tracked" in k:
            out["bn|" + k] = v.numpy()
    path = os.path.join(make_golden.OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name}: loss={losses['total'].mean().item():.6f} matches={int((pred['matches0'] > -1).sum())} "
          f"params={sum(p.numel() for p in model.parameters())} -> {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    torch.set_num_threads(8)
    run_superglue()
