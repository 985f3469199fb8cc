"""Generate tests/golden/gluestick_inter_l8_n160.npz by running the UNMODIFIED reference GlueStick
(gluefactory/models/matchers/gluestick.py) with intermediate line supervision on the CPU in fp64.  Test infrastructure
only; it needs the reference tree ($GLUEFACTORY_REFERENCE) and the omegaconf stand-in of oracle/_shim, like
oracle/make_golden.py, whose helpers it uses.  It writes no other fixture.

    python scripts/make_gluestick_inter_golden.py

Training mode (BatchNorm batch statistics), forward + loss + backward, B=2, N=160 points, L=24 lines, 8 GNN layers,
inter_supervision [0, 2] with loss.inter_supervision [0.3, 0.6]: block 2 takes the second weight, so a head weighted by
its block number instead of its position would read past the list.  Weights come from synthetic.make_gluestick_weights
over the PLUGIN's state_dict and are loaded strictly into the reference (which also proves the two module trees carry
identical names and shapes); inputs from synthetic.make_gluestick_batch.  Stored: predictions (the intermediate heads'
line_{l}_* included; of the point head's log-assignment, which tests/golden/gluestick_l4_n160.npz holds whole, only
tests/gluestick_inter_oracle.point_log_assignment_summary, to keep the file small), every loss entry, summarised parameter gradients (inter_line_proj.* included), the updated
BatchNorm running statistics, and as metadata the reference's state_dict key order for this configuration and for the
matcher section of configs/superpoint+lsd+gluestick-homography.yaml (18 layers, inter_supervision [2, 5]).
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden  # noqa: E402  (puts the reference and oracle/_shim on sys.path)
from gluefactory_b200 import synthetic  # noqa: E402
from tests.gluestick_inter_oracle import point_log_assignment_summary  # noqa: E402

# the matcher section of configs/superpoint+lsd+gluestick-homography.yaml
HOMOGRAPHY_CONF = {"input_dim": 256, "descriptor_dim": 256, "inter_supervision": [2, 5],
                   "GNN_layers": ["self", "cross"] * 9, "checkpointed": True}


def run_gluestick_inter(name="gluestick_inter_l8_n160", n_gnn=8, B=2, N=160, L=24, seed=151):
    from gluefactory.models import get_model
    from gluefactory_b200.matchers.gluestick import GlueStick as Plugin

    conf = {"GNN_layers": ["self", "cross"] * (n_gnn // 2), "filter_threshold": 0.2, "inter_supervision": [0, 2],
            "loss": {"nll_weight": 1.0, "nll_balancing": 0.5, "inter_supervision": [0.3, 0.6]}}
    sd = synthetic.make_gluestick_weights(Plugin(dict(conf)).state_dict(), seed=seed)
    model = get_model("matchers.gluestick")(dict(conf, name="matchers.gluestick")).double()
    assert list(model.state_dict().keys()) == list(sd.keys())
    model.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}, strict=True)
    model = model.train()
    data = synthetic.make_gluestick_batch(B, N, L, seed + 1, dtype=torch.float64)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    homography = get_model("matchers.gluestick")(dict(HOMOGRAPHY_CONF, name="matchers.gluestick"))
    out = {"meta|conf": np.array(repr(conf)), "meta|B": np.array(B), "meta|N": np.array(N), "meta|L": np.array(L),
           "meta|seed": np.array(seed), "meta|ref_keys": np.array(list(model.state_dict().keys())),
           "meta|homography_conf": np.array(repr(HOMOGRAPHY_CONF)),
           "meta|homography_ref_keys": np.array(list(homography.state_dict().keys()))}
    keys = ["matches0", "matches1", "matching_scores0", "matching_scores1", "line_matches0", "line_matches1",
            "line_matching_scores0", "line_log_assignment", "raw_line_scores"]
    for block in conf["inter_supervision"]:
        keys += [f"line_{block}_{k}" for k in ("log_assignment", "matches0", "matches1", "matching_scores0",
                                               "matching_scores1")]
    for k in keys:
        out["pred|" + k] = pred[k].detach().numpy()
    for k, v in point_log_assignment_summary(pred["log_assignment"].detach()).items():
        out["pred|" + k] = v.numpy()
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
    inter = " ".join(f"line_{b}={int((pred[f'line_{b}_matches0'] > -1).sum())}" for b in conf["inter_supervision"])
    print(f"{name}: loss={losses['total'].mean().item():.6f} point matches={int((pred['matches0'] > -1).sum())} "
          f"line matches={int((pred['line_matches0'] > -1).sum())} {inter} "
          f"params={sum(p.numel() for p in model.parameters())} -> {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    torch.set_num_threads(8)
    run_gluestick_inter()
