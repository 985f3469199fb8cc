"""Generate tests/golden/superglue_packed_l4.npz by running the UNMODIFIED reference SuperGlue
(gluefactory_nonfree/superglue.py) on the CPU in fp64 -- test infrastructure only; it needs the reference tree
($GLUEFACTORY_REFERENCE) and the omegaconf stand-in of oracle/_shim, like oracle/make_golden.py, whose import path it
uses.

    python scripts/make_superglue_packed_golden.py

Eval mode, 4 GNN layers, 50 Sinkhorn iterations, threshold 0.005 (random weights give flat assignments, whose mutual
scores sit near 0.007), one B = 1 call per pair at the sizes of PAIRS (one- and two-point views, sizes around 64 and
128, M != N both ways).  The packed GPU tests put these pairs into one NaN-padded call.  Weights come from synthetic.make_gluestick_weights over the plugin's state_dict, with the BatchNorm running
statistics moved away from (0, 1) so that eval-mode BatchNorm is not the identity; those statistics are stored.
Inputs come from synthetic.make_superglue_batch(1, m, n, seed), the seed stored per pair.  Stored per pair: the
log-assignment, matches and matching scores.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden  # noqa: E402  (puts the reference and oracle/_shim on sys.path)
from gluefactory_b200 import synthetic  # noqa: E402

PAIRS = [(1, 2), (2, 1), (63, 64), (65, 127), (128, 129), (150, 160), (97, 33)]
CONF = {"GNN_layers": ["self", "cross"] * 2, "num_sinkhorn_iterations": 50, "filter_threshold": 0.005, "weights": None}
WEIGHT_SEED = 41


def weights(plugin_state_dict, seed=WEIGHT_SEED):
    """Synthetic weights with running statistics away from (0, 1); returns (state dict, the running statistics)."""
    sd = synthetic.make_gluestick_weights(plugin_state_dict, seed=seed)
    g = torch.Generator().manual_seed(seed)
    bn = {}
    for k in sd:
        if k.endswith("running_mean"):
            sd[k] = bn[k] = 0.1 * torch.randn(sd[k].shape, generator=g, dtype=torch.float64).float()
        elif k.endswith("running_var"):
            sd[k] = bn[k] = (0.5 + torch.rand(sd[k].shape, generator=g, dtype=torch.float64)).float()
    return sd, bn


def run(name="superglue_packed_l4"):
    from gluefactory_nonfree.superglue import SuperGlue as Reference
    from gluefactory_b200.matchers.superglue import SuperGlue as Plugin

    sd, bn = weights(Plugin(dict(CONF)).state_dict())
    model = Reference(dict(CONF)).double()
    assert list(model.state_dict().keys()) == list(sd.keys())
    model.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}, strict=True)
    model = model.eval()
    out = {"meta|conf": np.array(repr(CONF)), "meta|weight_seed": np.array(WEIGHT_SEED),
           "meta|pairs": np.array(PAIRS)}
    out.update({"bn|" + k: v.numpy() for k, v in bn.items()})
    for i, (m, n) in enumerate(PAIRS):
        seed = 700 + i
        data = synthetic.make_superglue_batch(1, m, n, seed, dtype=torch.float64)
        for v in ("0", "1"):  # the reference reads view["image"].shape even when image_size is given
            data["view" + v]["image"] = torch.zeros(()).expand(1, 1, 1024, 1024)
        with torch.no_grad():
            pred = model(data)
        out[f"p{i}|seed"] = np.array(seed)
        for k in ["log_assignment", "matches0", "matches1", "matching_scores0", "matching_scores1"]:
            out[f"p{i}|{k}"] = pred[k][0].numpy()
        ms = pred["matching_scores0"][0]
        print(f"pair {i} ({m}, {n}): matches={int((pred['matches0'] > -1).sum())} "
              f"margin={float((ms[ms > 0] - CONF['filter_threshold']).abs().min()) if bool((ms > 0).any()) else None}")
    path = os.path.join(make_golden.OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name} -> {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    torch.set_num_threads(8)
    run()
