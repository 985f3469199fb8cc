"""Generate the loss-setting and label-extreme fixtures tests/golden/edge_*.npz by running the UNMODIFIED reference
matchers on the CPU in fp64, training mode: forward, loss and backward.  Test infrastructure only; it needs the reference
tree ($GLUEFACTORY_REFERENCE) and the omegaconf stand-in of oracle/_shim, like oracle/make_golden.py, whose helpers it
uses.  It writes no other fixture.

    python scripts/make_edge_golden.py

Every case runs the matchers with loss weights away from their symmetric defaults (LightGlue `gamma` 0 and 0.7,
`nll_balancing` 0.2 / 0.85 / 0.3 / 0.8, GlueStick `nll_weight` 2 and intermediate-head weights [0.25, 0.9]), so that a
swapped balance, a wrong layer-weight exponent or a dropped weight changes the stored values.  The labels come from
the synthetic homography labels and are then edited into the classes no other fixture has:

    edge_lg_a_labels     LightGlue 256 ch, 3 layers, gamma 0, nll_balancing 0.2, B 3, M 48, N 56: pair 0 as labelled,
                         pair 1 every label ignored (-2, no positives), pair 2 no negatives in view 1
    edge_lg_b_m1_n65     LightGlue 256 ch, 3 layers, gamma 0.7, nll_balancing 0.85, B 2, M 1, N 65: pair 0 its one view-0
                         point positive, pair 1 no positives
    edge_lg_c_m63_n130   the same loss settings, B 2, M 63, N 130: pair 1 has all of its positives in one row (one
                         view-0 point positive with four view-1 points)
    edge_sg_labels       SuperGlue, 2 GNN layers, nll_balancing 0.3, B 3, M 40, N 57: pair 1 no negatives in view 0,
                         pair 2 no positives
    edge_gs_labels       GlueStick, 4 GNN layers, inter_supervision [1, 0] weighted [0.25, 0.9], nll_balancing 0.8,
                         nll_weight 2, B 3, N 48, 8 lines: pair 1 no point or line negatives in view 1, pair 2 no point
                         or line positives

The edited labels are stored in each fixture (`label|*`); they cannot be rebuilt from the seeds.  The other inputs and
the weights are rebuilt from the stored seeds with gluefactory_b200.synthetic.  Stored besides: predictions, every loss
entry, summarised parameter gradients (oracle/make_golden.py `summarise`) and, for SuperGlue and GlueStick, the
BatchNorm running statistics after the backward.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden  # noqa: E402  (puts the reference and oracle/_shim on sys.path)
from gluefactory_b200 import synthetic  # noqa: E402

LG_A = dict(synthetic.DEFAULT_CONF, n_layers=3, filter_threshold=0.1,
            loss={"gamma": 0.0, "fn": "nll", "nll_balancing": 0.2})
LG_B = dict(synthetic.DEFAULT_CONF, n_layers=3, filter_threshold=0.1,
            loss={"gamma": 0.7, "fn": "nll", "nll_balancing": 0.85})
# name -> (conf, B, M, N, seed)
LG_CASES = {
    "edge_lg_a_labels": (LG_A, 3, 48, 56, 301),
    "edge_lg_b_m1_n65": (LG_B, 2, 1, 65, 303),
    "edge_lg_c_m63_n130": (LG_B, 2, 63, 130, 305),
}
SG_CONF = {"GNN_layers": ["self", "cross"], "filter_threshold": 0.2, "weights": None,
           "loss": {"nll_balancing": 0.3}}
GS_CONF = {"GNN_layers": ["self", "cross"] * 2, "filter_threshold": 0.2, "inter_supervision": [1, 0],
           "loss": {"nll_weight": 2.0, "nll_balancing": 0.8, "inter_supervision": [0.25, 0.9]}}


# ---- label edits (applied to the labels synthetic.make_pairs derived from the homography) ----
def ignore_all(asg, m0, m1, b):
    """Pair b: every point ignored (-2), so no positives and no negatives in either view."""
    asg[b] = False
    m0[b] = -2
    m1[b] = -2


def no_negatives(m, b):
    """Pair b: the unmatched points (-1) of this view become ignored (-2); its positives stay."""
    m[b] = torch.where(m[b] == -1, torch.full_like(m[b], -2), m[b])


def no_positives(asg, m0, m1, b):
    """Pair b: every positive becomes a negative on both sides."""
    asg[b] = False
    m0[b] = torch.where(m0[b] >= 0, torch.full_like(m0[b], -1), m0[b])
    m1[b] = torch.where(m1[b] >= 0, torch.full_like(m1[b], -1), m1[b])


def one_row(asg, m0, m1, b, i, cols):
    """Pair b: no positives but view-0 point i, positive with every view-1 point in `cols` (its label is the first)."""
    no_positives(asg, m0, m1, b)
    for j in cols:
        asg[b, i, j] = True
        m1[b, j] = i
    m0[b, i] = cols[0]


LABEL_EDITS = {
    "edge_lg_a_labels": lambda a, m0, m1: (ignore_all(a, m0, m1, 1), no_negatives(m1, 2)),
    "edge_lg_b_m1_n65": lambda a, m0, m1: (no_positives(a, m0, m1, 1), no_positives(a, m0, m1, 0),
                                           one_row(a, m0, m1, 0, 0, [17])),
    "edge_lg_c_m63_n130": lambda a, m0, m1: one_row(a, m0, m1, 1, 5, [3, 17, 40, 99]),
}


def _labels(data):
    return {"label|" + k: data[k].numpy() for k in ("gt_assignment", "gt_matches0", "gt_matches1")}


def run_lightglue(name, conf, B, M, N, seed):
    weights = synthetic.make_weights(conf, seed=seed)
    data = synthetic.make_pairs(B, N, seed=seed + 1, D=conf["input_dim"], M=M, dtype=torch.float64)
    LABEL_EDITS[name](data["gt_assignment"], data["gt_matches0"], data["gt_matches1"])
    model = make_golden.build_reference(conf, weights, torch.float64)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    out = {"meta|B": np.array(B), "meta|M": np.array(M), "meta|N": np.array(N), "meta|seed": np.array(seed),
           "meta|conf": np.array(repr(conf)), **_labels(data)}
    for k in ["matches0", "matches1", "matching_scores0", "matching_scores1", "log_assignment"]:
        out["pred|" + k] = pred[k].detach().numpy()
    for k, v in losses.items():
        out["loss|" + k] = v.detach().numpy() if torch.is_tensor(v) else np.array(v)
    for k, p in model.named_parameters():
        assert p.grad is not None, k
        out.update(make_golden.summarise("grad|" + k, p.grad))
    _save(name, out, f"loss={losses['total'].mean().item():.6f} matches={int((pred['matches0'] > -1).sum())}")


def run_superglue(name="edge_sg_labels", B=3, M=40, N=57, seed=311):
    from gluefactory_nonfree.superglue import SuperGlue as Reference
    from gluefactory_b200.matchers.superglue import SuperGlue as Plugin

    conf = SG_CONF
    sd = synthetic.make_gluestick_weights(Plugin(dict(conf)).state_dict(), seed=seed)
    model = Reference(dict(conf)).double()
    model.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}, strict=True)
    model = model.train()
    data = synthetic.make_superglue_batch(B, M, N, seed + 1, dtype=torch.float64)
    no_negatives(data["gt_matches0"], 1)
    no_positives(data["gt_assignment"], data["gt_matches0"], data["gt_matches1"], 2)
    for i in "01":  # the reference reads view["image"].shape even when image_size is given
        data["view" + i]["image"] = torch.zeros(()).expand(B, 1, 1024, 1024)
    pred = model(data)
    losses = model.loss(pred, data)
    losses["total"].mean().backward()
    out = {"meta|conf": np.array(repr(conf)), "meta|B": np.array(B), "meta|M": np.array(M), "meta|N": np.array(N),
           "meta|seed": np.array(seed), **_labels(data)}
    for k in ["sinkhorn_cost", "log_assignment", "matches0", "matches1", "matching_scores0", "matching_scores1"]:
        out["pred|" + k] = pred[k].detach().numpy()
    for k, v in losses.items():
        out["loss|" + k] = v.detach().numpy() if torch.is_tensor(v) else np.array(v)
    for k, p in model.named_parameters():
        out.update(make_golden.summarise("grad|" + k, p.grad))
    for k, v in model.state_dict().items():
        if "running_" in k or "num_batches_tracked" in k:
            out["bn|" + k] = v.numpy()
    _save(name, out, f"loss={losses['total'].mean().item():.6f}")


def run_gluestick(name="edge_gs_labels", B=3, N=48, L=8, seed=321):
    from gluefactory.models import get_model
    from gluefactory_b200.matchers.gluestick import GlueStick as Plugin

    conf = GS_CONF
    sd = synthetic.make_gluestick_weights(Plugin(dict(conf)).state_dict(), seed=seed)
    model = get_model("matchers.gluestick")(dict(conf, name="matchers.gluestick")).double()
    model.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}, strict=True)
    model = model.train()
    data = synthetic.make_gluestick_batch(B, N, L, seed + 1, dtype=torch.float64)
    for p in ("", "line_"):
        asg, m0, m1 = data[f"gt_{p}assignment"], data[f"gt_{p}matches0"], data[f"gt_{p}matches1"]
        no_negatives(m1, 1)
        no_positives(asg, m0, m1, 2)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    out = {"meta|conf": np.array(repr(conf)), "meta|B": np.array(B), "meta|N": np.array(N), "meta|L": np.array(L),
           "meta|seed": np.array(seed), **_labels(data)}
    for k in ("gt_line_assignment", "gt_line_matches0", "gt_line_matches1"):
        out["label|" + k] = data[k].numpy()
    keys = ["log_assignment", "matches0", "matches1", "matching_scores0", "matching_scores1", "line_log_assignment",
            "line_matches0", "line_matches1", "line_matching_scores0", "raw_line_scores"]
    for block in conf["inter_supervision"]:
        keys += [f"line_{block}_{k}" for k in ("log_assignment", "matches0", "matches1")]
    for k in keys:
        out["pred|" + k] = pred[k].detach().numpy()
    for k, v in losses.items():
        out["loss|" + k] = v.detach().numpy() if torch.is_tensor(v) else np.array(v)
    for k, p in model.named_parameters():
        assert p.grad is not None, k
        out.update(make_golden.summarise("grad|" + k, p.grad))
    for k, v in model.state_dict().items():
        if "running_" in k:
            out["bn|" + k] = v.numpy()
    _save(name, out, f"loss={losses['total'].mean().item():.6f}")


def _save(name, out, msg):
    path = os.path.join(make_golden.OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name}: {msg} -> {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    for name, (conf, B, M, N, seed) in LG_CASES.items():
        run_lightglue(name, conf, B, M, N, seed)
    run_superglue()
    run_gluestick()
