"""CPU oracle for the SuperGlue matcher (test infrastructure only): a plain-PyTorch restatement of
gluefactory_nonfree/superglue.py composed from the GlueStick oracle's building blocks (keypoint normalisation, Conv1d,
MLP with training-mode BatchNorm, multi-head attention with channel = d * H + h) and the Sinkhorn restatement of the
LightGlue oracle.  Pinned against the unmodified reference through tests/golden/superglue_l4_m150_n160.npz
(scripts/make_superglue_golden.py).

`w` is a flat dict under the reference's state_dict names.  `bn_stats`, when given, collects the batch mean / unbiased
variance per BatchNorm call (see oracle/gluestick_oracle.py); `running_stats` applies the reference's running-statistics
updates to them, including the second pass its checkpointed GNN layers make in the backward.
"""
import torch

from oracle.gluestick_oracle import _conv, _mlp, mha, normalize_keypoints
from oracle.lightglue_oracle import filter_matches, log_optimal_transport

MOMENTUM = 0.1


def superglue_forward(w, data, conf, bn_stats=None):
    """SuperGlue._forward (superglue.py:266-320) for non-empty keypoint sets."""
    layers = conf["GNN_layers"]
    D = conf.get("descriptor_dim", 256)
    n_enc = len(conf.get("keypoint_encoder", [32, 64, 128, 256])) + 1
    k0 = normalize_keypoints(data["keypoints0"], data["view0"]["image_size"])
    k1 = normalize_keypoints(data["keypoints1"], data["view1"]["image_size"])
    if conf.get("use_scores", True):
        k0 = torch.cat([k0, data["keypoint_scores0"][..., None]], -1)
        k1 = torch.cat([k1, data["keypoint_scores1"][..., None]], -1)
    d0 = data["descriptors0"] + _mlp(k0, w, "kenc.encoder", n_enc, bn_stats)
    d1 = data["descriptors1"] + _mlp(k1, w, "kenc.encoder", n_enc, bn_stats)
    for i, kind in enumerate(layers):
        pre = f"gnn.layers.{i}"
        s0, s1 = (d1, d0) if kind == "cross" else (d0, d1)
        out = []
        for x, src in ((d0, s0), (d1, s1)):
            out.append(x + _mlp(torch.cat([x, mha(x, src, w, pre + ".attn")], -1), w, pre + ".mlp", 2, bn_stats))
        d0, d1 = out
    md0, md1 = _conv(d0, w, "final_proj"), _conv(d1, w, "final_proj")
    cost = md0 @ md1.transpose(1, 2) / D**0.5
    scores = log_optimal_transport(cost, w["bin_score"], conf.get("num_sinkhorn_iterations", 50))
    m0, m1, ms0, ms1 = filter_matches(scores, conf.get("filter_threshold", 0.2))
    return {"sinkhorn_cost": cost, "log_assignment": scores, "matches0": m0, "matches1": m1, "matching_scores0": ms0,
            "matching_scores1": ms1}


def superglue_loss(w, pred, data, conf):
    """SuperGlue.loss (superglue.py:322-352)."""
    bal = conf.get("loss", {}).get("nll_balancing", 0.5)
    la = pred["log_assignment"]
    pos = data["gt_assignment"].to(la.dtype)
    num_pos = pos.sum((1, 2)).clamp(min=1.0)
    neg0, neg1 = (data["gt_matches0"] == -1).to(la.dtype), (data["gt_matches1"] == -1).to(la.dtype)
    num_neg = (neg0.sum(1) + neg1.sum(1)).clamp(min=1.0)
    nll_pos = -(la[:, :-1, :-1] * pos).sum((1, 2)) / num_pos
    nll_neg = (-(la[:, :-1, -1] * neg0).sum(1) - (la[:, -1, :-1] * neg1).sum(1)) / num_neg
    nll = bal * nll_pos + (1 - bal) * nll_neg
    return {"total": nll, "assignment_nll": nll, "nll_pos": nll_pos, "nll_neg": nll_neg, "num_matchable": num_pos,
            "num_unmatchable": num_neg, "bin_score": w["bin_score"][None]}


def running_stats(w, bn_stats, conf, backward=True):
    """The BatchNorm running statistics after one training forward (and, when `backward`, its backward) of the
    reference, from fresh ones in `w`: the keypoint encoder's BatchNorms update once per image; a GNN layer's MLP
    BatchNorm updates once per image in the forward and once more per image (image 0, then image 1) when the backward
    recomputes the checkpointed layer.  Returns {name: tensor} for running_mean / running_var / num_batches_tracked."""
    out = {}
    for name, calls in bn_stats.items():
        rm, rv = w[name + ".running_mean"].clone(), w[name + ".running_var"].clone()
        seq = list(calls) + (list(calls) if backward and name.startswith("gnn.") else [])
        for mean, var in seq:
            rm = (1 - MOMENTUM) * rm + MOMENTUM * mean
            rv = (1 - MOMENTUM) * rv + MOMENTUM * var
        out[name + ".running_mean"], out[name + ".running_var"] = rm, rv
        out[name + ".num_batches_tracked"] = torch.tensor(len(seq))
    return out
