"""CPU oracle for SuperGlue in eval mode (test infrastructure only): gluefactory_nonfree/superglue.py:266-320 composed
from the building blocks of oracle/gluestick_oracle.py (keypoint normalisation, Conv1d, multi-head attention with
channel = d * H + h) and the Sinkhorn and match-filter restatements of oracle/lightglue_oracle.py, with BatchNorm on
its running statistics (eps 1e-5).  tests/superglue_oracle.py is the training-mode twin.  Pinned against the unmodified
reference through tests/golden/superglue_packed_l4.npz (scripts/make_superglue_packed_golden.py).

`w` is a flat dict under the reference's state_dict names.
"""
import ast
import os

import numpy as np
import torch

from gluefactory_b200 import synthetic
from oracle.gluestick_oracle import EPS_BN, _conv, mha, normalize_keypoints
from oracle.lightglue_oracle import filter_matches, log_optimal_transport


def _mlp(x, w, pre, n_layers):
    """MLP(channels) of superglue.py:60-70 with eval-mode BatchNorm: conv, [BN, ReLU, conv]*."""
    for i in range(n_layers):
        x = _conv(x, w, f"{pre}.{3 * i}")
        if i < n_layers - 1:
            bn = f"{pre}.{3 * i + 1}"
            x = (x - w[bn + ".running_mean"]) / torch.sqrt(w[bn + ".running_var"] + EPS_BN) * w[bn + ".weight"] \
                + w[bn + ".bias"]
            x = torch.relu(x)
    return x


def superglue_forward_eval(w, data, conf):
    """SuperGlue._forward (superglue.py:266-320) in eval mode for non-empty keypoint sets."""
    D = conf.get("descriptor_dim", 256)
    n_enc = len(conf.get("keypoint_encoder", [32, 64, 128, 256])) + 1
    k0 = normalize_keypoints(data["keypoints0"], data["view0"]["image_size"])
    k1 = normalize_keypoints(data["keypoints1"], data["view1"]["image_size"])
    if conf.get("use_scores", True):
        k0 = torch.cat([k0, data["keypoint_scores0"][..., None]], -1)
        k1 = torch.cat([k1, data["keypoint_scores1"][..., None]], -1)
    d0 = data["descriptors0"] + _mlp(k0, w, "kenc.encoder", n_enc)
    d1 = data["descriptors1"] + _mlp(k1, w, "kenc.encoder", n_enc)
    for i, kind in enumerate(conf["GNN_layers"]):
        pre = f"gnn.layers.{i}"
        s0, s1 = (d1, d0) if kind == "cross" else (d0, d1)
        out = []
        for x, src in ((d0, s0), (d1, s1)):
            out.append(x + _mlp(torch.cat([x, mha(x, src, w, pre + ".attn")], -1), w, pre + ".mlp", 2))
        d0, d1 = out
    cost = _conv(d0, w, "final_proj") @ _conv(d1, w, "final_proj").transpose(1, 2) / D**0.5
    scores = log_optimal_transport(cost, w["bin_score"], conf.get("num_sinkhorn_iterations", 50))
    m0, m1, ms0, ms1 = filter_matches(scores, conf.get("filter_threshold", 0.2))
    return {"sinkhorn_cost": cost, "log_assignment": scores, "matches0": m0, "matches1": m1, "matching_scores0": ms0,
            "matching_scores1": ms1}


def load_fixture(golden, plugin_state_dict):
    """tests/golden/superglue_packed_l4.npz: (npz, conf, state dict with the stored running statistics, pairs as
    [(m, n, seed)])."""
    g = np.load(os.path.join(golden, "superglue_packed_l4.npz"))
    conf = ast.literal_eval(str(g["meta|conf"]))
    sd = synthetic.make_gluestick_weights(plugin_state_dict, seed=int(g["meta|weight_seed"]))
    for k in g:
        if k.startswith("bn|"):
            sd[k[3:]] = torch.from_numpy(g[k])
    pairs = [(int(m), int(n), int(g[f"p{i}|seed"])) for i, (m, n) in enumerate(g["meta|pairs"])]
    return g, conf, sd, pairs
