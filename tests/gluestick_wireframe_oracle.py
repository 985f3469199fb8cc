"""CPU oracle for GlueStick on wireframe inputs (test infrastructure only): gluefactory's GlueStick._forward
(gluestick.py:143-319) composed from the GlueStick oracle's building blocks (oracle/gluestick_oracle.py, whose functions
are left as they are for their existing callers), extended with what real wireframes need:
  * BatchNorm in eval mode (running statistics) as well as training mode;
  * views without keypoints (the reference's early-exit pred, gluestick.py:163-195) and views without lines (no line
    encoding, LineLayer or line head, zero / -1 line outputs, gluestick.py:213-240, 257-312, 734-740);
  * views given with `image` and without `image_size` (normalised with image.shape[-2:], gluestick.py:146-156);
  * intermediate line supervision (`inter_supervision`).
Pinned against the unmodified reference through tests/golden/gluestick_wireframe_*.npz
(scripts/make_gluestick_wireframe_golden.py).

`w` is a flat dict under the reference's state_dict names; `bn_stats` as in oracle/gluestick_oracle.py (training mode).
"""
import ast
import os

import numpy as np
import torch

from oracle import gluestick_oracle as G
from oracle.lightglue_oracle import filter_matches, log_double_softmax

CASES = ["a_eval", "b_train", "c_no_lines", "d_no_keypoints", "e_image_shape"]


def image_size(view, kpts):
    """view["image_size"], or (w, h) of view["image"].shape[-2:] (normalize_keypoints with a shape, gluestick.py:478-482)."""
    if "image_size" in view:
        return view["image_size"]
    h, w = view["image"].shape[-2:]
    return kpts.new_tensor([[w, h]])


class _Net:
    """The building blocks of oracle/gluestick_oracle.py with BatchNorm in training mode (batch statistics) or in eval
    mode (running statistics, eps 1e-5)."""

    def __init__(self, w, training, bn_stats=None):
        self.w, self.training, self.bn_stats = w, training, bn_stats

    def bn(self, x, name):
        if self.training:
            return G._bn(x, self.w, name, self.bn_stats)
        w = self.w
        return (x - w[name + ".running_mean"]) / torch.sqrt(w[name + ".running_var"] + G.EPS_BN) * w[name + ".weight"] \
            + w[name + ".bias"]

    def mlp(self, x, pre, n_layers):
        for i in range(n_layers):
            x = G._conv(x, self.w, f"{pre}.{3 * i}")
            if i < n_layers - 1:
                x = torch.relu(self.bn(x, f"{pre}.{3 * i + 1}"))
        return x

    def keypoint_encoder(self, kpts, scores):
        return self.mlp(torch.cat([kpts, scores[..., None]], -1), "kenc.encoder", 5)

    def endpoint_encoder(self, lines, scores):
        B, L = lines.shape[:2]
        off = lines[:, :, 1] - lines[:, :, 0]
        off = torch.stack([off, -off], 2).reshape(B, 2 * L, 2)
        inp = torch.cat([lines.reshape(B, 2 * L, 2), off, scores.repeat(1, 2)[..., None]], -1)
        return self.mlp(inp, "lenc.encoder", 5)

    def gnn_layer(self, d0, d1, i, kind):
        pre = f"gnn.layers.{i}.update"
        s0, s1 = (d1, d0) if kind == "cross" else (d0, d1)
        out = []
        for x, src in ((d0, s0), (d1, s1)):
            msg = G.mha(x, src, self.w, pre + ".attn")
            out.append(x + self.mlp(torch.cat([x, msg], -1), pre + ".mlp", 2))
        return out[0], out[1]

    def line_layer(self, d0, d1, enc0, enc1, idx0, idx1, j):
        """LineLayer (gluestick.py:589-691): messages averaged over the endpoints that share a junction."""
        out = []
        for d, enc, idx in ((d0, enc0, idx0), (d1, enc1, idx1)):
            B, n2 = idx.shape
            D = d.shape[-1]
            ld = torch.gather(d, 1, idx[..., None].expand(B, n2, D))
            other = ld.view(B, n2 // 2, 2, D).flip(2).reshape(B, n2, D)
            upd = self.mlp(torch.cat([ld, other, enc], -1), f"gnn.line_layers.{j}.mlp", 2)
            acc = torch.zeros_like(d).scatter_reduce(1, idx[..., None].expand(B, n2, D), upd, reduce="mean",
                                                     include_self=False)
            out.append(d + acc)
        return out[0], out[1]


def empty_pred(B, n0, n1, L0, L1, dtype=torch.float32):
    """gluestick.py:163-195 (log_assignment [B, M, N], line_matching_scores1 [B, N], no raw_line_scores)."""
    return {"log_assignment": torch.zeros(B, n0, n1, dtype=dtype), "matches0": torch.full((B, n0), -1),
            "matches1": torch.full((B, n1), -1), "matching_scores0": torch.zeros(B, n0, dtype=dtype),
            "matching_scores1": torch.zeros(B, n1, dtype=dtype),
            "line_log_assignment": torch.zeros(B, L0, L1, dtype=dtype), "line_matches0": torch.full((B, L0), -1),
            "line_matches1": torch.full((B, L1), -1), "line_matching_scores0": torch.zeros(B, L0, dtype=dtype),
            "line_matching_scores1": torch.zeros(B, n1, dtype=dtype)}


def gluestick_forward(w, data, conf, training, bn_stats=None):
    """GlueStick._forward (gluestick.py:143-319), no line attention; BatchNorm in training or eval mode."""
    net = _Net(w, training, bn_stats)
    inter_sup = conf.get("inter_supervision") or []
    layers = conf["GNN_layers"]
    D = conf.get("descriptor_dim", 256)
    th = conf.get("filter_threshold", 0.2)
    kp0, kp1 = data["keypoints0"], data["keypoints1"]
    B, n0 = kp0.shape[:2]
    n1 = kp1.shape[1]
    L0, L1 = data["lines0"].shape[1], data["lines1"].shape[1]
    if n0 == 0 or n1 == 0:
        return empty_pred(B, n0, n1, L0, L1, kp0.dtype)
    size0, size1 = image_size(data["view0"], kp0), image_size(data["view1"], kp1)
    d0, d1 = data["descriptors0"], data["descriptors1"]
    if "input_proj.weight" in w:
        d0, d1 = G._conv(d0, w, "input_proj"), G._conv(d1, w, "input_proj")
    d0 = d0 + net.keypoint_encoder(G.normalize_keypoints(kp0, size0), data["keypoint_scores0"])
    d1 = d1 + net.keypoint_encoder(G.normalize_keypoints(kp1, size1), data["keypoint_scores1"])
    lines = L0 > 0 and L1 > 0
    if lines:
        l0 = G.normalize_keypoints(data["lines0"].reshape(B, 2 * L0, 2), size0).reshape(B, L0, 2, 2)
        l1 = G.normalize_keypoints(data["lines1"].reshape(B, 2 * L1, 2), size1).reshape(B, L1, 2, 2)
        enc0 = net.endpoint_encoder(l0, data["line_scores0"])
        enc1 = net.endpoint_encoder(l1, data["line_scores1"])
        idx0, idx1 = data["lines_junc_idx0"].reshape(B, -1), data["lines_junc_idx1"].reshape(B, -1)
    inter = {}
    for i, kind in enumerate(layers):
        d0, d1 = net.gnn_layer(d0, d1, i, kind)
        if kind == "self" and lines:
            d0, d1 = net.line_layer(d0, d1, enc0, enc1, idx0, idx1, i // 2)
        if kind == "cross" and i // 2 in inter_sup:
            inter[i // 2] = (d0, d1)
    md0, md1 = G._conv(d0, w, "final_proj"), G._conv(d1, w, "final_proj")
    scores = log_double_softmax(md0 @ md1.transpose(1, 2) / D**0.5, w["bin_score"])
    m0, m1, ms0, ms1 = filter_matches(scores, th)
    pred = {"log_assignment": scores, "matches0": m0, "matches1": m1, "matching_scores0": ms0, "matching_scores1": ms1}
    if not lines:
        z = kp0.dtype
        pred.update({"line_log_assignment": torch.zeros(B, L0, L1, dtype=z), "line_matches0": torch.full((B, L0), -1),
                     "line_matches1": torch.full((B, L1), -1), "line_matching_scores0": torch.zeros(B, L0, dtype=z),
                     "line_matching_scores1": torch.zeros(B, L1, dtype=z), "raw_line_scores": torch.zeros(B, L0, L1, dtype=z)})
        return pred

    def line_head(e0, e1, proj):
        raw = G.line_scores_from_junctions(e0[:, :2 * L0], e1[:, :2 * L1], idx0, idx1, w, proj, D)
        la = log_double_softmax(raw, w["line_bin_score"])
        return (la, *filter_matches(la, th), raw)

    la, lm0, lm1, lms0, lms1, raw = line_head(d0, d1, "final_line_proj")
    pred.update({"line_log_assignment": la, "line_matches0": lm0, "line_matches1": lm1, "line_matching_scores0": lms0,
                 "line_matching_scores1": lms1, "raw_line_scores": raw})
    for k, block in enumerate(inter_sup):
        la, lm0, lm1, lms0, lms1, _ = line_head(*inter[block], f"inter_line_proj.{k}")
        pred.update({f"line_{block}_log_assignment": la, f"line_{block}_matches0": lm0, f"line_{block}_matches1": lm1,
                     f"line_{block}_matching_scores0": lms0, f"line_{block}_matching_scores1": lms1})
    return pred


def load_case(golden, name, dtype=torch.float64):
    """(golden dict, conf, weights seed, data) of tests/golden/gluestick_wireframe_{name}.npz; float inputs in `dtype`,
    a view stored without image_size gets a zero `image` of the stored shape."""
    g = dict(np.load(os.path.join(golden, f"gluestick_wireframe_{name}.npz"), allow_pickle=False))
    conf = ast.literal_eval(str(g["meta|conf"]))
    data = {"view0": {}, "view1": {}}
    for k, v in g.items():
        if not k.startswith("in|"):
            continue
        t = torch.from_numpy(v)
        t = t.to(dtype) if t.is_floating_point() else t
        key = k[len("in|"):]
        if key.startswith("image_size"):
            data["view" + key[-1]]["image_size"] = t
        elif key.startswith("image_shape"):
            data["view" + key[-1]]["image"] = torch.zeros(tuple(int(s) for s in v), dtype=dtype)
        else:
            data[key] = t
    return g, conf, int(g["meta|seed"]), data


def case_state_dict(g, state_dict_like):
    """The weights a fixture was made with: synthetic.make_gluestick_weights from its seed; in eval mode with the
    BatchNorm running statistics the reference's forward used (bn|*, kept in fp64; load_state_dict rounds them to the
    module's dtype)."""
    from gluefactory_b200 import synthetic

    sd = synthetic.make_gluestick_weights(state_dict_like, seed=int(g["meta|seed"]))
    if not bool(g["meta|training"]):
        for k in sd:
            if "running_" in k:
                sd[k] = torch.from_numpy(g["bn|" + k])  # fp64, as the reference ran
    return sd
