"""CPU oracle for GlueStick with intermediate line supervision (test infrastructure only): gluefactory's GlueStick with
`inter_supervision` set, composed from the GlueStick oracle's building blocks (oracle/gluestick_oracle.py, whose
functions are left as they are for their existing callers).  Pinned against the unmodified reference through
tests/golden/gluestick_inter_l8_n160.npz (scripts/make_gluestick_inter_golden.py).

`w` is a flat dict under the reference's state_dict names (`inter_line_proj.{k}.*` for the k-th listed block);
`bn_stats` as in oracle/gluestick_oracle.py.
"""
from oracle import gluestick_oracle as G
from oracle.lightglue_oracle import filter_matches, log_double_softmax


def point_log_assignment_summary(la, stride=8):
    """What the fixture keeps of the point head's [B, M+1, N+1] log-assignment (the line heads' are kept whole): every
    `stride`-th row and column (the bin row and column included at M = N = 160), and the row and column maxima of the
    inner block."""
    inner = la[:, :-1, :-1]
    return {"log_assignment_sub": la[:, ::stride, ::stride], "log_assignment_rowmax": inner.max(2).values,
            "log_assignment_colmax": inner.max(1).values}


def gluestick_forward(w, data, conf, bn_stats=None):
    """GlueStick._forward (gluestick.py:143-319) with lines present and no line attention.  For every block l of
    conf["inter_supervision"] the features after the cross layer i with i // 2 == l (AttentionalGNN.forward,
    gluestick.py:762-768) go through _get_line_matches with inter_line_proj[position of l] (gluestick.py:272-292)."""
    inter_sup = conf.get("inter_supervision") or []
    layers = conf["GNN_layers"]
    D = conf.get("descriptor_dim", 256)
    th = conf.get("filter_threshold", 0.2)
    size0, size1 = data["view0"]["image_size"], data["view1"]["image_size"]
    d0, d1 = data["descriptors0"], data["descriptors1"]
    if "input_proj.weight" in w:
        d0, d1 = G._conv(d0, w, "input_proj"), G._conv(d1, w, "input_proj")
    d0 = d0 + G.keypoint_encoder(G.normalize_keypoints(data["keypoints0"], size0), data["keypoint_scores0"], w, bn_stats)
    d1 = d1 + G.keypoint_encoder(G.normalize_keypoints(data["keypoints1"], size1), data["keypoint_scores1"], w, bn_stats)
    B, L0 = data["lines0"].shape[:2]
    L1 = data["lines1"].shape[1]
    l0 = G.normalize_keypoints(data["lines0"].reshape(B, 2 * L0, 2), size0).reshape(B, L0, 2, 2)
    l1 = G.normalize_keypoints(data["lines1"].reshape(B, 2 * L1, 2), size1).reshape(B, L1, 2, 2)
    enc0 = G.endpoint_encoder(l0, data["line_scores0"], w, bn_stats)
    enc1 = G.endpoint_encoder(l1, data["line_scores1"], w, bn_stats)
    idx0, idx1 = data["lines_junc_idx0"].reshape(B, -1), data["lines_junc_idx1"].reshape(B, -1)
    inter = {}
    for i, kind in enumerate(layers):
        d0, d1 = G.gnn_layer(d0, d1, w, i, kind, bn_stats)
        if kind == "self":
            d0, d1 = G.line_layer(d0, d1, enc0, enc1, idx0, idx1, w, i // 2, bn_stats)
        if kind == "cross" and i // 2 in inter_sup:
            inter[i // 2] = (d0, d1)
    md0, md1 = G._conv(d0, w, "final_proj"), G._conv(d1, w, "final_proj")
    scores = log_double_softmax(md0 @ md1.transpose(1, 2) / D**0.5, w["bin_score"])
    m0, m1, ms0, ms1 = filter_matches(scores, th)
    pred = {"log_assignment": scores, "matches0": m0, "matches1": m1, "matching_scores0": ms0, "matching_scores1": ms1}

    def line_head(e0, e1, proj):
        raw = G.line_scores_from_junctions(e0[:, :2 * L0], e1[:, :2 * L1], idx0, idx1, w, proj, D)
        la = log_double_softmax(raw, w["line_bin_score"])
        return (la, *filter_matches(la, th), raw)

    la, lm0, lm1, lms0, lms1, raw = line_head(d0, d1, "final_line_proj")
    pred.update({"line_log_assignment": la, "line_matches0": lm0, "line_matches1": lm1, "line_matching_scores0": lms0,
                 "line_matching_scores1": lms1, "raw_line_scores": raw})
    layer2idx = {block: k for k, block in enumerate(inter_sup)}
    for block in inter_sup:
        la, lm0, lm1, lms0, lms1, _ = line_head(*inter[block], f"inter_line_proj.{layer2idx[block]}")
        pred.update({f"line_{block}_log_assignment": la, f"line_{block}_matches0": lm0, f"line_{block}_matches1": lm1,
                     f"line_{block}_matching_scores0": lms0, f"line_{block}_matching_scores1": lms1})
    return pred


def gluestick_loss(w, pred, data, conf):
    """GlueStick.loss (gluestick.py:417-438), training branch: the final heads' terms (oracle/gluestick_oracle.py), then
    per listed block `line_{l}_assignment_nll`, added to the total as nll * nll_weight * loss.inter_supervision[position
    of l], against the final line head's ground truth and without statistics entries."""
    losses = G.gluestick_loss(w, pred, data, conf)
    inter_sup = conf.get("inter_supervision") or []
    lc = conf.get("loss", {})
    bal, wgt = lc.get("nll_balancing", 0.5), lc.get("nll_weight", 1.0)
    weights = lc.get("inter_supervision", [0.3, 0.6])
    layer2idx = {block: k for k, block in enumerate(inter_sup)}
    for block in inter_sup:
        nll, _, _ = G._sub_loss(pred[f"line_{block}_log_assignment"], data["gt_line_assignment"],
                                data["gt_line_matches0"], data["gt_line_matches1"], bal)
        losses[f"line_{block}_assignment_nll"] = nll
        losses["total"] = losses["total"] + nll * wgt * weights[layer2idx[block]]
    return losses
