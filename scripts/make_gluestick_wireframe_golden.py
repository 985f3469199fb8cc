"""Generate tests/golden/gluestick_wireframe_{a_eval,b_train,c_no_lines,d_no_keypoints,e_image_shape}.npz by running the
UNMODIFIED reference GlueStick (gluefactory/models/matchers/gluestick.py) on the CPU in fp64, on wireframes built by the
reference's own `lines_to_wireframe` (gluefactory/models/lines/wireframe.py; needs scikit-learn).  Test infrastructure
only; it needs the reference tree ($GLUEFACTORY_REFERENCE) and the omegaconf stand-in of oracle/_shim, like
oracle/make_golden.py, whose helpers it uses.  It writes no other fixture.

    python scripts/make_gluestick_wireframe_golden.py

Segments are seeded so that their endpoints cluster: most run between a few shared centres (some centres end 3 or more
segments), each endpoint jittered by 0.7 px, so that DBSCAN (nms_radius 3, as WireframeExtractor's default) merges them
into shared junctions; a few free segments end alone.  Keypoints closer than nms_radius to an endpoint are removed
(merge_points) or, with force_num_keypoints, replaced by random ones with score 0, and the junctions come first among
the nodes, as in WireframeExtractor._forward (wireframe.py:163-306).  View 1 is view 0 under a mild homography (its dense
descriptor map is view 0's warped), minus some segments and keypoints, plus others.

Cases (4 GNN blocks, 3 in b_train; weights from synthetic.make_gluestick_weights over the PLUGIN's state_dict, loaded strictly):
  a_eval          eval mode, B=1, BatchNorm running statistics that are not the defaults (`_calibrate`, stored as bn|*),
                  force_num_lines False; M != N, neither a multiple of 8; pred stored whole.
  b_train         training mode, B=2, force_num_lines / force_num_keypoints True (junctions padded with random ones that
                  no line touches), inter_supervision [1]; every loss entry, summarised parameter gradients, the updated
                  running statistics, and the predictions.
  c_no_lines      eval (as a_eval), view 1 without lines (L1 = 0).
  d_no_keypoints  eval, view 0 without keypoints or lines (M = 0).
  e_image_shape   eval, both views given with `image` (stored as its shape) and without `image_size`, of different sizes.
Inputs are stored as the tensors the matcher receives (in|*); the reference runs on them cast to fp64.  The descriptors
are rounded to fp16 and stored so (exact in fp32 and fp64), which halves the fixtures; everything else is float32 /
int64.
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

NMS_RADIUS = 3
S_DESC = 8
D = 256


def _segments(rs, W, H, n_centres, n_shared, n_free, n_hubs):
    """[L, 2, 2] segments: n_shared between centres (hubs first: each of the n_hubs first centres ends 3 or 4 of them),
    n_free with both endpoints alone; permuted."""
    centres = np.stack([rs.uniform(12, W - 12, n_centres), rs.uniform(12, H - 12, n_centres)], -1)
    pairs = []
    for h in range(n_hubs):
        for _ in range(3 + h % 2):
            pairs.append((h, rs.randint(n_hubs, n_centres)))
    while len(pairs) < n_shared:
        a, b = rs.choice(n_centres, 2, replace=False)
        pairs.append((a, b))
    seg = centres[np.array(pairs[:n_shared])] + 0.7 * rs.standard_normal((n_shared, 2, 2))
    ang = rs.uniform(0, np.pi, n_free)
    start = np.stack([rs.uniform(20, W - 20, n_free), rs.uniform(20, H - 20, n_free)], -1)
    end = np.clip(start + rs.uniform(20, 120, (n_free, 1)) * np.stack([np.cos(ang), np.sin(ang)], -1), 1, [W - 1, H - 1])
    return np.concatenate([seg, np.stack([start, end], 1)])[rs.permutation(n_shared + n_free)]


def _warp(p, Hm):
    q = np.concatenate([p, np.ones((len(p), 1))], 1) @ Hm.T
    return q[:, :2] / q[:, 2:]


def _dense_pair(rs, Hm, W, H):
    """Dense descriptor maps [1, D, H/8, W/8] of both views: view 1's samples view 0's through H^-1, plus noise."""
    h, w = H // S_DESC, W // S_DESC
    dense0 = torch.from_numpy(rs.standard_normal((1, D, h, w))).float()
    ys, xs = np.meshgrid((np.arange(h) + 0.5) * S_DESC, (np.arange(w) + 0.5) * S_DESC, indexing="ij")
    src = _warp(np.stack([xs.ravel(), ys.ravel()], -1), np.linalg.inv(Hm))
    grid = torch.from_numpy(src / np.array([W, H]) * 2 - 1).float().view(1, h, w, 2)
    dense1 = torch.nn.functional.grid_sample(dense0, grid, mode="bilinear", align_corners=False)
    dense1 = dense1 + 0.3 * torch.from_numpy(rs.standard_normal((1, D, h, w))).float()
    return dense0, dense1


def _view(rs, lines, kpts, dense, W, H, force):
    """WireframeExtractor._forward (merge_points, merge_line_endpoints) for one image: nodes = junctions then keypoints.
    force: force_num_lines / force_num_keypoints (pad the junctions to 2L, replace removed keypoints)."""
    from gluefactory.models.lines.wireframe import lines_to_wireframe, sample_descriptors_corner_conv

    L = len(lines)
    lines_t = torch.from_numpy(lines).float()[None]
    kp = torch.from_numpy(kpts).float()[None]
    kp_scores = torch.from_numpy(rs.uniform(0.05, 1, len(kpts))).float()[None]
    line_scores = torch.from_numpy(rs.uniform(0.05, 1, L)).float()[None]
    if L > 0:
        line_scores = line_scores / (line_scores.max(1)[0][:, None] + 1e-8)  # wireframe.py:175-176
    desc = sample_descriptors_corner_conv(kp, dense, S_DESC).mT
    if L > 0:
        remove = torch.any(torch.norm(kp[:, :, None] - lines_t.reshape(1, -1, 2)[:, None], dim=-1) < NMS_RADIUS, 2)
        if force:
            n = int(remove.sum())
            kp[remove] = torch.from_numpy(rs.uniform(0, 1, (n, 2))).float() * torch.tensor([[W - 1, H - 1]]).float()
            kp_scores[remove] = 0
            desc[0][remove[0]] = sample_descriptors_corner_conv(kp[0][remove[0]][None], dense, S_DESC)[0].T
        else:
            kp, kp_scores, desc = kp[:, ~remove[0]], kp_scores[:, ~remove[0]], desc[:, ~remove[0]]
        junc, junc_scores, junc_desc, _, new_lines, junc_idx, n_true = lines_to_wireframe(
            lines_t, line_scores, dense, s=S_DESC, nms_radius=NMS_RADIUS, force_num_lines=force, max_num_lines=L)
        nodes = torch.cat([junc[0], kp[0]])
        scores = torch.cat([junc_scores[0], kp_scores[0]])
        descs = torch.cat([junc_desc[0], desc[0]])
        lines_out, idx = new_lines[0], junc_idx[0]
    else:
        nodes, scores, descs = kp[0], kp_scores[0], desc[0]
        lines_out, idx, n_true = torch.zeros(0, 2, 2), torch.zeros(0, 2, dtype=torch.long), [0]
    # rounded to fp16: stored as such in the fixture, exactly the values the matcher and the reference receive
    return {"keypoints": nodes, "keypoint_scores": scores, "descriptors": descs.half().float(), "lines": lines_out,
            "lines_junc_idx": idx, "line_scores": line_scores[0], "num_junctions": int(n_true[0])}


def _pair(seed, W=640, H=480, n_shared=40, n_free=8, n_centres=30, n_hubs=5, n_kp=150, force=False, no_lines1=False,
          no_view0=False):
    rs = np.random.RandomState(seed)
    torch.manual_seed(seed)  # the random junctions of force_num_lines (wireframe.py:86-95)
    Hm = synthetic._random_homography(rs, 512.0, difficulty=0.3)
    dense0, dense1 = _dense_pair(rs, Hm, W, H)
    l0 = _segments(rs, W, H, n_centres, n_shared, n_free, n_hubs)
    k0 = np.stack([rs.uniform(2, W - 2, n_kp), rs.uniform(2, H - 2, n_kp)], -1)
    # view 1: 80 % of view 0's segments and keypoints under H (0.5 px noise), then new ones up to the same counts
    keep = rs.permutation(len(l0))[:int(0.8 * len(l0))]
    l1 = _warp(l0[keep].reshape(-1, 2), Hm).reshape(-1, 2, 2) + 0.5 * rs.standard_normal((len(keep), 2, 2))
    l1 = np.concatenate([l1, _segments(rs, W, H, 8, len(l0) - len(keep) - 2, 2, 1)])
    inside = np.all((l1 > 1) & (l1 < np.array([W - 1, H - 1])), (1, 2))
    l1 = l1[inside] if not force else np.clip(l1, 1, [W - 1, H - 1])
    kk = rs.permutation(n_kp)[:int(0.7 * n_kp)]
    k1 = np.concatenate([_warp(k0[kk], Hm) + 0.5 * rs.standard_normal((len(kk), 2)),
                         np.stack([rs.uniform(2, W - 2, n_kp - len(kk)), rs.uniform(2, H - 2, n_kp - len(kk))], -1)])
    k1 = np.clip(k1, 2, [W - 2, H - 2])[rs.permutation(n_kp)]
    if no_lines1:
        l1 = l1[:0]
    if no_view0:
        l0, k0 = l0[:0], k0[:0]
    v0 = _view(rs, l0, k0, dense0, W, H, force)
    v1 = _view(rs, l1, k1, dense1, W, H, force)
    return v0, v1, Hm


def _line_labels(idx0, idx1, m0, L0, L1):
    """A line of view 0 matches a line of view 1 when the point labels map its two junctions onto that line's two."""
    asg = torch.zeros(L0, L1, dtype=torch.bool)
    for a in range(L0):
        j = [int(m0[int(idx0[a, e])]) for e in (0, 1)]
        for b in range(L1):
            if j[0] >= 0 and sorted(j) == sorted(int(x) for x in idx1[b]) and j[0] != j[1]:
                asg[a, b] = True
    lm0 = torch.where(asg.any(1), asg.float().argmax(1), torch.full((L0,), -1, dtype=torch.long))
    lm1 = torch.where(asg.any(0), asg.float().argmax(0), torch.full((L1,), -1, dtype=torch.long))
    return asg, lm0, lm1


def _batch(views, sizes=None, shapes=None):
    """Stack per-image views ([(v0, v1), ...]) into the matcher's inputs."""
    data = {}
    for i in "01":
        for k in ("keypoints", "keypoint_scores", "descriptors", "lines", "lines_junc_idx", "line_scores"):
            data[f"{k}{i}"] = torch.stack([v[int(i)][k] for v in views])
    for i in "01":
        if shapes is not None:
            data[f"view{i}"] = {"image": torch.zeros(shapes[int(i)])}
        else:
            data[f"view{i}"] = {"image_size": torch.tensor([sizes[int(i)]] * len(views), dtype=torch.float32)}
    return data


def _calibrate(model, data, rs):
    """Eval-mode running statistics near the ones of a trained model: each BatchNorm's statistics of one training-mode
    forward on `data` (momentum 1: the last call's, image 1's for the shared modules), then moved off them (mean +
    0.05 N(0, 1), variance x U(0.8, 1.25)), so that the eval path cannot pass by using batch statistics."""
    bns = [m for m in model.modules() if isinstance(m, torch.nn.BatchNorm1d)]
    for m in bns:
        m.momentum = 1.0
    with torch.no_grad():
        model.train()(data)
        for m in bns:
            m.momentum = 0.1
            m.running_mean += 0.05 * torch.from_numpy(rs.standard_normal(m.running_mean.shape))
            m.running_var *= torch.from_numpy(rs.uniform(0.8, 1.25, m.running_var.shape))
            m.num_batches_tracked.zero_()


def _run(name, conf, data, seed, training, n_junctions, gt=None):
    from gluefactory.models import get_model
    from gluefactory_b200.matchers.gluestick import GlueStick as Plugin

    sd = synthetic.make_gluestick_weights(Plugin(dict(conf)).state_dict(), seed=seed)
    model = get_model("matchers.gluestick")(dict(conf, name="matchers.gluestick")).double()
    assert list(model.state_dict().keys()) == list(sd.keys())
    model.load_state_dict({k: (v.double() if v.is_floating_point() else v) for k, v in sd.items()}, strict=True)
    d64 = {k: ({kk: (vv.double() if vv.is_floating_point() else vv) for kk, vv in v.items()} if isinstance(v, dict) else
               (v.double() if v.is_floating_point() else v)) for k, v in {**data, **(gt or {})}.items()}
    if not training:
        _calibrate(model, d64, np.random.RandomState(seed + 1))
    model = model.train(training)
    out = {"meta|conf": np.array(repr(conf)), "meta|seed": np.array(seed), "meta|training": np.array(training),
           "meta|num_junctions": np.array(n_junctions)}
    for k, v in {**data, **(gt or {})}.items():
        if isinstance(v, dict):
            for kk, vv in v.items():
                out[f"in|{kk}{k[-1]}" if kk == "image_size" else f"in|image_shape{k[-1]}"] = (
                    vv.numpy() if kk == "image_size" else np.array(vv.shape))
        else:
            out["in|" + k] = (v.half() if k.startswith("descriptors") else v).numpy()
    if training:
        pred = model(d64)
        losses, _ = model.loss(pred, d64)
        losses["total"].mean().backward()
        for k, v in losses.items():
            out["loss|" + k] = v.detach().numpy() if torch.is_tensor(v) else np.array(v)
        for k, p in model.named_parameters():
            assert p.grad is not None, k
            out.update(make_golden.summarise("grad|" + k, p.grad))
    else:
        with torch.no_grad():
            pred = model(d64)
    # training: the running statistics after the step; eval: the ones the forward used
    for k, v in model.state_dict().items():
        if "running_" in k:
            out["bn|" + k] = v.numpy()
    for k, v in pred.items():
        if training and k == "log_assignment":  # kept as a summary, to keep the file small
            for kk, vv in point_log_assignment_summary(v.detach()).items():
                out["pred|" + kk] = vv.numpy()
        else:
            out["pred|" + k] = v.detach().numpy()
    path = os.path.join(make_golden.OUT, f"gluestick_wireframe_{name}.npz")
    np.savez_compressed(path, **out)
    M, N = data["keypoints0"].shape[1], data["keypoints1"].shape[1]
    L0, L1 = data["lines0"].shape[1], data["lines1"].shape[1]
    extra = f" loss={losses['total'].mean().item():.6f}" if training else ""
    print(f"{name}: M={M} N={N} L0={L0} L1={L1} junctions={n_junctions}{extra} "
          f"point matches={int((pred['matches0'] > -1).sum())} line matches={int((pred['line_matches0'] > -1).sum())} "
          f"max matching score={float(pred['matching_scores0'].max()) if pred['matching_scores0'].numel() else 0:.3f} "
          f"-> {path} ({os.path.getsize(path) / 1e6:.2f} MB)")
    return data, pred


def _degree_check(views):
    """Shared junctions: some junction ends 3 or more lines; some node is touched by no line."""
    for v in views:
        for view in v:
            idx = view["lines_junc_idx"].reshape(-1)
            if idx.numel() == 0:
                continue
            deg = torch.bincount(idx, minlength=len(view["keypoints"]))
            assert int(deg.max()) >= 3 and int((deg == 0).sum()) > 0, deg


def main():
    eval_conf = {"GNN_layers": ["self", "cross"] * 4, "filter_threshold": 0.2}
    size = [640.0, 480.0]
    # (a) eval, B = 1, unpadded
    v0, v1, _ = _pair(211)
    _degree_check([(v0, v1)])
    M, N = len(v0["keypoints"]), len(v1["keypoints"])
    assert M != N and M % 8 and N % 8, (M, N)
    _run("a_eval", eval_conf, _batch([(v0, v1)], sizes=(size, size)), 213, False, [v0["num_junctions"], v1["num_junctions"]])
    # (b) training, B = 2, padded wireframes, inter_supervision [1]
    # 3 GNN blocks (block 1 is then an intermediate one) and ~120 nodes per view keep the fixture small
    train_conf = dict(eval_conf, GNN_layers=["self", "cross"] * 3, inter_supervision=[1], loss={"nll_weight": 1.0, "nll_balancing": 0.5,
                                                              "inter_supervision": [0.3, 0.6]})
    views, hs = [], []
    for s in (221, 222):
        v0, v1, Hm = _pair(s, n_shared=26, n_free=4, n_centres=20, n_kp=60, force=True)
        views.append((v0, v1))
        hs.append(Hm)
    _degree_check(views)
    data = _batch(views, sizes=(size, size))
    gts = [synthetic.gt_matches_from_homography(data["keypoints0"][b:b + 1].double(), data["keypoints1"][b:b + 1].double(),
                                                torch.from_numpy(hs[b])[None]) for b in range(2)]
    gt = {"gt_assignment": torch.cat([g[0] for g in gts]), "gt_matches0": torch.cat([g[1] for g in gts]),
          "gt_matches1": torch.cat([g[2] for g in gts])}
    L0, L1 = data["lines0"].shape[1], data["lines1"].shape[1]
    lab = [_line_labels(data["lines_junc_idx0"][b], data["lines_junc_idx1"][b], gt["gt_matches0"][b], L0, L1)
           for b in range(2)]
    gt.update(gt_line_assignment=torch.stack([x[0] for x in lab]), gt_line_matches0=torch.stack([x[1] for x in lab]),
              gt_line_matches1=torch.stack([x[2] for x in lab]))
    assert int(gt["gt_line_assignment"].sum()) > 0
    _run("b_train", train_conf, data, 223, True, [[v[0]["num_junctions"], v[1]["num_junctions"]] for v in views], gt)
    # (c) eval, view 1 without lines
    v0, v1, _ = _pair(231, n_shared=20, n_free=4, n_centres=16, n_hubs=3, n_kp=60, no_lines1=True)
    _run("c_no_lines", eval_conf, _batch([(v0, v1)], sizes=(size, size)), 233, False,
         [v0["num_junctions"], v1["num_junctions"]])
    # (d) eval, view 0 without keypoints (and so without lines)
    v0, v1, _ = _pair(241, n_shared=20, n_free=4, n_centres=16, n_hubs=3, n_kp=60, no_view0=True)
    _run("d_no_keypoints", eval_conf, _batch([(v0, v1)], sizes=(size, size)), 243, False,
         [v0["num_junctions"], v1["num_junctions"]])
    # (e) eval, views given with `image` only, of different sizes (image 1 is wider than the points' range)
    v0, v1, _ = _pair(251, n_shared=20, n_free=4, n_centres=16, n_hubs=3, n_kp=60)
    _run("e_image_shape", eval_conf, _batch([(v0, v1)], shapes=((1, 1, 480, 640), (1, 3, 512, 700))), 253, False,
         [v0["num_junctions"], v1["num_junctions"]])


if __name__ == "__main__":
    torch.set_num_threads(8)
    main()
