"""GPU: line ground truth on the device (csrc/gt_lines.cu) -- the homography and depth components against the
reference's own labels (tests/golden/gt_lines_*.npz), the label pass alone against the reference's cost matrices,
the device assignment solver against scipy's results and the CPU restatement (oracle/line_gt_oracle.py), labels at
L = 512, and GlueStick training with device line labels (one CUDA graph; the MegaDepth-style depth pipeline)."""
import os

import numpy as np
import pytest
import torch

from gluefactory_b200 import ops, synthetic
from oracle import line_gt_oracle as O
from tests.test_line_gt_cpu import tie_heavy_costs
from tests.util import GOLDEN

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _load(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    return g, sorted({k.split("|")[0] for k in g})


def _meta(g, tag):
    B, L0, L1, seed, npts, dist, ov, mvt, h, w = g[f"{tag}|meta"]
    conf = {"use_points": False, "use_lines": True, "n_line_sampled_pts": int(npts), "line_perp_dist_th": float(dist),
            "overlap_th": float(ov), "min_visibility_th": float(mvt)}
    return int(B), int(L0), int(L1), int(seed), int(h), int(w), conf


def _t(g, tag, k):
    return torch.from_numpy(g[f"{tag}|{k}"]).to(DEV)


def _check_labels(pred, g, tag):
    assert pred["line_assignment"].dtype == torch.bool and pred["line_matches0"].dtype == torch.int64
    assert np.array_equal(pred["line_matches0"].cpu().numpy(), g[f"{tag}|matches0"]), tag
    assert np.array_equal(pred["line_matches1"].cpu().numpy(), g[f"{tag}|matches1"]), tag
    assert np.array_equal(pred["line_assignment"].nonzero().cpu().numpy(), g[f"{tag}|positives"]), tag


def test_homography_component_reproduces_reference_line_labels():
    from gluefactory_b200.matchers.homography_matcher import HomographyMatcher

    g, tags = _load("gt_lines_homography")
    for tag in tags:
        B, L0, L1, seed, h, w, conf = _meta(g, tag)
        img = torch.zeros(B, 1, h, w, device=DEV)
        data = {"lines0": _t(g, tag, "lines0"), "lines1": _t(g, tag, "lines1"), "valid_lines0": _t(g, tag, "valid_lines0"),
                "valid_lines1": _t(g, tag, "valid_lines1"), "H_0to1": _t(g, tag, "H"), "view0": {"image": img},
                "view1": {"image": img}}
        _check_labels(HomographyMatcher(conf)(data), g, tag)
        # the 4-value line layout gives the same labels
        data["lines0"] = data["lines0"].flatten(-2)
        _check_labels(HomographyMatcher(conf)(data), g, tag)
    torch.cuda.synchronize()


def test_depth_component_reproduces_reference_line_labels():
    from gluefactory_b200.matchers.depth_matcher import DepthMatcher

    g, tags = _load("gt_lines_pose_depth")
    for tag in tags:
        B, L0, L1, seed, h, w, conf = _meta(g, tag)
        sc = synthetic.to_device(synthetic.line_gt_scene("pose_depth", B, L0, L1, seed), DEV)
        img = torch.zeros(B, 1, h, w, device=DEV)
        data = {"lines0": sc["lines0"], "lines1": sc["lines1"], "valid_lines0": sc["valid_lines0"],
                "valid_lines1": sc["valid_lines1"],
                "view0": {"camera": synthetic.PinholeCamera(sc["K0"]), "depth": sc["depth0"], "image": img},
                "view1": {"camera": synthetic.PinholeCamera(sc["K1"]), "depth": sc["depth1"], "image": img},
                "T_0to1": synthetic.RigidPose(sc["R"], sc["t"])}
        assert torch.equal(data["lines0"].cpu(), torch.from_numpy(g[f"{tag}|lines0"]))
        _check_labels(DepthMatcher(conf)(data), g, tag)
    torch.cuda.synchronize()


@pytest.mark.parametrize("name,depth", [("gt_lines_homography", False), ("gt_lines_pose_depth", True)])
def test_label_pass_reproduces_reference_cost_matrix(name, depth):
    """The label pass alone, fed the reference's own projected points and masks."""
    g, tags = _load(name)
    for tag in tags:
        B, L0, L1, seed, h, w, conf = _meta(g, tag)
        segs = [ops.line_segments(_t(g, tag, f"lines{i}"), h, w) for i in "01"]
        masks = [_t(g, tag, k) for k in ("visible0", "visible1", "valid_pts0", "valid_pts1")] if depth else [None] * 4
        r = ops.gt_line_matches_from_projection(
            segs[0], segs[1], _t(g, tag, "pts0_1"), _t(g, tag, "pts1_0"), (h, w), (h, w), _t(g, tag, "valid_lines0"),
            _t(g, tag, "valid_lines1"), *masks, npts=conf["n_line_sampled_pts"], dist_th=conf["line_perp_dist_th"],
            overlap_th=conf["overlap_th"], min_visibility_th=conf["min_visibility_th"], return_cost=True)
        assert np.array_equal(r["cost"].cpu().numpy(), g[f"{tag}|cost"].astype(np.float64)), tag
        _check_labels(r, g, tag)


def _check_solver(C, r2c, c2r, rows, cols):
    R, Cn = C.shape
    want_r2c = np.full(R, -1)
    want_r2c[rows] = cols
    want_c2r = np.full(Cn, -1)
    want_c2r[cols] = rows
    assert np.array_equal(r2c, want_r2c) and np.array_equal(c2r, want_c2r)


def test_device_solver_equals_reference_assignments():
    for name in ("gt_lines_homography", "gt_lines_pose_depth"):
        g, tags = _load(name)
        for tag in tags:
            cost = torch.from_numpy(g[f"{tag}|cost"]).double().to(DEV)
            r2c, c2r = ops.linear_sum_assignment(cost)
            for b in range(cost.shape[0]):
                _check_solver(g[f"{tag}|cost"][b], r2c[b].cpu().numpy(), c2r[b].cpu().numpy(),
                              g[f"{tag}|assign_rows"][b], g[f"{tag}|assign_cols"][b])


@pytest.mark.parametrize("nr,nc", [(1, 1), (7, 13), (13, 7), (64, 64), (250, 250), (300, 512), (512, 300), (512, 512)])
def test_device_solver_equals_restatement(nr, nc):
    rs = np.random.RandomState(nr * 1000 + nc)
    B = 3
    Cs = np.stack([tie_heavy_costs(rs, nr, nc) for _ in range(B)])
    if nr >= 250:  # line-cost shaped: sparse products of two counts
        Cs = np.where(Cs < 1e6, -rs.randint(0, 51, size=Cs.shape) * rs.randint(0, 51, size=Cs.shape)
                      * (rs.uniform(size=Cs.shape) < 0.02), Cs)
    r2c, c2r = ops.linear_sum_assignment(torch.from_numpy(Cs).to(DEV))
    for b in range(B):
        rows, cols = O.linear_sum_assignment(Cs[b])
        _check_solver(Cs[b], r2c[b].cpu().numpy(), c2r[b].cpu().numpy(), rows, cols)


@pytest.mark.parametrize("L0,L1", [(512, 470), (430, 512)])
def test_labels_at_512_lines_equal_oracle(L0, L1):
    from gluefactory_b200.geometry import inv3x3, warp_points

    B, npts, h, w = 8, 50, 480, 640
    sc = synthetic.to_device(synthetic.line_gt_scene("homography", B, L0, L1, 300 + L0), DEV)
    r = ops.gt_line_matches_from_homography(sc["lines0"], sc["lines1"], sc["valid_lines0"], sc["valid_lines1"],
                                            (h, w), (h, w), sc["H_0to1"], npts=npts, min_visibility_th=0.5)
    segs = [ops.line_segments(sc[f"lines{i}"], h, w) for i in "01"]
    p01 = warp_points(ops.sample_line_points(segs[0], npts), sc["H_0to1"])
    p10 = warp_points(ops.sample_line_points(segs[1], npts), inv3x3(sc["H_0to1"]))
    cpu = lambda t: t.cpu()  # noqa: E731
    ref = O.line_labels(cpu(segs[0]), cpu(segs[1]), cpu(p01), cpu(p10), (h, w), (h, w), cpu(sc["valid_lines0"]),
                        cpu(sc["valid_lines1"]), npts=npts, min_visibility_th=0.5)
    assert torch.equal(r["line_matches0"].cpu(), ref["m0"]) and torch.equal(r["line_matches1"].cpu(), ref["m1"])
    assert torch.equal(r["line_assignment"].cpu(), ref["positive"])
    assert int(ref["positive"].sum()) > 100
    # the device sampling equals the restated sample_pts
    assert torch.equal(ops.sample_line_points(segs[0], npts).cpu(), O.sample_pts(cpu(segs[0]), npts).reshape(B, -1, 2))


def _gluestick_batch(B, N, L, seed):
    d = synthetic.make_gluestick_batch(B, N, L, seed)
    for i in "01":
        d[f"valid_lines{i}"] = torch.ones(B, L, dtype=torch.bool)
        d[f"view{i}"]["image"] = torch.zeros(B, 1, 1024, 1024)
    return d


def test_gluestick_step_with_device_line_labels_replays_as_one_cuda_graph():
    from gluefactory_b200.matchers.gluestick import GlueStick
    from gluefactory_b200.matchers.homography_matcher import HomographyMatcher
    from gluefactory_b200.trainer import MatcherTrainer

    conf = {"GNN_layers": ["self", "cross"] * 2, "filter_threshold": 0.2}

    def build():
        model = GlueStick(dict(conf, precision="bf16"))
        model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=31), strict=True)
        return model.to(DEV).train()

    data = synthetic.to_device(_gluestick_batch(2, 160, 24, 32), DEV)
    gt = HomographyMatcher({"use_lines": True, "th_positive": 3.0, "th_negative": 3.0})
    labels = gt(data)
    assert {"line_matches0", "line_matches1", "line_assignment", "matches0", "assignment"} <= set(labels)
    eager = MatcherTrainer(build(), lr=1e-4, ground_truth=gt)
    graphed = MatcherTrainer(build(), lr=1e-4, ground_truth=gt)
    graphed.capture(data, torch.device(DEV))
    for it in range(3):
        le, _ = eager.step(data)
        lg, _ = graphed.step_graphed(data)
        assert torch.isfinite(lg).all()
        assert abs(le.item() - lg.item()) < (1e-5 if it == 0 else 2e-3) * abs(le.item()), (it, le.item(), lg.item())


def test_gluestick_with_depth_line_ground_truth_trains():
    """Pipeline-shaped run as in the MegaDepth GlueStick config: ground_truth = depth_matcher with use_lines."""
    from gluefactory_b200.matchers.depth_matcher import DepthMatcher
    from gluefactory_b200.matchers.gluestick import GlueStick

    B, N, L, h, w = 2, 256, 32, 480, 640
    d = synthetic.make_gluestick_batch(B, N, L, 61)
    for k in ("keypoints0", "keypoints1", "lines0", "lines1"):
        d[k] = d[k] * 0.45  # into the 640 x 480 views
    sc = synthetic.pose_depth_scene(B, 1, 1, 62, W=w, H=h)
    for i in "01":
        d[f"view{i}"] = {"image_size": torch.tensor([[w, h]] * B, dtype=torch.float32), "image": torch.zeros(B, 1, h, w),
                         "camera": synthetic.PinholeCamera(sc[f"K{i}"]), "depth": sc[f"depth{i}"]}
        d[f"valid_lines{i}"] = torch.ones(B, L, dtype=torch.bool)
    d["T_0to1"] = synthetic.RigidPose(sc["R"], sc["t"])
    data = {k: (synthetic.to_device(v, DEV) if not k.startswith("view") else
                {kk: (vv.to(DEV) if hasattr(vv, "to") else vv) for kk, vv in v.items()}) for k, v in d.items()
            if not k.startswith("gt_") and k != "T_0to1"}
    data["T_0to1"] = d["T_0to1"].to(DEV)
    gt = DepthMatcher({"use_lines": True, "th_positive": 3.0, "th_negative": 5.0})
    data.update({f"gt_{k}": v for k, v in gt(data).items()})
    assert data["gt_line_matches0"].shape == (B, L) and data["gt_line_assignment"].shape == (B, L, L)
    model = GlueStick({"GNN_layers": ["self", "cross"] * 2, "precision": "bf16"})
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=63), strict=True)
    model = model.to(DEV).train()
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()
    assert torch.isfinite(losses["total"]).all() and torch.isfinite(losses["line_assignment_nll"]).all()
    assert all(p.grad is None or torch.isfinite(p.grad).all() for p in model.parameters())
