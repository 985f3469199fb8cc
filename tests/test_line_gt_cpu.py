"""CPU: the line ground-truth oracle (oracle/line_gt_oracle.py) against the reference's own labels
(tests/golden/gt_lines_*.npz) and against scipy's linear_sum_assignment; the ground-truth components' conf and
required keys with and without `use_lines`."""
import os

import numpy as np
import pytest
import torch

from oracle import line_gt_oracle as O
from tests.util import GOLDEN


def _case(g, tag, depth):
    B, L0, L1, seed, npts, dist, ov, mvt, h, w = g[f"{tag}|meta"]
    B, L0, L1, npts, h, w = int(B), int(L0), int(L1), int(npts), int(h), int(w)
    t = lambda k: torch.from_numpy(g[f"{tag}|{k}"])  # noqa: E731
    from gluefactory_b200 import ops

    segs = [ops.line_segments(t(f"lines{i}"), h, w) for i in "01"]  # clamping runs in torch: any device
    masks = {k: t(k) for k in ("visible0", "visible1", "valid_pts0", "valid_pts1")} if depth else {}
    return O.line_labels(segs[0], segs[1], t("pts0_1"), t("pts1_0"), (h, w), (h, w), t("valid_lines0"),
                         t("valid_lines1"), npts=npts, dist_th=float(dist), overlap_th=float(ov),
                         min_visibility_th=float(mvt), **masks)


@pytest.mark.parametrize("name,depth", [("gt_lines_homography", False), ("gt_lines_pose_depth", True)])
def test_oracle_reproduces_reference_line_labels(name, depth):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    tags = sorted({k.split("|")[0] for k in g})
    for tag in tags:
        r = _case(g, tag, depth)
        assert np.array_equal(r["cost"].numpy(), g[f"{tag}|cost"]), tag
        assert np.array_equal(r["positive"].nonzero().numpy(), g[f"{tag}|positives"]), tag
        assert np.array_equal(r["m0"].numpy(), g[f"{tag}|matches0"]), tag
        assert np.array_equal(r["m1"].numpy(), g[f"{tag}|matches1"]), tag
        for b, (rows, cols) in enumerate(r["assignment"]):
            assert np.array_equal(rows.numpy(), g[f"{tag}|assign_rows"][b])
            assert np.array_equal(cols.numpy(), g[f"{tag}|assign_cols"][b])
        assert int(r["positive"].sum()) > 0 and (r["m0"] == -2).any() and (r["m0"] == -1).any()


def tie_heavy_costs(rs, nr, nc):
    """Small integer costs (many ties), some rows / columns at 1e6, like the line costs."""
    C = -rs.randint(0, 4, size=(nr, nc)).astype(np.float64) * rs.randint(0, 3, size=(nr, nc))
    C[rs.uniform(size=nr) < 0.2] = 1e6
    C[:, rs.uniform(size=nc) < 0.2] = 1e6
    return C


def test_numpy_assignment_equals_scipy():
    scipy_opt = pytest.importorskip("scipy.optimize")
    rs = np.random.RandomState(7)
    for it in range(300):
        nr, nc = rs.randint(1, 14, size=2)
        C = tie_heavy_costs(rs, nr, nc)
        ref = scipy_opt.linear_sum_assignment(C)
        got = O.linear_sum_assignment(C)
        assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1]), (it, C)
    for nr, nc in ((60, 60), (45, 70), (70, 45)):
        C = -rs.randint(0, 30, size=(nr, nc)).astype(np.float64) * (rs.uniform(size=(nr, nc)) < 0.1)
        ref, got = scipy_opt.linear_sum_assignment(C), O.linear_sum_assignment(C)
        assert np.array_equal(ref[0], got[0]) and np.array_equal(ref[1], got[1])


@pytest.mark.parametrize("module,cls", [("homography_matcher", "HomographyMatcher"), ("depth_matcher", "DepthMatcher")])
def test_components_line_keys(module, cls):
    import importlib

    M = getattr(importlib.import_module(f"gluefactory_b200.matchers.{module}"), cls)
    base = M({})
    assert not base.conf.use_lines and base.conf.n_line_sampled_pts == 50 and base.conf.line_perp_dist_th == 5
    assert base.conf.overlap_th == 0.2 and base.conf.min_visibility_th == 0.5
    assert not {"lines0", "lines1", "valid_lines0", "valid_lines1"} & set(base.required_data_keys)
    lines = M({"use_lines": True})
    assert set(lines.required_data_keys) == set(base.required_data_keys) | {"lines0", "lines1", "valid_lines0",
                                                                             "valid_lines1"}
    assert M.required_data_keys == (["H_0to1"] if module == "homography_matcher" else ["view0", "view1", "T_0to1"])


def test_empty_line_sets_are_rejected():
    from gluefactory_b200 import ops

    with pytest.raises(ValueError):
        ops.line_segments(torch.zeros(1, 0, 2, 2), 480, 640)
