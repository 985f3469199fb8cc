"""CPU: the point-label restatement (tests/gt_points_oracle.py) reproduces the labels the unmodified reference
produced (tests/golden/gt_pose_depth*.npz: inputs of the O(M N) pass and its outputs), which is what licenses using it
as the reference of the GPU tests at sizes where no golden file exists; and its explicit tie rule is torch's CPU `min`."""
import os

import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.depth_matcher import _skew
from tests import gt_points_oracle as P
from tests.util import GOLDEN


def _scenes(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    return [(g, tag) for tag in sorted({k.split("|")[0] for k in g})]


SCENES = _scenes("gt_pose_depth") + _scenes("gt_pose_depth_masks")


def fundamental(sc):
    """F = K1^-T [t]x R K0^-1 in fp32, as DepthMatcher builds it."""
    return torch.inverse(sc["K1"]).transpose(-1, -2) @ (_skew(sc["t"]) @ sc["R"]) @ torch.inverse(sc["K0"])


def _labels(g, tag):
    B, M, N, seed, epi, cc = g[f"{tag}|meta"]
    sc = synthetic.pose_depth_scene(int(B), int(M), int(N), int(seed))  # K, R, t and keypoints; depth enters via the masks
    t = lambda k: torch.from_numpy(g[f"{tag}|{k}"])  # noqa: E731
    asg, m0, m1 = P.labels_from_reprojection(sc["kp0"], sc["kp1"], t("proj_0to1"), t("proj_1to0"), t("visible0"),
                                             t("visible1"), t("valid0"), t("valid1"), 3.0, 5.0)
    stats = {}
    if epi >= 0:
        dist = P.epipolar_distance_all(sc["kp0"], sc["kp1"], fundamental(sc))
        cand0 = (m0 == -2) & ~t("valid0")
        cand1 = (m1 == -2) & ~t("valid1")
        m0, m1, min0, min1 = P.epipolar_unmatched(m0, m1, t("valid0"), t("valid1"), dist, 5.0)
        mins = torch.cat([min0[cand0], min1[cand1]])
        stats = {"candidates": mins.numel(), "no_partner": int(torch.isinf(mins).sum()),
                 "excluded": int((mins > 5.0).sum()), "kept": int((mins <= 5.0).sum()),
                 "margin": float((mins[torch.isfinite(mins)] - 5.0).abs().min()) if torch.isfinite(mins).any() else 0.0}
    return asg, m0, m1, stats


@pytest.mark.parametrize("g,tag", SCENES, ids=[t for _, t in SCENES])
def test_restatement_reproduces_reference_labels(g, tag):
    asg, m0, m1, _ = _labels(g, tag)
    assert np.array_equal(m0.numpy(), g[f"{tag}|matches0"])
    assert np.array_equal(m1.numpy(), g[f"{tag}|matches1"])
    assert np.array_equal(asg.nonzero().numpy(), g[f"{tag}|positives"])


def test_golden_scenes_exercise_every_branch_of_the_epipolar_step():
    """Between them the stored scenes have candidates that are excluded, candidates that are kept, and candidates with
    no still-ignored partner at all; none of them sits within 1e-3 px of the threshold, so the fp64 evaluation and the
    reference's fp32 one cannot disagree on it."""
    tot = {"candidates": 0, "no_partner": 0, "excluded": 0, "kept": 0}
    for g, tag in SCENES:
        stats = _labels(g, tag)[3]
        if stats:
            assert stats["margin"] > 1e-3, (tag, stats)
            for k in tot:
                tot[k] += stats[k]
    assert tot["candidates"] > 100 and tot["excluded"] > tot["no_partner"] > 0 and tot["kept"] > 0, tot


def test_unmasked_restatement_equals_the_homography_restatement():
    from gluefactory_b200.geometry import warp_points

    d = synthetic.make_pairs(2, 333, seed=5, M=260, with_gt=False)
    kp0, kp1, H = d["keypoints0"], d["keypoints1"], d["H_0to1"]
    want = synthetic.gt_matches_from_homography(kp0, kp1, H, 3.0, 5.0)
    got = P.labels_from_reprojection(kp0, kp1, warp_points(kp0, H), warp_points(kp1, torch.inverse(H)), pos_th=3.0,
                                     neg_th=5.0)
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    assert int(got[0].sum()) > 50


def test_tie_rule_is_cpu_min():
    """Lowest index among equal values, duplicates, all-inf slices and NaN (first NaN) included."""
    gen = torch.Generator().manual_seed(0)
    d = torch.randint(0, 6, (64, 97), generator=gen).float()  # few distinct values: every row and column ties
    d[3] = float("inf")
    d[:, 11] = float("inf")
    d[5, 40] = d[5, 70] = float("nan")
    d[9, 0] = float("-inf")
    d[9, 50] = float("nan")
    for dim in (0, 1):
        assert torch.equal(P.first_min_index(d, dim), d.min(dim).indices)
    assert int((d == d.min(1, keepdim=True).values).sum(1).max()) > 5


def test_epipolar_distance_is_the_point_line_distance():
    """On a rectified pair (pure x translation, identity K) the epipolar line of (x, y) is the row y of the other
    view, so the symmetric distance is |y1 - y0| for every pair."""
    t = torch.tensor([[1.0, 0.0, 0.0]])
    F = _skew(t) @ torch.eye(3)[None]
    kp0, kp1 = torch.rand(1, 7, 2, generator=torch.Generator().manual_seed(1)) * 100, torch.rand(1, 5, 2) * 100
    dist = P.epipolar_distance_all(kp0, kp1, F)
    want = (kp0[:, :, None, 1] - kp1[:, None, :, 1]).abs().double()
    assert torch.allclose(dist, want, atol=1e-9)
