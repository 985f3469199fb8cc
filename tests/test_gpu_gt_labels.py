"""GPU: the ground-truth label kernels in the pose + depth configuration (csrc/gt.cu with visibility / validity masks,
its epipolar exclusion, and the depth variant of csrc/gt_lines.cu) against plain restatements of the same operations
(tests/gt_points_oracle.py, oracle/line_gt_oracle.py) at training sizes and at the edges of their launch shapes.

Labels are integers, so every comparison is exact, with one exception.  The epipolar distance of the kernel is a
plain fp32 expression that is not bit-identical to any torch one; a label of the exclusion pass may differ from the
fp64 restatement only where the fp64 minimum distance of that point lies within 1e-3 * th of th (5e-3 px at th = 5).
For scale: an fp32 evaluation of the same distances in torch differs from fp64 by up to 1.3e-3 px within 1 px of the
threshold in these scenes (640 x 480 views; each case records its own figure, see profiles/gt_label_tests_h100.md).
The number of points inside the band is recorded per case and bounded by 0.1 % of the points, so the band cannot
hide a wrong kernel.

Masks are drawn here, so that the shapes of invisibility are controlled: whole 64-row strips, whole columns, one lane's
columns, a whole batch element.  Failures name batch element, index, expected and got for the first mismatches."""
import functools

import pytest
import torch

from gluefactory_b200 import ops, synthetic
from gluefactory_b200.geometry import inv3x3, warp_points
from gluefactory_b200.matchers.depth_matcher import DepthMatcher, _skew, project, sample_depth
from oracle import line_gt_oracle as O
from tests import gt_points_oracle as P
from tests.util import report

pytestmark = pytest.mark.gpu
DEV = "cuda"


def assert_same(name, got, want, allowed=None):
    """Exact equality; `allowed` (bool, same shape) marks entries that may differ.  -> number of differing entries."""
    assert got.shape == want.shape and got.dtype == want.dtype, (name, got.shape, want.shape, got.dtype, want.dtype)
    diff = got != want
    bad = diff if allowed is None else diff & ~allowed
    if bool(bad.any()):
        first = bad.nonzero()[:5].tolist()
        rows = [f"batch {i[0]} index {tuple(i[1:])}: expected {want[tuple(i)].item()} got {got[tuple(i)].item()}" for i in first]
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.numel()} entries differ; " + "; ".join(rows))
    return int(diff.sum())


def _gen(seed):
    return torch.Generator().manual_seed(seed)


def _rand(shape, seed):
    return torch.rand(shape, generator=_gen(seed)).to(DEV)


# ---------------------------------------------------------------------------------------------------------------------
# masked point labels, kernel level
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=4)
def _points(B, M, N):
    """Keypoints of both views and their reprojections: 40 % of the view-1 points are view-0 points warped by a
    homography plus 0.5 px noise, the rest uniform in a 1024 x 1024 image."""
    d = synthetic.to_device(synthetic.make_pairs(B, N, seed=500 + B + M + N, D=4, M=M, with_gt=False), DEV)
    kp0, kp1, H = d["keypoints0"], d["keypoints1"], d["H_0to1"]
    return kp0, kp1, warp_points(kp0, H).contiguous(), warp_points(kp1, inv3x3(H)).contiguous()


PATTERNS = ["half", "all", "batch0_none", "strip1", "strip0", "lane5", "cols256", "superset", "valid_none"]


def _masks(pattern, B, M, N, seed=7):
    """visible0 [B,M], visible1 [B,N], valid0, valid1 (bool).  valid is a strict superset of visible (valid depth, but
    projected outside or inconsistent) except in "all" and "valid_none"."""
    dens = 0.5 if pattern in ("half", "valid_none", "superset") else 0.8
    v0, v1 = _rand((B, M), seed) < dens, _rand((B, N), seed + 1) < dens
    if pattern == "all":
        v0, v1 = torch.ones_like(v0), torch.ones_like(v1)
    elif pattern == "batch0_none":   # every row and column of one distance matrix is +inf
        v0[0], v1[0] = False, False
    elif pattern == "strip1":        # a whole 64-row strip of the scan kernel sees only +inf
        v0[:, 64:128] = False
    elif pattern == "strip0":        # the first finite strip of every column is not strip 0
        v0[:, :64] = False
    elif pattern == "lane5":         # one lane of the row pass sees only +inf
        v1[:, 5::32] = False
    elif pattern == "cols256":       # the first pass of the column loop sees only +inf
        v1[:, :256] = False
    val0, val1 = v0 | (_rand((B, M), seed + 2) < 0.5), v1 | (_rand((B, N), seed + 3) < 0.5)
    if pattern == "superset":        # much valid depth that is not visible
        val0, val1 = v0 | (_rand((B, M), seed + 2) < 0.9), v1 | (_rand((B, N), seed + 3) < 0.9)
    if pattern == "valid_none":
        val0, val1 = torch.zeros_like(v0), torch.zeros_like(v1)
    return v0, v1, val0, val1


def _check_point_labels(tag, pts, masks, pos_th, neg_th, dense=True):
    kp0, kp1, kp0_1, kp1_0 = pts
    r = ops.gt_matches_from_reprojection(kp0, kp1, kp0_1, kp1_0, *masks, pos_th=pos_th, neg_th=neg_th, dense=dense,
                                         dense_t=True)
    asg, m0, m1 = P.labels_from_reprojection(kp0, kp1, kp0_1, kp1_0, *masks, pos_th=pos_th, neg_th=neg_th)
    assert_same(tag + " matches0", r["matches0"], m0)
    assert_same(tag + " matches1", r["matches1"], m1)
    assert_same(tag + " assignment_t", r["assignment_t"], asg.transpose(1, 2))
    if dense:
        assert_same(tag + " assignment", r["assignment"], asg)
    else:
        assert "assignment" not in r
    # the labels are consistent with each other
    i = (m0 > -1).nonzero()
    assert bool((m1[i[:, 0], m0[m0 > -1]] == i[:, 1]).all()) and int(asg.sum()) == i.shape[0] == int((m1 > -1).sum())
    return asg, m0, m1


SHAPES = [(8, 2048, 2048), (3, 1000, 777), (2, 63, 31), (1, 1, 1), (1, 65, 257), (1, 5, 3000), (2, 2049, 2047)]


@pytest.mark.parametrize("pattern,pos_th,neg_th", [(p, 3.0, 5.0) for p in PATTERNS] + [("half", 3.0, 3.0), ("strip1", 3.0, 3.0)])
@pytest.mark.parametrize("B,M,N", SHAPES)
def test_masked_point_labels_equal_restatement(B, M, N, pattern, pos_th, neg_th):
    pts = _points(B, M, N)
    masks = _masks(pattern, B, M, N)
    tag = f"{B}x{M}x{N} {pattern} th=({pos_th},{neg_th})"
    asg, m0, m1 = _check_point_labels(tag, pts, masks, pos_th, neg_th)
    plain = ops.gt_matches_from_reprojection(*pts, pos_th=pos_th, neg_th=neg_th)
    if pattern == "all":  # all-true masks change nothing, bit for bit
        for k, v in (("matches0", m0), ("matches1", m1), ("assignment", asg)):
            assert_same(tag + " unmasked " + k, plain[k], v)
    elif min(M, N) >= 256:  # the scenario is not vacuous: every kind of label occurs and the masks matter
        npos, nun, nign = int(asg.sum()), int((m0 == -1).sum()), int((m0 == -2).sum())
        assert not torch.equal(plain["matches0"], m0) and not torch.equal(plain["matches1"], m1)
        assert int(plain["assignment"].sum()) > npos > 0 and nign > 0, (npos, nign)
        if pattern == "valid_none":
            assert nun == 0 and int((m1 == -1).sum()) == 0
        else:
            assert nun > 0 and int((m1 == -1).sum()) > 0
        if pattern == "batch0_none":
            assert int(asg[0].sum()) == 0 and int((m0[0] > -1).sum()) == 0
        if pattern == "superset":  # valid and visible differ on many points, and some of those are unmatched
            assert int(((m0 == -1) & ~masks[0]).sum()) > 0 and int(((m1 == -1) & ~masks[1]).sum()) > 0
    if pattern == "valid_none":
        assert int((m0 == -1).sum()) == 0 and int((m1 == -1).sum()) == 0


def test_masked_point_labels_sparse_outputs_at_batch_32():
    """The layout the matcher's loss asks for (no dense [B,M,N] mask, only its transpose) at the benchmark's batch."""
    B, M, N = 32, 2048, 2048
    asg, m0, _ = _check_point_labels("32x2048x2048 sparse", _points(B, M, N), _masks("half", B, M, N), 3.0, 5.0, dense=False)
    assert int(asg.sum()) > 32 * 50 and int((m0 == -1).sum()) > 0 and int((m0 == -2).sum()) > 0
    _points.cache_clear()


def _tie_points(B, M, N, seed):
    """Exact ties: a subset of pairs at distance 0 both ways, then 10 % of the points of each view overwritten with
    copies of other points of that view (reprojection included), so rows and columns hold equal minima at different
    indices, across lanes (any two columns) and across strips (rows more than 64 apart)."""
    kp0, kp1, kp0_1, kp1_0 = (t.clone() for t in _points(B, M, N))
    g = _gen(seed)
    S = min(M, N) // 5
    for b in range(B):
        i, j = torch.randperm(M, generator=g)[:S].to(DEV), torch.randperm(N, generator=g)[:S].to(DEV)
        kp0_1[b, i], kp1_0[b, j] = kp1[b, j], kp0[b, i]
        for kp, proj, n in ((kp1, kp1_0, N), (kp0, kp0_1, M)):
            dst = torch.randperm(n, generator=g)[:n // 10].to(DEV)
            src = torch.randint(0, n, (n // 10,), generator=g).to(DEV)
            kp[b, dst], proj[b, dst] = kp[b, src].clone(), proj[b, src].clone()
    return kp0, kp1, kp0_1, kp1_0


@pytest.mark.parametrize("masked", [False, True])
@pytest.mark.parametrize("B,M,N", [(2, 2048, 2048), (3, 1000, 777), (2, 63, 31)])
def test_point_labels_with_exact_ties(B, M, N, masked):
    pts = _tie_points(B, M, N, seed=B + M)
    masks = _masks("half", B, M, N, seed=11) if masked else (None,) * 4
    kp0, kp1, kp0_1, kp1_0 = pts
    d = torch.max(((kp0_1[0, :, None] - kp1[0, None]) ** 2).sum(-1), ((kp0[0, :, None] - kp1_0[0, None]) ** 2).sum(-1))
    tied_rows = int(((d == d.min(1, keepdim=True).values).sum(1) > 1).sum())
    tied_cols = int(((d == d.min(0, keepdim=True).values).sum(0) > 1).sum())
    assert tied_rows > M // 50 and tied_cols > N // 50, (tied_rows, tied_cols)
    asg, m0, m1 = _check_point_labels(f"ties {B}x{M}x{N} masked={masked}", pts, masks, 3.0, 5.0)
    if min(M, N) >= 256:
        assert int(asg.sum()) > 0 and int((m0 == -2).sum()) > 0


@pytest.mark.parametrize("masked", [False, True])
def test_point_labels_at_exact_thresholds(masked):
    """Reprojection errors that equal a threshold exactly (integer offsets, so the squared distances are exact):
    3 px is not a positive at th_positive 3 (`<`), 5 px is not unmatched at th_negative 5 (`>`)."""
    offs = torch.tensor([[0.0, 0.0], [2.0, 2.0], [3.0, 0.0], [3.0, 4.0], [4.0, 4.0], [0.0, 5.0]], device=DEV)
    B, M = 2, 600
    i = torch.arange(M, device=DEV)
    kp0 = torch.stack([100.0 * (i % 30), 100.0 * (i // 30)], -1).expand(B, M, 2).contiguous()
    kp1 = kp0 + 1000.0                      # view 1 is view 0 shifted; point i reprojects off[i % 6] away from its partner
    off = offs[i % 6]
    kp0_1, kp1_0 = kp1 + off, kp0 + off
    masks = (torch.ones(B, M, dtype=torch.bool, device=DEV),) * 4 if masked else (None,) * 4
    asg, m0, m1 = _check_point_labels(f"exact thresholds masked={masked}", (kp0, kp1, kp0_1, kp1_0), masks, 3.0, 5.0)
    want = torch.where(i % 6 < 2, i, torch.where(i % 6 == 4, torch.full_like(i, -1), torch.full_like(i, -2)))
    assert_same("exact thresholds: expected labels", m0, want.expand(B, M))
    assert_same("exact thresholds: expected labels", m1, want.expand(B, M))


# ---------------------------------------------------------------------------------------------------------------------
# epipolar exclusion
# ---------------------------------------------------------------------------------------------------------------------
def _fundamental(sc):
    """F = K1^-T [t]x R K0^-1 in fp32, as DepthMatcher builds it; one per batch element."""
    return torch.inverse(sc["K1"]).transpose(-1, -2) @ (_skew(sc["t"]) @ sc["R"]) @ torch.inverse(sc["K0"])


def _check_epipolar(tag, got0, got1, m0, m1, valid0, valid1, kp0, kp1, F, th):
    """got0 / got1: labels after the device pass on (m0, m1).  Exact against the fp64 restatement outside the band
    |min distance - th| <= 1e-3 th; labels that are not candidates never change.  -> restated labels."""
    F = F.float()
    epi = P.epipolar_distance_all(kp0, kp1, F, torch.float64)
    want0, want1, min0, min1 = P.epipolar_unmatched(m0, m1, valid0, valid1, epi, th)
    cand0, cand1 = (m0 == -2) & ~valid0, (m1 == -2) & ~valid1
    band0, band1 = cand0 & ((min0 - th).abs() <= 1e-3 * th), cand1 & ((min1 - th).abs() <= 1e-3 * th)
    flips = assert_same(tag + " matches0", got0, want0, band0) + assert_same(tag + " matches1", got1, want1, band1)
    assert_same(tag + " non-candidates of view 0", got0[~cand0][None], m0[~cand0][None])
    assert_same(tag + " non-candidates of view 1", got1[~cand1][None], m1[~cand1][None])
    in_band, total = int(band0.sum() + band1.sum()), m0.numel() + m1.numel()
    e32 = P.epipolar_distance_all(kp0, kp1, F, torch.float32)
    near = (epi - th).abs() < 1.0
    err32 = float((e32.double() - epi)[near].abs().max()) if bool(near.any()) else 0.0
    report("gt_epipolar " + tag, points=total, candidates=int(cand0.sum() + cand1.sum()),
           excluded=int((want0 != m0).sum() + (want1 != m1).sum()), in_band=in_band, flips_in_band=flips,
           torch_fp32_vs_fp64_px=err32)
    assert in_band <= 1e-3 * total, (tag, in_band, total)
    assert err32 < 1e-3 * th, (tag, err32)
    return want0, want1, cand0, cand1, min0, min1


def _epi_scene(B, M, N, no_depth, seed):
    """Scene keypoints, reprojections through the scene's depth, and drawn validity: a share `no_depth` of the points
    of each view has no valid depth (and so is not visible).  Labels before the pass come from the restatement."""
    sc = synthetic.to_device(synthetic.pose_depth_scene(B, M, N, seed), DEV)
    cam0, cam1, T = synthetic.PinholeCamera(sc["K0"]), synthetic.PinholeCamera(sc["K1"]), synthetic.RigidPose(sc["R"], sc["t"])
    d0, val0 = sample_depth(sc["kp0"], sc["depth0"])
    d1, val1 = sample_depth(sc["kp1"], sc["depth1"])
    val0, val1 = val0 & (_rand((B, M), seed + 1) >= no_depth), val1 & (_rand((B, N), seed + 2) >= no_depth)
    kp0_1, vis0 = project(sc["kp0"], d0, sc["depth1"], cam0, cam1, T, val0)
    kp1_0, vis1 = project(sc["kp1"], d1, sc["depth0"], cam1, cam0, T.inv(), val1)
    _, m0, m1 = P.labels_from_reprojection(sc["kp0"], sc["kp1"], kp0_1, kp1_0, vis0, vis1, val0, val1, 3.0, 5.0)
    return sc, m0, m1, val0, val1


@pytest.mark.parametrize("no_depth", [0.05, 0.5, 1.0])
@pytest.mark.parametrize("B,M,N", [(8, 2048, 2048), (3, 1000, 777), (2, 3, 2), (1, 2047, 2046)])
def test_epipolar_exclusion_equals_restatement(B, M, N, no_depth):
    sc, m0, m1, val0, val1 = _epi_scene(B, M, N, no_depth, seed=90 + B)
    F = _fundamental(sc)
    assert B == 1 or not torch.equal(F[0], F[1])
    got0, got1 = m0.clone(), m1.clone()
    ops.gt_epipolar_unmatched_(sc["kp0"], sc["kp1"], F, val0, val1, got0, got1, 5.0)
    want0, want1, cand0, cand1, _, _ = _check_epipolar(f"{B}x{M}x{N} no_depth={no_depth}", got0, got1, m0, m1, val0, val1,
                                                       sc["kp0"], sc["kp1"], F, 5.0)
    if M >= 1000:  # not vacuous: candidates on both sides, some excluded and some kept
        excluded = int((want0 != m0).sum() + (want1 != m1).sum())
        assert min(int(cand0.sum()), int(cand1.sum())) > 20 and 0 < excluded < int(cand0.sum() + cand1.sum())


@pytest.mark.parametrize("B,M,N", [(8, 2048, 2048), (2, 63, 31)])
def test_epipolar_exclusion_without_partners_and_without_candidates(B, M, N):
    sc, m0, m1, val0, val1 = _epi_scene(B, M, N, 0.5, seed=97)
    F = _fundamental(sc)
    # no point of view 1 is still ignored: every candidate of view 0 becomes unmatched, view 1 keeps its labels
    m1 = torch.where(m1 == -2, torch.full_like(m1, -1), m1)
    got0, got1 = m0.clone(), m1.clone()
    ops.gt_epipolar_unmatched_(sc["kp0"], sc["kp1"], F, val0, val1, got0, got1, 5.0)
    cand0 = (m0 == -2) & ~val0
    assert int(cand0.sum()) > 0
    assert_same("no partner: matches0", got0, torch.where(cand0, torch.full_like(m0, -1), m0))
    assert_same("no partner: matches1", got1, m1)
    # every point has valid depth: no candidates, nothing changes
    sc, m0, m1, _, _ = _epi_scene(B, M, N, 0.5, seed=98)
    got0, got1 = m0.clone(), m1.clone()
    ops.gt_epipolar_unmatched_(sc["kp0"], sc["kp1"], F, torch.ones_like(m0, dtype=torch.bool),
                               torch.ones_like(m1, dtype=torch.bool), got0, got1, 5.0)
    assert int((m0 == -2).sum()) > 0
    assert_same("no candidates: matches0", got0, m0)
    assert_same("no candidates: matches1", got1, m1)


# ---------------------------------------------------------------------------------------------------------------------
# through the component
# ---------------------------------------------------------------------------------------------------------------------
def _component_data(sc):
    B = sc["kp0"].shape[0]
    img = torch.zeros(B, 1, *sc["depth0"].shape[-2:], device=DEV)
    return {"keypoints0": sc["kp0"], "keypoints1": sc["kp1"],
            "view0": {"camera": synthetic.PinholeCamera(sc["K0"]), "depth": sc["depth0"], "image": img},
            "view1": {"camera": synthetic.PinholeCamera(sc["K1"]), "depth": sc["depth1"], "image": img},
            "T_0to1": synthetic.RigidPose(sc["R"], sc["t"])}


def _zero_blocks(sc):
    sc["depth0"][:, :, 320:420] = 0.0
    sc["depth0"][:, 400:, :] = 0.0
    sc["depth1"][:, 240:300, :] = 0.0
    sc["depth1"][:, :, :120] = 0.0
    return sc


def _check_component_points(tag, pred, data, conf):
    kp0, kp1 = data["keypoints0"], data["keypoints1"]
    v0, v1, T = data["view0"], data["view1"], data["T_0to1"]
    d0, val0 = sample_depth(kp0, v0["depth"])
    d1, val1 = sample_depth(kp1, v1["depth"])
    kp0_1, vis0 = project(kp0, d0, v1["depth"], v0["camera"], v1["camera"], T, val0, ccth=conf["th_consistency"])
    kp1_0, vis1 = project(kp1, d1, v0["depth"], v1["camera"], v0["camera"], T.inv(), val1, ccth=conf["th_consistency"])
    assert torch.equal(pred["visible0"], vis0) and torch.equal(pred["visible1"], vis1)
    assert int((val0 & ~vis0).sum()) > 0 and int((~val0).sum()) > 0.2 * val0.numel()
    asg, m0, m1 = P.labels_from_reprojection(kp0, kp1, kp0_1, kp1_0, vis0, vis1, val0, val1, conf["th_positive"],
                                             conf["th_negative"])
    assert_same(tag + " assignment", pred["assignment"], asg)
    assert_same(tag + " assignment_t", pred["assignment_t"], asg.transpose(1, 2))
    if conf["th_epi"] is None:
        assert_same(tag + " matches0", pred["matches0"], m0)
        assert_same(tag + " matches1", pred["matches1"], m1)
    else:  # thresholded with th_negative, as in the reference
        F = torch.inverse(v1["camera"].calibration_matrix()).transpose(-1, -2) @ (_skew(T.t) @ T.R) @ torch.inverse(
            v0["camera"].calibration_matrix())
        want0, _, _, _, _, _ = _check_epipolar(tag, pred["matches0"], pred["matches1"], m0, m1, val0, val1, kp0, kp1, F,
                                               conf["th_negative"])
        assert int((want0 != m0).sum()) > 0
    assert int(asg.sum()) > 100 * asg.shape[0] and int((m0 == -1).sum()) > 0 and int((m0 == -2).sum()) > 0


@pytest.mark.parametrize("th_epi,th_consistency", [(None, None), (5.0, None), (5.0, 3.0), (None, 3.0)])
def test_depth_matcher_points_at_2048(th_epi, th_consistency):
    sc = _zero_blocks(synthetic.to_device(synthetic.pose_depth_scene(4, 2048, 2048, 120), DEV))
    conf = {"th_positive": 3.0, "th_negative": 5.0, "th_epi": th_epi, "th_consistency": th_consistency,
            "transposed_assignment": True}
    data = _component_data(sc)
    _check_component_points(f"component epi={th_epi} cc={th_consistency}", DepthMatcher(conf)(data), data, conf)


# ---------------------------------------------------------------------------------------------------------------------
# depth line labels
# ---------------------------------------------------------------------------------------------------------------------
def _line_inputs(sc, npts):
    """Segments, projected sample points and the four point masks, through the component's own geometry."""
    h, w = sc["depth0"].shape[-2:]
    segs0, segs1 = ops.line_segments(sc["lines0"], h, w), ops.line_segments(sc["lines1"], h, w)
    pts0, pts1 = ops.sample_line_points(segs0, npts), ops.sample_line_points(segs1, npts)
    d0, val0 = sample_depth(pts0, sc["depth0"])
    d1, val1 = sample_depth(pts1, sc["depth1"])
    cam0, cam1, T = synthetic.PinholeCamera(sc["K0"]), synthetic.PinholeCamera(sc["K1"]), synthetic.RigidPose(sc["R"], sc["t"])
    pts0_1, vis0 = project(pts0, d0, sc["depth1"], cam0, cam1, T, val0)
    pts1_0, vis1 = project(pts1, d1, sc["depth0"], cam1, cam0, T.inv(), val1)
    return segs0, segs1, pts0_1, pts1_0, vis0, vis1, val0, val1


def _draw_line_masks(vis, val, npts, seed):
    """30 % of the lines without any visible point, another 30 % with valid depth on about a third of their points
    (below a min_visibility_th of 0.5, around one of 0.2), and no visible point in the whole first batch element."""
    B, L = vis.shape[0], vis.shape[1] // npts
    u = _rand((B, L), seed)
    vis, val = vis.view(B, L, npts).clone(), val.view(B, L, npts).clone()
    vis[u < 0.3] = False
    few = (_rand((B, L, npts), seed + 1) < 0.3) & ((u >= 0.3) & (u < 0.6))[:, :, None]
    val = torch.where(((u >= 0.3) & (u < 0.6))[:, :, None], few, val)
    vis = vis & val
    vis[0] = False
    return vis.reshape(B, -1), val.reshape(B, -1)


def _check_line_labels(tag, sc, inputs, npts, mvt, size):
    segs0, segs1, pts0_1, pts1_0, vis0, vis1, val0, val1 = inputs
    r = ops.gt_line_matches_from_projection(segs0, segs1, pts0_1, pts1_0, size, size, sc["valid_lines0"],
                                            sc["valid_lines1"], vis0, vis1, val0, val1, npts=npts, dist_th=5,
                                            overlap_th=0.2, min_visibility_th=mvt, return_cost=True)
    cost = r["cost"].clone()
    ref = O.line_labels(*(t.cpu() for t in (segs0, segs1, pts0_1, pts1_0)), size, size, sc["valid_lines0"].cpu(),
                        sc["valid_lines1"].cpu(), *(t.cpu() for t in (vis0, vis1, val0, val1)), npts=npts, dist_th=5,
                        overlap_th=0.2, min_visibility_th=mvt)
    assert_same(tag + " cost", cost.cpu(), ref["cost"].double())
    assert_same(tag + " line_matches0", r["line_matches0"].cpu(), ref["m0"])
    assert_same(tag + " line_matches1", r["line_matches1"].cpu(), ref["m1"])
    assert_same(tag + " line_assignment", r["line_assignment"].cpu(), ref["positive"])
    return ref


@pytest.mark.parametrize("B,L0,L1,npts,mvt,drawn", [
    (8, 512, 512, 50, 0.5, False), (8, 512, 470, 50, 0.2, True), (8, 430, 512, 50, 0.5, True),
    (2, 17, 33, 50, 0.5, False), (2, 17, 33, 21, 0.2, True), (2, 1, 1, 50, 0.5, False)])
def test_depth_line_labels_equal_oracle(B, L0, L1, npts, mvt, drawn):
    sc = synthetic.to_device(synthetic.line_gt_scene("pose_depth", B, max(L0, 17), max(L1, 33), 700 + L0 + L1 + npts), DEV)
    for i, L in (("0", L0), ("1", L1)):  # the scene generator needs a handful of lines: L = 1 keeps its first one
        sc[f"lines{i}"], sc[f"valid_lines{i}"] = sc[f"lines{i}"][:, :L].contiguous(), sc[f"valid_lines{i}"][:, :L].contiguous()
    if L0 == 1:
        sc["valid_lines0"][:], sc["valid_lines1"][:] = True, True
    inputs = list(_line_inputs(sc, npts))
    if drawn:
        inputs[4], inputs[6] = _draw_line_masks(inputs[4], inputs[6], npts, seed=L0)
        inputs[5], inputs[7] = _draw_line_masks(inputs[5], inputs[7], npts, seed=L1 + 1)
    ref = _check_line_labels(f"lines {B}x{L0}x{L1} npts={npts} mvt={mvt} drawn={drawn}", sc, inputs, npts, mvt,
                             tuple(sc["depth0"].shape[-2:]))
    if L0 >= 430:  # not vacuous: positives, unmatched and ignored lines, and lines without a visible point
        nvis0 = inputs[4].view(B, L0, npts).sum(-1)
        assert int(ref["positive"].sum()) > 100 and int((ref["m0"] == -1).sum()) > 0 and int((ref["m0"] == -2).sum()) > B * L0 // 20
        assert int((nvis0 == 0).sum()) > 0 and int(((nvis0 > 0) & (nvis0 < npts)).sum()) > 0
        if drawn:
            assert int(ref["positive"][0].sum()) == 0 and int(ref["positive"][1:].sum()) > 100


def test_depth_matcher_points_and_lines_end_to_end():
    B, M, L = 2, 2048, 512
    sc = synthetic.to_device(synthetic.line_gt_scene("pose_depth", B, L, L, 801), DEV)
    # keypoints for the line scene's cameras: uniform in view 0; 45 % of view 1 are reprojections + 0.7 px noise
    h, w = sc["depth0"].shape[-2:]
    span = torch.tensor([w - 4.0, h - 4.0], device=DEV)
    kp0, kp1 = _rand((B, M, 2), 802) * span + 2, _rand((B, M, 2), 803) * span + 2
    d0, val0 = sample_depth(kp0, sc["depth0"])
    proj, ok = project(kp0, d0, None, synthetic.PinholeCamera(sc["K0"]), synthetic.PinholeCamera(sc["K1"]),
                       synthetic.RigidPose(sc["R"], sc["t"]), val0)
    proj = proj + 0.7 * torch.randn(B, M, 2, generator=_gen(804)).to(DEV)
    ok = ok & ((proj > 2) & (proj < span + 2)).all(-1) & (torch.arange(M, device=DEV) < int(0.45 * M))
    sc.update(kp0=kp0, kp1=torch.where(ok[..., None], proj, kp1))
    sc = _zero_blocks(sc)
    conf = {"th_positive": 3.0, "th_negative": 5.0, "th_epi": 5.0, "th_consistency": None, "transposed_assignment": True,
            "use_lines": True, "use_points": True}
    data = _component_data(sc)
    data.update({k: sc[k] for k in ("lines0", "lines1", "valid_lines0", "valid_lines1")})
    pred = DepthMatcher(conf)(data)
    _check_component_points("end to end", pred, data, conf)
    segs0, segs1, pts0_1, pts1_0, vis0, vis1, val0, val1 = _line_inputs(sc, 50)
    size = tuple(sc["depth0"].shape[-2:])
    ref = O.line_labels(*(t.cpu() for t in (segs0, segs1, pts0_1, pts1_0)), size, size, sc["valid_lines0"].cpu(),
                        sc["valid_lines1"].cpu(), *(t.cpu() for t in (vis0, vis1, val0, val1)), npts=50, dist_th=5,
                        overlap_th=0.2, min_visibility_th=0.5)
    assert_same("end to end line_matches0", pred["line_matches0"].cpu(), ref["m0"])
    assert_same("end to end line_matches1", pred["line_matches1"].cpu(), ref["m1"])
    assert_same("end to end line_assignment", pred["line_assignment"].cpu(), ref["positive"])
    assert int(ref["positive"].sum()) > 100


# ---------------------------------------------------------------------------------------------------------------------
# inside a CUDA graph
# ---------------------------------------------------------------------------------------------------------------------
def test_depth_label_kernels_replay_in_a_cuda_graph():
    """Point labels with masks, the epipolar pass and the depth line labels captured on fixed-address inputs, replayed
    after the inputs were overwritten in place with a second scene: the replay equals the eager result on that scene."""
    B, M, N, L0, L1, npts = 2, 500, 400, 40, 37, 50

    def scene(seed):
        sc, m0, m1, val0, val1 = _epi_scene(B, M, N, 0.4, seed)
        cam0, cam1, T = synthetic.PinholeCamera(sc["K0"]), synthetic.PinholeCamera(sc["K1"]), synthetic.RigidPose(sc["R"], sc["t"])
        d0, _ = sample_depth(sc["kp0"], sc["depth0"])
        d1, _ = sample_depth(sc["kp1"], sc["depth1"])
        kp0_1, vis0 = project(sc["kp0"], d0, sc["depth1"], cam0, cam1, T, val0)
        kp1_0, vis1 = project(sc["kp1"], d1, sc["depth0"], cam1, cam0, T.inv(), val1)
        ls = synthetic.to_device(synthetic.line_gt_scene("pose_depth", B, L0, L1, seed), DEV)
        return [sc["kp0"], sc["kp1"], kp0_1.contiguous(), kp1_0.contiguous(), vis0, vis1, val0, val1, _fundamental(sc),
                ls["valid_lines0"], ls["valid_lines1"], *_line_inputs(ls, npts)]

    def run(t):
        out = ops.gt_matches_from_reprojection(*t[:8], pos_th=3.0, neg_th=5.0, dense=False, dense_t=True)
        ops.gt_epipolar_unmatched_(t[0], t[1], t[8], t[6], t[7], out["matches0"], out["matches1"], 5.0)
        lines = ops.gt_line_matches_from_projection(t[11], t[12], t[13], t[14], (480, 640), (480, 640), t[9], t[10],
                                                    *t[15:19], npts=npts, min_visibility_th=0.5)
        return [out["matches0"], out["matches1"], out["assignment_t"], lines["line_matches0"], lines["line_matches1"],
                lines["line_assignment"]]

    first, second = scene(130), scene(131)
    static = [t.clone() for t in first]
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        run(static)
    torch.cuda.current_stream().wait_stream(side)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        outs = run(static)
    eager_first, eager_second = [t.clone() for t in run(first)], [t.clone() for t in run(second)]
    assert not torch.equal(eager_first[0], eager_second[0]) and not torch.equal(eager_first[3], eager_second[3])
    graph.replay()
    for name, a, b in zip("m0 m1 assignment_t line_m0 line_m1 line_assignment".split(), outs, eager_first):
        assert_same("graph, first scene: " + name, a, b)
    for s, t in zip(static, second):
        s.copy_(t)
    for replay in range(2):
        graph.replay()
        for name, a, b in zip("m0 m1 assignment_t line_m0 line_m1 line_assignment".split(), outs, eager_second):
            assert_same(f"graph, second scene, replay {replay}: " + name, a, b)
    assert int((eager_second[0] > -1).sum()) > 0 and int((eager_second[3] > -1).sum()) > 0
