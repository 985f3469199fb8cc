"""Drop-in for gluefactory's `matchers.depth_matcher` -- the ground-truth component of the MegaDepth configs
(configs/superpoint+lightglue_megadepth.yaml: `ground_truth.name: matchers.depth_matcher`, th_positive 3,
th_negative 5, th_epi 5) -- with the O(M N) label pass on the device (SURVEY 8f row 1, second half).

Select it with `ground_truth.name: gluefactory_b200.matchers.depth_matcher`.  Same conf keys and output keys as the
reference (models/matchers/depth_matcher.py:17-89, geometry/gt_generation.py:13-106) except the dense `reward` map,
which has no consumer on the matcher's path.

The per-point geometry (depth sampling, un-projection, rigid transform, projection: O(M + N)) is done with torch ops
through the Camera / Pose objects the host framework puts in the batch (`data["view*"]["camera"]`, `data["T_0to1"]`;
duck-typed: `.image2cam`, `.cam2image`, `.calibration_matrix`, `.transform`, `.inv`, `.R`, `.t`), restating
geometry/depth.py:21-85.  The distance matrix, mutual nearest neighbours, thresholds and the epipolar exclusion --
everything the reference builds ~15 dense [B, M, N] temporaries for -- run in `lgb200_gt_from_reprojection` /
`lgb200_gt_epipolar_unmatched` without any dense temporary.

With `use_lines` the line labels (`line_matches0/1`, `line_assignment`) of `gt_line_matches_from_pose_depth`
(gt_generation.py:207-406) are added: the sampled line points go through the same `sample_depth` / `project` as the
keypoints, and the point-segment counting, the per-pair linear assignment (scipy's, on the host, in the reference)
and the labels run in csrc/gt_lines.cu without a host synchronisation.  Segments are clamped to `view*["depth"]`, the
"outside" test uses `view*["image"]`, and the reverse projection uses `T_0to1.inv()`, as in the reference (:286).
"""
import torch
import torch.nn.functional as F
from torch import nn

from .. import ops
from .lightglue import _Conf, _merge, _to_plain


def sample_depth(pts, depth_):
    """geometry/depth.py:8-26: bilinear sample where all four neighbours are valid, nearest otherwise."""
    depth = torch.where(depth_ > 0, depth_, depth_.new_tensor(float("nan")))[:, None]
    h, w = depth.shape[-2:]
    grid = (pts / pts.new_tensor([[w, h]]) * 2 - 1)[:, None]
    lin = F.grid_sample(depth, grid, align_corners=False, mode="bilinear")
    nn_ = F.grid_sample(depth, grid, align_corners=False, mode="nearest")
    interp = torch.where(torch.isnan(lin), nn_, lin)[:, :, 0].permute(0, 2, 1).squeeze(-1)
    return interp, (~torch.isnan(interp)) & (interp > 0)


def project(kpi, di, depthj, camera_i, camera_j, T_itoj, validi, ccth=None):
    """geometry/depth.py:39-71."""
    kpi_3d_j = T_itoj.transform(camera_i.image2cam(kpi) * di[..., None])
    kpi_j, validj = camera_j.cam2image(kpi_3d_j)
    validi = validi & validj
    if depthj is None or ccth is None:
        return kpi_j, validi & validj
    dj, validj = sample_depth(kpi_j, depthj)  # circle consistency
    kpi_j_3d_j = camera_j.image2cam(kpi_j) * dj[..., None]
    kpi_j_i, validj_i = camera_i.cam2image(T_itoj.inv().transform(kpi_j_3d_j))
    consistent = ((kpi - kpi_j_i) ** 2).sum(-1) < ccth
    return kpi_j, validi & consistent & validj_i & validj


def _skew(v):
    z = torch.zeros_like(v[..., 0])
    return torch.stack([z, -v[..., 2], v[..., 1], v[..., 2], z, -v[..., 0], -v[..., 1], v[..., 0], z], -1).reshape(
        v.shape[:-1] + (3, 3))


class DepthMatcher(nn.Module):
    default_conf = {
        "name": None,
        "trainable": False,
        "freeze_batch_normalization": False,
        "timeit": False,
        "use_points": True,
        "th_positive": 3.0,
        "th_negative": 5.0,
        "th_epi": None,
        "th_consistency": None,
        "use_lines": False,
        "n_line_sampled_pts": 50,
        "line_perp_dist_th": 5,
        "overlap_th": 0.2,
        "min_visibility_th": 0.5,
        "dense_assignment": True,  # plugin-only: materialise the boolean [B,M,N] assignment (the reference always does)
        # plugin-only: also emit `assignment_t`, the [B,N,M] transpose, in the same pass (saves the plugin matcher's loss a
        # 0.5 ms transpose per step: its fused assignment backward walks the mask by columns too)
        "transposed_assignment": False,
    }
    required_data_keys = ["view0", "view1", "T_0to1"]

    def __init__(self, conf=None):
        super().__init__()
        self.conf = conf = _Conf(_merge(self.default_conf, _to_plain(conf)))
        self.required_data_keys = list(self.required_data_keys)
        if conf.use_points:
            self.required_data_keys += ["keypoints0", "keypoints1"]
        if conf.use_lines:
            self.required_data_keys += ["lines0", "lines1", "valid_lines0", "valid_lines1"]

    @torch.no_grad()
    def forward(self, data):
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        with torch.autocast(device_type="cuda", enabled=False):  # reference: custom_fwd(cast_inputs=float32)
            result = self._labels(data) if self.conf.use_points else {}
            if self.conf.use_lines:
                result.update(self._line_labels(data))
        return result

    def _labels(self, data):
        conf = self.conf
        kp0, kp1 = data["keypoints0"].float(), data["keypoints1"].float()
        cam0, cam1 = data["view0"]["camera"], data["view1"]["camera"]
        T_0to1 = data["T_0to1"]
        T_1to0 = data.get("T_1to0", None)
        T_1to0 = T_0to1.inv() if T_1to0 is None else T_1to0
        depth0, depth1 = data["view0"].get("depth"), data["view1"].get("depth")
        if "depth_keypoints0" in data and "depth_keypoints1" in data:
            d0, valid0 = data["depth_keypoints0"], data["valid_depth_keypoints0"]
            d1, valid1 = data["depth_keypoints1"], data["valid_depth_keypoints1"]
        else:
            assert depth0 is not None and depth1 is not None
            d0, valid0 = sample_depth(kp0, depth0)
            d1, valid1 = sample_depth(kp1, depth1)
        kp0_1, visible0 = project(kp0, d0, depth1, cam0, cam1, T_0to1, valid0, ccth=conf.th_consistency)
        kp1_0, visible1 = project(kp1, d1, depth0, cam1, cam0, T_1to0, valid1, ccth=conf.th_consistency)
        out = ops.gt_matches_from_reprojection(kp0, kp1, kp0_1, kp1_0, visible0, visible1, valid0, valid1,
                                               pos_th=conf.th_positive, neg_th=conf.th_negative,
                                               dense=bool(conf.dense_assignment), dense_t=bool(conf.transposed_assignment))
        if conf.th_epi is not None:
            # F = K1^-T [t]x R K0^-1 (gt_generation.py:76-80, epipolar.py:7-9); note the reference thresholds the
            # epipolar distance with th_negative (neg_th), not with th_epi, which only switches the step on
            Fm = (torch.inverse(cam1.calibration_matrix()).transpose(-1, -2) @ (_skew(T_0to1.t) @ T_0to1.R)
                  @ torch.inverse(cam0.calibration_matrix()))
            ops.gt_epipolar_unmatched_(kp0, kp1, Fm, valid0, valid1, out["matches0"], out["matches1"], conf.th_negative)
        m0, m1 = out["matches0"], out["matches1"]
        out.update({"matching_scores0": (m0 > -1).float(), "matching_scores1": (m1 > -1).float(),
                    "depth_keypoints0": d0, "depth_keypoints1": d1, "proj_0to1": kp0_1, "proj_1to0": kp1_0,
                    "visible0": visible0, "visible1": visible1})
        return out

    def _line_labels(self, data):
        conf, npts = self.conf, self.conf.n_line_sampled_pts
        v0, v1 = data["view0"], data["view1"]
        segs0 = ops.line_segments(data["lines0"], *v0["depth"].shape[-2:])
        segs1 = ops.line_segments(data["lines1"], *v1["depth"].shape[-2:])
        pts0, pts1 = ops.sample_line_points(segs0, npts), ops.sample_line_points(segs1, npts)
        d0, valid0 = sample_depth(pts0, v0["depth"])
        d1, valid1 = sample_depth(pts1, v1["depth"])
        T_0to1 = data["T_0to1"]
        pts0_1, visible0 = project(pts0, d0, v1["depth"], v0["camera"], v1["camera"], T_0to1, valid0)
        pts1_0, visible1 = project(pts1, d1, v0["depth"], v1["camera"], v0["camera"], T_0to1.inv(), valid1)
        return ops.gt_line_matches_from_projection(
            segs0, segs1, pts0_1, pts1_0, v0["image"].shape[-2:], v1["image"].shape[-2:], data["valid_lines0"],
            data["valid_lines1"], visible0, visible1, valid0, valid1, npts=npts, dist_th=conf.line_perp_dist_th,
            overlap_th=conf.overlap_th, min_visibility_th=conf.min_visibility_th)

    def loss(self, pred, data):
        raise NotImplementedError


__main_model__ = DepthMatcher
