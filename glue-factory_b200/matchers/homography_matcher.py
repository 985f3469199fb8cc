"""Drop-in ground-truth "matcher" for homography pairs, computed on the GPU.

Mirrors gluefactory/models/matchers/homography_matcher.py:8-66 (the `ground_truth` component of TwoViewPipeline,
two_view_pipeline.py:54-56, 83-86, 98-100): same constructor, `default_conf`, `required_data_keys`, output keys and
`loss` behaviour.  Select it with `model.ground_truth.name: gluefactory_b200.matchers.homography_matcher`.
The point labels come from the device kernels of csrc/gt.cu (lgb200_gt_from_homography), which reproduce
`gt_matches_from_homography` (geometry/gt_generation.py:109-161) bit for bit; there is no CPU fallback.
With `use_lines` the line labels (`line_matches0/1`, `line_assignment`) of `gt_line_matches_from_homography`
(gt_generation.py:409-558) come from csrc/gt_lines.cu, including the per-pair linear assignment the reference solves
with scipy on the host, so the component never synchronises with the host and can run inside a captured CUDA graph.
Image sizes are read from `view0/1["image"]`, as the reference does.
"""
import torch
from torch import nn

from .. import ops
from .lightglue import _Conf, _merge, _to_plain


class HomographyMatcher(nn.Module):
    default_conf = {
        "name": None,
        "trainable": False,
        "freeze_batch_normalization": False,
        "timeit": False,
        # GT parameters for points (homography_matcher.py:10-13)
        "use_points": True,
        "th_positive": 3.0,
        "th_negative": 3.0,
        # GT parameters for lines
        "use_lines": False,
        "n_line_sampled_pts": 50,
        "line_perp_dist_th": 5,
        "overlap_th": 0.2,
        "min_visibility_th": 0.5,
        # plugin-only: also materialise the boolean [B,M,N] assignment (the reference always does)
        "dense_assignment": True,
        # plugin-only: also emit `assignment_t`, the [B,N,M] transpose, in the same pass (saves the plugin matcher's loss a
        # 0.5 ms transpose per step: its fused assignment backward walks the mask by columns too)
        "transposed_assignment": False,
    }
    required_data_keys = ["H_0to1"]

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
        # label generation is geometry in pixel units: always fp32, whatever autocast region the caller is in
        # (the pipeline runs ground_truth inside loss(), i.e. inside train.py's autocast block, :468-475)
        with torch.autocast(device_type="cuda", enabled=False):
            result = self._labels(data) if self.conf.use_points else {}
            if self.conf.use_lines:
                result.update(self._line_labels(data))
        return result

    def _labels(self, data):
        return ops.gt_matches_from_homography(data["keypoints0"], data["keypoints1"], data["H_0to1"],
                                              pos_th=self.conf.th_positive, neg_th=self.conf.th_negative,
                                              dense=bool(self.conf.dense_assignment),
                                              dense_t=bool(self.conf.transposed_assignment))

    def _line_labels(self, data):
        conf = self.conf
        return ops.gt_line_matches_from_homography(
            data["lines0"], data["lines1"], data["valid_lines0"], data["valid_lines1"], data["view0"]["image"].shape,
            data["view1"]["image"].shape, data["H_0to1"], npts=conf.n_line_sampled_pts, dist_th=conf.line_perp_dist_th,
            overlap_th=conf.overlap_th, min_visibility_th=conf.min_visibility_th)

    def loss(self, pred, data):
        raise NotImplementedError


__main_model__ = HomographyMatcher
