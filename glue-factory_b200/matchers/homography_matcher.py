"""Drop-in ground-truth "matcher" for homography pairs, computed on the GPU.

Mirrors gluefactory/models/matchers/homography_matcher.py:8-66 (the `ground_truth` component of TwoViewPipeline,
two_view_pipeline.py:54-56, 83-86, 98-100): same constructor, `default_conf`, `required_data_keys`, output keys and
`loss` behaviour.  Select it with `model.ground_truth.name: gluefactory_b200.matchers.homography_matcher`.
The point labels come from the device kernels of csrc/gt.cu (lgb200_gt_from_homography), which reproduce
`gt_matches_from_homography` (geometry/gt_generation.py:109-161) bit for bit; there is no CPU fallback.
Line ground truth (`use_lines`, gt_generation.py:401-..., needs the wireframe extractors) is outside the matcher
training path this library covers and raises.
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
        # GT parameters for lines (accepted for config compatibility; use_lines=True is not supported)
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
            raise NotImplementedError("gluefactory_b200 homography_matcher: line ground truth is not implemented")

    @torch.no_grad()
    def forward(self, data):
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        if not self.conf.use_points:
            return {}
        # label generation is geometry in pixel units: always fp32, whatever autocast region the caller is in
        # (the pipeline runs ground_truth inside loss(), i.e. inside train.py's autocast block, :468-475)
        with torch.autocast(device_type="cuda", enabled=False):
            return self._labels(data)

    def _labels(self, data):
        return ops.gt_matches_from_homography(data["keypoints0"], data["keypoints1"], data["H_0to1"],
                                              pos_th=self.conf.th_positive, neg_th=self.conf.th_negative,
                                              dense=bool(self.conf.dense_assignment),
                                              dense_t=bool(self.conf.transposed_assignment))

    def loss(self, pred, data):
        raise NotImplementedError


__main_model__ = HomographyMatcher
