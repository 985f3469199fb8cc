"""Generate tests/golden/gt_lines_homography.npz and gt_lines_pose_depth.npz from the UNMODIFIED reference's
gt_line_matches_from_homography / gt_line_matches_from_pose_depth (geometry/gt_generation.py:207-558) on the seeded
scenes of gluefactory_b200.synthetic.line_gt_scene (test infrastructure only; needs the reference tree and scipy).

    python oracle/make_line_golden.py

Besides inputs and outputs, each case stores what the reference computed on the way, recorded by wrapping the
functions it calls (the reference itself is not modified): the projected sample points and their masks, and every
cost matrix it hands to scipy's linear_sum_assignment together with the assignment scipy returned.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.environ.get("GLUEFACTORY_REFERENCE", "/root/reference")
sys.path.insert(0, os.path.join(HERE, "_shim"))
sys.path.insert(0, REF)
sys.path.insert(0, ROOT)

from gluefactory_b200 import synthetic  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")

# tag: (B, L0, L1, seed, npts, dist_th, overlap_th, min_visibility_th)
HOMOGRAPHY_CASES = {"a": (3, 60, 47, 101, 50, 5.0, 0.2, 0.5), "b": (2, 35, 52, 102, 50, 5.0, 0.2, 0.2),
                    "c": (1, 24, 24, 103, 20, 3.0, 0.3, 0.5)}
POSE_DEPTH_CASES = {"a": (2, 50, 41, 111, 50, 5.0, 0.2, 0.5), "b": (2, 30, 45, 112, 50, 5.0, 0.2, 0.5)}


class _Recorder:
    """Wraps attributes of a module, keeping every call's (positional arguments, result)."""

    def __init__(self, module, names):
        self.module, self.saved, self.calls = module, {}, {n: [] for n in names}
        for n in names:
            self.saved[n] = fn = getattr(module, n)
            setattr(module, n, self._wrap(n, fn))

    def _wrap(self, name, fn):
        def wrapped(*a, **k):
            r = fn(*a, **k)
            self.calls[name].append((a, r))
            return r
        return wrapped

    def close(self):
        for n, fn in self.saved.items():
            setattr(self.module, n, fn)


def _store(out, tag, sc, meta, pos, m0, m1, rec):
    out[f"{tag}|meta"] = np.array(meta, dtype=np.float64)
    for k in ("lines0", "lines1", "valid_lines0", "valid_lines1"):
        out[f"{tag}|{k}"] = sc[k].numpy()
    out[f"{tag}|positives"] = pos.nonzero().numpy()
    out[f"{tag}|matches0"], out[f"{tag}|matches1"] = m0.numpy(), m1.numpy()
    asg = rec.calls["linear_sum_assignment"]
    out[f"{tag}|cost"] = np.stack([np.asarray(a[0]) for a, _ in asg]).astype(np.int64)
    out[f"{tag}|assign_rows"] = np.stack([np.asarray(r[0]) for _, r in asg])
    out[f"{tag}|assign_cols"] = np.stack([np.asarray(r[1]) for _, r in asg])


def run_homography(out):
    from gluefactory.geometry import gt_generation as G

    for tag, (B, L0, L1, seed, npts, dist, ov, mvt) in HOMOGRAPHY_CASES.items():
        sc = synthetic.line_gt_scene("homography", B, L0, L1, seed)
        h, w = sc["image_size"]
        rec = _Recorder(G, ["warp_points_torch", "linear_sum_assignment"])
        try:
            pos, m0, m1 = G.gt_line_matches_from_homography(sc["lines0"], sc["lines1"], sc["valid_lines0"],
                                                            sc["valid_lines1"], (B, 1, h, w), (B, 1, h, w),
                                                            sc["H_0to1"], npts, dist, ov, mvt)
        finally:
            rec.close()
        _store(out, tag, sc, [B, L0, L1, seed, npts, dist, ov, mvt, h, w], pos, m0, m1, rec)
        out[f"{tag}|H"] = sc["H_0to1"].numpy()
        out[f"{tag}|pts0_1"] = rec.calls["warp_points_torch"][0][1].numpy()
        out[f"{tag}|pts1_0"] = rec.calls["warp_points_torch"][1][1].numpy()
        print(f"gt_lines_homography {tag}: positives={int(pos.sum())} unmatched0={int((m0 == -1).sum())} "
              f"ignored0={int((m0 == -2).sum())} unmatched1={int((m1 == -1).sum())}")


def run_pose_depth(out):
    from gluefactory.geometry import gt_generation as G
    from gluefactory.geometry.wrappers import Camera, Pose

    for tag, (B, L0, L1, seed, npts, dist, ov, mvt) in POSE_DEPTH_CASES.items():
        sc = synthetic.line_gt_scene("pose_depth", B, L0, L1, seed)
        h, w = sc["image_size"]
        T = Pose.from_Rt(sc["R"], sc["t"])
        data = {"view0": {"camera": Camera.from_calibration_matrix(sc["K0"]), "depth": sc["depth0"],
                          "image": torch.zeros(B, 1, h, w)},
                "view1": {"camera": Camera.from_calibration_matrix(sc["K1"]), "depth": sc["depth1"],
                          "image": torch.zeros(B, 1, h, w)},
                "T_0to1": T, "T_1to0": T.inv()}
        rec = _Recorder(G, ["sample_depth", "project", "linear_sum_assignment"])
        try:
            pos, m0, m1 = G.gt_line_matches_from_pose_depth(sc["lines0"], sc["lines1"], sc["valid_lines0"],
                                                            sc["valid_lines1"], data, npts, dist, ov, mvt)
        finally:
            rec.close()
        _store(out, tag, sc, [B, L0, L1, seed, npts, dist, ov, mvt, h, w], pos, m0, m1, rec)
        (_, (p01, vis0)), (_, (p10, vis1)) = rec.calls["project"]
        out[f"{tag}|pts0_1"], out[f"{tag}|pts1_0"] = p01.numpy(), p10.numpy()
        out[f"{tag}|visible0"], out[f"{tag}|visible1"] = vis0.numpy(), vis1.numpy()
        out[f"{tag}|valid_pts0"] = rec.calls["sample_depth"][0][1][1].numpy()
        out[f"{tag}|valid_pts1"] = rec.calls["sample_depth"][1][1][1].numpy()
        print(f"gt_lines_pose_depth {tag}: positives={int(pos.sum())} unmatched0={int((m0 == -1).sum())} "
              f"ignored0={int((m0 == -2).sum())} unmatched1={int((m1 == -1).sum())}")


if __name__ == "__main__":
    for name, fn in (("gt_lines_homography", run_homography), ("gt_lines_pose_depth", run_pose_depth)):
        out = {}
        fn(out)
        path = os.path.join(OUT, name + ".npz")
        np.savez_compressed(path, **out)
        print(name, "->", path, f"({os.path.getsize(path) / 1e6:.2f} MB)")
