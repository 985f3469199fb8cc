"""Generate tests/golden/superpoint_*.npz by running the UNMODIFIED reference SuperPoint
(gluefactory_nonfree/superpoint.py) on the CPU in fp32 -- test infrastructure only; it needs the reference tree
($GLUEFACTORY_REFERENCE) and the omegaconf stand-in of oracle/_shim, like oracle/make_golden.py.

    python scripts/make_superpoint_golden.py

Weights come from synthetic.make_superpoint_weights over the PLUGIN's state_dict and are loaded strictly into the
reference (which also proves the two module trees carry identical names and shapes).  The reference's constructor
fetches superpoint_v1.pth through torch.hub.load_state_dict_from_url; this script alone stubs that call with the
random state_dict, so nothing is downloaded.  Images come from synthetic.make_superpoint_images at sizes that are not
multiples of 8 or of the kernels' tiles.  Stored per case: the image (and image_size), the conf, the reference's dense
score map and dense descriptors (sparse_outputs False), and its keypoints, keypoint scores and descriptors.
"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden  # noqa: E402,F401  (puts the reference and oracle/_shim on sys.path)
from gluefactory_b200 import synthetic  # noqa: E402

WEIGHT_SEED = 7

# name: (B, C, H, W, image_size or None, conf overrides, image seed)
CASES = {
    "superpoint_gray_b2_75x101": (2, 1, 75, 101, None,
                                  {"max_num_keypoints": 64, "force_num_keypoints": True}, 1),
    "superpoint_rgb_b2_64x96": (2, 3, 64, 96, None,
                                {"max_num_keypoints": 128, "force_num_keypoints": True, "legacy_sampling": False,
                                 "nms_radius": 3, "detection_threshold": 0.0}, 2),
    "superpoint_imsize_b2_80x88": (2, 1, 80, 88, [[88.0, 70.0], [61.0, 80.0]],
                                   {"max_num_keypoints": 100, "force_num_keypoints": True}, 3),
    "superpoint_all_b1_120x136": (1, 1, 120, 136, None, {"max_num_keypoints": -1}, 4),
}


def reference_model(conf, sd):
    import torch.hub

    from gluefactory_nonfree.superpoint import SuperPoint as Reference

    saved = torch.hub.load_state_dict_from_url
    torch.hub.load_state_dict_from_url = lambda *a, **k: sd
    try:
        model = Reference(conf)
    finally:
        torch.hub.load_state_dict_from_url = saved
    model.load_state_dict(sd, strict=True)
    return model.eval()


def main():
    from gluefactory_b200.extractors.superpoint import SuperPoint as Plugin

    sd = synthetic.make_superpoint_weights(Plugin({"weights": None}).state_dict(), seed=WEIGHT_SEED)
    for name, (B, C, H, W, image_size, over, seed) in CASES.items():
        conf = dict(over)
        image = synthetic.make_superpoint_images(B, C, H, W, seed=seed)
        data = {"image": image}
        if image_size is not None:
            data["image_size"] = torch.tensor(image_size)
        torch.manual_seed(0)
        with torch.no_grad():
            dense = reference_model({**conf, "sparse_outputs": False}, sd)(data)
            pred = reference_model(conf, sd)(data)
        out = {
            "image": image.numpy(),
            "conf": np.array(json.dumps(conf)),
            "weight_seed": np.array(WEIGHT_SEED),
            "dense_scores": dense["keypoint_scores"].numpy(),
            "dense_descriptors": dense["descriptors"].numpy(),
            "keypoints": pred["keypoints"].numpy(),
            "keypoint_scores": pred["keypoint_scores"].numpy(),
            "descriptors": pred["descriptors"].numpy(),
        }
        if image_size is not None:
            out["image_size"] = np.array(image_size, np.float32)
        path = os.path.join(ROOT, "tests", "golden", name + ".npz")
        np.savez_compressed(path, **out)
        real = (pred["keypoint_scores"] > 0).sum(-1).tolist()
        print(f"{name}: keypoints {tuple(pred['keypoints'].shape)} real {real} -> {path}")


if __name__ == "__main__":
    main()
