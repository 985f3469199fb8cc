"""Generate tests/golden/sp_open_*.npz by running the UNMODIFIED reference SuperPoint-open
(gluefactory/models/extractors/superpoint_open.py) on the CPU in fp32 (not superpoint_*.npz: the non-free plugin's
tests take every file of that pattern) -- test infrastructure only; it needs the
reference tree ($GLUEFACTORY_REFERENCE) and the omegaconf stand-in of oracle/_shim, like oracle/make_golden.py.

    python scripts/make_superpoint_open_golden.py

Weights come from synthetic.make_superpoint_open_weights over the PLUGIN's state_dict, written to a temporary file and
passed as `weights`, so the reference loads them strictly and nothing is downloaded.  Images come from
synthetic.make_superpoint_images at sizes that are not multiples of 8 or of the kernels' tiles.  Training-mode cases
call the reference's BaseModel.train(), which leaves its BatchNorms on batch statistics unless
freeze_batch_normalization is set.  Stored per case: the image, the conf, `training`, the dense score map (before NMS)
and dense descriptors of a copy of the model in the same mode, the keypoints, scores and descriptors (and
dense_descriptors when asked for), and the running statistics after the call (`running`: every BatchNorm's
running_mean then running_var, in state_dict order).
"""
import copy
import json
import os
import sys
import tempfile

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden  # noqa: E402,F401  (puts the reference and oracle/_shim on sys.path)
from gluefactory_b200 import synthetic  # noqa: E402

WEIGHT_SEED = 11

# name: (B, C, H, W, training, conf overrides, image seed)
CASES = {
    "sp_open_gray_b2_75x101": (2, 1, 75, 101, False, {"max_num_keypoints": 64, "force_num_keypoints": True}, 1),
    "sp_open_rgb_b2_64x96": (2, 3, 64, 96, False, {"max_num_keypoints": 128, "force_num_keypoints": True,
                                                           "nms_radius": 3, "detection_threshold": 0.0}, 2),
    "sp_open_train_b3_72x90": (3, 1, 72, 90, True, {"max_num_keypoints": 96, "force_num_keypoints": True,
                                                            "nms_radius": 3, "detection_threshold": -1}, 3),
    "sp_open_frozen_b2_66x80": (2, 1, 66, 80, True, {"max_num_keypoints": 80, "force_num_keypoints": True,
                                                             "freeze_batch_normalization": True}, 4),
    "sp_open_all_b1_120x136": (1, 1, 120, 136, False, {}, 5),
    "sp_open_dense_b1_56x70": (1, 3, 56, 70, False, {"max_num_keypoints": 32, "dense_outputs": True}, 6),
}


def running(model):
    return np.concatenate([v.numpy().ravel() for k, v in model.state_dict().items()
                           if k.endswith("running_mean")] +
                          [v.numpy().ravel() for k, v in model.state_dict().items() if k.endswith("running_var")])


def dense(model, image):
    """The reference's dense score map before NMS and its dense descriptors, from its own modules."""
    if image.shape[1] == 3:
        image = (image * image.new_tensor([0.299, 0.587, 0.114]).view(1, 3, 1, 1)).sum(1, keepdim=True)
    features = model.backbone(image)
    desc = torch.nn.functional.normalize(model.descriptor(features), p=2, dim=1)
    scores = torch.nn.functional.softmax(model.detector(features), 1)[:, :-1]
    b, _, h, w = scores.shape
    scores = scores.permute(0, 2, 3, 1).reshape(b, h, w, 8, 8).permute(0, 1, 3, 2, 4).reshape(b, h * 8, w * 8)
    return scores, desc


def main():
    from gluefactory.models.extractors.superpoint_open import SuperPoint as Reference
    from gluefactory_b200.extractors.superpoint_open import SuperPointOpen as Plugin

    sd = synthetic.make_superpoint_open_weights(Plugin.state_dict_template(), seed=WEIGHT_SEED)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "superpoint_open_synthetic.pth")
        torch.save(sd, path)
        for name, (B, C, H, W, training, over, seed) in CASES.items():
            conf = dict(over)
            model = Reference({**conf, "weights": path, "trainable": False})
            model.train(training)
            image = synthetic.make_superpoint_images(B, C, H, W, seed=seed)
            torch.manual_seed(0)
            with torch.no_grad():
                scores, desc = dense(copy.deepcopy(model), image)
                pred = model({"image": image})
            out = {
                "image": image.numpy(),
                "conf": np.array(json.dumps(conf)),
                "training": np.array(training),
                "weight_seed": np.array(WEIGHT_SEED),
                "dense_scores": scores.numpy(),
                "dense_descriptors": desc.numpy(),
                "keypoints": pred["keypoints"].numpy(),
                "keypoint_scores": pred["keypoint_scores"].numpy(),
                "descriptors": pred["descriptors"].numpy(),
                "running": running(model),
            }
            if "dense_descriptors" in pred:
                out["dense_output"] = pred["dense_descriptors"].numpy()
            dst = os.path.join(ROOT, "tests", "golden", name + ".npz")
            np.savez_compressed(dst, **out)
            real = (pred["keypoint_scores"] > 0).sum(-1).tolist()
            print(f"{name}: keypoints {tuple(pred['keypoints'].shape)} real {real} -> {dst}")


if __name__ == "__main__":
    main()
