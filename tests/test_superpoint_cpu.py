"""CPU: the SuperPoint extractor plugin's surface (conf, module tree, a strict load into the reference module), its
refusals and its weight lookup, and the selection / sampling restatement the GPU tests use against the goldens made
by scripts/make_superpoint_golden.py."""
import glob
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gluefactory_b200 import synthetic  # noqa: E402
from gluefactory_b200.extractors.superpoint import SuperPoint  # noqa: E402
from tests.superpoint_oracle import border_ref, load_golden, nms_ref, sample_ref, select_ref  # noqa: E402

GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "superpoint_*.npz")))
NAMES = ["conv1a", "conv1b", "conv2a", "conv2b", "conv3a", "conv3b", "conv4a", "conv4b",
         "convPa", "convPb", "convDa", "convDb"]
REFERENCE_CONF = {
    "has_detector": True, "has_descriptor": True, "descriptor_dim": 256, "sparse_outputs": True,
    "dense_outputs": False, "nms_radius": 4, "refinement_radius": 0, "detection_threshold": 0.005,
    "max_num_keypoints": -1, "max_num_keypoints_val": None, "force_num_keypoints": False,
    "randomize_keypoints_training": False, "remove_borders": 4, "legacy_sampling": True,
}


def _reference():
    from oracle import stage_reference

    if stage_reference.import_reference() is None:
        return None
    from gluefactory_nonfree import superpoint

    return superpoint


def test_conf_and_module_tree():
    m = SuperPoint({"weights": None})
    for k, v in REFERENCE_CONF.items():
        assert m.conf[k] == v, k
    assert m.required_data_keys == ["image"]
    keys = list(m.state_dict().keys())
    assert keys == [f"{n}.{p}" for n in NAMES for p in ("weight", "bias")]
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert shapes["conv1a.weight"] == (64, 1, 3, 3) and shapes["conv3a.weight"] == (128, 64, 3, 3)
    assert shapes["convPb.weight"] == (65, 256, 1, 1) and shapes["convDb.weight"] == (256, 256, 1, 1)
    assert not any(p.requires_grad for p in m.parameters())


def test_strict_load_into_reference():
    ref = _reference()
    if ref is None:
        pytest.skip("reference not staged under oracle/_ref")
    assert {k: v for k, v in ref.SuperPoint.default_conf.items()} == REFERENCE_CONF
    sd = synthetic.make_superpoint_weights(SuperPoint({"weights": None}).state_dict(), seed=3)
    saved = torch.hub.load_state_dict_from_url
    torch.hub.load_state_dict_from_url = lambda *a, **k: sd
    try:
        r = ref.SuperPoint({})
    finally:
        torch.hub.load_state_dict_from_url = saved
    r.load_state_dict(SuperPoint({"weights": None}).state_dict(), strict=True)
    SuperPoint({"weights": None}).load_state_dict(r.state_dict(), strict=True)
    from gluefactory.models import get_model

    assert get_model("gluefactory_b200.extractors.superpoint") is SuperPoint


@pytest.mark.parametrize("conf", [
    {"trainable": True}, {"refinement_radius": 2}, {"has_detector": False, "sparse_outputs": False},
    {"has_descriptor": False, "sparse_outputs": False}, {"descriptor_dim": 128}, {"max_num_keypoints": 20000},
    {"nms_radius": 12},
])
def test_refused_confs(conf):
    with pytest.raises(NotImplementedError):
        SuperPoint({"weights": None, **conf})


def test_refused_forwards():
    m = SuperPoint({"weights": None, "randomize_keypoints_training": True, "max_num_keypoints": 8}).train()
    with pytest.raises(NotImplementedError, match="randomize"):
        m({"image": torch.zeros(1, 1, 16, 16)})
    m = SuperPoint({"weights": None})
    with pytest.raises(NotImplementedError, match="backward"):
        m({"image": torch.zeros(1, 1, 16, 16, requires_grad=True)})
    m.conv1a.weight.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="backward"):
        m({"image": torch.zeros(1, 1, 16, 16)})


def test_weights_lookup_never_downloads(tmp_path, monkeypatch):
    def no_download(*a, **k):
        raise AssertionError("download attempted")

    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", no_download)
    monkeypatch.setattr(torch.hub, "download_url_to_file", no_download)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    path = tmp_path / "checkpoints" / "superpoint_v1.pth"
    with pytest.raises(FileNotFoundError, match=str(path)):
        SuperPoint({})
    with pytest.raises(FileNotFoundError, match="nowhere.pth"):
        SuperPoint({"weights": str(tmp_path / "nowhere.pth")})
    sd = synthetic.make_superpoint_weights(SuperPoint({"weights": None}).state_dict(), seed=5)
    path.parent.mkdir()
    torch.save(sd, path)
    for w in ("default", str(path)):
        m = SuperPoint({"weights": w})
        for k, v in sd.items():
            assert torch.equal(m.state_dict()[k], v), k


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_golden_selection_restatement(path):
    """The restatement reproduces the reference's keypoints, scores and order from its own dense score map, and its
    descriptors from its dense descriptors: the GPU tests can use it at parameters the goldens do not cover."""
    g = load_golden(path)
    conf = {**REFERENCE_CONF, **g["conf"]}
    scores = torch.from_numpy(g["dense_scores"])
    s = border_ref(nms_ref(scores, conf["nms_radius"]), conf["remove_borders"],
                   torch.from_numpy(g["image_size"]) if "image_size" in g else None)
    sel = select_ref(s, conf["detection_threshold"], conf["max_num_keypoints"])
    kp_g, sc_g = torch.from_numpy(g["keypoints"]), torch.from_numpy(g["keypoint_scores"])
    for b, (kp, sc) in enumerate(sel):
        n = len(sc)
        assert torch.equal(kp + 0.5, kp_g[b, :n]) and torch.equal(sc, sc_g[b, :n])
        assert (sc_g[b, n:] == 0).all()
        desc = sample_ref(torch.from_numpy(g["dense_descriptors"][b:b + 1]), kp[None], conf["legacy_sampling"])
        torch.testing.assert_close(desc[0].float(), torch.from_numpy(g["descriptors"][b, :n]), rtol=0, atol=1e-5)
