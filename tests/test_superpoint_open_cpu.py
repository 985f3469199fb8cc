"""CPU: the SuperPoint-open extractor plugin's surface (conf, module tree, strict loads both ways with the reference,
resolution through glue-factory's get_model), its refusals and weight lookup, and the selection / sampling
restatement the GPU tests use, on the goldens made by scripts/make_superpoint_open_golden.py."""
import glob
import os
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gluefactory_b200 import synthetic  # noqa: E402
from gluefactory_b200.extractors.superpoint_open import SuperPointOpen  # noqa: E402
from tests.superpoint_oracle import border_ref, load_golden, nms_ref, sample_ref, select_ref  # noqa: E402

GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "sp_open_*.npz")))
REFERENCE_CONF = {
    "descriptor_dim": 256, "nms_radius": 4, "max_num_keypoints": None, "force_num_keypoints": False,
    "detection_threshold": 0.005, "remove_borders": 4, "channels": [64, 64, 128, 128, 256], "dense_outputs": None,
    "weights": None,
}


@pytest.fixture(scope="module")
def weights_path(tmp_path_factory):
    path = tmp_path_factory.mktemp("w") / "sp_open.pth"
    torch.save(synthetic.make_superpoint_open_weights(SuperPointOpen.state_dict_template(), seed=11), path)
    return str(path)


def _reference():
    from oracle import stage_reference

    if stage_reference.import_reference() is None:
        return None
    from gluefactory.models.extractors import superpoint_open

    return superpoint_open


def test_conf_and_module_tree(weights_path):
    m = SuperPointOpen({"weights": weights_path})
    for k, v in REFERENCE_CONF.items():
        if k != "weights":
            assert m.conf[k] == v, k
    assert m.required_data_keys == ["image"]
    keys = list(m.state_dict().keys())
    assert keys[:7] == ["backbone.0.0.conv.weight", "backbone.0.0.conv.bias", "backbone.0.0.bn.weight",
                        "backbone.0.0.bn.bias", "backbone.0.0.bn.running_mean", "backbone.0.0.bn.running_var",
                        "backbone.0.0.bn.num_batches_tracked"]
    assert len(keys) == 12 * 7 and keys[-1] == "descriptor.1.bn.num_batches_tracked"
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert shapes["backbone.2.0.conv.weight"] == (128, 64, 3, 3) and shapes["detector.1.conv.weight"] == (65, 256, 1, 1)
    assert shapes["descriptor.1.conv.weight"] == (256, 256, 1, 1)
    bns = [x for x in m.modules() if isinstance(x, torch.nn.BatchNorm2d)]
    assert len(bns) == 12 and all(b.eps == 1e-3 and b.momentum == 0.1 for b in bns)
    assert [type(x).__name__ for x in m.backbone[0]] == ["VGGBlock", "VGGBlock", "MaxPool2d"]
    assert len(m.backbone[3]) == 2
    assert isinstance(m.detector[1].activation, torch.nn.Identity)
    assert not any(p.requires_grad for p in m.parameters())


def test_freeze_batch_normalization(weights_path):
    m = SuperPointOpen({"weights": weights_path}).train()
    assert all(x.training for x in m.modules())
    m = SuperPointOpen({"weights": weights_path, "freeze_batch_normalization": True}).train()
    assert all(not x.training for x in m.modules() if isinstance(x, torch.nn.BatchNorm2d))
    assert m.backbone[0][0].conv.training


def test_sync_batchnorm_conversion(weights_path):
    """Under --distributed glue-factory converts every BatchNorm to nn.SyncBatchNorm (not a BatchNorm2d subclass):
    the plugin still finds all twelve, freezes them, and refuses momentum=None in bf16."""
    m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(
        SuperPointOpen({"weights": weights_path, "freeze_batch_normalization": True}))
    bns = m._batchnorms()
    assert len(bns) == 12 and all(isinstance(b, torch.nn.SyncBatchNorm) for b in bns)
    assert bns[0] is m.backbone[0][0].bn
    m.train()
    assert not any(b.training for b in bns) and m.backbone[0][0].conv.training
    m.detector[1].bn.momentum = None
    with pytest.raises(NotImplementedError, match="momentum"):
        m({"image": torch.zeros(1, 1, 16, 16)})


def test_reference_strict_load_both_ways(weights_path):
    ref = _reference()
    if ref is None:
        pytest.skip("reference not staged under oracle/_ref")
    assert dict(ref.SuperPoint.default_conf) == REFERENCE_CONF
    r = ref.SuperPoint({"weights": weights_path})
    mine = SuperPointOpen({"weights": weights_path})
    r.load_state_dict(mine.state_dict(), strict=True)
    mine.load_state_dict(r.state_dict(), strict=True)
    assert list(r.state_dict()) == list(mine.state_dict())
    from gluefactory.models import get_model

    assert get_model("gluefactory_b200.extractors.superpoint_open") is SuperPointOpen


@pytest.mark.parametrize("conf", [
    {"trainable": True}, {"channels": [32, 64, 128, 128, 256]}, {"descriptor_dim": 128},
    {"max_num_keypoints": 20000}, {"nms_radius": 10},
])
def test_refused_confs(conf, weights_path):
    with pytest.raises(NotImplementedError):
        SuperPointOpen({"weights": weights_path, **conf})


def test_refused_forwards(weights_path):
    m = SuperPointOpen({"weights": weights_path})
    with pytest.raises(NotImplementedError, match="backward"):
        m({"image": torch.zeros(1, 1, 16, 16, requires_grad=True)})
    with pytest.raises(ValueError, match="force_num_keypoints"):
        m({"image": torch.zeros(2, 1, 16, 16)})
    with pytest.raises(ValueError, match="8x8"):
        m({"image": torch.zeros(1, 1, 7, 16)})
    m.backbone[0][0].conv.weight.requires_grad_(True)
    with pytest.raises(NotImplementedError, match="backward"):
        m({"image": torch.zeros(1, 1, 16, 16)})


def test_weights_lookup_never_downloads(tmp_path, monkeypatch, weights_path):
    def no_download(*a, **k):
        raise AssertionError("download attempted")

    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", no_download)
    monkeypatch.setattr(torch.hub, "download_url_to_file", no_download)
    monkeypatch.setattr(torch.hub, "get_dir", lambda: str(tmp_path))
    default = tmp_path / "checkpoints" / "superpoint_v6_from_tf.pth"
    with pytest.raises(FileNotFoundError, match=str(default)):
        SuperPointOpen({})
    with pytest.raises(FileNotFoundError, match="nowhere.pth.*" + str(default)):
        SuperPointOpen({"weights": str(tmp_path / "nowhere.pth")})
    sd = torch.load(weights_path)
    default.parent.mkdir()
    torch.save(sd, default)
    for w in (None, str(tmp_path / "nowhere.pth"), weights_path):  # the reference's fallback to the default file
        m = SuperPointOpen({"weights": w})
        for k, v in sd.items():
            assert torch.equal(m.state_dict()[k], v), k


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_golden_selection_restatement(path):
    """The restatement reproduces the reference's keypoints, scores and order from its own dense score map (fixed
    border frame), and its descriptors from its dense descriptors sampled in fixed mode at kp + 0.5."""
    g = load_golden(path)
    conf = {**REFERENCE_CONF, **g["conf"]}
    s = border_ref(nms_ref(torch.from_numpy(g["dense_scores"]), conf["nms_radius"]), conf["remove_borders"])
    k = conf["max_num_keypoints"]
    sel = select_ref(s, conf["detection_threshold"], -1 if k is None else k)
    kp_g, sc_g = torch.from_numpy(g["keypoints"]), torch.from_numpy(g["keypoint_scores"])
    for b, (kp, sc) in enumerate(sel):
        n = len(sc)
        assert torch.equal(kp + 0.5, kp_g[b, :n]) and torch.equal(sc, sc_g[b, :n])
        assert (sc_g[b, n:] == 0).all()
        desc = sample_ref(torch.from_numpy(g["dense_descriptors"][b:b + 1]), kp[None] + 0.5, False)
        torch.testing.assert_close(desc[0].float(), torch.from_numpy(g["descriptors"][b, :n]), rtol=0, atol=1e-5)
    if "dense_output" in g:
        assert (g["dense_output"] == g["dense_descriptors"]).all()
