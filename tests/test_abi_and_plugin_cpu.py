"""CPU: the C-ABI library loads and exports every symbol of include/lgb200.h; the plugin honours
the reference's plugin surface (construction, names, state_dict) and fails loudly without a GPU."""
import json
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN_SURFACE = os.path.join(ROOT, "tests", "golden", "reference_plugin_surface.json")


@pytest.fixture(scope="module")
def built():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge

    return ge.build()


def test_library_exports_every_declared_symbol(built):
    from gluefactory_b200 import _lib

    hdr = open(os.path.join(ROOT, "include", "lgb200.h")).read()
    declared = set(re.findall(r"\b(lgb200_[a-z0-9_]+)\s*\(", hdr))
    assert declared and declared == set(_lib.SIGNATURES), declared ^ set(_lib.SIGNATURES)
    lib = _lib.load(check_device=False)
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.lgb200_abi_version() == 2
    # pure host queries are callable without a GPU
    assert lib.lgb200_assign_ws_bytes(2, 64, 64) == 2 * 2 * 64 * 8
    assert lib.lgb200_ln_gelu_bwd_parts(1000) == 125
    assert lib.lgb200_attn_bwd_ws_floats(64, 2048, 2048, 4) == 2 * 64 * 4 * 2048  # padded lse2 + delta only


def test_plugin_surface_matches_reference_names():
    from gluefactory_b200 import synthetic
    from gluefactory_b200.matchers import lightglue as plug

    model = plug.__main_model__({"name": "gluefactory_b200.matchers.lightglue", "n_layers": 3, "unknown_key": 1})
    names = [n for n, _ in model.named_parameters()]
    conf = dict(synthetic.DEFAULT_CONF, n_layers=3)
    assert names == [n for n, _ in synthetic.state_dict_spec(conf)]
    for n, shape in synthetic.state_dict_spec(conf):
        assert tuple(model.state_dict()[n].shape) == tuple(shape), n
    assert "confidence_thresholds" in model.state_dict()
    assert model.required_data_keys == ["keypoints0", "keypoints1", "descriptors0", "descriptors1"]
    disk = plug.LightGlue({"input_dim": 128, "n_layers": 1})
    assert tuple(disk.input_proj.weight.shape) == (256, 128)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback():
    from gluefactory_b200 import synthetic
    from gluefactory_b200._lib import Lgb200Error
    from gluefactory_b200.matchers.lightglue import LightGlue

    model = LightGlue({"n_layers": 1})
    data = synthetic.make_pairs(1, 64, seed=1)
    with pytest.raises(Lgb200Error, match="no CPU fallback"):
        model(data)


def test_dropin_through_reference_get_model():
    """The plugin must expose the reference's surface: the LightGlue state_dict layout and confidence thresholds, and the
    homography ground-truth component's required keys and defaults, as recorded from the unmodified reference in
    tests/golden/reference_plugin_surface.json (oracle/make_surface_golden.py).  Where the build staged the reference
    under oracle/_ref, gluefactory.models.get_model must also discover the plugin the way it discovers the reference
    matcher (models/__init__.py:7-30)."""
    from gluefactory_b200.matchers.homography_matcher import HomographyMatcher
    from gluefactory_b200.matchers.lightglue import LightGlue

    with open(GOLDEN_SURFACE) as f:
        g = json.load(f)
    lg = g["lightglue_n_layers2"]
    mine = LightGlue({"n_layers": 2})
    sd = mine.state_dict()
    assert list(sd.keys()) == lg["keys"]
    for k, shape in zip(lg["keys"], lg["shapes"]):
        assert list(sd[k].shape) == shape, k
    mine.load_state_dict({k: torch.zeros(shape) for k, shape in zip(lg["keys"], lg["shapes"])})  # strict
    assert torch.allclose(LightGlue({"n_layers": 2}).confidence_thresholds, torch.tensor(lg["confidence_thresholds"]))
    hm = g["homography_matcher"]
    assert sorted(HomographyMatcher({}).required_data_keys) == hm["required_data_keys"]
    for k, v in hm["default_conf"].items():
        assert HomographyMatcher.default_conf[k] == v, k

    saved = list(sys.path)
    try:
        from oracle import stage_reference

        if stage_reference.import_reference() is not None:
            _dropin_checks()
    finally:
        sys.path[:] = saved


def _dropin_checks():
    from gluefactory.models import get_model

    cls = get_model("gluefactory_b200.matchers.lightglue")
    ref_cls = get_model("matchers.lightglue")
    mine, ref = cls({"n_layers": 2}), ref_cls({"n_layers": 2})
    assert list(mine.state_dict().keys()) == list(ref.state_dict().keys())
    for k, v in ref.state_dict().items():
        assert mine.state_dict()[k].shape == v.shape, k
    mine.load_state_dict(ref.state_dict())  # strict
    assert torch.allclose(mine.confidence_thresholds, ref.confidence_thresholds)
    # TwoViewPipeline builds it from a config dict like any other matcher (two_view_pipeline.py:48-49)
    from gluefactory.models.two_view_pipeline import TwoViewPipeline

    pipe = TwoViewPipeline({"matcher": {"name": "gluefactory_b200.matchers.lightglue", "n_layers": 1},
                            "ground_truth": {"name": "gluefactory_b200.matchers.homography_matcher", "th_positive": 2.0},
                            "extractor": {"name": None}, "allow_no_extract": True})
    assert isinstance(pipe.matcher, cls)
    # the ground-truth component is discovered the same way (two_view_pipeline.py:54-56) and mirrors the reference's
    gt_cls, ref_gt = get_model("gluefactory_b200.matchers.homography_matcher"), get_model("matchers.homography_matcher")
    assert isinstance(pipe.ground_truth, gt_cls) and pipe.ground_truth.conf.th_positive == 2.0
    assert sorted(gt_cls({}).required_data_keys) == sorted(ref_gt({}).required_data_keys)
    for k, v in ref_gt.default_conf.items():
        assert gt_cls.default_conf[k] == v, k
    with pytest.raises(NotImplementedError):
        gt_cls({}).loss({}, {})
    if not torch.cuda.is_available():
        with pytest.raises(Exception):  # no CUDA device: the op refuses instead of falling back to the CPU
            gt_cls({})({"H_0to1": torch.eye(3)[None], "keypoints0": torch.zeros(1, 4, 2), "keypoints1": torch.zeros(1, 4, 2)})


def test_lightglue_rejects_removed_precision_mode():
    """`precision` takes `bf16` or `fp32`; a config naming the former `bf16x3` mode fails at construction rather than
    running some other numeric path.  `fp32` meets the goldens that mode was held to."""
    from gluefactory_b200.matchers.lightglue import LightGlue

    with pytest.raises(AssertionError, match="bf16x3"):
        LightGlue({"precision": "bf16x3", "n_layers": 1})


def test_mask_counts_host_fallback():
    from gluefactory_b200 import ops

    m = (torch.rand(2, 9, 13, generator=torch.Generator().manual_seed(1)) < 0.3)
    r, c = ops.mask_counts(m.view(torch.uint8))
    assert torch.equal(r, m.sum(2).float()) and torch.equal(c, m.sum(1).float())
