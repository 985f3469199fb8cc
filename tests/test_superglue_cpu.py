"""CPU: the SuperGlue plugin's surface and its fp64 oracle (tests/superglue_oracle.py) against the fixture produced by the
unmodified reference (tests/golden/superglue_l4_m150_n160.npz, scripts/make_superglue_golden.py: forward + loss +
backward in fp64, training mode).  The plugin's numerics run on the GPU (tests/test_gpu_superglue.py)."""
import ast
import os
import sys

import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.superglue import SuperGlue
from tests import superglue_oracle as SO
from tests.util import GOLDEN, check_grad_summary

NAME = "superglue_l4_m150_n160"


def load_golden():
    g = dict(np.load(os.path.join(GOLDEN, NAME + ".npz"), allow_pickle=False))
    conf = ast.literal_eval(str(g["meta|conf"]))
    B, M, N, seed = (int(g["meta|" + k]) for k in ("B", "M", "N", "seed"))
    return g, conf, B, M, N, seed


def golden_weights(conf, seed, dtype=torch.float64):
    sd = synthetic.make_gluestick_weights(SuperGlue(dict(conf)).state_dict(), seed=seed)
    return {k: (v.to(dtype) if v.is_floating_point() else v) for k, v in sd.items()}


def test_oracle_matches_reference_golden():
    g, conf, B, M, N, seed = load_golden()
    w = golden_weights(conf, seed)
    params = {k: w[k].clone().requires_grad_(True) for k, _ in SuperGlue(dict(conf)).named_parameters()}
    ww = {**w, **params}
    data = synthetic.make_superglue_batch(B, M, N, seed + 1, dtype=torch.float64)
    stats = {}
    pred = SO.superglue_forward(ww, data, conf, stats)
    losses = SO.superglue_loss(ww, pred, data, conf)
    losses["total"].mean().backward()
    for k in ("matches0", "matches1"):
        assert np.array_equal(pred[k].numpy(), g["pred|" + k]), k
    for k in ("sinkhorn_cost", "log_assignment", "matching_scores0", "matching_scores1"):
        np.testing.assert_allclose(pred[k].detach().numpy(), g["pred|" + k], rtol=1e-9, atol=1e-9, err_msg=k)
    assert set(losses) == {k[len("loss|"):] for k in g if k.startswith("loss|")}
    for k, v in losses.items():
        np.testing.assert_allclose(v.detach().numpy(), g["loss|" + k], rtol=1e-9, atol=1e-12, err_msg=k)
    for k, p in params.items():
        if float(g[f"grad|{k}|norm"]) < 1e-9:  # conv bias in front of a BatchNorm: zero in theory, rounding noise
            assert p.grad.norm().item() < 1e-9, k
            continue
        check_grad_summary(g, k, p.grad, rtol=1e-9)
    # the running statistics after backward: kenc once per image, GNN MLPs twice per image (checkpoint recompute)
    rs = SO.running_stats(w, stats, conf)
    assert {k[len("bn|"):] for k in g if k.startswith("bn|")} == set(rs)
    for k, v in rs.items():
        np.testing.assert_allclose(v.numpy(), g["bn|" + k], rtol=1e-9, atol=1e-12, err_msg=k)


def test_state_dict_layout_equals_reference_fixture():
    g, conf, *_ = load_golden()
    model = SuperGlue(dict(conf))
    grads = {k[len("grad|"):].rsplit("|", 1)[0] for k in g if k.startswith("grad|")}
    assert grads == {n for n, _ in model.named_parameters()}
    assert {k[len("bn|"):] for k in g if k.startswith("bn|")} == \
        {k for k in model.state_dict() if "running_" in k or "num_batches_tracked" in k}
    # initialisation quirks kept from the reference: proj = deepcopy(merge), zero last biases
    attn = model.gnn.layers[0].attn
    for p in attn.proj:
        assert torch.equal(p.weight, attn.merge.weight) and torch.equal(p.bias, attn.merge.bias)
    assert not model.kenc.encoder[-1].bias.any() and not model.gnn.layers[0].mlp[-1].bias.any()
    assert model.kenc.encoder[0].weight.shape[1] == 3
    assert SuperGlue({"weights": None, "use_scores": False}).kenc.encoder[0].weight.shape[1] == 2


def test_conf_surface():
    assert SuperGlue.default_conf["weights"] == "outdoor"
    assert SuperGlue.default_conf["num_sinkhorn_iterations"] == 50
    assert SuperGlue({"weights": None, "some_unknown_key": 3, "GNN_layers": ["self"]}).conf.some_unknown_key == 3
    with pytest.raises(NotImplementedError):
        SuperGlue({"weights": None, "descriptor_dim": 128})


def test_pretrained_weights_come_from_the_cache_only(tmp_path, monkeypatch):
    """"outdoor" / "indoor" are read from torch-hub's checkpoint cache and never downloaded."""
    monkeypatch.setenv("TORCH_HOME", str(tmp_path))
    monkeypatch.setattr(torch.hub, "_hub_dir", None, raising=False)
    expected = os.path.join(str(tmp_path), "hub", "checkpoints", "superglue_outdoor.pth")
    with pytest.raises(FileNotFoundError, match="superglue_outdoor.pth"):
        SuperGlue({"GNN_layers": ["self"]})
    with pytest.raises(FileNotFoundError, match="superglue_indoor.pth"):
        SuperGlue({"weights": "indoor", "GNN_layers": ["self"]})
    # present in the cache: loaded (strictly) from there
    src = SuperGlue({"weights": None, "GNN_layers": ["self", "cross"]})
    os.makedirs(os.path.dirname(expected))
    torch.save(src.state_dict(), expected)
    got = SuperGlue({"GNN_layers": ["self", "cross"]})
    for k, v in src.state_dict().items():
        assert torch.equal(got.state_dict()[k], v), k
    # any other string is a local file
    local = str(tmp_path / "mine.pth")
    torch.save(src.state_dict(), local)
    assert torch.equal(SuperGlue({"weights": local, "GNN_layers": ["self", "cross"]}).bin_score, src.bin_score)


def test_dropin_through_reference_get_model():
    """Where the build staged the reference under oracle/_ref: glue-factory's get_model discovers the plugin,
    TwoViewPipeline builds it from a config, and the reference module's state_dict loads into it strictly."""
    saved = list(sys.path)
    try:
        from oracle import stage_reference

        if stage_reference.import_reference() is None:
            pytest.skip("reference not staged under oracle/_ref")
        from gluefactory.models import get_model
        from gluefactory.models.two_view_pipeline import TwoViewPipeline
        from gluefactory_nonfree.superglue import SuperGlue as Reference

        cls = get_model("gluefactory_b200.matchers.superglue")
        assert cls is SuperGlue
        conf = {"weights": None, "GNN_layers": ["self", "cross"]}
        mine, ref = cls(dict(conf)), Reference(dict(conf))
        assert list(mine.state_dict().keys()) == list(ref.state_dict().keys())
        mine.load_state_dict(ref.state_dict())  # strict
        assert sorted(cls.required_data_keys) == sorted(Reference.required_data_keys)
        for k, v in Reference.default_conf.items():
            got = SuperGlue.default_conf[k]
            assert (dict(got) if isinstance(got, dict) else got) == (dict(v) if isinstance(v, dict) else v), k
        pipe = TwoViewPipeline({"matcher": {"name": "gluefactory_b200.matchers.superglue", "weights": None,
                                            "GNN_layers": ["self", "cross"]},
                                "extractor": {"name": None}, "allow_no_extract": True})
        assert isinstance(pipe.matcher, cls)
    finally:
        sys.path[:] = saved
