"""CPU: GlueStick on wireframes, and pretrained weights by name.

The fp64 oracle (tests/gluestick_wireframe_oracle.py) against the fixtures the unmodified reference produced on
wireframes from its own `lines_to_wireframe` (tests/golden/gluestick_wireframe_*.npz,
scripts/make_gluestick_wireframe_golden.py): shared junctions in eval and training mode, a view without lines, a view
without keypoints, views given with `image` only.  The plugin's pred for a view without keypoints needs no kernel and is
checked here; the numerics run on the GPU (tests/test_gpu_gluestick_wireframe.py).

Weight resolution of the GlueStick and LightGlue plugins: a name is looked up on the local disk in the reference's order
(glue-factory's DATA_PATH, taken from a stand-in `gluefactory.settings`, then torch-hub's cache under TORCH_HOME) and
never downloaded: torch.hub.load_state_dict_from_url is replaced by a function that fails the test."""
import os
import sys
import types

import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.gluestick import GlueStick
from gluefactory_b200.matchers.lightglue import LightGlue
from tests import gluestick_wireframe_oracle as O
from tests.gluestick_inter_oracle import point_log_assignment_summary
from tests.util import GOLDEN, check_grad_summary


def _oracle_run(name):
    g, conf, _, data = O.load_case(GOLDEN, name)
    training = bool(g["meta|training"])
    w = {k: (v.double() if v.is_floating_point() else v)
         for k, v in O.case_state_dict(g, GlueStick(dict(conf)).state_dict()).items()}
    params = {k: v.requires_grad_(True) for k, v in w.items() if v.is_floating_point() and "running_" not in k}
    stats = {} if training else None
    pred = O.gluestick_forward({**w, **params}, data, conf, training, bn_stats=stats)
    return g, conf, data, w, params, stats, pred


@pytest.mark.parametrize("name", O.CASES)
def test_oracle_matches_reference_golden(name):
    g, conf, data, w, params, stats, pred = _oracle_run(name)
    if "pred|log_assignment_sub" in g:
        pred = {**pred, **point_log_assignment_summary(pred["log_assignment"])}
    stored = {k[len("pred|"):] for k in g if k.startswith("pred|")}
    got = set(pred) - ({"log_assignment"} if "pred|log_assignment_sub" in g else set())
    assert stored == got, stored ^ got
    for k in stored:
        ref = g["pred|" + k]
        assert tuple(pred[k].shape) == ref.shape, k
        if "matches" in k and "scores" not in k:
            assert pred[k].dtype == torch.int64 and np.array_equal(pred[k].numpy(), ref), k
        else:
            np.testing.assert_allclose(pred[k].detach().numpy(), ref, rtol=1e-9, atol=1e-9, err_msg=k)
    if not bool(g["meta|training"]):
        return
    # b_train: loss entries, every parameter gradient, the running statistics after the step
    from tests import gluestick_inter_oracle as I

    losses = I.gluestick_loss({**w, **params}, pred, data, conf)
    losses["total"].mean().backward()
    assert set(losses) == {k[len("loss|"):] for k in g if k.startswith("loss|")}
    assert "line_1_assignment_nll" in losses
    for k, v in losses.items():
        np.testing.assert_allclose(v.detach().numpy(), g["loss|" + k], rtol=1e-9, atol=1e-12, err_msg=k)
    for k, p in params.items():
        if float(g[f"grad|{k}|norm"]) < 1e-9:  # a conv bias in front of a BatchNorm: zero in theory, rounding noise
            assert p.grad.norm().item() < 1e-8, k
            continue
        check_grad_summary(g, k, p.grad, rtol=1e-9)
    for name_, calls in stats.items():
        rm, rv = torch.zeros_like(calls[0][0]), torch.ones_like(calls[0][1])
        for mean, var_unbiased in calls:
            rm, rv = 0.9 * rm + 0.1 * mean, 0.9 * rv + 0.1 * var_unbiased
        np.testing.assert_allclose(rm.numpy(), g["bn|" + name_ + ".running_mean"], rtol=1e-9, atol=1e-12, err_msg=name_)
        np.testing.assert_allclose(rv.numpy(), g["bn|" + name_ + ".running_var"], rtol=1e-9, atol=1e-12, err_msg=name_)


def test_fixtures_hold_shared_junctions_and_untouched_nodes():
    """The wireframes are what merge_line_endpoints makes: junctions ending 3 or more lines, nodes no line touches;
    case a has M != N, neither a multiple of 8; b pads its junctions (force_num_lines)."""
    for name in ("a_eval", "b_train"):
        g, _, _, data = O.load_case(GOLDEN, name)
        for i in "01":
            idx, n = data[f"lines_junc_idx{i}"], data[f"keypoints{i}"].shape[1]
            for b in range(idx.shape[0]):
                deg = torch.bincount(idx[b].reshape(-1), minlength=n)
                assert int(deg.max()) >= 3 and int((deg == 0).sum()) > 0
                assert int((deg[:2 * idx.shape[1]] == 0).sum()) > 0  # inside the line head's first 2L nodes too
    g, _, _, data = O.load_case(GOLDEN, "a_eval")
    M, N = data["keypoints0"].shape[1], data["keypoints1"].shape[1]
    assert M != N and M % 8 and N % 8 and data["keypoints0"].shape[0] == 1
    assert (g["pred|matches0"] > -1).sum() > 0 and (g["pred|line_matches0"] > -1).sum() > 0


def test_degenerate_pred_of_a_view_without_keypoints():
    """The reference's early-exit pred (gluestick.py:163-195), key for key, with its dtypes and shapes, two of which are
    not what the names suggest: log_assignment is [B, M, N] (no bins) and line_matching_scores1 is [B, N]."""
    g, conf, _, data = O.load_case(GOLDEN, "d_no_keypoints", dtype=torch.float32)
    pred = GlueStick(dict(conf)).eval()(data)
    B, M, N = 1, 0, data["keypoints1"].shape[1]
    L0, L1 = 0, data["lines1"].shape[1]
    assert N > 0 and L1 > 0 and N != L1
    shapes = {"log_assignment": (B, M, N), "matches0": (B, M), "matches1": (B, N), "matching_scores0": (B, M),
              "matching_scores1": (B, N), "line_log_assignment": (B, L0, L1), "line_matches0": (B, L0),
              "line_matches1": (B, L1), "line_matching_scores0": (B, L0), "line_matching_scores1": (B, N)}
    assert set(pred) == set(shapes) == {k[len("pred|"):] for k in g if k.startswith("pred|")}
    for k, shape in shapes.items():
        assert tuple(pred[k].shape) == shape == g["pred|" + k].shape, k
        assert pred[k].dtype == (torch.int64 if "matches" in k and "scores" not in k else torch.float32), k
        assert np.array_equal(pred[k].numpy(), g["pred|" + k]), k


# ---------------------------------------------------------------------------------------------- weights by name
@pytest.fixture
def caches(tmp_path, monkeypatch):
    """DATA_PATH of a stand-in gluefactory.settings, TORCH_HOME, and no download."""
    data_path = tmp_path / "data"
    data_path.mkdir()
    pkg, settings = types.ModuleType("gluefactory"), types.ModuleType("gluefactory.settings")
    settings.DATA_PATH = data_path
    pkg.settings = settings
    monkeypatch.setitem(sys.modules, "gluefactory", pkg)
    monkeypatch.setitem(sys.modules, "gluefactory.settings", settings)
    monkeypatch.setenv("TORCH_HOME", str(tmp_path / "torch"))

    def no_download(*args, **kwargs):
        pytest.fail(f"a download was attempted: {args} {kwargs}")

    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", no_download)
    return data_path, tmp_path / "torch" / "hub" / "checkpoints"


def _no_gluefactory(monkeypatch):
    monkeypatch.setitem(sys.modules, "gluefactory", None)
    monkeypatch.setitem(sys.modules, "gluefactory.settings", None)


GS_CONF = {"GNN_layers": ["self", "cross"] * 2}


def _gs_state(seed):
    return synthetic.make_gluestick_weights(GlueStick(dict(GS_CONF)).state_dict(), seed=seed)


def _assert_same_state(a, b):
    a, b = a.state_dict(), b.state_dict()
    assert list(a) == list(b)
    for k in a:
        assert torch.equal(a[k], b[k]), k


def test_gluestick_weights_by_name_from_data_path(caches):
    data_path, _ = caches
    sd = _gs_state(301)
    fname = data_path / "weights" / "checkpoint_GlueStick_MD_v0.1_arxiv.tar"
    fname.parent.mkdir()
    torch.save(sd, fname)
    by_name = GlueStick(dict(GS_CONF, weights="checkpoint_GlueStick_MD"))
    by_path = GlueStick(dict(GS_CONF, weights=str(fname)))
    _assert_same_state(by_name, by_path)
    assert torch.equal(by_name.state_dict()["final_proj.weight"], sd["final_proj.weight"])
    # a full glue-factory checkpoint ("model" with the pipeline's matcher. / DDP module. prefixes) under another version
    torch.save({"model": {"module.matcher." + k: v for k, v in _gs_state(302).items()}},
               data_path / "weights" / "checkpoint_GlueStick_MD_v0.2.tar")
    wrapped = GlueStick(dict(GS_CONF, weights="checkpoint_GlueStick_MD", version="v0.2"))
    assert torch.equal(wrapped.state_dict()["bin_score"], _gs_state(302)["bin_score"])


def test_gluestick_existing_path_wins_over_the_name(caches, tmp_path, monkeypatch):
    data_path, _ = caches
    (data_path / "weights").mkdir()
    torch.save(_gs_state(311), data_path / "weights" / "mine_v0.1_arxiv.tar")
    torch.save(_gs_state(312), tmp_path / "mine")
    monkeypatch.chdir(tmp_path)
    model = GlueStick(dict(GS_CONF, weights="mine"))
    assert torch.equal(model.state_dict()["final_proj.weight"], _gs_state(312)["final_proj.weight"])


def test_gluestick_missing_name_lists_every_path(caches):
    data_path, _ = caches
    with pytest.raises(FileNotFoundError) as e:
        GlueStick(dict(GS_CONF, weights="checkpoint_GlueStick_MD"))
    msg = str(e.value)
    assert "'checkpoint_GlueStick_MD'" in msg
    assert str(data_path / "weights" / "checkpoint_GlueStick_MD_v0.1_arxiv.tar") in msg
    assert not (data_path / "weights").exists()  # nothing is created either


def test_gluestick_without_gluefactory_skips_data_path(tmp_path, monkeypatch):
    _no_gluefactory(monkeypatch)
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", lambda *a, **k: pytest.fail("download attempted"))
    with pytest.raises(FileNotFoundError) as e:
        GlueStick(dict(GS_CONF, weights="checkpoint_GlueStick_MD"))
    assert "tried: checkpoint_GlueStick_MD (" in str(e.value)
    torch.save(_gs_state(321), tmp_path / "w.tar")
    model = GlueStick(dict(GS_CONF, weights=str(tmp_path / "w.tar")))
    assert torch.equal(model.state_dict()["line_bin_score"], _gs_state(321)["line_bin_score"])


LG_CONF = {"n_layers": 2}


def _lg_state(seed):
    return {k: v for k, v in synthetic.make_weights(dict(synthetic.DEFAULT_CONF, **LG_CONF), seed=seed).items()}


def _legacy(sd):
    """The key names of the first LightGlue releases: transformers.{i}.self_attn.* was self_attn.{i}.*, likewise
    cross_attn (lightglue.py:384-391)."""
    out = {}
    for k, v in sd.items():
        parts = k.split(".")
        out[".".join([parts[2], parts[1]] + parts[3:]) if parts[0] == "transformers" else k] = v
    return out


def test_lightglue_weights_by_name_from_the_hub_cache(caches):
    _, hub = caches
    hub.mkdir(parents=True)
    sd = _lg_state(331)
    legacy = _legacy(sd)
    assert "self_attn.1.Wqkv.weight" in legacy and "cross_attn.0.to_qk.bias" in legacy
    torch.save(legacy, hub / "superpoint_v0-1_arxiv.pth")
    by_name = LightGlue(dict(LG_CONF, weights="superpoint"))
    by_path = LightGlue(dict(LG_CONF, weights=str(hub / "superpoint_v0-1_arxiv.pth")))
    _assert_same_state(by_name, by_path)
    for k, v in sd.items():  # the legacy names were renamed on load
        assert torch.equal(by_name.state_dict()[k], v), k
    torch.save(_lg_state(332), hub / "disk_v0-2.pth")
    other = LightGlue(dict(LG_CONF, weights="disk", weights_from_version="v0.2"))
    assert torch.equal(other.state_dict()["posenc.Wr.weight"], _lg_state(332)["posenc.Wr.weight"])


def test_lightglue_data_path_comes_before_the_hub_cache(caches):
    data_path, hub = caches
    hub.mkdir(parents=True)
    torch.save(_lg_state(341), hub / "superpoint_v0-1_arxiv.pth")
    torch.save(_lg_state(342), data_path / "superpoint")
    model = LightGlue(dict(LG_CONF, weights="superpoint"))
    assert torch.equal(model.state_dict()["posenc.Wr.weight"], _lg_state(342)["posenc.Wr.weight"])


def test_lightglue_missing_name_lists_every_path(caches):
    data_path, hub = caches
    with pytest.raises(FileNotFoundError) as e:
        LightGlue(dict(LG_CONF, weights="aliked"))
    msg = str(e.value)
    for path in ("aliked", str(data_path / "aliked"), str(hub / "aliked_v0-1_arxiv.pth")):
        assert path in msg, (path, msg)


def test_lightglue_without_gluefactory_skips_data_path(tmp_path, monkeypatch):
    _no_gluefactory(monkeypatch)
    monkeypatch.setenv("TORCH_HOME", str(tmp_path / "torch"))
    monkeypatch.setattr(torch.hub, "load_state_dict_from_url", lambda *a, **k: pytest.fail("download attempted"))
    hub = tmp_path / "torch" / "hub" / "checkpoints"
    with pytest.raises(FileNotFoundError) as e:
        LightGlue(dict(LG_CONF, weights="sift"))
    assert f"tried: sift, {hub / 'sift_v0-1_arxiv.pth'} (" in str(e.value)
    hub.mkdir(parents=True)
    torch.save(_lg_state(351), hub / "sift_v0-1_arxiv.pth")
    model = LightGlue(dict(LG_CONF, weights="sift"))
    assert torch.equal(model.state_dict()["posenc.Wr.weight"], _lg_state(351)["posenc.Wr.weight"])


def test_superglue_weights_resolution_is_unchanged(tmp_path, monkeypatch):
    """SuperGlue keeps its own lookup: torch-hub's cache only, no DATA_PATH."""
    from gluefactory_b200.matchers.superglue import SuperGlue

    monkeypatch.setenv("TORCH_HOME", str(tmp_path / "torch"))
    path = os.path.join(str(tmp_path / "torch"), "hub", "checkpoints", "superglue_outdoor.pth")
    with pytest.raises(FileNotFoundError, match="superglue_outdoor.pth") as e:
        SuperGlue._weights_path("outdoor")
    assert path in str(e.value)
