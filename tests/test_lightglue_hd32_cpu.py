"""CPU: LightGlue at head dimension 32 -- `descriptor_dim 128` with 4 heads and `descriptor_dim 256` with 8 heads.  The
fp64 oracle (oracle/lightglue_oracle.py) against the fixtures produced by the unmodified reference
(scripts/make_lightglue_hd32_golden.py), the plugin's state_dict layout, the head dims it refuses, and the rotary and
position-encoder entry points of the C ABI at head dim 32.  The numerics run on the GPU (tests/test_gpu_rope_hd32.py,
tests/test_gpu_lightglue_hd32.py).  The eval-mode point-pruning fixture has no oracle counterpart (the oracle restates
the training path); the GPU test holds the plugin to it."""
import os
import re
import sys

import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.lightglue import LightGlue
from oracle import lightglue_oracle as O
from tests.util import GOLDEN, check_grad_summary, load_case

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HD32_CASES = ["lg_hd32_d128_h4_l3_n128", "lg_hd32_d128_h4_l3_m80_n112", "lg_hd32_d256_h8_l2_n128",
              "lg_hd32_sift_d128_h4_l2_n96"]


@pytest.mark.parametrize("name", HD32_CASES)
def test_oracle_matches_reference_golden(name):
    g, conf, w, data = load_case(name)
    assert conf["descriptor_dim"] // conf["num_heads"] == 32
    assert tuple(w["posenc.Wr.weight"].shape) == (16, 4 if conf.get("add_scale_ori") else 2)
    for p in w.values():
        p.requires_grad_(True)
    pred = O.lightglue_forward(w, data, conf)
    losses = O.lightglue_loss(w, pred, data, conf, training=True)
    losses["total"].mean().backward()
    assert np.array_equal(pred["matches0"].numpy(), g["pred|matches0"])
    assert np.array_equal(pred["matches1"].numpy(), g["pred|matches1"])
    assert (g["pred|matches0"] > -1).sum() > 20  # the index comparison is not vacuous
    np.testing.assert_allclose(pred["matching_scores0"].detach().numpy(), g["pred|matching_scores0"], rtol=1e-9, atol=1e-12)
    np.testing.assert_allclose(pred["log_assignment"].detach().numpy(), g["pred|log_assignment"], rtol=1e-9, atol=1e-9)
    for k in ["total", "last", "assignment_nll", "nll_pos", "nll_neg", "num_matchable", "num_unmatchable",
              "confidence", "row_norm"]:
        # the reference evaluates the confidence BCE against a float32 target even in double mode (lightglue.py:91-92):
        # 1e-6 on the two entries that include it, as for the head-dim-64 fixtures
        rtol = 1e-6 if k in ("total", "confidence") else 1e-9
        np.testing.assert_allclose(losses[k].detach().numpy(), g["loss|" + k], rtol=rtol, atol=1e-12, err_msg=k)
    for k, p in w.items():
        check_grad_summary(g, k, p.grad, rtol=1e-6)


def test_pruning_fixture_is_a_head_dim_32_pruning_case():
    import ast

    g = dict(np.load(os.path.join(GOLDEN, "lg_hd32_d128_h4_adaptive_prune.npz")))
    conf = ast.literal_eval(str(g["meta|conf"]))
    assert conf["descriptor_dim"] // conf["num_heads"] == 32 and conf["width_confidence"] > 0
    assert float(g["meta|min_margin"]) > 2e-4
    M, N, L = int(g["meta|M"]), int(g["meta|N"]), conf["n_layers"]
    kept0 = g["pred|log_assignment"].shape[1] - 1
    assert 20 < kept0 < M - 20 and int((g["pred|prune0"] == L).sum()) == kept0
    assert g["pred|matches0"].shape == (1, M) and g["pred|matches1"].shape == (1, N)


@pytest.mark.parametrize("D,H", [(128, 4), (256, 8)])
def test_state_dict_layout_equals_reference(D, H):
    """Names and shapes from the synthetic spec (which the fixtures' reference modules loaded), and -- where the build
    staged the reference under oracle/_ref -- names, order and shapes of the reference module itself, loaded strictly."""
    conf = dict(synthetic.DEFAULT_CONF, descriptor_dim=D, input_dim=D, num_heads=H, n_layers=3)
    model = LightGlue(dict(conf))
    sd = {k: v for k, v in model.state_dict().items() if k != "confidence_thresholds"}
    spec = synthetic.state_dict_spec(conf)
    assert list(sd) == [n for n, _ in spec]
    for n, shape in spec:
        assert tuple(sd[n].shape) == shape, n
    assert tuple(model.posenc.Wr.weight.shape) == (16, 2)
    assert tuple(LightGlue(dict(conf, add_scale_ori=True)).posenc.Wr.weight.shape) == (16, 4)
    saved = list(sys.path)
    try:
        from oracle import stage_reference

        if stage_reference.import_reference() is None:
            return
        from gluefactory.models import get_model

        ref = get_model("matchers.lightglue")(dict(conf, name="matchers.lightglue"))
        assert list(ref.state_dict().keys()) == list(model.state_dict().keys())
        for k, v in ref.state_dict().items():
            assert model.state_dict()[k].shape == v.shape, k
        model.load_state_dict(ref.state_dict())  # strict
    finally:
        sys.path[:] = saved


@pytest.mark.parametrize("D,H", [(256, 2), (256, 16), (128, 8), (512, 4), (256, 3)])
def test_head_dims_other_than_32_and_64_raise(D, H):
    with pytest.raises(NotImplementedError, match="head_dim"):
        LightGlue({"descriptor_dim": D, "input_dim": D, "num_heads": H})


@pytest.fixture(scope="module")
def built():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge

    return ge.build()


def test_rope_head_dim_entry_points_are_declared_bound_and_exported(built):
    from gluefactory_b200 import _lib

    hdr = open(os.path.join(ROOT, "include", "lgb200.h")).read()
    lib = _lib.load(check_device=False)
    for name, base in (("lgb200_rope_split_fwd_hd", "lgb200_rope_split_fwd"),
                       ("lgb200_rope_split_bwd_hd", "lgb200_rope_split_bwd")):
        decl = re.search(r"\b" + name + r"\s*\(([^)]*)\)", hdr)
        base_decl = re.search(r"\b" + base + r"\s*\(([^)]*)\)", hdr)
        assert decl and base_decl, name
        args = [a.strip() for a in decl.group(1).split(",")]
        base_args = [a.strip() for a in base_decl.group(1).split(",")]
        # the same arguments as the head-dim-64 entry point, with `int head_dim` in front of the stream
        assert args == base_args[:-1] + ["int head_dim"] + base_args[-1:], name
        restype, argtypes = _lib.SIGNATURES[name]
        assert len(argtypes) == len(args) and argtypes[-2] is _lib._i, name
        assert _lib.SIGNATURES[base][1] == argtypes[:-2] + argtypes[-1:], name
        assert hasattr(lib, name) and _lib.KERNELS_PER_CALL[name] == _lib.KERNELS_PER_CALL[base], name


def test_rope_head_dims_other_than_32_and_64_are_refused(built):
    """The argument checks run before any CUDA call, so they are visible without a GPU: a head dim other than 32 or 64
    is LGB200_ERR_UNSUPPORTED.  The pointers are never dereferenced."""
    from gluefactory_b200 import _lib

    lib = _lib.load(check_device=False)
    p = [_lib.ctypes.c_void_p(256 * (i + 1)) for i in range(8)]
    for hd in (0, 16, 48, 128):
        for dt in (_lib.F32, _lib.BF16):
            assert lib.lgb200_rope_split_fwd_hd(*p[:5], 4096, 4, dt, hd, None) == -3, hd
            assert b"head_dim" in lib.lgb200_last_error()
            assert lib.lgb200_rope_split_bwd_hd(*p, 4096, 4, dt, hd, None) == -3, hd
            assert b"head_dim" in lib.lgb200_last_error()


def test_posenc_wgrad_refuses_other_angle_counts(built):
    """C = head_dim / 2 angles: 32 or 16.  Anything else is refused before any CUDA call."""
    from gluefactory_b200 import _lib

    lib = _lib.load(check_device=False)
    p = [_lib.ctypes.c_void_p(256 * (i + 1)) for i in range(3)]
    for C in (0, 8, 24, 33, 64):
        for kd in (2, 4):
            assert lib.lgb200_posenc_wgrad(*p, 1000, C, kd, None) == -1, C
            assert b"C must be 32 or 16" in lib.lgb200_last_error()
