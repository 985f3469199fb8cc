"""CPU: GlueStick with 128-channel descriptors (the DISK variant of the shipped GlueStick configs: 4 heads of 32
channels).  The fp64 oracle (oracle/gluestick_oracle.py) against the fixture produced by the unmodified reference
(tests/golden/gluestick_d128_l4_n160.npz, scripts/make_gluestick_d128_golden.py), the plugin's state_dict layout,
the widths it refuses, and the head-dimension entry points of the C ABI.  The numerics run on the GPU
(tests/test_gpu_attention_hd32.py, tests/test_gpu_gluestick_d128.py)."""
import ast
import os
import re
import sys

import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.gluestick import GlueStick
from tests.util import GOLDEN, check_grad_summary

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAME = "gluestick_d128_l4_n160"


def load_golden():
    g = dict(np.load(os.path.join(GOLDEN, NAME + ".npz"), allow_pickle=False))
    conf = ast.literal_eval(str(g["meta|conf"]))
    B, N, L, seed = (int(g["meta|" + k]) for k in ("B", "N", "L", "seed"))
    return g, conf, B, N, L, seed


def test_oracle_matches_reference_golden():
    from oracle import gluestick_oracle as G

    g, conf, B, N, L, seed = load_golden()
    assert conf["descriptor_dim"] == conf["input_dim"] == 128
    w = {k: (v.double() if v.is_floating_point() else v)
         for k, v in synthetic.make_gluestick_weights(GlueStick(dict(conf)).state_dict(), seed=seed).items()}
    params = {k: v.requires_grad_(True) for k, v in w.items() if v.is_floating_point() and "running_" not in k}
    ww = {**w, **params}
    data = synthetic.make_gluestick_batch(B, N, L, seed + 1, D=128, dtype=torch.float64)
    stats = {}
    pred = G.gluestick_forward(ww, data, conf, bn_stats=stats)
    losses = G.gluestick_loss(ww, pred, data, conf)
    losses["total"].mean().backward()
    for k in ["matches0", "matches1", "line_matches0", "line_matches1"]:
        assert np.array_equal(pred[k].numpy(), g["pred|" + k]), k
    for k in ["log_assignment", "line_log_assignment", "raw_line_scores", "matching_scores0", "matching_scores1",
              "line_matching_scores0"]:
        np.testing.assert_allclose(pred[k].detach().numpy(), g["pred|" + k], rtol=1e-9, atol=1e-9, err_msg=k)
    assert set(losses) == {k[len("loss|"):] for k in g if k.startswith("loss|")}
    for k, v in losses.items():
        np.testing.assert_allclose(v.detach().numpy(), g["loss|" + k], rtol=1e-9, atol=1e-12, err_msg=k)
    for k, p in params.items():
        if float(g[f"grad|{k}|norm"]) < 1e-9:  # a conv bias in front of a BatchNorm: zero in theory, rounding noise
            assert p.grad.norm().item() < 1e-8, k
            continue
        check_grad_summary(g, k, p.grad, rtol=1e-9)
    # running statistics: momentum 0.1, one update per call (image 0 then image 1)
    assert {k[len("bn|"):].rsplit(".", 1)[0] for k in g if k.startswith("bn|")} == set(stats)
    for name, calls in stats.items():
        rm, rv = torch.zeros_like(calls[0][0]), torch.ones_like(calls[0][1])
        for mean, var_unbiased in calls:
            rm, rv = 0.9 * rm + 0.1 * mean, 0.9 * rv + 0.1 * var_unbiased
        np.testing.assert_allclose(rm.numpy(), g["bn|" + name + ".running_mean"], rtol=1e-9, atol=1e-12, err_msg=name)
        np.testing.assert_allclose(rv.numpy(), g["bn|" + name + ".running_var"], rtol=1e-9, atol=1e-12, err_msg=name)


def test_state_dict_layout_equals_reference():
    """Names from the fixture (every parameter has a gradient there, every running statistic an entry), shapes from the
    fixture's full-size entries, and -- where the build staged the reference under oracle/_ref -- names and shapes of
    the reference module itself, loaded strictly."""
    g, conf, *_ = load_golden()
    model = GlueStick(dict(conf))
    sd = model.state_dict()
    assert {k[len("grad|"):].rsplit("|", 1)[0] for k in g if k.startswith("grad|")} == {n for n, _ in model.named_parameters()}
    assert {k[len("bn|"):] for k in g if k.startswith("bn|")} == {k for k in sd if "running_" in k}
    for k in g:
        if k.startswith("grad|") and k.endswith("|full"):
            name = k[len("grad|"):-len("|full")]
            assert tuple(sd[name].shape) == g[k].shape, name
        elif k.startswith("bn|"):
            assert tuple(sd[k[len("bn|"):]].shape) == g[k].shape, k
    assert tuple(model.final_proj.weight.shape) == (128, 128, 1)
    assert tuple(model.gnn.layers[0].update.attn.proj[0].weight.shape) == (128, 128, 1)
    assert tuple(model.gnn.line_layers[0].mlp[0].weight.shape) == (256, 384, 1)
    assert not hasattr(model, "input_proj")
    assert tuple(GlueStick(dict(conf, input_dim=256)).input_proj.weight.shape) == (128, 256, 1)
    saved = list(sys.path)
    try:
        from oracle import stage_reference

        if stage_reference.import_reference() is None:
            return
        from gluefactory.models import get_model

        ref = get_model("matchers.gluestick")(dict(conf, name="matchers.gluestick"))
        assert list(ref.state_dict().keys()) == list(sd.keys())
        for k, v in ref.state_dict().items():
            assert sd[k].shape == v.shape, k
        model.load_state_dict(ref.state_dict())  # strict
    finally:
        sys.path[:] = saved


@pytest.mark.parametrize("D", [64, 96, 192, 512])
def test_unsupported_descriptor_dim_raises(D):
    with pytest.raises(NotImplementedError, match="128 or 256"):
        GlueStick({"descriptor_dim": D, "input_dim": D})


@pytest.fixture(scope="module")
def built():
    sys.path.insert(0, ROOT)
    import __graft_entry__ as ge

    return ge.build()


def test_head_dim_entry_points_are_declared_bound_and_exported(built):
    from gluefactory_b200 import _lib

    hdr = open(os.path.join(ROOT, "include", "lgb200.h")).read()
    lib = _lib.load(check_device=False)
    for name, base in (("lgb200_attn_fwd_hd", "lgb200_attn_fwd"), ("lgb200_attn_bwd_hd", "lgb200_attn_bwd")):
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


def test_head_dims_other_than_32_and_64_are_refused(built):
    """The argument checks run before any CUDA call, so they are visible without a GPU: a head dim other than 32 or 64
    is LGB200_ERR_UNSUPPORTED, and so is the shared-qk backward (dq == dk) at 32.  The pointers are never dereferenced."""
    from gluefactory_b200 import _lib

    lib = _lib.load(check_device=False)
    p = [_lib.ctypes.c_void_p(256 * (i + 1)) for i in range(10)]
    for hd in (0, 16, 48, 65, 128):
        assert lib.lgb200_attn_fwd_hd(*p[:5], 2, 70, 90, 4, 1, 0.2, _lib.BF16, hd, None) == -3, hd
        assert lib.lgb200_attn_bwd_hd(*p, 2, 70, 90, 4, 1, 0.2, _lib.F32, hd, None) == -3, hd
        assert b"head_dim" in lib.lgb200_last_error()
    q, dq = p[0], p[6]
    assert lib.lgb200_attn_bwd_hd(q, q, *p[2:6], dq, dq, *p[8:], 2, 64, 64, 4, 1, 0.2, _lib.BF16, 32, None) == -3
    assert b"head_dim 64 only" in lib.lgb200_last_error()
    # the workspace does not depend on the head dim
    assert lib.lgb200_attn_bwd_ws_floats(2, 70, 90, 4) == 2 * 2 * 4 * 128
