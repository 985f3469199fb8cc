"""GPU: the kernel launches of the 128-channel and 8-head models (LightGlue at descriptor_dim 128 / 4 heads and 256 / 8
heads, GlueStick at 128 channels) against fp64 at their training sizes, with the launch tables checked against what the
engine and the matchers actually launch.

A. Launch census.  ops.linear, wgrad_bf16, gemm_bf16, attn_fwd / attn_bwd / attn_bwd_shared_qk, assign_fused_stats /
   assign_fused_bwd, colsum and head_token_fwd / head_token_bwd are wrapped by recording shims (the engine, LinearFn and
   the matchers look them up through the ops module), and one bf16 training step (forward, loss, backward) runs per
   model configuration at a small size.  Each call is reduced to a signature without its token or keypoint counts
   (sizes that are not channel widths print as "n"); every signature must be a row of this file's tables or of the
   benchmark-shape lists of tests/test_gpu_tensor_core_kernels.py, and every row of this file's tables must be seen.
   linear: (N, K, w_is_kn, bias, out dtype, accumulate, A pitch / K, W pitch / its width, W column offset / its
   width, C pitch / N); wgrad: (M, N, dy pitch / M, x pitch / N); gemm_bf16: (M, N, K, A / B MN-major, out dtype).

B. GEMMs at training size, exact and bounded (units, operands and bounds of test_gpu_tensor_core_kernels): every
   linear / wgrad / gemm_bf16 row of the tables at its configuration's token count (LightGlue: 32 pairs x 2 x 2048 =
   131072 tokens; GlueStick: 8 pairs x 2 x 3072 nodes = 49152).  W is a column block of a wider matrix where the engine
   passes one (ffn.0's W0[:, D:] and W0[:, :D]: pitch 2D, column offset D or 0), A and C are column blocks where the
   engine's are, and the columns of C's buffer outside C must keep their NaN pattern.  Each test asserts the property
   its row exists for: more than 132 A-panel items with one n-tile (N <= 128: several items per persistent CTA, the
   next panel prefetched after the item's B loads), a pitched W, or the split count of the split-K weight gradient.

C. Attention at head dim 32 (bounds of tests/test_gpu_attention_hd32.py): LightGlue's launch, 64 sequences x 2048
   keypoints at 4 and 8 heads, self (kv_shift 0) and cross (kv_shift 32), every sequence checked against fp64, each
   launch run twice (bit-identical) into guarded buffers; 8 heads at three tile-edge pairs; and
   engine._attend_bwd_shared_qk at head dim 32 (dq and dk written separately, added in bf16) against the fp64 total
   gradient of the shared tensor, dQ of its own direction plus dK of the other:
       |dqk - (dQ + dK)| <= bdQ + bdK + UBF |dQ + dK|
   (attn_ref's bounds of the two bf16 gradients, and the rounding of their bf16 sum).

D. The fused assignment head at D = 128 runs at the training launch through ASSIGN_SHAPES of
   test_gpu_tensor_core_kernels.  head_token_bwd at 131072 tokens and D = 128 (the one-channel-slot template with half
   of each warp's slots empty), and the back-to-back column sums over the 128-channel layer's widths, with the chains
   of tests/test_gpu_step_kernels.py.

E. CPU negative controls: each new check rejects a wrong answer built from its own reference.

Budget: under 3 minutes and 20 GiB peak device memory on one H100, recorded by the module fixture.
"""
import ast
import math
import os
import time

import numpy as np
import pytest
import torch

from gluefactory_b200 import _lib, engine, ops, synthetic
from tests.test_gpu_attention_hd32 import SCALE as SCALE32
from tests.test_gpu_attention_hd32 import _inputs as _inputs32
from tests.test_gpu_attention_hd32 import _run as _run32
from tests.test_gpu_tensor_core_kernels import (BENCH_LINEAR, DEV, F32_GUARD, BF16_GUARD, U32, UBF, _addend,
                                                _cpu_gen, _draw, _gemm_case, _gen, _splitk_chain, _trunc_bf16, _within,
                                                _Worst, attn_ref, check_attn_fwd, check_exact, gemm_bound)
from tests.util import GOLDEN, report

GPU = pytest.mark.gpu
TOK_LG = 131072  # LightGlue: 32 pairs x (2048 + 2048) keypoints
TOK_GS = 49152   # GlueStick: 8 pairs x (3072 + 3072) nodes
SMS = 132        # persistent CTAs of the dense GEMMs on an H100 SXM
BF, F32 = "bf16", "f32"


@pytest.fixture(scope="module", autouse=True)
def _file_budget():
    """Wall time and peak device memory of this file (the machines running it are shared)."""
    if not torch.cuda.is_available():
        yield
        return
    torch.cuda.reset_peak_memory_stats()
    t = time.time()
    yield
    torch.cuda.synchronize()
    report("test_gpu_layer_launches", seconds=time.time() - t,
           peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)


# ================================================================================================
# launch tables
# ================================================================================================
# linear rows: (name, T, N, K, w_is_kn, bias, out, accumulate, A pitch / K, W pitch / width, W offset / width,
#               C pitch / N, property).  property: "panel" = A-panel kernel with one n-tile and > 132 items;
#               "w_pitch" = W a column block of ffn.0's weight; "" = the launch form only.
LINEAR_ROWS = [
    # LightGlue, D = 128, 4 heads (131072 tokens)
    ("d128 qkv", TOK_LG, 384, 128, False, True, BF, False, 2, 1, 0, 1, ""),
    ("d128 out / to_out", TOK_LG, 128, 128, False, True, BF, False, 1, 1, 0, 2, "panel"),
    ("d128 to_qk / to_v", TOK_LG, 128, 128, False, True, BF, False, 2, 1, 0, 1, "panel"),
    ("d128 final_proj", TOK_LG, 128, 128, False, True, BF, False, 1, 1, 0, 1, "panel"),
    ("d128 ffn.0", TOK_LG, 256, 256, False, True, BF, False, 1, 1, 0, 1, ""),
    ("d128 ffn.3", TOK_LG, 128, 256, False, True, BF, False, 1, 1, 0, 1, "panel"),
    ("d128 ffn.3 dgrad", TOK_LG, 256, 128, True, False, BF, False, 1, 1, 0, 1, ""),
    ("d128 ffn.0 dgrad W0[:, D:]", TOK_LG, 128, 256, True, False, BF, False, 1, 2, 1, 1, "panel w_pitch"),
    ("d128 ffn.0 dgrad += W0[:, :D]", TOK_LG, 128, 256, True, False, F32, True, 1, 2, 0, 1, "panel w_pitch"),
    ("d128 out / to_out / final_proj dgrad", TOK_LG, 128, 128, True, False, BF, False, 1, 1, 0, 1, "panel"),
    ("d128 to_qk / to_v dgrad +=", TOK_LG, 128, 128, True, False, F32, True, 1, 1, 0, 1, "panel"),
    ("d128 qkv dgrad +=", TOK_LG, 128, 384, True, False, F32, True, 1, 1, 0, 1, ""),
    # LightGlue, D = 256 (4 or 8 heads): the forms the benchmark-shape list does not have
    ("d256 qkv", TOK_LG, 768, 256, False, True, BF, False, 2, 1, 0, 1, ""),
    ("d256 out / to_out", TOK_LG, 256, 256, False, True, BF, False, 1, 1, 0, 2, ""),
    ("d256 to_qk / to_v", TOK_LG, 256, 256, False, True, BF, False, 2, 1, 0, 1, ""),
    ("d256 ffn.3 dgrad", TOK_LG, 512, 256, True, False, BF, False, 1, 1, 0, 1, ""),
    ("d256 ffn.0 dgrad W0[:, D:]", TOK_LG, 256, 512, True, False, BF, False, 1, 2, 1, 1, "w_pitch"),
    ("d256 ffn.0 dgrad += W0[:, :D]", TOK_LG, 256, 512, True, False, F32, True, 1, 2, 0, 1, "w_pitch"),
    ("d256 to_qk / to_v dgrad +=", TOK_LG, 256, 256, True, False, F32, True, 1, 1, 0, 1, ""),
    # GlueStick's 1x1 convolutions (LinearFn; 49152 nodes) at 128 and 256 channels
    ("gluestick conv 64->128", TOK_GS, 128, 64, False, True, BF, False, 1, 1, 0, 1, "panel"),
    ("gluestick conv 64->128 dgrad", TOK_GS, 64, 128, True, False, BF, False, 1, 1, 0, 1, "panel"),
    ("gluestick conv 128->256", TOK_GS, 256, 128, False, True, BF, False, 1, 1, 0, 1, ""),
    ("gluestick conv 128->256 dgrad", TOK_GS, 128, 256, True, False, BF, False, 1, 1, 0, 1, "panel"),
    ("gluestick d128 conv 384->256", TOK_GS, 256, 384, False, True, BF, False, 1, 1, 0, 1, ""),
    ("gluestick d128 conv 384->256 dgrad", TOK_GS, 384, 256, True, False, BF, False, 1, 1, 0, 1, ""),
    ("gluestick d256 conv 768->512", TOK_GS, 512, 768, False, True, BF, False, 1, 1, 0, 1, ""),
    ("gluestick d256 conv 768->512 dgrad", TOK_GS, 768, 512, True, False, BF, False, 1, 1, 0, 1, ""),
    ("gluestick d256 conv 512->512 dgrad", TOK_GS, 512, 512, True, False, BF, False, 1, 1, 0, 1, ""),
]
# wgrad rows: (name, T, M, N, dy pitch / M, x pitch / N, least split count on a 114..132-SM H100)
WGRAD_ROWS = [
    ("d128 qkv: dqkv^T x16", TOK_LG, 384, 128, 1, 2, 34),
    ("d128 out / to_out / final_proj", TOK_LG, 128, 128, 1, 1, 100),
    ("d128 to_qk / to_v: d^T x1_16", TOK_LG, 128, 128, 1, 2, 100),
    ("d128 ffn.3", TOK_LG, 128, 256, 1, 1, 50),
    ("d256 qkv: dqkv^T x16", TOK_LG, 768, 256, 1, 2, 8),
    ("d256 to_qk / to_v: d^T x1_16", TOK_LG, 256, 256, 1, 2, 25),
    ("gluestick conv 64->128", TOK_GS, 128, 64, 1, 1, 100),
    ("gluestick conv 128->256", TOK_GS, 256, 128, 1, 1, 50),
    ("gluestick d128 conv 384->256", TOK_GS, 256, 384, 1, 1, 19),
    ("gluestick d256 conv 768->512", TOK_GS, 512, 768, 1, 1, 4),
]
# gemm_bf16 rows: (name, batch, M, N, K, a_mn, b_mn, out)
GEMM_ROWS = [
    ("gluestick d128 sim", 8, 2048, 2048, 128, False, False, F32),
    ("gluestick d128 d(a)", 8, 2048, 128, 2048, False, True, BF),
    ("gluestick d128 d(b)", 8, 2048, 128, 2048, True, True, BF),
]
# attention rows: (entry, H, head dim, kv_shift kind, Nq == Nk); tested here (hd 32) or by the hd-64 suites
ATTN_ROWS = [(e, H, hd, s, True) for e in ("attn_fwd", "attn_bwd") for H, hd in ((4, 32), (8, 32)) for s in ("0", "half")] \
    + [(e, H, hd, "0", False) for e in ("attn_fwd", "attn_bwd") for H, hd in ((4, 32), (8, 32))] \
    + [("attn_bwd_shared_qk", 4, 64, "half", True)]
# head_token_fwd is a per-token kernel (no cross-CTA reduction), checked by test_gpu_kernels::test_head_token_kernels
OTHER_ROWS = [("assign_fused_stats", 128), ("assign_fused_bwd", 128), ("head_token_fwd", 128, BF, True),
              ("head_token_fwd", 128, BF, False), ("head_token_bwd", 128, BF), ("colsum", 384, BF), ("colsum", 128, BF),
              ("colsum", 256, BF)]

# the signatures the hd-64 / 256-channel suites already test (tests/test_gpu_tensor_core_kernels.py,
# tests/test_gpu_step_kernels.py, tests/test_gpu_kernels.py)
_DT = {torch.bfloat16: BF, torch.float32: F32}
KNOWN = {("linear", N, K, kn, bias, _DT[odt], acc, 1, 1, 0, 1) for _, _, N, K, kn, bias, odt, acc in BENCH_LINEAR}
KNOWN |= {("wgrad", M, N, 1, 1) for M, N in [(768, 256), (256, 256), (512, 512), (256, 512)]}
KNOWN |= {("gemm_bf16", "n", "n", 256, False, False, F32), ("gemm_bf16", "n", 256, "n", False, True, BF),
          ("gemm_bf16", "n", 256, "n", True, True, BF)}
KNOWN |= {(e, 4, 64, s, True) for e in ("attn_fwd", "attn_bwd") for s in ("0", "half")}
KNOWN |= {(e, 4, 64, "0", False) for e in ("attn_fwd", "attn_bwd")}
KNOWN |= {("assign_fused_stats", 256), ("assign_fused_bwd", 256), ("head_token_fwd", 256, BF, True),
          ("head_token_fwd", 256, BF, False),
          ("head_token_bwd", 256, BF), ("colsum", 768, BF), ("colsum", 256, BF), ("colsum", 512, BF)}


def _lin_sig(row):
    _, _, N, K, kn, bias, odt, acc, ap, wp, wo, cp, _ = row
    return ("linear", N, K, kn, bias, odt, acc, ap, wp, wo, cp)


def table_signatures():
    """{signature: row name} of this file's tables."""
    t = {_lin_sig(r): r[0] for r in LINEAR_ROWS}
    t.update({("wgrad", M, N, dp, xp): name for name, _, M, N, dp, xp, _ in WGRAD_ROWS})
    t.update({("gemm_bf16", "n" if M > 512 else M, "n" if N > 512 else N, "n" if K > 512 else K, am, bm, o): name
              for name, _, M, N, K, am, bm, o in GEMM_ROWS})
    t.update({r: " ".join(map(str, r)) for r in ATTN_ROWS + OTHER_ROWS})
    return t


def check_census(seen):
    """seen: {configuration: set of signatures}.  Every signature is a table row (or already known); every row of this
    file's tables is seen by some configuration."""
    tables = table_signatures()
    missing = sorted({(cfg, s) for cfg, sigs in seen.items() for s in sigs if s not in tables and s not in KNOWN},
                     key=repr)
    assert not missing, "launch signatures outside the tables:\n" + "\n".join(f"  {c}: {s!r}" for c, s in missing)
    everything = set().union(*seen.values()) if seen else set()
    unseen = sorted((n for s, n in tables.items() if s not in everything), key=repr)
    assert not unseen, f"table rows no configuration launches: {unseen}"


# ================================================================================================
# A. launch census
# ================================================================================================
def _n(x):
    return x if x in (32, 64, 128, 256, 384, 512, 768) else "n"


def _ratio(pitch, width):
    r = pitch / width
    return int(r) if r == int(r) else round(r, 4)


def _signature(name, args, kw):
    a = dict(kw)
    if name == "linear":
        x, w = args[0], args[1]
        kn = a.get("w_is_kn", args[5] if len(args) > 5 else False)
        bias = a.get("bias", args[2] if len(args) > 2 else None)
        out = a.get("out", args[3] if len(args) > 3 else None)
        odt = out.dtype if out is not None else a.get("out_dtype", args[4] if len(args) > 4 else torch.bfloat16)
        acc = a.get("accumulate", args[6] if len(args) > 6 else False)
        K = x.shape[1]
        N = w.shape[1] if kn else w.shape[0]
        width = w.shape[1]
        off = (w.storage_offset() % w.stride(0)) if w.stride(0) != width else 0
        return ("linear", N, K, bool(kn), bias is not None, _DT[odt], bool(acc), _ratio(x.stride(0), K),
                _ratio(w.stride(0), width), _ratio(off, width), _ratio(out.stride(0), N) if out is not None else 1)
    if name == "wgrad_bf16":
        dy, x = args[0], args[1]
        return ("wgrad", dy.shape[1], x.shape[1], _ratio(dy.stride(0), dy.shape[1]), _ratio(x.stride(0), x.shape[1]))
    if name == "gemm_bf16":
        x, y = args[0], args[1]
        am, bm = a.get("a_mn_major", False), a.get("b_mn_major", False)
        M, K = (x.shape[2], x.shape[1]) if am else (x.shape[1], x.shape[2])
        N = y.shape[2] if bm else y.shape[1]
        return ("gemm_bf16", _n(M), _n(N), _n(K), bool(am), bool(bm), _DT[a.get("out_dtype", torch.float32)])
    if name in ("attn_fwd", "attn_bwd"):
        q, k = args[0], args[1]
        shift = args[3] if name == "attn_fwd" else args[6]
        kind = "0" if shift == 0 else ("half" if 2 * shift == q.shape[0] else str(shift))
        return (name, q.shape[2], q.shape[3], kind, q.shape[1] == k.shape[1])
    if name == "attn_bwd_shared_qk":
        return (name, args[0].shape[2], args[0].shape[3], "half", True)
    if name in ("assign_fused_stats", "assign_fused_bwd"):
        return (name, args[0].shape[2])
    if name == "colsum":
        return (name, args[0].shape[1], _DT[args[0].dtype])
    if name == "head_token_fwd":
        cdt, wt = (args[5], args[3]) if len(args) > 5 else (kw["cdt"], kw.get("wt", args[3] if len(args) > 3 else None))
        return (name, args[0].shape[1], _DT[cdt], wt is not None)
    if name == "head_token_bwd":
        return (name, args[0].shape[1], _DT[args[1].dtype] if args[1] is not None else None)
    raise KeyError(name)


SHIMMED = ("linear", "wgrad_bf16", "gemm_bf16", "attn_fwd", "attn_bwd", "attn_bwd_shared_qk", "assign_fused_stats",
           "assign_fused_bwd", "colsum", "head_token_fwd", "head_token_bwd")


def _record(monkeypatch, sigs):
    for name in SHIMMED:
        orig = getattr(ops, name)

        def shim(*args, _orig=orig, _name=name, **kw):
            sigs.add(_signature(_name, args, kw))
            return _orig(*args, **kw)

        monkeypatch.setattr(ops, name, shim)


def _lightglue_step(D, H, M, N):
    from gluefactory_b200.matchers.lightglue import LightGlue

    conf = dict(synthetic.DEFAULT_CONF, descriptor_dim=D, input_dim=D, num_heads=H, n_layers=2, precision="bf16")
    model = LightGlue(conf)
    model.load_state_dict(synthetic.make_weights(conf, seed=D + H), strict=False)
    model = model.to(DEV).train()
    data = synthetic.to_device(synthetic.make_pairs(2, N, seed=M + N, D=D, M=M), DEV)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()


def _gluestick_step(D):
    from gluefactory_b200.matchers.gluestick import GlueStick

    name = "gluestick_d128_l4_n160" if D == 128 else "gluestick_l4_n160"
    conf = ast.literal_eval(str(np.load(os.path.join(GOLDEN, name + ".npz"))["meta|conf"]))
    model = GlueStick(dict(conf, precision="bf16"))
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=D), strict=True)
    model = model.to(DEV).train()
    data = synthetic.to_device(synthetic.make_gluestick_batch(2, 200, 40, D, D=D), DEV)
    pred = model(data)
    losses, _ = model.loss(pred, data)
    losses["total"].mean().backward()


CENSUS = {  # keypoint counts that are not channel widths, so that their dimensions print as "n"
    "lightglue d256 h4": lambda: _lightglue_step(256, 4, 200, 200),
    "lightglue d256 h4 M!=N": lambda: _lightglue_step(256, 4, 168, 200),
    "lightglue d128 h4": lambda: _lightglue_step(128, 4, 200, 200),
    "lightglue d128 h4 M!=N": lambda: _lightglue_step(128, 4, 168, 200),
    "lightglue d256 h8": lambda: _lightglue_step(256, 8, 200, 200),
    "lightglue d256 h8 M!=N": lambda: _lightglue_step(256, 8, 168, 200),
    "gluestick d256": lambda: _gluestick_step(256),
    "gluestick d128": lambda: _gluestick_step(128),
}


@GPU
def test_launch_census(monkeypatch):
    """Every launch of a bf16 training step of each configuration is a row of the tables, and every row is launched."""
    seen = {}
    for cfg, step in CENSUS.items():
        sigs = set()
        with monkeypatch.context() as m:
            _record(m, sigs)
            step()
        torch.cuda.synchronize()
        seen[cfg] = sigs
        report(f"census {cfg}", **{f"s{i}": repr(s).replace(" ", "") for i, s in enumerate(sorted(sigs, key=repr))})
    check_census(seen)


# ================================================================================================
# B. GEMMs at training size
# ================================================================================================
def _block(rows, width, pitch, off, dtype, fill, exact, g, K):
    """A [rows, width] column block at column offset off * width of a [rows, pitch * width] matrix of NaN / values."""
    if pitch == 1:
        return _draw((rows, width), exact, g, K) if fill else torch.empty(rows, width, device=DEV, dtype=dtype)
    big = _draw((rows, pitch * width), exact, g, K) if fill else torch.empty(rows, pitch * width, device=DEV,
                                                                               dtype=dtype)
    return big[:, off * width:(off + 1) * width]


def _linear_pitched(T, N, K, kn, bias, odt, acc, ap, wp, wo, cp, exact, seed, tag, chunk=16384):
    """ops.linear with A a column block of a [T, ap K] matrix, W a column block (pitch wp x width, column offset
    wo x width) of a wider weight, and C the first N columns of a [T, cp N] buffer (+ 8 columns) whose other columns
    must keep their NaN pattern."""
    g = _gen(seed)
    out_dtype = torch.bfloat16 if odt == BF else torch.float32
    a = _block(T, K, ap, 1 if ap > 1 else 0, torch.bfloat16, True, exact, g, K)
    wshape = (K, N) if kn else (N, K)
    wt = _block(wshape[0], wshape[1], wp, wo, torch.bfloat16, True, exact, g, K)
    assert wt.stride(0) == wp * wshape[1] and wt.storage_offset() == wo * wshape[1]
    bv = _addend((N,), exact, g, 2 ** 15) if bias else None
    alpha = 0.5 if exact else 0.7
    cbig = torch.empty(T, cp * N + 8, device=DEV, dtype=out_dtype)
    cbig.view(torch.int32 if out_dtype == torch.float32 else torch.int16).fill_(
        F32_GUARD if out_dtype == torch.float32 else BF16_GUARD)
    out = cbig[:, :N]
    c0 = None
    if acc:
        c0 = _addend((T, N), exact, g, 2 ** 20)
        out.copy_(c0)
    keep = cbig[:, N:].clone()
    ops.linear(a, wt, bias=bv, out=out, w_is_kn=kn, accumulate=acc, alpha=alpha)
    assert torch.equal(cbig[:, N:].view(torch.uint8), keep.view(torch.uint8)), (tag, "stray write")
    del keep
    W64 = wt.double().t() if kn else wt.double()  # [N, K]
    w = _Worst(tag)
    wide = []
    for s in range(0, T, chunk):
        A64 = a[s:s + chunk].double()
        ref = alpha * (A64 @ W64.t())
        add = None
        if bias:
            ref = ref + bv.double()
            add = bv.double().abs().expand_as(ref)
        if acc:
            ref = ref + c0[s:s + chunk].double()
            add = c0[s:s + chunk].double().abs() + (add if add is not None else 0)
        got = out[s:s + chunk]
        if exact:
            wide.append(check_exact(got, ref, f"{tag} rows {s}", log=False))
        else:
            w("C", (got.double() - ref).abs(), gemm_bound(A64.abs() @ W64.abs().t(), K, alpha, ref, out_dtype, add))
    if exact:
        report(tag, mismatches=0, wider_than_bf16=sum(wide) / len(wide))
    else:
        w.report()
    return sum(wide) / len(wide) if wide else None


@GPU
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "bounded"])
@pytest.mark.parametrize("row", LINEAR_ROWS, ids=[r[0] for r in LINEAR_ROWS])
def test_linear_layer_launches(row, exact):
    name, T, N, K, kn, bias, odt, acc, ap, wp, wo, cp, prop = row
    tiles_m = -(-T // 128)
    if "panel" in prop:  # A-panel kernel (K <= 256), one n-tile, several items per persistent CTA
        assert K <= 256 and N <= 128 and tiles_m > SMS, (name, T)
    if "w_pitch" in prop:
        assert wp > 1 and kn, name
    wide = _linear_pitched(T, N, K, kn, bias, odt, acc, ap, wp, wo, cp, exact, seed=N + 3 * K + wo,
                           tag=f"linear {name} T={T} {'exact' if exact else 'bounded'}")
    if exact and odt == BF:
        assert wide > 0.5, wide  # most results are rounded: a truncating store cannot hide


@GPU
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "bounded"])
@pytest.mark.parametrize("row", WGRAD_ROWS, ids=[r[0] for r in WGRAD_ROWS])
def test_wgrad_layer_launches(row, exact):
    """dW = dy^T x over all tokens, split-K; x a column block of a [T, 2N] buffer where the engine passes one."""
    name, T, M, N, dp, xp, least = row
    n_chain, splits = _splitk_chain(M, N, T)
    assert splits >= least, (name, splits)
    g = _gen(M + 7 * N + xp)
    dy = _block(T, M, dp, 0, torch.bfloat16, True, exact, g, T)
    x = _block(T, N, xp, 0, torch.bfloat16, True, exact, g, T)
    out = torch.full((M, N), float("nan"), device=DEV)
    ops.wgrad_bf16(dy, x, out=out)
    again = torch.full_like(out, float("nan"))
    ops.wgrad_bf16(dy, x, out=again)
    assert torch.equal(out, again), (name, "split-K sum order")
    del again
    ref = torch.zeros(M, N, device=DEV, dtype=torch.float64)
    absprod = torch.zeros_like(ref)
    for s in range(0, T, 16384):
        d64, x64 = dy[s:s + 16384].double(), x[s:s + 16384].double()
        ref += d64.t() @ x64
        absprod += d64.abs().t() @ x64.abs()
    tag = f"wgrad {name} T={T} {M}x{N} splits={splits} {'exact' if exact else 'bounded'}"
    if exact:
        check_exact(out, ref, tag)
    else:
        _within((out.double() - ref).abs(), gemm_bound(absprod, n_chain, 1.0, ref, torch.float32), tag)


@GPU
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "bounded"])
@pytest.mark.parametrize("row", GEMM_ROWS, ids=[r[0] for r in GEMM_ROWS])
def test_gemm_layer_launches(row, exact):
    name, batch, M, N, K, am, bm, odt = row
    wide = _gemm_case(batch, M, N, K, am, bm, torch.bfloat16 if odt == BF else torch.float32, exact, seed=M + N + K,
                      again=True, tag=f"gemm {name} {'exact' if exact else 'bounded'}")
    if exact and odt == BF:
        assert wide > 0.5, wide


# ================================================================================================
# C. attention at head dim 32
# ================================================================================================
@GPU
@pytest.mark.parametrize("shift", [0, 32], ids=["self", "cross"])
@pytest.mark.parametrize("H", [4, 8])
def test_hd32_lightglue_launch(H, shift):
    """64 sequences (32 pairs x 2 images) x 2048 keypoints, head dim 32: every sequence against fp64, forward and
    backward run twice (bit-identical), outputs in guarded buffers."""
    _run32(64, 2048, 2048, H, shift, "randn", seed=40 + H + shift, again=True, tag=f"attn hd32 lightglue H={H} "
                                                                                   f"shift={shift}")


@GPU
@pytest.mark.parametrize("Nq,Nk", [(65, 129), (1000, 63), (129, 1000)])
def test_hd32_eight_heads_tile_edges(Nq, Nk):
    _run32(2, Nq, Nk, 8, (Nq + Nk) % 2, "randn", seed=Nq * 13 + Nk, tag=f"attn hd32 H=8 Nq={Nq} Nk={Nk}")


def shared_qk_bound(r_own, r_other):
    """fp64 total gradient of a shared query / key tensor (dQ of its own direction plus dK of the other) and the bound
    of dq and dk rounded to bf16 separately, then added in bf16."""
    ref = r_own["dQ"] + r_other["dK"]
    return ref, r_own["bdQ"] + r_other["bdK"] + UBF * ref.abs()


def check_bf16_sum(dqk, dq, dk, tag):
    """dqk == dq + dk rounded to nearest-even in bf16, bit for bit.  The fp64 bound above cannot see how the last add
    rounds: its dS-rounding terms alone are over 11 UBF |dQ + dK| (measured on the randn, rising and spike regimes), so
    the add is checked exactly against the separately computed bf16 dq and dk."""
    want = (dq.float() + dk.float()).to(torch.bfloat16)
    bad = ~(dqk == want)
    assert not bad.any(), (tag, "bf16 add", int(bad.sum()), dqk[bad][:4].tolist(), want[bad][:4].tolist())


@GPU
@pytest.mark.parametrize("H", [4, 8])
@pytest.mark.parametrize("B,M,N", [(32, 2048, 2048), (3, 1000, 777)], ids=["M=N", "M!=N"])
def test_hd32_shared_qk_backward(B, M, N, H):
    """engine._attend_bwd_shared_qk at head dim 32 (LightGlue's cross block at 128 channels / 4 heads and 256 / 8):
    dqk against the fp64 total gradient of the shared tensor, and equal to the bf16 sum of the separately launched
    dq and dk; dv against fp64."""
    sizes = (B, M, N)
    g = _gen(B + M + H)
    T = B * (M + N)
    qk = (torch.randn(T, H * 32, device=DEV, generator=g) * 1.5).to(torch.bfloat16)
    v = torch.randn(T, H * 32, device=DEV, generator=g).to(torch.bfloat16)
    do = torch.randn(T, H * 32, device=DEV, generator=g).to(torch.bfloat16)
    out, lses = engine._attend_fwd(qk, qk, v, sizes, H, cross=True)
    dqk, dv = engine._attend_bwd_shared_qk(qk, v, out, lses, do, sizes, H)
    again = engine._attend_bwd_shared_qk(qk, v, out, lses, do, sizes, H)
    assert torch.equal(again[0], dqk) and torch.equal(again[1], dv)
    del again
    dq, dk, dv2 = engine._attend_bwd(qk, qk, v, out, lses, do, sizes, H, cross=True)
    assert torch.equal(dv2, dv)
    check_bf16_sum(dqk, dq, dk, f"attn hd32 shared_qk H={H} M={M} N={N}")
    del dq, dk, dv2
    # token ranges of the 2B sequences: image 0 of pair b, then image 1 of pair b
    seq = [(b * M, M) for b in range(B)] + [(B * M + b * N, N) for b in range(B)]
    tag = f"attn hd32 shared_qk H={H} B={B} M={M} N={N}"
    w = _Worst(tag)
    view = lambda t, s: t[s[0]:s[0] + s[1]].view(s[1], H, 32)  # noqa: E731
    for i in range(2 * B):
        p = (i + B) % (2 * B)
        si, sp = seq[i], seq[p]
        r_ip = attn_ref(view(qk, si), view(qk, sp), view(v, sp), SCALE32, view(out, si), view(do, si))
        r_pi = attn_ref(view(qk, sp), view(qk, si), view(v, si), SCALE32, view(out, sp), view(do, sp))
        check_attn_fwd(view(out, si), lses[0][i] if M == N else lses[i // B][i % B], r_ip, w)
        ref, bound = shared_qk_bound(r_ip, r_pi)
        w("dqk", (view(dqk, si).double() - ref).abs(), bound)
        w("dv", (view(dv, si).double() - r_pi["dV"]).abs(), r_pi["bdV"])
        del r_ip, r_pi
    w.report()


# ================================================================================================
# D. CUDA-core kernels at width 128
# ================================================================================================
@GPU
def test_head_token_bwd_d128_at_training_size():
    T, D = TOK_LG, 128
    g = _gen(31)
    x = torch.randn(T, D, device=DEV, generator=g) + torch.randn(D, device=DEV, generator=g)
    dmdw = torch.randn(T, D, device=DEV, generator=g).to(torch.bfloat16)
    dzt = torch.randn(T, 2, device=DEV, generator=g) + 0.5
    wm = torch.randn(D, device=DEV, generator=g) * 0.1
    dx, dW2, db2 = ops.head_token_bwd(x, dmdw, dzt, wm)
    again = ops.head_token_bwd(x, dmdw, dzt, wm)
    assert all(torch.equal(a, b) for a, b in zip((dx, dW2, db2), again))
    del again
    tag = f"head_token_bwd T={T} D={D} bf16"
    x64, z64 = x.double(), dzt.double()
    ref = dmdw.double() + z64[:, :1] * wm.double()
    _within((dx.double() - ref).abs(), U32 * (dmdw.double().abs() + (z64[:, :1] * wm.double()).abs()), f"{tag} dx")
    del ref
    # the launch: 592 CTAs of 8 warps; per warp over ceil(T / (592 * 8)) tokens, the 8 warps, then 592 CTA partials
    parts = _lib.load().lgb200_head_token_bwd_ws_floats(D) // (2 * D + 2)
    assert parts == 592, parts
    chain = -(-T // (parts * 8)) + 8 + parts
    _within((dW2.double() - z64.t() @ x64).abs(), chain * U32 * (z64.abs().t() @ x64.abs()), f"{tag} dW2")
    _within((db2.double() - z64.sum(0)).abs(), chain * U32 * z64.abs().sum(0), f"{tag} db2")


@GPU
def test_colsum_d128_widths_back_to_back():
    """The 128-channel layer's bias gradients: widths 384, 128, 256 and 128 one after the other on one set of arrival
    counters (the repeated width must come back bit-identical)."""
    g = _gen(19)
    widths = (384, 128, 256, 128)
    mats = {wd: (torch.randn(TOK_LG, wd, device=DEV, generator=g) + torch.randn(wd, device=DEV, generator=g))
            .to(torch.bfloat16) for wd in (384, 128, 256)}
    outs = [(wd, ops.colsum(mats[wd])) for wd in widths]
    assert torch.equal(outs[1][1], outs[3][1])
    for wd, got in outs[:3]:
        a = mats[wd].double()
        nslabs = _lib.load().lgb200_colsum_slabs(TOK_LG, wd)
        rps = -(-TOK_LG // nslabs)
        chain = -(-rps // 32) + 32 + nslabs
        _within((got.double() - a.sum(0)).abs(), chain * U32 * a.abs().sum(0), f"colsum w={wd} bf16 (d128 layer)")


# ================================================================================================
# E. negative controls (CPU, no library call)
# ================================================================================================
def test_census_check_rejects_an_unknown_launch_and_an_unseen_row():
    rows = set(table_signatures())
    check_census({"all": rows})
    with pytest.raises(AssertionError, match="outside the tables"):
        check_census({"all": rows | {("linear", 128, 256, True, False, F32, False, 1, 2, 1, 1)}})  # dmsg in fp32
    with pytest.raises(AssertionError, match="no configuration launches"):
        check_census({"all": rows - {_lin_sig(LINEAR_ROWS[7])}})


def _int_operands(g, M, N, K):
    r = int(math.isqrt(2 ** 23 // K))
    return (torch.randint(-r, r + 1, (M, K), generator=g).double(), torch.randint(-r, r + 1, (N, K), generator=g).double())


def test_pitched_w_checks_reject_the_wrong_half_and_the_wrong_pitch():
    """dmsg = dh W0[:, D:] (pitch 2D, offset D): the other half, and the block read with pitch D, both fail."""
    g = _cpu_gen(11)
    T, D = 300, 64
    dh, _ = _int_operands(g, T, 1, 2 * D)
    W0 = torch.randint(-90, 91, (2 * D, 2 * D), generator=g).double()
    w = W0[:, D:]
    ex = 0.5 * (dh @ w)
    check_exact((0.5 * (dh @ w)).float(), ex, "control pitched W", log=False)
    with pytest.raises(AssertionError):
        check_exact((0.5 * (dh @ W0[:, :D])).float(), ex, "control W0 other half", log=False)
    flat = W0.flatten()[D:D + 2 * D * D].view(2 * D, D)  # [2D, D] read from offset D with pitch D instead of 2D
    with pytest.raises(AssertionError):
        check_exact((0.5 * (dh @ flat)).float(), ex, "control W0 pitch N", log=False)
    bnd = gemm_bound(0.5 * dh.abs() @ w.abs(), 2 * D, 1.0, ex, torch.bfloat16)
    _within((ex.float().to(torch.bfloat16).double() - ex).abs(), bnd, "control", log=False)
    with pytest.raises(AssertionError):
        _within(((0.5 * (dh @ flat)).float().to(torch.bfloat16).double() - ex).abs(), bnd, "control", log=False)


def test_panel_check_rejects_a_reused_panel():
    """A-panel GEMM with one n-tile and two items on a CTA: the rows of item i + 132 computed from item i's panel fail
    both checks."""
    g = _cpu_gen(12)
    M, N, K = (SMS + 2) * 128, 128, 128
    a, w = _int_operands(g, M, N, K)
    ex = 0.5 * (a @ w.t())
    stale = ex.clone()
    stale[SMS * 128:] = ex[:2 * 128]  # items 132, 133 from the panels of items 0, 1
    check_exact(ex.float().to(torch.bfloat16), ex, "control panel", log=False)
    with pytest.raises(AssertionError):
        check_exact(stale.float().to(torch.bfloat16), ex, "control panel reused", log=False)
    ab, wb = (t.to(torch.bfloat16).double() for t in (torch.randn(M, K, generator=g), torch.randn(N, K, generator=g)))
    ref = ab @ wb.t()
    bnd = gemm_bound(ab.abs() @ wb.abs().t(), K, 1.0, ref, torch.bfloat16)
    bad = ref.clone()
    bad[SMS * 128:] = ref[:2 * 128]
    _within((ref.float().to(torch.bfloat16).double() - ref).abs(), bnd, "control", log=False)
    with pytest.raises(AssertionError):
        _within((bad.float().to(torch.bfloat16).double() - ref).abs(), bnd, "control", log=False)


def test_splitk_checks_reject_a_missing_k_range():
    """Split-K over 8192 tokens in 128 splits of kps = 1 k-block (64 tokens): one split's range left out fails."""
    g = _cpu_gen(13)
    T, M, N, kps, splits = 8192, 64, 72, 1, 128
    r = int(math.isqrt(2 ** 23 // T))
    dy = torch.randint(-r, r + 1, (T, M), generator=g).double()
    x = torch.randint(-r, r + 1, (T, N), generator=g).double()
    ex = dy.t() @ x
    check_exact(ex.float(), ex, "control split-K", log=False)
    s = 77
    lo, hi = s * kps * 64, (s + 1) * kps * 64
    drop = ex - dy[lo:hi].t() @ x[lo:hi]
    with pytest.raises(AssertionError):
        check_exact(drop.float(), ex, "control split-K range", log=False)
    db, xb = (torch.randn(T, c, generator=g).to(torch.bfloat16).double() for c in (M, N))
    ref = db.t() @ xb
    bnd = gemm_bound(db.abs().t() @ xb.abs(), 64 * kps + splits, 1.0, ref, torch.float32)
    _within((ref.float().double() - ref).abs(), bnd, "control", log=False)
    with pytest.raises(AssertionError):
        _within((ref - db[lo:hi].t() @ xb[lo:hi]).float().double().sub(ref).abs(), bnd, "control", log=False)


def test_shared_qk_check_rejects_a_missing_dk_and_a_truncating_add():
    """Without the other direction's dK the fp64 bound fails; a truncating bf16 add fails the exact sum check."""
    q, _, v, do = (t[0] for t in _inputs32(2, 130, 130, 2, "randn", 9, dev="cpu"))
    qk = q  # sequence 0's shared query / key tensor; sequence 1 is its partner
    qk1, _, v1, do1 = (t[1] for t in _inputs32(2, 130, 130, 2, "randn", 9, dev="cpu"))
    o0 = attn_ref(qk, qk1, v1, SCALE32)["O"].to(torch.bfloat16)
    o1 = attn_ref(qk1, qk, v, SCALE32)["O"].to(torch.bfloat16)
    r_own = attn_ref(qk, qk1, v1, SCALE32, o0, do)
    r_other = attn_ref(qk1, qk, v, SCALE32, o1, do1)
    ref, bound = shared_qk_bound(r_own, r_other)
    dq, dk = r_own["dQ"].to(torch.bfloat16), r_other["dK"].to(torch.bfloat16)
    ok = (dq.double() + dk.double()).float().to(torch.bfloat16)
    _within((ok.double() - ref).abs(), bound, "control shared qk", log=False)
    with pytest.raises(AssertionError):
        _within((dq.double() - ref).abs(), bound, "control shared qk without dk", log=False)
    check_bf16_sum(ok, dq, dk, "control shared qk")
    with pytest.raises(AssertionError, match="bf16 add"):
        check_bf16_sum(_trunc_bf16(dq.double() + dk.double()), dq, dk, "control shared qk truncating add")
