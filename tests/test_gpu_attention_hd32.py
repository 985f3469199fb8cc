"""GPU: the attention kernels at head dimension 32 (lgb200_attn_fwd_hd / lgb200_attn_bwd_hd; GlueStick with 128-channel
descriptors and 4 heads) element by element against fp64, with the bound-based checks, guarded outputs and logit
regimes of tests/test_gpu_tensor_core_kernels.py.

Bounds: those of test_gpu_tensor_core_kernels.attn_ref, written for a 64-term dot product; at 32 terms the S error term
is half as large, so the bounds hold with that much room on the S error and are unchanged elsewhere.  Scale = 32^-0.5.

fp32 CUDA-core path (precision "fp32"): plain fp32 arithmetic, so the bound is attn_ref's with the fp32 unit in
place of the tensor cores' and with no bf16 rounding:
    eps32 = 32 U32 scale (|q| |k|) + 4 U32 + 3 U32 (|S| + |max S|)     (expf of an fp32 difference)
    O     2 (P eps32)|V| + 2 (P eps32)1 |O| + (2 Nk + 64) U32 P|V| + U32 |O|
          (the P V and row-sum chains, Nk steps each, and the rescales at each new running maximum)
    dQ    scale (2 A (eps32 + 32 U32) + (2 Nk + 64) U32 A) |K| + U32 |dQ|     (dK, dV likewise over the queries)
          A = P o (|dO| |V|^T + rowsum(|dO| o |O|)): the second term also covers the rounding of delta's own sum

Shapes: GlueStick's C5 launch (2048 points + 512 lines = 3072 nodes per image, 4 heads) as self-attention, a cross
launch with Nq != Nk, and every pair of tile edges Nq, Nk in {1, 63, 64, 65, 127, 128, 129, 1000}.  The large launches
run twice and must agree bit for bit.  The negative controls show that each check rejects a deliberately wrong result.
"""
import pytest
import torch

from gluefactory_b200 import _lib, ops
from gluefactory_b200._lib import call, ptr, stream_ptr
from tests.test_gpu_tensor_core_kernels import (DEV, U32, _cpu_gen, _gen, _guarded, _guards_intact, _trunc_bf16,
                                                _within, _Worst, attn_ref, check_attn_bwd, check_attn_fwd)

GPU = pytest.mark.gpu
HD = 32
SCALE = HD ** -0.5


def _inputs(B, Nq, Nk, H, regime, seed, dev=DEV, dtype=torch.bfloat16):
    """q, k, v, dout [B, N, H, 32]; the regimes of test_gpu_tensor_core_kernels._attn_inputs (randn, spike, rising,
    zero_q), with the spike and the rise scaled so the logits span the same range at this scale."""
    g = _gen(seed) if dev == DEV else _cpu_gen(seed)
    q = torch.randn(B, Nq, H, HD, device=dev, generator=g) * 1.5
    k = torch.randn(B, Nk, H, HD, device=dev, generator=g)
    v = torch.randn(B, Nk, H, HD, device=dev, generator=g)
    do = torch.randn(B, Nq, H, HD, device=dev, generator=g)
    if regime == "spike":  # the last key (in a partial tile when Nk % 64 != 0) ~40 above every other logit
        q[..., 0] = 8.0
        k[..., 0] = 0.0
        k[:, Nk - 1, :, 0] = 40.0 / (8.0 * SCALE)
    elif regime == "rising":  # the running maximum grows in every key tile
        q[..., 0] = 8.0
        k[..., 0] = torch.linspace(0.0, 60.0 / (8.0 * SCALE), Nk, device=dev)[None, :, None]
    elif regime == "zero_q":  # every p is 1: out = mean of V
        q.zero_()
        v = 1.25 + 0.1 * v
    return tuple(t.to(dtype).contiguous() for t in (q, k, v, do))


def _fwd_guarded(q, k, v, shift):
    B, Nq, H, _ = q.shape
    go = _guarded((B, Nq, H, HD), q.dtype, 2 * H * HD)
    gl = _guarded((B, H, Nq), torch.float32, 64)
    call("lgb200_attn_fwd_hd", ptr(q), ptr(k), ptr(v), ptr(go[1]), ptr(gl[1]), B, Nq, k.shape[1], H, shift,
         float(SCALE), ops._code(q.dtype), HD, stream_ptr())
    return go, gl


def _bwd_guarded(q, k, v, out, lse, do, shift):
    B, Nq, H, _ = q.shape
    Nk = k.shape[1]
    gq = _guarded((B, Nq, H, HD), q.dtype, 2 * H * HD)
    gk = _guarded((B, Nk, H, HD), q.dtype, 2 * H * HD)
    gv = _guarded((B, Nk, H, HD), q.dtype, 2 * H * HD)
    ws = torch.empty(_lib.load().lgb200_attn_bwd_ws_floats(B, Nq, Nk, H), device=DEV)
    call("lgb200_attn_bwd_hd", ptr(q), ptr(k), ptr(v), ptr(out), ptr(lse), ptr(do), ptr(gq[1]), ptr(gk[1]),
         ptr(gv[1]), ptr(ws), B, Nq, Nk, H, shift, float(SCALE), ops._code(q.dtype), HD, stream_ptr())
    return gq, gk, gv


def attn_ref_f32(q, k, v, out=None, do=None):
    """fp64 attention of one sequence with the fp32 CUDA-core bounds of the module docstring."""
    Q, K, V = (t.double().permute(1, 0, 2) for t in (q, k, v))
    Nq, Nk = Q.shape[1], K.shape[1]
    S = SCALE * (Q @ K.transpose(1, 2))
    m = S.amax(-1, keepdim=True)
    P = torch.softmax(S, -1)
    lse = torch.logsumexp(S, -1)
    eps = (HD * U32 * SCALE) * (Q.abs() @ K.abs().transpose(1, 2)) + 4 * U32 + 3 * U32 * (S.abs() + m.abs())
    Pe = P * eps
    aV = V.abs()
    O = P @ V
    Pe1 = Pe.sum(-1, keepdim=True)
    r = dict(O=O, lse=lse, bO=2 * (Pe @ aV) + 2 * Pe1 * O.abs() + (2 * Nk + 64) * U32 * (P @ aV) + U32 * O.abs(),
             blse=Pe1.squeeze(-1) + (2 * Nk + 64) * U32 + 4 * U32 * (m.squeeze(-1).abs() + lse.abs()))
    if do is not None:
        dO, Os = do.double().permute(1, 0, 2), out.double().permute(1, 0, 2)
        delta = (dO * Os).sum(-1, keepdim=True)
        dS = P * (dO @ V.transpose(1, 2) - delta)
        A = P * (dO.abs() @ aV.transpose(1, 2) + (dO.abs() * Os.abs()).sum(-1, keepdim=True))
        r["dV"], r["dQ"], r["dK"] = P.transpose(1, 2) @ dO, SCALE * (dS @ K), SCALE * (dS.transpose(1, 2) @ Q)
        r["bdV"] = (2 * Pe + (2 * Nq + 64) * U32 * P).transpose(1, 2) @ dO.abs() + U32 * r["dV"].abs()
        W = 2 * A * (eps + HD * U32) + (2 * Nk + 64) * U32 * A
        r["bdQ"] = SCALE * (W @ K.abs()) + U32 * r["dQ"].abs()
        W = 2 * A * (eps + HD * U32) + (2 * Nq + 64) * U32 * A
        r["bdK"] = SCALE * (W.transpose(1, 2) @ Q.abs()) + U32 * r["dK"].abs()
    return {key: (t if key in ("lse", "blse") else t.permute(1, 0, 2)) for key, t in r.items()}


def _run(B, Nq, Nk, H, shift, regime, seed, again=False, tag="", fp32=False):
    q, k, v, do = _inputs(B, Nq, Nk, H, regime, seed, dtype=torch.float32 if fp32 else torch.bfloat16)
    go, gl = _fwd_guarded(q, k, v, shift)
    out, lse = go[1], gl[1]
    gq, gk, gv = _bwd_guarded(q, k, v, out, lse, do, shift)
    if again:
        out2, lse2 = ops.attn_fwd(q, k, v, shift, SCALE)
        assert torch.equal(out, out2) and torch.equal(lse, lse2), (tag, "forward not bit-identical")
        again_ = ops.attn_bwd(q, k, v, out, lse, do, shift, SCALE)
        assert all(torch.equal(a, b[1]) for a, b in zip(again_, (gq, gk, gv))), (tag, "backward not bit-identical")
        del out2, lse2, again_
    w = _Worst(tag)
    for b in range(B):
        kb = (b + shift) % B
        if fp32:
            r = attn_ref_f32(q[b], k[kb], v[kb], out[b], do[b])
        else:
            r = attn_ref(q[b], k[kb], v[kb], SCALE, out[b], do[b])
        check_attn_fwd(out[b], lse[b], r, w)
        check_attn_bwd(gq[1][b], gk[1][kb], gv[1][kb], r, w)
        del r
    w.report()
    for gb in (go, gl, gq, gk, gv):
        _guards_intact(gb, tag)


@GPU
def test_hd32_gluestick_self_attention_shape():
    """GlueStick's C5 self-attention launch: 3072 nodes, 4 heads, forward and backward twice (bit-identical)."""
    _run(4, 3072, 3072, 4, 0, "randn", seed=101, again=True, tag="attn hd32 self 3072")


@GPU
def test_hd32_cross_attention_ragged_shape():
    """Cross-attention between images of different sizes (Nq != Nk), both directions in one launch."""
    _run(2, 3072, 2600, 4, 1, "randn", seed=102, again=True, tag="attn hd32 cross 3072x2600")


EDGES = (1, 63, 64, 65, 127, 128, 129, 1000)


@GPU
@pytest.mark.parametrize("Nk", EDGES)
@pytest.mark.parametrize("Nq", EDGES)
def test_hd32_tile_edges(Nq, Nk):
    _run(2, Nq, Nk, 4, (Nq + Nk) % 2, "randn", seed=Nq * 11 + Nk, tag=f"attn hd32 Nq={Nq} Nk={Nk}")


@GPU
@pytest.mark.parametrize("regime", ["spike", "rising", "zero_q"])
@pytest.mark.parametrize("Nq,Nk", [(129, 65), (300, 1000)])
def test_hd32_logit_regimes(regime, Nq, Nk):
    _run(2, Nq, Nk, 2, 1, regime, seed=Nq + Nk, tag=f"attn hd32 {regime} Nq={Nq} Nk={Nk}")


@GPU
@pytest.mark.parametrize("Nq,Nk", [(3072, 3072), (129, 1000), (1, 65), (1000, 63)])
def test_hd32_fp32_cuda_core_path(Nq, Nk):
    """precision "fp32": the CUDA-core kernels at head dim 32, forward and backward, against fp64."""
    B = 2
    _run(B, Nq, Nk, 4, (Nq + Nk) % 2, "randn", seed=Nq + 3 * Nk, again=Nq == 3072, tag=f"attn hd32 fp32 Nq={Nq} Nk={Nk}",
         fp32=True)


@GPU
def test_hd32_guard_check_sees_a_stray_write():
    """Control for the guard rows: one element written past the output is seen."""
    g = _guarded((2, 3, 4, HD), torch.bfloat16, 8)
    _guards_intact(g, "control")
    g[0][-1] = 0.0
    with pytest.raises(AssertionError, match="guard rows overwritten"):
        _guards_intact(g, "control")


def test_hd32_checks_reject_wrong_answers():
    """CPU controls at head dim 32: each check rejects a wrong result built from its own reference."""
    w = lambda name, e, b: _within(e, b, name, log=False)  # noqa: E731
    q, k, v, do = (t[0] for t in _inputs(1, 70, 150, 1, "randn", 6, dev="cpu"))
    r = attn_ref(q, k, v, SCALE, attn_ref(q, k, v, SCALE)["O"].to(torch.bfloat16), do)
    check_attn_fwd(r["O"].to(torch.bfloat16), r["lse"].float(), r, w)
    check_attn_bwd(r["dQ"].to(torch.bfloat16), r["dK"].to(torch.bfloat16), r["dV"].to(torch.bfloat16), r, w)
    # forward: a key tile left out (out, then lse); a truncating bf16 store
    keep = torch.cat([torch.arange(0, 64), torch.arange(128, 150)])
    r_drop = attn_ref(q, k[keep], v[keep], SCALE, r["O"].to(torch.bfloat16), do)
    for got_o, got_l in ((r_drop["O"], r["lse"]), (r["O"], r_drop["lse"])):
        with pytest.raises(AssertionError):
            check_attn_fwd(got_o.to(torch.bfloat16), got_l.float(), r, w)
    zq, zk, zv, _ = (t[0] for t in _inputs(1, 70, 150, 1, "zero_q", 4, dev="cpu"))
    rz = attn_ref(zq, zk, zv, SCALE)
    with pytest.raises(AssertionError):
        check_attn_fwd(_trunc_bf16(rz["O"]), rz["lse"].float(), rz, w)
    # backward: dQ from a key tile left out; dK / dV from a query tile left out
    with pytest.raises(AssertionError):
        check_attn_bwd(r_drop["dQ"].to(torch.bfloat16), r["dK"].to(torch.bfloat16), r["dV"].to(torch.bfloat16), r, w)
    qk = torch.arange(64, 70)
    r_q = attn_ref(q[qk], k, v, SCALE, r["O"][qk].to(torch.bfloat16), do[qk])
    with pytest.raises(AssertionError):
        check_attn_bwd(r["dQ"].to(torch.bfloat16), r_q["dK"].to(torch.bfloat16), r["dV"].to(torch.bfloat16), r, w)
    with pytest.raises(AssertionError):
        check_attn_bwd(r["dQ"].to(torch.bfloat16), r["dK"].to(torch.bfloat16), r_q["dV"].to(torch.bfloat16), r, w)
    # fp32 path: the exact result passes; bf16-rounded outputs and gradients (what the tensor-core path gives) do not
    q, k, v, do = (t[0] for t in _inputs(1, 70, 150, 1, "randn", 7, dev="cpu", dtype=torch.float32))
    r = attn_ref_f32(q, k, v, attn_ref_f32(q, k, v)["O"].float(), do)
    check_attn_fwd(r["O"].float(), r["lse"].float(), r, w)
    check_attn_bwd(r["dQ"].float(), r["dK"].float(), r["dV"].float(), r, w)
    with pytest.raises(AssertionError):
        check_attn_fwd(r["O"].to(torch.bfloat16), r["lse"].float(), r, w)
    for i in range(3):
        grads = [r[n].float() for n in ("dQ", "dK", "dV")]
        grads[i] = grads[i].to(torch.bfloat16)
        with pytest.raises(AssertionError):
            check_attn_bwd(*grads, r, w)
