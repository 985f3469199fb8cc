"""GPU: the rotary split (lgb200_rope_split_{fwd,bwd}_hd) and the position-encoder weight gradient (lgb200_posenc_wgrad)
at head dimension 32 -- LightGlue with descriptor_dim 128 / 4 heads or 256 / 8 heads -- element by element against
fp64 restatements of lightglue.py:42-49, 62 and 156-160.

Wqkv feature = h*96 + d*3 + {q,k,v}; theta [T, 16]; the rotation pairs adjacent channels (2i, 2i+1) by theta[:, i].
Bounds are per element: the kernel computes in fp32 from the stored operands and rounds once to the output dtype, so
|got - ref| <= u_out |ref| + 1e-5 (|a| + |b|) for a rotated pair (a, b) (u_out = 2^-8 in bf16, 2^-23 in fp32), and the
dtheta / weight-gradient sums are held to a multiple of the unit round-off times the sum of absolute terms.  Each check
has a negative control that must fail it: the angles the head-dim-64 kernel would apply to a head-dim-32 buffer (theta
read with a row stride of 32 across heads of 64), and the rotation applied to swapped pairs (channel i with i + 16,
the non-interleaved convention)."""
import pytest
import torch

from gluefactory_b200 import _lib, ops
from gluefactory_b200._lib import call, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = "cuda"
HD = 32
BENCH_T = 2 * 32 * 2048  # both images of the benchmark's 32 pairs at 2048 points


def _u(dtype):
    return 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -23


def _inputs(T, H, dtype, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    qkv = torch.randn(T, H * 3 * HD, device=DEV, generator=g).to(dtype)
    theta = (torch.rand(T, HD // 2, device=DEV, generator=g) * 8 - 4).contiguous()  # |kp Wr^T| of a few radians
    return qkv, theta


def _rot(t, theta, pairs="adjacent"):
    """t [T, H, hd] fp64, theta [T, hd/2] or per head [T, H, hd/2] -> rotated t.  pairs="adjacent": (2i, 2i+1)
    (lightglue.py:42-49); "halves": (i, i + hd/2), the convention this kernel must NOT implement (negative control)."""
    th = theta[:, None] if theta.dim() == 2 else theta
    c, s = torch.cos(th), torch.sin(th)
    out = torch.empty_like(t)
    if pairs == "adjacent":
        a, b = t[..., 0::2], t[..., 1::2]
        out[..., 0::2], out[..., 1::2] = a * c - b * s, b * c + a * s
    else:
        h = t.shape[-1] // 2
        a, b = t[..., :h], t[..., h:]
        out[..., :h], out[..., h:] = a * c - b * s, b * c + a * s
    return out


def _theta64(theta, H):
    """The angles the head-dim-64 kernel would apply to this buffer (negative control).  Its Wqkv layout h*192 + d*3
    of H/2 heads is the same memory order as h*96 + d*3 of H heads, so what tells the two apart is the angles: it reads
    theta with a row stride of 32 and gives pair p (0..31) of a 64-channel head -- 32-channel heads 2h, 2h + 1 --
    angle p.  Defined for the first T/2 tokens: [T/2, H, 16]."""
    Th = theta.shape[0] // 2
    return theta.double().reshape(-1)[: Th * 32].view(Th, 1, 2, 16).expand(Th, H // 2, 2, 16).reshape(Th, H, 16)


def _split(qkv, H):
    """fp64 q, k, v [T, H, 32] of a Wqkv output (feature = h*96 + d*3 + {q,k,v}, lightglue.py:156-158)."""
    x = qkv.double().view(qkv.shape[0], H, HD, 3)
    return x[..., 0], x[..., 1], x[..., 2]


def _pair_sum(t):
    """|a| + |b| for each element of the rotation pair (2i, 2i+1) it belongs to; t [T, H, hd]."""
    a = t.abs()
    return a[..., 0::2].repeat_interleave(2, -1) + a[..., 1::2].repeat_interleave(2, -1)


def _close(got, ref, bound):
    err = (got.double() - ref).abs()
    return bool((err <= bound).all()), float((err / bound.clamp(min=1e-30)).max())


def _fwd_check(q, k, v, qkv, theta, H, dtype, control=None):
    """control: None (the kernel's contract), "hd64" (angles as the head-dim-64 kernel reads them), "halves"."""
    q0, k0, v0 = _split(qkv, H)
    th, pairs, T = theta.double(), "adjacent", qkv.shape[0]
    if control == "hd64":
        th = _theta64(theta, H)
        T = th.shape[0]
    elif control == "halves":
        pairs = "halves"
    ok, worst = True, 0.0
    for got, ref, src in ((q, _rot(q0[:T], th, pairs), q0), (k, _rot(k0[:T], th, pairs), k0), (v, v0[:T], None)):
        bound = _u(dtype) * ref.abs() + (1e-5 * _pair_sum(src[:T]) if src is not None else 0.0)
        o, w = _close(got[:T].view(T, H, HD), ref, bound)
        ok, worst = ok and o, max(worst, w)
    return ok, worst


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("T,H", [(BENCH_T, 4), (1003, 4), (777, 8)])
def test_rope_fwd_hd32_against_fp64(T, H, dtype):
    qkv, theta = _inputs(T, H, dtype, seed=T + H)
    q, k, v = ops.rope_fwd(qkv, theta, H)
    assert q.shape == (T, H * HD)
    ok, worst = _fwd_check(q, k, v, qkv, theta, H, dtype)
    assert ok, worst
    # negative controls: the head-dim-64 kernel's angles, and the rotation applied to the other pairing
    assert not _fwd_check(q, k, v, qkv, theta, H, dtype, control="hd64")[0]
    assert not _fwd_check(q, k, v, qkv, theta, H, dtype, control="halves")[0]
    # deterministic
    q2, k2, v2 = ops.rope_fwd(qkv, theta, H)
    assert torch.equal(q, q2) and torch.equal(k, k2) and torch.equal(v, v2)


def _bwd_ref(qkv, theta, grads, H, pairs="adjacent"):
    """fp64 autograd of the forward restatement: d(qkv) in the interleaved layout and d(theta).  theta may be per
    head ([T, H, 16], the hd64 control); qkv and grads are cut to its token count."""
    T = theta.shape[0]
    x = qkv[:T].double().requires_grad_(True)
    th = theta.double().requires_grad_(True)
    t = x.view(T, H, HD, 3)
    outs = (_rot(t[..., 0], th, pairs), _rot(t[..., 1], th, pairs), t[..., 2])
    torch.autograd.backward(outs, [g[:T].double().view(T, H, HD) for g in grads])
    return x.grad, th.grad


def _bwd_bounds(q, k, grads, H, dtype):
    """Per-element bounds of dqkv (the rotation of the incoming gradients, rounded once) and the sum of absolute terms
    of dtheta (over heads and q / k of dq'[2i+1] q'[2i] - dq'[2i] q'[2i+1]; q' is the stored rotated value)."""
    T = q.shape[0]
    gq, gk, gv = (g.double().view(T, H, HD) for g in grads)
    dq_b = (_u(dtype) + 1e-5) * _pair_sum(gq)  # |R(-theta) g| <= |a| + |b|
    dk_b = (_u(dtype) + 1e-5) * _pair_sum(gk)
    dqkv_b = torch.stack([dq_b, dk_b, _u(dtype) * gv.abs()], -1).reshape(T, H * 3 * HD)
    terms = 0.0
    for g, r in ((gq, q), (gk, k)):
        r = r.double().view(T, H, HD).abs()
        ga = g.abs()
        terms = terms + (ga[..., 1::2] * r[..., 0::2] + ga[..., 0::2] * r[..., 1::2]).sum(1)
    return dqkv_b, terms


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
@pytest.mark.parametrize("T,H", [(BENCH_T, 4), (1003, 4), (777, 8)])
def test_rope_bwd_hd32_against_fp64_accumulates_dtheta(T, H, dtype):
    """Two calls (two layers) into one dtheta that starts non-zero: dqkv of each call in the interleaved layout, and
    dtheta = start + both calls' contributions."""
    g = torch.Generator(device=DEV).manual_seed(7 * T + H)
    qkv1, theta = _inputs(T, H, dtype, seed=T + H)
    qkv2 = torch.randn(qkv1.shape, device=DEV, generator=g).to(dtype)
    start = torch.randn(theta.shape, device=DEV, generator=g)
    dtheta = start.clone()
    ref_dth = start.double()
    bound_dth = torch.zeros_like(ref_dth)
    for qkv in (qkv1, qkv2):
        q, k, v = ops.rope_fwd(qkv, theta, H)
        grads = tuple(torch.randn(q.shape, device=DEV, generator=g).to(dtype) for _ in range(3))
        dqkv, out = ops.rope_bwd(*grads, q, k, theta, H, dtheta=dtheta)
        assert out is dtheta and dqkv.shape == qkv.shape
        ref_dqkv, ref_t = _bwd_ref(qkv, theta, grads, H)
        dqkv_b, terms = _bwd_bounds(q, k, grads, H, dtype)
        ok, worst = _close(dqkv, ref_dqkv, dqkv_b)
        assert ok, ("dqkv", worst)
        # negative controls: the head-dim-64 kernel's angles, and the other pairing
        th64 = _theta64(theta, H)
        Th = th64.shape[0]
        assert not _close(dqkv[:Th], _bwd_ref(qkv, th64, grads, H)[0], dqkv_b[:Th])[0]
        assert not _close(dqkv, _bwd_ref(qkv, theta, grads, H, pairs="halves")[0], dqkv_b)[0]
        ref_dth = ref_dth + ref_t
        # q' is stored in the dtype (up to u_out of each term), then fp32 sums over 4H terms
        bound_dth = bound_dth + (2 * _u(dtype) + 4 * H * 2.0 ** -23) * terms
    ok, worst = _close(dtheta, ref_dth, bound_dth + 2.0 ** -22 * (ref_dth.abs() + start.double().abs()))
    assert ok, ("dtheta", worst)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32])
def test_rope_hd_entry_point_at_64_is_the_base_entry_point(dtype):
    """lgb200_rope_split_{fwd,bwd}_hd with head_dim 64 give the bits of lgb200_rope_split_{fwd,bwd}."""
    T, H = 4099, 4
    g = torch.Generator(device=DEV).manual_seed(5)
    qkv = torch.randn(T, H * 192, device=DEV, generator=g).to(dtype)
    theta = torch.randn(T, 32, device=DEV, generator=g)
    outs = []
    for hd_arg in (None, 64):
        q, k, v = (torch.empty(T, H * 64, device=DEV, dtype=dtype) for _ in range(3))
        args = (ptr(qkv), ptr(theta), ptr(q), ptr(k), ptr(v), T, H, ops._code(dtype))
        if hd_arg is None:
            call("lgb200_rope_split_fwd", *args, stream_ptr())
        else:
            call("lgb200_rope_split_fwd_hd", *args, hd_arg, stream_ptr())
        gq, gk, gv = (torch.randn(q.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(9 + i)).to(dtype)
                      for i in range(3))
        dqkv = torch.empty_like(qkv)
        dtheta = torch.full_like(theta, 0.5)
        args = (ptr(gq), ptr(gk), ptr(gv), ptr(q), ptr(k), ptr(theta), ptr(dqkv), ptr(dtheta), T, H, ops._code(dtype))
        if hd_arg is None:
            call("lgb200_rope_split_bwd", *args, stream_ptr())
        else:
            call("lgb200_rope_split_bwd_hd", *args, hd_arg, stream_ptr())
        outs.append((q, k, v, dqkv, dtheta))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def _wgrad(gr, kp):
    T, C = gr.shape
    kd = kp.shape[1]
    nb = _lib.load().lgb200_posenc_wgrad_blocks()
    part = torch.empty(nb, C, kd, device=DEV, dtype=torch.float32)
    call("lgb200_posenc_wgrad", ptr(gr), ptr(kp), ptr(part), T, C, kd, stream_ptr())
    return part.sum(0)


@pytest.mark.parametrize("T", [BENCH_T, 1003, 5])
@pytest.mark.parametrize("kd", [2, 4])
def test_posenc_wgrad_16_angles_against_fp64(T, kd):
    """dWr [16, kd] = sum_t g[t] kp[t]^T, g = dtheta [T, 16]; fixed reduction order, so the same bits every call.  The
    PosencTheta backward takes the same path."""
    g = torch.Generator(device=DEV).manual_seed(T + kd)
    gr = torch.randn(T, 16, device=DEV, generator=g)
    kp = torch.rand(T, kd, device=DEV, generator=g) * 2 - 1
    dw = _wgrad(gr, kp)
    ref = gr.double().t() @ kp.double()
    absum = gr.double().abs().t() @ kp.double().abs()
    nb = _lib.load().lgb200_posenc_wgrad_blocks()
    steps = T // (nb * 16) + 1 + 16 + nb  # sequential additions of one term, worst case
    err = (dw.double() - ref).abs()
    assert (err <= steps * 2.0 ** -24 * absum + 1e-30).all(), float((err / absum).max())
    assert torch.equal(dw, _wgrad(gr, kp))
    # negative control: the same buffer read with the 32-angle stride is a different contraction
    if T % 2 == 0:
        wrong = gr.double().view(T // 2, 32).t() @ kp.double()[: T // 2]
        assert not torch.allclose(dw.double(), wrong[:16], rtol=1e-3, atol=1e-3)
    # through autograd: theta = kp Wr^T, Wr [16, kd]
    w = torch.randn(16, kd, device=DEV, generator=g, requires_grad=True)
    ops.PosencTheta.apply(kp, w).backward(gr)
    assert torch.equal(w.grad, dw)
