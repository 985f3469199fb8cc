"""CPU: the bounds of tests/superpoint_open_oracle.py that tests/test_gpu_superpoint_open_shapes.py holds the
SuperPoint-open BatchNorm kernels to.  Each bound must hold for the kernels' formulas evaluated in fp32 in another
order (the folded affine, spo_bn_setup and its element formula, the bf16 store, the running update); each comparison
must reject a one-ulp change of its worst element, a swapped channel and a swapped image; the sum and running-update
restatements must reject a biased variance used for the unbiased one and a rank's local count used for the global
one."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import superpoint_open_oracle as oo  # noqa: E402
from tests import superpoint_oracle as so  # noqa: E402

EPS = 1e-3


def _bn(C, seed):
    """Buffers as the GPU tests draw them: both signs, running_var over 1e-3 .. 1e2, near-zero weights."""
    g = torch.Generator().manual_seed(seed)
    rv = 10.0 ** (torch.rand(C, generator=g) * 5 - 3)
    w = (torch.rand(C, generator=g) + 0.5) * torch.sqrt(rv) * (torch.randint(0, 2, (C,), generator=g) * 2 - 1)
    w[::8] = (torch.rand(w[::8].shape, generator=g) * 2 - 1) * 1e-3
    return w, (torch.rand(C, generator=g) * 2 - 1) * 0.2, torch.rand(C, generator=g) * 2 - 1, rv


def _acts(B, H, W, C, seed, relu=True):
    """bf16-exact activations [B, H, W, C] with a dead channel, a constant one and one of large mean, small spread."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B, H, W, C, generator=g) * (torch.rand(C, generator=g) * 2 + 0.1) + torch.randn(C, generator=g)
    x = F.relu(x) if relu else x
    x[..., 0] = 0
    x[..., 1] = 0.75
    x[..., 2] = 6 + 0.02 * torch.randn(B, H, W, generator=g)
    return x.to(torch.bfloat16).float()


def _worst_ulp(out, ref, bound, k=1):
    """out with its worst element (largest error to bound) moved k ulps further from the reference."""
    ratio = ((out.double() - ref).abs() / bound).reshape(-1)
    i = int(torch.argmax(ratio))
    o = out.clone(memory_format=torch.contiguous_format)
    iv = o.view(-1).view({torch.bfloat16: torch.int16, torch.float32: torch.int32}[o.dtype])
    away = (float(o.view(-1)[i]) >= float(ref.reshape(-1)[i])) == (float(o.view(-1)[i]) >= 0)
    iv[i] += k if away else -k
    return o


def _worst_rel(out, ref, bound, rel):
    """out with its worst element moved further from the reference by rel of its magnitude."""
    i = int(torch.argmax(((out.double() - ref).abs() / bound).reshape(-1)))
    o = out.clone(memory_format=torch.contiguous_format)
    d = float(o.view(-1)[i]) - float(ref.reshape(-1)[i])
    o.view(-1)[i] += rel * abs(float(o.view(-1)[i])) * (1 if d >= 0 else -1)
    return o


def _rejects(out, ref, bound, chan_dim, rel=None):
    """The comparison passes on out and fails on its worst element moved one ulp (the bf16 outputs, whose bounds are
    about half an ulp) or, for the fp32 softmax and L2 outputs (bounds of a few hundred ulps, for expf, the sums and
    the norm), moved by `rel` of its value; on two channels swapped; and (out [B, ...]) on two images swapped."""
    r = so.assert_within(out, ref, bound)
    with pytest.raises(AssertionError):
        so.assert_within(_worst_ulp(out, ref, bound) if rel is None else _worst_rel(out, ref, bound, rel), ref, bound)
    sw = out.clone()
    idx = [slice(None)] * out.dim()
    a, b = list(idx), list(idx)
    a[chan_dim], b[chan_dim] = 3, 4
    sw[tuple(a)], sw[tuple(b)] = out[tuple(b)], out[tuple(a)]
    with pytest.raises(AssertionError):
        so.assert_within(sw, ref, bound)
    with pytest.raises(AssertionError):
        so.assert_within(out.flip(0), ref, bound)
    return r


# ---- eval mode: the folded affine ------------------------------------------------------------------------------------
@pytest.mark.parametrize("pool", [False, True])
def test_folded_affine_bound_holds_and_rejects(pool):
    B, H, W, C = 2, 12, 10, 64
    g_, b_, rm, rv = _bn(C, seed=1 + pool)
    r = _acts(B, H, W, C, seed=3).permute(0, 3, 1, 2)  # the fp32 staged ReLU output, NCHW
    acc = 1e-6 * r.abs()  # a conv accumulation error, within the E the test passes
    r32 = (r.double() + acc * torch.sign(torch.randn(r.shape, generator=torch.Generator().manual_seed(4)))).float()
    s, t = oo.fold32(g_, b_, rm, rv, EPS)
    v = oo.fma32(r32, s.view(1, -1, 1, 1), t.view(1, -1, 1, 1))
    z, e = oo.folded_affine(r.double(), acc, g_, b_, rm, rv, EPS)
    if pool:
        out = F.max_pool2d(v, 2, 2).to(torch.bfloat16)
        ref = F.max_pool2d(z, 2, 2)
        bound = so.pool_bf16_bound(ref, e)
    else:
        out, ref, bound = v.to(torch.bfloat16), z, so.relu_bf16_bound(z, e)
    assert _rejects(out, ref, bound, 1) > 0.3  # the bf16 store dominates: the bound is tight
    # the pool of the un-normalised map, then the affine: wrong with negative scales
    if pool:
        bad = oo.fma32(F.max_pool2d(r32, 2, 2), s.view(1, -1, 1, 1), t.view(1, -1, 1, 1)).to(torch.bfloat16)
        with pytest.raises(AssertionError):
            so.assert_within(bad, ref, bound)
    # the affine before the ReLU
    pre = r32 - 0.5
    bad = oo.fma32(pre, s.view(1, -1, 1, 1), t.view(1, -1, 1, 1)).clamp_min(0)
    with pytest.raises(AssertionError):
        so.assert_within(bad if not pool else F.max_pool2d(bad, 2, 2), ref,
                         bound if not pool else so.pool_bf16_bound(ref, e))


def test_folded_affine_heads_bound_holds():
    """Softmax and L2 normalisation of folded logits: the fp32 restatement within softmax_bound / l2n_bound."""
    g_, b_, rm, rv = _bn(65, seed=7)
    y = torch.randn(2, 65, 5, 6, generator=torch.Generator().manual_seed(8), dtype=torch.float64) * 2
    s, t = oo.fold32(g_, b_, rm, rv, EPS)
    logit = oo.fma32(y.float(), s.view(1, -1, 1, 1), t.view(1, -1, 1, 1))
    z, e = oo.folded_affine(y, torch.zeros_like(y), g_, b_, rm, rv, EPS)
    p, bound = oo.softmax_bound(z, e)
    so.assert_within(F.softmax(logit, 1)[:, :-1], p, bound)
    g2, b2, rm2, rv2 = _bn(256, seed=9)
    y2 = torch.randn(2, 256, 4, 3, generator=torch.Generator().manual_seed(10), dtype=torch.float64)
    s2, t2 = oo.fold32(g2, b2, rm2, rv2, EPS)
    a = oo.fma32(y2.float(), s2.view(1, -1, 1, 1), t2.view(1, -1, 1, 1))
    z2, e2 = oo.folded_affine(y2, torch.zeros_like(y2), g2, b2, rm2, rv2, EPS)
    o, bound2 = oo.l2n_bound(z2, e2)
    _rejects(F.normalize(a, dim=1), o, bound2, 1, rel=2.0 ** -10)


# ---- training mode: sums, the normalisation and the running update ---------------------------------------------------
def _stats(x):
    st = oo.Stats(x.shape[-1], x.device)
    for b in range(x.shape[0]):
        st.add(x[b])
    for b in range(x.shape[0]):
        st.add_centred(x[b])
    return st


def _kernel_sums(x):
    """bn_stats in another order: fp64 sums over the flattened rows in reverse."""
    x = x.reshape(-1, x.shape[-1]).double().flip(0)
    return torch.cat([x.sum(0), (x * x).sum(0), x.new_tensor([float(x.shape[0])])])


@pytest.mark.parametrize("op", ["plain", "pool", "softmax", "l2n"])
def test_bn_apply_bound_holds_and_rejects(op):
    C = {"plain": 64, "pool": 128, "softmax": 65, "l2n": 256}[op]
    x = _acts(3, 8, 10, C, seed=C, relu=op in ("plain", "pool"))
    g_, b_, _, _ = _bn(C, seed=C + 1)
    st = _stats(x)
    sums = _kernel_sums(x)
    so.assert_within(sums, st.sums(), st.sum_bound())
    mu, rs = oo.bn_setup32(sums, EPS)
    v = oo.bn_apply32(x, mu, rs, g_, b_)
    z, e = oo.bn_apply_ref(x.double(), st, g_, b_, EPS)
    if op == "plain":
        out, ref, bound, cd = v.to(torch.bfloat16), z, so.relu_bf16_bound(z, e), -1
        assert bool((out[..., :2] == b_[:2].to(torch.bfloat16)).all())  # dead and constant channels: exactly beta
    elif op == "pool":
        out = F.max_pool2d(v.permute(0, 3, 1, 2), 2, 2).to(torch.bfloat16)
        ref = F.max_pool2d(z.permute(0, 3, 1, 2), 2, 2)
        out, ref, bound, cd = out, ref, so.pool_bf16_bound(ref, e.permute(0, 3, 1, 2)), 1
    elif op == "softmax":
        p, bound = so.softmax_bound(z.permute(0, 3, 1, 2), e.permute(0, 3, 1, 2))
        out, ref, cd = F.softmax(v, -1)[..., :64].permute(0, 3, 1, 2), p, 1
    else:
        o, bound = so.l2n_bound(z.permute(0, 3, 1, 2), e.permute(0, 3, 1, 2))
        out, ref, cd = F.normalize(v, dim=-1).permute(0, 3, 1, 2), o, 1
    _rejects(out, ref, bound, cd, rel=None if op in ("plain", "pool") else 2.0 ** -10)
    if op == "softmax":  # the dustbin left un-normalised
        bad = torch.cat([v[..., :64], x[..., 64:65]], -1)
        with pytest.raises(AssertionError):
            so.assert_within(F.softmax(bad, -1)[..., :64].permute(0, 3, 1, 2), ref, bound)


def test_one_pass_variance_cancellation_is_covered():
    """A channel of mean 6 and spread 0.02 over many rows: the fp64 one-pass variance is within kernel_stat_bounds of
    the two-pass one, and the bound there is wider than for a centred channel, but stays far below the variance."""
    x = _acts(16, 32, 32, 8, seed=21)
    st = _stats(x)
    sums = _kernel_sums(x)
    n = st.n
    m = sums[:8] / n
    var_k = (sums[8:16] / n - m * m).clamp_min(0)
    em, dvar = st.kernel_stat_bounds()
    assert bool(((var_k - st.var).abs() <= dvar).all())
    assert bool(((m - st.mean).abs() <= em).all())
    rel = dvar / st.var
    assert rel[2] > 1e3 * rel[3] and rel[2] < 1e-4
    assert float(var_k[1]) == 0.0 and float(var_k[0]) == 0.0


@pytest.mark.parametrize("momentum", [0.1, 0.37])
def test_running_update_bound_holds_and_rejects(momentum):
    C = 64
    x = _acts(2, 5, 7, C, seed=31)  # n = 70: n / (n - 1) is far outside the fp32 roundings
    _, _, rm0, rv0 = _bn(C, seed=32)
    st = _stats(x)
    sums = _kernel_sums(x)
    (rm_ref, rm_b), (rv_ref, rv_b) = oo.running_ref(st, rm0, rv0, momentum)
    rm, rv = oo.running_update32(sums, rm0, rv0, momentum)
    so.assert_within(rm, rm_ref, rm_b)
    so.assert_within(rv, rv_ref, rv_b)
    for o, ref, b in ((rm, rm_ref, rm_b), (rv, rv_ref, rv_b)):  # the bound is four fp32 roundings wide
        with pytest.raises(AssertionError):
            so.assert_within(_worst_ulp(o, ref, b, 8), ref, b)
    # the biased variance for the unbiased one
    _, rv_biased = oo.running_update32(sums, rm0, rv0, momentum, unbiased=False)
    with pytest.raises(AssertionError):
        so.assert_within(rv_biased, rv_ref, rv_b)
    # one rank's local count for the global one (the sums of all ranks, the count of one of two)
    local = sums.clone()
    local[2 * C] = st.n // 2
    rm_l, rv_l = oo.running_update32(local, rm0, rv0, momentum)
    with pytest.raises(AssertionError):
        so.assert_within(rm_l, rm_ref, rm_b)
    with pytest.raises(AssertionError):
        so.assert_within(rv_l, rv_ref, rv_b)


def test_sums_reject_local_count_and_missing_image():
    x = _acts(4, 6, 8, 64, seed=41)
    st = _stats(x)
    sums = _kernel_sums(x)
    so.assert_within(sums, st.sums(), st.sum_bound())
    local = _kernel_sums(x[:2])  # one rank's sums and count, not exchanged
    with pytest.raises(AssertionError):
        so.assert_within(local, st.sums(), st.sum_bound())
    short = sums.clone()
    short[-1] -= 1
    with pytest.raises(AssertionError):
        so.assert_within(short, st.sums(), st.sum_bound())
    # normalising with one rank's statistics instead of the exchanged ones
    g_, b_, _, _ = _bn(64, seed=42)
    z, e = oo.bn_apply_ref(x.double(), st, g_, b_, EPS)
    bound = so.relu_bf16_bound(z, e)
    mu, rs = oo.bn_setup32(local, EPS)
    with pytest.raises(AssertionError):
        so.assert_within(oo.bn_apply32(x, mu, rs, g_, b_).to(torch.bfloat16), z, bound)
