"""GPU: the forward-only attention over packed sequences of different lengths (lgb200_attn_fwd_varlen), which LightGlue's
adaptive depth / width runs on a batch of pairs.

Seven sequences of 1, 63, 64, 65, 127, 2048 and 0 tokens lie in one token-major buffer, with guard rows between them and
around them.  Self-attention: each sequence attends to itself; cross-attention: each to another sequence of a different
length, one sequence to the empty one (it does no work).  Every sequence is checked against fp64 attention of its own
tokens -- bf16 with the element-wise bounds of tests/test_gpu_tensor_core_kernels.py (attn_ref), fp32 within 2e-5
relative -- and every output row and lse entry that belongs to no computed sequence must keep its guard value.  A
uniform batch run through the packed entry point equals the uniform kernel bit for bit, the property the adaptive path
relies on for a single pair.

Budget: a few seconds and well under 1 GiB of device memory on one H100, recorded by the module fixture."""
import time

import pytest
import torch

from gluefactory_b200 import ops
from gluefactory_b200._lib import call, ptr, stream_ptr
from tests.test_gpu_tensor_core_kernels import _within, attn_ref
from tests.util import report

pytestmark = pytest.mark.gpu
DEV = "cuda"
LENS = [1, 63, 64, 65, 127, 2048, 0]
PARTNER = [6, 2, 1, 5, 3, 4, 0]  # cross-attention: sequence s attends to the keys of sequence PARTNER[s]
GAP = 5                          # guard rows before, between and after the sequences
OUT_GUARD, LSE_GUARD, IN_GUARD = 512.0, -12345.0, 3.0


@pytest.fixture(scope="module", autouse=True)
def _file_budget():
    """Wall time and peak device memory of this file (the machines running it are shared)."""
    torch.cuda.reset_peak_memory_stats()
    t = time.time()
    yield
    torch.cuda.synchronize()
    report("test_gpu_attention_varlen", seconds=time.time() - t, peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)


def _layout():
    offs, r = [], GAP
    for n in LENS:
        offs.append(r)
        r += n + GAP
    return offs, r


def _inputs(T, H, hd, dtype, seed):
    g = torch.Generator(device="cpu").manual_seed(seed)
    offs, _ = _layout()
    qkv = []
    for _ in range(3):
        t = torch.full((T, H, hd), IN_GUARD)
        for o, n in zip(offs, LENS):
            t[o:o + n] = torch.randn(n, H, hd, generator=g)
        qkv.append(t.to(DEV, dtype))
    return qkv


@pytest.mark.parametrize("cross", [False, True], ids=["self", "cross"])
@pytest.mark.parametrize("hd,H", [(64, 4), (32, 8)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_varlen_against_fp64_per_sequence(dtype, hd, H, cross):
    offs, T = _layout()
    q, k, v = _inputs(T, H, hd, dtype, seed=hd + 7 * H + int(cross))
    partner = PARTNER if cross else list(range(len(LENS)))
    i32 = dict(device=DEV, dtype=torch.int32)
    q_off, q_len = torch.tensor(offs, **i32), torch.tensor(LENS, **i32)
    k_off, k_len = q_off[partner].contiguous(), q_len[partner].contiguous()
    out = torch.full_like(q, OUT_GUARD)
    scale = hd ** -0.5
    out, lse = ops.attn_fwd_varlen(q, k, v, q_off, q_len, k_off, k_len, max(LENS), scale, out=out)
    torch.cuda.synchronize()
    written = torch.zeros(T, dtype=torch.bool)
    worst = 0.0
    for s, (o, n) in enumerate(zip(offs, LENS)):
        ko, kn = offs[partner[s]], LENS[partner[s]]
        if n == 0 or kn == 0:
            continue
        written[o:o + n] = True
        got, gl = out[o:o + n], lse[:, o:o + n]
        if dtype == torch.bfloat16:
            r = attn_ref(q[o:o + n], k[ko:ko + kn], v[ko:ko + kn], scale)
            worst = max(worst, _within((got.double() - r["O"]).abs(), r["bO"], f"varlen out s{s}", log=False),
                        _within((gl.double() - r["lse"]).abs(), r["blse"], f"varlen lse s{s}", log=False))
        else:
            Q, K, V = (t.double().permute(1, 0, 2) for t in (q[o:o + n], k[ko:ko + kn], v[ko:ko + kn]))
            S = scale * Q @ K.transpose(1, 2)
            O = (torch.softmax(S, -1) @ V).permute(1, 0, 2)
            L = torch.logsumexp(S, -1)
            worst = max(worst, _within((got.double() - O).abs(), 2e-5 * (1 + O.abs()), f"varlen out s{s}", log=False),
                        _within((gl.double() - L).abs(), 2e-5 * (1 + L.abs()), f"varlen lse s{s}", log=False))
    report(f"varlen {dtype} hd{hd} H{H} {'cross' if cross else 'self'}", max_err_over_bound=worst)
    assert written.any()
    untouched = out[~written.to(DEV)]
    assert torch.equal(untouched, torch.full_like(untouched, OUT_GUARD)), "rows outside the sequences were written"


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_varlen_lse_rows_outside_sequences_untouched(dtype):
    """The entry point called with a guard-filled lse [H, T]: no entry outside the computed sequences is written."""
    offs, T = _layout()
    H, hd = 4, 64
    q, k, v = _inputs(T, H, hd, dtype, seed=5)
    i32 = dict(device=DEV, dtype=torch.int32)
    q_off, q_len = torch.tensor(offs, **i32), torch.tensor(LENS, **i32)
    out = torch.full_like(q, OUT_GUARD)
    lse = torch.full((H, T), LSE_GUARD, device=DEV)
    call("lgb200_attn_fwd_varlen", ptr(q), ptr(k), ptr(v), ptr(out), ptr(lse), ptr(q_off), ptr(q_len), ptr(q_off),
         ptr(q_len), len(LENS), max(LENS), T, T, H, hd ** -0.5, ops._code(dtype), hd, stream_ptr())
    torch.cuda.synchronize()
    written = torch.zeros(T, dtype=torch.bool)
    for o, n in zip(offs, LENS):
        written[o:o + n] = True
    outside = lse[:, ~written.to(DEV)]
    assert torch.equal(outside, torch.full_like(outside, LSE_GUARD))
    assert torch.isfinite(lse[:, written.to(DEV)]).all()


@pytest.mark.parametrize("hd,H", [(64, 4), (32, 8)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("B,Nq,Nk", [(2, 192, 192), (1, 150, 203)])
def test_varlen_equals_uniform_kernel_bitwise(B, Nq, Nk, dtype, hd, H):
    """Sequences of one length packed back to back compute what the uniform kernel computes, bit for bit, in the
    self (Nq == Nk) and the cross layout (both directions of B pairs; Nq != Nk: one direction)."""
    g = torch.Generator(device="cpu").manual_seed(Nq + Nk + hd)
    i32 = dict(device=DEV, dtype=torch.int32)
    scale = hd ** -0.5
    q = torch.randn(2 * B, Nq, H, hd, generator=g).to(DEV, dtype)
    kv = [torch.randn(2 * B, Nk, H, hd, generator=g).to(DEV, dtype) for _ in range(2)]
    if Nq == Nk:  # [image0 of every pair; image1 of every pair], kv_shift = B: each query batch attends to its partner
        ref, ref_lse = ops.attn_fwd(q, kv[0], kv[1], B, scale)
        off = torch.arange(2 * B, **i32) * Nq
        ln = torch.full((2 * B,), Nq, **i32)
        part = ((torch.arange(2 * B, device=DEV) + B) % (2 * B)) * Nq
        out, lse = ops.attn_fwd_varlen(q.view(-1, H, hd), kv[0].view(-1, H, hd), kv[1].view(-1, H, hd), off, ln,
                                       part.to(torch.int32), ln, Nq, scale)
        assert torch.equal(out.view_as(ref), ref)
        assert torch.equal(lse.view(H, 2 * B, Nq).permute(1, 0, 2), ref_lse)
    else:
        ref, ref_lse = ops.attn_fwd(q, kv[0], kv[1], 0, scale)
        qo, ko = torch.arange(2 * B, **i32) * Nq, torch.arange(2 * B, **i32) * Nk
        out, lse = ops.attn_fwd_varlen(q.view(-1, H, hd), kv[0].view(-1, H, hd), kv[1].view(-1, H, hd), qo,
                                       torch.full((2 * B,), Nq, **i32), ko, torch.full((2 * B,), Nk, **i32), Nq, scale)
        assert torch.equal(out.view_as(ref), ref)
        assert torch.equal(lse.view(H, 2 * B, Nq).permute(1, 0, 2), ref_lse)


def _adaptive_layout(seed):
    """32 pairs packed back to back, pair-major, without guard rows, as LightGlue's adaptive forward packs them after
    a stop / prune step: lengths in [1, 2048] (tile edges among them), three stopped pairs of length 0, and the last
    segment ending at T."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    lens = torch.randint(1, 2049, (64,), generator=g).tolist()
    lens[:12] = [1, 2, 63, 64, 65, 127, 129, 2047, 2048, 1000, 31, 33]
    for b in (5, 17, 26):  # stopped pairs
        lens[2 * b] = lens[2 * b + 1] = 0
    lens[-2:] = [777, 1531]
    offs = [0]
    for n in lens[:-1]:
        offs.append(offs[-1] + n)
    return offs, lens, offs[-1] + lens[-1]


@pytest.mark.parametrize("cross", [False, True], ids=["self", "cross"])
@pytest.mark.parametrize("hd,H", [(64, 4), (32, 4), (32, 8)])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_varlen_adaptive_layout_against_fp64(dtype, hd, H, cross):
    """Segments of unequal lengths back to back: a partial key tile of one sequence reads the first tokens of the next.
    Those tokens' keys and values are scaled up (keys x 8, values x 64), so a leak would dominate the softmax; each
    sequence must still equal fp64 attention over its own keys (cross: its partner's, s ^ 1)."""
    offs, lens, T = _adaptive_layout(seed=hd + H)
    g = torch.Generator(device="cpu").manual_seed(7 * hd + H + int(cross))
    q, k, v = (torch.randn(T, H, hd, generator=g) for _ in range(3))
    for o, n in zip(offs, lens):  # the first tokens of every segment: the keys just past the previous one's end
        k[o:o + min(n, 16)] *= 8.0
        v[o:o + min(n, 16)] *= 64.0
    q, k, v = (t.to(DEV, dtype) for t in (q, k, v))
    partner = [s ^ 1 for s in range(64)] if cross else list(range(64))
    i32 = dict(device=DEV, dtype=torch.int32)
    q_off, q_len = torch.tensor(offs, **i32), torch.tensor(lens, **i32)
    k_off, k_len = q_off[partner].contiguous(), q_len[partner].contiguous()
    scale = hd ** -0.5
    out, lse = ops.attn_fwd_varlen(q, k, v, q_off, q_len, k_off, k_len, max(lens), scale)
    torch.cuda.synchronize()
    worst = 0.0
    for s, (o, n) in enumerate(zip(offs, lens)):
        ko, kn = offs[partner[s]], lens[partner[s]]
        if n == 0 or kn == 0:
            continue
        got, gl = out[o:o + n], lse[:, o:o + n]
        if dtype == torch.bfloat16:
            r = attn_ref(q[o:o + n], k[ko:ko + kn], v[ko:ko + kn], scale)
            worst = max(worst, _within((got.double() - r["O"]).abs(), r["bO"], f"adaptive layout out s{s}", log=False),
                        _within((gl.double() - r["lse"]).abs(), r["blse"], f"adaptive layout lse s{s}", log=False))
        else:
            Q, K, V = (t.double().permute(1, 0, 2) for t in (q[o:o + n], k[ko:ko + kn], v[ko:ko + kn]))
            S = scale * Q @ K.transpose(1, 2)
            P = torch.softmax(S, -1)
            O = (P @ V).permute(1, 0, 2)
            L = torch.logsumexp(S, -1)
            # 2e-5 relative to the magnitudes summed, plus the fp32 rounding of the scores (32 u |q| . |k| each),
            # which the scaled keys make large: it moves each p by p dS, so O by sum_j p_j dS_j (|v_j| + |O|)
            dS = 32 * 2.0 ** -24 * scale * (Q.abs() @ K.abs().transpose(1, 2))
            PdS = P * dS
            bO = (2e-5 * (1 + P @ V.abs()) + PdS @ V.abs() + PdS.sum(-1, keepdim=True) * (P @ V).abs()).permute(1, 0, 2)
            bL = 2e-5 * (1 + L.abs()) + PdS.sum(-1)
            worst = max(worst, _within((got.double() - O).abs(), bO, f"adaptive layout out s{s}", log=False),
                        _within((gl.double() - L).abs(), bL, f"adaptive layout lse s{s}", log=False))
    report(f"varlen adaptive layout {dtype} hd{hd} H{H} {'cross' if cross else 'self'}", T=T,
           max_err_over_bound=worst)
