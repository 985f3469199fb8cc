"""GPU: the Hopper tensor-core kernels (csrc/gemm_tc.cu, csrc/attn_tc.cu, csrc/assign_tc.cu) element by element against
plain fp64 evaluations of the same operations on the same bf16 operands, at the benchmark's launch shapes (32 pairs of
2048 + 2048 keypoints = 131072 tokens, 64 attention sequences) and at tile edges.  References are torch fp64 on the
device, split per sequence / batch so that no N x N fp64 tensor over ~0.5 GB is alive at once.

Units:
  U32  = 2^-24   fp32 unit round-off (one rounding of an fp32 add, multiply or fma)
  UACC = 2^-23   one fp32 accumulation step of the tensor cores; twice U32 so that an accumulator that truncates
                 instead of rounding to nearest still meets the bound
  UBF  = 2^-8    bf16 rounding to nearest-even (8-bit significand: off by at most 2^-8 of the value)
  EX2  = 2^-21   relative error of ex2.approx.ftz.f32 (2^-22 per the PTX ISA), doubled for the fp32 rounding of its
                 argument

GEMMs (ops.gemm_bf16, ops.linear on the A-panel and the generic kernel, ops.wgrad_bf16 = split-K):
  exact   integer operands with |a| |b| K <= 2^23, alpha = 1/2, integer bias and initial C: every partial sum is a
          multiple of 1/2 below 2^23, which fp32 holds exactly in any summation order.  fp32 C must equal the exact
          result bit for bit, bf16 C must equal it rounded to nearest-even.  Zero tolerance: a dropped or repeated
          k-block, a wrong tile or split-K partial, or a truncating bf16 store fails.
  bounded randn operands:
          |C - C64| <= |alpha| n UACC (|A| |B|^T) + U32 |C64| + [bf16 C] UBF |C64|
                       + [bias / accumulate] U32 (|alpha| |A| |B|^T + |bias| + |C0|)
          n = K for one pass; split-K: the longest chain, 64 ceil(k-blocks / splits) + splits.

Attention (lgb200_attn_fwd / lgb200_attn_bwd, shared-qk backward), per (sequence, head), scale = 1/8, P = softmax(S):
  S error   dS_j = 64 UACC scale (|q| |k_j|); each p_j is off by a relative eps_j = dS_j + EX2 + 3 U32 (|S_j| + |max S|)
            (its exponent is an fp32 fma of S and the running maximum)
  O         2 UBF P'|V| + UBF |O| + 2 (P eps)|V| + 2 (P eps)1 |O| + n_o U32 P|V|
            P' = P without the keys at the row's maximum: their unnormalised p is exp2(0) = 1, which bf16 holds, so
            only the other keys' p carry the rounding of P to bf16; c = 2 covers that rounding (1) and the fp32
            rescales by the running maximum.  n_o = 2 Nk + Nk/4 + Nk/64 + 16: the P V accumulation (UACC per key), the
            row sum l (Nk/4 per lane, then the quad) and one rescale per key tile.
  lse       (P eps)1 + (Nk/4 + 16) U32 + 4 U32 (|max S| + |lse|)     (absolute)
  dV        2 UBF P^T|dO| + UBF |dV| + 2 (P eps)^T|dO| + Nq UACC P^T|dO|
  dQ, dK    through A = P o (|dO||V|^T + |delta|), delta = rowsum(dO o O) of the STORED bf16 O (what the kernel reads;
            the reference uses the same delta): dS = P o (dP - delta) is rounded to bf16 (UBF |dS| <= UBF A), and is
            off before that by A (eps + 64 UACC) (p and dP);
            dQ: scale (2 UBF A + 2 A eps' + Nk UACC A)|K| + UBF |dQ|,  dK: scale (...)^T |Q| + UBF |dK|,
            eps' = eps + 64 UACC; c = 2 on the dS rounding for the fp32 products around it.
  q = 0     every p is exactly 1, so P' = 0 and O = mean of the Nk valid values of V with V ~ 1.25: the bound is then
            ~0.6 bf16 ulp of O, so a padded key leaking into l, or a truncating store, fails.

Fused assignment head (assign_fused_stats / assign_fused_bwd), per pair, s = alpha md0 md1^T:
  es        D UACC alpha (|md0| |md1|^T), the error of s
  lse_row   (Pr eps_r)1 + (N/4 + 16) U32 + 4 U32 (|max s| + |lse|), eps_r = es + EX2 + 3 U32 (|s| + |max s|)
            (lse_col likewise over columns)
  scores    sb = 2 es + b(lse_row) + b(lse_col) + 4 U32 (2|s| + |lse_row| + |lse_col| + |ls0| + |ls1|)
  rowmax    max_j sb (the maximum of perturbed values moves by at most the largest perturbation); colmax likewise
  argmax    rowarg == fp64 argmax where the fp64 top-2 margin exceeds 2 max_j sb (asserted for >= 90 % of the rows);
            every other row's pick scores within 2 max_j sb of the maximum
  pos_row_sum  sum_j gt (2 es + b(lse_row) + b(lse_col) + 6 U32 (2|s| + |lse_row| + |lse_col| + |ls1|))
               + (N/4 + 4) U32 sum_j gt |2 s - lse_row - lse_col|
  dmd0      (2 UBF |dsim| + 2 ddsim + N UACC |dsim|) |md1| + UBF |dmd0|, ddsim = gc (Pr rowcnt eps_r' + Pc colcnt eps_c'),
            eps' = es + b(lse) + EX2 + 4 U32 (|s| + |lse|): dsim is rounded to bf16 before its product; dmd1 likewise.
  labels as match lists (gt = gt_t = NULL): STATS reads no mask for its LSE / max / argmax outputs, which must equal the
            mask mode's bit for bit.  assign_pos_fwd from the descriptors is held to the bound of
            tests/test_gpu_sparse_labels.py, (2 D + 8) U32 (2 alpha |md0_i| . |md1_j| + |lse_row_i| + |lse_col_j|) at
            the kernel's own LSEs.  The fused backward then rounds X = dsim' md1 to bf16, dsim' = dsim without its
            2 gc entries at the positives, and assign_pos_bwd adds 2 gc md1[gt0[i]] to that bf16 value in one fp32 fma
            and rounds again: dmd0 is within b1 = (2 UBF |dsim'| + 2 ddsim + N UACC |dsim'|) |md1| + UBF |X| (the
            mask mode's bound for the partial product) plus (UBF + U32) (|dmd0| + b1) for the second rounding of a
            value already off by b1; dmd1 likewise.

Every check takes a NaN as a failure (unwritten outputs show as NaN) and records its largest err / bound through
tests.util.report.  Attention outputs, lse, dq / dk / dv and d(mdesc) land in buffers with NaN-pattern guard rows on
both sides, which must come back unchanged; the benchmark-shaped attention and GEMM launches are run twice and must agree
bit for bit.  The negative controls at the end run on the CPU: each check function rejects a wrong answer built from
its own reference (bf16 truncation, a k-block left out, a key tile left out, a stale softmax maximum, padded keys in
the row sum, a swapped pair of argmax indices).

Budget: under 3 minutes and 20 GiB peak device memory on one H100, recorded by the module fixture.
"""
import math
import time

import pytest
import torch

from gluefactory_b200 import _lib, ops
from gluefactory_b200._lib import call, ptr, stream_ptr
from tests.util import report

GPU = pytest.mark.gpu
DEV = "cuda"
U32, UACC, UBF, EX2 = 2.0 ** -24, 2.0 ** -23, 2.0 ** -8, 2.0 ** -21
TOK = 131072  # tokens of the benchmark's step: 32 pairs x (2048 + 2048)
SCALE = 0.125  # attention scale of head_dim 64
BF16_GUARD, F32_GUARD = 0x7FA5, 0x7FA5A5A5  # NaN bit patterns of the guard rows


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
    report("test_gpu_tensor_core_kernels", seconds=time.time() - t,
           peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)


def _gen(seed, dev=DEV):
    return torch.Generator(device=dev).manual_seed(seed)


def _within(err, bound, tag, log=True):
    """err <= bound elementwise (a NaN error fails: an output left unwritten shows as NaN); returns (and records) the
    largest err / bound."""
    err, bound = err.double(), bound.double()
    ratio = (err / bound.clamp(min=1e-300)).max().item() if err.numel() else 0.0
    if log:
        report(tag, max_err_over_bound=ratio)
    bad = ~(err <= bound)
    assert not bad.any(), (tag, int(bad.sum()), ratio, err[bad][:4].tolist(), bound[bad][:4].tolist())
    return ratio


class _Worst:
    """Largest err / bound per quantity over the chunks of one case, reported once."""

    def __init__(self, tag):
        self.tag, self.r = tag, {}

    def __call__(self, name, err, bound):
        r = _within(err, bound, f"{self.tag} {name}", log=False)
        self.r[name] = max(self.r.get(name, 0.0), r)

    def report(self):
        report(self.tag, **{f"{k}_err_over_bound": v for k, v in self.r.items()})


def _trunc_bf16(x):
    """x rounded toward zero to bf16 (a truncating epilogue; negative control)."""
    b = x.float().contiguous().view(torch.int32) & -65536
    return b.view(torch.float32).to(torch.bfloat16)


# ================================================================================================
# check functions (device-agnostic: the negative controls run them on the CPU)
# ================================================================================================
def gemm_bound(absprod, n, alpha, ref, out_dtype, addend_abs=None):
    """The GEMM error bound of the module docstring; absprod = |A| |B|^T, addend_abs = |bias| + |C0| (or None)."""
    b = abs(alpha) * n * UACC * absprod + U32 * ref.abs()
    if addend_abs is not None:
        b = b + U32 * (abs(alpha) * absprod + addend_abs)
    if out_dtype == torch.bfloat16:
        b = b + UBF * ref.abs()
    return b


def check_gemm(got, ref, bound, tag, log=True):
    return _within((got.double() - ref).abs(), bound, tag, log=log)


def check_exact(got, exact, tag, log=True):
    """got == exact (fp64, exactly representable in fp32) in got's dtype: fp32 bit for bit, bf16 rounded to
    nearest-even.  Returns the share of elements that need more than bf16's 8 significant bits."""
    want = exact.to(got.dtype)
    bad = ~(got == want)
    wide = (exact != exact.float().to(torch.bfloat16).double()).double().mean().item() if exact.numel() else 0.0
    if log:
        report(tag, mismatches=int(bad.sum()), wider_than_bf16=wide)
    assert not bad.any(), (tag, int(bad.sum()), got[bad][:4].tolist(), want[bad][:4].tolist())
    return wide


def attn_ref(q, k, v, scale=SCALE, out=None, do=None):
    """fp64 attention of one sequence, q [Nq,H,64], k / v [Nk,H,64] (the kernel's bf16 values), with the bounds of the
    module docstring.  With out (the kernel's stored O) and do: the backward too, delta taken from out."""
    Q, K, V = (t.double().permute(1, 0, 2) for t in (q, k, v))  # [H, N, 64]
    Nq, Nk = Q.shape[1], K.shape[1]
    S = scale * (Q @ K.transpose(1, 2))
    m = S.amax(-1, keepdim=True)
    E = torch.exp(S - m)
    P = E / E.sum(-1, keepdim=True)
    del E
    lse = (m + torch.log(torch.exp(S - m).sum(-1, keepdim=True))).squeeze(-1)
    eps = (64 * UACC * scale) * (Q.abs() @ K.abs().transpose(1, 2)) + EX2 + 3 * U32 * (S.abs() + m.abs())
    Pe = P * eps
    aV = V.abs()
    O = P @ V
    PV = P @ aV
    PVx = torch.where(S < m, P, torch.zeros_like(P)) @ aV
    n_o = 2 * Nk + Nk / 4 + Nk / 64 + 16
    Pe1 = Pe.sum(-1, keepdim=True)
    r = dict(O=O, lse=lse,
             bO=2 * UBF * PVx + UBF * O.abs() + 2 * (Pe @ aV) + 2 * Pe1 * O.abs() + n_o * U32 * PV,
             blse=Pe1.squeeze(-1) + (Nk / 4 + 16) * U32 + 4 * U32 * (m.squeeze(-1).abs() + lse.abs()))
    if do is not None:
        dO = do.double().permute(1, 0, 2)
        Os = out.double().permute(1, 0, 2)
        delta = (dO * Os).sum(-1, keepdim=True)
        adO = dO.abs()
        dS = P * (dO @ V.transpose(1, 2) - delta)
        A = P * (adO @ aV.transpose(1, 2) + delta.abs())
        r["dV"] = P.transpose(1, 2) @ dO
        r["dQ"] = scale * (dS @ K)
        r["dK"] = scale * (dS.transpose(1, 2) @ Q)
        del dS
        r["bdV"] = ((2 * UBF + Nq * UACC) * P + 2 * Pe).transpose(1, 2) @ adO + UBF * r["dV"].abs()
        W = (2 * UBF + Nk * UACC) * A + 2 * A * (eps + 64 * UACC)
        r["bdQ"] = scale * (W @ K.abs()) + UBF * r["dQ"].abs()
        W = (2 * UBF + Nq * UACC) * A + 2 * A * (eps + 64 * UACC)
        r["bdK"] = scale * (W.transpose(1, 2) @ Q.abs()) + UBF * r["dK"].abs()
    # back to the kernel's layouts: O / dQ [Nq,H,64], dK / dV [Nk,H,64], lse [H,Nq]
    return {key: (t if key in ("lse", "blse") else t.permute(1, 0, 2)) for key, t in r.items()}


def check_attn_fwd(out, lse, r, w):
    w("out", (out.double() - r["O"]).abs(), r["bO"])
    w("lse", (lse.double() - r["lse"]).abs(), r["blse"])


def check_attn_bwd(dq, dk, dv, r, w):
    w("dq", (dq.double() - r["dQ"]).abs(), r["bdQ"])
    w("dk", (dk.double() - r["dK"]).abs(), r["bdK"])
    w("dv", (dv.double() - r["dV"]).abs(), r["bdV"])


def _lse_with_bound(s, es, dim):
    """logsumexp of s over dim and its absolute bound (module docstring)."""
    mx = s.amax(dim, keepdim=True)
    lse = mx + torch.log(torch.exp(s - mx).sum(dim, keepdim=True))
    P = torch.exp(s - lse)
    eps = es + EX2 + 3 * U32 * (s.abs() + mx.abs())
    n = s.shape[dim]
    b = (P * eps).sum(dim, keepdim=True) + (n / 4 + 16) * U32 + 4 * U32 * (mx.abs() + lse.abs())
    return lse, b, P


def assign_ref(md0, md1, alpha, ls0, ls1, gt, gc, lists=False):
    """fp64 assignment head of one pair: md0 [M,D], md1 [N,D] bf16, ls0 [M], ls1 [N], gt [M,N] bool, gc scalar.
    lists: the d(mdesc) bounds of the mask-free backward followed by assign_pos_bwd (module docstring)."""
    A, Bm = md0.double(), md1.double()
    D = A.shape[1]
    s = alpha * (A @ Bm.t())
    es = (D * UACC * alpha) * (A.abs() @ Bm.abs().t())
    lr, blr, Pr = _lse_with_bound(s, es, 1)
    lc, blc, Pc = _lse_with_bound(s, es, 0)
    l0, l1 = ls0.double()[:, None], ls1.double()[None, :]
    sc = (s - lr) + (s - lc) + (l0 + l1)
    sb = 2 * es + blr + blc + 4 * U32 * (2 * s.abs() + lr.abs() + lc.abs() + l0.abs() + l1.abs())
    g = gt.double()
    t = 2 * s - lr - lc
    r = dict(lse_row=lr[:, 0], b_lse_row=blr[:, 0], lse_col=lc[0], b_lse_col=blc[0], sc=sc,
             rowmax=sc.amax(1), b_rowmax=sb.amax(1), colmax=sc.amax(0), b_colmax=sb.amax(0),
             pos_row_sum=(g * t).sum(1),
             b_pos=(g * (2 * es + blr + blc + 6 * U32 * (2 * s.abs() + lr.abs() + lc.abs() + l1.abs()))).sum(1)
             + (s.shape[1] / 4 + 4) * U32 * (g * t.abs()).sum(1))
    rowcnt, colcnt = g.sum(1, keepdim=True), g.sum(0, keepdim=True)
    dsim = gc * (2 * g - Pr * rowcnt - Pc * colcnt)
    er = es + blr + EX2 + 4 * U32 * (s.abs() + lr.abs())
    ec = es + blc + EX2 + 4 * U32 * (s.abs() + lc.abs())
    ddsim = abs(gc) * (Pr * rowcnt * er + Pc * colcnt * ec)
    M, N = s.shape
    r["dmd0"] = dsim @ Bm
    r["dmd1"] = dsim.t() @ A
    if not lists:
        r["b_dmd0"] = ((2 * UBF + N * UACC) * dsim.abs() + 2 * ddsim) @ Bm.abs() + UBF * r["dmd0"].abs()
        r["b_dmd1"] = ((2 * UBF + M * UACC) * dsim.abs() + 2 * ddsim).t() @ A.abs() + UBF * r["dmd1"].abs()
        return r
    part = dsim - 2 * gc * g  # what the fused kernel contracts without masks
    b1 = ((2 * UBF + N * UACC) * part.abs() + 2 * ddsim) @ Bm.abs() + UBF * (part @ Bm).abs()
    r["b_dmd0"] = b1 + (UBF + U32) * (r["dmd0"].abs() + b1)
    b1 = ((2 * UBF + M * UACC) * part.abs() + 2 * ddsim).t() @ A.abs() + UBF * (part.t() @ A).abs()
    r["b_dmd1"] = b1 + (UBF + U32) * (r["dmd1"].abs() + b1)
    return r


def check_argmax(arg, sc, bmax, dim, tag, w=None, min_share=0.9):
    """arg (the kernel's first argmax along dim) against the fp64 scores sc: equal to the fp64 argmax wherever the
    fp64 top-2 margin exceeds twice the score bound bmax (at least min_share of the lines qualify); elsewhere a pick
    within 2 bmax of the maximum."""
    arg = arg.long()
    top = sc.topk(2, dim=dim).values if sc.shape[dim] > 1 else torch.cat([sc.amax(dim, keepdim=True)] * 2, dim)
    top = top.movedim(dim, -1)
    margin = top[..., 0] - top[..., 1]
    sure = margin > 2 * bmax if sc.shape[dim] > 1 else torch.ones_like(margin, dtype=torch.bool)
    ref = sc.argmax(dim)
    share = sure.double().mean().item()
    assert share >= min_share, (tag, "rows with a clear maximum", share)
    bad = sure & (arg != ref)
    assert not bad.any(), (tag, "argmax", int(bad.sum()), arg[bad][:4].tolist(), ref[bad][:4].tolist())
    assert ((arg >= 0) & (arg < sc.shape[dim])).all(), (tag, "argmax out of range")
    picked = sc.gather(dim, arg.unsqueeze(dim)).squeeze(dim)
    slack = top[..., 0] - picked
    assert (slack <= 2 * bmax).all(), (tag, "argmax pick", slack.max().item())
    if w is not None:
        w.r[f"{tag}_clear_share"] = share
    return share


# ================================================================================================
# 1. GEMMs
# ================================================================================================
def _draw(shape, exact, g, K=None):
    """bf16 operands: integers |x| <= r with r^2 K <= 2^23 (r <= 256, bf16-exact) when exact, else randn."""
    if exact:
        r = min(256, int(math.isqrt(2 ** 23 // K)))
        return torch.randint(-r, r + 1, shape, device=DEV, generator=g).to(torch.bfloat16)
    return torch.randn(*shape, device=DEV, generator=g).to(torch.bfloat16)


def _addend(shape, exact, g, big):
    if exact:
        return torch.randint(-big, big + 1, shape, device=DEV, generator=g).float()
    return torch.randn(*shape, device=DEV, generator=g)


def _gemm_case(batch, M, N, K, a_mn, b_mn, out_dtype, exact, seed, again=False, tag=""):
    g = _gen(seed)
    a = _draw((batch, K, M) if a_mn else (batch, M, K), exact, g, K)
    b = _draw((batch, K, N) if b_mn else (batch, N, K), exact, g, K)
    alpha = 0.5 if exact else 0.37
    c = ops.gemm_bf16(a, b, a_mn_major=a_mn, b_mn_major=b_mn, out_dtype=out_dtype, alpha=alpha)
    if again:
        assert torch.equal(c, ops.gemm_bf16(a, b, a_mn_major=a_mn, b_mn_major=b_mn, out_dtype=out_dtype, alpha=alpha))
    w = _Worst(tag)
    wide = []
    for i in range(batch):
        A64 = a[i].double().t() if a_mn else a[i].double()  # [M, K]
        B64 = b[i].double().t() if b_mn else b[i].double()  # [N, K]
        ref = alpha * (A64 @ B64.t())
        if exact:
            wide.append(check_exact(c[i], ref, f"{tag} b={i}", log=False))
        else:
            w("C", (c[i].double() - ref).abs(), gemm_bound(A64.abs() @ B64.abs().t(), K, alpha, ref, out_dtype))
    if exact:
        report(tag, mismatches=0, wider_than_bf16=sum(wide) / len(wide))
    else:
        w.report()
    return sum(wide) / len(wide) if wide else None


def _linear_case(M, N, K, *, w_is_kn, bias, out_dtype, accumulate, exact, seed, a_pad=0, c_off=0, again=False,
                 tag="", chunk=16384):
    """ops.linear with A a column block of a [M, K + a_pad] matrix and C the columns [c_off, c_off + N) of a
    [M, N + 8] buffer whose other columns must keep their NaN pattern."""
    g = _gen(seed)
    a = _draw((M, K + a_pad), exact, g, K)[:, a_pad:]
    wt = _draw((K, N) if w_is_kn else (N, K), exact, g, K)
    bv = _addend((N,), exact, g, 2 ** 15) if bias else None
    alpha = 0.5 if exact else 0.7
    cbig = torch.empty(M, N + 8, device=DEV, dtype=out_dtype)
    cbig.view(torch.int32 if out_dtype == torch.float32 else torch.int16).fill_(
        F32_GUARD if out_dtype == torch.float32 else BF16_GUARD)
    out = cbig[:, c_off:c_off + N]
    c0 = None
    if accumulate:
        c0 = _addend((M, N), exact, g, 2 ** 20)
        out.copy_(c0)
    keep = cbig.clone()
    ops.linear(a, wt, bias=bv, out=out, w_is_kn=w_is_kn, accumulate=accumulate, alpha=alpha)
    outside = torch.ones(M, N + 8, dtype=torch.bool, device=DEV)
    outside[:, c_off:c_off + N] = False
    assert torch.equal(cbig[outside].view(torch.uint8), keep[outside].view(torch.uint8)), (tag, "stray write")
    if again:
        assert torch.equal(out, ops.linear(a, wt, bias=bv, out_dtype=out_dtype, w_is_kn=w_is_kn, alpha=alpha)), tag
    W64 = wt.double().t() if w_is_kn else wt.double()  # [N, K]
    w = _Worst(tag)
    wide = []
    for s in range(0, M, chunk):
        A64 = a[s:s + chunk].double()
        ref = alpha * (A64 @ W64.t())
        add = None
        if bias:
            ref = ref + bv.double()
            add = bv.double().abs().expand_as(ref)
        if accumulate:
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


def _splitk_chain(M, N, K):
    """Longest summation chain of the split-K GEMM: 64 ceil(k-blocks / splits) products, then the splits."""
    splits = _lib.load().lgb200_gemm_splitk_ws_floats(M, N, K) // (M * N)
    nk = -(-K // 64)
    return 64 * -(-nk // splits) + splits, splits


def _wgrad_case(T, M, N, exact, seed, pad=0, tag="", chunk=16384):
    g = _gen(seed)
    dy = _draw((T, M + pad), exact, g, T)[:, pad:]
    a = _draw((T, N + pad), exact, g, T)[:, pad:]
    out = torch.full((M, N), float("nan"), device=DEV)
    ops.wgrad_bf16(dy, a, out=out)
    again = torch.full_like(out, float("nan"))
    ops.wgrad_bf16(dy, a, out=again)
    assert torch.equal(out, again), (tag, "split-K sum order")
    ref = torch.zeros(M, N, device=DEV, dtype=torch.float64)
    absprod = torch.zeros_like(ref)
    for s in range(0, T, chunk):
        d64, a64 = dy[s:s + chunk].double(), a[s:s + chunk].double()
        ref += d64.t() @ a64
        absprod += d64.abs().t() @ a64.abs()
    n, splits = _splitk_chain(M, N, T)
    if exact:
        check_exact(out, ref, tag)
    else:
        _within((out.double() - ref).abs(), gemm_bound(absprod, n, 1.0, ref, torch.float32), f"{tag} splits={splits}")


# (name, M, N, K, w_is_kn, bias, out dtype, accumulate): the layer step's launches at 131072 tokens
BENCH_LINEAR = [
    ("qkv", TOK, 768, 256, False, True, torch.bfloat16, False),          # A-panel
    ("out", TOK, 256, 256, False, True, torch.bfloat16, False),          # A-panel
    ("ffn0", TOK, 512, 512, False, True, torch.bfloat16, False),         # generic
    ("ffn1", TOK, 256, 512, False, True, torch.bfloat16, False),         # generic
    ("qkv.dgrad", TOK, 256, 768, True, False, torch.float32, True),      # generic, TMA reduce-add
    ("out.dgrad", TOK, 256, 256, True, False, torch.bfloat16, False),    # A-panel, MN-major W
    ("ffn0.dgrad", TOK, 512, 512, True, False, torch.float32, True),     # generic, TMA reduce-add
    ("ffn1.dgrad", TOK, 512, 256, True, False, torch.float32, True),     # A-panel, TMA reduce-add
]


@GPU
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "bounded"])
@pytest.mark.parametrize("case", BENCH_LINEAR, ids=[c[0] for c in BENCH_LINEAR])
def test_linear_bench_shapes(case, exact):
    name, M, N, K, kn, bias, odt, acc = case
    wide = _linear_case(M, N, K, w_is_kn=kn, bias=bias, out_dtype=odt, accumulate=acc, exact=exact, seed=K + N,
                        again=not acc and K <= 256, tag=f"linear {name} T={M} {'exact' if exact else 'bounded'}")
    if exact and odt == torch.bfloat16:
        assert wide > 0.5, wide  # most results are rounded: a truncating store cannot hide


@GPU
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "bounded"])
@pytest.mark.parametrize("M,N", [(768, 256), (256, 256), (512, 512), (256, 512)])
def test_wgrad_bench_shapes(M, N, exact):
    """The step's weight gradients dy^T x over the 131072 tokens; dy and x are column blocks of wider matrices."""
    _wgrad_case(TOK, M, N, exact, seed=M + N, pad=8 if M == 256 else 0,
                tag=f"wgrad T={TOK} {M}x{N} {'exact' if exact else 'bounded'}")


@GPU
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "bounded"])
@pytest.mark.parametrize("n", [2048, 1024])
def test_gluestick_similarity_gemms(n, exact):
    """GlueStick's similarity and its two backward GEMMs (matchers/gluestick.py::_BmmNT) at 8 pairs: 2048 points and
    1024 line endpoints.  8 x 16 x 16 = 2048 output tiles: the persistent loop goes round ~16 times."""
    kind = "exact" if exact else "bounded"
    _gemm_case(8, n, n, 256, False, False, torch.float32, exact, seed=n, again=True, tag=f"bmm_nt sim n={n} {kind}")
    wide = _gemm_case(8, n, 256, n, False, True, torch.bfloat16, exact, seed=n + 1, tag=f"bmm_nt da n={n} {kind}")
    wide2 = _gemm_case(8, n, 256, n, True, True, torch.bfloat16, exact, seed=n + 2, tag=f"bmm_nt db n={n} {kind}")
    if exact:
        assert wide > 0.5 and wide2 > 0.5, (wide, wide2)


LAYOUTS = [(False, False), (False, True), (True, False), (True, True)]


@GPU
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "bounded"])
@pytest.mark.parametrize("out_dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("a_mn,b_mn", LAYOUTS)
def test_gemm_bf16_edges(a_mn, b_mn, out_dtype, exact):
    """Ragged M, N and K at every layout (MN-major operands need M / N % 8 == 0: their row pitch), batch 3."""
    Ms = [8, 72, 136] if a_mn else [1, 63, 65, 129]
    Ns = [8, 72, 136] if b_mn else [8, 72, 130, 136]
    i = 0
    for M in Ms:
        for N in Ns:
            for K in (8, 56, 72, 256, 264):
                i += 1
                _gemm_case(3, M, N, K, a_mn, b_mn, out_dtype, exact, seed=i,
                           tag=f"gemm_bf16 {int(a_mn)}{int(b_mn)} {str(out_dtype)[6:]} {M}x{N}x{K} "
                               f"{'exact' if exact else 'bounded'}")


@GPU
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "bounded"])
@pytest.mark.parametrize("K", [8, 56, 72, 256, 264])
def test_linear_edges(K, exact):
    """K <= 256: the A-panel kernel; K = 264: the generic one.  Each (M, N) pair runs a different combination of
    w_is_kn, bias, output (bf16 / fp32 / fp32 accumulate) and C placement: 16-byte aligned (TMA epilogue), 8-byte
    aligned (paired register stores) or odd (scalar register stores), with A a row-strided column block."""
    combos = [(kn, bias, out, c_off) for kn in (False, True) for bias in (False, True)
              for out in ("bf16", "f32", "acc") for c_off in (0, 2, 1)]
    shapes = [(M, N) for M in (1, 63, 65, 129) for N in (8, 72, 130, 136)]
    for i, (kn, bias, out, c_off) in enumerate(combos):
        M, N = shapes[i % len(shapes)]
        if kn and N % 8:
            N = 136  # w [K, N] is read MN-major: its pitch N must be a multiple of 8
        odt = torch.bfloat16 if out == "bf16" else torch.float32
        _linear_case(M, N, K, w_is_kn=kn, bias=bias, out_dtype=odt, accumulate=out == "acc", exact=exact,
                     seed=1000 + 37 * K + i, a_pad=8 * (i % 2), c_off=c_off,
                     tag=f"linear {M}x{N}x{K} kn={int(kn)} bias={int(bias)} {out} c_off={c_off} "
                         f"{'exact' if exact else 'bounded'}")


@GPU
@pytest.mark.parametrize("exact", [True, False], ids=["exact", "bounded"])
def test_wgrad_edges(exact):
    """Split-K with few tokens (one split), a ragged last k-block, and column-slice operands."""
    i = 0
    for T in (8, 56, 264, 4097):
        for M in (8, 72, 136):
            for N in (8, 72, 136):
                i += 1
                _wgrad_case(T, M, N, exact, seed=500 + i, pad=8 * (i % 2),
                            tag=f"wgrad T={T} {M}x{N} {'exact' if exact else 'bounded'}")


# ================================================================================================
# 2. attention
# ================================================================================================
def _guarded(shape, dtype, guard):
    """A tensor of `shape` inside a flat buffer with `guard` elements before and after, all set to a NaN pattern."""
    n = math.prod(shape)
    buf = torch.empty(n + 2 * guard, device=DEV, dtype=dtype)
    buf.view(torch.int16 if dtype == torch.bfloat16 else torch.int32).fill_(
        BF16_GUARD if dtype == torch.bfloat16 else F32_GUARD)
    return buf, buf[guard:guard + n].view(shape), guard


def _guards_intact(g, tag):
    buf, _, guard = g
    bits = buf.view(torch.int16 if buf.dtype == torch.bfloat16 else torch.int32)
    pat = BF16_GUARD if buf.dtype == torch.bfloat16 else F32_GUARD
    assert (bits[:guard] == pat).all() and (bits[-guard:] == pat).all(), (tag, "guard rows overwritten")


def _attn_fwd_guarded(q, k, v, shift):
    B, Nq, H, _ = q.shape
    Nk = k.shape[1]
    go = _guarded((B, Nq, H, 64), torch.bfloat16, 2 * H * 64)
    gl = _guarded((B, H, Nq), torch.float32, 64)
    call("lgb200_attn_fwd", ptr(q), ptr(k), ptr(v), ptr(go[1]), ptr(gl[1]), B, Nq, Nk, H, shift, float(SCALE),
         _lib.BF16, stream_ptr())
    return go, gl


def _attn_bwd_guarded(q, k, v, out, lse, do, shift, shared=False):
    B, Nq, H, _ = q.shape
    Nk = k.shape[1]
    gq = _guarded((B, Nq, H, 64), torch.bfloat16, 2 * H * 64)
    gk = gq if shared else _guarded((B, Nk, H, 64), torch.bfloat16, 2 * H * 64)
    gv = _guarded((B, Nk, H, 64), torch.bfloat16, 2 * H * 64)
    ws = torch.empty(_lib.load().lgb200_attn_bwd_ws_floats(B, Nq, Nk, H), device=DEV)
    call("lgb200_attn_bwd", ptr(q), ptr(k), ptr(v), ptr(out), ptr(lse), ptr(do), ptr(gq[1]), ptr(gk[1]), ptr(gv[1]),
         ptr(ws), B, Nq, Nk, H, shift, float(SCALE), _lib.BF16, stream_ptr(), launches=2 if shared else None)
    return gq, gk, gv


def _attn_inputs(B, Nq, Nk, H, regime, seed, shared=False):
    """bf16 q, k, v, dout.  Regimes: randn (logits ~ randn * 1.5); spike (the last key, in a partial tile when
    Nk % 64 != 0, sits ~40 above every other logit of every row); rising (logits climb ~60 over the keys, so the
    running maximum grows in every key tile); zero_q (q = 0: every p is 1, out = mean of V, V ~ 1.25)."""
    g = _gen(seed)
    q = torch.randn(B, Nq, H, 64, device=DEV, generator=g) * 1.5
    k = q if shared else torch.randn(B, Nk, H, 64, device=DEV, generator=g)
    v = torch.randn(B, Nk, H, 64, device=DEV, generator=g)
    do = torch.randn(B, Nq, H, 64, device=DEV, generator=g)
    if regime == "spike":
        q[..., 0] = 8.0
        k[..., 0] = 0.0
        k[:, Nk - 1, :, 0] = 40.0  # 8 * 40 / 8 = 40
    elif regime == "rising":
        q[..., 0] = 8.0
        k[..., 0] = torch.linspace(0.0, 60.0, Nk, device=DEV)[None, :, None]
    elif regime == "zero_q":
        q.zero_()
        v = 1.25 + 0.1 * v
    bf = lambda t: t.to(torch.bfloat16).contiguous()  # noqa: E731
    q = bf(q)
    return q, (q if shared else bf(k)), bf(v), bf(do)


def _attn_run(B, Nq, Nk, H, shift, regime, seed, bwd=True, again=False, tag=""):
    q, k, v, do = _attn_inputs(B, Nq, Nk, H, regime, seed)
    go, gl = _attn_fwd_guarded(q, k, v, shift)
    out, lse = go[1], gl[1]
    if again:
        out2, lse2 = ops.attn_fwd(q, k, v, shift, SCALE)
        assert torch.equal(out, out2) and torch.equal(lse, lse2), (tag, "forward not bit-identical")
        del out2, lse2
    if bwd:
        gq, gk, gv = _attn_bwd_guarded(q, k, v, out, lse, do, shift)
        if again:
            again_ = ops.attn_bwd(q, k, v, out, lse, do, shift, SCALE)
            assert all(torch.equal(a, b[1]) for a, b in zip(again_, (gq, gk, gv))), (tag, "backward not bit-identical")
            del again_
    w = _Worst(tag)
    for b in range(B):
        kb = (b + shift) % B
        r = attn_ref(q[b], k[kb], v[kb], SCALE, out[b] if bwd else None, do[b] if bwd else None)
        check_attn_fwd(out[b], lse[b], r, w)
        if bwd:
            check_attn_bwd(gq[1][b], gk[1][kb], gv[1][kb], r, w)
        del r
    w.report()
    for gb in (go, gl) + ((gq, gk, gv) if bwd else ()):
        _guards_intact(gb, tag)


@GPU
@pytest.mark.parametrize("shift", [0, 32], ids=["self", "cross"])
def test_attention_bench_shape(shift):
    """The step's attention launch: 64 sequences (32 pairs x 2 images) x 2048 tokens x 4 heads, forward and backward,
    each run twice (bit-identical), into guarded buffers."""
    _attn_run(64, 2048, 2048, 4, shift, "randn", seed=7 + shift, again=True, tag=f"attn bench shift={shift}")


@GPU
def test_attention_shared_qk_bench_shape():
    """Shared-qk cross-attention backward at 32 pairs: dqk = dq + dk of the shared tensor, dv, against fp64."""
    B, N, H = 64, 2048, 4
    qk, _, v, do = _attn_inputs(B, N, N, H, "randn", seed=21, shared=True)
    out, lse = ops.attn_fwd(qk, qk, v, B // 2, SCALE)
    gq, _, gv = _attn_bwd_guarded(qk, qk, v, out, lse, do, B // 2, shared=True)
    dqk, dv = gq[1], gv[1]
    again, dv2 = ops.attn_bwd_shared_qk(qk, v, out, lse, do, SCALE)
    assert torch.equal(again, dqk) and torch.equal(dv2, dv)
    del again, dv2
    w = _Worst("attn shared_qk bench")
    for b in range(B):
        p = (b + B // 2) % B
        r_bp = attn_ref(qk[b], qk[p], v[p], SCALE, out[b], do[b])  # b's queries on p's keys: dQ_b
        r_pb = attn_ref(qk[p], qk[b], v[b], SCALE, out[p], do[p])  # p's queries on b's keys: dK_b, dV_b
        ref = r_bp["dQ"] + r_pb["dK"]
        bound = r_bp["bdQ"] + r_pb["bdK"] - UBF * (r_bp["dQ"].abs() + r_pb["dK"].abs()) + UBF * ref.abs()
        w("dqk", (dqk[b].double() - ref).abs(), bound)
        w("dv", (dv[b].double() - r_pb["dV"]).abs(), r_pb["bdV"])
        del r_bp, r_pb
    w.report()
    _guards_intact(gq, "attn shared_qk dqk")
    _guards_intact(gv, "attn shared_qk dv")


RAGGED = [(nq, nk) for nq in (1, 63, 64, 65, 129, 2049) for nk in (1, 63, 64, 65, 129, 2049) if nq != nk]


@GPU
@pytest.mark.parametrize("H", [1, 4])
@pytest.mark.parametrize("Nq,Nk", RAGGED)
def test_attention_ragged(Nq, Nk, H):
    """Nq != Nk as GlueStick calls it (self-attention layout, kv_shift 0), and a cross launch (kv_shift 1)."""
    _attn_run(2, Nq, Nk, H, (Nq + Nk) % 2, "randn", seed=Nq * 7 + Nk + H, tag=f"attn Nq={Nq} Nk={Nk} H={H}")


@GPU
@pytest.mark.parametrize("regime", ["randn", "spike", "rising", "zero_q"])
@pytest.mark.parametrize("Nq,Nk", [(200, 2049), (129, 65), (300, 1000)])
def test_attention_logit_regimes(regime, Nq, Nk):
    _attn_run(2, Nq, Nk, 2, 1, regime, seed=Nq + Nk, tag=f"attn {regime} Nq={Nq} Nk={Nk}")


# ================================================================================================
# 3. fused assignment head
# ================================================================================================
def _assign_inputs(B, M, N, D, seed):
    """Pair kinds by b % 4: a partial matching; no positives; a partial matching plus full-positive rows (every 7th);
    about a quarter of all pairs positive."""
    g = _gen(seed)
    md0 = (torch.randn(B, M, D, device=DEV, generator=g) * 2).to(torch.bfloat16)
    md1 = (torch.randn(B, N, D, device=DEV, generator=g) * 2).to(torch.bfloat16)
    ls0 = torch.nn.functional.logsigmoid(torch.randn(B, M, device=DEV, generator=g))
    ls1 = torch.nn.functional.logsigmoid(torch.randn(B, N, device=DEV, generator=g))
    gt = torch.zeros(B, M, N, device=DEV, dtype=torch.bool)
    K = max(1, min(M, N) // 3)
    for b in range(B):
        kind = b % 4
        if kind in (0, 2):
            gt[b, torch.randperm(M, device=DEV, generator=g)[:K], torch.randperm(N, device=DEV, generator=g)[:K]] = True
        if kind == 2:
            gt[b, 0::7] = True
        if kind == 3:
            gt[b] = torch.rand(M, N, device=DEV, generator=g) < 0.25
    gc = (torch.rand(B, device=DEV, generator=g) + 0.1) * D ** -0.5
    return md0, md1, D ** -0.5, ls0, ls1, gt, gc


def _assign_lists(B, M, N, seed):
    """One-to-one match lists gt0 [B,M] / gt1 [B,N] with -1 and -2 labels: pair 0 without positives, every other pair
    with min(M, N) // 3 positives at random rows and columns; a tenth of the unmatched points ignored."""
    g = torch.Generator().manual_seed(seed)
    m0 = torch.full((B, M), -1, dtype=torch.long)
    m1 = torch.full((B, N), -1, dtype=torch.long)
    K = max(1, min(M, N) // 3)
    for b in range(1, B):
        i, j = torch.randperm(M, generator=g)[:K], torch.randperm(N, generator=g)[:K]
        m0[b, i], m1[b, j] = j, i
    m0[(torch.rand(B, M, generator=g) < 0.1) & (m0 < 0)] = -2
    m1[(torch.rand(B, N, generator=g) < 0.1) & (m1 < 0)] = -2
    return m0.to(DEV), m1.to(DEV)


ASSIGN_SHAPES = [(32, 2048, 2048, 256), (32, 2048, 2048, 128), (4, 384, 320, 64), (4, 300, 257, 128), (4, 191, 321, 192), (4, 1000, 777, 256)]


# every shape with the mask (ids as before the lists mode existed) and with match lists ("-lists")
ASSIGN_CASES = [pytest.param(*s, labels, id="-".join(map(str, s)) + ("" if labels == "mask" else "-lists"))
                for labels in ("mask", "lists") for s in ASSIGN_SHAPES]


@GPU
@pytest.mark.parametrize("B,M,N,D,labels", ASSIGN_CASES)
def test_assign_fused_against_fp64(B, M, N, D, labels):
    md0, md1, alpha, ls0, ls1, gt, gc = _assign_inputs(B, M, N, D, seed=B + M + N + D)
    if labels == "lists":  # the same labels as a mask, for the mask mode's outputs and the reference
        m0, m1 = _assign_lists(B, M, N, seed=B * M + N + D)
        gt = torch.zeros(B, M, N, device=DEV, dtype=torch.bool).scatter_(2, m0.clamp(min=0)[..., None],
                                                                       (m0 >= 0)[..., None])
    gt_u8 = gt.view(torch.uint8)
    f = ops.assign_fused_stats(md0, md1, alpha, ls0, ls1, gt_u8=gt_u8)
    rowcnt, colcnt = gt_u8.sum(2, dtype=torch.float32), gt_u8.sum(1, dtype=torch.float32)
    g0 = _guarded((B * M, D), torch.bfloat16, 2 * D)
    g1 = _guarded((B * N, D), torch.bfloat16, 2 * D)
    if labels == "mask":
        gt_t = gt_u8.transpose(1, 2).contiguous()
        ops.assign_fused_bwd(md0, md1, alpha, f["lse_row"], f["lse_col"], gt_u8, gt_t, gc, rowcnt, colcnt, g0[1], g1[1])
    else:
        fl = ops.assign_fused_stats(md0, md1, alpha, ls0, ls1, gt_u8=None)
        assert fl["pos_row_sum"] is None
        for k in ("lse_row", "lse_col", "rowmax", "rowarg", "colmax", "colarg"):
            assert torch.equal(fl[k], f[k]), k  # STATS reads no mask for these
        rowcnt, colcnt, _ = ops.match_list_counts(m0, m1)
        pos = ops.assign_pos_fwd(m0, m1, fl["lse_row"], fl["lse_col"], alpha, md0, md1)
        a, c = md0.double(), md1.double()
        j = m0.clamp(min=0)
        cj = c.gather(1, j[..., None].expand(-1, -1, D))
        lcj = fl["lse_col"].double().gather(1, j)
        lr = fl["lse_row"].double()
        want = torch.where(m0 >= 0, 2 * alpha * (a * cj).sum(-1) - lr - lcj, torch.zeros_like(lr))
        bound = torch.where(m0 >= 0, (2 * D + 8) * U32 * (2 * alpha * (a.abs() * cj.abs()).sum(-1) + lr.abs() + lcj.abs()),
                            torch.zeros_like(lr))
        _within((pos.double() - want).abs(), bound, f"assign lists B={B} M={M} N={N} D={D} pos_fwd")
        del a, c, cj, fl
        ops.assign_fused_bwd(md0, md1, alpha, f["lse_row"], f["lse_col"], None, None, gc, rowcnt, colcnt, g0[1], g1[1])
        ops.assign_pos_bwd(md0, md1, gc, m0, m1, g0[1], g1[1])
    dmd0, dmd1 = g0[1].view(B, M, D), g1[1].view(B, N, D)
    if B == 32:  # the benchmark's launch: a second call is bit-identical
        f2 = ops.assign_fused_stats(md0, md1, alpha, ls0, ls1, gt_u8=gt_u8)
        assert all(torch.equal(f[k], f2[k]) for k in ("lse_row", "lse_col", "rowmax", "rowarg", "colmax", "colarg",
                                                      "pos_row_sum"))
        del f2
    tag = f"assign {labels} B={B} M={M} N={N} D={D}"
    w = _Worst(tag)
    for b in range(B):
        r = assign_ref(md0[b], md1[b], alpha, ls0[b], ls1[b], gt[b], gc[b].item(), lists=labels == "lists")
        for k in ("lse_row", "lse_col", "rowmax", "colmax"):
            w(k, (f[k][b].double() - r[k]).abs(), r["b_" + k])
        w("pos_row_sum", (f["pos_row_sum"][b].double() - r["pos_row_sum"]).abs(), r["b_pos"])
        check_argmax(f["rowarg"][b], r["sc"], r["b_rowmax"], 1, f"{tag} b={b} rowarg")
        check_argmax(f["colarg"][b], r["sc"], r["b_colmax"], 0, f"{tag} b={b} colarg")
        w("dmd0", (dmd0[b].double() - r["dmd0"]).abs(), r["b_dmd0"])
        w("dmd1", (dmd1[b].double() - r["dmd1"]).abs(), r["b_dmd1"])
        if (b == 0) if labels == "lists" else (b % 4 == 1):  # no positives: nothing to differentiate
            assert not dmd0[b].any() and not dmd1[b].any() and not f["pos_row_sum"][b].any()
        del r
    w.report()
    _guards_intact(g0, f"{tag} dmd0")
    _guards_intact(g1, f"{tag} dmd1")


# ================================================================================================
# 4. negative controls: each check rejects a wrong answer built from its own reference (CPU, no library call)
# ================================================================================================
def _cpu_gen(seed):
    return torch.Generator().manual_seed(seed)


def test_gemm_checks_reject_truncation_and_a_missing_k_block():
    g = _cpu_gen(1)
    M, N, K = 65, 72, 256
    a = torch.randn(M, K, generator=g).to(torch.bfloat16).double()
    b = torch.randn(N, K, generator=g).to(torch.bfloat16).double()
    ref = a @ b.t()
    bnd = gemm_bound(a.abs() @ b.abs().t(), K, 1.0, ref, torch.bfloat16)
    check_gemm(ref.float().to(torch.bfloat16), ref, bnd, "control gemm rn", log=False)  # the right answer passes
    with pytest.raises(AssertionError):
        check_gemm(_trunc_bf16(ref), ref, bnd, "control gemm trunc", log=False)
    drop = a.clone()
    drop[:, 192:256] = 0  # the last 64-wide k-block left out
    bnd32 = gemm_bound(a.abs() @ b.abs().t(), K, 1.0, ref, torch.float32)
    with pytest.raises(AssertionError):
        check_gemm((drop @ b.t()).float(), ref, bnd32, "control gemm k-block", log=False)
    # exact form
    r = int(math.isqrt(2 ** 23 // K))
    ai = torch.randint(-r, r + 1, (M, K), generator=g).double()
    bi = torch.randint(-r, r + 1, (N, K), generator=g).double()
    ex = 0.5 * (ai @ bi.t())
    assert check_exact(ex.float().to(torch.bfloat16), ex, "control exact rn", log=False) > 0.5
    with pytest.raises(AssertionError):
        check_exact(_trunc_bf16(ex), ex, "control exact trunc", log=False)
    ai[:, 192:256] = 0
    with pytest.raises(AssertionError):
        check_exact((0.5 * (ai @ bi.t())).float(), ex, "control exact k-block", log=False)


def _cpu_attn(Nq, Nk, regime, seed):
    g = _cpu_gen(seed)
    q = torch.randn(Nq, 1, 64, generator=g) * 1.5
    k = torch.randn(Nk, 1, 64, generator=g)
    v = torch.randn(Nk, 1, 64, generator=g)
    do = torch.randn(Nq, 1, 64, generator=g)
    if regime == "rising":
        q[..., 0] = 8.0
        k[..., 0] = torch.linspace(0.0, 60.0, Nk)[:, None]
    elif regime == "zero_q":
        q.zero_()
        v = 1.25 + 0.1 * v
    return tuple(t.to(torch.bfloat16) for t in (q, k, v, do))


def _online_softmax(q, k, v, stale_tile=None):
    """fp64 flash-attention forward, 64-key tiles, online maximum; at stale_tile the accumulated O is not rescaled to
    the new maximum (l is)."""
    Q, K, V = (t.double()[:, 0] for t in (q, k, v))
    m = torch.full((Q.shape[0], 1), -math.inf, dtype=torch.float64)
    l = torch.zeros_like(m)
    o = torch.zeros(Q.shape[0], 64, dtype=torch.float64)
    for j, s in enumerate(range(0, K.shape[0], 64)):
        S = SCALE * Q @ K[s:s + 64].t()
        m_new = torch.maximum(m, S.amax(1, keepdim=True))
        a = torch.exp(m - m_new)
        p = torch.exp(S - m_new)
        l = l * a + p.sum(1, keepdim=True)
        o = (o if j == stale_tile else o * a) + p @ V[s:s + 64]
        m = m_new
    return (o / l)[:, None, :], (m + torch.log(l)).t()


def test_attention_checks_reject_wrong_answers():
    w = lambda name, e, b: _within(e, b, name, log=False)  # noqa: E731
    # the online-softmax restatement is the reference, and passes
    q, k, v, do = _cpu_attn(70, 150, "rising", 3)
    o_ok, lse_ok = _online_softmax(q, k, v)
    r = attn_ref(q, k, v, SCALE, o_ok.to(torch.bfloat16), do)
    check_attn_fwd(o_ok.to(torch.bfloat16), lse_ok.float(), r, w)
    # the last key tile rescaled with a stale maximum (the maximum grows in every tile of the rising regime)
    o_st, lse_st = _online_softmax(q, k, v, stale_tile=2)
    with pytest.raises(AssertionError):
        check_attn_fwd(o_st.to(torch.bfloat16), lse_st.float(), r, w)
    # one key tile left out (randn logits: every tile carries weight)
    q, k, v, do = _cpu_attn(70, 150, "randn", 6)
    o_ok, _ = _online_softmax(q, k, v)
    r = attn_ref(q, k, v, SCALE, o_ok.to(torch.bfloat16), do)
    keep = torch.cat([torch.arange(0, 64), torch.arange(128, 150)])
    r_drop = attn_ref(q, k[keep], v[keep], SCALE)
    for got_o, got_l in ((r_drop["O"], r["lse"]), (r["O"], r_drop["lse"])):
        with pytest.raises(AssertionError):
            check_attn_fwd(got_o.to(torch.bfloat16), got_l.float(), r, w)
    r_drop = attn_ref(q, k[keep], v[keep], SCALE, o_ok.to(torch.bfloat16), do)
    w("dq", (r["dQ"].to(torch.bfloat16).double() - r["dQ"]).abs(), r["bdQ"])
    with pytest.raises(AssertionError):
        w("dq", (r_drop["dQ"].to(torch.bfloat16).double() - r["dQ"]).abs(), r["bdQ"])
    # q = 0: a truncating store, and padded keys leaking into the row sum, are both seen
    q, k, v, do = _cpu_attn(70, 150, "zero_q", 4)
    r = attn_ref(q, k, v, SCALE)
    check_attn_fwd(r["O"].to(torch.bfloat16), r["lse"].float(), r, w)
    with pytest.raises(AssertionError):
        check_attn_fwd(_trunc_bf16(r["O"]), r["lse"].float(), r, w)
    leak = v.double().sum(0, keepdim=True) / 192  # 150 keys summed, divided by three whole tiles
    with pytest.raises(AssertionError):
        check_attn_fwd(leak.expand_as(r["O"]).to(torch.bfloat16), r["lse"].float(), r, w)


def test_assign_checks_reject_a_swapped_argmax_pair():
    g = _cpu_gen(5)
    M, N, D = 100, 90, 64
    md0 = (torch.randn(M, D, generator=g) * 2).to(torch.bfloat16)
    md1 = (torch.randn(N, D, generator=g) * 2).to(torch.bfloat16)
    ls0 = torch.nn.functional.logsigmoid(torch.randn(M, generator=g))
    ls1 = torch.nn.functional.logsigmoid(torch.randn(N, generator=g))
    gt = torch.zeros(M, N, dtype=torch.bool)
    gt[torch.arange(30), torch.arange(30)] = True
    r = assign_ref(md0, md1, D ** -0.5, ls0, ls1, gt, 0.1)
    arg = r["sc"].argmax(1)
    check_argmax(arg, r["sc"], r["b_rowmax"], 1, "control argmax")
    sure = (r["sc"].topk(2, dim=1).values.diff(dim=1).neg()[:, 0] > 2 * r["b_rowmax"])
    i = int(sure.nonzero()[0])
    j = int(next(jj for jj in sure.nonzero()[:, 0].tolist() if arg[jj] != arg[i]))
    bad = arg.clone()
    bad[i], bad[j] = arg[j], arg[i]
    with pytest.raises(AssertionError):
        check_argmax(bad, r["sc"], r["b_rowmax"], 1, "control argmax swapped")
    # pos_row_sum with one positive of row 0 left out
    s0 = D ** -0.5 * (md0[0].double() @ md1[0].double())
    miss = r["pos_row_sum"].clone()
    miss[0] -= 2 * s0 - r["lse_row"][0] - r["lse_col"][0]
    with pytest.raises(AssertionError):
        _within((miss - r["pos_row_sum"]).abs(), r["b_pos"], "control pos", log=False)
