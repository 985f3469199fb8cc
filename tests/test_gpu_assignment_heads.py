"""GPU: the kernels that turn the last similarity into a prediction, element by element against fp64 at the benchmark's
shape (32 pairs of 2048 x 2048) and at ragged edges:
  * the unfused assignment passes of csrc/assign.cu: lgb200_assign_lse (row LSE + per-strip column partials, then the
    strip merge), lgb200_assign_scores (dense log-assignment, row / column max and argmax, positive-weighted row sums,
    row_norm) and lgb200_assign_bwd (d sim of the positive NLL term, fp32 or bf16), and lgb200_filter_matches;
  * GlueStick's head, lgb200_log_double_softmax[_dev] (csrc/heads.cu), and the closed-form backward
    heads_grad.log_double_softmax_backward;
  * SuperGlue's head, the persistent cooperative Sinkhorn pair lgb200_sinkhorn_fwd / lgb200_sinkhorn_bwd.
Each pass is fed the previous pass's kernel outputs (the scores pass gets the kernel's LSE vectors, the filter gets the
kernel's argmax, the backward the kernel's potentials), so an error cannot hide behind an upstream one.  References are
torch fp64 on the device, a few pairs at a time.

Units:
  U32 = 2^-24   fp32 unit round-off (one rounding of an fp32 add, subtract or multiply is off by at most U32 of its result)
  UBF = 2^-8    bf16 round-to-nearest of an output (8-bit significand)
  SO  = 1 + 2^-12  second-order slack: chains of n <= 4096 roundings compound to at most n U32 (1 + 2^-12)
  __expf(d) is off by at most 2 + floor(1.173 |d|) ulp of its result (CUDA programming guide), i.e. a relative
  2 U32 (2 + 1.173 |d|); expf / logf / log1pf by at most 2 / 1 / 1 ulp.  A sum of n-link sequential fp32 additions of
  terms t is off by at most n U32 sum |t|.

Bounds (x = the fp32 similarity, evaluated in fp64):
  lse_row / lse_col   sum_j p_j eps_j + n U32 + 4 U32 log(sum_j exp(x_j - m)) + 2 U32 |lse|, p = softmax(x), m = max x,
            eps_j = U32 (6 (K + 1) + 5 (m - x_j)): the first __expf of a term and its K later rescales by the moving
            maximum (their arguments add up to m - x_j: the reference a term is taken against is never below it), each
            with the rounding of its argument and of its product.
            rows: K = ceil(N/128) + 5 (one rescale per 128-column chunk, five warp merges), n = ceil(N/128) + 17 (the
            per-lane chain over chunks, the 4-term tree, three roundings per warp merge);
            columns: K = 1 (one rescale per strip partial in the merge), n = ceil(S/8) + 21, S = ceil(M/32) strips
            (4 rows per warp, 8 warps, the strided strip loop of the merge, its 8-group sum, the product).
  scores    bit-equal to fp32 torch ((x - lr) + (x - lc)) + (ls0 + ls1) on the kernel's lr / lc; against fp64 of the same
            inputs U32 (|x - lr| + |x - lc| + |2x - lr - lc| + |ls0 + ls1| + |s|).  Dustbin column = dust0, dustbin
            row = dust1, corner = 0, exactly.
  max / arg rowmax / colmax equal the maximum of the kernel's own scores; rowarg / colarg are the LOWEST maximising index.
            Against fp64: the argmax equals the fp64 argmax wherever the fp64 top-2 margin exceeds twice the largest
            score bound of the row (column).
  pos_row_sum  sum_j gt U32 (|x - lr| + |x - lc| + |t|) + (4 ceil(N/128) + 5) U32 sum_j gt |t|, t = 2x - lr - lc
            (4 columns per lane and chunk, then the 5-level warp sum); exactly 0 for rows without positives.
  row_expsum   sum over the row's scores and dust0 of 2 U32 (2 + 1.173 |s|) e^s + (4 ceil(N/128) + 6) U32 sum e^s.
  d sim     2 c gt - e^(x - lr) c rowcnt - e^(x - lc) c colcnt:
            U32 [E_r (6 + 3.5 |x - lr|) + E_c (6 + 3.5 |x - lc|)] + U32 (2 |c| gt + E_r + E_c + |ref|),
            E_r = e^(x - lr) |c rowcnt| (the __expf, its argument, c * count, the product); bf16: that bound plus
            UBF (|ref| + bound).  Exact case: with zero counts d sim = 2c, whose bf16 store must be round-to-nearest.
  filter    m0 / m1 / matching scores bit-equal to a torch restatement of lightglue.py:293-309 on the same device (both
            sides use CUDA's expf; the library is built without --use_fast_math).
  log_double_softmax  from the kernel's own lse (read back from its workspace), L = logaddexp(lse, bin) is off by
            b_L = U32 (5 e + |lse - bin| e + 2 log1p(e) + |L|), e = exp(-|lse - bin|);
            inner 0.5 (b_Lr + b_Lc) + 0.5 U32 (|x - Lr| + |x - Lc| + |2x - Lr - Lc|), bin column b_Lr + U32 |bin - Lr|,
            bin row b_Lc + U32 |bin - Lc|, corner 0.  Host and device bin give bit-identical output.
  its backward (heads_grad, fp32 torch on the kernel's output) against fp64 autograd of gluestick.py:772-783: the lse
            it reads back (bin - score) is off from the fp64 one by a measured d, so each softmax factor is off by
            expm1(d + U32 |x - lse|) + 5 U32; the row / column gradient sums by (n + 1) U32 sum |terms| (torch's
            reduction order is not fixed: n = the reduced length); the subtractions by U32 of their operands; d bin
            sums B max(M, N) terms, in an order torch does not fix, so its bound allows a chain that long and the d bin
            check rejects only gross errors.
  Sinkhorn  no a-priori bound for an iterated fixed point: a plain fp32 torch evaluation of the same iterations
            (forward) and of the same reverse sweep on the kernel's potentials (backward) measures the fp32 floor
            against fp64, per element class (dense, dustbin row, dustbin column); the kernel must be within 4x that
            floor, plus 16 U32 (1 + |ref|), elementwise.  This runs at 1, 3 and 100 iterations: by 100 the output has
            converged and no longer shows a missing iteration or a wrong start, so the first two carry that.  The
            stored potentials of every iteration (which the backward consumes) are each checked against one fp64
            half-iteration applied to the kernel's previous one, under the LSE bound (see check_history).

Dense outputs (scores, d sim, log_double_softmax and Sinkhorn outputs) are written into buffers with NaN-pattern guard
rows before and after, which must come back unchanged, and every unwritten output starts as NaN (a NaN error fails).  At
the benchmark shape a second call of every kernel must be bit-identical.  The negative controls at the end run on the
CPU without the library: each check rejects a wrong answer built from its own reference (lse_col without the last strip,
a tie broken to the highest index, the dustbin column shifted by one, a truncating bf16 store, >= in the filter, the bin
left out of the column softmax, a Sinkhorn iteration fewer, a reverse sweep whose last step reads v_0 in place of 0, a
Sinkhorn history shifted by one iteration or started from a wrong v).

Budget: about a minute and under 6 GiB peak device memory on one H100, recorded by the module fixture.
"""
import math
import time
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from gluefactory_b200 import _lib, heads_grad, ops
from gluefactory_b200._lib import call, ptr, stream_ptr
from gluefactory_b200.matchers.gluestick import GlueStick
from gluefactory_b200.matchers.lightglue import LightGlue
from tests.util import report

GPU = pytest.mark.gpu
DEV = "cuda"
U32, UBF, SO = 2.0 ** -24, 2.0 ** -8, 1.0 + 2.0 ** -12
BF16_GUARD, F32_GUARD = 0x7FA5, 0x7FA5A5A5  # NaN bit patterns of the guard rows
BENCH = (32, 2048, 2048)  # pairs x keypoints x keypoints of the benchmark's step
SK_ITERS = 100  # SuperGlue's sinkhorn_iterations


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
    report("test_gpu_assignment_heads", seconds=time.time() - t,
           peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)


def _gen(seed, dev=DEV):
    return torch.Generator(device=dev).manual_seed(seed)


def _randn(*shape, g, scale=1.0):
    return torch.randn(*shape, device=g.device, generator=g) * scale


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


def _chunks(B, M, N):
    """Pair slices small enough for a handful of fp64 [pairs, M, N] planes (128 MiB each at the benchmark's shape)."""
    step = max(1, 2 ** 24 // (M * N))
    return [slice(b, min(B, b + step)) for b in range(0, B, step)]


def _same_bits(a, b):
    if a.dtype in (torch.float32, torch.bfloat16):
        it = torch.int32 if a.dtype == torch.float32 else torch.int16
        return torch.equal(a.contiguous().view(it), b.contiguous().view(it))
    return torch.equal(a, b)


def _trunc_bf16(x):
    """x rounded toward zero to bf16 (a truncating store; negative control)."""
    b = x.float().contiguous().view(torch.int32) & -65536
    return b.view(torch.float32).to(torch.bfloat16)


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


# ================================================================================================
# kernel calls (every output starts as NaN; dense outputs between guard rows)
# ================================================================================================
def _nan(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def _assign_lse(sim):
    B, M, N = sim.shape
    lr, lc = _nan(B, M), _nan(B, N)
    ws = torch.empty(_lib.load().lgb200_assign_ws_bytes(B, M, N), device=DEV, dtype=torch.uint8)
    call("lgb200_assign_lse", ptr(sim), ptr(lr), ptr(lc), ptr(ws), B, M, N, stream_ptr())
    return lr, lc


def _assign_scores(c, lr, lc):
    sim = c["sim"]
    B, M, N = sim.shape
    g = _guarded((B, M + 1, N + 1), torch.float32, N + 1)
    st = {"scores": g[1], "rowmax": _nan(B, M), "colmax": _nan(B, N), "pos_row_sum": _nan(B, M),
          "row_expsum": _nan(B, M), "rowarg": torch.full((B, M), -7, device=DEV, dtype=torch.int32),
          "colarg": torch.full((B, N), -7, device=DEV, dtype=torch.int32)}
    ws = torch.empty(_lib.load().lgb200_assign_ws_bytes(B, M, N), device=DEV, dtype=torch.uint8)
    call("lgb200_assign_scores", ptr(sim), ptr(lr), ptr(lc), ptr(c["ls0"]), ptr(c["ls1"]), ptr(c["d0"]), ptr(c["d1"]),
         ptr(c["gt"]), ptr(st["scores"]), ptr(st["rowmax"]), ptr(st["rowarg"]), ptr(st["colmax"]), ptr(st["colarg"]),
         ptr(st["pos_row_sum"]), ptr(st["row_expsum"]), ptr(ws), B, M, N, stream_ptr())
    _guards_intact(g, "assign_scores")
    return st


def _assign_bwd(sim, lr, lc, gt, gc, rowcnt, colcnt, dtype):
    B, M, N = sim.shape
    g = _guarded((B, M, N), dtype, N)
    call("lgb200_assign_bwd", ptr(sim), ptr(lr), ptr(lc), ptr(gt), ptr(gc), ptr(rowcnt), ptr(colcnt), ptr(g[1]),
         _lib.BF16 if dtype == torch.bfloat16 else _lib.F32, B, M, N, stream_ptr())
    _guards_intact(g, "assign_bwd")
    return g[1]


def _lds(sim, beta, on_device):
    """lgb200_log_double_softmax[_dev] -> (scores, the kernel's lse_row, lse_col read back from its workspace)."""
    B, M, N = sim.shape
    g = _guarded((B, M + 1, N + 1), torch.float32, N + 1)
    ws = torch.empty(_lib.load().lgb200_heads_ws_bytes(B, M, N), device=DEV, dtype=torch.uint8)
    if on_device:
        bs = torch.tensor([beta], device=DEV, dtype=torch.float32)
        call("lgb200_log_double_softmax_dev", ptr(sim), ptr(bs), ptr(g[1]), ptr(ws), B, M, N, stream_ptr())
    else:
        call("lgb200_log_double_softmax", ptr(sim), float(beta), ptr(g[1]), ptr(ws), B, M, N, stream_ptr())
    _guards_intact(g, "log_double_softmax")
    lse = ws[:4 * B * (M + N)].view(torch.float32)  # workspace layout: [lse_row B*M][lse_col B*N][...]
    return g[1], lse[:B * M].view(B, M), lse[B * M:].view(B, N)


def _sk_fwd(sim, alpha, iters):
    B, M, N = sim.shape
    g = _guarded((B, M + 1, N + 1), torch.float32, N + 1)
    uh, vh = _nan(iters, B, M + 1), _nan(iters, B, N + 1)
    ws = torch.empty(_lib.load().lgb200_heads_ws_bytes(B, M, N), device=DEV, dtype=torch.uint8)
    call("lgb200_sinkhorn_fwd", ptr(sim), float(alpha), int(iters), ptr(g[1]), ptr(uh), ptr(vh), ptr(ws), B, M, N,
         stream_ptr())
    _guards_intact(g, "sinkhorn_fwd")
    return g[1], uh, vh


def _sk_bwd(sim, alpha, iters, grad, uh, vh):
    B, M, N = sim.shape
    g = _guarded((B, M, N), torch.float32, N)
    dzr, dzc = _nan(B, N + 1), _nan(B, M)
    ws = torch.empty(_lib.load().lgb200_heads_ws_bytes(B, M, N), device=DEV, dtype=torch.uint8)
    call("lgb200_sinkhorn_bwd", ptr(sim), float(alpha), int(iters), ptr(grad), ptr(uh), ptr(vh), ptr(g[1]), ptr(dzr),
         ptr(dzc), ptr(ws), B, M, N, stream_ptr())
    _guards_intact(g, "sinkhorn_bwd")
    return g[1], dzr, dzc


# ================================================================================================
# references and checks (device-agnostic: the negative controls run them on the CPU)
# ================================================================================================
def lse_ref(x, dim, rescales, chain, rounded_terms=False):
    """fp64 logsumexp of the fp32 x along dim and its bound (module docstring).  rounded_terms: the kernel forms each
    term as an fp32 sum (Sinkhorn's Z + v), off by U32 |x_j| before its exponential."""
    x = x.double()
    m = x.amax(dim, keepdim=True)
    e = torch.exp(x - m)
    s = e.sum(dim, keepdim=True)
    ls = torch.log(s)
    lse = m + ls
    eps = U32 * (6 * (rescales + 1) + 5 * (m - x) + (x.abs() if rounded_terms else 0))
    b = SO * ((e * eps).sum(dim, keepdim=True) / s + chain * U32 + 4 * U32 * ls + 2 * U32 * lse.abs())
    return lse.squeeze(dim), b.squeeze(dim)


def check_lse(lr, lc, x, w):
    M, N = x.shape[1:]
    C, S = -(-N // 128), -(-M // 32)
    r, br = lse_ref(x, 2, C + 5, C + 17)
    w("lse_row", (lr.double() - r).abs(), br)
    c, bc = lse_ref(x, 1, 1, -(-S // 8) + 21)
    w("lse_col", (lc.double() - c).abs(), bc)


def scores_exact(x, lr, lc, ls0, ls1):
    """The kernel's association of the log-assignment in fp32 torch (every op one IEEE rounding)."""
    return ((x - lr[:, :, None]) + (x - lc[:, None, :])) + (ls0[:, :, None] + ls1[:, None, :])


def check_scores_exact(sc, x, lr, lc, ls0, ls1, d0, d1):
    M, N = x.shape[1:]
    assert _same_bits(sc[:, :M, :N], scores_exact(x, lr, lc, ls0, ls1)), "scores differ from the fp32 evaluation"
    assert _same_bits(sc[:, :M, N], d0), "dustbin column != dust0"
    assert _same_bits(sc[:, M, :N], d1), "dustbin row != dust1"
    assert (sc[:, M, N] == 0).all(), "corner != 0"


def scores_ref(x, lr, lc, ls0, ls1):
    x = x.double()
    a, c = x - lr.double()[:, :, None], x - lc.double()[:, None, :]
    l01 = ls0.double()[:, :, None] + ls1.double()[:, None, :]
    s = a + c + l01
    return s, SO * U32 * (a.abs() + c.abs() + (a + c).abs() + l01.abs() + s.abs())


def check_lowest_argmax(val, arg, s, dim):
    """val == max of s along dim exactly, arg == the lowest index attaining it (not torch's tie rule)."""
    mx = s.amax(dim)
    idx = torch.arange(s.shape[dim], device=s.device)
    idx = idx[:, None] if dim == 1 else idx
    low = torch.where(s == mx.unsqueeze(dim), idx, s.shape[dim]).amin(dim)
    assert _same_bits(val, mx), "max differs from the maximum of the scores"
    bad = arg.long() != low
    assert not bad.any(), ("argmax is not the lowest maximising index", int(bad.sum()))


def check_margin_argmax(arg, s64, b, dim):
    """arg == fp64 argmax wherever the fp64 top-2 margin exceeds twice the largest bound along dim; returns the share
    of such (decidable) rows."""
    if s64.shape[dim] == 1:
        assert (arg == 0).all()
        return 1.0
    top = s64.topk(2, dim=dim).values
    safe = (top.select(dim, 0) - top.select(dim, 1)) > 2 * b.amax(dim)
    bad = safe & (arg.long() != s64.argmax(dim))
    assert not bad.any(), ("argmax differs from fp64 where the margin decides it", int(bad.sum()))
    return safe.double().mean().item()


def bwd_ref(x, lr, lc, gt, gc, rowcnt, colcnt):
    """fp64 2 c gt - e^(x - lr) c rowcnt - e^(x - lc) c colcnt (SURVEY A.4 / assign.cu) and its fp32 bound."""
    x = x.double()
    dr, dc = x - lr.double()[:, :, None], x - lc.double()[:, None, :]
    cr = (gc.double()[:, None] * rowcnt.double())[:, :, None]
    cc = (gc.double()[:, None] * colcnt.double())[:, None, :]
    er, ec = torch.exp(dr) * cr, torch.exp(dc) * cc
    two = 2 * gc.double()[:, None, None] * gt.double()
    ref = two - er - ec
    er, ec = er.abs(), ec.abs()
    b = SO * U32 * (er * (6 + 3.5 * dr.abs()) + ec * (6 + 3.5 * dc.abs()) + two.abs() + er + ec + ref.abs())
    return ref, b


def check_dsim(d, ref, b, w):
    if d.dtype == torch.bfloat16:
        b = b * (1 + UBF) + UBF * ref.abs()
    w(f"dsim_{str(d.dtype)[6:]}", (d.double() - ref).abs(), b)


def check_exact_bf16(got, want_f32):
    """A bf16 store of exactly representable fp32 values: round to nearest-even, bit for bit."""
    want = want_f32.to(torch.bfloat16)
    bad = ~(got.view(torch.int16) == want.view(torch.int16))
    assert not bad.any(), ("bf16 store is not round-to-nearest", int(bad.sum()))


def filter_ref(rowmax, rowarg, colarg, th, ge=False):
    """lightglue.py:293-309 restated on the pass-2 maxima: mutual nearest neighbours whose exp(score) exceeds th.
    ge: >= in place of > (negative control)."""
    m0, m1 = rowarg.long(), colarg.long()
    i0 = torch.arange(m0.shape[1], device=m0.device)[None]
    i1 = torch.arange(m1.shape[1], device=m1.device)[None]
    mutual0 = i0 == m1.gather(1, m0)
    mutual1 = i1 == m0.gather(1, m1)
    zero = rowmax.new_zeros(())
    ms0 = torch.where(mutual0, rowmax.exp(), zero)
    ms1 = torch.where(mutual1, ms0.gather(1, m1), zero)
    valid0 = mutual0 & ((ms0 >= th) if ge else (ms0 > th))
    valid1 = mutual1 & valid0.gather(1, m1)
    return torch.where(valid0, m0, -1), torch.where(valid1, m1, -1), ms0, ms1


def check_filter(got, want, tag):
    for name, a, b in zip(("m0", "m1", "ms0", "ms1"), got, want):
        assert _same_bits(a, b), (tag, name, int((a != b).sum()))


def _logaddexp_bound(a, beta):
    L = torch.logaddexp(a, torch.full_like(a, beta))
    d = (a - beta).abs()
    e = torch.exp(-d)
    return L, U32 * (5 * e + d * e + 2 * torch.log1p(e) + L.abs())


def lds_ref(x, lr, lc, beta):
    """gluestick.py:772-783 in fp64 from the kernel's lse vectors: (inner, bin column, bin row) and their bounds."""
    x = x.double()
    Lr, br = _logaddexp_bound(lr.double(), beta)
    Lc, bc = _logaddexp_bound(lc.double(), beta)
    a, c = x - Lr[:, :, None], x - Lc[:, None, :]
    inner = (a + c) / 2
    b_in = SO * (0.5 * (br[:, :, None] + bc[:, None, :]) + 0.5 * U32 * (a.abs() + c.abs() + (a + c).abs()))
    col, row = beta - Lr, beta - Lc
    return (inner, b_in), (col, SO * (br + U32 * col.abs())), (row, SO * (bc + U32 * row.abs()))


def check_lds(out, x, lr, lc, beta, w):
    M, N = x.shape[1:]
    (inner, b_in), (col, b_col), (row, b_row) = lds_ref(x, lr, lc, beta)
    w("inner", (out[:, :M, :N].double() - inner).abs(), b_in)
    w("bin_col", (out[:, :M, N].double() - col).abs(), b_col)
    w("bin_row", (out[:, M, :N].double() - row).abs(), b_row)
    assert (out[:, M, N] == 0).all(), "corner != 0"


def lds_restated(sim, beta):
    """gluestick.py:772-783 (log_double_softmax) in the dtype of sim; beta a 0-dim tensor."""
    B, M, N = sim.shape
    s0 = torch.log_softmax(torch.cat([sim, beta.expand(B, M, 1)], 2), 2)
    s1 = torch.log_softmax(torch.cat([sim, beta.expand(B, 1, N)], 1), 1)
    out = sim.new_zeros(B, M + 1, N + 1)
    out[:, :M, :N] = (s0[:, :, :N] + s1[:, :M, :]) / 2
    out[:, :M, N] = s0[:, :, N]
    out[:, M, :N] = s1[:, M, :]
    return out


def _sk_marginals(B, M, N, dtype, dev):
    norm = -math.log(M + N)
    log_mu = torch.full((B, M + 1), norm, dtype=dtype, device=dev)
    log_mu[:, M] = math.log(N) + norm
    log_nu = torch.full((B, N + 1), norm, dtype=dtype, device=dev)
    log_nu[:, N] = math.log(M) + norm
    return norm, log_mu, log_nu


def _sk_coupling(sim, alpha, dtype):
    B, M, N = sim.shape
    Z = torch.empty(B, M + 1, N + 1, dtype=dtype, device=sim.device)
    Z[:, :M, :N] = sim
    Z[:, :M, N] = alpha
    Z[:, M, :] = alpha
    return Z


def sk_potentials(sim, alpha, iters, dtype, v_init=None):
    """superglue.py:186-214 (log_optimal_transport): log-domain Sinkhorn on the bordered coupling Z, marginals
    [1..1, N] / (M+N) and [1..1, M] / (M+N), from v = 0 (v_init: another start; negative control).  Returns Z, norm
    and the potentials of every iteration, uh [iters, B, M+1] and vh [iters, B, N+1]."""
    B, M, N = sim.shape
    Z = _sk_coupling(sim, alpha, dtype)
    norm, log_mu, log_nu = _sk_marginals(B, M, N, dtype, sim.device)
    u, us, vs = torch.zeros_like(log_mu), [], []
    v = torch.zeros_like(log_nu) if v_init is None else v_init.to(dtype)
    for _ in range(iters):
        u = log_mu - torch.logsumexp(Z + v[:, None, :], 2)
        v = log_nu - torch.logsumexp(Z + u[:, :, None], 1)
        us.append(u)
        vs.append(v)
    return Z, norm, torch.stack(us), torch.stack(vs)


def sk_fwd_ref(sim, alpha, iters, dtype):
    """log_optimal_transport's output: Z + u + v shifted by log(M+N)."""
    Z, norm, uh, vh = sk_potentials(sim, alpha, iters, dtype)
    return Z + uh[-1][:, :, None] + vh[-1][:, None, :] - norm


def check_history(uh, vh, sim, alpha, R, S, w):
    """Every stored potential against one fp64 half-iteration applied to the kernel's own previous iterate:
    u_k = log_mu - LSE_j(Z + v_{k-1}) (v_{-1} = 0), v_k = log_nu - LSE_i(Z + u_k).  Bounds: the LSE bound with
    the terms' fp32 sums, K rescales and a 3K-link chain, where
      u (row phase, warp per row): K = ceil(N/128) + 10 (at most two lse4 per 256 columns, one per 128, three lse1,
        five warp merges, the dustbin column); the dustbin row takes one lse1 per 32 columns, K = ceil(N/32) + 6;
      v (strip partials of R rows, merged over S strips): K = ceil(R/4) + ceil(S/128) + 11, the dustbin column
        (one lse1 per row) R + ceil(S/128) + 11;
    plus the fp32 marginal constants and the final subtraction, 3 U32 (|log(M+N)| + log max(M, N)) + U32 |u|."""
    B, M, N = sim.shape
    Z = _sk_coupling(sim, alpha, torch.float64)
    norm, log_mu, log_nu = _sk_marginals(B, M, N, torch.float64, sim.device)
    Kr = torch.full((M + 1, 1), -(-N // 128) + 10.0, dtype=torch.float64, device=sim.device)
    Kr[M] = -(-N // 32) + 6.0
    Kc = torch.full((N + 1,), -(-R // 4) + -(-S // 128) + 11.0, dtype=torch.float64, device=sim.device)
    Kc[N] = R + -(-S // 128) + 11.0
    slack = 3 * U32 * (abs(norm) + math.log(max(M, N)))
    for k in range(uh.shape[0]):
        vp = vh[k - 1].double() if k else torch.zeros(B, N + 1, dtype=torch.float64, device=sim.device)
        lse, b = lse_ref(Z + vp[:, None, :], 2, Kr, 3 * Kr, rounded_terms=True)
        u = log_mu - lse
        w("u_history", (uh[k].double() - u).abs(), SO * (b + slack + U32 * u.abs()))
        lse, b = lse_ref(Z + uh[k].double()[:, :, None], 1, Kc, 3 * Kc, rounded_terms=True)
        v = log_nu - lse
        w("v_history", (vh[k].double() - v).abs(), SO * (b + slack + U32 * v.abs()))


def sk_bwd_ref(sim, alpha, grad, uh, vh, dtype, v_init=None):
    """d(sum grad * out)/dZ of the iterations above by reverse sweep over the given potentials u_k = uh[k],
    v_k = vh[k]: with Q_k = exp(Z + u_k + v_k - log_nu) and P_k = exp(Z + v_{k-1} + u_k - log_mu),
        dZ -= Q_k dv ;  du -= rowsum(Q_k dv) ;  dZ -= P_k du ;  dv = -colsum(P_k du) ;  du = 0     for k = iters .. 1,
    from dZ = grad, du = rowsum(grad), dv = colsum(grad); v_{-1} = 0 (v_init: another value; negative control).
    Returns the bordered dZ."""
    B, M, N = sim.shape
    Z = _sk_coupling(sim, alpha, dtype)
    _, log_mu, log_nu = _sk_marginals(B, M, N, dtype, sim.device)
    dZ = grad.to(dtype).clone()
    du, dv = dZ.sum(2), dZ.sum(1)
    for k in range(uh.shape[0] - 1, -1, -1):
        u_k, v_k = uh[k].to(dtype), vh[k].to(dtype)
        v_p = vh[k - 1].to(dtype) if k else (torch.zeros_like(v_k) if v_init is None else v_init.to(dtype))
        Qd = torch.exp(Z + u_k[:, :, None] + (v_k - log_nu)[:, None, :]) * dv[:, None, :]
        dZ -= Qd
        du = du - Qd.sum(2)
        Pd = torch.exp(Z + v_p[:, None, :] + (u_k - log_mu)[:, :, None]) * du[:, :, None]
        dZ -= Pd
        dv = -Pd.sum(1)
        du = torch.zeros_like(du)
    return dZ


def check_floor(got, ref, ref32, name, w):
    """|got - ref| <= 4 max|ref32 - ref| + 16 U32 (1 + |ref|) elementwise (ref32: the plain fp32 evaluation)."""
    floor = (ref32.double() - ref).abs().max()
    w(name, (got.double() - ref).abs(), 4 * floor + 16 * U32 * (1 + ref.abs()))


def _sk_classes(out, M, N):
    return {"dense": out[:, :M, :N], "dustbin_row": out[:, M, :], "dustbin_col": out[:, :M, N]}


# ================================================================================================
# 1. lgb200_assign_lse
# ================================================================================================
LSE_SHAPES = [BENCH] + [(3, M, N) for M in (1, 33, 2047) for N in (5, 127, 129, 2049, 2050, 2051)]


def _lse_case(B, M, N, regime, seed):
    g = _gen(seed)
    if regime == "constant":  # lse = x + log N on every row
        return _randn(B, M, 1, g=g, scale=4.0).expand(B, M, N).contiguous()
    x = _randn(B, M, N, g=g, scale=4.0)
    if regime == "spike":  # every third row has one entry 60 above everything else of its pair
        i = torch.arange(0, M, 3, device=DEV)
        x[:, i, (5 * i + 1) % N] = x.amax((1, 2))[:, None] + 60.0
    elif regime == "offset":
        x += 1000.0
    return x


@GPU
@pytest.mark.parametrize("regime", ["randn", "spike", "offset", "constant"])
@pytest.mark.parametrize("B,M,N", LSE_SHAPES)
def test_assign_lse_against_fp64(B, M, N, regime):
    x = _lse_case(B, M, N, regime, seed=M + 7 * N + len(regime))
    lr, lc = _assign_lse(x)
    w = _Worst(f"assign_lse B={B} M={M} N={N} {regime}")
    for sl in _chunks(B, M, N):
        check_lse(lr[sl], lc[sl], x[sl], w)
    w.report()


# ================================================================================================
# 2. lgb200_assign_scores
# ================================================================================================
# exact ties at the maximum: copies of a dominant column (row argmax) at these offsets fall inside one lane's 4 columns
# (+1, +3), in the next lane (+4), in the next 128-column chunk (+128, +132); copies of a dominant row (column argmax)
# in the same warp (+8), the next warp (+1), the next strip (+32) and the last strip (+2016)
COL_TWINS = ([1], [4], [128], [3, 4, 128, 132])
ROW_TWINS = ([8], [1], [32], [1, 8, 32, 2016])


def _scores_case(B, M, N, seed, density=0.001):
    """Pairs b % 8 < 4: randn * 4.  Pairs b % 8 >= 4: randn plus a dominant row and column (20 + randn / 2) and exact
    copies of them (with their matchability) at the offsets above, so most rows and columns tie at their maximum.
    gt at the given density, with one row of positives only and one row without any."""
    g = _gen(seed)
    sim = _randn(B, M, N, g=g, scale=4.0)
    z0, z1 = _randn(B, M, g=g, scale=2.0), _randn(B, N, g=g, scale=2.0)
    ties = []
    for b in range(4, B, 1):
        if b % 8 < 4:
            continue
        k = b % 4
        i0, j0 = 2 + k, 4 * (3 + k)
        if i0 >= M or j0 >= N:
            continue
        sim[b] = _randn(M, N, g=g)
        sim[b, i0, :] = 20 + _randn(N, g=g, scale=0.5)
        sim[b, :, j0] = 20 + _randn(M, g=g, scale=0.5)
        rt = [i0 + d for d in ROW_TWINS[k] if i0 + d < M]
        ct = [j0 + d for d in COL_TWINS[k] if j0 + d < N]
        sim[b, rt, :] = sim[b, i0, :].clone()
        sim[b, :, ct] = sim[b, :, j0, None].clone()
        z0[b, rt], z1[b, ct] = z0[b, i0].item(), z1[b, j0].item()
        ties.append((b, rt, ct))
    gt = torch.rand(B, M, N, device=DEV, generator=g) < density
    if M > 6:
        gt[:, 5, :], gt[:, 6, :] = True, False
    return {"sim": sim, "ls0": F.logsigmoid(z0), "ls1": F.logsigmoid(z1), "d0": F.logsigmoid(-z0),
            "d1": F.logsigmoid(-z1), "gt": gt.to(torch.uint8).contiguous(), "ties": ties}


SCORE_SHAPES = [BENCH, (8, 2047, 2051), (8, 33, 129), (8, 1, 5), (8, 2047, 127), (8, 33, 2050)]


@GPU
@pytest.mark.parametrize("B,M,N", SCORE_SHAPES)
def test_assign_scores_against_fp32_and_fp64(B, M, N):
    c = _scores_case(B, M, N, seed=3 * M + N)
    lr, lc = _assign_lse(c["sim"])
    st = _assign_scores(c, lr, lc)
    tag = f"assign_scores B={B} M={M} N={N}"
    w = _Worst(tag)
    C = -(-N // 128)
    decided = []
    for sl in _chunks(B, M, N):
        x, sc = c["sim"][sl], st["scores"][sl]
        ls0, ls1, d0, d1 = (c[k][sl] for k in ("ls0", "ls1", "d0", "d1"))
        inner = sc[:, :M, :N]
        # bit equality with the same IEEE operations, dustbins and corner
        check_scores_exact(sc, x, lr[sl], lc[sl], ls0, ls1, d0, d1)
        # maxima of the kernel's own scores, lowest maximising index
        check_lowest_argmax(st["rowmax"][sl], st["rowarg"][sl], inner, 2)
        check_lowest_argmax(st["colmax"][sl], st["colarg"][sl], inner, 1)
        # against fp64 of the same inputs
        s64, bs = scores_ref(x, lr[sl], lc[sl], ls0, ls1)
        w("scores", (inner.double() - s64).abs(), bs)
        decided.append(check_margin_argmax(st["rowarg"][sl], s64, bs, 2))
        check_margin_argmax(st["colarg"][sl], s64, bs, 1)
        # the TokenConfidence labels: argmax over [scores | dustbin], the dustbin winning only when strictly larger
        z = torch.zeros_like(d0.double())
        fin0 = LightGlue._argmax_with_dustbin(st["rowmax"][sl], st["rowarg"][sl], d0, N)
        check_margin_argmax(fin0, torch.cat([s64, d0.double()[:, :, None]], 2), torch.cat([bs, z[:, :, None]], 2), 2)
        z = torch.zeros_like(d1.double())
        fin1 = LightGlue._argmax_with_dustbin(st["colmax"][sl], st["colarg"][sl], d1, M)
        check_margin_argmax(fin1, torch.cat([s64, d1.double()[:, None, :]], 1), torch.cat([bs, z[:, None, :]], 1), 1)
        del s64, bs
        # positive-weighted row sums on the kernel's lse
        gt = c["gt"][sl].double()
        a, cc = x.double() - lr[sl].double()[:, :, None], x.double() - lc[sl].double()[:, None, :]
        t = a + cc
        ref = (gt * t).sum(2)
        b = SO * U32 * ((gt * (a.abs() + cc.abs() + t.abs())).sum(2) + (4 * C + 5) * (gt * t.abs()).sum(2))
        w("pos_row_sum", (st["pos_row_sum"][sl].double() - ref).abs(), b)
        empty = gt.sum(2) == 0
        assert (st["pos_row_sum"][sl][empty] == 0).all()
        del a, cc, t, gt
        # row_norm: sum of exp over the row's kernel scores and its dustbin
        s = inner.double()
        e, ed = torch.exp(s), torch.exp(d0.double())
        ref = e.sum(2) + ed
        b = SO * (2 * U32 * ((e * (2 + 1.173 * s.abs())).sum(2) + ed * (2 + 1.173 * d0.double().abs()))
                  + (4 * C + 6) * U32 * ref)
        w("row_expsum", (st["row_expsum"][sl].double() - ref).abs(), b)
        del s, e
    # the designed ties sit at the maxima of most rows / columns of their pairs
    for b, rt, ct in c["ties"]:
        inner = st["scores"][b, :M, :N]
        if ct:
            tied = ((inner == inner.amax(1, keepdim=True)).sum(1) >= 2).sum().item()
            assert tied >= M // 2, (b, "row ties", tied)
            assert (st["rowarg"][b] <= 4 * (3 + b % 4)).float().mean() > 0.5
        if rt:
            tied = ((inner == inner.amax(0, keepdim=True)).sum(0) >= 2).sum().item()
            assert tied >= N // 2, (b, "column ties", tied)
    w.report()
    report(tag, rows_decided_by_margin=sum(decided) / len(decided), tie_pairs=len(c["ties"]))


# ================================================================================================
# 3. lgb200_assign_bwd
# ================================================================================================
BWD_SHAPES = [BENCH, (4, 33, 2051), (4, 2047, 127), (3, 1, 5), (4, 129, 2050)]


@GPU
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("B,M,N", BWD_SHAPES)
def test_assign_bwd_against_fp64(B, M, N, dtype):
    g = _gen(11 * M + N)
    sim = _randn(B, M, N, g=g, scale=4.0)
    gt = (torch.rand(B, M, N, device=DEV, generator=g) < (0.001 if M * N > 2 ** 20 else 0.01)).to(torch.uint8)
    rowcnt, colcnt = gt.sum(2).float(), gt.sum(1).float()
    rowcnt[:, ::5] = 0.0  # zero counts: the skipped terms
    colcnt[:, 1::7] = 0.0
    rowcnt[:, 3::11] += 2.0
    gc = _randn(B, g=g)
    gc[0] = 0.0  # a pair without weight
    lr, lc = _assign_lse(sim)
    d = _assign_bwd(sim, lr, lc, gt, gc, rowcnt, colcnt, dtype)
    w = _Worst(f"assign_bwd B={B} M={M} N={N}")
    for sl in _chunks(B, M, N):
        ref, b = bwd_ref(sim[sl], lr[sl], lc[sl], gt[sl], gc[sl], rowcnt[sl], colcnt[sl])
        check_dsim(d[sl], ref, b, w)
        del ref, b
    assert not d[0].float().any(), "c = 0 must give d sim = 0"
    w.report()


def _bf16_exact_case(M, N, dev):
    """Zero counts, so d sim = 2c on the positives and 0 elsewhere; 2c = 2^e (1 + k 2^-9) lands 1/4, 3/4, 1/2 (a tie,
    to even) or 0 of a bf16 ulp past the grid, of either sign."""
    ks = [3, 1, 6, 7, 11, 4, 3, 5]
    es = [0, -3, 5, 1, -6, 2, 9, -1]
    sg = [1, -1, 1, -1, 1, -1, -1, 1]
    gc = torch.tensor([s * 2.0 ** e * (1 + k * 2.0 ** -9) for s, e, k in zip(sg, es, ks)], device=dev)
    gt = torch.rand(len(ks), M, N, generator=torch.Generator(device=dev).manual_seed(5), device=dev) < 0.3
    want = torch.where(gt, 2 * gc[:, None, None], torch.zeros((), device=dev))
    return gc, gt.to(torch.uint8), want


@GPU
@pytest.mark.parametrize("N", [128, 131])  # the vector (pack_bf16) and the scalar store
def test_assign_bwd_bf16_store_rounds_to_nearest(N):
    M = 67
    gc, gt, want = _bf16_exact_case(M, N, DEV)
    B = gc.shape[0]
    sim = _randn(B, M, N, g=_gen(6), scale=4.0)
    lr, lc = _assign_lse(sim)
    zero_r, zero_c = torch.zeros(B, M, device=DEV), torch.zeros(B, N, device=DEV)
    d32 = _assign_bwd(sim, lr, lc, gt, gc, zero_r, zero_c, torch.float32)
    assert _same_bits(d32, want)
    assert (_trunc_bf16(want) != want.to(torch.bfloat16)).any()  # the case tells the two roundings apart
    check_exact_bf16(_assign_bwd(sim, lr, lc, gt, gc, zero_r, zero_c, torch.bfloat16), want)


# ================================================================================================
# 4. lgb200_filter_matches (and GlueStick's _matches)
# ================================================================================================
def _thresholds(ms0):
    """0, exactly exp(rowmax) of chosen mutual rows (the test is strict), and above every score."""
    pos = ms0[ms0 > 0].sort().values
    picks = [float(pos[0]), float(pos[len(pos) // 2]), float(pos[-1])] if len(pos) else []
    return [0.0] + picks + [float(ms0.max()) + 1.0]


@GPU
def test_filter_matches_against_torch_restatement():
    B, M, N = BENCH
    c = _scores_case(B, M, N, seed=21)
    lr, lc = _assign_lse(c["sim"])
    st = _assign_scores(c, lr, lc)
    rowmax, rowarg, colarg = st["rowmax"], st["rowarg"], st["colarg"]
    base = filter_ref(rowmax, rowarg, colarg, 0.0)
    chains = (~(colarg.long().gather(1, rowarg.long()) == torch.arange(M, device=DEV))).sum().item()
    assert chains > 0  # non-mutual rows
    for th in _thresholds(base[2]):
        want = filter_ref(rowmax, rowarg, colarg, th)
        check_filter(ops.filter_matches(rowmax, rowarg, colarg, th), want, f"filter th={th}")
        if th > 0 and (base[2] == th).any():
            assert ((base[2] == th) & (want[0] >= 0)).sum() == 0  # rows at the threshold are rejected
        # GlueStick's path: torch's max over the same scores, int32 indices
        gs = GlueStick._matches(SimpleNamespace(conf=SimpleNamespace(filter_threshold=th)), st["scores"])
        inner = st["scores"][:, :-1, :-1]
        mx0, mx1 = inner.max(2), inner.max(1)
        check_filter(gs, filter_ref(mx0.values, mx0.indices, mx1.indices, th), f"gluestick th={th}")
    # synthetic chains i -> i -> i + 1 -> i + 1 -> ..., every third row mutual
    g = _gen(22)
    Ms, Ns = 300, 257
    ra = (torch.arange(Ms, device=DEV) % Ns).to(torch.int32).repeat(2, 1).contiguous()
    j = torch.arange(Ns, device=DEV)
    ca = torch.where(j % 3 == 0, j, (j + 1) % Ms).to(torch.int32).repeat(2, 1).contiguous()
    rm = _randn(2, Ms, g=g) - 1.0
    for th in _thresholds(filter_ref(rm, ra, ca, 0.0)[2]):
        check_filter(ops.filter_matches(rm, ra, ca, th), filter_ref(rm, ra, ca, th), f"filter chains th={th}")
    report("filter_matches", non_mutual_rows=chains)


# ================================================================================================
# 5. lgb200_log_double_softmax[_dev] and its backward
# ================================================================================================
def _line_scores(B, L, nj, g):
    """GlueStick's line scores (gluestick.py:327-329): a junction similarity gathered per line endpoint, best of the two
    endpoint orderings.  Few junctions, so many lines share both endpoints: exact duplicates."""
    sj = _randn(B, nj, nj, g=g, scale=3.0)
    idx0 = torch.randint(0, nj, (B, 2 * L), device=DEV, generator=g)
    idx1 = torch.randint(0, nj, (B, 2 * L), device=DEV, generator=g)
    s = torch.gather(sj, 2, idx1[:, None, :].expand(B, nj, 2 * L))
    s = torch.gather(s, 1, idx0[:, :, None].expand(B, 2 * L, 2 * L)).reshape(B, L, 2, L, 2)
    return (0.5 * torch.maximum(s[:, :, 0, :, 0] + s[:, :, 1, :, 1], s[:, :, 0, :, 1] + s[:, :, 1, :, 0])).contiguous()


def _lds_sim(kind, seed):
    g = _gen(seed)
    if kind == "points":  # scripts/prof_gluestick.py: 8 pairs x 2048 points
        return _randn(8, 2048, 2048, g=g, scale=4.0)
    if kind == "lines":  # ... and 512 lines
        return _line_scores(8, 512, 24, g)
    M, N = {"ragged_a": (33, 129), "ragged_b": (1, 5), "ragged_c": (2047, 2051)}[kind]
    return _randn(3, M, N, g=g, scale=4.0)


BINS = [0.7, -30.0, 30.0]


@GPU
@pytest.mark.parametrize("beta", BINS)
@pytest.mark.parametrize("kind", ["points", "lines", "ragged_a", "ragged_b", "ragged_c"])
def test_log_double_softmax_against_fp64(kind, beta):
    sim = _lds_sim(kind, seed=len(kind))
    B, M, N = sim.shape
    if kind == "lines":
        assert torch.unique(sim[0]).numel() < sim[0].numel()  # exact duplicates
    beta = float(torch.tensor(beta, dtype=torch.float32))  # the kernel's fp32 bin
    out, lr, lc = _lds(sim, beta, on_device=False)
    out_dev, lr_dev, lc_dev = _lds(sim, beta, on_device=True)
    assert _same_bits(out, out_dev), "host and device bin paths differ"
    w = _Worst(f"log_double_softmax {kind} B={B} M={M} N={N} bin={beta}")
    for sl in _chunks(B, M, N):
        check_lse(lr[sl], lc[sl], sim[sl], w)
        check_lds(out[sl], sim[sl], lr[sl], lc[sl], beta, w)
    w.report()


@GPU
@pytest.mark.parametrize("beta", BINS)
@pytest.mark.parametrize("kind", ["lines", "ragged_a", "ragged_b", "ragged_c"])
def test_log_double_softmax_backward_against_fp64_autograd(kind, beta):
    sim = _lds_sim(kind, seed=100 + len(kind))
    B, M, N = sim.shape
    bt = torch.tensor(beta, device=DEV, dtype=torch.float32)
    grad = _randn(B, M + 1, N + 1, g=_gen(101))
    out, _, _ = _lds(sim, float(bt), on_device=True)
    dsim, dbin = heads_grad.log_double_softmax_backward(sim, bt, out, grad)
    s64, b64 = sim.double().requires_grad_(True), bt.double().requires_grad_(True)
    (lds_restated(s64, b64) * grad.double()).sum().backward()
    with torch.no_grad():
        x, bd = sim.double(), float(bt)
        Lr = torch.logaddexp(torch.logsumexp(x, 2), torch.tensor(bd, device=DEV, dtype=torch.float64))
        Lc = torch.logaddexp(torch.logsumexp(x, 1), torch.tensor(bd, device=DEV, dtype=torch.float64))
        used_r, used_c = (bt - out[:, :M, N]).double(), (bt - out[:, M, :N]).double()  # what the backward reads back
        gi = grad[:, :M, :N].double() * 0.5
        R0, C1 = gi.sum(2) + grad[:, :M, N].double(), gi.sum(1) + grad[:, M, :N].double()
        eR0 = (N + 1) * U32 * (gi.abs().sum(2) + grad[:, :M, N].double().abs())
        eC1 = (M + 1) * U32 * (gi.abs().sum(1) + grad[:, M, :N].double().abs())
        Pr, Pc = torch.exp(x - Lr[:, :, None]), torch.exp(x - Lc[:, None, :])
        epsR = torch.expm1((used_r - Lr).abs()[:, :, None] + U32 * (x - used_r[:, :, None]).abs()) + 5 * U32
        epsC = torch.expm1((used_c - Lc).abs()[:, None, :] + U32 * (x - used_c[:, None, :]).abs()) + 5 * U32
        tR, tC = Pr * R0.abs()[:, :, None], Pc * C1.abs()[:, None, :]
        ref = s64.grad
        b = SO * (tR * epsR + Pr * eR0[:, :, None] * (1 + epsR) + tC * epsC + Pc * eC1[:, None, :] * (1 + epsC)
                  + U32 * (2 * gi.abs() + tR + tC + ref.abs()))
        tag = f"lds_backward {kind} B={B} M={M} N={N} bin={beta}"
        _within((dsim.double() - ref).abs(), b, f"{tag} dsim")
        # d bin = sum_i (g_iN - e^(s_iN) r0_i) + sum_j (g_Mj - e^(s_Mj) c1_j), s the stored bin entries
        EN, EM = torch.exp(bd - Lr), torch.exp(bd - Lc)
        eN = torch.expm1((out[:, :M, N].double() - (bd - Lr)).abs()) + 5 * U32
        eM = torch.expm1((out[:, M, :N].double() - (bd - Lc)).abs()) + 5 * U32
        termN = grad[:, :M, N].double() - EN * R0
        termM = grad[:, M, :N].double() - EM * C1
        # torch does not fix the order of its two .sum() reductions, so the chain bound has to allow a sequential
        # chain of all B max(M, N) terms (at most 6153 here).  This check therefore rejects only gross errors
        # (~B max(M, N) U32 of sum |terms|, i.e. a wrong formula or a term of typical size left out at the largest
        # shape sits near the bound); the elementwise d sim check above carries the precision of this backward.
        bN = EN * (R0.abs() * eN + eR0 * (1 + eN)) + U32 * termN.abs()
        bM = EM * (C1.abs() * eM + eC1 * (1 + eM)) + U32 * termM.abs()
        bbin = SO * (bN.sum() + bM.sum() + (B * max(M, N) + 1) * U32 * (termN.abs().sum() + termM.abs().sum())
                     + U32 * b64.grad.abs())
        _within((dbin.double() - b64.grad).abs(), bbin, f"{tag} dbin")


# ================================================================================================
# 6. Sinkhorn (lgb200_sinkhorn_fwd / _bwd)
# ================================================================================================
def _sk_geometry(B, M, N, nsm):
    """sk_plan of csrc/heads.cu: S strips of R rows per pair, grid, whether the strips live in shared memory."""
    S = 1 if B >= nsm else nsm // B
    S = min(S, M)
    R = -(-M // S)
    S = -(-M // R)
    vec_b = 3 * ((N + 1 + 3) & ~3) + 2 * ((R + 1 + 3) & ~3)
    cached = B * S <= nsm and (vec_b + R * N) * 4 <= 200 * 1024
    return S, R, min(B * S, nsm), cached


SK_PLANS = ["pairs_over_sms", "m_below_strips", "m_below_strips_b2", "partial_last_strip", "partial_last_strip_b2"]


def _sk_shape(plan, nsm):
    return {"pairs_over_sms": (nsm + 8, 70, 61), "m_below_strips": (1, 50, 203), "m_below_strips_b2": (2, 20, 300),
            "partial_last_strip": (1, 997, 1001), "partial_last_strip_b2": (2, 301, 129)}[plan]


@GPU
@pytest.mark.parametrize("iters", [1, 3, SK_ITERS])  # 1 and 3: every iteration, the first one's v = 0 and the
@pytest.mark.parametrize("plan", SK_PLANS)          # reverse sweep's last step (v_{-1} = 0) change the result
def test_sinkhorn_against_fp64_and_the_fp32_floor(plan, iters):
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    B, M, N = _sk_shape(plan, nsm)
    S, R, grid, cached = _sk_geometry(B, M, N, nsm)
    if plan == "pairs_over_sms":
        assert B * S > grid and not cached  # items wrap round the grid, rows read from global memory
    elif plan.startswith("m_below_strips"):
        assert M < nsm // B and R == 1
    else:
        assert M % R != 0 and N % 4 != 0  # the dustbin row joins a partial last strip; ragged columns
    g = _gen(31 + M)
    sim = _randn(B, M, N, g=g, scale=3.0)
    alpha = float(torch.tensor(0.9, dtype=torch.float32))
    grad = _randn(B, M + 1, N + 1, g=g)
    out, uh, vh = _sk_fwd(sim, alpha, iters)
    dsim, dzr, dzc = _sk_bwd(sim, alpha, iters, grad, uh, vh)
    w = _Worst(f"sinkhorn {plan} iters={iters} B={B} M={M} N={N} S={S} R={R} grid={grid} cached={int(cached)}")
    ref = sk_fwd_ref(sim, alpha, iters, torch.float64)
    ref32 = sk_fwd_ref(sim, alpha, iters, torch.float32)
    got, r64, r32 = _sk_classes(out, M, N), _sk_classes(ref, M, N), _sk_classes(ref32, M, N)
    for k in got:
        check_floor(got[k], r64[k], r32[k], f"fwd_{k}", w)
    # the stored potentials (what the backward consumes), each against one fp64 step from the kernel's previous one
    check_history(uh, vh, sim, alpha, R, S, w)
    # the backward on the kernel's own potentials
    dZ = sk_bwd_ref(sim, alpha, grad, uh, vh, torch.float64)
    dZ32 = sk_bwd_ref(sim, alpha, grad, uh, vh, torch.float32)
    check_floor(dsim, dZ[:, :M, :N], dZ32[:, :M, :N], "bwd_dense", w)
    check_floor(dzr, dZ[:, M, :], dZ32[:, M, :], "bwd_dustbin_row", w)
    check_floor(dzc, dZ[:, :M, N], dZ32[:, :M, N], "bwd_dustbin_col", w)
    w.report()


# ================================================================================================
# 7. determinism at the benchmark shape (every dense output also between guard rows)
# ================================================================================================
@GPU
def test_second_call_is_bit_identical_at_the_benchmark_shape():
    B, M, N = BENCH
    c = _scores_case(B, M, N, seed=77)
    sim = c["sim"]
    lr, lc = _assign_lse(sim)
    lr2, lc2 = _assign_lse(sim)
    assert _same_bits(lr, lr2) and _same_bits(lc, lc2), "assign_lse"
    st = _assign_scores(c, lr, lc)
    st2 = _assign_scores(c, lr, lc)
    for k in st:
        assert _same_bits(st[k], st2[k]), ("assign_scores", k)
    del st2
    f1 = ops.filter_matches(st["rowmax"], st["rowarg"], st["colarg"], 0.05)
    f2 = ops.filter_matches(st["rowmax"], st["rowarg"], st["colarg"], 0.05)
    check_filter(f1, f2, "filter_matches repeat")
    del st
    gc = _randn(B, g=_gen(78))
    rc, cc = c["gt"].sum(2).float(), c["gt"].sum(1).float()
    for dt in (torch.float32, torch.bfloat16):
        d1 = _assign_bwd(sim, lr, lc, c["gt"], gc, rc, cc, dt)
        d2 = _assign_bwd(sim, lr, lc, c["gt"], gc, rc, cc, dt)
        assert _same_bits(d1, d2), ("assign_bwd", dt)
        del d1, d2
    o1 = _lds(sim, 0.7, on_device=False)[0]
    for dev in (False, True):
        assert _same_bits(o1, _lds(sim, 0.7, on_device=dev)[0]), ("log_double_softmax", dev)
    del o1
    alpha, grad = 0.9, _randn(B, M + 1, N + 1, g=_gen(79))
    out, uh, vh = _sk_fwd(sim, alpha, SK_ITERS)
    out2, uh2, vh2 = _sk_fwd(sim, alpha, SK_ITERS)
    assert _same_bits(out, out2) and _same_bits(uh, uh2) and _same_bits(vh, vh2), "sinkhorn_fwd"
    del out, out2, uh2, vh2
    r1 = _sk_bwd(sim, alpha, SK_ITERS, grad, uh, vh)
    r2 = _sk_bwd(sim, alpha, SK_ITERS, grad, uh, vh)
    assert all(_same_bits(a, b) for a, b in zip(r1, r2)), "sinkhorn_bwd"


# ================================================================================================
# 8. negative controls: each check rejects a wrong answer built from its own reference (CPU, no library call)
# ================================================================================================
def _cpu_gen(seed):
    return torch.Generator().manual_seed(seed)


def _reject(fn, *args):
    with pytest.raises(AssertionError):
        fn(*args)


def test_lse_check_rejects_a_column_lse_without_the_last_strip():
    x = torch.randn(2, 100, 37, generator=_cpu_gen(1)) * 4
    w = lambda name, e, b: _within(e, b, name, log=False)  # noqa: E731
    lr, lc = torch.logsumexp(x, 2), torch.logsumexp(x, 1)  # fp32 torch: the right answer passes
    check_lse(lr, lc, x, w)
    x[0, 3, 5] = 1000.0 + x[0, 3, 5]
    check_lse(torch.logsumexp(x, 2), torch.logsumexp(x, 1), x, w)
    _reject(check_lse, torch.logsumexp(x, 2), torch.logsumexp(x[:, :96], 1), x, w)  # rows 96..99: strip 3 of 4


def _cpu_scores_case(seed, B=2, M=70, N=133):
    g = _cpu_gen(seed)
    x = torch.randn(B, M, N, generator=g) * 4
    x[:, :, 9] = x[:, :, 5]  # an exact tie of columns 5 and 9 on every row
    z0, z1 = torch.randn(B, M, generator=g) * 2, torch.randn(B, N, generator=g) * 2
    z1[:, 9] = z1[:, 5]
    x[:, :, 5] += 30.0
    x[:, :, 9] += 30.0
    lr, lc = torch.logsumexp(x, 2), torch.logsumexp(x, 1)
    lc[:, 9] = lc[:, 5]  # (the CPU reduction need not treat the two columns alike)
    return x, lr, lc, F.logsigmoid(z0), F.logsigmoid(z1), F.logsigmoid(-z0), F.logsigmoid(-z1)


def test_argmax_check_rejects_a_tie_broken_to_the_highest_index():
    x, lr, lc, ls0, ls1, _, _ = _cpu_scores_case(2)
    s = scores_exact(x, lr, lc, ls0, ls1)
    mx = s.amax(2)
    assert ((s == mx[..., None]).sum(2) >= 2).float().mean() > 0.5  # most rows tied at their maximum
    low = torch.where(s == mx[..., None], torch.arange(s.shape[2]), -1)
    check_lowest_argmax(mx, low.masked_fill(low < 0, 10 ** 6).amin(2), s, 2)
    _reject(check_lowest_argmax, mx, low.amax(2), s, 2)


def test_scores_check_rejects_a_shifted_dustbin_column():
    x, lr, lc, ls0, ls1, d0, d1 = _cpu_scores_case(3)
    B, M, N = x.shape
    sc = torch.zeros(B, M + 1, N + 1)
    sc[:, :M, :N] = scores_exact(x, lr, lc, ls0, ls1)
    sc[:, :M, N], sc[:, M, :N] = d0, d1
    check_scores_exact(sc, x, lr, lc, ls0, ls1, d0, d1)
    bad = sc.clone()
    bad[:, :M, N] = d0.roll(1, 1)
    _reject(check_scores_exact, bad, x, lr, lc, ls0, ls1, d0, d1)
    # another association (the log-sigmoids added one at a time) is caught by the bit-exact check only: it is as close
    # to fp64 as the kernel's, so the fp64 bound accepts it
    other = (((x - lr[:, :, None]) + (x - lc[:, None, :])) + ls0[:, :, None]) + ls1[:, None, :]
    assert not _same_bits(other, sc[:, :M, :N])
    bad = sc.clone()
    bad[:, :M, :N] = other
    _reject(check_scores_exact, bad, x, lr, lc, ls0, ls1, d0, d1)
    s64, b = scores_ref(x, lr, lc, ls0, ls1)
    w = lambda name, e, bb: _within(e, bb, name, log=False)  # noqa: E731
    w("scores", (sc[:, :M, :N].double() - s64).abs(), b)
    # the fp64 comparison rejects a wrong value: ls1 left out of the scores
    wrong = (x - lr[:, :, None]) + (x - lc[:, None, :]) + ls0[:, :, None]
    _reject(w, "scores", (wrong.double() - s64).abs(), b)


def test_bwd_checks_reject_a_truncating_bf16_store():
    _, _, want = _bf16_exact_case(67, 131, "cpu")
    check_exact_bf16(want.to(torch.bfloat16), want)
    _reject(check_exact_bf16, _trunc_bf16(want), want)
    # the bounded form too, at a size where d sim spans many binades
    g = _cpu_gen(4)
    x = torch.randn(2, 40, 53, generator=g) * 4
    gt = (torch.rand(2, 40, 53, generator=g) < 0.1).to(torch.uint8)
    gc = torch.tensor([1.3, -0.7])
    ref, b = bwd_ref(x, torch.logsumexp(x, 2), torch.logsumexp(x, 1), gt, gc, gt.sum(2).float(), gt.sum(1).float())
    w = lambda name, e, bb: _within(e, bb, name, log=False)  # noqa: E731
    check_dsim(ref.float(), ref, b, w)
    check_dsim(ref.to(torch.bfloat16), ref, b, w)
    _reject(check_dsim, _trunc_bf16(ref), ref, b, w)


def test_filter_check_rejects_ge_in_place_of_gt():
    g = _cpu_gen(5)
    B, M, N = 2, 90, 70
    s = torch.randn(B, M, N, generator=g) * 3 - 2
    rowmax, ra = s.max(2)
    ca = s.max(1).indices
    ra, ca = ra.int(), ca.int()
    base = filter_ref(rowmax, ra, ca, 0.0)
    th = float(base[2][base[2] > 0].median())
    want = filter_ref(rowmax, ra, ca, th)
    check_filter(want, filter_ref(rowmax, ra, ca, th), "control filter")
    _reject(check_filter, filter_ref(rowmax, ra, ca, th, ge=True), want, "control filter ge")


def test_lds_check_rejects_the_bin_missing_from_the_column_softmax():
    g = _cpu_gen(6)
    x = torch.randn(2, 45, 38, generator=g) * 4
    beta = float(torch.tensor(0.7))
    w = lambda name, e, b: _within(e, b, name, log=False)  # noqa: E731
    lr, lc = torch.logsumexp(x, 2), torch.logsumexp(x, 1)
    right = lds_restated(x.double(), torch.tensor(beta, dtype=torch.float64))
    check_lds(right.float(), x, lr, lc, beta, w)
    Lr = torch.logaddexp(lr.double(), torch.tensor(beta, dtype=torch.float64))
    wrong = right.clone()
    wrong[:, :45, :38] = ((x.double() - Lr[:, :, None]) + (x.double() - lc.double()[:, None, :])) / 2
    wrong[:, 45, :38] = beta - lc.double()
    _reject(check_lds, wrong.float(), x, lr, lc, beta, w)


def _cpu_sk_case():
    """The partial_last_strip_b2 plan of the GPU test (2 x 301 x 129 on 132 SMs: 61 strips of 5 rows)."""
    g = _cpu_gen(7)
    x = torch.randn(2, 301, 129, generator=g) * 3
    S, R, _, _ = _sk_geometry(2, 301, 129, 132)
    return x, torch.randn(2, 302, 130, generator=g), S, R


def test_sinkhorn_checks_reject_a_missing_iteration_and_a_wrong_start():
    x, grad, S, R = _cpu_sk_case()
    w = lambda name, e, b: _within(e, b, name, log=False)  # noqa: E731
    # one iteration fewer, at an iteration count the GPU test runs
    it = 3
    ref, ref32 = sk_fwd_ref(x, 0.9, it, torch.float64), sk_fwd_ref(x, 0.9, it, torch.float32)
    check_floor(ref32, ref, ref32, "control sinkhorn", w)
    _reject(check_floor, sk_fwd_ref(x, 0.9, it - 1, torch.float32), ref, ref32, "control sinkhorn", w)
    # the reverse sweep's last step taking v_0 in place of v_{-1} = 0
    _, _, uh, vh = sk_potentials(x, 0.9, it, torch.float32)
    dZ, dZ32 = sk_bwd_ref(x, 0.9, grad, uh, vh, torch.float64), sk_bwd_ref(x, 0.9, grad, uh, vh, torch.float32)
    check_floor(dZ32, dZ, dZ32, "control sinkhorn bwd", w)
    _reject(check_floor, sk_bwd_ref(x, 0.9, grad, uh, vh, torch.float32, v_init=vh[0]), dZ, dZ32, "control", w)
    # at 100 iterations the output has converged, but the stored history has not: the fp32 history passes, and one
    # shifted by an iteration, or one started from a wrong v, is rejected
    _, _, uh, vh = sk_potentials(x, 0.9, SK_ITERS, torch.float32)
    check_history(uh, vh, x, 0.9, R, S, w)
    _reject(check_history, torch.cat([uh[1:], uh[-1:]]), torch.cat([vh[1:], vh[-1:]]), x, 0.9, R, S, w)
    _, _, uh, vh = sk_potentials(x, 0.9, SK_ITERS, torch.float32, v_init=torch.full((2, 130), 0.5))
    _reject(check_history, uh, vh, x, 0.9, R, S, w)


def test_sinkhorn_reverse_sweep_matches_autograd():
    """The reverse-sweep reference (sk_bwd_ref) against fp64 autograd through the restated iterations."""
    g = _cpu_gen(8)
    B, M, N, it = 2, 7, 9, 6
    x = (torch.randn(B, M, N, generator=g, dtype=torch.float64) * 3).requires_grad_(True)
    grad = torch.randn(B, M + 1, N + 1, generator=g, dtype=torch.float64)
    (sk_fwd_ref(x, 0.9, it, torch.float64) * grad).sum().backward()
    with torch.no_grad():
        _, _, uh, vh = sk_potentials(x, 0.9, it, torch.float64)
        dZ = sk_bwd_ref(x, 0.9, grad, uh, vh, torch.float64)
    torch.testing.assert_close(dZ[:, :M, :N], x.grad, rtol=1e-10, atol=1e-12)
