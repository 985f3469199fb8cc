"""GPU: the CUDA-core kernels that run between the GEMMs of every layer step, and the loss terms of every supervised
layer, against plain fp64 evaluations of the same operations on the same (bf16-rounded where the kernel reads bf16)
inputs.  Shapes reach the benchmark's token count (32 pairs of 2048 + 2048 keypoints = 131072 tokens), so grid-stride
loops go round many times and multi-CTA reductions combine hundreds of partials; edges are ragged tails, degenerate
pairs, ties, overflowing logits and arrival counters shared between calls.

Every bound below names the error it allows for:
  U32  = 2^-24   fp32 unit round-off; a sum whose longest chain of sequential fp32 additions has n links is off by at
                 most n * U32 * sum(|terms|), so reductions are checked per column against that, not against the result
  UBF  = 2^-8    bf16 output rounding (8-bit significand; round to nearest is off by less than 2^-8 relative)
  ERF  = 1.5e-7  |error| of the Abramowitz-Stegun 7.1.26 erf approximation inside the GELU
"""
import ctypes
import math
import time

import pytest
import torch
import torch.nn.functional as F

from gluefactory_b200 import _lib, ops
from gluefactory_b200._lib import Lgb200Error, call, ptr, stream_ptr
from tests.util import rel_err, report

pytestmark = pytest.mark.gpu
DEV = "cuda"
U32, UBF, ERF = 2.0 ** -24, 2.0 ** -8, 1.5e-7
TOK = 131072  # tokens of the benchmark's step: 32 pairs x (2048 + 2048)


@pytest.fixture(scope="module", autouse=True)
def _file_budget():
    """Wall time and peak device memory of this file (the machines running it are shared)."""
    torch.cuda.reset_peak_memory_stats()
    t = time.time()
    yield
    torch.cuda.synchronize()
    report("test_gpu_step_kernels", seconds=time.time() - t, peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(*shape, g, scale=1.0):
    return torch.randn(*shape, device=DEV, generator=g) * scale


def _rnd(dtype):
    """Rounding of one output element, relative."""
    return UBF if dtype == torch.bfloat16 else U32


def _within(err, bound, tag, **kw):
    """err <= bound elementwise (a NaN error fails: an output left unwritten shows as NaN); records the largest
    err / bound."""
    err, bound = err.double(), bound.double()
    ratio = (err / bound.clamp(min=1e-300)).max().item() if err.numel() else 0.0
    report(tag, max_err_over_bound=ratio, **kw)
    bad = ~(err <= bound)
    assert not bad.any(), (tag, int(bad.sum()), ratio, err[bad][:4].tolist(), bound[bad][:4].tolist())


# ================================================================================================
# 1. loss terms of a supervised layer (lgb200_head_terms_fwd / _bwd)
# ================================================================================================
def _terms_case(B, M, N, seed, with_fin):
    """Kernel inputs for B pairs.  Pair kinds cycle by b % 4: ordinary, no positives, no negatives, every token positive.
    Logits of +-90 (exp overflows fp32) in both columns of zt; a fifth of the rows and columns have a dustbin score equal
    to their row / column max, bit for bit, with the final argmax on the inner argmax (the strict rule labels them 1)."""
    g = _gen(seed)
    TM, TN = B * M, B * N
    zt = _randn(TM + TN, 2, g=g, scale=3.0)
    zt[0::37, 0], zt[5::37, 0], zt[11::37, 1], zt[17::37, 1] = 90.0, -90.0, 90.0, -90.0
    cnt = lambda *s: (torch.rand(*s, device=DEV, generator=g) < 0.3).float() * torch.randint(  # noqa: E731
        1, 3, s, device=DEV, generator=g).float()
    rowcnt, colcnt = cnt(B, M), cnt(B, N)
    neg0 = ((rowcnt == 0) & (torch.rand(B, M, device=DEV, generator=g) < 0.8)).float()
    neg1 = ((colcnt == 0) & (torch.rand(B, N, device=DEV, generator=g) < 0.8)).float()
    for b in range(B):
        if b % 4 == 1:  # no positives: num_pos clamps to 1
            rowcnt[b], colcnt[b] = 0.0, 0.0
        elif b % 4 == 2:  # no negatives: num_neg clamps to 1 + 1
            neg0[b], neg1[b] = 0.0, 0.0
        elif b % 4 == 3:  # every token positive
            rowcnt[b].clamp_(min=1.0), colcnt[b].clamp_(min=1.0)
            neg0[b], neg1[b] = 0.0, 0.0
    # sum_j gt_ij (2 sim - lse_r - lse_c) <= 0, zero for rows without positives
    pos_row_sum = -rowcnt * (torch.rand(B, M, device=DEV, generator=g) * 8 + 0.1)
    num_pos = rowcnt.sum(1).clamp(min=1.0)
    num_neg = neg0.sum(1).clamp(min=1.0) + neg1.sum(1).clamp(min=1.0)  # as matchers/lightglue.py passes it
    _, du = ops.head_logsig(zt)  # the kernel's own fp32 dustbin scores: the labels are decisions taken on them
    du0, du1 = du[:TM].view(B, M), du[TM:].view(B, N)
    rowarg = torch.randint(0, N, (B, M), device=DEV, generator=g, dtype=torch.int32)
    colarg = torch.randint(0, M, (B, N), device=DEV, generator=g, dtype=torch.int32)
    off = lambda *s: (torch.rand(*s, device=DEV, generator=g) * 2 + 0.05) * torch.where(  # noqa: E731
        torch.rand(*s, device=DEV, generator=g) < 0.5, -1.0, 1.0)
    rowmax, colmax = du0 + off(B, M), du1 + off(B, N)
    rowmax[:, 0::5], colmax[:, 2::5] = du0[:, 0::5], du1[:, 2::5]  # ties
    fin0 = fin1 = None
    if with_fin:
        def fin(arg, width, s):
            r = torch.rand(*s, device=DEV, generator=g)
            other = torch.randint(0, width, s, device=DEV, generator=g, dtype=torch.int32)
            return torch.where(r < 0.4, arg, torch.where(r < 0.7, torch.full_like(arg, width), other))
        fin0, fin1 = fin(rowarg, N, (B, M)), fin(colarg, M, (B, N))
        fin0[:, 0::5], fin1[:, 2::5] = rowarg[:, 0::5], colarg[:, 2::5]
    return dict(zt=zt, pos_row_sum=pos_row_sum, rowcnt=rowcnt, colcnt=colcnt, neg0=neg0, neg1=neg1, rowmax=rowmax,
                rowarg=rowarg, colmax=colmax, colarg=colarg, fin0=fin0, fin1=fin1, num_pos=num_pos, num_neg=num_neg,
                du=du, B=B, M=M, N=N)


def _terms_prefix(c, Bp):
    """The first Bp pairs of a case (zt is [side-0 tokens of all pairs; side-1 tokens of all pairs])."""
    B, M, N = c["B"], c["M"], c["N"]
    out = {k: (v[:Bp] if torch.is_tensor(v) and v.shape[0] == B else v) for k, v in c.items()}
    out["zt"] = torch.cat([c["zt"][:Bp * M], c["zt"][B * M:B * M + Bp * N]])
    out["du"] = torch.cat([c["du"][:Bp * M], c["du"][B * M:B * M + Bp * N]])
    out["B"] = Bp
    return out


def _terms_fwd(c, bal, counters):
    B, M, N = c["B"], c["M"], c["N"]
    out = torch.full((4, B), float("nan"), device=DEV)
    ws = torch.empty(4 * B * ((M + N + 255) // 256), device=DEV)
    call("lgb200_head_terms_fwd", ptr(c["zt"]), ptr(c["pos_row_sum"]), ptr(c["rowcnt"]), ptr(c["colcnt"]),
         ptr(c["neg0"]), ptr(c["neg1"]), ptr(c["rowmax"]), ptr(c["rowarg"]), ptr(c["colmax"]), ptr(c["colarg"]),
         ptr(c["fin0"]), ptr(c["fin1"]), ptr(c["num_pos"]), ptr(c["num_neg"]), float(bal), ptr(out[0]), ptr(out[1]),
         ptr(out[2]), ptr(out[3]), ptr(ws), ptr(counters), B, M, N, stream_ptr())
    return out  # nll, nll_pos, nll_neg, conf


def _terms_bwd(c, bal, g_nll, g_conf):
    dzt = torch.full_like(c["zt"], float("nan"))
    call("lgb200_head_terms_bwd", ptr(c["zt"]), ptr(c["rowcnt"]), ptr(c["colcnt"]), ptr(c["neg0"]), ptr(c["neg1"]),
         ptr(c["rowmax"]), ptr(c["rowarg"]), ptr(c["colmax"]), ptr(c["colarg"]), ptr(c["fin0"]), ptr(c["fin1"]),
         ptr(c["num_pos"]), ptr(c["num_neg"]), float(bal), ptr(g_nll), ptr(g_conf), ptr(dzt), c["B"], c["M"], c["N"],
         stream_ptr())
    return dzt


def _terms_ref(c, bal, zt64):
    """losses.py:weight_loss (NLL with positives / negatives balanced by bal) and TokenConfidence.loss in fp64.
    Returns the four outputs and, per pair, sum(|terms|) of nll_pos, nll_neg and conf (the scales of their errors)."""
    B, M, N, d = c["B"], c["M"], c["N"], lambda k: c[k].double()  # noqa: E731
    z0, z1 = zt64[:B * M].view(B, M, 2), zt64[B * M:].view(B, N, 2)
    ls0, ls1, du0, du1 = F.logsigmoid(z0[..., 0]), F.logsigmoid(z1[..., 0]), F.logsigmoid(-z0[..., 0]), F.logsigmoid(-z1[..., 0])
    pt = [d("pos_row_sum"), d("rowcnt") * ls0, d("colcnt") * ls1]
    nt = [d("neg0") * du0, d("neg1") * du1]
    nll_pos = -sum(t.sum(1) for t in pt) / d("num_pos")
    nll_neg = -sum(t.sum(1) for t in nt) / d("num_neg")
    nll = bal * nll_pos + (1 - bal) * nll_neg
    s_pos = sum(t.abs().sum(1) for t in pt) / d("num_pos")
    # the kernel forms du = log sigmoid(z) - z: its round-off is that of |z|, not of |du| (they differ for z << 0)
    s_neg = ((d("neg0") * (du0.abs() + z0[..., 0].abs())).sum(1)
             + (d("neg1") * (du1.abs() + z1[..., 0].abs())).sum(1)).detach() / d("num_neg")
    if c["fin0"] is None:
        conf = torch.zeros_like(nll)
    else:
        kdu0, kdu1 = c["du"][:B * M].view(B, M), c["du"][B * M:].view(B, N)
        arg0 = torch.where(kdu0 > c["rowmax"], N, c["rowarg"])  # the dustbin wins only when strictly larger
        arg1 = torch.where(kdu1 > c["colmax"], M, c["colarg"])
        bce = F.binary_cross_entropy_with_logits
        conf = (bce(z0[..., 1], (c["fin0"] == arg0).double(), reduction="none").mean(1)
                + bce(z1[..., 1], (c["fin1"] == arg1).double(), reduction="none").mean(1)) / 2
    return (nll, nll_pos, nll_neg, conf), (bal * s_pos + (1 - bal) * s_neg, s_pos, s_neg, conf.abs())


TERM_SHAPES = [(1, 1), (255, 1), (256, 256), (1000, 777), (2048, 2048)]


@pytest.mark.parametrize("with_fin", [False, True])
@pytest.mark.parametrize("bal", [0.0, 0.5, 1.0])
@pytest.mark.parametrize("M,N", TERM_SHAPES)
@pytest.mark.parametrize("B", [1, 3, 32])
def test_head_terms_against_fp64(B, M, N, bal, with_fin):
    c = _terms_case(B, M, N, seed=1000 * B + M + 7 * N, with_fin=with_fin)
    out = _terms_fwd(c, bal, torch.zeros(B, device=DEV, dtype=torch.int32))
    zt64 = c["zt"].double().requires_grad_(True)
    ref, scale = _terms_ref(c, bal, zt64)
    # per pair: warp (5) + block (8) + chunk (<= 16) partial sums, ~4 roundings per term and 3 in the final scaling
    chain = 5 + 8 + (M + N + 255) // 256 + 8
    tag = f"head_terms_fwd B={B} M={M} N={N} bal={bal} fin={with_fin}"
    for i, name in enumerate(("nll", "nll_pos", "nll_neg", "conf")):
        _within((out[i].double() - ref[i].detach()).abs(), chain * U32 * scale[i], f"{tag} {name}")
    if not with_fin:
        assert torch.equal(out[3], torch.zeros_like(out[3]))
    # backward against fp64 autograd of the same loss, for random upstream gradients
    g = _gen(B + M + N)
    g_nll, g_conf = _randn(B, g=g), _randn(B, g=g)
    (ref[0] * g_nll.double() + ref[3] * g_conf.double()).sum().backward()
    dzt = _terms_bwd(c, bal, g_nll, g_conf)
    # per token, |d/dz_match| <= |g_nll| (bal cnt / num_pos + (1 - bal) neg / num_neg), |d/dz_tok| <= |g_conf| / (2 L);
    # sigmoid, the divisions and the products: under 16 roundings of that magnitude
    b0, b1 = torch.arange(B, device=DEV).repeat_interleave(M), torch.arange(B, device=DEV).repeat_interleave(N)
    bt = torch.cat([b0, b1])
    cnt = torch.cat([c["rowcnt"].reshape(-1), c["colcnt"].reshape(-1)]).double()
    ng = torch.cat([c["neg0"].reshape(-1), c["neg1"].reshape(-1)]).double()
    mx = g_nll.double().abs()[bt] * (bal * cnt / c["num_pos"].double()[bt] + (1 - bal) * ng / c["num_neg"].double()[bt])
    L = torch.cat([torch.full((B * M,), M, device=DEV), torch.full((B * N,), N, device=DEV)]).double()
    my = g_conf.double().abs()[bt] * 0.5 / L if with_fin else torch.zeros_like(mx)
    err = (dzt.double() - zt64.grad).abs()
    _within(err[:, 0], 16 * U32 * mx, f"head_terms_bwd {tag} dz_match")
    _within(err[:, 1], 16 * U32 * my, f"head_terms_bwd {tag} dz_tok")
    assert err.norm() <= 16 * U32 * torch.stack([mx, my], 1).norm(), rel_err(dzt, zt64.grad)


def test_head_terms_counters_shared_across_calls():
    """The per-pair arrival counters reset themselves: calls with B = 32, 3, 1 and 32 on one counter buffer give, pair
    for pair, bit-identical results, and leave every counter at zero."""
    c = _terms_case(32, 2048, 2048, seed=5, with_fin=True)
    counters = torch.zeros(64, device=DEV, dtype=torch.int32)
    first = _terms_fwd(c, 0.5, counters)
    assert torch.isfinite(first).all()
    for Bp in (3, 1, 32):
        out = _terms_fwd(_terms_prefix(c, Bp), 0.5, counters)
        assert torch.equal(out, first[:, :Bp]), Bp
        assert torch.equal(counters, torch.zeros_like(counters)), Bp


# ================================================================================================
# 2. LayerNorm + GELU of the FFN (lgb200_ln_gelu_fwd / _bwd)
# ================================================================================================
EPS_LN = 1e-5


def _ln_case(T, W, dtype, seed):
    g = _gen(seed)
    x = _randn(T, W, g=g, scale=2.0) + _randn(T, 1, g=g)
    if T >= 7:
        x[1] = -1.5  # constant row: variance 0, rstd = eps^-1/2
        x[3::977] = 1e3 + _randn(x[3::977].shape[0], W, g=g)  # large common offset
        x[5] = -1e3 + _randn(W, g=g)
    gamma, beta = 1 + _randn(W, g=g, scale=0.1), _randn(W, g=g, scale=0.1)
    return x.to(dtype), gamma, beta, _randn(T, W, g=g).to(dtype)


def _ln_ref_chunks(x, gamma, beta, dy, chunk):
    """fp64 LayerNorm + exact-erf GELU and its autograd gradients, chunk by chunk of tokens."""
    W = x.shape[1]
    for s in range(0, x.shape[0], chunk):
        xr = x[s:s + chunk].double().requires_grad_(True)
        gr, br = gamma.double().requires_grad_(True), beta.double().requires_grad_(True)
        u = F.layer_norm(xr, (W,), gr, br, EPS_LN)
        y = F.gelu(u)
        dy64 = dy[s:s + chunk].double()
        dx, dg, db = torch.autograd.grad(y, (xr, gr, br), dy64)
        with torch.no_grad():
            var, mu = torch.var_mean(xr, 1, correction=0)
            rstd = (var + EPS_LN).rsqrt()
            h = (xr - mu[:, None]) * rstd[:, None]
            # error of the normalised input: the fp32 mean is off by ~U32 |mean|, which h sees times rstd
            k = 1 + mu.abs() * rstd
        yield s, dict(y=y.detach(), mean=mu, rstd=rstd, h=h, u=u.detach(), dx=dx, dg=dg, db=db, dy=dy64, k=k,
                      absmean=xr.abs().mean(1))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("T", [1, 7, 1001, 4097, TOK])
@pytest.mark.parametrize("W", [256, 512, 1024])
def test_ln_gelu_against_fp64(W, T, dtype):
    x, gamma, beta, dy = _ln_case(T, W, dtype, seed=W + T)
    y, mean, rstd = ops.ln_gelu_fwd(x, gamma, beta, EPS_LN)
    dx, dg, db, dxs = ops.ln_gelu_bwd(dy, x, gamma, beta, mean, rstd, want_dxsum=True)
    # two calls are bit-equal.  In the backward this is the check that can see a race on the row sums the warps of
    # a token exchange through shared memory (the s_rows double buffer); such a race corrupts only some runs, so
    # a broken buffer flip is caught with a probability that depends on timing, at T = 131072 (W = 512 or 1024),
    # where the backward is repeated a few times (about 1 ms per call) to raise that probability.
    y2, mean2, rstd2 = ops.ln_gelu_fwd(x, gamma, beta, EPS_LN)
    assert torch.equal(y, y2) and torch.equal(mean, mean2) and torch.equal(rstd, rstd2)
    del y2, mean2, rstd2
    for _ in range(8 if T == TOK else 1):
        again = ops.ln_gelu_bwd(dy, x, gamma, beta, mean, rstd, want_dxsum=True)
        assert all(torch.equal(a, b) for a, b in zip((dx, dg, db, dxs), again))
        del again
    R = _rnd(dtype)
    nch = W // 256
    # a row sum of the forward: 4 NCH pair sums per lane, then 5 shuffle levels; mean = sum / W (exact)
    n_row = 4 * nch + 6
    # round-off of the normalisation and the GELU, and of the backward's row sums, in units of U32 k: bounds set at
    # 4-8x the worst measured on an H100 (y: 3.5 U32 k (1 + |u|); dx: 1 U32 k per row magnitude)
    c_y, c_dx = 16, 8
    parts = _lib.load().lgb200_ln_gelu_bwd_parts(T)
    slots = 8 // nch
    # dgamma / dbeta / dxsum: per-slot token loop, the slots of a CTA, then the sum over the CTA partials, plus the
    # round-off of each term
    chain = -(-T // (parts * slots)) + slots + parts + c_y
    tag = f"ln_gelu W={W} T={T} {str(dtype)[6:]}"
    acc = {k: torch.zeros(W, device=DEV, dtype=torch.float64) for k in ("dg", "db", "dxs", "sdg", "sdb", "sdxs")}
    worst = dict(y=0.0, dx=0.0, mean=0.0, rstd=0.0)
    normal_err = dict(y=0.0, dx=0.0)
    normal_ref = dict(y=0.0, dx=0.0)
    for s, r in _ln_ref_chunks(x, gamma, beta, dy, chunk=8192 if W == 1024 else 16384):
        n = r["y"].shape[0]
        k = r["k"][:, None]
        # y: fp32 round-off through the normalisation (k) and the GELU, the erf approximation, the output rounding
        ey = (y[s:s + n].double() - r["y"]).abs()
        by = (ERF + c_y * U32 * k) * (1 + r["u"].abs()) + R * r["y"].abs()
        worst["y"] = max(worst["y"], (ey / by).max().item())
        assert (ey <= by).all(), (tag, "y", s)
        # mean: n_row roundings of sum(|x|) / W
        em = (mean[s:s + n].double() - r["mean"]).abs()
        worst["mean"] = max(worst["mean"], (em / (n_row * U32 * r["absmean"])).max().item())
        assert (em <= n_row * U32 * r["absmean"]).all(), (tag, "mean", s)
        # rstd, relative: the two-pass variance is a chain of 8 NCH + 7 fp32 roundings (+ eps: one more), halved by the
        # square root, and rsqrtf adds at most 2 ulp: (4 NCH + 6) U32 = n_row U32; the mean's error adds
        # (mean error * rstd)^2 / 2, which only rows with a large common offset (large k) can see
        er = (rstd[s:s + n].double() - r["rstd"]).abs() / r["rstd"]
        br = n_row * U32 + 0.5 * (n_row * U32 * r["k"]) ** 2
        worst["rstd"] = max(worst["rstd"], (er / br).max().item())
        assert (er <= br).all(), (tag, "rstd", s)
        # dx, per row: magnitude rstd max|dy g| (1 + max|h|); erf approximation and round-off of gelu', the two row
        # means, the output rounding
        hmax = r["h"].abs().amax(1, keepdim=True)
        srow = r["rstd"][:, None] * (r["dy"] * gamma.double()).abs().amax(1, keepdim=True) * (1 + hmax)
        edx = (dx[s:s + n].double() - r["dx"]).abs()
        bdx = (2 * ERF + c_dx * U32 * k) * srow + R * r["dx"].abs()
        worst["dx"] = max(worst["dx"], (edx / bdx).max().item())
        assert (edx <= bdx).all(), (tag, "dx", s)
        ok = r["k"] < 16  # rows without a large common offset (their error is k times that of the others)
        normal_err["y"] += (ey[ok] ** 2).sum().item()
        normal_ref["y"] += (r["y"][ok] ** 2).sum().item()
        normal_err["dx"] += (edx[ok] ** 2).sum().item()
        normal_ref["dx"] += (r["dx"][ok] ** 2).sum().item()
        # reductions over tokens: a term dz (dz h for dgamma) is off by ~(ERF + c_y U32 k (1 + |h|)) |dy|, a term of
        # dxsum by what dx is off by above; the sum adds chain U32 of sum(|terms|)
        dz = r["dy"].abs() * (1 + r["h"].abs()) * k
        acc["dg"] += r["dg"]
        acc["db"] += r["db"]
        acc["dxs"] += r["dx"].sum(0)
        acc["sdg"] += (dz * (1 + r["h"].abs())).sum(0)
        acc["sdb"] += dz.sum(0)
        acc["sdxs"] += ((r["dx"].abs() + srow) * k).sum(0)
    report(tag, **{f"{k}_err_over_bound": v for k, v in worst.items()})
    # norm-relative, over the rows without a large offset
    ny = math.sqrt(normal_err["y"] / max(normal_ref["y"], 1e-300))
    ndx = math.sqrt(normal_err["dx"] / max(normal_ref["dx"], 1e-300))
    report(tag, y_rel=ny, dx_rel=ndx)
    assert ny < 2 * ERF + c_y * U32 + R and ndx < 2 * ERF + c_y * U32 + R, (ny, ndx)
    for got, ref, sc, name in ((dg, acc["dg"], acc["sdg"], "dgamma"), (db, acc["db"], acc["sdb"], "dbeta"),
                               (dxs, acc["dxs"], acc["sdxs"], "dxsum")):
        _within((got.double() - ref).abs(), (2 * ERF + chain * U32) * sc, f"{tag} {name}", rel=rel_err(got, ref))


# ================================================================================================
# 3. residual add + cast (lgb200_residual_add_cast, _pitched, lgb200_add_f32_cast)
# ================================================================================================
SENT = 1e30  # never the sum of two unit normals


@pytest.mark.parametrize("with_y", [False, True])
@pytest.mark.parametrize("rem", [0, 1, 7])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_residual_add_cast_bit_exact(dtype, rem, with_y):
    """x_out = x + y and x_cast = (dtype) x_out are torch's fp32 add and cast, bit for bit, including the scalar tail
    (numel % 8 != 0); nothing past numel is written."""
    n = 8 * 65537 + rem
    g = _gen(31 + rem)
    x = _randn(n, g=g)
    y = _randn(n, g=g).to(dtype) if with_y else None
    xo = torch.full((n + 16,), SENT, device=DEV)
    xc = torch.full((n + 16,), SENT, device=DEV, dtype=dtype)
    call("lgb200_residual_add_cast", ptr(x), ptr(y), ptr(xo) if with_y else None, ptr(xc), n, ops._code(dtype),
         stream_ptr())
    s = x + y.float() if with_y else x
    assert torch.equal(xc[:n], s.to(dtype)) and (xc[n:] == SENT).all()
    if with_y:
        assert torch.equal(xo[:n], s) and (xo[n:] == SENT).all()


@pytest.mark.parametrize("with_y", [False, True])
@pytest.mark.parametrize("T", [7, 4097])
@pytest.mark.parametrize("D", [128, 256])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_residual_add_cast_pitched_keeps_sentinels(dtype, D, T, with_y):
    """The cast copy lands in big[1:T+1, pad:pad+D] of a sentinel-filled [T+3, 2D+2 pad] buffer, as it lands in the
    left half of the [x | msg] operand of ffn.0: bit-equal to torch, and every other element keeps its sentinel."""
    pad = 8
    g = _gen(D + T)
    x = _randn(T, D, g=g)
    y = _randn(T, D, g=g).to(dtype) if with_y else None
    big = torch.full((T + 3, 2 * D + 2 * pad), SENT, device=DEV, dtype=dtype)
    view = big[1:T + 1, pad:pad + D]
    x_new, _ = ops.residual_add_cast(x, y, dtype, out_cast=view)
    s = x + y.float() if with_y else x
    assert torch.equal(x_new, s)
    assert torch.equal(view, s.to(dtype))
    keep = torch.ones_like(big, dtype=torch.bool)
    keep[1:T + 1, pad:pad + D] = False
    assert (big[keep] == SENT).all()


@pytest.mark.parametrize("rem", [0, 1, 7])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_add_f32_cast_bit_exact(dtype, rem):
    n = 8 * 40961 + rem
    g = _gen(77 + rem)
    x0, y = _randn(n, g=g), _randn(n, g=g, scale=3.0)
    x = x0.clone()
    x_out, xc = ops.add_f32_cast_(x, y, dtype)
    assert x_out.data_ptr() == x.data_ptr()
    assert torch.equal(x, x0 + y) and torch.equal(xc, (x0 + y).to(dtype))


# ================================================================================================
# 4. rotary backward (lgb200_rope_split_bwd accumulates into dtheta)
# ================================================================================================
def _rot64(x, th):
    """rotate consecutive channel pairs (2p, 2p+1) of x [T, H, 64] by th [T, 32] (lightglue.py:42-49)"""
    c, s = th.cos()[:, None, :], th.sin()[:, None, :]
    x0, x1 = x[..., 0::2], x[..., 1::2]
    return torch.stack([x0 * c - x1 * s, x1 * c + x0 * s], -1).flatten(-2)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("H", [1, 4])
@pytest.mark.parametrize("T", [1, 333, TOK])
def test_rope_bwd_accumulates_into_dtheta(T, H, dtype):
    g = _gen(T + H)
    q, k = _randn(T, H * 64, g=g).to(dtype), _randn(T, H * 64, g=g).to(dtype)  # rotated, as saved by forward
    dq, dk, dv = (_randn(T, H * 64, g=g).to(dtype) for _ in range(3))
    theta = _randn(T, 32, g=g, scale=3.0)
    dtheta0 = _randn(T, 32, g=g)
    dtheta = dtheta0.clone()
    dqkv, _ = ops.rope_bwd(dq, dk, dv, q, k, theta, H, dtheta=dtheta)
    dqkv2, _ = ops.rope_bwd(dq, dk, dv, q, k, theta, H, dtheta=dtheta)
    assert torch.equal(dqkv, dqkv2)
    R = _rnd(dtype)
    tag = f"rope_bwd T={T} H={H} {str(dtype)[6:]}"
    worst = dict(dtheta=0.0, dqkv=0.0)
    for s in range(0, T, 32768):
        sl = slice(s, s + 32768)
        n = theta[sl].shape[0]
        v64 = lambda t: t[sl].double().view(n, H, 64)  # noqa: E731
        th = theta[sl].double().requires_grad_(True)
        qu = _rot64(v64(q), -th.detach()).requires_grad_(True)  # un-rotated inputs of the forward
        ku = _rot64(v64(k), -th.detach()).requires_grad_(True)
        loss = (_rot64(qu, th) * v64(dq)).sum() + (_rot64(ku, th) * v64(dk)).sum()
        gth, gq, gk = torch.autograd.grad(loss, (th, qu, ku))
        # dtheta_p = sum over heads of 4 products: 4H sequential additions, then two accumulations
        a, b = v64(dq), v64(dk)
        qq, kk = v64(q), v64(k)
        sc = ((a[..., 1::2] * qq[..., 0::2]).abs() + (a[..., 0::2] * qq[..., 1::2]).abs()
              + (b[..., 1::2] * kk[..., 0::2]).abs() + (b[..., 0::2] * kk[..., 1::2]).abs()).sum(1)
        want = dtheta0[sl].double() + 2 * gth
        e = (dtheta[sl].double() - want).abs()
        bnd = (4 * H + 4) * U32 * (dtheta0[sl].double().abs() + 2 * sc)
        worst["dtheta"] = max(worst["dtheta"], (e / bnd).max().item())
        assert (e <= bnd).all(), (tag, "dtheta", s)
        # dqkv interleaves (R(-theta) dq, R(-theta) dk, dv) per channel; each is two products of |dq| and sincos
        ref = torch.stack([gq, gk, v64(dv)], -1).reshape(n, H * 192)
        pair = lambda t: (t[..., 0::2].abs() + t[..., 1::2].abs()).repeat_interleave(2, -1)  # noqa: E731
        mag = torch.stack([pair(a), pair(b), torch.zeros_like(a)], -1).reshape(n, H * 192)
        e = (dqkv[sl].double() - ref).abs()
        bnd = 8 * U32 * mag + R * ref.abs()
        worst["dqkv"] = max(worst["dqkv"], (e / bnd.clamp(min=1e-300)).max().item())
        assert (e <= bnd).all(), (tag, "dqkv", s)
    report(tag, **{f"{k}_err_over_bound": v for k, v in worst.items()})


# ================================================================================================
# 5. token-head backward, position-encoder weight gradient, column sums at the benchmark's size
# ================================================================================================
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_head_token_bwd_at_bench_size(dtype):
    T, D = TOK, 256
    g = _gen(3)
    x = _randn(T, D, g=g) + _randn(D, g=g)  # non-zero column means: a lost partial shows
    dmdw = _randn(T, D, g=g).to(dtype)
    dzt = _randn(T, 2, g=g) + 0.5
    wm = _randn(D, g=g, scale=0.1)
    dx, dW2, db2 = ops.head_token_bwd(x, dmdw, dzt, wm)
    again = ops.head_token_bwd(x, dmdw, dzt, wm)
    assert all(torch.equal(a, b) for a, b in zip((dx, dW2, db2), again))
    del again
    tag = f"head_token_bwd T={T} D={D} {str(dtype)[6:]}"
    x64, z64 = x.double(), dzt.double()
    ref = dmdw.double() + z64[:, :1] * wm.double()
    _within((dx.double() - ref).abs(), U32 * (dmdw.double().abs() + (z64[:, :1] * wm.double()).abs()), f"{tag} dx")
    del ref
    # per warp over ceil(T / (592 * 8)) tokens, 8 warps, then 592 CTA partials in order
    chain = -(-T // (592 * 8)) + 8 + 592
    _within((dW2.double() - z64.t() @ x64).abs(), chain * U32 * (z64.abs().t() @ x64.abs()), f"{tag} dW2")
    _within((db2.double() - z64.sum(0)).abs(), chain * U32 * z64.abs().sum(0), f"{tag} db2")


@pytest.mark.parametrize("kd", [2, 4])
def test_posenc_wgrad_at_bench_size(kd):
    T = TOK
    g = _gen(kd)
    gth = _randn(T, 32, g=g) + 0.3
    kp = _randn(T, kd, g=g) * 100 + 200  # pixel coordinates
    nb = _lib.load().lgb200_posenc_wgrad_blocks()
    parts = [torch.full((nb, 32, kd), float("nan"), device=DEV) for _ in range(2)]
    for p in parts:
        call("lgb200_posenc_wgrad", ptr(gth), ptr(kp), ptr(p), T, 32, kd, stream_ptr())
    assert torch.equal(parts[0], parts[1])
    got = parts[0].double().sum(0)
    ref = gth.double().t() @ kp.double()
    # per warp-slot over ceil(T / (nb * 8)) tokens, then the 8 slots of a CTA (the partials are summed here in fp64)
    chain = -(-T // (nb * 8)) + 8
    _within((got - ref).abs(), chain * U32 * (gth.double().abs().t() @ kp.double().abs()), f"posenc_wgrad kd={kd}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_colsum_widths_back_to_back(dtype):
    """A layer's backward sums columns of widths 768, 256 and 512 one after the other on one set of arrival counters."""
    g = _gen(9)
    mats = {w: (_randn(TOK, w, g=g) + _randn(w, g=g)).to(dtype) for w in (768, 256, 512)}
    outs = [(w, ops.colsum(mats[w])) for w in (768, 256, 512, 768)]
    assert torch.equal(outs[0][1], outs[3][1])
    for w, got in outs[:3]:
        a = mats[w].double()
        nslabs = _lib.load().lgb200_colsum_slabs(TOK, w)
        rps = -(-TOK // nslabs)
        chain = -(-rps // 32) + 32 + nslabs  # per thread, the 32 row lanes, the slab partials in order
        _within((got.double() - a.sum(0)).abs(), chain * U32 * a.abs().sum(0), f"colsum w={w} {str(dtype)[6:]}")


# ================================================================================================
# 6. misaligned pointers are refused on the host, before any launch
# ================================================================================================
def _misaligned_each(fn, ptrs):
    """Call fn with each pointer in turn moved 4 bytes off its 16-byte boundary; every call must be refused."""
    for i in range(len(ptrs)):
        args = [ctypes.c_void_p(p + (4 if j == i else 0)) for j, p in enumerate(ptrs)]
        with pytest.raises(Lgb200Error, match="misaligned"):
            fn(*args)


def test_misaligned_pointers_are_refused():
    buf = [torch.zeros(64 * 1024, device=DEV) for _ in range(10)]
    p = [b.data_ptr() for b in buf]
    s = stream_ptr()
    for dt in (_lib.F32, _lib.BF16):
        _misaligned_each(lambda x, y, xo, xc: call("lgb200_residual_add_cast_pitched", x, y, xo, xc, 4, 64, 128, dt, s),
                         p[:4])
        _misaligned_each(lambda x, y, xo, xc: call("lgb200_residual_add_cast", x, y, xo, xc, 256, dt, s), p[:4])
        _misaligned_each(lambda x, y, xo, xc: call("lgb200_add_f32_cast", x, y, xo, xc, 256, dt, s), p[:4])
        _misaligned_each(lambda src, dst: call("lgb200_cast_bf16", src, dst, 256, s), p[:2])
        _misaligned_each(lambda x, ga, be, y: call("lgb200_ln_gelu_fwd", x, ga, be, y, ctypes.c_void_p(p[8]),
                                                   ctypes.c_void_p(p[9]), 8, 256, 1e-5, dt, s), p[:4])
        _misaligned_each(lambda dy, x, ga, be, dx: call("lgb200_ln_gelu_bwd", dy, x, ga, be, ctypes.c_void_p(p[8]),
                                                        ctypes.c_void_p(p[9]), dx, ctypes.c_void_p(p[5]),
                                                        ctypes.c_void_p(p[6]), ctypes.c_void_p(p[7]), 8, 256, dt, s),
                         p[:5])
        _misaligned_each(lambda qkv, th, q, k, v: call("lgb200_rope_split_fwd", qkv, th, q, k, v, 8, 1, dt, s), p[:5])
        _misaligned_each(lambda *a: call("lgb200_rope_split_bwd", *a, 8, 1, dt, s), p[:8])
    torch.cuda.synchronize()
