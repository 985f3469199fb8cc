"""Error bounds and fp32 restatements for the SuperPoint-open BatchNorm paths (csrc/superpoint.cu, the `spo_*` entry
points, and lgb200_bn_stats / lgb200_bn_running_update of csrc/elementwise.cu), used by
tests/test_gpu_superpoint_open_shapes.py and checked on the CPU by tests/test_superpoint_open_restatements_cpu.py.

Notation: u = 2^-24 (fp32), u64 = 2^-53 (fp64), gamma(n) = n u / (1 - n u) bounds the relative error of n
roundings (Higham's lemma).  Every bound is element-wise, fp64, and derived from the kernels' operation order; none
has a tuning constant.

Eval mode (running statistics).  bn_affine forms, in fp32 on the device, s' = g / sqrt(rv + eps) (three roundings,
one of them under the square root, and eps itself rounded: |s' - s| <= gamma(3) |s|) and t' = b - rm s' (product and
difference: |t' - t| <= gamma(5) |rm s| + u |b|).  The epilogue evaluates fmaf(r, s', t') on the staged fp32 value
r, itself within E of the exact r* (E from conv_acc_bound; ReLU is 1-Lipschitz).  The reference is the unfolded
BatchNorm (r* - rm) / sqrt(rv + eps) g + b of the same fp32 buffers, so the fold's roundings count as error.

Training mode (batch statistics).  lgb200_bn_stats sums x and x^2 of n exact terms (a bf16 or fp32 value and its
square are exact in fp64) in some order: each sum is within gamma64(n - 1) of the sum of |terms|.  spo_bn_setup
forms in fp64 m = S1 / n and the one-pass variance S2 / n - m^2, whose error is that of S2 / n and of m^2, so it is
largest against the variance where |m| is large against the spread; then in fp32 mu = fl(m) and
rs = 1 / sqrt(fl(var) + eps).  The element is fmaf((x - mu) rs, g, b).  The reference is fp64 BatchNorm with the
two-pass variance sum (x - m)^2 / n.
"""
import torch

from tests.superpoint_oracle import U, U_BF16, l2n_bound, pool_bf16_bound, relu_bf16_bound, softmax_bound  # noqa

U64 = 2.0 ** -53


def gamma(n, u=U):
    return n * u / (1 - n * u)


# ---- eval mode: the folded affine ------------------------------------------------------------------------------------
def bn_view(t, dim, ndim):
    """A [C] tensor as fp64, shaped to broadcast along `dim` of an ndim-dimensional tensor."""
    shape = [1] * ndim
    shape[dim] = -1
    return t.detach().double().reshape(shape)


def folded_affine(r, E, g, b, rm, rv, eps, dim=1):
    """r: fp64 value before the BatchNorm (ReLU output or logits), E its bound; g, b, rm, rv: the module's fp32 [C]
    buffers.  -> (z, e): the unfolded fp64 BatchNorm (r - rm) / sqrt(rv + eps) g + b, and the bound on the kernel's
    fmaf(r', s', t') before any store."""
    g, b, rm, rv = (bn_view(t, dim, r.dim()).to(r.device) for t in (g, b, rm, rv))
    z = (r - rm) / torch.sqrt(rv + eps) * g + b
    s = g / torch.sqrt(rv + eps)
    e = (E * s.abs() * (1 + gamma(3)) + gamma(3) * (r * s).abs() + gamma(5) * (rm * s).abs() + U * b.abs()) * (1 + U)
    return z, e + U * z.abs()


# ---- training mode: batch statistics ---------------------------------------------------------------------------------
class Stats:
    """Per-channel fp64 statistics of one BatchNorm's input, accumulated over chunks of [*, C] values: the sums
    S1 = sum x, S2 = sum x^2, A = sum |x| and n, then (second pass) Q = sum (x - m)^2 about the reference mean."""

    def __init__(self, C, device):
        z = (lambda: torch.zeros(C, dtype=torch.float64, device=device))
        self.S1, self.S2, self.A, self.Q = z(), z(), z(), z()
        self.n = 0

    def add(self, x):
        x = x.reshape(-1, x.shape[-1]).double()
        self.S1 += x.sum(0)
        self.S2 += (x * x).sum(0)
        self.A += x.abs().sum(0)
        self.n += x.shape[0]

    def add_centred(self, x):
        x = x.reshape(-1, x.shape[-1]).double() - self.mean
        self.Q += (x * x).sum(0)

    @property
    def mean(self):
        return self.S1 / self.n

    @property
    def var(self):
        """Biased two-pass variance (after every add_centred)."""
        return self.Q / self.n

    def sums(self):
        """The bn_stats layout [S1 | S2 | n]."""
        return torch.cat([self.S1, self.S2, self.S1.new_tensor([float(self.n)])])

    def sum_bound(self):
        """|kernel sums - these sums| for the bn_stats layout: both are fp64 sums of the same n exact terms in two
        orders, each within gamma64(n - 1) of the sum of |terms|; the count is exact."""
        g = gamma(self.n - 1, U64) * (1 + gamma(self.n, U64))
        return torch.cat([2 * g * self.A, 2 * g * self.S2, self.S1.new_zeros(1)])

    def kernel_stat_bounds(self):
        """(em, dvar): bounds on |m_k - mean| and |var_k - var| for the mean and one-pass variance spo_bn_setup and
        lgb200_bn_running_update form in fp64 from the kernel's sums, against this reference's mean and two-pass
        variance.  The reference's own error (its sums, and the two-pass sum of squares) is included."""
        n, m, v = self.n, self.mean, self.var
        infl = 1 + gamma(n + 4, U64)
        e1 = 2 * gamma(n - 1, U64) * self.A * infl      # |S1_k - S1_ref|, S1_ref within gamma(n-1) A of exact
        e2 = 2 * gamma(n - 1, U64) * self.S2 * infl
        em_ref = gamma(n, U64) * self.A / n * infl       # |mean_ref - exact mean|
        em = (e1 / n) * (1 + U64) + U64 * (m.abs() + e1 / n) + em_ref * 2
        dsq = (e2 / n) * (1 + U64) + U64 * self.S2 / n * infl
        dmm = em * (2 * m.abs() + em) * (1 + U64) + U64 * m * m
        dvar_k = (dsq + dmm) * (1 + U64) + U64 * (v + dsq + dmm)
        dvar_ref = gamma(n + 3, U64) * (v + em_ref ** 2) * infl + em_ref ** 2
        return em, dvar_k + dvar_ref


def bn_apply_ref(x, st, g, b, eps, dim=-1):
    """x: the kernel's input values (fp64, any layout with channels along `dim`, exactly the stored bf16 / fp32);
    st: Stats of the whole batch.  -> (z, e): fp64 BatchNorm with the reference statistics, and the bound on the
    kernel's fmaf((x - mu) rs, g, b) before any store (spo_bn_setup's fp32 mu and rs from the kernel's fp64 one-pass
    statistics; the subtraction, the product and the FMA)."""
    nd = x.dim()
    dim = dim % nd
    em, dvar = st.kernel_stat_bounds()
    m, v = st.mean, st.var
    V = v + eps
    # fl32(var) + fl32(eps), rounded: |V_k - V| <= dvar (1 + gamma2) + gamma2 V
    rho = (dvar * (1 + gamma(2)) + gamma(2) * V) / V
    assert bool((rho < 0.5).all()), "statistics too uncertain for a bound"
    drs = (1 + rho / (2 * (1 - rho) ** 1.5)) * (1 + gamma(2)) - 1   # sqrt and reciprocal roundings
    dmu = em + U * (m.abs() + em)                                    # mu = fl32(m_k)
    rs = 1 / torch.sqrt(V)
    m_, rs_, drs_, dmu_ = (bn_view(t, dim, nd) for t in (m, rs, drs, dmu))
    g_, b_ = bn_view(g, dim, nd).to(x.device), bn_view(b, dim, nd).to(x.device)
    D = x - m_
    z = D * rs_ * g_ + b_
    err_p = D.abs() * rs_ * ((1 + gamma(2)) * (1 + drs_) - 1) + dmu_ * rs_ * (1 + gamma(2)) * (1 + drs_)
    e = g_.abs() * err_p * (1 + U) + U * z.abs()
    return z, e


def running_ref(st, rm0, rv0, momentum):
    """torch's running-statistics step in fp64: (1 - momentum) r + momentum stat, with the unbiased variance
    var n / (n - 1), and its bound for lgb200_bn_running_update: the fp64 mean and variance within
    kernel_stat_bounds, n / (n - 1) (two fp64 roundings), the fp32 casts, the fp32 momentum and 1 - momentum, the two
    products and the sum (contracted into an FMA or not)."""
    n = st.n
    em, dvar = st.kernel_stat_bounds()
    m = st.mean
    vu = st.var * n / (n - 1)
    dvu = dvar * n / (n - 1) * (1 + gamma(2, U64)) + gamma(2, U64) * vu
    out = []
    for r0, stat, dstat in ((rm0, m, em), (rv0, vu, dvu)):
        r0 = r0.detach().double().to(stat.device)
        ref = (1 - momentum) * r0 + momentum * stat
        e = (gamma(3) * r0.abs() + momentum * (dstat * (1 + gamma(3)) + gamma(3) * stat.abs())) * (1 + U)
        out.append((ref, e + U * ref.abs()))
    return out


# ---- fp32 restatements of the kernels, in another order (CPU) -------------------------------------------------------
def fma32(a, b, c):
    """fmaf emulated: the fp64 a * b + c (the product of two fp32 values is exact in fp64) rounded once to fp32."""
    return (a.double() * b.double() + c.double()).float()


def fold32(g, b, rm, rv, eps):
    """bn_affine's fp32 fold."""
    s = g.float() / torch.sqrt(rv.float() + eps)
    return s, b.float() - rm.float() * s


def bn_setup32(sums, eps):
    """spo_bn_setup: fp64 mean and one-pass variance from [S1 | S2 | n], then fp32 mu and rs."""
    C = (sums.numel() - 1) // 2
    n = sums[2 * C]
    m = sums[:C] / n
    var = (sums[C:2 * C] / n - m * m).clamp_min(0.0)
    eps32 = torch.tensor(eps, dtype=torch.float32)
    return m.float(), 1.0 / torch.sqrt(var.float() + eps32)


def bn_apply32(x, mu, rs, g, b):
    """spo_bn on channel-last fp32 x: fmaf((x - mu) * rs, g, b)."""
    return fma32((x.float() - mu) * rs, g.float(), b.float())


def running_update32(sums, rm, rv, momentum, unbiased=True):
    """lgb200_bn_running_update in fp32 (the sum evaluated as fmaf(momentum, stat, (1 - momentum) r))."""
    C = rm.numel()
    n = sums[2 * C]
    m = sums[:C] / n
    var = (sums[C:2 * C] / n - m * m).clamp_min(0.0)
    if unbiased:
        var = var * n / (n - 1.0)
    mom = torch.tensor(momentum, dtype=torch.float32)
    one_m = 1.0 - mom
    return (fma32(mom.expand(C), m.float(), one_m * rm.float()), fma32(mom.expand(C), var.float(), one_m * rv.float()))
