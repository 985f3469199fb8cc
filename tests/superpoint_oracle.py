"""Plain torch restatements of SuperPoint's keypoint selection and descriptor sampling, used by the extractor tests.

nms_ref / select_ref follow the reference's formulas step for step (max-pool comparisons, two suppression rounds, the
border frame, `scores > threshold`, torch.topk when there are more than k candidates), so on the same fp32 score map
they give the same keypoints, scores and order.  sample_ref restates bilinear grid_sample (zeros padding) and the L2
normalisation in fp64.
"""
import numpy as np
import torch
import torch.nn.functional as F


def nms_ref(scores, radius):
    def pool(x):
        return F.max_pool2d(x, kernel_size=2 * radius + 1, stride=1, padding=radius)

    zeros = torch.zeros_like(scores)
    keep = scores == pool(scores)
    for _ in range(2):
        supp = pool(keep.float()) > 0
        s2 = torch.where(supp, zeros, scores)
        keep = keep | ((s2 == pool(s2)) & ~supp)
    return torch.where(keep, scores, zeros)


def border_ref(scores, rb, image_size=None):
    s = scores.clone()
    if rb:
        s[:, :rb] = -1
        s[:, :, :rb] = -1
        if image_size is not None:
            for i in range(s.shape[0]):
                w, h = image_size[i]
                s[i, int(h) - rb:] = -1
                s[i, :, int(w) - rb:] = -1
        else:
            s[:, -rb:] = -1
            s[:, :, -rb:] = -1
    return s


def select_ref(s, threshold, k):
    """Per image: (keypoints [n, 2] as (x, y) float, scores [n]), reference order; ties within topk by lower index."""
    out = []
    for b in range(s.shape[0]):
        ys, xs = torch.where(s[b] > threshold)
        sc = s[b][ys, xs]
        kp = torch.stack([xs, ys], -1).float()
        if 0 < k < len(sc):
            # descending score, then ascending row-major index (which torch.where order already is)
            order = sorted(range(len(sc)), key=lambda i: (-float(sc[i]), i))[:k]
            order = torch.tensor(order, dtype=torch.long)
            kp, sc = kp[order], sc[order]
        out.append((kp, sc))
    return out


def sample_ref(desc, kpts, legacy, s=8):
    """desc [B, C, h, w], kpts [B, K, 2] (x, y) score-map pixels -> [B, K, C], fp64."""
    desc = desc.double()
    kpts = kpts.double()
    B, C, h, w = desc.shape
    if legacy:
        k = (kpts - s / 2 + 0.5) / torch.tensor([w * s - s / 2 - 0.5, h * s - s / 2 - 0.5], dtype=torch.float64)
        k = k * 2 - 1
        ix, iy = (k[..., 0] + 1) / 2 * (w - 1), (k[..., 1] + 1) / 2 * (h - 1)
    else:
        k = kpts / (torch.tensor([w, h], dtype=torch.float64) * s) * 2 - 1
        ix, iy = ((k[..., 0] + 1) * w - 1) / 2, ((k[..., 1] + 1) * h - 1) / 2
    out = torch.zeros(B, kpts.shape[1], C, dtype=torch.float64)
    x0, y0 = torch.floor(ix), torch.floor(iy)
    for dx in (0, 1):
        for dy in (0, 1):
            xx, yy = x0 + dx, y0 + dy
            wt = (1 - (ix - xx).abs()) * (1 - (iy - yy).abs())
            ok = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
            xi, yi = xx.clamp(0, w - 1).long(), yy.clamp(0, h - 1).long()
            for b in range(B):
                v = desc[b][:, yi[b], xi[b]].T  # [K, C]
                out[b] += (wt[b] * ok[b])[:, None] * v
    return F.normalize(out, p=2, dim=-1)


def load_golden(path):
    g = dict(np.load(path))
    g["conf"] = __import__("json").loads(str(g["conf"]))
    return g


# ---- exact selection restatement, vectorised ------------------------------------------------------------------------
def select_ref_fast(s, threshold, k):
    """select_ref with numpy: candidates `s > threshold` in row-major order; when 0 < k < count, the first k of
    np.lexsort((index, -score)), i.e. descending score and, within exact ties, ascending row-major index."""
    W = s.shape[-1]
    out = []
    for b in range(s.shape[0]):
        v = s[b].detach().cpu().reshape(-1).numpy()
        idx = np.nonzero(v > np.float32(threshold))[0]
        sc = v[idx]
        if 0 < k < len(idx):
            order = np.lexsort((idx, -sc))[:k]
            idx, sc = idx[order], sc[order]
        kp = np.stack([idx % W, idx // W], -1).astype(np.float32).reshape(-1, 2)
        out.append((torch.from_numpy(kp), torch.from_numpy(np.ascontiguousarray(sc, dtype=np.float32))))
    return out


def tie_stats(s_b, threshold, k):
    """For one map with more than k candidates: (count of candidates equal to the k-th largest score, how many of those
    the top k takes, the 1024-pixel chunks the tie group touches).  The kernel gathers in 1024-pixel chunks, so a group
    that touches several chunks and is cut inside carries its row-major rank across chunks."""
    v = s_b.detach().cpu().reshape(-1).numpy()
    idx = np.nonzero(v > np.float32(threshold))[0]
    sc = v[idx]
    kth = np.sort(sc)[::-1][k - 1]
    eq = idx[sc == kth]
    taken = k - int((sc > kth).sum())
    return len(eq), taken, sorted(set((eq // 1024).tolist()))


# ---- comparisons ----------------------------------------------------------------------------------------------------
def bits(t):
    """The raw bits of a float tensor as integers (so -0.0 != 0.0 and NaN patterns compare)."""
    t = t.detach().contiguous()
    return t.view({torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float64: torch.int64}[t.dtype])


def assert_bits_equal(out, ref, tag=""):
    assert out.shape == ref.shape and out.dtype == ref.dtype, (tag, out.shape, ref.shape, out.dtype, ref.dtype)
    diff = bits(out) != bits(ref)
    if diff.any():
        i = int(torch.nonzero(diff.reshape(-1))[0])
        raise AssertionError(f"{tag}: {int(diff.sum())} of {diff.numel()} differ, first at flat index {i}: "
                             f"{out.reshape(-1)[i].item()!r} vs {ref.reshape(-1)[i].item()!r}")


def assert_within(out, ref, bound, tag=""):
    """|out - ref| <= bound element-wise (fp64), every output finite.  Returns the worst error-to-bound ratio."""
    out64 = out.detach().double()
    ref64, bound64 = ref.detach().double().to(out64.device), bound.detach().double().to(out64.device)
    assert out.shape == ref.shape == bound.shape, (tag, out.shape, ref.shape, bound.shape)
    assert torch.isfinite(out64).all(), f"{tag}: non-finite output"
    err = (out64 - ref64).abs()
    ratio = (err / bound64.clamp_min(1e-300)).max().item()
    if not bool((err <= bound64).all()):
        i = int(torch.argmax((err - bound64).reshape(-1)))
        raise AssertionError(f"{tag}: worst error-to-bound ratio {ratio:.3g}, at flat index {i}: "
                             f"out {out64.reshape(-1)[i].item()!r} ref {ref64.reshape(-1)[i].item()!r} "
                             f"bound {bound64.reshape(-1)[i].item():.3g}")
    return ratio


def assert_selection(kp, sc, cnt, ref, tag=""):
    """Kernel selection of one image (kp [cap, 2], sc [cap], cnt) against (kp_ref [n, 2], sc_ref [n]) truncated to cap:
    count, keypoints and scores of the kept slots bit for bit."""
    kp_ref, sc_ref = ref
    n = min(len(sc_ref), kp.shape[0])
    assert int(cnt) == n, f"{tag}: count {int(cnt)} vs {n}"
    assert_bits_equal(kp[:n].cpu(), kp_ref[:n], tag + " keypoints")
    assert_bits_equal(sc[:n].cpu(), sc_ref[:n], tag + " scores")


# ---- guarded outputs ------------------------------------------------------------------------------------------------
GUARD_BITS = {torch.float32: 0x7FA5A5A5, torch.bfloat16: 0x7FA5, torch.int32: 0x7FA5A5A5}  # NaN patterns
_INT = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.int32: torch.int32}


class Guarded:
    """`shape` elements between `guard` sentinel elements on each side, all set to a NaN bit pattern before the call;
    `.t` is the output view (16-byte aligned when `guard` keeps it so), `.check()` asserts both guards are intact and,
    with `full`, that every output element was written."""

    def __init__(self, shape, dtype, device, guard=64):
        n = 1
        for d in shape:
            n *= d
        self.n, self.guard, self.dtype = n, guard, dtype
        self.buf = torch.empty(n + 2 * guard, device=device, dtype=dtype)
        self.ibuf = self.buf.view(_INT[dtype])
        self.ibuf.fill_(GUARD_BITS[dtype])
        self.t = self.buf[guard:guard + n].view(shape)

    def check(self, tag="", full=True):
        pat = GUARD_BITS[self.dtype]
        g = self.guard
        assert bool((self.ibuf[:g] == pat).all()), f"{tag}: the guard before the output was overwritten"
        assert bool((self.ibuf[g + self.n:] == pat).all()), f"{tag}: the guard after the output was overwritten"
        if full:
            left = int((self.ibuf[g:g + self.n] == pat).sum())
            assert left == 0, f"{tag}: {left} output elements were never written"


# ---- derived error bounds -------------------------------------------------------------------------------------------
U = 2.0 ** -24       # fp32 unit roundoff (round to nearest)
U_ACC = 2.0 ** -23   # one fp32 accumulator add that may truncate
U_BF16 = 2.0 ** -8   # bf16 unit roundoff (8-bit significand)


def conv_acc_bound(mag, K):
    """fp32 accumulation of K products plus the bias add: each add may err by 2^-23 of a partial sum, and every partial
    sum is at most mag = conv(|x|, |w|) + |b|."""
    return (K + 1) * U_ACC * mag


def relu_bf16_bound(ref, acc_bound):
    """ReLU is 1-Lipschitz; the bf16 store rounds the fp32 value, itself within acc_bound of the exact one."""
    return acc_bound + U_BF16 * (ref.abs() + acc_bound)


def pool_bf16_bound(ref_pooled, acc_bound):
    """max of four values moves by at most the largest of the four inputs' errors; then the bf16 store."""
    e = F.max_pool2d(acc_bound, 2, 2)
    return e + U_BF16 * (ref_pooled.abs() + e)


def softmax_bound(logits, acc_bound):
    """logits, acc_bound [B, 65, h, w] fp64 -> (p [B, 64, h, w], bound).  Exact softmax: |dp_c| <= p_c (e^{2 dl} - 1)
    with dl = max_c |d logit_c|.  Arithmetic of p = expf(l - m) / sum expf(l - m) in fp32: the subtraction (u |l - m|),
    expf (2 ulp = 2^-22), the 65-term positive sum (64 u) and the division (u), relative to p."""
    p = F.softmax(logits, 1)
    dl = acc_bound.amax(1, keepdim=True)
    L = logits.amax(1, keepdim=True) - logits.amin(1, keepdim=True) + dl
    rel = torch.expm1(2 * dl) + 2 * (2.0 ** -22 + U * L) + 66 * U
    return p[:, :-1], (p * rel)[:, :-1] + 2.0 ** -126


def l2n_bound(y, acc_bound):
    """y, acc_bound [B, C, h, w] fp64 -> (y / |y|, bound).  |a/|a| - b/|b||_c <= (|d_c| + |b_c / |b|| |d|) / (|b| - |d|)
    for a = b + d; the kernel's sum of squares (8 terms per lane, then 5 shuffle levels), sqrt, reciprocal and product
    add at most 16 u relative to each output."""
    ny = y.norm(dim=1, keepdim=True)
    nE = acc_bound.norm(dim=1, keepdim=True)
    o = y / ny
    return o, (acc_bound + o.abs() * nE) / (ny - nE) + 16 * U * o.abs()


def sample_unnormalised(desc, kpts, legacy, s=8):
    """sample_ref without the final normalisation: desc [B, C, h, w] -> [B, K, C] fp64."""
    desc = desc.double()
    kpts = kpts.double()
    B, C, h, w = desc.shape
    if legacy:
        k = (kpts - s / 2 + 0.5) / torch.tensor([w * s - s / 2 - 0.5, h * s - s / 2 - 0.5], dtype=torch.float64)
        k = k * 2 - 1
        ix, iy = (k[..., 0] + 1) / 2 * (w - 1), (k[..., 1] + 1) / 2 * (h - 1)
    else:
        k = kpts / (torch.tensor([w, h], dtype=torch.float64) * s) * 2 - 1
        ix, iy = ((k[..., 0] + 1) * w - 1) / 2, ((k[..., 1] + 1) * h - 1) / 2
    out = torch.zeros(B, kpts.shape[1], C, dtype=torch.float64)
    x0, y0 = torch.floor(ix), torch.floor(iy)
    for dx in (0, 1):
        for dy in (0, 1):
            xx, yy = x0 + dx, y0 + dy
            wt = (1 - (ix - xx).abs()) * (1 - (iy - yy).abs())
            ok = (xx >= 0) & (xx < w) & (yy >= 0) & (yy < h)
            xi, yi = xx.clamp(0, w - 1).long(), yy.clamp(0, h - 1).long()
            for b in range(B):
                out[b] += (wt[b] * ok[b])[:, None] * desc[b][:, yi[b], xi[b]].T
    return out


def sample_bound(desc, kpts, legacy):
    """desc [B, C, h, w], kpts [B, K, 2] -> (sample_ref, element-wise bound) in fp64.

    The kernel's sample a differs from the exact a* at the fp32 keypoint by
      * the four fp32 weighted adds (and the weight product): 5 u sum_t wt_t |d_t| <= 5 u max|d|;
      * the sample coordinate: ix, iy come from five or six fp32 operations on values at most 2, scaled by w or h,
        so |d ix| <= 8 u (w + 1) and |d iy| <= 8 u (h + 1); bilinear interpolation is Lipschitz in each coordinate
        with constant max |d_i - d_j| <= 2 max|d| (across cell edges and the zero padding too).
    With E the resulting bound on |a - a*|_2, |a/|a| - a*/|a*||_c <= E (1 + |o_c|) / (|a*| - E), and the kernel's
    normalisation adds 16 u relative, as in l2n_bound."""
    B, C, h, w = desc.shape
    a = sample_unnormalised(desc, kpts, legacy)
    dmax = desc.double().norm(dim=1).max().item()
    E = 5 * U * dmax + 2 * dmax * 8 * U * ((w + 1) + (h + 1))
    na = a.norm(dim=-1, keepdim=True)
    o = a / na
    return o, E * (1 + o.abs()) / (na - E) + 16 * U * o.abs()


# ---- inputs ---------------------------------------------------------------------------------------------------------
def warp_zero_fill(img, seed, strength=0.15):
    """A random perspective warp of img [B, C, H, W] with zeros outside the source, as cv2.warpPerspective fills it:
    bilinear sampling of a homography that moves each corner by up to `strength` of the image size."""
    B, C, H, W = img.shape
    g = torch.Generator(device="cpu").manual_seed(seed)
    src = torch.tensor([[-1.0, -1.0], [1.0, -1.0], [1.0, 1.0], [-1.0, 1.0]], dtype=torch.float64)
    dst = src + (torch.rand(4, 2, generator=g, dtype=torch.float64) * 2 - 1) * 2 * strength
    A = []
    for (x, y), (u, v) in zip(dst.tolist(), src.tolist()):  # homography from output to input coordinates
        A.append([x, y, 1, 0, 0, 0, -u * x, -u * y])
        A.append([0, 0, 0, x, y, 1, -v * x, -v * y])
    h = torch.linalg.solve(torch.tensor(A, dtype=torch.float64), src.reshape(-1))
    Hm = torch.cat([h, torch.ones(1, dtype=torch.float64)]).reshape(3, 3)
    ys, xs = torch.meshgrid(torch.linspace(-1, 1, H, dtype=torch.float64), torch.linspace(-1, 1, W, dtype=torch.float64),
                            indexing="ij")
    p = torch.stack([xs, ys, torch.ones_like(xs)], -1) @ Hm.T
    grid = (p[..., :2] / p[..., 2:]).float()[None].expand(B, H, W, 2).to(img.device)
    return F.grid_sample(img, grid, mode="bilinear", padding_mode="zeros", align_corners=True)


# ---- score maps with plateaus ---------------------------------------------------------------------------------------
def blob_map(B, H, W, seed, levels=None, n=60):
    """Score-like maps in [0, 0.2): Gaussian bumps of radius 1.5 - 6 (drawn within 5 radii of their centre) over a
    faint floor; with `levels`, quantised to that many steps, so bump tops and the floor become plateaus of exactly
    equal scores."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    out = torch.empty(B, H, W, dtype=torch.float32)
    for b in range(B):
        m = 0.002 * torch.rand(H, W, generator=g, dtype=torch.float64)
        for _ in range(n):
            cy, cx = float(torch.rand(1, generator=g)) * H, float(torch.rand(1, generator=g)) * W
            s, a = 1.5 + 4.5 * float(torch.rand(1, generator=g)), 0.2 * float(torch.rand(1, generator=g))
            y0, y1 = max(0, int(cy - 5 * s)), min(H, int(cy + 5 * s) + 1)
            x0, x1 = max(0, int(cx - 5 * s)), min(W, int(cx + 5 * s) + 1)
            yy = torch.arange(y0, y1, dtype=torch.float64)[:, None]
            xx = torch.arange(x0, x1, dtype=torch.float64)[None, :]
            m[y0:y1, x0:x1] = torch.maximum(m[y0:y1, x0:x1],
                                            a * torch.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * s * s)))
        if levels:
            m = torch.floor(m * levels / 0.2) * (0.2 / levels)
        out[b] = m.float()
    return out


def region_map(B, H, W, seed, cell=37):
    """Piecewise-constant maps: `cell`-pixel blocks, each one of five values (0 included)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    vals = torch.tensor([0.0, 0.004, 0.0125, 0.05, 0.125], dtype=torch.float32)
    blocks = vals[torch.randint(0, 5, (B, (H + cell - 1) // cell, (W + cell - 1) // cell), generator=g)]
    return blocks.repeat_interleave(cell, 1).repeat_interleave(cell, 2)[:, :H, :W].contiguous()
