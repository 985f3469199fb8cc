"""Plain torch restatement of the O(M N) point-label pass of the pose + depth ground truth
(gluefactory/geometry/gt_generation.py:46-91, geometry/epipolar.py:59-72), written from its behaviour; the GPU tests
compare csrc/gt.cu against it at sizes where no golden file exists, and tests/test_gt_points_oracle_cpu.py pins it to
the reference's own labels (tests/golden/gt_pose_depth*.npz).

Dense and device-agnostic, one batch element at a time (three [M, N] matrices live at once, 48 MB at 2048 x 2048).
Distances use the elementwise fp32 order of the reference (`(a - b) ** 2` summed over the last axis, `torch.max`,
`torch.where(mask, dist, inf)`).  Argmin ties are resolved here, explicitly, as "lowest index" and a NaN as the
minimum (first NaN) -- what `Tensor.min` does on the CPU, where the reference's labels were produced, but not a
documented property of it on other devices.
"""
import torch

IGNORE, UNMATCHED = -2, -1


def first_min_index(d, dim):
    """Index of the minimum along `dim`, the lowest index among equal values; a NaN counts as the minimum (the first
    NaN wins), as in torch's CPU `min`.  An all-inf slice gives index 0."""
    nan = torch.isnan(d)
    hit = torch.where(nan.any(dim, keepdim=True), nan, d == d.min(dim, keepdim=True).values)
    return hit.to(torch.uint8).argmax(dim)  # argmax returns the first maximal value


def labels_from_reprojection(kp0, kp1, kp0_1, kp1_0, visible0=None, visible1=None, valid0=None, valid1=None,
                             pos_th=3.0, neg_th=5.0):
    """kp0 [B,M,2], kp1 [B,N,2], kp0_1 = kp0 projected into view 1, kp1_0 the converse; visible* / valid* bool [B,M] /
    [B,N] or None (= all true).  -> assignment bool [B,M,N], m0 [B,M], m1 [B,N] int64 (index, -1 unmatched, -2 ignored).

    A pair's distance is the larger of its two squared reprojection errors, +inf unless both points are visible in the
    other view.  Positives: mutual nearest neighbours below pos_th^2.  Unmatched: best one-way reprojection error
    (over ALL partners, visible or not) above neg_th^2, and a valid depth.  Everything else is ignored."""
    B = kp0.shape[0]
    asg, m0s, m1s = [], [], []
    for b in range(B):
        d0 = ((kp0_1[b, :, None] - kp1[b, None]) ** 2).sum(-1)
        d1 = ((kp0[b, :, None] - kp1_0[b, None]) ** 2).sum(-1)
        dist = torch.max(d0, d1)
        if visible0 is not None:
            dist = torch.where(visible0[b].bool()[:, None] & visible1[b].bool()[None], dist, dist.new_tensor(float("inf")))
        min0, min1 = first_min_index(dist, 1), first_min_index(dist, 0)
        ismin0 = torch.zeros_like(dist, dtype=torch.bool).scatter_(1, min0[:, None], True)
        ismin1 = torch.zeros_like(dist, dtype=torch.bool).scatter_(0, min1[None], True)
        positive = ismin0 & ismin1 & (dist < pos_th ** 2)
        neg0, neg1 = d0.min(1).values > neg_th ** 2, d1.min(0).values > neg_th ** 2
        if valid0 is not None:
            neg0, neg1 = neg0 & valid0[b].bool(), neg1 & valid1[b].bool()
        m0 = torch.where(positive.any(1), min0, torch.full_like(min0, IGNORE))
        m1 = torch.where(positive.any(0), min1, torch.full_like(min1, IGNORE))
        m0s.append(torch.where(neg0, torch.full_like(m0, UNMATCHED), m0))
        m1s.append(torch.where(neg1, torch.full_like(m1, UNMATCHED), m1))
        asg.append(positive)
    return torch.stack(asg), torch.stack(m0s), torch.stack(m1s)


def epipolar_distance_all(kp0, kp1, F, dtype=torch.float64, eps=1e-15):
    """Symmetric epipolar distance of every pair, [B,M,N]: |b^T F a| averaged over its two normalisations, the norm of
    the first two coordinates of F a (the line of a in view 1) and of F^T b (the line of b in view 0)."""
    a = torch.cat([kp0, torch.ones_like(kp0[..., :1])], -1).to(dtype)   # [B,M,3]
    bq = torch.cat([kp1, torch.ones_like(kp1[..., :1])], -1).to(dtype)  # [B,N,3]
    F = F.to(dtype)
    Fa = a @ F.transpose(-1, -2)   # [B,M,3]: F a
    Ftb = bq @ F                   # [B,N,3]: F^T b
    num = (Fa @ bq.transpose(-1, -2)).abs()
    n0 = (Fa[..., 0] ** 2 + Fa[..., 1] ** 2 + eps).sqrt()[:, :, None]
    n1 = (Ftb[..., 0] ** 2 + Ftb[..., 1] ** 2 + eps).sqrt()[:, None, :]
    return (num / n0 + num / n1) / 2


def epipolar_unmatched(m0, m1, valid0, valid1, epi, th):
    """A point without valid depth whose label is still "ignored" becomes unmatched when every still-ignored point of
    the other view is further than `th` from it in `epi` (no such partner at all: min over nothing = inf > th).  Both
    views are judged on the labels before the update.  -> new m0, new m1, and the minimum distance per point over its
    still-ignored partners, min0 [B,M], min1 [B,N]."""
    ign0, ign1 = m0 == IGNORE, m1 == IGNORE
    masked = torch.where(ign0[:, :, None] & ign1[:, None, :], epi, epi.new_tensor(float("inf")))
    min0, min1 = masked.min(2).values, masked.min(1).values
    new0 = torch.where(ign0 & ~valid0.bool() & (min0 > th), torch.full_like(m0, UNMATCHED), m0)
    new1 = torch.where(ign1 & ~valid1.bool() & (min1 > th), torch.full_like(m1, UNMATCHED), m1)
    return new0, new1, min0, min1
