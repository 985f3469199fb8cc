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
