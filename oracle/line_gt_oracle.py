"""CPU restatement of the line ground truth (gluefactory/geometry/gt_generation.py:164-558) and of the linear
assignment it solves with scipy, written from the math; the GPU tests compare csrc/gt_lines.cu against it (the GPU
machines have neither the reference nor, necessarily, scipy).

`line_labels` starts from the clamped segments and the projected sample points (the reference's own, stored in the
fixtures, or any others) and follows the reference step by step in torch on the CPU, pair by pair and in chunks of
segments, so no [B, L0, L1, npts] tensor is built.  The rotation into a segment's frame is evaluated as
fma(R[j,1], c1, R[j,0] * c0) -- the rounding of torch.einsum on the CPU (:198) -- with the product exact in float64.
"""
import numpy as np
import torch


def linear_sum_assignment(cost):
    """Shortest augmenting path (Crouse's rectangular variant of Jonker-Volgenant), with the tie rules of scipy's
    linear_sum_assignment: columns are scanned from a `remaining` list that starts reversed and loses its picked entry
    by a move of the last one; among equal path costs the last unassigned column in that order wins, else the first.
    Returns (rows, cols) sorted by row, as scipy does."""
    C = np.asarray(cost, dtype=np.float64)
    tr = C.shape[0] > C.shape[1]
    if tr:
        C = C.T
    nr, nc = C.shape
    u, v = np.zeros(nr), np.zeros(nc)
    col4row, row4col = np.full(nr, -1), np.full(nc, -1)
    for cur in range(nr):
        shortest, path = np.full(nc, np.inf), np.full(nc, -1)
        SR, SC = np.zeros(nr, bool), np.zeros(nc, bool)
        remaining = list(range(nc - 1, -1, -1))
        minval, i, sink = 0.0, cur, -1
        while sink < 0:
            SR[i] = True
            rem = np.asarray(remaining)
            r = minval + C[i, rem] - u[i] - v[rem]
            upd = r < shortest[rem]
            shortest[rem[upd]] = r[upd]
            path[rem[upd]] = i
            sh = shortest[rem]
            lowest = sh.min()
            cand = np.flatnonzero(sh == lowest)
            free = cand[row4col[rem[cand]] == -1]
            index = free[-1] if len(free) else cand[0]
            minval, j = lowest, rem[index]
            SC[j] = True
            remaining[index] = remaining[-1]
            remaining.pop()
            if row4col[j] == -1:
                sink = j
            else:
                i = row4col[j]
        u[cur] += minval
        others = np.flatnonzero(SR)
        others = others[others != cur]
        u[others] += minval - shortest[col4row[others]]
        v[SC] -= minval - shortest[SC]
        j = sink
        while True:
            i = path[j]
            row4col[j] = i
            col4row[i], j = j, col4row[i]
            if i == cur:
                break
    if tr:
        order = np.argsort(col4row)
        return col4row[order], order
    return np.arange(nr), col4row


def sample_pts(segs, npts):
    """segs [..., 4] -> [..., npts, 2] (:164-170)."""
    d = (segs[..., 2:4] - segs[..., :2]) / (npts - 1)
    return (segs[..., :2, None] + d[..., None] * torch.arange(npts).to(segs)).transpose(-1, -2)


def _fma32(a, b, c):
    """fp32 fma(a, b, c): the product is exact in float64."""
    return (a.double() * b.double() + c.double()).float()


def close_counts(segs, pts, dist_th, weight=None, chunk=64):
    """segs [La,4], pts [Lb,npts,2] -> int64 [La, Lb]: points of each b-line within dist_th of segment a and
    overlapping it (torch_perp_dist, :173-204, and :309-316), weighted by `weight` [Lb,npts] (bool) when given."""
    d = segs[:, 2:] - segs[:, :2]
    size = torch.norm(d, dim=-1).half()
    nd = d / size[:, None]
    size = size.float()
    out = []
    for s in range(0, segs.shape[0], chunk):
        c = pts[None] - segs[s:s + chunk, None, None, 2:]
        n0, n1 = nd[s:s + chunk, 0, None, None], nd[s:s + chunk, 1, None, None]
        r0 = _fma32(n1, c[..., 1], n0 * c[..., 0])
        r1 = _fma32(n0, c[..., 1], (-n1) * c[..., 0])
        close = (r1.abs() < dist_th) & (r0 <= 0) & (r0.abs() <= size[s:s + chunk, None, None])
        if weight is not None:
            close = close & weight[None]
        out.append(close.sum(-1))
    return torch.cat(out)


def _outside(pts, h, w, npts, mvt):
    out = (pts < 0).any(-1) | (pts >= torch.tensor([w, h]).to(pts)).any(-1)
    return out.reshape(-1, npts).float().mean(-1) >= (1 - mvt)


def line_labels(segs0, segs1, pts0_1, pts1_0, size0, size1, valid_lines0, valid_lines1, visible0=None, visible1=None,
                valid_pts0=None, valid_pts1=None, npts=50, dist_th=5, overlap_th=0.2, min_visibility_th=0.5):
    """Batched CPU labels.  segs [B,L,4] clamped, pts0_1 [B,L0*npts,2] (view-0 points in view 1, image size1 = (h, w)),
    masks [B,L*npts] or None (homography variant).  Returns dict: positive bool [B,L0,L1], m0, m1 int64, cost int64
    [B,L0,L1], and the assignment (rows, cols) per pair."""
    depth = visible0 is not None
    B, L0, L1 = segs0.shape[0], segs0.shape[1], segs1.shape[1]
    (h0, w0), (h1, w1) = size0, size1
    res = {"positive": [], "m0": [], "m1": [], "cost": [], "assignment": []}
    for b in range(B):
        p01, p10 = pts0_1[b].reshape(L0, npts, 2), pts1_0[b].reshape(L1, npts, 2)
        vis0 = visible0[b].reshape(L0, npts) if depth else None
        vis1 = visible1[b].reshape(L1, npts) if depth else None
        out_of0 = _outside(p10, h0, w0, npts, min_visibility_th)  # [L1]
        out_of1 = _outside(p01, h1, w1, npts, min_visibility_th)  # [L0]
        c0 = close_counts(segs0[b], p10, dist_th, vis1)        # [L0, L1]
        c1t = close_counts(segs1[b], p01, dist_th, vis0).t()   # [L0, L1]
        num = c0 * c1t
        if depth:
            mask = (c1t > vis0.float().sum(-1)[:, None] * overlap_th) & (c0 > vis1.float().sum(-1)[None] * overlap_th)
        else:
            mask = (c1t > npts * overlap_th) & (c0 > npts * overlap_th) & ~out_of0[None] & ~out_of1[:, None]
        unmatched0 = ~mask.any(1) | out_of1
        unmatched1 = ~mask.any(0) | out_of0
        ignore0, ignore1 = ~valid_lines0[b].bool(), ~valid_lines1[b].bool()
        if depth:
            ignore0 = ignore0 | (valid_pts0[b].reshape(L0, npts).float().mean(-1) < min_visibility_th)
            ignore1 = ignore1 | (valid_pts1[b].reshape(L1, npts).float().mean(-1) < min_visibility_th)
        cost = -num
        cost[unmatched0 | ignore0] = 1000000
        cost[:, unmatched1 | ignore1] = 1000000
        rows, cols = linear_sum_assignment(cost.numpy())
        rows, cols = torch.from_numpy(np.asarray(rows)).long(), torch.from_numpy(np.asarray(cols)).long()
        pos = torch.zeros(L0, L1, dtype=torch.bool)
        pos[rows, cols] = True
        pos = pos & mask
        pos[unmatched0 | ignore0] = False
        pos[:, unmatched1 | ignore1] = False
        m0 = torch.full((L0,), -1, dtype=torch.long).scatter_(0, rows, cols)
        m1 = torch.full((L1,), -1, dtype=torch.long).scatter_(0, cols, rows)
        m0[~pos.any(1) | unmatched0] = -1
        m0[ignore0] = -2
        m1[~pos.any(0) | unmatched1] = -1
        m1[ignore1] = -2
        for k, val in (("positive", pos), ("m0", m0), ("m1", m1), ("cost", cost), ("assignment", (rows, cols))):
            res[k].append(val)
    return {k: (v if k == "assignment" else torch.stack(v)) for k, v in res.items()}
