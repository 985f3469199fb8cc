"""fp64 restatements of GlueStick's fixed-order LineLayer and line-head kernels (ops.JunctionGather, ops.JunctionMean,
ops.LineScores) and of the junction layout they run on, written from the formulas and not from the kernels' loops:
  * brute_layout: the JunctionLayout of one view by Python loops;
  * junction_sum: the backward of the endpoint gather [x[tgt[e]] ; x[tgt[e ^ 1]]];
  * junction_mean_bwd: the backward of the scatter-mean in upd;
  * line_scores / line_scores_bwd: raw = 0.5 * maximum(s[a0,c0] + s[a1,c1], s[a0,c1] + s[a1,c0]) and its gradient with
    torch.maximum's rule (the larger branch takes the gradient, each takes half on an exact tie, both take it when
    either is NaN, nothing leaks through a branch that takes none);
and the reference's own torch formulas (reference_line_layer_parts, reference_line_scores, gluestick.py:589-691 and
336-376), whose autograd pins the restatements on the CPU.  Everything works on CPU tensors."""
import torch


def brute_layout(idx, n, P):
    """(tgt, order, tgt_sorted, ptr) of one view by loops: idx [B, 2 L] junction indices, n nodes per pair, P the line
    heads' rows.  order: endpoints sorted by token row, ties by endpoint index; ptr [B, P + 1]."""
    B, E2 = idx.shape
    tgt = [b * n + int(idx[b, k]) for b in range(B) for k in range(E2)]
    order = sorted(range(len(tgt)), key=lambda e: (tgt[e], e))
    ptr = [[sum(1 for t in tgt if t < b * n + r) for r in range(P + 1)] for b in range(B)]
    return (torch.tensor(tgt), torch.tensor(order), torch.tensor([tgt[e] for e in order]), torch.tensor(ptr))


def reference_line_layer_parts(x, idx, B):
    """The reference's endpoint gather of one view (x [B*n, D], idx [B, 2L]): [x[flat] ; the other end's] [E, 2D]."""
    D, n, n2 = x.shape[1], x.shape[0] // B, idx.shape[1]
    flat = (idx + torch.arange(B)[:, None] * n).reshape(-1)
    ld = x.index_select(0, flat)
    other = ld.view(B, n2 // 2, 2, D).flip(2).reshape(B * n2, D)
    return torch.cat([ld, other], 1), flat


def reference_junction_mean(x, upd, flat):
    D = x.shape[1]
    return x + torch.zeros_like(x).scatter_reduce(0, flat[:, None].expand(-1, D), upd, reduce="mean", include_self=False)


def junction_sum(src, tgt, T, D):
    """dx [T, D] with dx[r] = sum over endpoints e with tgt[e] == r of src[e, :D] + src[e ^ 1, D:2D]."""
    src = src.double()
    partner = torch.arange(tgt.numel()) ^ 1
    return torch.zeros(T, D, dtype=torch.float64).index_add_(0, tgt.long(), src[:, :D] + src[partner, D:2 * D])


def junction_mean_bwd(g, tgt):
    """d upd [E, D] = g[tgt[e]] / (number of endpoints at tgt[e])."""
    cnt = torch.bincount(tgt.long(), minlength=g.shape[0]).to(g.dtype)
    return g[tgt.long()] / cnt[tgt.long()][:, None]


def reference_line_scores(s, idx0, idx1):
    """gluestick.py:348-361 on s [B, P0, P1]: the two gathers, the two sums, maximum, scale."""
    B = s.shape[0]
    n20, n21 = idx0.shape[1], idx1.shape[1]
    s = torch.gather(s, 2, idx1[:, None, :].expand(B, s.shape[1], n21))
    s = torch.gather(s, 1, idx0[:, :, None].expand(B, n20, n21)).reshape(B, n20 // 2, 2, n21 // 2, 2)
    return 0.5 * torch.maximum(s[:, :, 0, :, 0] + s[:, :, 1, :, 1], s[:, :, 0, :, 1] + s[:, :, 1, :, 0])


def line_scores(sim, junc0, junc1):
    return reference_line_scores(sim.double(), junc0.long(), junc1.long())


def line_scores_bwd(graw, sim, junc0, junc1, m=None, n=None, absolute=False):
    """d sim [G, P0, P1] fp64 for graw [G, L0, L1]; lines i >= m[g] / j >= n[g] take no part.  absolute: the sum of the
    contributions' magnitudes instead (the scale of an fp32 summation's rounding)."""
    sim, graw = sim.double(), graw.double()
    G, P0, P1 = sim.shape
    L0, L1 = junc0.shape[1] // 2, junc1.shape[1] // 2
    out = torch.zeros(G, P0, P1, dtype=torch.float64)
    for g in range(G):
        a, c = junc0[g].long().view(L0, 2), junc1[g].long().view(L1, 2)
        S = sim[g]
        st = S[a[:, 0]][:, c[:, 0]] + S[a[:, 1]][:, c[:, 1]]
        sw = S[a[:, 0]][:, c[:, 1]] + S[a[:, 1]][:, c[:, 0]]
        tie = st == sw
        w_st = torch.where(tie, 0.5, torch.where(st < sw, 0.0, 1.0)).double()
        w_sw = torch.where(tie, 0.5, torch.where(st > sw, 0.0, 1.0)).double()
        d = 0.5 * graw[g]
        keep = torch.ones(L0, L1, dtype=torch.bool)
        if m is not None:
            keep = (torch.arange(L0)[:, None] < int(m[g])) & (torch.arange(L1)[None, :] < int(n[g]))
        c_st = torch.where((w_st == 0) | ~keep, 0.0, d * w_st)
        c_sw = torch.where((w_sw == 0) | ~keep, 0.0, d * w_sw)
        if absolute:
            c_st, c_sw = c_st.abs(), c_sw.abs()
        for (p, q), contrib in (((0, 0), c_st), ((1, 1), c_st), ((0, 1), c_sw), ((1, 0), c_sw)):
            rows = a[:, p][:, None].expand(L0, L1)
            cols = c[:, q][None, :].expand(L0, L1)
            out[g].index_put_((rows.reshape(-1), cols.reshape(-1)), contrib.reshape(-1), accumulate=True)
    return out


def wireframe_junctions(B, L, n, seed, hubs=((3, 8), (7, 5)), degenerate=(13, 14), pool=None):
    """lines_junc_idx [B, L, 2] of a wireframe with shared junctions: endpoints drawn from `pool` (default: 2 L / 2.5)
    junction nodes, so most junctions end two or more lines; junction h ends lines 0.. of each (h, k) in `hubs` (degree
    >= k); the lines in `degenerate` have both ends at one junction; nodes from `pool` up to n are no line's junction."""
    gen = torch.Generator().manual_seed(seed)
    pool = pool or max(4, int(2 * L / 2.5))
    assert pool <= min(n, 2 * L)
    idx = torch.randint(0, pool, (B, L, 2), generator=gen)
    start = 0
    for h, k in hubs:
        idx[:, start:start + k, start % 2] = h
        start += k
    for l in degenerate:
        if l < L:
            idx[:, l, 1] = idx[:, l, 0]
    return idx
