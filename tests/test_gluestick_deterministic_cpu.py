"""CPU: the junction layout GlueStick's fixed-order line kernels run on, against brute force, and the fp64 restatements
of their backward formulas (tests/gluestick_deterministic_oracle.py) against torch.autograd of the reference's own
formulas in fp64: the endpoint gather with its partner flip, the scatter-mean over junctions, and the line scores'
gathers + maximum, ties and NaN included.  No GPU: this pins the formulas the kernels implement independently of it."""
import pytest
import torch

from gluefactory_b200.matchers.gluestick import junction_layout
from tests import gluestick_deterministic_oracle as O


def _idx(B, L, n, seed):
    idx = O.wireframe_junctions(B, L, n, seed, hubs=((3, 4), (5, 3)), degenerate=(7, 9))
    return idx.reshape(B, 2 * L)


@pytest.mark.parametrize("B,L,n", [(3, 9, 20), (2, 9, 12), (1, 1, 1), (4, 13, 40)])
def test_junction_layout_matches_brute_force(B, L, n):
    """Shared junctions, a junction of degree >= 4, degenerate lines, node rows no line touches (rows 8.. at n = 20 /
    40), and fewer nodes than endpoints (n = 12 < 2 L: the heads' rows P = n)."""
    if n == 1:
        idx = torch.zeros(B, 2, dtype=torch.int64)
    else:
        idx = O.wireframe_junctions(B, L, n, 5 + B, hubs=((3, 4),), degenerate=(5,), pool=min(8, n, 2 * L))
        idx = idx.reshape(B, 2 * L)
    P = min(n, 2 * L)
    lay = junction_layout(idx, n, P)
    tgt, order, tgt_sorted, ptr = O.brute_layout(idx, n, P)
    assert all(t.dtype == torch.int32 for t in (lay.tgt, lay.order, lay.tgt_sorted, lay.junc, lay.ptr))
    assert torch.equal(lay.tgt.long(), tgt) and torch.equal(lay.order.long(), order)
    assert torch.equal(lay.tgt_sorted.long(), tgt_sorted) and torch.equal(lay.ptr.long(), ptr)
    assert torch.equal(lay.junc.long(), idx)
    if n > 1:
        deg = torch.bincount(idx[0], minlength=n)
        assert deg.max() >= 4 and (deg == 0).any()
    # every endpoint of pair b at junction r < P is listed under (b, r), in endpoint order
    for b in range(B):
        for r in range(P):
            got = lay.order[lay.ptr[b, r]:lay.ptr[b, r + 1]].tolist()
            assert got == [b * 2 * L + k for k in range(2 * L) if int(idx[b, k]) == r], (b, r)


def test_gather_backward_restatement_matches_autograd():
    """d x of the reference's endpoint gather [x[flat] ; flip] = per junction, the sum of its endpoints' first block and
    of their partners' second block (the partner flip folded into the reads)."""
    B, L, n, D = 3, 11, 30, 8
    idx = _idx(B, L, n, 1)
    x = torch.randn(B * n, D, dtype=torch.float64, requires_grad=True)
    out, flat = O.reference_line_layer_parts(x, idx, B)
    g = torch.randn_like(out)
    out.backward(g)
    lay = junction_layout(idx, n, min(n, 2 * L))
    got = O.junction_sum(g, lay.tgt, B * n, D)
    torch.testing.assert_close(got, x.grad, rtol=1e-12, atol=1e-12)
    assert torch.equal(lay.tgt.long(), flat)
    # the flip matters: without it the gradient differs wherever a line's ends sit at different junctions
    wrong = torch.zeros_like(got).index_add_(0, flat, g[:, :D] + g[:, D:])
    assert not torch.allclose(wrong, x.grad)


def test_mean_backward_restatement_matches_autograd():
    """x + scatter_reduce(mean, include_self=False): d x = g, d upd[e] = g[tgt[e]] / count(tgt[e])."""
    B, L, n, D = 2, 13, 40, 4
    idx = _idx(B, L, n, 2)
    lay = junction_layout(idx, n, min(n, 2 * L))
    x = torch.randn(B * n, D, dtype=torch.float64, requires_grad=True)
    upd = torch.randn(B * 2 * L, D, dtype=torch.float64, requires_grad=True)
    y = O.reference_junction_mean(x, upd, lay.tgt.long())
    g = torch.randn_like(y)
    y.backward(g)
    assert torch.equal(x.grad, g)
    torch.testing.assert_close(O.junction_mean_bwd(g, lay.tgt), upd.grad, rtol=0, atol=0)
    assert torch.bincount(lay.tgt.long()).max() >= 3


def _line_case(seed, L0=7, L1=5, P0=10, P1=9, G=2, integers=True):
    gen = torch.Generator().manual_seed(seed)
    # small integers make ties between the two endpoint orderings frequent and every sum exact in fp64
    sim = torch.randint(-3, 4, (G, P0, P1), generator=gen).double() if integers else \
        torch.randn(G, P0, P1, generator=gen, dtype=torch.float64)
    j0 = torch.randint(0, P0, (G, L0, 2), generator=gen)
    j1 = torch.randint(0, P1, (G, L1, 2), generator=gen)
    j0[:, 0, 1] = j0[:, 0, 0]  # degenerate lines
    j1[:, 1, 1] = j1[:, 1, 0]
    j0[:, 2:5, 0] = 4  # junction 4 of view 0 ends three more lines
    graw = torch.randint(-4, 5, (G, L0, L1), generator=gen).double()
    return sim, j0.reshape(G, -1), j1.reshape(G, -1), graw


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_line_score_backward_restatement_matches_autograd(seed):
    sim, j0, j1, graw = _line_case(seed)
    s = sim.clone().requires_grad_(True)
    raw = O.reference_line_scores(s, j0, j1)
    raw.backward(graw)
    assert torch.equal(O.line_scores(sim, j0, j1), raw.detach())
    got = O.line_scores_bwd(graw, sim, j0, j1)
    assert torch.equal(got, s.grad)  # every term and sum is exact here
    st = sim[0][j0[0, 0::2]][:, j1[0, 0::2]] + sim[0][j0[0, 1::2]][:, j1[0, 1::2]]
    sw = sim[0][j0[0, 0::2]][:, j1[0, 1::2]] + sim[0][j0[0, 1::2]][:, j1[0, 0::2]]
    assert (st == sw).sum() > 1  # ties (the degenerate lines among them) took part
    # lines past (m, n) take no part
    m, n = torch.tensor([5, 7]), torch.tensor([5, 3])
    s2 = sim.clone().requires_grad_(True)
    raw2 = O.reference_line_scores(s2, j0, j1)
    mask = (torch.arange(7)[None, :, None] < m[:, None, None]) & (torch.arange(5)[None, None, :] < n[:, None, None])
    raw2.backward(graw * mask)
    assert torch.equal(O.line_scores_bwd(graw, sim, j0, j1, m, n), s2.grad)


def test_line_score_tie_gives_half_to_each_ordering():
    """An exact tie between two different endpoint orderings: torch.maximum gives each branch half, so each of the
    four similarity entries receives a quarter of the raw score's gradient (first-wins would give two of them half)."""
    sim = torch.tensor([[[1.0, 2.0], [3.0, 4.0]]], dtype=torch.float64)  # s[0,0] + s[1,1] == s[0,1] + s[1,0]
    j = torch.tensor([[0, 1]])
    s = sim.clone().requires_grad_(True)
    O.reference_line_scores(s, j, j).backward(torch.tensor([[[8.0]]], dtype=torch.float64))
    assert torch.equal(s.grad, torch.full((1, 2, 2), 2.0, dtype=torch.float64))
    assert torch.equal(O.line_scores_bwd(torch.tensor([[[8.0]]]), sim, j, j), s.grad)
    # a degenerate line (both ends at junction 0) ties its orderings too
    s = sim.clone().requires_grad_(True)
    j0 = torch.tensor([[0, 0]])
    O.reference_line_scores(s, j0, j).backward(torch.tensor([[[8.0]]], dtype=torch.float64))
    assert torch.equal(O.line_scores_bwd(torch.tensor([[[8.0]]]), sim, j0, j), s.grad)


def test_line_score_nan_follows_torch_maximum():
    """A NaN on one branch: torch.maximum returns NaN and passes the gradient to both branches; an infinite gradient on
    a branch that takes none does not leak into it as inf * 0 = NaN."""
    sim = torch.tensor([[[float("nan"), 2.0], [3.0, 4.0]]], dtype=torch.float64)
    j = torch.tensor([[0, 1]])
    s = sim.clone().requires_grad_(True)
    raw = O.reference_line_scores(s, j, j)
    raw.backward(torch.tensor([[[8.0]]], dtype=torch.float64))
    assert torch.isnan(raw).all() and torch.isnan(O.line_scores(sim, j, j)).all()
    assert torch.equal(s.grad, torch.full((1, 2, 2), 4.0, dtype=torch.float64))
    assert torch.equal(O.line_scores_bwd(torch.tensor([[[8.0]]]), sim, j, j), s.grad)

    sim, j0, j1, graw = _line_case(7, integers=False)
    sim[0, int(j0[0, 6]), int(j1[0, 3])] = float("nan")
    graw[1, 0, 0] = float("inf")
    s = sim.clone().requires_grad_(True)
    raw = O.reference_line_scores(s, j0, j1)
    raw.backward(graw)
    ref = O.line_scores(sim, j0, j1)
    assert torch.equal(torch.isnan(ref), torch.isnan(raw.detach())) and torch.isnan(ref).any()
    got = O.line_scores_bwd(graw, sim, j0, j1)
    assert torch.isinf(s.grad).any() and not torch.isnan(s.grad).any()
    torch.testing.assert_close(got, s.grad, rtol=1e-12, atol=1e-12)
