"""CPU: labels as match lists instead of the [B, M, N] assignment mask.

1. Every shipped ground-truth golden holds one-to-one labels: the dense assignment equals the one-hot of matches0 and
   matches1 is its inverse, so the match lists carry everything the mask does.
2. fp64 restatements of the sparse loss terms and gradients (one gathered entry per row; dsim = gc (2 gt - softmax_row
   rowcnt - softmax_col colcnt) with gt from the list) against torch autograd of the reference's dense formulas
   (losses.py:6-25 weight_loss on lightglue.py's sigmoid log double softmax), with -1 / -2 labels, rows and pairs
   without positives, and M != N.
3. The consistency rule of ops.match_list_counts: equal positive counts per pair, NaN otherwise.
"""
import os

import numpy as np
import pytest
import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _tags(g):
    return sorted({k.split("|")[0] for k in g if k.endswith("|positives")})


@pytest.mark.parametrize("name", ["gt_homography", "gt_pose_depth", "gt_pose_depth_masks", "gt_lines_homography",
                                  "gt_lines_pose_depth"])
def test_golden_labels_are_one_to_one(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz"), allow_pickle=False))
    tags = _tags(g)
    assert tags
    for t in tags:
        m0, m1, p = g[f"{t}|matches0"], g[f"{t}|matches1"], g[f"{t}|positives"]
        B, M = m0.shape
        N = m1.shape[1]
        dense = np.zeros((B, M, N), bool)
        dense[p[:, 0], p[:, 1], p[:, 2]] = True
        onehot = np.zeros((B, M, N), bool)
        b, i = np.nonzero(m0 >= 0)
        onehot[b, i, m0[b, i]] = True
        assert np.array_equal(dense, onehot), (name, t)
        onehot1 = np.zeros((B, M, N), bool)
        b, j = np.nonzero(m1 >= 0)
        onehot1[b, m1[b, j], j] = True
        assert np.array_equal(dense, onehot1), (name, t)


def _lists(B, M, N, seed):
    g = torch.Generator().manual_seed(seed)
    m0 = torch.full((B, M), -1, dtype=torch.long)
    m1 = torch.full((B, N), -1, dtype=torch.long)
    for b in range(1, B):  # pair 0 has no positive
        k = int(torch.randint(0, min(M, N) + 1, (1,), generator=g))
        i, j = torch.randperm(M, generator=g)[:k], torch.randperm(N, generator=g)[:k]
        m0[b, i], m1[b, j] = j, i
    m0[(m0 < 0) & (torch.rand(B, M, generator=g) < 0.3)] = -2
    m1[(m1 < 0) & (torch.rand(B, N, generator=g) < 0.3)] = -2
    return m0, m1


def _dense(m0, N):
    B, M = m0.shape
    gt = torch.zeros(B, M, N, dtype=torch.float64)
    b, i = torch.nonzero(m0 >= 0, as_tuple=True)
    gt[b, i, m0[b, i]] = 1.0
    return gt


def _weight_loss(la, gt, m0, m1):
    """losses.py:6-25 with the weights of lightglue.py:598-603 (mask inside, unmatched indicators in the bins)."""
    B, M1, N1 = la.shape
    w = torch.zeros_like(la)
    w[:, :-1, :-1] = gt
    w[:, :-1, -1] = (m0 == -1).double()
    w[:, -1, :-1] = (m1 == -1).double()
    sc = la * w
    num_pos = w[:, :-1, :-1].sum((1, 2)).clamp(min=1.0)
    num_neg = (w[:, :-1, -1].sum(1) + w[:, -1, :-1].sum(1)).clamp(min=1.0)
    return -sc[:, :-1, :-1].sum((1, 2)) / num_pos, -(sc[:, :-1, -1].sum(1) + sc[:, -1, :-1].sum(1)) / num_neg


def _log_assignment(sim, z0, z1):
    """lightglue.py:256-269 (sigmoid_log_double_softmax) in fp64."""
    B, M, N = sim.shape
    ls0, ls1 = torch.nn.functional.logsigmoid(z0), torch.nn.functional.logsigmoid(z1)
    la = sim.new_zeros(B, M + 1, N + 1)
    la[:, :M, :N] = sim.log_softmax(2) + sim.log_softmax(1) + ls0[..., None] + ls1[:, None]
    la[:, :M, N] = torch.nn.functional.logsigmoid(-z0)
    la[:, M, :N] = torch.nn.functional.logsigmoid(-z1)
    return la


@pytest.mark.parametrize("B,M,N", [(3, 17, 29), (2, 40, 9), (4, 1, 6), (2, 33, 33)])
def test_sparse_formulas_match_dense_autograd(B, M, N):
    g = torch.Generator().manual_seed(M * 100 + N)
    sim = (3 * torch.randn(B, M, N, generator=g, dtype=torch.float64)).requires_grad_(True)
    z0 = torch.randn(B, M, generator=g, dtype=torch.float64)
    z1 = torch.randn(B, N, generator=g, dtype=torch.float64)
    m0, m1 = _lists(B, M, N, M + N)
    la = _log_assignment(sim, z0, z1)
    la.retain_grad()
    nll_pos, nll_neg = _weight_loss(la, _dense(m0, N), m0, m1)
    gpos = torch.randn(B, generator=g, dtype=torch.float64)
    (nll_pos * gpos + nll_neg).sum().backward()

    # sparse restatement: one gathered entry per row, counts from the lists
    pos = m0 >= 0
    j = m0.clamp(min=0)
    rowcnt, colcnt = pos.double(), (m1 >= 0).double()
    num_pos = rowcnt.sum(1).clamp(min=1.0)
    assert torch.equal(num_pos, (m1 >= 0).double().sum(1).clamp(min=1.0))
    s = sim.detach()
    lse_r, lse_c = s.logsumexp(2), s.logsumexp(1)
    pos_row_sum = torch.where(pos, 2 * s.gather(2, j[..., None])[..., 0] - lse_r - lse_c.gather(1, j),
                              torch.zeros_like(lse_r))
    ls0, ls1 = torch.nn.functional.logsigmoid(z0), torch.nn.functional.logsigmoid(z1)
    sparse_pos = -((pos_row_sum + rowcnt * ls0).sum(1) + (colcnt * ls1).sum(1)) / num_pos
    assert torch.allclose(sparse_pos, nll_pos.detach(), rtol=1e-12, atol=1e-12)
    # d nll_pos / d la: -1 / num_pos at (i, gt0[i]), nothing else in the inner block
    dla = torch.zeros(B, M, N, dtype=torch.float64)
    b, i = torch.nonzero(pos, as_tuple=True)
    dla[b, i, m0[b, i]] = -(gpos / num_pos)[b]
    gneg_part = la.grad[:, :-1, :-1] - dla
    assert torch.allclose(gneg_part, torch.zeros_like(gneg_part), atol=1e-12)
    # d nll_pos / d sim = gc (2 gt - softmax_row rowcnt - softmax_col colcnt) with gc = -g / num_pos (engine.py)
    gc = (-gpos / num_pos)[:, None, None]
    gt = _dense(m0, N)
    dsim = gc * (2 * gt - s.softmax(2) * rowcnt[..., None] - s.softmax(1) * colcnt[:, None])
    assert torch.allclose(sim.grad, dsim, rtol=1e-10, atol=1e-12)
    # the same gradient as rank-1 pieces: the positive entry is one index per row (and per column)
    dsim_sparse = gc * (-s.softmax(2) * rowcnt[..., None] - s.softmax(1) * colcnt[:, None])
    dsim_sparse[b, i, m0[b, i]] += 2 * gc[b, 0, 0]
    assert torch.allclose(dsim_sparse, dsim, rtol=0, atol=1e-15)


def test_match_list_counts_nan_on_disagreeing_lists():
    from gluefactory_b200 import ops

    m0, m1 = _lists(3, 20, 25, 7)
    rowcnt, colcnt, num_pos = ops.match_list_counts(m0, m1)
    assert torch.equal(num_pos, rowcnt.sum(1).clamp(min=1.0)) and torch.isfinite(num_pos).all()
    b = 1 if (m0[1] >= 0).any() else 2
    bad = m1.clone()
    bad[b, m0[b][m0[b] >= 0][0]] = -1
    _, _, num_bad = ops.match_list_counts(m0, bad)
    assert torch.isnan(num_bad[b]) and torch.isfinite(num_bad[torch.arange(3) != b]).all()
