"""CPU: the packed layout LightGlue builds from `num_keypoints0/1` (segments, index maps, source rows) against a plain
restatement, the layout of equal counts against the uniform packing of the adaptive forward, and the refusals that
need no device."""
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.lightglue import LightGlue, keypoint_counts, ragged_layout, segment_rows


def _restated(n0, n1, M, N):
    """Pair by pair: the tokens are [image 0 of every pair; image 1 of every pair]."""
    B = len(n0)
    seg = [[0] * (2 * B) for _ in range(4)]
    ind, src0, src1, pid0, pid1 = [], [], [], [], []
    t = 0
    for b in range(B):
        seg[0][2 * b], seg[1][2 * b] = t, n0[b]
        ind += list(range(n0[b]))
        src0 += [b * M + i for i in range(n0[b])]
        pid0 += [b] * n0[b]
        t += n0[b]
    for b in range(B):
        seg[0][2 * b + 1], seg[1][2 * b + 1] = t, n1[b]
        ind += list(range(n1[b]))
        src1 += [b * N + j for j in range(n1[b])]
        pid1 += [b] * n1[b]
        t += n1[b]
    for s in range(2 * B):
        seg[2][s], seg[3][s] = seg[0][s ^ 1], seg[1][s ^ 1]
    return seg, ind, src0, src1, pid0, pid1


@pytest.mark.parametrize("n0,n1,M,N", [([1], [1], 1, 1), ([5, 1, 64, 65], [128, 129, 1, 7], 70, 130),
                                        ([2048, 1, 1000], [1, 2048, 999], 2048, 2048), ([3] * 300, [4] * 300, 3, 9)])
def test_layout_against_restatement(n0, n1, M, N):
    lay = ragged_layout(torch.tensor(n0), torch.tensor(n1), M, N)
    seg, ind, src0, src1, pid0, pid1 = _restated(n0, n1, M, N)
    assert lay.seg.dtype == torch.int32 and lay.ind.dtype == torch.int32
    assert lay.seg.tolist() == seg and lay.ind.tolist() == ind
    assert lay.src0.tolist() == src0 and lay.src1.tolist() == src1
    assert lay.pid0.tolist() == pid0 and lay.pid1.tolist() == pid1


def test_equal_counts_give_the_uniform_packing():
    """Full counts lay the tokens out as the adaptive forward always has: pair b's views at b M and B M + b N."""
    B, M, N = 3, 5, 7
    lay = ragged_layout(torch.full((B,), M), torch.full((B,), N), M, N)
    off = torch.stack([torch.arange(B) * M, B * M + torch.arange(B) * N], 1).reshape(-1)
    ln = torch.tensor([M, N]).repeat(B)
    seg = torch.stack([off, ln, off.view(B, 2).flip(1).reshape(-1), ln.view(B, 2).flip(1).reshape(-1)])
    assert torch.equal(lay.seg, seg.int())
    assert torch.equal(lay.ind, torch.cat([torch.arange(M).repeat(B), torch.arange(N).repeat(B)]).int())


def test_segment_rows():
    rows, k, i = segment_rows(torch.tensor([10, 0, 50]), torch.tensor([2, 0, 3]))
    assert rows.tolist() == [10, 11, 50, 51, 52] and k.tolist() == [0, 0, 2, 2, 2] and i.tolist() == [0, 1, 0, 1, 2]


def _data(B=2, M=6, N=5):
    return {"keypoints0": torch.rand(B, M, 2), "keypoints1": torch.rand(B, N, 2), "descriptors0": torch.rand(B, M, 256),
            "descriptors1": torch.rand(B, N, 256)}


def test_counts_parsing():
    d = _data()
    assert keypoint_counts(d, 2, 6, 5) is None
    n0, n1 = keypoint_counts(dict(d, num_keypoints1=torch.tensor([1, 5], dtype=torch.int16)), 2, 6, 5)
    assert n0.tolist() == [6, 6] and n1.tolist() == [1, 5] and n0.dtype == n1.dtype == torch.int64


@pytest.mark.parametrize("bad,msg", [(torch.tensor([0, 3]), "1 .. 6"), (torch.tensor([7, 3]), "1 .. 6"),
                                     (torch.tensor([-1, 3]), "1 .. 6"), (torch.tensor([2.0, 3.0]), "integer"),
                                     (torch.tensor([True, True]), "integer"), ([2, 3], "integer"),
                                     (torch.tensor([2, 3, 4]), "shape"), (torch.tensor([[2, 3]]), "shape")])
def test_refusals_without_a_device(bad, msg):
    model = LightGlue(dict(synthetic.DEFAULT_CONF, n_layers=2)).eval()
    with pytest.raises(ValueError, match=msg):
        model(dict(_data(), num_keypoints0=bad))


def test_counts_refused_in_training_mode():
    model = LightGlue(dict(synthetic.DEFAULT_CONF, n_layers=2)).train()
    with pytest.raises(ValueError, match="eval mode"):
        model(dict(_data(), num_keypoints0=torch.tensor([3, 6])))
