"""CPU: the host side of GlueStick's packed batches (num_keypoints0/1, num_lines0/1): the endpoint-to-token map and the
junction order against plain restatements, and the count refusals that need no device."""
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.gluestick import GlueStick, endpoint_layout, junction_order


def test_endpoint_layout_against_plain_restatement():
    nl = torch.tensor([3, 0, 1, 5, 2])
    nk = torch.tensor([4, 9, 1, 20, 7])
    lined = torch.tensor([True, True, True, False, True])
    Lp = 6
    lsrc, lpid, esrc, epid, ssrc, bound = endpoint_layout(nl, nk, Lp, lined)
    want = {k: [] for k in ("lsrc", "lpid", "esrc", "epid", "ssrc", "bound")}
    for b in range(5):
        if not lined[b]:
            continue
        L = int(nl[b])
        for line in range(L):
            want["lsrc"].append(b * Lp + line)
            want["lpid"].append(b)
            for end in range(2):
                e = 2 * line + end
                want["esrc"].append(b * 2 * Lp + e)
                want["epid"].append(b)
                want["ssrc"].append(b * Lp + e % L)  # scores.repeat(1, 2): endpoint e takes line e % L's score
                want["bound"].append(min(int(nk[b]), 2 * L))
    for k, got in zip(want, (lsrc, lpid, esrc, epid, ssrc, bound)):
        assert got.tolist() == want[k], k


def test_junction_order_is_a_stable_sort():
    g = torch.Generator().manual_seed(0)
    tgt = torch.randint(0, 50, (400,), generator=g).int()
    order, srt = junction_order(tgt)
    plain = sorted(range(400), key=lambda e: (int(tgt[e]), e))  # by row, then endpoint order
    assert order.dtype == srt.dtype == torch.int32
    assert order.tolist() == plain
    assert srt.tolist() == [int(tgt[e]) for e in plain]


def _data(B=2, N=24, L=4):
    return synthetic.make_gluestick_batch(B, N, L, 3)


@pytest.mark.parametrize("key,value,match", [
    ("num_keypoints0", torch.tensor([3.0, 4.0]), "integer"),
    ("num_lines1", torch.tensor([[1, 2]]), "shape"),
    ("num_keypoints1", torch.tensor([0, 5]), r"1 \.\. 24"),
    ("num_keypoints0", torch.tensor([25, 5]), r"1 \.\. 24"),
    ("num_lines0", torch.tensor([-1, 2]), r"0 \.\. 4"),
    ("num_lines1", torch.tensor([5, 2]), r"0 \.\. 4"),
])
def test_count_refusals(key, value, match):
    model = GlueStick({"GNN_layers": ["self", "cross"]}).eval()
    data = _data()
    data[key] = value
    with pytest.raises(ValueError, match=match):
        model(data)


def test_counts_refused_in_training_mode():
    model = GlueStick({"GNN_layers": ["self", "cross"]}).train()
    data = _data()
    data["num_lines0"] = torch.tensor([1, 2])
    with pytest.raises(ValueError, match="eval mode"):
        model(data)


def test_loss_refused_on_a_packed_pred():
    model = GlueStick({"GNN_layers": ["self", "cross"]}).eval()
    with pytest.raises(ValueError, match="num_keypoints0/1"):
        model.loss({"_b200_packed": True}, _data())
