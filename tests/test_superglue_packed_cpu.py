"""CPU: the reference fixture of SuperGlue's packed evaluation (tests/golden/superglue_packed_l4.npz, eval mode) against
the fp64 eval-mode restatement, per pair, and the refusals of num_keypoints0/1 that need no device."""
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.superglue import SuperGlue
from tests import superglue_eval_oracle as O
from tests.util import GOLDEN


def test_fixture_against_fp64_eval_oracle():
    conf = {"GNN_layers": ["self", "cross"] * 2, "weights": None}
    g, conf, sd, pairs = O.load_fixture(GOLDEN, SuperGlue(conf).state_dict())
    w = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    assert any(p[0] != p[1] for p in pairs) and min(min(p[:2]) for p in pairs) == 1
    for i, (m, n, seed) in enumerate(pairs):
        data = synthetic.make_superglue_batch(1, m, n, seed, dtype=torch.float64)
        ref = O.superglue_forward_eval(w, data, conf)
        la = torch.from_numpy(g[f"p{i}|log_assignment"])
        assert la.shape == (m + 1, n + 1)
        assert (ref["log_assignment"][0] - la).abs().max() <= 1e-9 * la.abs().max(), (m, n)
        for k in ("matches0", "matches1"):
            assert torch.equal(ref[k][0], torch.from_numpy(g[f"p{i}|{k}"])), (m, n, k)
        for k in ("matching_scores0", "matching_scores1"):
            torch.testing.assert_close(ref[k][0], torch.from_numpy(g[f"p{i}|{k}"]), rtol=1e-9, atol=1e-12)
    assert sum(int((torch.from_numpy(g[f"p{i}|matches0"]) > -1).sum()) for i in range(len(pairs))) > 10


def _data(B=2, M=24, N=20):
    return synthetic.make_superglue_batch(B, M, N, 3)


@pytest.mark.parametrize("key,value,match", [
    ("num_keypoints0", torch.tensor([3.0, 4.0]), "integer"),
    ("num_keypoints1", torch.tensor([[1, 2]]), "shape"),
    ("num_keypoints1", torch.tensor([0, 5]), r"1 \.\. 20"),
    ("num_keypoints0", torch.tensor([25, 5]), r"1 \.\. 24"),
    ("num_keypoints0", [3, 4], "integer"),
])
def test_count_refusals(key, value, match):
    model = SuperGlue({"GNN_layers": ["self", "cross"], "weights": None}).eval()
    data = _data()
    data[key] = value
    with pytest.raises(ValueError, match=match):
        model(data)


def test_counts_refused_in_training_mode():
    model = SuperGlue({"GNN_layers": ["self", "cross"], "weights": None}).train()
    data = _data()
    data["num_keypoints1"] = torch.tensor([1, 2])
    with pytest.raises(ValueError, match="eval mode"):
        model(data)


def test_loss_refused_on_a_packed_pred():
    model = SuperGlue({"GNN_layers": ["self", "cross"], "weights": None}).eval()
    with pytest.raises(ValueError, match="num_keypoints0/1"):
        model.loss({"_b200_packed": True}, _data())
