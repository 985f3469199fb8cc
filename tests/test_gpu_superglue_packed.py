"""GPU: SuperGlue inference on batches of pairs with their own keypoint counts (`num_keypoints0/1`, eval mode).

The packed Sinkhorn kernel (ops.log_optimal_transport_varlen) over 300+ pairs of lengths 1-2048, at 0, 1 and 50
iterations: a batch is bit-identical to its pairs sent one at a time, matches the uniform kernel on [1, m, n] (1e-5
relative, equal argmaxes) and an fp64 restatement of superglue.py:186-214, never reads the padding of sim, and keeps
every entry of its output it does not own.

The plugin: each pair of one packed call must get what a one-pair call on its truncated inputs returns, in the padded
original indexing:
  * against packed calls made one pair at a time: bf16 bit-identical, fp32 equal matches and log-assignments within 1e-5;
  * against the uniform one-pair path, and for the reference fixture's pairs (tests/golden/superglue_packed_l4.npz)
    inside one NaN-padded call against the fp64 reference, at tests/test_gpu_superglue.py's bounds per precision;
  * NaN / Inf padding changes no output bit; out-of-range valid keypoints and `loss` on a packed pred are refused."""
import math

import pytest
import torch

from gluefactory_b200 import ops, synthetic
from gluefactory_b200.matchers.superglue import SuperGlue
from oracle.lightglue_oracle import log_optimal_transport as lot64
from tests import superglue_eval_oracle as O
from tests.util import GOLDEN, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
KEYS = ["keypoints", "descriptors", "keypoint_scores"]
SENTINEL = 7.25
BIN = 0.9
# per precision, the bounds of tests/test_gpu_superglue.py against the fp64 reference (log-assignment, relative)
BOUND = {"fp32": 1e-4, "bf16": 5e-3}


# ---------------------------------------------------------------------------------------------- kernel
def _kernel_batches():
    """Two launches' worth of pairs: the long and edge lengths padded to 2048, and 300 short pairs padded to 160."""
    big = [(1, 1), (1, 2048), (2048, 1), (2048, 2048), (31, 33), (33, 31), (32, 32), (127, 129), (129, 127),
           (128, 128), (300, 257), (1000, 31), (64, 1500)]
    r = torch.Generator().manual_seed(1)
    small = [(int(a), int(b)) for a, b in torch.randint(1, 161, (300, 2), generator=r)]
    small += [(31, 32), (33, 32), (127, 128), (129, 128), (160, 1), (1, 160)]
    return {"big": big, "small": small}


def _sim(lens, fill, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    M, N = max(m for m, _ in lens), max(n for _, n in lens)
    sim = torch.full((len(lens), M, N), fill, device=DEV)
    for i, (m, n) in enumerate(lens):
        sim[i, :m, :n] = 3 * torch.randn(m, n, device=DEV, generator=g)
    return sim


def _run_varlen(sim, lens, iters, rows, Bo, Mo, No):
    out = torch.full((Bo, Mo + 1, No + 1), SENTINEL, device=DEV)
    pairs = torch.stack([torch.tensor([m for m, _ in lens]), torch.tensor([n for _, n in lens]), rows]).to(DEV).int()
    return ops.log_optimal_transport_varlen(sim, torch.tensor(BIN, device=DEV), iters, pairs, out)


def _own(got, m, n, Mo, No):
    """Pair block of a packed output row in the one-pair [m + 1, n + 1] form."""
    r = torch.cat([torch.arange(m), torch.tensor([Mo])]).to(got.device)
    c = torch.cat([torch.arange(n), torch.tensor([No])]).to(got.device)
    return got[r][:, c]


def _argmax_agree(a, b, dim):
    """Equal argmax of a and b along dim, except where b's top two are within 1e-5 of each other (a near-tie)."""
    ia, ib = a.argmax(dim), b.argmax(dim)
    if torch.equal(ia, ib):
        return True
    bad = (ia != ib).nonzero()
    va = b.gather(dim, ia.unsqueeze(dim)).squeeze(dim)
    vb = b.gather(dim, ib.unsqueeze(dim)).squeeze(dim)
    return bool(((vb - va).abs()[ia != ib] < 1e-5 * vb.abs()[ia != ib].clamp(min=1)).all()) and bad.shape[0] <= 2


@pytest.mark.parametrize("iters", [0, 1, 50])
@pytest.mark.parametrize("which", ["big", "small"])
def test_varlen_sinkhorn_kernel(which, iters):
    lens = _kernel_batches()[which]
    G = len(lens)
    sim = _sim(lens, float("nan"), seed=7 + G)
    M, N = sim.shape[1:]
    Bo, Mo, No = G + 3, M + 2, N + 5
    rows = torch.randperm(Bo, generator=torch.Generator().manual_seed(2))[:G]
    out = _run_varlen(sim, lens, iters, rows, Bo, Mo, No)
    # NaN or Inf in the padding of sim changes no output bit
    for fill in (float("inf"), -float("inf")):
        other = _run_varlen(torch.where(sim.isnan(), fill, sim), lens, iters, rows, Bo, Mo, No)
        assert torch.equal(other, out), fill
    bin_t = torch.tensor(BIN, device=DEV)
    owned = torch.zeros(Bo, Mo + 1, No + 1, dtype=torch.bool, device=DEV)
    for i, (m, n) in enumerate(lens):
        r = int(rows[i])
        got = _own(out[r], m, n, Mo, No)
        one_sim = sim[i:i + 1, :m, :n].contiguous()
        # one pair at a time through the same entry point: bit-identical
        one = _run_varlen(one_sim, [(m, n)], iters, torch.tensor([0]), 1, m, n)[0]
        assert torch.equal(got, one), (m, n, iters)
        # the uniform kernel on [1, m, n]: the same iterations with another strip plan
        uni = ops.log_optimal_transport(one_sim, bin_t, iters)[0]
        assert rel_err(got, uni) < 1e-5, (m, n, iters, rel_err(got, uni))
        inner, uinner = got[:m, :n], uni[:m, :n]
        assert _argmax_agree(inner, uinner, 1) and _argmax_agree(inner, uinner, 0), (m, n, iters)
        # fp64 restatement of superglue.py:186-214 on the same fp32 costs
        ref = lot64(one_sim.double().cpu(), BIN, iters)[0]
        assert rel_err(got, ref) < (1e-6 if iters == 0 else 2e-5), (m, n, iters, rel_err(got, ref))
        rr = torch.cat([torch.arange(m), torch.tensor([Mo])]).to(DEV)
        cc = torch.cat([torch.arange(n), torch.tensor([No])]).to(DEV)
        owned[r, rr[:, None], cc[None, :]] = True
    assert torch.all(out[~owned] == SENTINEL)


# ---------------------------------------------------------------------------------------------- plugin
SHAPES = [(1, 2), (2, 1), (63, 64), (65, 127), (128, 129), (80, 72), (160, 150), (64, 65), (33, 160)]
PADS = (160, 160)


def _fixture_model(precision):
    model = SuperGlue({"GNN_layers": ["self", "cross"] * 2, "weights": None})
    g, conf, sd, pairs = O.load_fixture(GOLDEN, model.state_dict())
    model = SuperGlue(dict(conf, precision=precision))
    model.load_state_dict(sd, strict=True)
    return model.to(DEV).eval(), g, conf, pairs


def _pair(seed, m, n):
    return synthetic.make_superglue_batch(1, m, n, seed)


def _pad(t, n, fill):
    shp = list(t.shape)
    shp[1] = n - shp[1]
    return torch.cat([t, torch.full(shp, fill, dtype=t.dtype)], 1)


def _batch(pairs, pads, fill=float("nan")):
    data = {}
    for v, P in enumerate(pads):
        for k in KEYS:
            data[f"{k}{v}"] = torch.cat([_pad(p[f"{k}{v}"], P, fill) for p in pairs])
        data[f"view{v}"] = {"image_size": torch.cat([p[f"view{v}"]["image_size"] for p in pairs])}
        data[f"num_keypoints{v}"] = torch.tensor([p[f"keypoints{v}"].shape[1] for p in pairs])
    return data


def _run(model, data):
    with torch.no_grad():
        return model(synthetic.to_device(data, DEV))


def _block(pred, b, m, n, M, N):
    la = pred["log_assignment"][b]
    r = torch.cat([torch.arange(m), torch.tensor([M])]).to(la.device)
    c = torch.cat([torch.arange(n), torch.tensor([N])]).to(la.device)
    return {"log_assignment": la[r][:, c], "sinkhorn_cost": pred["sinkhorn_cost"][b, :m, :n],
            "matches0": pred["matches0"][b, :m], "matches1": pred["matches1"][b, :n],
            "matching_scores0": pred["matching_scores0"][b, :m], "matching_scores1": pred["matching_scores1"][b, :n]}


def _outside_is_empty(pred, b, m, n, M, N):
    la = pred["log_assignment"][b]
    own = torch.zeros_like(la, dtype=torch.bool)
    rr = torch.cat([torch.arange(m), torch.tensor([M])]).to(la.device)
    cc = torch.cat([torch.arange(n), torch.tensor([N])]).to(la.device)
    own[rr[:, None], cc[None, :]] = True
    assert torch.all(la[~own] == float("-inf"))
    cost = pred["sinkhorn_cost"][b].clone()
    cost[:m, :n] = 0
    assert torch.all(cost == 0)
    assert torch.all(pred["matches0"][b, m:] == -1) and torch.all(pred["matches1"][b, n:] == -1)
    assert torch.all(pred["matching_scores0"][b, m:] == 0) and torch.all(pred["matching_scores1"][b, n:] == 0)


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_packed_batch_matches_one_pair_calls(precision):
    model, *_ = _fixture_model(precision)
    pairs = [_pair(100 + i, *s) for i, s in enumerate(SHAPES)]
    pred = _run(model, _batch(pairs, PADS))
    M, N = PADS
    for b, (p, (m, n)) in enumerate(zip(pairs, SHAPES)):
        _outside_is_empty(pred, b, m, n, M, N)
        got = _block(pred, b, m, n, M, N)
        single = _block(_run(model, _batch([p], (m, n))), 0, m, n, m, n)  # packed, one pair, no padding
        for k in got:
            if precision == "bf16" or "matches" in k:
                assert torch.equal(got[k], single[k]), (b, k)
            else:
                torch.testing.assert_close(got[k], single[k], rtol=0, atol=1e-5, msg=f"{b} {k}")
        uni = _run(model, p)
        assert rel_err(got["log_assignment"], uni["log_assignment"][0]) < BOUND[precision], b
        if precision == "fp32":
            assert torch.equal(got["matches0"], uni["matches0"][0].long()), b
            assert torch.equal(got["matches1"], uni["matches1"][0].long()), b


@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_reference_fixture_inside_a_nan_padded_batch(precision):
    model, g, conf, fx = _fixture_model(precision)
    pairs = [synthetic.make_superglue_batch(1, m, n, seed) for m, n, seed in fx]
    pads = (max(m for m, _, _ in fx) + 3, max(n for _, n, _ in fx) + 1)
    pred = _run(model, _batch(pairs, pads))
    for i, (m, n, _) in enumerate(fx):
        got = _block(pred, i, m, n, *pads)
        ref = torch.from_numpy(g[f"p{i}|log_assignment"])
        assert rel_err(got["log_assignment"], ref) < BOUND[precision], (m, n)
        if precision == "fp32":
            for k in ("matches0", "matches1"):
                assert torch.equal(got[k].cpu(), torch.from_numpy(g[f"p{i}|{k}"])), (m, n, k)


def test_padding_is_never_read_and_calls_are_deterministic():
    model, *_ = _fixture_model("bf16")
    pairs = [_pair(400 + i, *s) for i, s in enumerate(SHAPES)]
    base = _run(model, _batch(pairs, PADS, fill=0.0))
    for fill in (float("nan"), float("inf"), -float("inf"), 0.0):
        pred = _run(model, _batch(pairs, PADS, fill=fill))
        for k in base:
            if torch.is_tensor(base[k]):
                assert torch.equal(pred[k], base[k]), (fill, k)


def test_refusals_on_the_device():
    model, *_ = _fixture_model("bf16")
    pairs = [_pair(500 + i, *s) for i, s in enumerate(SHAPES[:3])]
    data = _batch(pairs, PADS)
    pred = _run(model, data)
    with pytest.raises(ValueError, match="loss"):
        model.loss(pred, synthetic.to_device(data, DEV))
    bad = dict(data)
    bad["keypoints1"] = data["keypoints1"].clone()
    bad["keypoints1"][2, 10] = 1e6  # a valid keypoint of pair 2, far outside its image
    with pytest.raises(AssertionError):
        _run(model, bad)
    bad["num_keypoints1"] = torch.tensor([2, 1, 10])  # the same row is now padding: never read
    _run(model, bad)
    with pytest.raises(ValueError, match=r"1 \.\. 160"):
        _run(model, dict(data, num_keypoints0=torch.tensor([1, 161, 3])))


def test_abi_has_the_packed_entry_point():
    from gluefactory_b200 import _lib

    lib = _lib.load()
    assert hasattr(lib, "lgb200_sinkhorn_varlen") and hasattr(lib, "lgb200_sinkhorn_varlen_ws_bytes")
    assert math.isfinite(float(lib.lgb200_sinkhorn_varlen_ws_bytes(3, 100, 200)))
