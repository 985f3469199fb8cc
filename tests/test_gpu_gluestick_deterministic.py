"""GPU: GlueStick's fixed-order LineLayer and line-head kernels, and the bit-reproducible training they give on
wireframes with shared junctions.

Kernels (ops.JunctionGather / JunctionMean / LineScores) against the fp64 restatements of
tests/gluestick_deterministic_oracle.py, at D 128 and 256, line counts not a multiple of 8, similarity widths across a
256-thread block and a junction ending >= 8 lines.  An fp32 sum of k terms is within k * 2^-24 * (sum of |terms|) of
the exact sum; the bounds below take 4 * 2^-24 * k_max * (sum of |terms|) per entry.  The forward raw scores must equal
the torch formula bit for bit, NaN included, and every result must repeat bit for bit.

End to end, on tests/golden/gluestick_wireframe_b_train.npz (shared junctions, padded, inter_supervision [1]) and on a
harder seeded wireframe (B = 4, hubs ending 9 and 5 lines, degenerate lines), in fp32 and bf16, at 128 and 256
channels: forward + loss + backward twice from the same state, and the captured trainer step replayed twice from the
same saved state, give the same bits, and the replay equals the eager step."""
import copy

import pytest
import torch

from gluefactory_b200 import ops, synthetic
from gluefactory_b200.matchers.gluestick import GlueStick, junction_layout
from gluefactory_b200.trainer import MatcherTrainer
from tests import gluestick_deterministic_oracle as O
from tests import gluestick_wireframe_oracle as W
from tests.util import GOLDEN

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 2.0 ** -24


def _wire(B, L, n, seed):
    idx = O.wireframe_junctions(B, L, n, seed, hubs=((3, 9), (7, 5)), degenerate=(14, 15, 16))
    return idx.reshape(B, 2 * L)


def _max_degree(idx, n):
    return int(torch.bincount((idx + torch.arange(idx.shape[0])[:, None] * n).reshape(-1)).max())


def _bound(k, mag):
    return 4 * EPS * k * mag + 1e-30


@pytest.mark.parametrize("D", [128, 256])
def test_junction_gather_and_mean_against_fp64(D):
    B, L, n = 3, 37, 90
    idx = _wire(B, L, n, 11)
    lay_c = junction_layout(idx, n, min(n, 2 * L))
    lay = junction_layout(idx.to(DEV), n, min(n, 2 * L))
    assert torch.bincount(lay_c.tgt.long()).max() >= 8
    for a, b in zip(lay, lay_c):
        assert torch.equal(a.cpu(), b)
    gen = torch.Generator().manual_seed(D)
    x = torch.randn(B * n, D, generator=gen)
    cat_g = torch.randn(B * 2 * L, 3 * D, generator=gen)  # the gradient of [gather ; encoding], as the MLP returns it
    xd = x.to(DEV).requires_grad_(True)
    out = ops.JunctionGather.apply(xd, lay.tgt, lay.order, lay.tgt_sorted)
    ref_out, _ = O.reference_line_layer_parts(x.double(), idx, B)
    assert torch.equal(out.detach().cpu().double(), ref_out)
    g = cat_g.to(DEV)
    out.backward(g[:, :2 * D])  # a column slice of a wider matrix: the kernel reads it in place (row pitch 3 D)
    k = int(torch.bincount(lay_c.tgt.long()).max()) * 2
    ref = O.junction_sum(cat_g[:, :2 * D], lay_c.tgt, B * n, D)
    mag = O.junction_sum(cat_g[:, :2 * D].abs(), lay_c.tgt, B * n, D)
    err = (xd.grad.cpu().double() - ref).abs()
    assert (err <= _bound(k, mag)).all(), float((err / _bound(k, mag)).max())
    assert (xd.grad.cpu()[torch.bincount(lay_c.tgt.long(), minlength=B * n) == 0] == 0).all()
    first = xd.grad.clone()
    xd.grad = None
    ops.JunctionGather.apply(xd, lay.tgt, lay.order, lay.tgt_sorted).backward(g[:, :2 * D].contiguous())
    assert torch.equal(xd.grad, first)

    upd = torch.randn(B * 2 * L, D, generator=gen)
    xm, um = x.to(DEV).requires_grad_(True), upd.to(DEV).requires_grad_(True)
    y = ops.JunctionMean.apply(xm, um, lay.tgt, lay.order, lay.tgt_sorted)
    ref_y = O.reference_junction_mean(x.double(), upd.double(), lay_c.tgt.long())
    mag_y = x.double().abs() + O.reference_junction_mean(torch.zeros_like(x).double(), upd.double().abs(),
                                                         lay_c.tgt.long())
    assert ((y.detach().cpu().double() - ref_y).abs() <= _bound(k + 2, mag_y)).all()
    gy = torch.randn(B * n, D, generator=gen)
    y.backward(gy.to(DEV))
    assert torch.equal(xm.grad.cpu(), gy)
    assert torch.equal(um.grad.cpu(), O.junction_mean_bwd(gy, lay_c.tgt).float())  # the same IEEE division
    y2 = ops.JunctionMean.apply(xm.detach(), um.detach(), lay.tgt, lay.order, lay.tgt_sorted)
    assert torch.equal(y2, y.detach())


def _scores_case(G, L0, L1, n0, n1, seed):
    idx0, idx1 = _wire(G, L0, n0, seed), _wire(G, L1, n1, seed + 1)
    P0, P1 = min(n0, 2 * L0), min(n1, 2 * L1)
    gen = torch.Generator().manual_seed(seed)
    sim = torch.randn(G, P0, P1, generator=gen)
    hubs = sim[:, :8, :8]  # small integers here: exact ties among the hubs' lines
    hubs.copy_(torch.randint(-2, 3, hubs.shape, generator=gen))
    graw = torch.randn(G, L0, L1, generator=gen)
    return idx0, idx1, sim, graw


def _line_scores(sim, idx0, idx1, n0, n1, grad=True):
    G, P0, P1 = sim.shape
    L0, L1 = idx0.shape[1] // 2, idx1.shape[1] // 2
    lay0, lay1 = junction_layout(idx0.to(DEV), n0, P0), junction_layout(idx1.to(DEV), n1, P1)
    pairs = torch.tensor([[L0] * G, [L1] * G], dtype=torch.int32, device=DEV)
    s = sim.to(DEV).requires_grad_(grad)
    raw = ops.LineScores.apply(s, lay0.junc, lay1.junc, pairs, lay0.order, lay0.ptr, lay1.order, lay1.ptr)
    return s, raw


@pytest.mark.parametrize("G,L0,L1,n0,n1", [(2, 37, 45, 90, 160), (3, 150, 141, 250, 300), (1, 5, 3, 6, 6)])
def test_line_scores_against_torch_and_fp64(G, L0, L1, n0, n1):
    """Raw scores bit-identical to the torch formula on the same fp32 sim; d sim within the fp32 summation bound of the
    fp64 restatement, 0 where no line reads it; both repeat bit for bit."""
    idx0, idx1, sim, graw = _scores_case(G, L0, L1, n0, n1, 3 + L0)
    s, raw = _line_scores(sim, idx0, idx1, n0, n1)
    torch_raw = O.reference_line_scores(sim.to(DEV), idx0.to(DEV), idx1.to(DEV))
    assert torch.equal(raw.detach(), torch_raw)
    raw.backward(graw.to(DEV))
    ref = O.line_scores_bwd(graw, sim, idx0, idx1)
    mag = O.line_scores_bwd(graw, sim, idx0, idx1, absolute=True)
    k = _max_degree(idx0, n0) * _max_degree(idx1, n1)
    err = (s.grad.cpu().double() - ref).abs()
    assert (err <= _bound(k, mag)).all(), float((err / _bound(k, mag)).max())
    assert (s.grad.cpu()[mag == 0] == 0).all()
    first = s.grad.clone()
    s2, raw2 = _line_scores(sim, idx0, idx1, n0, n1)
    raw2.backward(graw.to(DEV))
    assert torch.equal(raw2, raw) and torch.equal(s2.grad, first)


def test_line_scores_nan_like_torch():
    """A NaN in sim: the same raw NaNs as the torch formula, and d sim as torch's autograd (both branches of a NaN
    maximum take the gradient; an infinite gradient does not leak through a branch that takes none)."""
    G, L0, L1, n0, n1 = 2, 21, 19, 50, 50
    idx0, idx1, sim, graw = _scores_case(G, L0, L1, n0, n1, 5)
    sim[0, int(idx0[0, 6]), int(idx1[0, 3])] = float("nan")
    graw[1, 2, 2] = float("inf")
    s, raw = _line_scores(sim, idx0, idx1, n0, n1)
    st = sim.to(DEV).requires_grad_(True)
    torch_raw = O.reference_line_scores(st, idx0.to(DEV), idx1.to(DEV))
    assert torch.isnan(torch_raw).any()
    assert torch.equal(torch.isnan(raw), torch.isnan(torch_raw))
    assert torch.equal(raw.nan_to_num(), torch_raw.detach().nan_to_num())
    raw.backward(graw.to(DEV))
    torch_raw.backward(graw.to(DEV))
    assert torch.isinf(st.grad).any()
    assert torch.equal(torch.isnan(s.grad), torch.isnan(st.grad)) and torch.equal(torch.isinf(s.grad), torch.isinf(st.grad))
    fin = torch.isfinite(st.grad)
    torch.testing.assert_close(s.grad[fin], st.grad[fin], rtol=1e-5, atol=1e-5)
    ref = O.line_scores_bwd(graw, sim, idx0, idx1)
    assert torch.equal(torch.isinf(s.grad.cpu()), torch.isinf(ref))


# ------------------------------------------------------------------------------------------------ end to end
SMALL_CONF = {"GNN_layers": ["self", "cross"] * 2, "filter_threshold": 0.2, "inter_supervision": [1],
              "loss": {"nll_weight": 1.0, "nll_balancing": 0.5, "inter_supervision": [0.3, 0.6]}}


def _hard_case(D, seed=91, B=4, N=128, L=44):
    """make_gluestick_batch with its lines replaced by a wireframe: junctions of degree 9 and 5, degenerate lines,
    nodes no line touches; each line's endpoints are its junctions' keypoints."""
    d = synthetic.make_gluestick_batch(B, N, L, seed, D=D)
    for i in "01":
        idx = _wire(B, L, N, seed + int(i)).view(B, L, 2)
        d[f"lines_junc_idx{i}"] = idx
        kp = d[f"keypoints{i}"]
        d[f"lines{i}"] = torch.stack([kp[b][idx[b].reshape(-1)] for b in range(B)]).view(B, L, 2, 2)
    model_conf = dict(SMALL_CONF, descriptor_dim=D, input_dim=D)
    return model_conf, seed, d


def _case(name, D, precision):
    if name == "b_train":
        g, conf, _, data = W.load_case(GOLDEN, "b_train", dtype=torch.float32)
        model = GlueStick(dict(conf, precision=precision))
        model.load_state_dict(W.case_state_dict(g, model.state_dict()), strict=True)
    else:
        conf, seed, data = _hard_case(D)
        model = GlueStick(dict(conf, precision=precision))
        model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=seed), strict=True)
    return model.to(DEV).train(), synthetic.to_device(data, DEV)


CASES = [("b_train", 256), ("hard", 128), ("hard", 256)]


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name,D", CASES)
def test_forward_backward_repeats_bit_for_bit(name, D, precision):
    model, data = _case(name, D, precision)
    start = {k: v.clone() for k, v in model.state_dict().items()}
    runs = []
    for _ in range(2):
        model.load_state_dict(start)
        model.zero_grad(set_to_none=True)
        pred = model(data)
        losses, _ = model.loss(pred, data)
        losses["total"].mean().backward()
        runs.append(({k: v.detach().clone() for k, v in losses.items() if torch.is_tensor(v)},
                     {k: p.grad.clone() for k, p in model.named_parameters()},
                     {k: v.clone() for k, v in model.state_dict().items() if "running_" in k},
                     pred["raw_line_scores"].detach().clone()))
    (l0, g0, r0, w0), (l1, g1, r1, w1) = runs
    assert torch.isfinite(l0["total"]).all()
    assert set(l0) == set(l1) and all(torch.equal(l0[k], l1[k]) for k in l0), name
    for k in g0:
        assert torch.equal(g0[k], g1[k]), k
    for k in r0:
        assert torch.equal(r0[k], r1[k]), k
    assert torch.equal(w0, w1)
    if name == "hard":  # the wireframe has what it is meant to have
        j = data["lines_junc_idx0"].reshape(4, -1)
        assert int(torch.bincount(j[0]).max()) >= 9 and bool((j[:, 28] == j[:, 29]).all())


@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("name,D", CASES)
def test_captured_step_replays_bit_for_bit_and_equals_eager(name, D, precision):
    model, data = _case(name, D, precision)
    eager_model, _ = _case(name, D, precision)
    start = {k: v.clone() for k, v in model.state_dict().items()}
    graphed = MatcherTrainer(model, lr=1e-4)
    opt_start = copy.deepcopy(graphed.state_dict())
    graphed.capture(data, torch.device(DEV))
    outs = []
    for _ in range(2):
        model.load_state_dict(start)  # in place: the weights are views of the captured flat buffer
        graphed.load_state_dict(copy.deepcopy(opt_start))
        loss, _ = graphed.step_graphed(data)
        torch.cuda.synchronize()
        st = graphed.state_dict()["optimizer"]["state"]
        outs.append((loss.clone(), {k: v.clone() for k, v in model.state_dict().items()},
                     {i: {k: v.clone() for k, v in s.items()} for i, s in st.items()}))
    (la, sa, oa), (lb, sb, ob) = outs
    assert torch.isfinite(la).all() and torch.equal(la, lb)
    for k in sa:
        assert torch.equal(sa[k], sb[k]), k
    assert oa.keys() == ob.keys() and all(torch.equal(oa[i][k], ob[i][k]) for i in oa for k in oa[i])
    eager = MatcherTrainer(eager_model, lr=1e-4)
    le, _ = eager.step(data)
    assert torch.equal(le, la), (le.item(), la.item())
    for k, v in eager_model.state_dict().items():
        assert torch.equal(v, sa[k]), k
