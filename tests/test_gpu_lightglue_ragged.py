"""GPU: LightGlue inference on batches of pairs with their own keypoint counts (`num_keypoints0/1`), and the packed
varlen assignment head behind it (ops.assign_varlen).

Contract: pair b of a ragged call returns what a one-pair call on its truncated inputs returns -- with adaptive depth /
width off (the plain forward), depth only, width only and both.  Matches, prune counts and stop layers are exact; bf16
is bit-identical everywhere; fp32 log-assignments, scores and states are within 1e-5 (the GEMMs of the fp32 path
are cuBLAS calls whose blocking may change with the packed row count).  Every output key keeps the padded convention of
the module docstring: -inf rows / columns, -1 matches and zero scores, prune counts and states at padded points.

Also: NaN / Inf in every padded input change no output; the adaptive reference fixtures
(tests/golden/lg_adaptive_*.npz, adaptive_prune) hold to the bars of test_gpu_lightglue_adaptive_reference.py when
their pairs run as one ragged call inside larger, NaN-padded views; the varlen head is bit-identical to per-pair
uniform ops.assign_stats + ops.filter_matches at lengths 1 to 2048 and at 300 pairs, with index maps from a pruning
step and NaN in the similarity padding; and the refusals that need a device.

Budget: about a minute and under 6 GiB of device memory on one H100, recorded by the module fixture."""
import ast
import os
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from gluefactory_b200 import ops, synthetic
from gluefactory_b200.matchers.lightglue import LightGlue
from tests.test_gpu_lightglue_adaptive_batch import _calibrate_confidence, _pick_depth, _token_stats
from tests.test_gpu_lightglue_adaptive_reference import _check_la, load_fixture
from tests.util import GOLDEN, report

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture(scope="module", autouse=True)
def _file_budget():
    """Wall time and peak device memory of this file (the machines running it are shared)."""
    torch.cuda.reset_peak_memory_stats()
    t = time.time()
    yield
    torch.cuda.synchronize()
    report("test_gpu_lightglue_ragged", seconds=time.time() - t, peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)


def _build(conf, weights, precision):
    model = LightGlue(dict(conf, precision=precision))
    missing, unexpected = model.load_state_dict({k: v.float() for k, v in weights.items()}, strict=False)
    assert not unexpected and missing in ([], ["confidence_thresholds"])
    return model.to(DEV).eval()


def _pair(m, n, D, seed, frac):
    p = synthetic.make_pairs(1, n, seed=seed, D=D, M=m, frac=frac)
    return {"keypoints0": p["keypoints0"], "keypoints1": p["keypoints1"], "descriptors0": p["descriptors0"],
            "descriptors1": p["descriptors1"], "view0": {"image_size": p["view0"]["image_size"]},
            "view1": {"image_size": p["view1"]["image_size"]}}


def _ragged(pairs, M, N, fill=None, seed=0):
    """Pairs padded to [B, M, N] views; the padding is `fill` (NaN, Inf, ...) or, when None, random finite values
    unlike any real keypoint."""
    g = torch.Generator().manual_seed(seed)
    B = len(pairs)
    out = {}
    for key, L in (("keypoints0", M), ("keypoints1", N), ("descriptors0", M), ("descriptors1", N)):
        shp = (B, L, pairs[0][key].shape[-1])
        t = torch.randn(shp, generator=g) * 1e3 if fill is None else torch.full(shp, fill)
        for b, p in enumerate(pairs):
            t[b, :p[key].shape[1]] = p[key][0]
        out[key] = t
    out["view0"] = {"image_size": torch.cat([p["view0"]["image_size"] for p in pairs])}
    out["view1"] = {"image_size": torch.cat([p["view1"]["image_size"] for p in pairs])}
    out["num_keypoints0"] = torch.tensor([p["keypoints0"].shape[1] for p in pairs])
    out["num_keypoints1"] = torch.tensor([p["keypoints1"].shape[1] for p in pairs], dtype=torch.int32)
    return synthetic.to_device(out, DEV)


def _survivors(la_b, M, N):
    """Rows / columns of a pair's [M+1, N+1] log-assignment that hold scores, plus the dustbins."""
    r = torch.where(torch.isfinite(la_b[:M, N]))[0]
    c = torch.where(torch.isfinite(la_b[M, :N]))[0]
    return torch.cat([r, r.new_tensor([M])]), torch.cat([c, c.new_tensor([N])])


def _close(got, ref, exact, tag):
    if exact:
        assert torch.equal(got, ref), (tag, float((got - ref).abs().max()) if got.shape == ref.shape else got.shape)
    else:
        np.testing.assert_allclose(got.cpu().numpy(), ref.cpu().numpy(), rtol=1e-5, atol=1e-5, err_msg=tag)
    return float((got - ref).abs().max()) if got.numel() else 0.0


def _check_padding(pred, counts, M, N, D):
    n0, n1 = counts
    B = len(n0)
    la = pred["log_assignment"]
    assert la.shape == (B, M + 1, N + 1) and pred["stop_layer"].shape == (B,)
    assert pred["ref_descriptors0"].shape == (B, 1, M, D) and pred["ref_descriptors1"].shape == (B, 1, N, D)
    for b in range(B):
        a, c = n0[b], n1[b]
        assert torch.isneginf(la[b, a:M]).all() and torch.isneginf(la[b, :, c:N]).all(), b
        assert (pred["matches0"][b, a:] == -1).all() and (pred["matches1"][b, c:] == -1).all(), b
        for k, v in (("matching_scores0", a), ("prune0", a), ("matching_scores1", c), ("prune1", c)):
            assert (pred[k][b, v:] == 0).all(), (b, k)
        assert (pred["ref_descriptors0"][b, 0, a:] == 0).all() and (pred["ref_descriptors1"][b, 0, c:] == 0).all()


def _check_against_single(pb, ps, b, n0, n1, M, N, exact, L, tag):
    """Pair b of the ragged pred pb against the one-pair pred ps of its truncated inputs."""
    for k, n in (("matches0", n0), ("matches1", n1), ("prune0", n0), ("prune1", n1)):
        assert torch.equal(pb[k][b, :n], ps[k][0]), (tag, k)
    assert int(pb["stop_layer"][b]) == int(ps.get("stop_layer", L - 1)), tag
    for k, n in (("matching_scores0", n0), ("matching_scores1", n1)):
        _close(pb[k][b, :n], ps[k][0], exact, f"{tag} {k}")
    rows, cols = _survivors(pb["log_assignment"][b], M, N)
    worst = _close(pb["log_assignment"][b][rows][:, cols], ps["log_assignment"][0], exact, f"{tag} log_assignment")
    for j, (idx, n) in enumerate(((rows[:-1], n0), (cols[:-1], n1))):
        assert int(idx.max()) < n, tag
        _close(pb[f"ref_descriptors{j}"][b, 0, idx], ps[f"ref_descriptors{j}"][0, -1], exact, f"{tag} ref{j}")
    return worst


# counts: 1, the tile edges 63-65 / 127-129, the padded maximum and M != N (pruning needs a few points per view)
COUNTS = {"plain": ([1, 64, 129, 300, 127, 65], [63, 260, 128, 1, 65, 200]),
          "depth": ([1, 64, 129, 300, 127, 65], [63, 260, 128, 1, 65, 200]),
          "width": ([63, 300, 129, 127, 65], [260, 64, 128, 200, 65]),
          "both": ([63, 300, 129, 127, 65], [260, 64, 128, 200, 65])}
MODES = {"plain": (False, False), "depth": (True, False), "width": (False, True), "both": (True, True)}


@pytest.mark.parametrize("mode", list(MODES))
@pytest.mark.parametrize("D,H", [(256, 4), (128, 4)])
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_ragged_equals_one_pair_calls(precision, D, H, mode):
    M, N, L = 300, 260, 5
    n0, n1 = COUNTS[mode]
    conf = dict(synthetic.DEFAULT_CONF, descriptor_dim=D, input_dim=D, num_heads=H, n_layers=L)
    w = synthetic.make_weights(conf, seed=500 + D)
    pairs = [_pair(a, c, D, seed=600 + D + 7 * i, frac=float(f))
             for i, (a, c, f) in enumerate(zip(n0, n1, np.linspace(0.1, 0.8, len(n0))))]
    use_depth, use_width = MODES[mode]
    dc, wc = -1, -1
    if use_depth or use_width:
        ratios, match, pre, thr = _token_stats(conf, w, precision, pairs)
        if use_depth:
            w = _calibrate_confidence(w, pre, thr)
            ratios, match, _, _ = _token_stats(conf, w, precision, pairs)
            dc, n_stops = _pick_depth(ratios, L)
            assert dc is not None and n_stops >= 2, ratios
        if use_width:
            wc = 1.0 - (float(match[0].median()) if use_depth else min(float(m.quantile(0.3)) for m in match))
    model = _build(dict(conf, depth_confidence=dc, width_confidence=wc), w, precision)
    with torch.no_grad():
        pb = model(_ragged(pairs, M, N))
        singles = [model(synthetic.to_device(p, DEV)) for p in pairs]
    _check_padding(pb, (n0, n1), M, N, D)
    worst = 0.0
    for b, ps in enumerate(singles):
        worst = max(worst, _check_against_single(pb, ps, b, n0[b], n1[b], M, N, precision == "bf16", L,
                                                 f"{precision} D{D} {mode} pair {b}"))
    stops = pb["stop_layer"].tolist()
    kept = [int((pb["prune0"][b, :n0[b]] == pb["prune0"][b, :n0[b]].max()).sum()) for b in range(len(n0))]
    report(f"ragged {precision} D{D} H{H} {mode}", la_max_abs=worst, stops=str(stops), kept0=str(kept))
    if use_depth and not use_width:
        assert len(set(stops)) >= 2, stops
    if use_width:
        assert len(set(kept)) >= 2, kept
    with pytest.raises(ValueError, match="num_keypoints"):
        model.loss(pb, {})


@pytest.mark.parametrize("mode", ["plain", "both"])
def test_nan_and_inf_padding_change_nothing(mode):
    """Padding of zeros against padding of NaN and of +Inf in keypoints, descriptors, scales and orientations, with
    scale / orientation inputs on and no image sizes (each pair's bounding box normalises its keypoints)."""
    M, N, D = 200, 180, 256
    conf = dict(synthetic.DEFAULT_CONF, n_layers=4, add_scale_ori=True,
                depth_confidence=0.9 if mode == "both" else -1, width_confidence=0.99 if mode == "both" else -1)
    model = _build(conf, synthetic.make_weights(conf, seed=11), "bf16")
    n0, n1 = [150, 1, 200, 90], [180, 40, 7, 129]
    pairs = [_pair(a, c, D, seed=20 + i, frac=0.5) for i, (a, c) in enumerate(zip(n0, n1))]
    if mode == "both":
        n0[1], n1[2] = 30, 30
        pairs[1], pairs[2] = _pair(30, 40, D, seed=21, frac=0.5), _pair(200, 30, D, seed=22, frac=0.5)
    g = torch.Generator().manual_seed(3)
    for p in pairs:
        for j in (0, 1):
            n = p[f"keypoints{j}"].shape[1]
            p[f"scales{j}"] = torch.rand(1, n, generator=g) * 3
            p[f"oris{j}"] = (torch.rand(1, n, generator=g) - 0.5) * 6
    preds = []
    for fill in (0.0, float("nan"), float("inf")):
        data = _ragged(pairs, M, N, fill=fill)
        for j, L in ((0, M), (1, N)):
            for k in ("scales", "oris"):
                t = torch.full((len(pairs), L), fill, device=DEV)
                for b, p in enumerate(pairs):
                    t[b, :p[f"{k}{j}"].shape[1]] = p[f"{k}{j}"][0].to(DEV)
                data[f"{k}{j}"] = t
            del data[f"view{j}"]
        with torch.no_grad():
            preds.append(model(data))
    for k, v in preds[0].items():
        if isinstance(v, torch.Tensor):
            for other in preds[1:]:
                assert torch.equal(v, other[k]), (mode, k)
    _check_padding(preds[0], (n0, n1), M, N, D)
    with torch.no_grad():  # the bounding box of the valid points only: a one-pair call without image sizes
        b = 0
        single = {k: v for k, v in pairs[b].items() if not k.startswith("view")}
        ps = model(synthetic.to_device(single, DEV))
    _check_against_single(preds[0], ps, b, n0[b], n1[b], M, N, True, 4, f"nan padding {mode}")


@pytest.mark.parametrize("name", ["lg_adaptive_a_depth", "lg_adaptive_b_both", "lg_adaptive_c_d128_both",
                                  "lg_adaptive_d_long", "adaptive_prune"])
def test_reference_fixtures_in_one_ragged_call(name):
    """Every pair of a fixture in one ragged call, in reversed order, inside views padded with NaN to 1.25 x the
    fixture's sizes (the fixtures differ in weights, so each is its own call), against the reference's results."""
    if name == "adaptive_prune":
        g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
        conf = ast.literal_eval(str(g["meta|conf"]))
        seed, M, N = int(g["meta|seed"]), int(g["meta|M"]), int(g["meta|N"])
        w = synthetic.make_weights(conf, seed=seed)
        pairs = [_pair(M, N, conf["input_dim"], seed=seed + 1, frac=0.4)]
        ref = {f"p0|{k}": g[f"pred|{k}"] for k in ("prune0", "prune1", "matches0", "matches1", "matching_scores0",
                                                   "matching_scores1", "log_assignment")}
        ref["p0|stop_layer"] = np.array(conf["n_layers"] - 1)
        pairs = pairs + [_pair(M // 2, N + 7, conf["input_dim"], seed=seed + 9, frac=0.2)]  # a second, other-sized pair
        check = [0]
    else:
        ref, conf, w, pairs = load_fixture(name)
        M, N = int(ref["meta|M"]), int(ref["meta|N"])
        check = list(range(len(pairs)))
    Mp, Np = M + M // 4 + 1, N + N // 4 + 3
    model = _build(conf, w, "fp32")
    order = list(range(len(pairs)))[::-1]
    with torch.no_grad():
        pred = model(_ragged([pairs[j] for j in order], Mp, Np, fill=float("nan")))
    assert pred["log_assignment"].shape == (len(pairs), Mp + 1, Np + 1)
    worst = 0.0
    for b, j in enumerate(order):
        if j not in check:
            continue
        p, tag = f"p{j}|", f"{name} pair {j}"
        assert int(pred["stop_layer"][b]) == int(ref[p + "stop_layer"]), tag
        for k, n in (("prune0", M), ("prune1", N), ("matches0", M), ("matches1", N)):
            got = pred[k][b].cpu().numpy()
            assert np.array_equal(got[:n], ref[p + k][0].astype(got.dtype)), (tag, k)
            assert (got[n:] == (-1 if k.startswith("matches") else 0)).all(), (tag, k)
        for k, n in (("matching_scores0", M), ("matching_scores1", N)):
            np.testing.assert_allclose(pred[k][b, :n].cpu().numpy(), ref[p + k][0], rtol=1e-3, atol=1e-6, err_msg=tag)
        la = pred["log_assignment"][b].cpu().numpy()
        p0, p1 = ref[p + "prune0"][0], ref[p + "prune1"][0]
        rows = np.concatenate([np.flatnonzero(p0 == p0.max()), [Mp]])
        cols = np.concatenate([np.flatnonzero(p1 == p1.max()), [Np]])
        assert np.isneginf(la[np.setdiff1d(np.arange(Mp + 1), rows)]).all(), tag
        assert np.isneginf(la[:, np.setdiff1d(np.arange(Np + 1), cols)]).all(), tag
        worst = max(worst, _check_la(la[np.ix_(rows, cols)], ref, p, tag))
    report(f"ragged reference {name}", la_max_abs=worst, stops=str(pred["stop_layer"].tolist()))


def _head_case(lens, Mo, No, seed, prune):
    """G pairs of (m, n) from lens; their original index maps come from a pruning step (sorted survivors of Mo / No
    points) when `prune`, else 0 .. m-1; the similarity is padded to the longest pair with NaN."""
    g = torch.Generator().manual_seed(seed)
    G = len(lens)
    Mg, Ng = max(m for m, _ in lens), max(n for _, n in lens)
    sim = torch.full((G, Mg, Ng), float("nan"))
    z = torch.full((2, G, max(Mg, Ng)), float("nan"))
    ind0, ind1 = torch.zeros(G, Mg, dtype=torch.int32), torch.zeros(G, Ng, dtype=torch.int32)
    for k, (m, n) in enumerate(lens):
        sim[k, :m, :n] = torch.randn(m, n, generator=g) * 3
        z[0, k, :m], z[1, k, :n] = torch.randn(m, generator=g), torch.randn(n, generator=g)
        ind0[k, :m] = (torch.randperm(Mo, generator=g)[:m].sort().values if prune else torch.arange(m)).int()
        ind1[k, :n] = (torch.randperm(No, generator=g)[:n].sort().values if prune else torch.arange(n)).int()
    out_b = torch.randperm(G, generator=g)
    return sim, z[0, :, :Mg], z[1, :, :Ng], ind0, ind1, out_b


@pytest.mark.parametrize("case", ["lengths_1_to_2048", "300_pairs"])
def test_varlen_head_bitwise_against_uniform(case):
    """ops.assign_varlen against per-pair uniform ops.assign_stats(dense=True) + ops.filter_matches on [1, m, n]."""
    if case == "lengths_1_to_2048":
        lens = [(1, 1), (1, 2048), (2048, 1), (63, 65), (64, 64), (65, 129), (127, 128), (129, 31), (2048, 2048),
                (1000, 1537), (33, 4), (257, 255)]
        Mo, No = 2100, 2100
    else:
        g = torch.Generator().manual_seed(5)
        lens = [tuple(int(v) for v in torch.randint(1, 140, (2,), generator=g)) for _ in range(300)]
        Mo, No = 150, 160
    for prune in (False, True):
        sim, z0, z1, ind0, ind1, out_b = _head_case(lens, Mo if prune else max(m for m, _ in lens),
                                                    No if prune else max(n for _, n in lens), 7, prune)
        Mo_, No_ = (Mo, No) if prune else (sim.shape[1], sim.shape[2])
        G = len(lens)
        sim, z0, z1, ind0, ind1 = (t.to(DEV) for t in (sim, z0, z1, ind0, ind1))
        pairs = torch.tensor([[m for m, _ in lens], [n for _, n in lens], out_b.tolist()], dtype=torch.int32,
                             device=DEV)
        out = {"scores": torch.full((G, Mo_ + 1, No_ + 1), -float("inf"), device=DEV),
               "m0": torch.full((G, Mo_), -1, dtype=torch.int64, device=DEV),
               "m1": torch.full((G, No_), -1, dtype=torch.int64, device=DEV),
               "ms0": torch.zeros(G, Mo_, device=DEV), "ms1": torch.zeros(G, No_, device=DEV)}
        th = 0.1
        st = ops.assign_varlen(sim, F.logsigmoid(z0), F.logsigmoid(z1), F.logsigmoid(-z0), F.logsigmoid(-z1), pairs,
                               ind0, ind1, th, out)
        written = torch.zeros(G, Mo_ + 1, No_ + 1, dtype=torch.bool, device=DEV)
        for k, (m, n) in enumerate(lens):
            s = ops.assign_stats(sim[k:k + 1, :m, :n].contiguous(), F.logsigmoid(z0[k:k + 1, :m]),
                                 F.logsigmoid(z1[k:k + 1, :n]), F.logsigmoid(-z0[k:k + 1, :m]),
                                 F.logsigmoid(-z1[k:k + 1, :n]), dense=True)
            a0, a1, s0, s1 = ops.filter_matches(s["rowmax"], s["rowarg"], s["colarg"], th)
            b = int(out_b[k])
            r = torch.cat([ind0[k, :m].long(), torch.tensor([Mo_], device=DEV)])
            c = torch.cat([ind1[k, :n].long(), torch.tensor([No_], device=DEV)])
            tag = f"{case} prune={prune} pair {k} ({m}, {n})"
            assert torch.equal(out["scores"][b][r[:, None], c[None, :]], s["scores"][0]), tag
            written[b][r[:, None], c[None, :]] = True
            i0, i1 = ind0[k, :m].long(), ind1[k, :n].long()
            assert torch.equal(out["m0"][b, i0], torch.where(a0[0] < 0, -1, i1[a0[0].clamp(min=0)])), tag
            assert torch.equal(out["m1"][b, i1], torch.where(a1[0] < 0, -1, i0[a1[0].clamp(min=0)])), tag
            assert torch.equal(out["ms0"][b, i0], s0[0]) and torch.equal(out["ms1"][b, i1], s1[0]), tag
            for key in ("rowmax", "rowarg", "row_expsum"):
                assert torch.equal(st[key][k, :m], s[key][0]), (tag, key)
            for key in ("colmax", "colarg"):
                assert torch.equal(st[key][k, :n], s[key][0]), (tag, key)
            keep0 = torch.ones(Mo_, dtype=torch.bool, device=DEV)
            keep0[i0] = False
            keep1 = torch.ones(No_, dtype=torch.bool, device=DEV)
            keep1[i1] = False
            assert (out["m0"][b, keep0] == -1).all() and (out["ms0"][b, keep0] == 0).all(), tag
            assert (out["m1"][b, keep1] == -1).all() and (out["ms1"][b, keep1] == 0).all(), tag
        assert torch.isneginf(out["scores"][~written]).all(), case
    report(f"varlen head {case}", pairs=len(lens))


def test_refusals_on_device():
    conf = dict(synthetic.DEFAULT_CONF, n_layers=2)
    model = _build(conf, synthetic.make_weights(conf, seed=1), "bf16")
    data = _ragged([_pair(20, 30, 256, seed=1, frac=0.5), _pair(40, 10, 256, seed=2, frac=0.5)], 40, 30)
    with torch.no_grad():
        pred = model(data)
    with pytest.raises(ValueError, match="num_keypoints"):
        model.loss(pred, data)
    for bad, msg in ((torch.tensor([0, 10], device=DEV), "1 .. 40"), (torch.tensor([41, 10], device=DEV), "1 .. 40"),
                     (torch.tensor([20.0, 40.0], device=DEV), "integer"), (torch.tensor([[20, 40]], device=DEV), "shape")):
        with pytest.raises(ValueError, match=msg):
            model(dict(data, num_keypoints0=bad))
    model.train()
    with pytest.raises(ValueError, match="eval mode"):
        model(data)
