"""GPU: GlueStick inference on batches of pairs with their own keypoint and line counts (`num_keypoints0/1`,
`num_lines0/1`, eval mode).  Each pair of one packed call must get what a one-pair call on its truncated inputs returns,
in the padded original indexing:
  * against packed calls made one pair at a time: bf16 bit-identical, fp32 equal matches and log-assignments within 1e-5;
  * against the uniform one-pair path: tests/test_gpu_gluestick.py's bounds per precision;
  * fp32 against the fp64 eval oracle (tests/gluestick_wireframe_oracle.py) per pair;
  * the reference's wireframe fixtures a_eval, c_no_lines and e_image_shape as pairs of a NaN-padded packed call;
  * padding (NaN / Inf, junction indices of -1 or out of range) changes no output bit;
and the three packed kernels against the uniform head, the torch formula and an fp64 restatement."""
import numpy as np
import pytest
import torch

from gluefactory_b200 import _lib, ops, synthetic
from gluefactory_b200.matchers.gluestick import GlueStick, junction_order
from tests import gluestick_wireframe_oracle as O
from tests.util import GOLDEN, rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
PT_KEYS = ["keypoints", "descriptors", "keypoint_scores"]
LN_KEYS = ["lines", "line_scores", "lines_junc_idx"]
# (n0, n1, L0, L1): counts 1, 2, 63-65, 127-129, 2 L and the padded maximum; 0, 1 and the maximum lines; M != N
SHAPES = [(1, 2, 1, 1), (2, 1, 0, 3), (63, 64, 40, 1), (65, 127, 20, 36), (128, 129, 7, 0), (80, 72, 40, 36),
          (160, 150, 40, 36), (64, 65, 1, 36)]
PADS = (160, 150, 40, 36)


def _pair(seed, n0, n1, L0, L1, D=256):
    """One synthetic pair (B = 1) with shared junctions: each line's endpoints are keypoints among the first
    min(n, 2 L), drawn with repetition, so several lines may end at one junction."""
    n = max(n0, n1, 2 * max(L0, L1, 1))
    d = synthetic.make_gluestick_batch(1, n, max(L0, L1, 1), seed, D=D)
    g = torch.Generator().manual_seed(seed)
    out = {"view0": d["view0"], "view1": d["view1"]}
    for v, (nk, nl) in enumerate(((n0, L0), (n1, L1))):
        for k in PT_KEYS:
            out[f"{k}{v}"] = d[f"{k}{v}"][:, :nk]
        junc = torch.randint(0, max(1, min(nk, 2 * nl)), (1, nl, 2), generator=g)
        out[f"lines_junc_idx{v}"] = junc
        out[f"lines{v}"] = out[f"keypoints{v}"][0][junc.reshape(-1)].reshape(1, nl, 2, 2)
        out[f"line_scores{v}"] = d[f"line_scores{v}"][:, :nl]
    return out


def _pad(t, n, fill):
    shp = list(t.shape)
    shp[1] = n - shp[1]
    return torch.cat([t, torch.full(shp, fill, dtype=t.dtype)], 1)


def _batch(pairs, pads, fill=float("nan"), junc_fill=-1):
    """Pad one-pair dicts to pads = (M, N, L0, L1) and stack them; returns (data, counts)."""
    M, N, Lp0, Lp1 = pads
    data = {"view0": {}, "view1": {}}
    for v, (P, Lp) in enumerate(((M, Lp0), (N, Lp1))):
        for k in PT_KEYS:
            data[f"{k}{v}"] = torch.cat([_pad(p[f"{k}{v}"], P, fill) for p in pairs])
        for k in LN_KEYS:
            f = junc_fill if k == "lines_junc_idx" else fill
            data[f"{k}{v}"] = torch.cat([_pad(p[f"{k}{v}"], Lp, f) for p in pairs])
        view = pairs[0][f"view{v}"]
        if "image_size" in view:
            data[f"view{v}"]["image_size"] = torch.cat([p[f"view{v}"]["image_size"] for p in pairs])
        else:
            data[f"view{v}"]["image"] = view["image"]
        for key, k in (("num_keypoints", "keypoints"), ("num_lines", "lines")):
            data[f"{key}{v}"] = torch.tensor([p[f"{k}{v}"].shape[1] for p in pairs])
    return data


def _model(precision, D=256, seed=5, inter=True):
    conf = {"GNN_layers": ["self", "cross"] * 3, "descriptor_dim": D, "input_dim": D, "filter_threshold": 0.05}
    if inter:
        conf["inter_supervision"] = [1]
    model = GlueStick(dict(conf, precision=precision))
    sd = synthetic.make_gluestick_weights(model.state_dict(), seed=seed)
    g = torch.Generator().manual_seed(seed)
    for k in sd:  # running statistics away from (0, 1), so that eval-mode BatchNorm is not the identity
        if k.endswith("running_mean"):
            sd[k] = 0.1 * torch.randn(sd[k].shape, generator=g)
        elif k.endswith("running_var"):
            sd[k] = 0.5 + torch.rand(sd[k].shape, generator=g)
    model.load_state_dict(sd, strict=True)
    return model.to(DEV).eval(), conf


def _run(model, data):
    with torch.no_grad():
        return model(synthetic.to_device(data, DEV))


def _heads(model):
    return [("", "M", "N"), ("line_", "L0", "L1")] + [(f"line_{b}_", "L0", "L1")
                                                      for b in model.conf.inter_supervision or []]


def _block(pred, b, prefix, m, n, M, N):
    """Pair b's outputs of head `prefix` in the one-pair form (bins moved back next to the block)."""
    la = pred[prefix + "log_assignment"][b]
    r = torch.cat([torch.arange(m), torch.tensor([M])]).to(la.device)
    c = torch.cat([torch.arange(n), torch.tensor([N])]).to(la.device)
    return {"log_assignment": la[r][:, c], "matches0": pred[prefix + "matches0"][b, :m],
            "matches1": pred[prefix + "matches1"][b, :n], "matching_scores0": pred[prefix + "matching_scores0"][b, :m],
            "matching_scores1": pred[prefix + "matching_scores1"][b, :n]}


def _outside_is_empty(pred, b, prefix, m, n, M, N):
    """Every entry pair b's head does not own: -inf log-assignment, -1 matches, 0 scores."""
    la = pred[prefix + "log_assignment"][b].clone()
    own = torch.zeros_like(la, dtype=torch.bool)
    if m and n:
        rr = torch.cat([torch.arange(m), torch.tensor([M])]).to(la.device)
        cc = torch.cat([torch.arange(n), torch.tensor([N])]).to(la.device)
        own[rr[:, None], cc[None, :]] = True
    assert torch.all(la[~own] == float("-inf"))
    mm0 = m if (m and n) else 0
    mm1 = n if (m and n) else 0
    assert torch.all(pred[prefix + "matches0"][b, mm0:] == -1) and torch.all(pred[prefix + "matches1"][b, mm1:] == -1)
    assert torch.all(pred[prefix + "matching_scores0"][b, mm0:] == 0)
    assert torch.all(pred[prefix + "matching_scores1"][b, mm1:] == 0)


def _one_pair_keys(one, prefix):
    return {k: one[prefix + k] for k in ("log_assignment", "matches0", "matches1", "matching_scores0",
                                         "matching_scores1")}


def _extents(shape, prefix):
    n0, n1, L0, L1 = shape
    if prefix == "":
        return n0, n1
    return (L0, L1) if (L0 and L1) else (0, 0)


@pytest.mark.parametrize("precision,D", [("bf16", 256), ("fp32", 256), ("bf16", 128), ("fp32", 128)])
def test_packed_batch_matches_one_pair_calls(precision, D):
    model, _ = _model(precision, D)
    pairs = [_pair(100 + i, *s, D=D) for i, s in enumerate(SHAPES)]
    pred = _run(model, _batch(pairs, PADS))
    M, N, Lp0, Lp1 = PADS
    pads = {"M": M, "N": N, "L0": Lp0, "L1": Lp1}
    for b, (p, s) in enumerate(zip(pairs, SHAPES)):
        single = _run(model, _batch([p], tuple(int(x) for x in s)))  # packed, one pair, no padding
        uniform = _run(model, p)
        for prefix, kM, kN in _heads(model):
            m, n = _extents(s, prefix)
            _outside_is_empty(pred, b, prefix, m, n, pads[kM], pads[kN])
            if not (m and n):
                continue
            got = _block(pred, b, prefix, m, n, pads[kM], pads[kN])
            ref = _block(single, 0, prefix, m, n, s[0 if kM == "M" else 2], s[1 if kN == "N" else 3])
            for k in got:
                if precision == "bf16" or "matches" in k:
                    assert torch.equal(got[k], ref[k]), (b, prefix, k)
                else:
                    torch.testing.assert_close(got[k], ref[k], rtol=0, atol=1e-5, msg=f"{b} {prefix}{k}")
            uni = _one_pair_keys(uniform, prefix)
            e = rel_err(got["log_assignment"], uni["log_assignment"][0])
            assert e < (1e-4 if precision == "fp32" else 2e-2), (b, prefix, e)
            if precision == "fp32":
                assert torch.equal(got["matches0"], uni["matches0"][0]), (b, prefix)
                assert torch.equal(got["matches1"], uni["matches1"][0]), (b, prefix)
        L0, L1 = _extents(s, "line_")
        raw = pred["raw_line_scores"][b]
        assert torch.all(raw[L0:] == 0) and torch.all(raw[:, L1:] == 0)
        if L0 and precision == "bf16":
            assert torch.equal(raw[:L0, :L1], single["raw_line_scores"][0]), b


def test_packed_fp32_against_fp64_eval_oracle():
    model, conf = _model("fp32")
    pairs = [_pair(200 + i, *s) for i, s in enumerate(SHAPES)]
    pred = _run(model, _batch(pairs, PADS))
    w = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    M, N, Lp0, Lp1 = PADS
    pads = {"M": M, "N": N, "L0": Lp0, "L1": Lp1}
    for b, (p, s) in enumerate(zip(pairs, SHAPES)):
        p64 = {k: ({kk: vv.double() for kk, vv in v.items()} if isinstance(v, dict) else
                   (v.double() if v.is_floating_point() else v)) for k, v in p.items()}
        ref = O.gluestick_forward(w, p64, dict(conf, descriptor_dim=256), training=False)
        for prefix, kM, kN in _heads(model):
            m, n = _extents(s, prefix)
            if not (m and n):
                continue
            got = _block(pred, b, prefix, m, n, pads[kM], pads[kN])
            assert torch.equal(got["matches0"].cpu(), ref[prefix + "matches0"][0]), (b, prefix)
            assert torch.equal(got["matches1"].cpu(), ref[prefix + "matches1"][0]), (b, prefix)
            assert rel_err(got["log_assignment"], ref[prefix + "log_assignment"][0]) < 1e-4, (b, prefix)


@pytest.mark.parametrize("name", ["a_eval", "c_no_lines", "e_image_shape"])
def test_reference_fixtures_inside_a_nan_padded_batch(name):
    g, conf, _, fx = O.load_case(GOLDEN, name, dtype=torch.float32)
    model = GlueStick(dict(conf, precision="fp32"))
    model.load_state_dict(O.case_state_dict(g, model.state_dict()), strict=True)
    model = model.to(DEV).eval()
    D = fx["descriptors0"].shape[-1]
    fx = {k: ({kk: vv[:1] for kk, vv in v.items()} if isinstance(v, dict) else v[:1]) for k, v in fx.items()}
    n0, n1 = fx["keypoints0"].shape[1], fx["keypoints1"].shape[1]
    L0, L1 = fx["lines0"].shape[1], fx["lines1"].shape[1]
    side = []
    for i, s in enumerate([(17, 9, 4, 3), (n0 + 5, n1 + 3, L0 + 2, L1 + 4)]):
        p = _pair(300 + i, *s, D=D)
        for v in (0, 1):
            p[f"view{v}"] = fx[f"view{v}"]
        side.append(p)
    pads = tuple(max(t) for t in zip(*[(q["keypoints0"].shape[1], q["keypoints1"].shape[1], q["lines0"].shape[1],
                                        q["lines1"].shape[1]) for q in side + [fx]]))
    pred = _run(model, _batch([side[0], fx, side[1]], pads))
    M, N, Lp0, Lp1 = pads
    stored = {k[len("pred|"):] for k in g if k.startswith("pred|")}
    for prefix, m, n, PM, PN in (("", n0, n1, M, N), ("line_", L0, L1, Lp0, Lp1)):
        if not (m and n):
            _outside_is_empty(pred, 1, prefix, 0, 0, PM, PN)
            continue
        got = _block(pred, 1, prefix, m, n, PM, PN)
        for k, v in got.items():
            if prefix + k not in stored:
                continue
            ref = g["pred|" + prefix + k]
            if "matches" in k:
                assert np.array_equal(v.cpu().numpy(), ref[0]), (prefix, k)
            elif "log_assignment" in k:
                assert rel_err(v, torch.from_numpy(ref[0])) < 1e-4, (prefix, k)
                np.testing.assert_allclose(v.cpu().numpy(), ref[0], rtol=1e-3, atol=1e-3, err_msg=prefix + k)
            else:
                np.testing.assert_allclose(v.cpu().numpy(), ref[0], rtol=1e-3, atol=1e-4, err_msg=prefix + k)
    if L0 and L1:
        np.testing.assert_allclose(pred["raw_line_scores"][1, :L0, :L1].cpu().numpy(), g["pred|raw_line_scores"][0],
                                   rtol=1e-3, atol=1e-3)


def test_padding_is_never_read_and_calls_are_deterministic():
    model, _ = _model("bf16")
    pairs = [_pair(400 + i, *s) for i, s in enumerate(SHAPES)]
    base = _run(model, _batch(pairs, PADS, fill=0.0, junc_fill=0))
    again = _run(model, _batch(pairs, PADS, fill=0.0, junc_fill=0))
    for fill, junc in ((float("nan"), -1), (float("inf"), 10 ** 6), (-float("inf"), -7)):
        pred = _run(model, _batch(pairs, PADS, fill=fill, junc_fill=junc))
        for k in base:
            if torch.is_tensor(base[k]):
                assert torch.equal(pred[k], base[k]), (fill, k)
    for k in base:
        if torch.is_tensor(base[k]):
            assert torch.equal(again[k], base[k]), k


def test_refusals_on_the_device():
    model, _ = _model("bf16")
    pairs = [_pair(500 + i, *s) for i, s in enumerate(SHAPES[:3])]
    data = _batch(pairs, PADS)
    bad = dict(data)
    bad["lines_junc_idx0"] = data["lines_junc_idx0"].clone()
    bad["lines_junc_idx0"][2, 0, 0] = min(63, 2 * 40)  # pair 2: n0 = 63, L0 = 40 -> bound 63
    with pytest.raises(ValueError, match="lines_junc_idx"):
        _run(model, bad)
    bad["lines_junc_idx0"][2, 0, 0] = -1
    with pytest.raises(ValueError, match="lines_junc_idx"):
        _run(model, bad)
    pred = _run(model, data)
    with pytest.raises(ValueError, match="loss"):
        model.loss(pred, synthetic.to_device(data, DEV))


# ---------------------------------------------------------------------------------------------- kernels
def test_varlen_log_double_softmax_bit_identical_to_uniform():
    g = torch.Generator(device=DEV).manual_seed(0)
    lens = [(1, 1), (1, 2048), (2048, 1), (7, 9), (63, 65), (129, 127), (300, 257), (2048, 2048), (31, 1000)]
    lens += [(int(a), int(b)) for a, b in torch.randint(1, 40, (300, 2), generator=torch.Generator().manual_seed(1))]
    G = len(lens)
    M, N = max(m for m, _ in lens), max(n for _, n in lens)
    Bo, Mo, No = G + 3, M + 5, N + 2
    sim = torch.full((G, M, N), float("nan"), device=DEV)
    for i, (m, n) in enumerate(lens):
        sim[i, :m, :n] = 4 * torch.randn(m, n, device=DEV, generator=g)
    bin_score = torch.tensor(0.7, device=DEV)
    rows = torch.randperm(Bo, generator=torch.Generator().manual_seed(2))[:G]
    pairs = torch.stack([torch.tensor([m for m, _ in lens]), torch.tensor([n for _, n in lens]), rows]).to(DEV).int()
    out = {"scores": torch.full((Bo, Mo + 1, No + 1), float("-inf"), device=DEV),
           "m0": torch.full((Bo, Mo), -1, device=DEV, dtype=torch.int64),
           "m1": torch.full((Bo, No), -1, device=DEV, dtype=torch.int64),
           "ms0": torch.zeros(Bo, Mo, device=DEV), "ms1": torch.zeros(Bo, No, device=DEV)}
    ops.log_double_softmax_varlen(sim, bin_score, pairs, 0.01, out)
    for i, (m, n) in enumerate(lens):
        r = int(rows[i])
        ref = ops.log_double_softmax(sim[i:i + 1, :m, :n].contiguous(), bin_score)[0]
        got = out["scores"][r]
        assert torch.equal(got[:m, :n], ref[:m, :n]) and torch.equal(got[:m, No], ref[:m, n]), (m, n)
        assert torch.equal(got[Mo, :n], ref[m, :n]) and torch.equal(got[Mo, No], ref[m, n]), (m, n)
        inner = ref[:m, :n]
        mx0, mx1 = inner.max(1), inner.max(0)
        m0, m1, ms0, ms1 = ops.filter_matches(mx0.values[None].contiguous(), mx0.indices.int()[None].contiguous(),
                                              mx1.indices.int()[None].contiguous(), 0.01)
        assert torch.equal(out["m0"][r, :m], m0[0]) and torch.equal(out["m1"][r, :n], m1[0]), (m, n)
        assert torch.equal(out["ms0"][r, :m], ms0[0]) and torch.equal(out["ms1"][r, :n], ms1[0]), (m, n)
    untouched = torch.ones(Bo, dtype=torch.bool)
    untouched[rows] = False
    assert torch.all(out["scores"][untouched] == float("-inf")) and torch.all(out["m0"][untouched] == -1)


def test_line_scores_kernel_equals_torch_formula():
    g = torch.Generator(device=DEV).manual_seed(3)
    lens = [(1, 1), (40, 36), (0, 5), (17, 1), (3, 30)]
    lens = [(a, b) for a, b in lens if a and b]
    G = len(lens)
    L0, L1 = max(a for a, _ in lens), max(b for _, b in lens)
    P0, P1 = 2 * L0 + 3, 2 * L1 + 1
    sim = torch.randn(G, P0, P1, device=DEV, generator=g)
    junc0 = torch.full((G, 2 * L0), -5, device=DEV, dtype=torch.int32)
    junc1 = torch.full((G, 2 * L1), 10 ** 6, device=DEV, dtype=torch.int32)
    for i, (a, b) in enumerate(lens):
        junc0[i, :2 * a] = torch.randint(0, min(P0, 2 * a), (2 * a,), device=DEV, generator=g).int()
        junc1[i, :2 * b] = torch.randint(0, min(P1, 2 * b), (2 * b,), device=DEV, generator=g).int()
    pairs = torch.tensor(lens, device=DEV, dtype=torch.int32).t().contiguous()
    raw = ops.line_scores_varlen(sim, junc0, junc1, pairs, L0, L1)
    for i, (a, b) in enumerate(lens):
        idx0, idx1 = junc0[i:i + 1, :2 * a].long(), junc1[i:i + 1, :2 * b].long()
        s = torch.gather(sim[i:i + 1], 2, idx1[:, None, :].expand(1, P0, 2 * b))
        s = torch.gather(s, 1, idx0[:, :, None].expand(1, 2 * a, 2 * b)).reshape(1, a, 2, b, 2)
        ref = 0.5 * torch.maximum(s[:, :, 0, :, 0] + s[:, :, 1, :, 1], s[:, :, 0, :, 1] + s[:, :, 1, :, 0])
        assert torch.equal(raw[i, :a, :b], ref[0]), (a, b)
        assert torch.all(raw[i, a:] == 0) and torch.all(raw[i, :, b:] == 0)


def test_junction_mean_against_fp64_and_pair_order():
    g = torch.Generator().manual_seed(4)
    D, sizes = 256, [5, 1, 40, 17, 64]
    tgt, upd, off = [], [], 0
    for n in sizes:  # pair p owns token rows off .. off + n - 1; 3n endpoints with many shared junctions
        tgt.append(off + torch.randint(0, n, (3 * n,), generator=g))
        off += n
    x = torch.randn(off, D, generator=g)
    upd = torch.randn(sum(3 * n for n in sizes), D, generator=g)
    t = torch.cat(tgt)
    ref = x.double().clone()
    for r in t.unique():
        ref[r] += upd[t == r].double().mean(0)
    order, srt = junction_order(t.int().to(DEV))
    got = ops.junction_mean_(x.to(DEV), upd.to(DEV), order, srt)
    assert torch.allclose(got.double().cpu(), ref, rtol=0, atol=1e-5)
    # the same pairs in another order: every pair's rows come out bit-identical
    perm = [3, 0, 4, 2, 1]
    starts = torch.tensor([0] + sizes).cumsum(0)
    estarts = torch.tensor([0] + [3 * n for n in sizes]).cumsum(0)
    xs, us, ts, new_off = [], [], [], 0
    for p in perm:
        xs.append(x[starts[p]:starts[p + 1]])
        us.append(upd[estarts[p]:estarts[p + 1]])
        ts.append(tgt[p] - starts[p] + new_off)
        new_off += sizes[p]
    order2, srt2 = junction_order(torch.cat(ts).int().to(DEV))
    got2 = ops.junction_mean_(torch.cat(xs).to(DEV), torch.cat(us).to(DEV), order2, srt2)
    o = 0
    for p in perm:
        assert torch.equal(got2[o:o + sizes[p]], got[starts[p]:starts[p + 1]]), p
        o += sizes[p]


def test_abi_has_the_packed_entry_points():
    lib = _lib.load()
    for name in ("lgb200_log_double_softmax_varlen", "lgb200_line_scores_varlen", "lgb200_junction_mean_varlen"):
        assert hasattr(lib, name)
