"""CPU: the restatements and comparison helpers that tests/test_gpu_superpoint_shapes.py checks the SuperPoint kernels
with.  select_ref_fast must equal select_ref (the reference's order) on the goldens and on maps full of exact ties; each
comparison helper must reject a one-ulp, one-index or swapped-tie perturbation; the derived bounds must hold for fp32
arithmetic done in another order, and must stay far from vacuous."""
import glob
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests import superpoint_oracle as so  # noqa: E402

GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "superpoint_*.npz")))


def _tied_maps():
    """Small post-NMS maps with plateaus (quantised bumps, constant blocks, one constant map) and the border frame."""
    maps = [so.blob_map(2, 45, 70, seed=1, levels=6), so.region_map(2, 45, 70, seed=2, cell=9),
            torch.full((1, 45, 70), 0.03)]
    return [so.border_ref(so.nms_ref(m, 2), 4) for m in maps]


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
@pytest.mark.parametrize("k", [-1, 1, 7, 40, 512])
def test_select_fast_equals_select_ref_golden(path, k):
    s = so.border_ref(so.nms_ref(torch.from_numpy(so.load_golden(path)["dense_scores"]), 3), 4)
    for thr in (0.0, 0.005):
        for (a, sa), (b, sb) in zip(so.select_ref_fast(s, thr, k), so.select_ref(s, thr, k)):
            so.assert_bits_equal(a, b, "keypoints")
            so.assert_bits_equal(sa, sb, "scores")


@pytest.mark.parametrize("thr", [0.0, 0.005, -1.0])
def test_select_fast_equals_select_ref_ties(thr):
    for s in _tied_maps():
        n = int((s > thr).sum(dim=(1, 2)).max())
        for k in (1, 2, 17, n // 3, n - 1, n, n + 1):
            for (a, sa), (b, sb) in zip(so.select_ref_fast(s, thr, k), so.select_ref(s, thr, k)):
                so.assert_bits_equal(a, b, "keypoints")
                so.assert_bits_equal(sa, sb, "scores")
    # the tie fixtures really are tied at the cut: the constant map's one group spans every chunk of the image
    s = _tied_maps()[2]
    eq, taken, chunks = so.tie_stats(s[0], thr, 100)
    assert eq == 37 * 62 and taken == 100 and chunks == [0, 1, 2]


def test_select_fast_ties_go_to_lower_index():
    s = torch.zeros(1, 4, 600)
    s[0, 0, 5] = s[0, 3, 590] = s[0, 1, 10] = 0.5  # three equal scores in different 1024-pixel chunks
    s[0, 2, 2] = 0.7
    kp, sc = so.select_ref_fast(s, 0.0, 3)[0]
    assert kp.tolist() == [[2.0, 2.0], [5.0, 0.0], [10.0, 1.0]] and sc.tolist() == pytest.approx([0.7, 0.5, 0.5])
    kp, _ = so.select_ref_fast(s, 0.0, 4)[0]  # no more than k: row-major order
    assert kp.tolist() == [[5.0, 0.0], [10.0, 1.0], [2.0, 2.0], [590.0, 3.0]]


# ---- negative controls ------------------------------------------------------------------------------------------------
def _ulp_up(t, i):
    t = t.clone()
    t.view(-1).view(torch.int32)[i] += 1
    return t


def test_bits_equal_rejects_one_ulp():
    x = torch.rand(5, 7)
    so.assert_bits_equal(x, x.clone())
    with pytest.raises(AssertionError):
        so.assert_bits_equal(_ulp_up(x, 11), x)
    with pytest.raises(AssertionError):
        so.assert_bits_equal(-torch.zeros(3), torch.zeros(3))


def test_selection_rejects_ulp_index_and_swapped_tie():
    s = _tied_maps()[0]
    ref = so.select_ref_fast(s, 0.0, 50)[0]
    kp, sc = ref[0].clone(), ref[1].clone()
    so.assert_selection(kp, sc, 50, ref)
    with pytest.raises(AssertionError):
        so.assert_selection(kp, _ulp_up(sc, 3), 50, ref)
    kp1 = kp.clone()
    kp1[7, 0] += 1  # one index off
    with pytest.raises(AssertionError):
        so.assert_selection(kp1, sc, 50, ref)
    with pytest.raises(AssertionError):
        so.assert_selection(kp, sc, 49, ref)
    i = next(i for i in range(49) if sc[i] == sc[i + 1] and not torch.equal(kp[i], kp[i + 1]))
    kp2 = kp.clone()
    kp2[[i, i + 1]] = kp2[[i + 1, i]]  # two tied candidates swapped: same scores, other order
    with pytest.raises(AssertionError):
        so.assert_selection(kp2, sc, 50, ref)


def test_within_rejects_one_ulp_past_the_bound():
    ref = torch.rand(64, dtype=torch.float64)
    bound = torch.full_like(ref, 2.0 ** -20)
    out = (ref + bound).float()
    exact = ref + bound  # out's value, shifted to where the bound is met exactly
    assert so.assert_within(exact, ref, bound) <= 1.0
    past = torch.nextafter(exact, torch.full_like(exact, 2.0))
    with pytest.raises(AssertionError):
        so.assert_within(past, ref, bound)
    with pytest.raises(AssertionError):
        so.assert_within(out.double().clone().index_fill_(0, torch.tensor([3]), float("nan")), ref, bound)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.int32])
def test_guards_reject_overwrite_and_unwritten(dtype):
    g = so.Guarded((3, 5), dtype, "cpu", guard=8)
    g.t.copy_(torch.ones(3, 5).to(dtype))
    g.check("ok")
    g.ibuf[g.guard + g.n] = 0  # one element past the output
    with pytest.raises(AssertionError, match="after"):
        g.check("past")
    g = so.Guarded((3, 5), dtype, "cpu", guard=8)
    g.t.copy_(torch.ones(3, 5).to(dtype))
    g.ibuf[g.guard - 1] = 0  # one element before it
    with pytest.raises(AssertionError, match="before"):
        g.check("before")
    g = so.Guarded((3, 5), dtype, "cpu", guard=8)
    g.t[:2].copy_(torch.ones(2, 5).to(dtype))  # the last row never written
    with pytest.raises(AssertionError, match="never written"):
        g.check("unwritten")


# ---- the derived bounds hold for fp32 arithmetic in another order, and are tight enough to mean something -------------
def _bf16(t):
    return t.to(torch.bfloat16).double()


@pytest.mark.parametrize("cin,cout,ks", [(64, 64, 3), (128, 65, 1), (256, 256, 1)])
def test_conv_bounds_hold_for_fp32(cin, cout, ks):
    g = torch.Generator(device="cpu").manual_seed(cin + cout)
    x = _bf16(torch.rand(1, cin, 9, 13, generator=g))
    w = _bf16(torch.randn(cout, cin, ks, ks, generator=g) * (2.0 / (cin * ks * ks)) ** 0.5 * 4)
    b = torch.rand(cout, generator=g, dtype=torch.float64) * 0.1 - 0.05
    y = F.conv2d(x, w, b, padding=ks // 2)
    E = so.conv_acc_bound(F.conv2d(x.abs(), w.abs(), b.abs(), padding=ks // 2), ks * ks * cin)
    y32 = F.conv2d(x.float(), w.float(), b.float(), padding=ks // 2)  # fp32, another summation order
    assert so.assert_within(y32, y, E) < 1.0
    r = so.assert_within(F.relu(y32).to(torch.bfloat16), F.relu(y), so.relu_bf16_bound(F.relu(y), E))
    assert r < 1.0
    pooled = F.max_pool2d(F.relu(y), 2, 2)
    so.assert_within(F.max_pool2d(F.relu(y32), 2, 2).to(torch.bfloat16), pooled, so.pool_bf16_bound(pooled, E[..., :8, :12]))
    # far from vacuous: the typical accumulation bound is below one bf16 rounding of the value
    assert float((E / y.abs().clamp_min(1e-3)).median()) < so.U_BF16
    if cout == 65:
        p, bound = so.softmax_bound(y, E)
        so.assert_within(F.softmax(y32, 1)[:, :-1], p, bound)
        assert float((bound / p).max()) < 1e-2
    if cout == 256:
        o, bound = so.l2n_bound(y, E)
        so.assert_within(F.normalize(y32, dim=1), o, bound)
        assert float(bound.max()) < 1e-3


@pytest.mark.parametrize("legacy", [True, False])
@pytest.mark.parametrize("h,w", [(60, 80), (150, 200)])
def test_sample_coordinate_error_bound(legacy, h, w):
    """The kernel's fp32 sample coordinate, restated op by op in fp32 (rounded after every operation), stays within the
    8 u (w + 1) that sample_bound assumes."""
    rs = np.random.RandomState(h + legacy)
    kx = np.concatenate([np.arange(8 * w, dtype=np.float32), (rs.rand(4096) * (8 * w - 1)).astype(np.float32)])
    f = np.float32
    if legacy:
        t = (kx - f(4.0) + f(0.5)) / f(w * 8.0 - 4.0 - 0.5)
        t = t * f(2) - f(1)
        ix = ((t + f(1)) / f(2)) * f(w - 1)
        ref = ((kx.astype(np.float64) - 3.5) / (8.0 * w - 4.5)) * (w - 1)
    else:
        t = kx / f(w * 8.0) * f(2) - f(1)
        ix = ((t + f(1)) * f(w) - f(1)) / f(2)
        ref = (kx.astype(np.float64) / (8.0 * w) * 2 * w - 1) / 2
    assert np.abs(ix.astype(np.float64) - ref).max() <= 8 * so.U * (w + 1)


def test_sample_bound_holds_for_fp32():
    g = torch.Generator(device="cpu").manual_seed(0)
    desc = F.normalize(torch.randn(1, 128, 20, 30, generator=g), dim=1)
    kp = torch.rand(1, 500, 2, generator=g) * torch.tensor([239.0, 159.0])
    for legacy in (True, False):
        o, bound = so.sample_bound(desc, kp, legacy)
        o32 = F.normalize(so.sample_unnormalised(desc, kp, legacy).float(), dim=-1)
        so.assert_within(o32, o, bound)
        assert float(bound.max()) < 1e-3
