"""GPU: the SuperPoint kernels (csrc/superpoint.cu) at the launches the shipped configurations make, against fp64 and
exact restatements (tests/superpoint_oracle.py), with every output between sentinel guards.

Shipped settings (glue-factory configs): homography pre-training 480x640, nms_radius 3, threshold 0, 512 forced
keypoints; MegaDepth training 1024 on the long side, 2048; evaluation 1600 on the long side, 1024; GlueStick
nms_radius 4, 1000.

Error bounds of the convolutions (element-wise, derived, no tuning constant).  With x and w the kernel's bf16 inputs,
y = conv(x, w) + b in fp64 and A = conv(|x|, |w|) + |b|:
  * the wgmma accumulation of K = ks^2 Cin exact bf16 products in fp32, each add allowed 2^-23 of a partial sum (the
    accumulator may truncate), plus the bias add: |acc - y| <= E = (K + 1) 2^-23 A;
  * ReLU epilogue: ReLU is 1-Lipschitz, then the bf16 store (unit roundoff 2^-8): E + 2^-8 (|ref| + E);
  * pooled epilogue: the max of four values moves by at most the largest of their bounds, then the bf16 store;
  * softmax epilogue: |dp_c| <= p_c (e^{2 max|dl|} - 1), plus fp32 rounding of l - m, expf (2 ulp), the 65-term sum
    and the division, relative to p;
  * L2 epilogue: |a/|a| - y/|y||_c <= (E_c + |o_c| |E|) / (|y| - |E|), plus 16 u relative for the sum of squares,
    sqrt, reciprocal and product.
conv1a is nine fp32 FMAs on the fp32 image: 10 u A, then the bf16 store.  Sampling: see sample_bound.

NMS, border removal, counting and selection are comparisons only, so they are checked bit for bit against nms_ref,
border_ref and select_ref_fast.  Worst error-to-bound ratios are printed (`-s`) for the record in
profiles/superpoint_tests_h100.md.
"""
import os
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gluefactory_b200 import _lib, synthetic  # noqa: E402
from gluefactory_b200.extractors import superpoint as sp  # noqa: E402
from tests import superpoint_oracle as so  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
RB = 4  # remove_borders of every shipped configuration


def _p(t):
    return _lib.ptr(t)


def _report(tag, ratio):
    print(f"[ratio] {tag}: {ratio:.3g}")


def _model(conf, precision="bf16"):
    m = sp.SuperPoint({"weights": None, "precision": precision, **conf})
    m.load_state_dict(synthetic.make_superpoint_weights(m.state_dict(), seed=7))
    return m.to(DEV).eval()


def _images(B, H, W, seed, warped=()):
    """B distinct gray images; those in `warped` are perspective-warped with zeros outside, as warpPerspective fills."""
    img = synthetic.make_superpoint_images(B, 1, H, W, seed=seed)
    for b in warped:
        img[b:b + 1] = so.warp_zero_fill(img[b:b + 1], seed=seed + b)
    return img.to(DEV).contiguous()


# ---- 1. launch census -----------------------------------------------------------------------------------------------
SETTINGS = {  # name: (conf, B, H, W, per-image image_size)
    "homography": ({"nms_radius": 3, "detection_threshold": 0.0, "max_num_keypoints": 512,
                    "force_num_keypoints": True}, 2, 480, 640, True),
    "megadepth": ({"nms_radius": 3, "detection_threshold": 0.0, "max_num_keypoints": 2048,
                   "force_num_keypoints": True}, 1, 768, 1024, True),
    "evaluation": ({"nms_radius": 3, "detection_threshold": 0.0, "max_num_keypoints": 1024}, 1, 1200, 1600, False),
    "gluestick": ({"nms_radius": 4, "max_num_keypoints": 1000, "force_num_keypoints": True}, 2, 480, 640, True),
}
# every entry-point signature the shipped settings launch, and the test that runs it at training size ("contract-only":
# accepted by the entry point, launched by no shipped setting, tested at its contract only)
CONV_LAYERS = [  # sp_conv: (Cin, Cout, ks, epilogue, ldx, channel offset), in dense_bf16's order
    ("1b", (64, 64, 3, sp.EP_POOL, 64, 0)), ("2a", (64, 64, 3, sp.EP_RELU, 64, 0)),
    ("2b", (64, 64, 3, sp.EP_POOL, 64, 0)), ("3a", (64, 128, 3, sp.EP_RELU, 64, 0)),
    ("3b", (128, 128, 3, sp.EP_POOL, 128, 0)), ("4a", (128, 128, 3, sp.EP_RELU, 128, 0)),
    ("4b", (128, 128, 3, sp.EP_RELU, 128, 0)), ("PaDa", (128, 512, 3, sp.EP_RELU, 128, 0)),
    ("Pb", (256, 65, 1, sp.EP_SOFTMAX, 512, 0)), ("Db", (256, 256, 1, sp.EP_L2N, 512, 256)),
]
CENSUS = {
    **{("sp_conv", sig): "test_conv_training_sizes" for _, sig in CONV_LAYERS},
    ("sp_conv1a", (1,)): "test_conv_training_sizes",
    ("sp_conv1a", (3,)): "contract-only",  # RGB input; tests/test_gpu_superpoint.py::test_conv1a
    ("sp_nms", (3, RB, True)): "test_nms_training_sizes",
    ("sp_nms", (3, RB, False)): "test_nms_training_sizes",
    ("sp_nms", (4, RB, True)): "test_nms_training_sizes",
    ("sp_select", (512, "forced", 0.0)): "test_select_sweep",
    ("sp_select", (2048, "forced", 0.0)): "test_select_sweep",
    ("sp_select", (1000, "forced", 0.005)): "test_select_sweep",
    ("sp_select", (1024, "count", 0.0)): "test_pipeline_shipped",
    ("sp_count", (0.0,)): "test_nms_training_sizes",
    ("sp_sample", (256, 1)): "test_sample",
}


def _census_run(name, precision):
    conf, B, H, W, isz = SETTINGS[name]
    m = _model(conf, precision)
    data = {"image": _images(B, H, W, seed=3)}
    if isz:
        data["image_size"] = torch.tensor([[W, H]] * B, dtype=torch.float32)
    seen, outs = [], []
    real = _lib.call

    def rec(entry, *args, **kw):
        a = [x.value if hasattr(x, "value") else x for x in args]
        if entry == "lgb200_sp_conv1a":
            seen.append(("sp_conv1a", (a[1],)))
            outs.append(a[4])
        elif entry == "lgb200_sp_conv":
            base = max(o for o in outs if o <= a[0])  # the activation this launch reads: an earlier launch's output
            seen.append(("sp_conv", (a[8], a[9], a[10], a[11], a[1], (a[0] - base) // 2)))
            outs.append(a[4])
        elif entry == "lgb200_sp_nms":
            seen.append(("sp_nms", (a[6], a[7], a[1] is not None)))
        elif entry == "lgb200_sp_select":
            seen.append(("sp_select", (a[2], "forced" if a[4] is not None else "count", round(a[1], 6))))
        elif entry == "lgb200_sp_count":
            seen.append(("sp_count", (round(a[1], 6),)))
        elif entry == "lgb200_sp_sample":
            seen.append(("sp_sample", (a[7], a[8])))
        return real(entry, *args, **kw)

    _lib.call = rec
    try:
        m(data)
        torch.cuda.synchronize()
    finally:
        _lib.call = real
    return seen


@pytest.mark.parametrize("name", list(SETTINGS))
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_launch_census(name, precision):
    seen = _census_run(name, precision)
    for row in seen:
        assert row in CENSUS, f"{name} {precision}: untabled launch {row}"
    entries = {e for e, _ in seen}
    assert {"sp_nms", "sp_select", "sp_sample"} <= entries
    assert (("sp_conv" in entries) == (precision == "bf16")) and (("sp_conv1a" in entries) == (precision == "bf16"))
    if precision == "bf16":  # the whole encoder and both heads, in order
        assert [sig for e, sig in seen if e == "sp_conv"] == [sig for _, sig in CONV_LAYERS]
    # every row that is not contract-only names a test of this file
    for row, test in CENSUS.items():
        assert test == "contract-only" or callable(globals().get(test)), (row, test)
    # and the swept parameters of those tests cover the row
    for (entry, sig), test in CENSUS.items():
        if entry == "sp_nms":
            assert sig[0] in TRAINING_RADII and sig[1] == RB
        elif entry == "sp_select" and test == "test_select_sweep":
            assert sig[0] in SELECT_K and sig[2] in SELECT_THR
        elif entry == "sp_sample":
            assert sig[0] in SAMPLE_C
        elif entry == "sp_count":
            assert sig[0] in SELECT_THR


# ---- 2. convolutions at training sizes ------------------------------------------------------------------------------
def _conv1a_ref(img, w, b):
    """fp64 ReLU(conv1a) of one gray image [1, 1, H, W] and its element-wise bound, NHWC."""
    x, w64, b64 = img.double(), w.double().view(64, 1, 3, 3), b.double()
    y = F.conv2d(x, w64, b64, padding=1)
    A = F.conv2d(x.abs(), w64.abs(), b64.abs(), padding=1)
    ref = F.relu(y)
    return ref.permute(0, 2, 3, 1), so.relu_bf16_bound(ref, 10 * so.U * A).permute(0, 2, 3, 1)


def _launch_conv(x, wk, bias, sig):
    cin, cout, ks, ep, ldx, c0 = sig
    B, H, W, _ = x.shape
    if ep == sp.EP_POOL:
        shape, dtype = (B, H // 2, W // 2, cout), torch.bfloat16
    elif ep == sp.EP_RELU:
        shape, dtype = (B, H, W, cout), torch.bfloat16
    elif ep == sp.EP_SOFTMAX:
        shape, dtype = (B, 8 * H, 8 * W), torch.float32
    else:
        shape, dtype = (B, H, W, cout), torch.float32
    g = so.Guarded(shape, dtype, DEV, guard=max(1024, shape[-1] * shape[-2]))
    _lib.call("lgb200_sp_conv", x.data_ptr() + 2 * c0, ldx, _p(wk), _p(bias), _p(g.t), B, H, W, cin, cout, ks, ep,
              _lib.stream_ptr())
    return g


def _conv_ref(xb, wk, bias, sig):
    """fp64 reference and bound of one image's launch: xb [1, H, W, ldx] bf16, wk [Npad, ks*ks*Cin] bf16."""
    cin, cout, ks, ep, ldx, c0 = sig
    x = xb[..., c0:c0 + cin].permute(0, 3, 1, 2).double()
    w = wk[:cout].view(cout, ks, ks, cin).permute(0, 3, 1, 2).double()
    b = bias[:cout].double()
    y = F.conv2d(x, w, b, padding=ks // 2)
    E = so.conv_acc_bound(F.conv2d(x.abs(), w.abs(), b.abs(), padding=ks // 2), ks * ks * cin)
    del x
    if ep == sp.EP_RELU:
        ref = F.relu(y)
        return ref.permute(0, 2, 3, 1), so.relu_bf16_bound(ref, E).permute(0, 2, 3, 1)
    if ep == sp.EP_POOL:
        ref = F.max_pool2d(F.relu(y), 2, 2)
        return ref.permute(0, 2, 3, 1), so.pool_bf16_bound(ref, E).permute(0, 2, 3, 1)
    if ep == sp.EP_SOFTMAX:
        p, bound = so.softmax_bound(y, E)
        _, _, h, w_ = p.shape

        def d2s(t):
            return t.permute(0, 2, 3, 1).reshape(1, h, w_, 8, 8).permute(0, 1, 3, 2, 4).reshape(1, 8 * h, 8 * w_)

        return d2s(p), d2s(bound)
    o, bound = so.l2n_bound(y, E)
    return o.permute(0, 2, 3, 1), bound.permute(0, 2, 3, 1)


@pytest.mark.parametrize("H,W", [(480, 640), (768, 1024), (1003, 767)])
def test_conv_training_sizes(H, W):
    """dense_bf16's launches, layer by layer, each on the kernel's own output of the layer before, against fp64; two
    distinct images, the second warped with zero fill; every launch guarded and repeated bit for bit."""
    m = _model({})
    pk = m._kernel_weights()
    img = _images(2, H, W, seed=H + W, warped=(1,))
    g = so.Guarded((2, H, W, 64), torch.bfloat16, DEV, guard=W * 64)
    _lib.call("lgb200_sp_conv1a", _p(img), 1, _p(pk["1a"][0]), _p(pk["1a"][1]), _p(g.t), 2, H, W, _lib.stream_ptr())
    g.check("conv1a")
    worst = {}
    for b in range(2):
        ref, bound = _conv1a_ref(img[b:b + 1], *pk["1a"])
        worst["1a"] = max(worst.get("1a", 0), so.assert_within(g.t[b:b + 1], ref, bound, f"conv1a image {b}"))
    x = g.t
    pd = None
    for name, sig in CONV_LAYERS:
        wk, bias = pk[name]
        src = pd if name in ("Pb", "Db") else x
        out = _launch_conv(src, wk, bias, sig)
        out.check(name)
        again = _launch_conv(src, wk, bias, sig)
        so.assert_bits_equal(again.t, out.t, f"{name} repeat")
        del again
        for b in range(2):
            ref, bound = _conv_ref(src[b:b + 1], wk, bias, sig)
            r = so.assert_within(out.t[b:b + 1], ref, bound, f"{name} {H}x{W} image {b}")
            worst[name] = max(worst.get(name, 0), r)
            del ref, bound
        if name == "PaDa":
            pd = out.t
        elif name not in ("Pb", "Db"):
            x = out.t
    for k, v in worst.items():
        _report(f"conv {k} {H}x{W}", v)


def test_conv1a_past_the_grid_cap():
    """B H W > 2^25: the grid is capped at 65535 * 16 blocks of 256 threads, so each thread loops.  The whole output
    must be written (sentinel-filled before), the first, a middle and the last image must match fp64, and a second
    launch must give the same bits (per-image position-weighted checksums)."""
    B, H, W = 112, 480, 640
    assert B * H * W > 2 ** 25
    m = _model({})
    w, bias = m._kernel_weights()["1a"]
    picks = (0, B // 2, B - 1)
    img = torch.rand(B, 1, H, W, device=DEV, generator=torch.Generator(device=DEV).manual_seed(5))
    img[list(picks)] = _images(3, H, W, seed=17, warped=(1,))
    g = so.Guarded((B, H, W, 64), torch.bfloat16, DEV, guard=W * 64)
    n_img = H * W * 64
    wpos = torch.arange(n_img, device=DEV, dtype=torch.int64) % 65521 + 1

    def launch_and_hash():
        g.ibuf.fill_(so.GUARD_BITS[torch.bfloat16])
        _lib.call("lgb200_sp_conv1a", _p(img), 1, _p(w), _p(bias), _p(g.t), B, H, W, _lib.stream_ptr())
        g.check("conv1a grid cap", full=False)
        hashes = []
        for b in range(B):
            v = g.t[b].view(torch.int16).reshape(-1)
            assert not bool((v == so.GUARD_BITS[torch.bfloat16]).any()), f"image {b} not fully written"
            hashes.append(int((v.to(torch.int64) * wpos).sum()))
        return hashes

    try:
        h1 = launch_and_hash()
        worst = 0.0
        for b in picks:
            ref, bound = _conv1a_ref(img[b:b + 1], w, bias)
            worst = max(worst, so.assert_within(g.t[b:b + 1], ref, bound, f"conv1a image {b} of {B}"))
            del ref, bound
        keep = g.t[list(picks)].clone()
        h2 = launch_and_hash()
        assert h1 == h2
        so.assert_bits_equal(g.t[list(picks)], keep, "conv1a repeat")
        _report("conv1a past the grid cap", worst)
    finally:
        del g, img
        torch.cuda.empty_cache()


# ---- 3. NMS ---------------------------------------------------------------------------------------------------------
TRAINING_RADII = (3, 4)


def _nms_launch(s, r, rb, isz):
    g = so.Guarded(tuple(s.shape), torch.float32, DEV, guard=max(64, s.shape[-1]))
    _lib.call("lgb200_sp_nms", _p(s), _p(isz), _p(g.t), s.shape[0], s.shape[1], s.shape[2], r, rb, _lib.stream_ptr())
    g.check(f"nms r={r}")
    return g.t


def _nms_check(s, r, rb, isz=None, tag=""):
    out = _nms_launch(s, r, rb, isz)
    ref = so.border_ref(so.nms_ref(s, r), rb, None if isz is None else isz.cpu())
    so.assert_bits_equal(out, ref, f"nms {tag} r={r} rb={rb} {tuple(s.shape)}")
    for thr in (0.0, 0.005, -1.0):
        c = sp.count(out, thr)
        assert c.tolist() == (ref > thr).sum(dim=(1, 2)).tolist(), (tag, thr)
    return out


def _plateau_maps(H, W, seed):
    """Random scores, quantised bumps, constant blocks and a constant map: [4, H, W] on the device."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    rnd = torch.rand(1, H, W, generator=g) ** 8 * 0.05
    return torch.cat([rnd, so.blob_map(1, H, W, seed, levels=5, n=max(4, H * W // 400)),
                      so.region_map(1, H, W, seed, cell=max(2, min(H, W) // 5)), torch.full((1, H, W), 0.02)]).to(DEV)


@pytest.mark.parametrize("r", range(10))
def test_nms_every_radius(r):
    """Sizes one below, at, one above and twice-plus-one the output tile T = 96 - 10 r, and 1, so every seam offset of
    the 5r halo runs; plateau maps; remove_borders cycling 0, 1, 4, with and without per-image sizes."""
    T = 96 - 10 * r
    sizes = sorted({1, T - 1, T, T + 1, 2 * T + 1})
    i = 0
    for H in sizes:
        for W in sizes:
            s = _plateau_maps(H, W, seed=100 * r + i)
            rb = (0, 1, 4)[i % 3]
            isz = torch.tensor([[W, H], [W - 0.5, H - 1.7], [W + 3.0, H + 3.0], [rb + 0.3, rb + 0.9]],
                               device=DEV) if i % 2 else None
            _nms_check(s, r, rb, isz, f"{H}x{W}")
            i += 1


def _extractor_map(H, W, seed):
    """The bf16 extractor's dense score map of a warped image: zero-filled corners give flat regions."""
    return _model({}).dense_bf16(_images(1, H, W, seed=seed, warped=(0,)))[0]


@pytest.mark.parametrize("H,W", [(480, 640), (768, 1024), (1200, 1600)])
def test_nms_training_sizes(H, W):
    maps = torch.cat([_extractor_map(H, W, seed=H), _plateau_maps(H, W, seed=W)[:2]])
    isz = torch.tensor([[W, H], [W - 100.6, H - 37.2], [W, H - 8]], device=DEV)
    for r in TRAINING_RADII:
        _nms_check(maps, r, RB, None, f"{H}x{W}")
        _nms_check(maps, r, RB, isz, f"{H}x{W} image_size")


@pytest.mark.parametrize("rb", [0, 1, 4])
def test_nms_border_image_size(rb):
    """Per-image sizes that are fractional (int truncation), larger than the map, and smaller than rb, so the far
    border's slice start is negative (Python wraps it) or exactly 0."""
    H, W = 61, 83
    s = _plateau_maps(H, W, seed=rb)
    s = torch.cat([s, s[:2]])  # six images
    isz = torch.tensor([[82.9, 60.99], [200.0, 300.0], [rb - 2.5, rb - 0.5], [float(rb), float(rb)], [rb + 0.7, 3.2],
                        [0.5, 1.5]], device=DEV)
    for r in (0, 3, 4):
        _nms_check(s, r, rb, isz, "image_size")


# ---- 4. selection ---------------------------------------------------------------------------------------------------
SELECT_K = (1, 2, 511, 512, 1000, 1024, 1025, 2048, 2049, 4096, 16384)
SELECT_THR = (0.0, 0.005, -1.0)


class _SelRef:
    """select_ref_fast, with each image's full (score, index) order computed once per threshold."""

    def __init__(self, s, thr):
        self.W = s.shape[-1]
        self.full = so.select_ref_fast(s, thr, -1)  # row-major
        self.sorted = []
        for kp, sc in self.full:
            idx = (kp[:, 1].long() * self.W + kp[:, 0].long()).numpy()
            order = np.lexsort((idx, -sc.numpy()))
            self.sorted.append((kp[order], sc[order]))

    def __call__(self, b, k):
        n = len(self.full[b][1])
        return self.sorted[b] if 0 < k < n else self.full[b]

    def count(self, b):
        return len(self.full[b][1])


def _select_launch(s, thr, k, cap, uniform=None, pad_hi=None):
    B = s.shape[0]
    gk = so.Guarded((B, cap, 2), torch.float32, DEV)
    gs = so.Guarded((B, cap), torch.float32, DEV)
    gc = so.Guarded((B,), torch.int32, DEV)
    _lib.call("lgb200_sp_select", _p(s), float(thr), int(k), int(cap), _p(uniform), _p(pad_hi), _p(gk.t), _p(gs.t),
              _p(gc.t), B, s.shape[1], s.shape[2], _lib.stream_ptr())
    for g, t in ((gk, "keypoints"), (gs, "scores"), (gc, "counts")):
        g.check(f"select k={k} {t}", full=uniform is not None or t == "counts")
    return gk.t, gs.t, gc.t


def _select_maps():
    """B = 4 post-NMS maps at 480x640: a warped extractor map, quantised bumps (plateau maxima survive NMS as ties), a
    constant map (every cell kept, one tie group over the whole image), all through the NMS kernel; then 300 isolated
    peaks on a floor of -1, and a map of -1 alone: no candidate at any threshold."""
    H, W = 480, 640
    ext = _extractor_map(H, W, seed=11)
    blobs = so.blob_map(1, H, W, seed=12, levels=5, n=600).to(DEV)
    const = torch.full((1, H, W), 0.02, device=DEV)
    sparse = torch.full((1, H, W), -1.0, device=DEV)  # below every threshold: only the peaks are candidates
    g = torch.Generator(device="cpu").manual_seed(13)
    ys, xs = torch.randint(8, H - 8, (300,), generator=g), torch.randint(8, W - 8, (300,), generator=g)
    sparse[0, ys, xs] = torch.rand(300, generator=g).to(DEV) * 0.1 + 0.01
    return torch.cat([_nms_check(torch.cat([ext, blobs, const]), 3, RB, None, "selection maps"), sparse,
                      torch.full((1, H, W), -1.0, device=DEV)])


@pytest.mark.parametrize("thr", SELECT_THR)
def test_select_sweep(thr):
    s = _select_maps()
    ref = _SelRef(s, thr)
    B = s.shape[0]
    counts = [ref.count(b) for b in range(B)]
    assert counts[4] == 0 and 0 < counts[3] < 512 and counts[2] > 16384
    if thr >= 0:  # at -1 every cell NMS returns (suppressed ones score 0) is a candidate: the three NMS maps tie
        assert len(set(counts)) == B
    ks = list(SELECT_K) + [c + d for c in counts[:4] for d in (-1, 0, 1) if 0 < c + d <= sp.MAX_K]
    u = torch.rand(B, max(ks), 2, device=DEV, generator=torch.Generator(device=DEV).manual_seed(1))
    pad_hi = torch.full((1,), 480.0, device=DEV)
    ties_cut = 0
    for k in sorted(set(ks)):
        kp, sc, cnt = _select_launch(s, thr, k, k, u[:, :k].contiguous(), pad_hi)
        for b in range(B):
            r = ref(b, k)
            n = min(len(r[1]), k)
            so.assert_selection(kp[b], sc[b], cnt[b], r, f"thr={thr} k={k} image {b}")
            pad = kp[b, n:]
            assert bool((sc[b, n:] == 0).all())
            if n:
                lo, hi = kp[b, :n].min(0).values, kp[b, :n].max(0).values
                assert bool(((pad >= lo) & (pad <= hi)).all()), (k, b)
            else:
                assert bool(((pad >= 0) & (pad < 480.0)).all()), (k, b)
            if b == 2:  # the tie fixture: one tie group over the whole image, cut by every k
                eq, taken, chunks = so.tie_stats(s[b], thr, k)
                assert eq > taken >= 1 and len(chunks) > 1, (k, b, eq, taken, chunks[:4])
                ties_cut += 1
        # the non-forced launch: cap = the kept count, nothing written past it
        if k in (512, 1024, 2048):
            cap = max(1, min(counts[0], k))
            kp1, sc1, cnt1 = _select_launch(s[:1], thr, k, cap)
            so.assert_selection(kp1[0], sc1[0], cnt1[0], ref(0, k), f"thr={thr} k={k} cap={cap}")
    assert ties_cut >= len(SELECT_K)


# ---- 5. sampling ----------------------------------------------------------------------------------------------------
SAMPLE_C = (256, 128)


@pytest.mark.parametrize("C", SAMPLE_C)
@pytest.mark.parametrize("legacy", [True, False])
@pytest.mark.parametrize("h,w", [(60, 80), (96, 128), (150, 200)])
def test_sample(C, legacy, h, w):
    B, K = 4, 2048
    g = torch.Generator(device="cpu").manual_seed(C + h + legacy)
    desc = F.normalize(torch.randn(B, h, w, C, generator=g), dim=-1)
    ints = torch.stack([torch.randint(0, 8 * w, (B, K // 2), generator=g),
                        torch.randint(0, 8 * h, (B, K // 2), generator=g)], -1).float()
    ints[:, :4] = torch.tensor([[0, 0], [8 * w - 1, 8 * h - 1], [8 * w - 1, 0], [0, 8 * h - 1]], dtype=torch.float32)
    ints[:, 4:8, 0] = 8 * w - 1  # last column
    ints[:, 8:12, 1] = 8 * h - 1  # last row
    sub = torch.rand(B, K // 2, 2, generator=g) * torch.tensor([8 * w - 1.0, 8 * h - 1.0])
    kp = torch.cat([ints, sub], 1).contiguous()
    out = so.Guarded((B, K, C), torch.float32, DEV, guard=C)
    _lib.call("lgb200_sp_sample", _p(desc.to(DEV)), _p(kp.to(DEV)), _p(out.t), B, K, h, w, C, int(legacy),
              _lib.stream_ptr())
    out.check("sample")
    ref, bound = so.sample_bound(desc.permute(0, 3, 1, 2), kp, legacy)
    _report(f"sample C={C} legacy={legacy} {h}x{w}", so.assert_within(out.t.cpu(), ref, bound, "sample"))


# ---- 6. the pipeline at the shipped settings --------------------------------------------------------------------------
PIPELINES = {  # name: (conf, B, H, W, warped, image sizes or None, train mode)
    "homography": ({"nms_radius": 3, "detection_threshold": 0.0, "max_num_keypoints": 512,
                    "force_num_keypoints": True}, 4, 480, 640, (1, 3),
                   [[640, 480], [600.5, 470.2], [640, 480], [512, 400]], True),
    "homography_val": ({"nms_radius": 3, "detection_threshold": 0.0, "max_num_keypoints": 512,
                        "max_num_keypoints_val": 1024, "force_num_keypoints": True}, 2, 480, 640, (0,),
                       [[640, 480], [630.0, 475.0]], False),
    "megadepth": ({"nms_radius": 3, "detection_threshold": 0.0, "max_num_keypoints": 2048,
                   "force_num_keypoints": True}, 2, 768, 1024, (1,), [[1024, 768], [1024, 700]], True),
    "evaluation": ({"nms_radius": 3, "detection_threshold": 0.0, "max_num_keypoints": 1024}, 1, 1200, 1600, (), None,
                   False),
}


def _check_sparse(pred, scores, desc, conf, k, isz, forced, tag):
    """The plugin's keypoints and scores against the restatement on its own dense maps, bit for bit in the kept slots;
    descriptors within sample_bound."""
    s_ref = so.border_ref(so.nms_ref(scores, conf["nms_radius"]), RB, None if isz is None else isz.cpu())
    ref = so.select_ref_fast(s_ref, conf.get("detection_threshold", 0.005), k)
    worst = 0.0
    for b, (kp, sc) in enumerate(ref):
        n = min(len(sc), pred["keypoints"].shape[1])
        assert n > 0
        so.assert_bits_equal(pred["keypoints"][b, :n].cpu() - 0.5, kp[:n], f"{tag} image {b} keypoints")
        so.assert_bits_equal(pred["keypoint_scores"][b, :n].cpu(), sc[:n], f"{tag} image {b} scores")
        if forced:
            assert bool((pred["keypoint_scores"][b, n:] == 0).all())
        else:
            assert pred["keypoints"].shape[1] == n
        o, bound = so.sample_bound(desc[b:b + 1].permute(0, 3, 1, 2).cpu(), kp[None, :n], conf.get("legacy_sampling",
                                                                                                      True))
        worst = max(worst, so.assert_within(pred["descriptors"][b:b + 1, :n].cpu(), o, bound, f"{tag} descriptors"))
    return [min(len(sc), pred["keypoints"].shape[1]) for _, sc in ref], worst


@pytest.mark.parametrize("name", list(PIPELINES))
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_pipeline_shipped(name, precision):
    conf, B, H, W, warped, sizes, train = PIPELINES[name]
    m = _model(conf, precision)
    m.train(train)
    k = conf["max_num_keypoints"] if train or "max_num_keypoints_val" not in conf else conf["max_num_keypoints_val"]
    forced = conf.get("force_num_keypoints", False)
    img = _images(B, H, W, seed=H + B, warped=warped)
    data = {"image": img}
    isz = None
    if sizes is not None:
        isz = torch.tensor(sizes, dtype=torch.float32)
        data["image_size"] = isz
    pred = m(data)
    scores, desc = (m.dense_bf16 if precision == "bf16" else m.dense_fp32)(img)
    assert pred["keypoints"].shape[1] == (k if forced else pred["keypoints"].shape[1])
    kept, worst = _check_sparse(pred, scores, desc, conf, k, isz, forced, f"{name} {precision}")
    _report(f"pipeline {name} {precision} descriptors", worst)
    # each image alone gives the bits it gets inside the batch: the sparse kernels on its slice of the dense maps, and
    # (bf16, all our kernels) the whole forward
    for b in range(B):
        n = kept[b]
        db = {"image": img[b:b + 1]}
        if isz is not None:
            db["image_size"] = isz[b:b + 1]
        alone = [m._sparse(db, img[b:b + 1], scores[b:b + 1], desc[b:b + 1])]
        if precision == "bf16":
            alone.append(m(db))
        for a in alone:
            for key in ("keypoints", "keypoint_scores", "descriptors"):
                so.assert_bits_equal(a[key][0, :n], pred[key][b, :n], f"{name} image {b} alone {key}")
