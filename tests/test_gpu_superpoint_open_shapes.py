"""GPU: the SuperPoint-open BatchNorm paths (csrc/superpoint.cu `spo_*`, lgb200_bn_stats and
lgb200_bn_running_update) at the launches and batches the shipped configurations make, against fp64 with the derived
bounds of tests/superpoint_open_oracle.py, with every output between sentinel guards.

Shipped settings (glue-factory configs): superpoint-open+lightglue_homography, 128 RGB images at 480x640 per view in
training mode (threshold -1, nms_radius 3, 512 forced keypoints); superpoint-open+lightglue_megadepth, 32 RGB images at
1024x1024 (2048 keypoints); evaluation in eval mode, one image, 1024 keypoints, up to 1600 on the long side;
freeze_batch_normalization training, which takes the eval-mode path.

  1. launch census: every entry-point signature these settings make, each a row naming the test that runs it;
  2. eval mode: the folded BatchNorm epilogues layer by layer at 480x640, 1024x1024 and 1003x767;
  3. training mode at B = 128 x 480x640 and B = 32 x 1024x1024: the batch sums, the running update and the
     normalisation of every BatchNorm, with a dead, a constant and a large-mean channel in every layer;
  4. conv1a on RGB past the grid cap;
  5. whole-batch calls past element 2^31 (training, B = 128) and 2^32 (eval, B = 256) against calls on slices of the
     batch, bit for bit.

Worst error-to-bound ratios are printed with `-s` ("[ratio]"), and each test's time and peak memory ("[cost]"), for the
record in profiles/superpoint_open_tests_h100.md.

The synthetic BatchNorms have running_mean of both signs, running_var spread log-uniformly over 1e-3 to 1e2, and
weights of both signs, every eighth one near zero.  The other weights scale with sqrt(running_var), so the folded scale
stays O(1) and activations keep their size through the twelve layers: otherwise the score logits saturate the softmax
and its check says little.
"""
import os
import sys
import time
import types

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gluefactory_b200 import _lib, ops, synthetic  # noqa: E402
from gluefactory_b200.extractors import superpoint_open as spo  # noqa: E402
from tests import superpoint_open_oracle as oo  # noqa: E402
from tests import superpoint_oracle as so  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS = 1e-3  # every SuperPoint-open BatchNorm
GRAY = (0.299, 0.587, 0.114)


def _p(t):
    return _lib.ptr(t)


def _report(tag, ratio):
    print(f"[ratio] {tag}: {ratio:.3g}")


@pytest.fixture(autouse=True)
def _cost(request):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    torch.cuda.synchronize()
    print(f"[cost] {request.node.name}: {time.perf_counter() - t0:.1f} s, peak "
          f"{torch.cuda.max_memory_allocated() / 2 ** 30:.2f} GiB")
    torch.cuda.empty_cache()


@pytest.fixture(scope="module")
def weights_path(tmp_path_factory):
    path = tmp_path_factory.mktemp("w") / "sp_open.pth"
    torch.save(synthetic.make_superpoint_open_weights(spo.SuperPointOpen.state_dict_template(), seed=11), path)
    return str(path)


def _bn_buffers(m, seed):
    """running_mean U(-1, 1); running_var log-uniform on [1e-3, 1e2]; weight of either sign, |weight| in
    [0.5, 1.5] sqrt(running_var), every eighth one in (-1e-3, 1e-3); bias U(-0.2, 0.2)."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for bn in m._batchnorms():
            C = bn.num_features
            rv = 10.0 ** (torch.rand(C, generator=g) * 5 - 3)
            w = (torch.rand(C, generator=g) + 0.5) * torch.sqrt(rv) * (torch.randint(0, 2, (C,), generator=g) * 2 - 1)
            w[::8] = (torch.rand(w[::8].shape, generator=g) * 2 - 1) * 1e-3
            bn.running_mean.copy_(torch.rand(C, generator=g) * 2 - 1)
            bn.running_var.copy_(rv)
            bn.weight.copy_(w)
            bn.bias.copy_((torch.rand(C, generator=g) * 2 - 1) * 0.2)
    return m


def _model(weights_path, conf=None, train=False, precision="bf16", seed=5, sync=False):
    m = spo.SuperPointOpen({**(conf or {}), "weights": weights_path, "precision": precision})
    _bn_buffers(m, seed)
    if sync:
        m = torch.nn.SyncBatchNorm.convert_sync_batchnorm(m)
    return m.to(DEV).train(train)


def _images(B, C, H, W, seed, warped=()):
    """B distinct images in [0, 1] on the device: four synthetic bases, each image shifted, scaled and given its own
    noise; those in `warped` perspective-warped with zero fill."""
    base = synthetic.make_superpoint_images(4, C, H, W, seed=seed).to(DEV)
    g = torch.Generator(device=DEV).manual_seed(seed)
    img = torch.empty(B, C, H, W, device=DEV)
    for b in range(B):
        img[b] = torch.roll(base[b % 4], shifts=((7 * b) % H, (13 * b) % W), dims=(-2, -1))
    img.mul_(torch.rand(B, 1, 1, 1, generator=g, device=DEV) * 0.5 + 0.5)
    img.add_(torch.rand(B, C, H, W, generator=g, device=DEV) * 0.05).clamp_(0, 1)
    for b in warped:
        img[b:b + 1] = so.warp_zero_fill(img[b:b + 1], seed=seed + b)
    return img.contiguous()


def _gray32(img):
    """The kernels' gray conversion, rounded per operation: (r .299 + g .587) + b .114 in fp32."""
    if img.shape[1] == 1:
        return img
    c = [torch.tensor(v, dtype=torch.float32, device=img.device) for v in GRAY]
    return (img[:, 0:1] * c[0] + img[:, 1:2] * c[1]) + img[:, 2:3] * c[2]


def _written(g, B, tag):
    """Both guards intact and, image by image, no sentinel left in the output."""
    g.check(tag, full=False)
    pat = so.GUARD_BITS[g.dtype]
    flat = g.ibuf[g.guard:g.guard + g.n].view(B, -1)
    step = max(1, (1 << 28) // flat.shape[1])
    for b0 in range(0, B, step):
        left = (flat[b0:b0 + step] == pat).any(1)
        assert not bool(left.any()), f"{tag}: image {b0 + int(torch.nonzero(left)[0])} not fully written"


def _hashes(g, B):
    """Per-image position-weighted checksums of a guarded output's bits."""
    flat = g.ibuf[g.guard:g.guard + g.n].view(B, -1)
    w = torch.arange(flat.shape[1], device=DEV, dtype=torch.int64) % 65521 + 1
    return [int((flat[b].to(torch.int64) * w).sum()) for b in range(B)]


# ---- launches into guarded outputs -----------------------------------------------------------------------------------
def _conv1a(img, w, b, scale=None, shift=None):
    B, C, H, W = img.shape
    g = so.Guarded((B, H, W, 64), torch.bfloat16, DEV, guard=W * 64)
    if scale is None:
        _lib.call("lgb200_sp_conv1a", _p(img), C, _p(w), _p(b), _p(g.t), B, H, W, _lib.stream_ptr())
    else:
        _lib.call("lgb200_spo_conv1a", _p(img), C, _p(w), _p(b), _p(scale), _p(shift), _p(g.t), B, H, W,
                  _lib.stream_ptr())
    return g


def _conv(x, w, b, sig, scale=None, shift=None):
    """sig = (cin, cout, ks, epilogue, ldx, c0, affine): lgb200_spo_conv when affine or raw, else lgb200_sp_conv."""
    cin, cout, ks, ep, ldx, c0, aff = sig
    B, H, W, _ = x.shape
    assert x.shape[-1] == ldx
    shape, dtype = {spo.EP_POOL: ((B, H // 2, W // 2, cout), torch.bfloat16),
                    spo.EP_RELU: ((B, H, W, cout), torch.bfloat16),
                    spo.EP_SOFTMAX: ((B, 8 * H, 8 * W), torch.float32),
                    spo.EP_L2N: ((B, H, W, cout), torch.float32),
                    spo.EP_RAW: ((B, H, W, -(-cout // 128) * 128), torch.float32)}[ep]
    g = so.Guarded(shape, dtype, DEV, guard=max(1024, shape[-1] * shape[-2]))
    if aff or ep == spo.EP_RAW:
        _lib.call("lgb200_spo_conv", x.data_ptr() + 2 * c0, ldx, _p(w), _p(b), _p(scale), _p(shift), _p(g.t), B, H, W,
                  cin, cout, ks, ep, _lib.stream_ptr())
    else:
        _lib.call("lgb200_sp_conv", x.data_ptr() + 2 * c0, ldx, _p(w), _p(b), _p(g.t), B, H, W, cin, cout, ks, ep,
                  _lib.stream_ptr())
    return g


def _bn_apply(y, sums, bn, op):
    B, H, W, _ = y.shape
    C = bn.num_features
    shape, dtype = {spo.BN_PLAIN: ((B, H, W, C), torch.bfloat16), spo.BN_POOL: ((B, H // 2, W // 2, C), torch.bfloat16),
                    spo.BN_SOFTMAX: ((B, 8 * H, 8 * W), torch.float32), spo.BN_L2N: ((B, H, W, C), torch.float32)}[op]
    g = so.Guarded(shape, dtype, DEV, guard=max(1024, shape[-1] * shape[-2]))
    _lib.call("lgb200_spo_bn_apply", _p(y), _p(sums), _p(bn.weight.float().contiguous()),
              _p(bn.bias.float().contiguous()), float(bn.eps), _p(g.t), B, H, W, C, int(op), _lib.stream_ptr())
    return g


def _d2s(p):
    """[1, 64, h, w] -> the depth-to-space score map [1, 8h, 8w]."""
    _, _, h, w = p.shape
    return p.permute(0, 2, 3, 1).reshape(1, h, w, 8, 8).permute(0, 1, 3, 2, 4).reshape(1, 8 * h, 8 * w)


# ---- 1. launch census ------------------------------------------------------------------------------------------------
HOMOGRAPHY = {"max_num_keypoints": 512, "force_num_keypoints": True, "detection_threshold": -1, "nms_radius": 3}
MEGADEPTH = {"max_num_keypoints": 2048, "force_num_keypoints": True, "detection_threshold": -1, "nms_radius": 3}
SETTINGS = {  # name: (conf, B, image channels, H, W, training)
    "homography": (HOMOGRAPHY, 2, 3, 480, 640, True),
    "megadepth": (MEGADEPTH, 2, 3, 1024, 1024, True),
    "frozen": ({**HOMOGRAPHY, "freeze_batch_normalization": True}, 2, 3, 480, 640, True),
    "hpatches": ({"max_num_keypoints": 1024, "detection_threshold": -1, "nms_radius": 3}, 1, 1, 480, 640, False),
    "megadepth1500": ({"max_num_keypoints": 2048, "detection_threshold": -1, "nms_radius": 3}, 1, 3, 1200, 1600,
                      False),
}
R, P, S, L, RAW = spo.EP_RELU, spo.EP_POOL, spo.EP_SOFTMAX, spo.EP_L2N, spo.EP_RAW
# eval mode (running statistics, also freeze_batch_normalization): dense_bf16's conv launches, in order, as
# (cin, cout, ks, epilogue, ldx, channel offset, affine)
EVAL_CONVS = [("1b", (64, 64, 3, P, 64, 0, True)), ("2a", (64, 64, 3, R, 64, 0, True)),
              ("2b", (64, 64, 3, P, 64, 0, True)), ("3a", (64, 128, 3, R, 64, 0, True)),
              ("3b", (128, 128, 3, P, 128, 0, True)), ("4a", (128, 128, 3, R, 128, 0, True)),
              ("4b", (128, 128, 3, R, 128, 0, True)), ("PaDa", (128, 512, 3, R, 128, 0, True)),
              ("Pb", (256, 65, 1, S, 512, 0, True)), ("Db", (256, 256, 1, L, 512, 256, True))]
BF16, F32 = _lib.BF16, _lib.F32
# training mode: per BatchNorm, the conv writing the pre-BatchNorm activation (ReLU'd bf16, or raw fp32 logits for the
# heads), then bn_stats (C, dtype), bn_running_update (C, momentum) and spo_bn_apply (op, C)
TRAIN_LAYERS = [  # (name, conv signature, stats signature, bn C, apply op)
    ("1a", None, (64, BF16), 64, spo.BN_PLAIN), ("1b", (64, 64, 3, R, 64, 0, False), (64, BF16), 64, spo.BN_POOL),
    ("2a", (64, 64, 3, R, 64, 0, False), (64, BF16), 64, spo.BN_PLAIN),
    ("2b", (64, 64, 3, R, 64, 0, False), (64, BF16), 64, spo.BN_POOL),
    ("3a", (64, 128, 3, R, 64, 0, False), (128, BF16), 128, spo.BN_PLAIN),
    ("3b", (128, 128, 3, R, 128, 0, False), (128, BF16), 128, spo.BN_POOL),
    ("4a", (128, 128, 3, R, 128, 0, False), (128, BF16), 128, spo.BN_PLAIN),
    ("4b", (128, 128, 3, R, 128, 0, False), (128, BF16), 128, spo.BN_PLAIN),
    ("Pa", (128, 256, 3, R, 128, 0, False), (256, BF16), 256, spo.BN_PLAIN),
    ("Da", (128, 256, 3, R, 128, 0, False), (256, BF16), 256, spo.BN_PLAIN),
    ("Pb", (256, 65, 1, RAW, 256, 0, False), (128, F32), 65, spo.BN_SOFTMAX),
    ("Db", (256, 256, 1, RAW, 256, 0, False), (256, F32), 256, spo.BN_L2N),
]


def _expected(training, C):
    if not training:
        return [("spo_conv1a", (C, True))] + [("spo_conv", sig) for _, sig in EVAL_CONVS]
    rows = []
    for name, sig, stats, c, op in TRAIN_LAYERS:
        rows.append(("sp_conv1a", (C, False)) if sig is None else ("spo_conv" if sig[3] == RAW else "sp_conv", sig))
        rows += [("bn_stats", stats), ("bn_running_update", (c, 0.1)), ("spo_bn_apply", (op, c))]
    return rows


T_EVAL, T_TRAIN = "test_eval_epilogues_training_sizes", "test_training_chain"
T_CAP = "test_conv1a_rgb_past_the_grid_cap"
CENSUS = {
    ("spo_conv1a", (3, True)): T_EVAL + ", " + T_CAP,
    ("spo_conv1a", (1, True)): T_EVAL,
    ("sp_conv1a", (3, False)): T_TRAIN + ", " + T_CAP,
    **{("spo_conv", sig): T_EVAL for _, sig in EVAL_CONVS},
    **{("spo_conv" if sig[3] == RAW else "sp_conv", sig): T_TRAIN for _, sig, _, _, _ in TRAIN_LAYERS if sig},
    **{("bn_stats", st): T_TRAIN for _, _, st, _, _ in TRAIN_LAYERS},
    **{("bn_running_update", (c, 0.1)): T_TRAIN for _, _, _, c, _ in TRAIN_LAYERS},
    **{("spo_bn_apply", (op, c)): T_TRAIN for _, _, _, c, op in TRAIN_LAYERS},
}
CONV_ENTRIES = {"sp_conv1a", "spo_conv1a", "sp_conv", "spo_conv"}


def _census_run(name, precision, weights_path):
    conf, B, C, H, W, training = SETTINGS[name]
    m = _model(weights_path, conf, train=training, precision=precision)
    img = _images(B, C, H, W, seed=3)
    seen, outs = [], []
    real = _lib.call

    def offset(x, ldx):
        """The channel offset of a conv's input: into the latest earlier output that starts less than one pixel
        (ldx bf16 channels) before it."""
        base = next(o for o in reversed(outs) if 0 <= x - o < 2 * ldx)
        return (x - base) // 2

    def rec(entry, *args, **kw):
        a = [x.value if hasattr(x, "value") else x for x in args]
        if entry in ("lgb200_sp_conv1a", "lgb200_spo_conv1a"):
            aff = entry == "lgb200_spo_conv1a"
            seen.append((entry[7:], (a[1], aff)))
            outs.append(a[6] if aff else a[4])
        elif entry == "lgb200_sp_conv":
            seen.append(("sp_conv", (a[8], a[9], a[10], a[11], a[1], offset(a[0], a[1]), False)))
            outs.append(a[4])
        elif entry == "lgb200_spo_conv":
            seen.append(("spo_conv", (a[10], a[11], a[12], a[13], a[1], offset(a[0], a[1]), a[4] is not None)))
            outs.append(a[6])
        elif entry == "lgb200_bn_stats":
            seen.append(("bn_stats", (a[5], a[6])))
        elif entry == "lgb200_bn_running_update":
            seen.append(("bn_running_update", (a[4], round(a[3], 6))))
        elif entry == "lgb200_spo_bn_apply":
            seen.append(("spo_bn_apply", (a[10], a[9])))
            outs.append(a[5])
        return real(entry, *args, **kw)

    _lib.call = ops.call = rec  # ops binds `call` at import (bn_stats, bn_running_update)
    try:
        with torch.no_grad():
            m({"image": img})
        torch.cuda.synchronize()
    finally:
        _lib.call = ops.call = real
    return seen


@pytest.mark.parametrize("name", list(SETTINGS))
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_launch_census(name, precision, weights_path):
    conf, B, C, H, W, training = SETTINGS[name]
    seen = _census_run(name, precision, weights_path)
    for row in seen:
        assert row in CENSUS, f"{name} {precision}: untabled launch {row}"
    if precision == "fp32":  # the parity path runs the module's own torch layers
        assert not any(e in CONV_ENTRIES or e == "spo_bn_apply" for e, _ in seen), seen
    else:  # the whole layer sequence, in dense_bf16's order
        batch_stats = training and not conf.get("freeze_batch_normalization")
        assert seen == _expected(batch_stats, C), seen
    for row, tests in CENSUS.items():  # every row names tests of this file, or says contract-only with a reason
        for t in tests.split(", "):
            assert t.startswith("contract-only") or callable(globals().get(t)), (row, t)


# ---- 2. eval mode: the folded epilogues at training sizes ------------------------------------------------------------
def _eval_bn(m):
    """name -> (weight, bias, running_mean, running_var) of the BatchNorm each eval launch folds; PaDa's the
    concatenation of Pa's and Da's."""
    bns = {n: b.bn for n, b in zip(["1a", "1b", "2a", "2b", "3a", "3b", "4a", "4b"], m._blocks())}
    bns.update(Pa=m.detector[0].bn, Pb=m.detector[1].bn, Da=m.descriptor[0].bn, Db=m.descriptor[1].bn)
    out = {k: (b.weight, b.bias, b.running_mean, b.running_var) for k, b in bns.items()}
    out["PaDa"] = tuple(torch.cat([a, d]) for a, d in zip(out["Pa"], out["Da"]))
    return out


def _eval_affines(m):
    """The plugin's own bn_affine output per launch, as dense_bf16 passes it."""
    blocks = m._blocks()
    aff = {n: spo.bn_affine(b.bn) for n, b in zip(["1a", "1b", "2a", "2b", "3a", "3b", "4a", "4b"], blocks)}
    (pa, pb), (da, db) = m.detector, m.descriptor
    aff["PaDa"] = tuple(torch.cat([a, d]) for a, d in zip(spo.bn_affine(pa.bn), spo.bn_affine(da.bn)))
    aff["Pb"] = tuple(F.pad(t, (0, 128 - 65)) for t in spo.bn_affine(pb.bn))
    aff["Db"] = spo.bn_affine(db.bn)
    return aff


def _conv1a_eval_ref(img, w, b, bn):
    """fp64 BatchNorm(ReLU(conv1a)) of one image [1, C, H, W] (gray rounded as the kernel rounds it) and its bound,
    NHWC: nine fp32 FMAs (10 u A), the folded affine, the bf16 store."""
    x, w64, b64 = _gray32(img).double(), w.double().view(64, 1, 3, 3), b.double()
    y = F.conv2d(x, w64, b64, padding=1)
    E = 10 * oo.U * F.conv2d(x.abs(), w64.abs(), b64.abs(), padding=1)
    z, e = oo.folded_affine(F.relu(y), E, *bn, EPS)
    return z.permute(0, 2, 3, 1), oo.relu_bf16_bound(z, e).permute(0, 2, 3, 1)


def _conv_eval_ref(xb, wk, bias, sig, bn):
    """fp64 reference and bound of one image's eval-mode launch: xb [1, H, W, ldx] bf16, wk [Npad, ks*ks*cin]."""
    cin, cout, ks, ep, ldx, c0, _ = sig
    x = xb[..., c0:c0 + cin].permute(0, 3, 1, 2).double()
    w = wk[:cout].view(cout, ks, ks, cin).permute(0, 3, 1, 2).double()
    b = bias[:cout].double()
    y = F.conv2d(x, w, b, padding=ks // 2)
    E = so.conv_acc_bound(F.conv2d(x.abs(), w.abs(), b.abs(), padding=ks // 2), ks * ks * cin)
    del x
    bn = tuple(t[:cout] for t in bn)
    if ep == R:
        z, e = oo.folded_affine(F.relu(y), E, *bn, EPS)
        return z.permute(0, 2, 3, 1), oo.relu_bf16_bound(z, e).permute(0, 2, 3, 1)
    if ep == P:  # the max of the affine values: with negative scales, not the affine of the max
        z, e = oo.folded_affine(F.relu(y), E, *bn, EPS)
        zp = F.max_pool2d(z, 2, 2)
        return zp.permute(0, 2, 3, 1), oo.pool_bf16_bound(zp, e).permute(0, 2, 3, 1)
    z, e = oo.folded_affine(y, E, *bn, EPS)
    if ep == S:
        p, bound = oo.softmax_bound(z, e)
        return _d2s(p), _d2s(bound)
    o, bound = oo.l2n_bound(z, e)
    return o.permute(0, 2, 3, 1), bound.permute(0, 2, 3, 1)


@pytest.mark.parametrize("H,W,C", [(480, 640, 3), (1024, 1024, 3), (1003, 767, 1)])
def test_eval_epilogues_training_sizes(H, W, C, weights_path):
    """dense_bf16's eval-mode launches layer by layer, each on the kernel's own output of the layer before, with the
    plugin's own bn_affine, against the unfolded fp64 BatchNorm; two images, the second warped with zero fill; every
    launch guarded and repeated bit for bit."""
    m = _model(weights_path)
    pk = m._kernel_weights()
    aff, bns = _eval_affines(m), _eval_bn(m)
    img = _images(2, C, H, W, seed=H + W, warped=(1,))
    w1, b1 = pk["enc"][0]
    g = _conv1a(img, w1, b1, *aff["1a"])
    _written(g, 2, "conv1a")
    so.assert_bits_equal(_conv1a(img, w1, b1, *aff["1a"]).t, g.t, "conv1a repeat")
    worst = {}
    for b in range(2):
        ref, bound = _conv1a_eval_ref(img[b:b + 1], w1, b1, bns["1a"])
        worst["1a"] = max(worst.get("1a", 0), so.assert_within(g.t[b:b + 1], ref, bound, f"conv1a image {b}"))
    weights = dict(zip(["1b", "2a", "2b", "3a", "3b", "4a", "4b"], pk["enc"][1:]))
    weights.update(PaDa=pk["PaDa"], Pb=pk["Pb"], Db=pk["Db"])
    x, pd = g.t, None
    for name, sig in EVAL_CONVS:
        wk, bias = weights[name]
        src = pd if name in ("Pb", "Db") else x
        out = _conv(src, wk, bias, sig, *aff[name])
        _written(out, 2, name)
        so.assert_bits_equal(_conv(src, wk, bias, sig, *aff[name]).t, out.t, f"{name} repeat")
        for b in range(2):
            ref, bound = _conv_eval_ref(src[b:b + 1], wk, bias, sig, bns[name])
            r = so.assert_within(out.t[b:b + 1], ref, bound, f"{name} {H}x{W} image {b}")
            worst[name] = max(worst.get(name, 0), r)
            del ref, bound
        if name == "PaDa":
            pd = out.t
        elif name not in ("Pb", "Db"):
            x = out.t
    for k, v in worst.items():
        _report(f"eval {k} {H}x{W}", v)


# ---- 3. training mode at the shipped batches -------------------------------------------------------------------------
DEAD, CONST, BIGMEAN = 0, 1, 2  # edited output channels of every conv


def _edge_channels(m):
    """In every conv: channel 0 dead (zero weights; bias -0.5 before a ReLU, 0 in the heads' raw logits), channel 1
    constant (zero weights, bias 0.75: variance exactly 0), channel 2 with mean about 6 and a spread about a hundred
    times smaller (weights scaled by 0.01, bias 6)."""
    convs = [b.conv for b in m._blocks()] + [m.detector[0].conv, m.descriptor[0].conv, m.detector[1].conv,
                                             m.descriptor[1].conv]
    with torch.no_grad():
        for i, c in enumerate(convs):
            head = i >= 10
            c.weight[DEAD] = 0
            c.bias[DEAD] = 0.0 if head else -0.5
            c.weight[CONST] = 0
            c.bias[CONST] = 0.75
            c.weight[BIGMEAN] *= 0.01
            c.bias[BIGMEAN] = 6.0


def _stats(y, C):
    """Two passes of fp64 statistics over the first C channels of y [B, h, w, ld], in chunks of images."""
    B = y.shape[0]
    step = max(1, (1 << 26) // (y[0].numel()))
    st = oo.Stats(C, y.device)
    for b0 in range(0, B, step):
        st.add(y[b0:b0 + step, ..., :C])
    for b0 in range(0, B, step):
        st.add_centred(y[b0:b0 + step, ..., :C])
    return st


def _check_bn(y, bn, op, picks, worst, tag, momenta=(0.1, 0.37)):
    """One training-mode BatchNorm on the kernel's own pre-BatchNorm activation y: bn_stats against fp64 sums, the
    running update against torch's formula in fp64 (at each momentum, the first on the module itself), and
    spo_bn_apply on the picked images against fp64 BatchNorm with the fp64 statistics, every image written and a
    second launch with the same per-image checksums.  Returns the guarded output."""
    B, h, w, ld = y.shape
    C = bn.num_features
    st = _stats(y, C)
    sums = ops.bn_stats(y.view(-1, ld))
    if ld != C:  # Pb's padded logits: the plugin's 65-of-128 slice
        sums = torch.cat([sums[:C], sums[ld:ld + C], sums[2 * ld:]])
    assert float(sums[2 * C]) == st.n == B * h * w
    r = so.assert_within(sums, st.sums(), st.sum_bound(), f"{tag} bn_stats")
    worst["sums"] = max(worst.get("sums", 0), r)
    for mom in momenta:
        tgt = bn if mom == 0.1 else types.SimpleNamespace(
            running_mean=bn.running_mean.clone(), running_var=bn.running_var.clone(), momentum=mom,
            num_batches_tracked=bn.num_batches_tracked.clone())
        assert tgt.momentum == mom
        rm0, rv0, nbt = tgt.running_mean.clone(), tgt.running_var.clone(), int(tgt.num_batches_tracked)
        ops.bn_running_update(sums, tgt)
        (rm_ref, rm_b), (rv_ref, rv_b) = oo.running_ref(st, rm0, rv0, mom)
        r = max(so.assert_within(tgt.running_mean, rm_ref, rm_b, f"{tag} running_mean momentum {mom}"),
                so.assert_within(tgt.running_var, rv_ref, rv_b, f"{tag} running_var momentum {mom}"))
        worst["running"] = max(worst.get("running", 0), r)
        assert int(tgt.num_batches_tracked) == nbt + 1
    out = _bn_apply(y, sums, bn, op)
    _written(out, B, f"{tag} bn_apply")
    again = _bn_apply(y, sums, bn, op)
    assert _hashes(again, B) == _hashes(out, B), f"{tag}: a second bn_apply differs"
    del again
    for b in picks:
        xb = y[b:b + 1, ..., :C].double()
        z, e = oo.bn_apply_ref(xb, st, bn.weight, bn.bias, EPS)
        if op == spo.BN_PLAIN:
            ref, bound = z, oo.relu_bf16_bound(z, e)
        elif op == spo.BN_POOL:
            zp = F.max_pool2d(z.permute(0, 3, 1, 2), 2, 2)
            ref, bound = zp.permute(0, 2, 3, 1), oo.pool_bf16_bound(zp, e.permute(0, 3, 1, 2)).permute(0, 2, 3, 1)
        elif op == spo.BN_SOFTMAX:
            p, bound = oo.softmax_bound(z.permute(0, 3, 1, 2), e.permute(0, 3, 1, 2))
            ref, bound = _d2s(p), _d2s(bound)
        else:
            o, bound = oo.l2n_bound(z.permute(0, 3, 1, 2), e.permute(0, 3, 1, 2))
            ref, bound = o.permute(0, 2, 3, 1), bound.permute(0, 2, 3, 1)
        r = so.assert_within(out.t[b:b + 1], ref, bound, f"{tag} bn_apply image {b} of {B}")
        worst[tag] = max(worst.get(tag, 0), r)
        del xb, z, e, ref, bound
    # the edited channels: one-pass statistics exact, and a dead or constant channel normalises to exactly beta
    S1, S2, n = sums[:C].double(), sums[C:2 * C].double(), sums[2 * C].double()
    assert float(S1[DEAD]) == 0.0 and float(S2[DEAD]) == 0.0, tag
    v = float(y[0, 0, 0, CONST])
    assert float(S1[CONST]) == v * st.n and float(S2[CONST]) == v * v * st.n, tag
    assert float(S2[CONST] / n - (S1[CONST] / n) ** 2) == 0.0, tag
    if op in (spo.BN_PLAIN, spo.BN_POOL):
        for c in (DEAD, CONST):
            beta = bn.bias[c].to(torch.bfloat16)
            assert bool((out.t[..., c] == beta).all()), f"{tag}: channel {c} is not bf16(beta)"
    return out


TRAIN_CASES = [(128, 480, 640), (32, 1024, 1024), (2, 56, 72)]


@pytest.mark.parametrize("B,H,W", TRAIN_CASES)
def test_training_chain(B, H, W, weights_path):
    """dense_bf16's training-mode launches at the shipped batches (and a small one, where the unbiased variance's
    n / (n - 1) is visible in fp32), layer by layer on RGB images, each layer freed before the next.  At B = 128 the
    last image of every full-resolution 64-channel map lies past element 2^31 (2^31 / (480 640 64) = 109.2)."""
    m = _model(weights_path, train=True)
    _edge_channels(m)
    pk = m._kernel_weights()
    picks = sorted({0, B // 2, B - 1})
    img = _images(B, 3, H, W, seed=B + H, warped=(min(1, B - 1),))
    if B * H * W * 64 > 2 ** 31:
        assert (B - 1) * H * W * 64 > 2 ** 31
    bn_of = {n: b.bn for n, b in zip(["1a", "1b", "2a", "2b", "3a", "3b", "4a", "4b"], m._blocks())}
    bn_of.update(Pa=m.detector[0].bn, Da=m.descriptor[0].bn, Pb=m.detector[1].bn, Db=m.descriptor[1].bn)
    weights = dict(zip(["1a", "1b", "2a", "2b", "3a", "3b", "4a", "4b"], pk["enc"]))
    weights.update(Pa=pk["Pa"], Da=pk["Da"], Pb=pk["Pb"], Db=pk["Db"])
    worst = {}
    x = xa = None
    for name, sig, _, _, op in TRAIN_LAYERS:
        if sig is None:
            y = _conv1a(img, *weights[name])
            del img
        else:
            src = xa[name[0]] if name in ("Pb", "Db") else x
            y = _conv(src, *weights[name], sig)
        _written(y, B, f"{name} conv")
        out = _check_bn(y.t, bn_of[name], op, picks, worst, name)
        del y
        if name in ("Pa", "Da"):
            xa = xa or {}
            xa[name[0]] = out.t
        elif name not in ("Pb", "Db"):
            x = out.t
        del out
        if name == "Da":
            x = None
        torch.cuda.empty_cache()
    for k, v in worst.items():
        _report(f"training {k} B={B} {H}x{W}", v)


# ---- 4. conv1a on RGB past the grid cap ------------------------------------------------------------------------------
def test_conv1a_rgb_past_the_grid_cap(weights_path):
    """B H W 8 = 3.1e8 threads of work against a grid capped at 65535 * 16 blocks of 256: each thread loops.  Both
    the plain (training) and the affine (eval) conv1a on RGB: the first, a middle and the last image against fp64
    with the kernel's gray rounding, every image written, and a second launch with the same per-image checksums."""
    B, H, W = 128, 480, 640
    assert B * H * W * 8 > 65535 * 16 * 256
    m = _model(weights_path)
    w, bias = m._kernel_weights()["enc"][0]
    bn = m._blocks()[0].bn
    aff = spo.bn_affine(bn)
    img = _images(B, 3, H, W, seed=31, warped=(B - 1,))
    picks = (0, B // 2, B - 1)
    worst = {}
    for kind in ("plain", "affine"):
        args = () if kind == "plain" else aff
        g = _conv1a(img, w, bias, *args)
        _written(g, B, f"conv1a {kind}")
        for b in picks:
            if kind == "plain":
                x, w64, b64 = _gray32(img[b:b + 1]).double(), w.double().view(64, 1, 3, 3), bias.double()
                y = F.conv2d(x, w64, b64, padding=1)
                E = 10 * oo.U * F.conv2d(x.abs(), w64.abs(), b64.abs(), padding=1)
                ref, bound = F.relu(y).permute(0, 2, 3, 1), oo.relu_bf16_bound(F.relu(y), E).permute(0, 2, 3, 1)
            else:
                ref, bound = _conv1a_eval_ref(img[b:b + 1], w, bias, (bn.weight, bn.bias, bn.running_mean,
                                                                     bn.running_var))
            worst[kind] = max(worst.get(kind, 0), so.assert_within(g.t[b:b + 1], ref, bound,
                                                                   f"conv1a {kind} image {b} of {B}"))
            del ref, bound
        h1 = _hashes(g, B)
        del g
        g = _conv1a(img, w, bias, *args)
        _written(g, B, f"conv1a {kind} again")
        assert _hashes(g, B) == h1, f"conv1a {kind}: a second launch differs"
        del g
        torch.cuda.empty_cache()
    for k, v in worst.items():
        _report(f"conv1a RGB {k} B={B}", v)


# ---- 5. batch-offset invariance past 2^31 and 2^32 -------------------------------------------------------------------
def _running(m):
    sd = m.state_dict()
    return torch.cat([v.float().ravel() for k, v in sd.items() if "running" in k or k.endswith("num_batches_tracked")])


def test_ranks_equal_whole_batch_b128(monkeypatch, weights_path):
    """The homography training setting at B = 128 as 4 emulated SyncBatchNorm ranks of 32 images.  Each rank's
    exchange records its local sums and hands back the whole batch's: its keypoints, scores, descriptors and dense
    descriptors must equal its slice of the whole-batch call bit for bit, its running statistics the whole batch's,
    and the ranks' local sums must add up to the whole batch's.  No rank holds an element past 2^31, so a 32-bit
    offset anywhere in the chain shows up as a mismatch."""
    B, ranks, H, W = 128, 4, 480, 640
    conf = {**HOMOGRAPHY, "dense_outputs": True}
    img = _images(B, 3, H, W, seed=41, warped=(1, 77, 127))
    totals = []

    def record(bn):
        assert isinstance(bn, torch.nn.SyncBatchNorm) and bn.training
        return lambda t: totals.append(t.clone())
    monkeypatch.setattr(ops, "bn_exchange", record)
    whole = _model(weights_path, conf, train=True, sync=True)
    torch.manual_seed(0)
    ref = whole({"image": img})
    ref = {k: v.clone() for k, v in ref.items()}
    run_whole = _running(whole)
    del whole
    torch.cuda.empty_cache()
    assert len(totals) == 12
    parts = []
    n = B // ranks
    for r in range(ranks):
        sl = slice(r * n, (r + 1) * n)
        calls = iter(range(len(totals)))
        local = []

        def exchange(bn):
            assert isinstance(bn, torch.nn.SyncBatchNorm) and bn.training

            def ex(t):
                local.append(t.clone())
                t.copy_(totals[next(calls)])
            return ex
        monkeypatch.setattr(ops, "bn_exchange", exchange)
        m = _model(weights_path, conf, train=True, sync=True)
        torch.manual_seed(0)
        out = m({"image": img[sl].contiguous()})
        for k in ("keypoints", "keypoint_scores", "descriptors", "dense_descriptors"):
            so.assert_bits_equal(out[k], ref[k][sl], f"rank {r} {k}")
        so.assert_bits_equal(_running(m), run_whole, f"rank {r} running statistics")
        parts.append(local)
        del m, out
    for i, t in enumerate(totals):
        s = sum(p[i] for p in parts)
        # fp64 sums of the same terms in another grouping: far inside 1e-9 of the largest entry
        torch.testing.assert_close(s, t, rtol=1e-9, atol=1e-9 * float(t.abs().max()), msg=f"BatchNorm {i}: local sums")


def test_eval_b256_equals_chunks(weights_path):
    """Eval mode at B = 256 x 480x640 (every full-resolution 64-channel map has 5.0e9 elements, past 2^32): the
    whole batch equals 8 calls of 32 images bit for bit."""
    B, n, H, W = 256, 32, 480, 640
    conf = {**HOMOGRAPHY, "dense_outputs": True}
    m = _model(weights_path, conf)
    img = _images(B, 3, H, W, seed=43, warped=(3, 200, 255))
    torch.manual_seed(0)
    ref = m({"image": img})
    for c in range(B // n):
        sl = slice(c * n, (c + 1) * n)
        out = m({"image": img[sl].contiguous()})
        for k in ("keypoints", "keypoint_scores", "descriptors", "dense_descriptors"):
            so.assert_bits_equal(out[k], ref[k][sl], f"images {sl.start}-{sl.stop - 1} {k}")
