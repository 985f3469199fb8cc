"""GPU: the SuperPoint extractor's kernels (csrc/superpoint.cu) against fp64 and the reference goldens
(scripts/make_superpoint_golden.py), its determinism and CUDA-graph replay, and a matcher training step fed by it."""
import glob
import os
import sys

import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gluefactory_b200 import synthetic  # noqa: E402
from gluefactory_b200.extractors import superpoint as sp  # noqa: E402
from tests.superpoint_oracle import border_ref, load_golden, nms_ref, sample_ref, select_ref  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda"
GOLDEN = sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "superpoint_*.npz")))
IDS = [os.path.basename(p)[:-4] for p in GOLDEN]


def _model(conf, precision):
    m = sp.SuperPoint({"weights": None, "precision": precision, **conf})
    m.load_state_dict(synthetic.make_superpoint_weights(m.state_dict(), seed=7))
    return m.to(DEV).eval()


def _close(out, ref, rtol, atol):
    err = (out.double() - ref).abs()
    bound = rtol * ref.abs() + atol
    assert torch.isfinite(out).all()
    assert (err <= bound).all(), f"max err {err.max().item():.3g}, worst ratio {(err / bound).max().item():.3g}"


# ---- 1. each conv kernel against fp64 at tile edges and odd sizes ----------------------------------------------------
@pytest.mark.parametrize("H,W", [(8, 16), (13, 21), (17, 35)])
@pytest.mark.parametrize("C", [1, 3])
def test_conv1a(H, W, C):
    g = torch.Generator(device="cpu").manual_seed(H * W + C)
    img = torch.rand(2, C, H, W, generator=g)
    w, b = torch.randn(64, 1, 3, 3, generator=g) * 0.3, torch.randn(64, generator=g) * 0.1
    out = sp.conv1a(img.to(DEV), w.reshape(64, 9).to(DEV), b.to(DEV))
    gray = img.double() if C == 1 else (img * torch.tensor([0.299, 0.587, 0.114]).view(1, 3, 1, 1)).sum(1, True).double()
    ref = F.relu(F.conv2d(gray, w.double(), b.double(), padding=1)).permute(0, 2, 3, 1)
    _close(out.cpu(), ref, 2 ** -8, 1e-5)


CONVS = [  # (Cin, Cout, ksize, epilogue)
    (64, 64, 3, sp.EP_RELU), (64, 64, 3, sp.EP_POOL), (64, 128, 3, sp.EP_RELU), (128, 128, 3, sp.EP_POOL),
    (128, 128, 3, sp.EP_RELU), (128, 512, 3, sp.EP_RELU), (256, 65, 1, sp.EP_SOFTMAX), (256, 256, 1, sp.EP_L2N),
]


@pytest.mark.parametrize("H,W", [(8, 16), (9, 17), (15, 33), (24, 40)])
@pytest.mark.parametrize("cin,cout,ks,ep", CONVS)
def test_conv_kernel(H, W, cin, cout, ks, ep):
    g = torch.Generator(device="cpu").manual_seed(1000 * cin + cout + H * W + ep)
    x = torch.rand(2, H, W, cin, generator=g).to(torch.bfloat16)
    scale = (2.0 / (cin * ks * ks)) ** 0.5 * (4.0 if ep == sp.EP_SOFTMAX else 1.0)
    w = (torch.randn(cout, cin, ks, ks, generator=g) * scale).to(torch.bfloat16)
    b = torch.randn(cout, generator=g) * 0.1
    npad = 128 if ep == sp.EP_SOFTMAX else cout
    wk = F.pad(w.permute(0, 2, 3, 1).reshape(cout, -1), (0, 0, 0, npad - cout)).contiguous()
    out = sp.conv(x.to(DEV), wk.to(DEV), F.pad(b, (0, npad - cout)).to(DEV), cout, ks, ep).cpu()
    y = F.conv2d(x.double().permute(0, 3, 1, 2), w.double(), b.double(), padding=ks // 2)
    if ep == sp.EP_RELU:
        _close(out, F.relu(y).permute(0, 2, 3, 1), 2 ** -8, 1e-4)
    elif ep == sp.EP_POOL:
        _close(out, F.max_pool2d(F.relu(y), 2, 2).permute(0, 2, 3, 1), 2 ** -8, 1e-4)
    elif ep == sp.EP_SOFTMAX:
        p = F.softmax(y, 1)[:, :-1]
        p = p.permute(0, 2, 3, 1).reshape(2, H, W, 8, 8).permute(0, 1, 3, 2, 4).reshape(2, 8 * H, 8 * W)
        _close(out, p, 1e-5, 1e-7)
    else:
        _close(out, F.normalize(y, dim=1).permute(0, 2, 3, 1), 1e-5, 1e-6)


def test_conv_channel_offset():
    """convDb reads the convDa half of the fused Pa / Da activation (pitch 512, channel offset 256)."""
    g = torch.Generator(device="cpu").manual_seed(5)
    pd = torch.rand(2, 11, 19, 512, generator=g).to(torch.bfloat16)
    w = (torch.randn(256, 256, generator=g) * 0.09).to(torch.bfloat16)
    b = torch.randn(256, generator=g) * 0.1
    out = sp.conv(pd.to(DEV), w.to(DEV), b.to(DEV), 256, 1, sp.EP_L2N, cin=256, c0=256).cpu()
    ref = F.normalize(pd[..., 256:].double() @ w.double().T + b.double(), dim=-1)
    _close(out, ref, 1e-5, 1e-6)


# ---- 2. NMS + selection on the golden score maps: bit-identical to the reference restatement ------------------------
@pytest.mark.parametrize("path", GOLDEN, ids=IDS)
@pytest.mark.parametrize("radius", [3, 4])
@pytest.mark.parametrize("thr", [0.0, 0.005])
@pytest.mark.parametrize("k", [-1, 512, 40])
def test_nms_select_golden(path, radius, thr, k):
    g = load_golden(path)
    scores = torch.from_numpy(g["dense_scores"])
    isz = torch.from_numpy(g["image_size"]) if "image_size" in g else None
    s_ref = border_ref(nms_ref(scores, radius), 4, isz)
    s = sp.nms(scores.to(DEV), radius, 4, None if isz is None else isz.to(DEV))
    assert torch.equal(s.cpu(), s_ref)
    ref = select_ref(s_ref, thr, k)
    for b, (kp, sc) in enumerate(ref):
        kk, ks, cnt = sp.select(s[b:b + 1], thr, k, len(sc))
        assert cnt.item() == len(sc)
        assert torch.equal(kk[0].cpu(), kp) and torch.equal(ks[0].cpu(), sc)
    assert sp.count(s, thr).tolist() == [int((s_ref[b] > thr).sum()) for b in range(s_ref.shape[0])]


@pytest.mark.parametrize("path", GOLDEN, ids=IDS)
def test_forced_padding(path):
    """A count above the number of candidates: the candidates first, then padding in the kept keypoints' range."""
    g = load_golden(path)
    s = sp.nms(torch.from_numpy(g["dense_scores"]).to(DEV), 4, 4)
    n = sp.count(s, 0.005).cpu()
    cap = int(n.max()) + 37
    u = torch.rand(s.shape[0], cap, 2, device=DEV)
    kp, sc, cnt = sp.select(s, 0.005, cap, cap, u, torch.full((1,), 50.0, device=DEV))
    assert torch.equal(cnt.cpu(), n)
    for b in range(s.shape[0]):
        m = int(n[b])
        real, pad = kp[b, :m], kp[b, m:]
        assert (sc[b, m:] == 0).all() and (sc[b, :m] > 0.005).all() and pad.shape[0] >= 37
        assert (pad >= real.min(0).values).all() and (pad <= real.max(0).values).all()
    # no candidate at all: padding inside (0, pad_hi)
    kp, sc, cnt = sp.select(torch.zeros_like(s), 0.5, 16, 16, u[:, :16].contiguous(), torch.full((1,), 50.0, device=DEV))
    assert (cnt == 0).all() and (sc == 0).all() and (kp >= 0).all() and (kp <= 50).all()


# ---- 3. descriptor sampling against fp64 -------------------------------------------------------------------------
@pytest.mark.parametrize("legacy", [True, False])
@pytest.mark.parametrize("h,w", [(9, 12), (15, 17)])
def test_sample(legacy, h, w):
    g = torch.Generator(device="cpu").manual_seed(h * w + legacy)
    desc = F.normalize(torch.randn(2, h, w, 256, generator=g), dim=-1)
    kp = torch.rand(2, 300, 2, generator=g) * torch.tensor([8 * w + 2, 8 * h + 2]) - 1  # edges and just outside
    out = sp.sample(desc.to(DEV), kp.to(DEV), legacy).cpu()
    ref = sample_ref(desc.permute(0, 3, 1, 2), kp, legacy)
    _close(out, ref, 1e-5, 2e-6)


# ---- 4. end to end against the goldens ------------------------------------------------------------------------------
def _run(g, precision, **over):
    m = _model({**g["conf"], **over}, precision)
    data = {"image": torch.from_numpy(g["image"]).to(DEV)}
    if "image_size" in g:
        data["image_size"] = torch.from_numpy(g["image_size"])
    return m, data, m(data)


def _real(g):
    return (torch.from_numpy(g["keypoint_scores"]) > 0).sum(-1).tolist()


@pytest.mark.parametrize("path", GOLDEN, ids=IDS)
def test_end_to_end_fp32(path):
    g = load_golden(path)
    _, _, dense = _run(g, "fp32", sparse_outputs=False)
    ref_s, ref_d = torch.from_numpy(g["dense_scores"]), torch.from_numpy(g["dense_descriptors"])
    _close(dense["keypoint_scores"].cpu(), ref_s.double(), 1e-4, 1e-4 * ref_s.abs().max().item())
    _close(dense["descriptors"].cpu(), ref_d.double(), 1e-4, 1e-5)
    _, _, pred = _run(g, "fp32")
    for b, n in enumerate(_real(g)):
        kr = torch.from_numpy(g["keypoints"][b, :n])
        k = pred["keypoints"][b, :n].cpu()
        sr = torch.from_numpy(g["keypoint_scores"][b, :n])
        ref_set = {tuple(p) for p in kr.tolist()}
        mine = {tuple(p) for p in k.tolist()}
        # keypoints may differ only where two candidates' scores are closer than the tolerance
        diff = ref_set ^ mine
        if diff:
            edges = (sr.min().item(), g["conf"].get("detection_threshold", 0.005))  # the k-th score, the threshold
            assert all(min(abs(float(ref_s[b, int(y - 0.5), int(x - 0.5)]) - e) for e in edges) < 1e-4 * sr.max().item()
                       for x, y in diff), diff
        shared = [i for i, p in enumerate(k.tolist()) if tuple(p) in ref_set]
        idx_ref = {tuple(p): i for i, p in enumerate(kr.tolist())}
        for i in shared:
            j = idx_ref[tuple(k[i].tolist())]
            torch.testing.assert_close(pred["descriptors"][b, i].cpu(), torch.from_numpy(g["descriptors"][b, j]),
                                       rtol=0, atol=1e-4)
    assert pred["descriptors"].shape[-1] == 256 and pred["keypoints"].shape[:2] == pred["keypoint_scores"].shape


BF16_RECALL, BF16_COSINE = 0.95, 0.999  # measured on H100: recall >= 0.98, median cosine 0.99999 (fp32: exact sets)


@pytest.mark.parametrize("path", GOLDEN, ids=IDS)
def test_end_to_end_bf16(path):
    g = load_golden(path)
    _, _, pred = _run(g, "bf16")
    recalls, cosines = [], []
    for b, n in enumerate(_real(g)):
        kr = {tuple(p): i for i, p in enumerate(g["keypoints"][b, :n].tolist())}
        k = pred["keypoints"][b].cpu().tolist()
        hits = [(i, kr[tuple(p)]) for i, p in enumerate(k[:n]) if tuple(p) in kr]
        recalls.append(len(hits) / max(n, 1))
        for i, j in hits:
            cosines.append(float(pred["descriptors"][b, i].cpu() @ torch.from_numpy(g["descriptors"][b, j])))
    cos = torch.tensor(cosines)
    print(f"bf16 {os.path.basename(path)}: recall {recalls} cosine min {cos.min():.4f} median {cos.median():.5f}")
    assert min(recalls) >= BF16_RECALL and cos.median() >= BF16_COSINE


# ---- 5. determinism and CUDA-graph replay -----------------------------------------------------------------------
@pytest.mark.parametrize("precision", ["bf16", "fp32"])
def test_repeat_and_graph_replay(precision):
    g = load_golden(next(p for p in GOLDEN if "gray" in p))  # force_num_keypoints: no host read
    m, data, a = _run(g, precision)
    torch.manual_seed(3)
    a = m(data)
    torch.manual_seed(3)
    b = m(data)
    for k in a:
        assert torch.equal(a[k], b[k]), k
    static = {"image": data["image"].clone()}
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        m(static)  # warm-up: weight packing and kernel attributes
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        out = m(static)
    torch.manual_seed(11)
    graph.replay()
    torch.cuda.synchronize()
    eager = m(static)
    n = _real(g)
    for bi, c in enumerate(n):  # padding is random; the real keypoints and all descriptors of them must agree
        assert torch.equal(out["keypoints"][bi, :c], eager["keypoints"][bi, :c])
        assert torch.equal(out["keypoint_scores"][bi], eager["keypoint_scores"][bi])
        assert torch.equal(out["descriptors"][bi, :c], eager["descriptors"][bi, :c])


# ---- 6. a homography pre-training step fed by the extractor ----------------------------------------------------------
def test_training_step_with_extractor():
    from gluefactory_b200.matchers.homography_matcher import HomographyMatcher
    from gluefactory_b200.matchers.lightglue import LightGlue
    from gluefactory_b200.trainer import MatcherTrainer

    B, S, K = 2, 128, 96
    ext = _model({"max_num_keypoints": K, "force_num_keypoints": True, "detection_threshold": 0.0}, "bf16").train()
    img0 = synthetic.make_superpoint_images(B, 1, S, S, seed=21).to(DEV)
    # view 1: view 0 shifted by (16, 8) pixels, whole 8-pixel cells, so the keypoints shift with it; H_0to1 the shift
    Hs = torch.tensor([[1.0, 0.0, 16.0], [0.0, 1.0, 8.0], [0.0, 0.0, 1.0]], device=DEV).expand(B, 3, 3).contiguous()
    img1 = torch.roll(img0, shifts=(8, 16), dims=(-2, -1))
    size = torch.full((B, 2), float(S), device=DEV)
    f0, f1 = ext({"image": img0, "image_size": size}), ext({"image": img1, "image_size": size})
    data = {"keypoints0": f0["keypoints"], "keypoints1": f1["keypoints"], "descriptors0": f0["descriptors"],
            "descriptors1": f1["descriptors"], "view0": {"image_size": size}, "view1": {"image_size": size},
            "H_0to1": Hs}
    gt = HomographyMatcher({"th_positive": 3.0, "th_negative": 3.0})
    tr = MatcherTrainer(LightGlue({"n_layers": 2}).to(DEV), lr=1e-4, ground_truth=gt)
    before = [p.detach().clone() for p in ext.parameters()]
    loss, losses = tr.step(data)
    assert torch.isfinite(loss).all()
    assert (gt(data)["matches0"] > -1).any()
    assert all(torch.equal(a, b) for a, b in zip(before, ext.parameters()))
    assert not any(p.requires_grad for p in ext.parameters())
