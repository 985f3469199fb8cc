"""Seeded synthetic weights, keypoint pairs and ground-truth labels.

Everything here is host-side input construction (numpy `RandomState`, whose
stream is frozen across numpy versions, so the same seed gives the same
tensors in the build container and on the GPU box).  It is shared by
`bench.py`, the tests and `oracle/make_golden.py`.

The pair recipe follows SURVEY.md section 8(d): N uniformly drawn keypoints in
a 1024x1024 image, a random homography, 40 % planted correspondences with
0.5 px noise and correlated descriptors, the rest random; view 1 permuted.
Ground truth restates `gt_matches_from_homography`
(/root/reference/gluefactory/geometry/gt_generation.py:109-161) with the
thresholds of configs/superpoint+lightglue_homography.yaml:22-25.
"""
import math

import numpy as np
import torch

from .geometry import warp_points

DEFAULT_CONF = {
    "name": "lightglue",
    "input_dim": 256,
    "descriptor_dim": 256,
    "n_layers": 9,
    "num_heads": 4,
    "filter_threshold": 0.0,
    "loss": {"gamma": 1.0, "fn": "nll", "nll_balancing": 0.5},
}


def state_dict_spec(conf):
    """(name, shape) list in the reference's state_dict order
    (/root/reference/gluefactory/models/matchers/lightglue.py:343-372)."""
    D, L, Din = conf["descriptor_dim"], conf["n_layers"], conf["input_dim"]
    H = conf["num_heads"]
    dh = D // H
    spec = []
    if Din != D:
        spec += [("input_proj.weight", (D, Din)), ("input_proj.bias", (D,))]
    spec += [("posenc.Wr.weight", (dh // 2, 2 + 2 * bool(conf.get("add_scale_ori", False))))]
    for i in range(L):
        p = f"transformers.{i}.self_attn"
        spec += [(p + ".Wqkv.weight", (3 * D, D)), (p + ".Wqkv.bias", (3 * D,)),
                 (p + ".out_proj.weight", (D, D)), (p + ".out_proj.bias", (D,)),
                 (p + ".ffn.0.weight", (2 * D, 2 * D)), (p + ".ffn.0.bias", (2 * D,)),
                 (p + ".ffn.1.weight", (2 * D,)), (p + ".ffn.1.bias", (2 * D,)),
                 (p + ".ffn.3.weight", (D, 2 * D)), (p + ".ffn.3.bias", (D,))]
        p = f"transformers.{i}.cross_attn"
        spec += [(p + ".to_qk.weight", (D, D)), (p + ".to_qk.bias", (D,)),
                 (p + ".to_v.weight", (D, D)), (p + ".to_v.bias", (D,)),
                 (p + ".to_out.weight", (D, D)), (p + ".to_out.bias", (D,)),
                 (p + ".ffn.0.weight", (2 * D, 2 * D)), (p + ".ffn.0.bias", (2 * D,)),
                 (p + ".ffn.1.weight", (2 * D,)), (p + ".ffn.1.bias", (2 * D,)),
                 (p + ".ffn.3.weight", (D, 2 * D)), (p + ".ffn.3.bias", (D,))]
    for i in range(L):
        p = f"log_assignment.{i}"
        spec += [(p + ".matchability.weight", (1, D)), (p + ".matchability.bias", (1,)),
                 (p + ".final_proj.weight", (D, D)), (p + ".final_proj.bias", (D,))]
    for i in range(L - 1):
        p = f"token_confidence.{i}.token.0"
        spec += [(p + ".weight", (1, D)), (p + ".bias", (1,))]
    return spec


def make_weights(conf, seed=0, dtype=torch.float32):
    """Deterministic random-init weights under the reference's parameter names.

    Linear layers: U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weight and bias
    (torch's default nn.Linear init); LayerNorm affine perturbed away from
    (1, 0) so that its gradients are exercised; posenc.Wr ~ N(0, 1)
    (lightglue.py:58 with gamma = 1).
    """
    rs = np.random.RandomState(seed)
    out = {}
    spec = state_dict_spec(conf)
    shapes = dict(spec)
    for name, shape in spec:
        if name == "posenc.Wr.weight":
            a = rs.standard_normal(shape)
        elif ".ffn.1." in name:
            a = (1.0 if name.endswith("weight") else 0.0) + 0.1 * rs.standard_normal(shape)
        else:
            wshape = shape if name.endswith("weight") else shapes[name[: -len("bias")] + "weight"]
            bound = 1.0 / math.sqrt(wshape[-1])
            a = rs.uniform(-bound, bound, size=shape)
        out[name] = torch.from_numpy(np.ascontiguousarray(a)).to(dtype)
    return out


# ----------------------------------------------------------------------------
# ground truth (restated; runs on whatever device the keypoints live on)
# ----------------------------------------------------------------------------
@torch.no_grad()
def gt_matches_from_homography(kp0, kp1, Hm, pos_th=3.0, neg_th=3.0):
    """Restates geometry/gt_generation.py:109-161: reprojection distance both
    ways, mutual nearest neighbours below pos_th are positives, points whose
    best reprojection error exceeds neg_th are unmatched (-1), the rest are
    ignored (-2)."""
    kp0_1 = warp_points(kp0, Hm)
    kp1_0 = warp_points(kp1, torch.inverse(Hm))
    d0 = ((kp0_1[:, :, None] - kp1[:, None]) ** 2).sum(-1)
    d1 = ((kp0[:, :, None] - kp1_0[:, None]) ** 2).sum(-1)
    dist = torch.max(d0, d1)
    min0 = dist.min(-1).indices
    min1 = dist.min(-2).indices
    ismin0 = torch.zeros_like(dist, dtype=torch.bool).scatter_(-1, min0[..., None], True)
    ismin1 = torch.zeros_like(dist, dtype=torch.bool).scatter_(-2, min1[:, None], True)
    positive = ismin0 & ismin1 & (dist < pos_th**2)
    neg0 = d0.min(-1).values > neg_th**2
    neg1 = d1.min(-2).values > neg_th**2
    m0 = torch.where(positive.any(-1), min0, torch.full_like(min0, -2))
    m1 = torch.where(positive.any(-2), min1, torch.full_like(min1, -2))
    m0 = torch.where(neg0, torch.full_like(m0, -1), m0)
    m1 = torch.where(neg1, torch.full_like(m1, -1), m1)
    return positive, m0, m1


def _random_homography(rs, size, difficulty=0.7):
    """4-corner perturbation homography (in the spirit of
    geometry/homography.py:40-107), solved by DLT."""
    s = float(size)
    src = np.array([[0, 0], [s, 0], [s, s], [0, s]], dtype=np.float64)
    dst = src + rs.uniform(-0.25 * difficulty * s / 2, 0.25 * difficulty * s / 2, size=(4, 2))
    A = []
    for (x, y), (u, v) in zip(src, dst):
        A.append([-x, -y, -1, 0, 0, 0, u * x, u * y, u])
        A.append([0, 0, 0, -x, -y, -1, v * x, v * y, v])
    _, _, vt = np.linalg.svd(np.asarray(A))
    Hm = vt[-1].reshape(3, 3)
    return Hm / Hm[2, 2]


def make_pairs(B, N, seed=1234, D=256, image_size=1024, frac=0.4, M=None, with_gt=True,
               dtype=torch.float32):
    """Synthetic batch in the matcher's input contract
    (models/two_view_pipeline.py:80-81; lightglue.py:416-455)."""
    M = N if M is None else M
    rs = np.random.RandomState(seed)
    S = float(image_size)
    kp0 = np.zeros((B, M, 2)); kp1 = np.zeros((B, N, 2))
    de0 = np.zeros((B, M, D)); de1 = np.zeros((B, N, D))
    Hs = np.zeros((B, 3, 3))
    for b in range(B):
        Hm = _random_homography(rs, S)
        Hs[b] = Hm
        k0 = rs.uniform(0.5, S - 0.5, size=(M, 2))
        K = int(frac * min(M, N))
        ph = np.concatenate([k0[:K], np.ones((K, 1))], 1) @ Hm.T
        w1 = ph[:, :2] / ph[:, 2:] + 0.5 * rs.standard_normal((K, 2))
        k1 = rs.uniform(0.5, S - 0.5, size=(N, 2))
        inside = np.all((w1 > 0.5) & (w1 < S - 0.5), 1)
        k1[:K][inside] = w1[inside]
        f0 = rs.standard_normal((M, D))
        f0 /= np.linalg.norm(f0, axis=1, keepdims=True)
        f1 = rs.standard_normal((N, D))
        f1[:K][inside] = (f0[:K] + 0.3 * rs.standard_normal((K, D)) / math.sqrt(D))[inside]
        f1 /= np.linalg.norm(f1, axis=1, keepdims=True)
        perm = rs.permutation(N)
        kp0[b], kp1[b], de0[b], de1[b] = k0, k1[perm], f0, f1[perm]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dtype)
    size = torch.full((B, 2), S, dtype=dtype)
    data = {
        "keypoints0": t(kp0), "keypoints1": t(kp1),
        "descriptors0": t(de0), "descriptors1": t(de1),
        "view0": {"image_size": size.clone()}, "view1": {"image_size": size.clone()},
        "H_0to1": t(Hs),
    }
    if with_gt:
        gts = [gt_matches_from_homography(data["keypoints0"][b:b + 1].double(), data["keypoints1"][b:b + 1].double(),
                                          data["H_0to1"][b:b + 1].double()) for b in range(B)]  # per pair: bounded memory
        data.update({"gt_assignment": torch.cat([g[0] for g in gts]), "gt_matches0": torch.cat([g[1] for g in gts]),
                     "gt_matches1": torch.cat([g[2] for g in gts])})
    return data


def add_scale_ori_inputs(data, seed):
    """Per-keypoint scale / orientation of SIFT-style extractors (the extra inputs of `add_scale_ori`, lightglue.py:426-443)."""
    rs = np.random.RandomState(seed)
    for i in "01":
        k = data[f"keypoints{i}"]
        data[f"scales{i}"] = torch.from_numpy(rs.uniform(0.5, 4.0, size=tuple(k.shape[:2]))).to(k.dtype)
        data[f"oris{i}"] = torch.from_numpy(rs.uniform(-3.14, 3.14, size=tuple(k.shape[:2]))).to(k.dtype)
    return data


def to_device(data, device, non_blocking=False):
    """Recursive .to(device) over the nested batch dict
    (utils/tensor.py:30-34 batch_to_device)."""
    if isinstance(data, dict):
        return {k: to_device(v, device, non_blocking) for k, v in data.items()}
    if torch.is_tensor(data):
        return data.to(device, non_blocking=non_blocking)
    return data


# ----------------------------------------------------------------------------
# GlueStick (points + lines; BASELINE.json configs[4])
# ----------------------------------------------------------------------------
def make_gluestick_batch(B, N, L, seed, D=256, dtype=torch.float32):
    """Synthetic GlueStick batch (SURVEY 8d, config 5 shape): the first 2L keypoints of each view are the endpoints of L
    independent segments (wireframe.py:246-253, 290-294: lines_junc_idx = arange(2L).view(L, 2)), the rest plain
    keypoints.  Point labels from the homography restatement; a segment of view 0 matches a segment of view 1 when both
    endpoints correspond (either order)."""
    d = make_pairs(B, N, seed=seed, D=D, dtype=dtype)
    rs = np.random.RandomState(seed + 7)
    out = dict(d)
    for i in "01":
        kp = d[f"keypoints{i}"]
        out[f"lines{i}"] = kp[:, :2 * L].reshape(B, L, 2, 2).clone()
        out[f"lines_junc_idx{i}"] = torch.arange(2 * L).view(1, L, 2).repeat(B, 1, 1)
        out[f"line_scores{i}"] = torch.from_numpy(rs.uniform(0, 1, size=(B, L))).to(dtype)
        out[f"keypoint_scores{i}"] = torch.from_numpy(rs.uniform(0, 1, size=(B, N))).to(dtype)
    m0 = d["gt_matches0"][:, :2 * L].reshape(B, L, 2)
    asg = torch.zeros(B, L, L, dtype=torch.bool)
    for b in range(B):
        for a in range(L):
            e0, e1 = int(m0[b, a, 0]), int(m0[b, a, 1])
            if 0 <= e0 < 2 * L and 0 <= e1 < 2 * L and e0 // 2 == e1 // 2 and e0 != e1:
                asg[b, a, e0 // 2] = True
    lm0 = torch.where(asg.any(2), asg.float().argmax(2), torch.full((B, L), -1, dtype=torch.long))
    lm1 = torch.where(asg.any(1), asg.float().argmax(1), torch.full((B, L), -1, dtype=torch.long))
    out.update(gt_line_assignment=asg, gt_line_matches0=lm0, gt_line_matches1=lm1)
    return out


def make_gluestick_weights(state_dict_like, seed=0, dtype=torch.float32):
    """Deterministic weights for a GlueStick state_dict (names / shapes taken from `state_dict_like`, e.g. the plugin
    module's own state_dict, whose tree equals the reference's): conv weights and biases U(-1/sqrt(fan_in), ..),
    BatchNorm affine perturbed around (1, 0), bin scores around 1, running statistics left at their defaults."""
    rs = np.random.RandomState(seed)
    shapes = {k: tuple(v.shape) for k, v in state_dict_like.items()}
    out = {}
    for k, shp in shapes.items():
        if k.endswith("num_batches_tracked"):
            out[k] = torch.zeros((), dtype=torch.long)
        elif k.endswith("running_mean"):
            out[k] = torch.zeros(shp, dtype=dtype)
        elif k.endswith("running_var"):
            out[k] = torch.ones(shp, dtype=dtype)
        elif len(shp) == 0:
            out[k] = torch.tensor(1.0 + 0.1 * rs.standard_normal(), dtype=dtype)
        elif k[: k.rfind(".")] + ".running_mean" in shapes:  # BatchNorm affine
            base = 1.0 if k.endswith("weight") else 0.0
            out[k] = torch.from_numpy(base + 0.1 * rs.standard_normal(shp)).to(dtype)
        else:
            wshape = shp if k.endswith("weight") else shapes[k[: -len("bias")] + "weight"]
            bound = 1.0 / math.sqrt(wshape[1])
            out[k] = torch.from_numpy(rs.uniform(-bound, bound, size=shp)).to(dtype)
    return out


def make_superglue_batch(B, M, N, seed, D=256, dtype=torch.float32):
    """Synthetic SuperGlue batch: make_pairs (keypoints, descriptors, homography labels; M view-0 and N view-1 points)
    plus per-keypoint detection scores in [0, 1)."""
    d = make_pairs(B, N, seed=seed, D=D, M=M, dtype=dtype)
    rs = np.random.RandomState(seed + 7)
    for i, n in (("0", M), ("1", N)):
        d[f"keypoint_scores{i}"] = torch.from_numpy(rs.uniform(0, 1, size=(B, n))).to(dtype)
    return d


# ----------------------------------------------------------------------------
# pose + depth ground truth (MegaDepth-style supervision, matchers/depth_matcher.py)
# ----------------------------------------------------------------------------
def pose_depth_scene(B, M, N, seed, W=640, H=480):
    """Synthetic two-view scene for the pose + depth ground truth: a tilted plane seen by two pinhole cameras; depth
    maps in closed form (with a band of invalid depth), 45 % of the view-1 keypoints are reprojections of view-0
    keypoints + 0.7 px noise, the rest uniform.  Returns plain tensors (K, R, t, depths, keypoints)."""
    rs = np.random.RandomState(seed)
    K = np.array([[520.0, 0, W / 2], [0, 520.0, H / 2], [0, 0, 1]])
    out = {k: [] for k in ("K0", "K1", "R", "t", "depth0", "depth1", "kp0", "kp1")}
    for b in range(B):
        ang = rs.uniform(-0.12, 0.12, size=3)
        Rx = np.array([[1, 0, 0], [0, np.cos(ang[0]), -np.sin(ang[0])], [0, np.sin(ang[0]), np.cos(ang[0])]])
        Ry = np.array([[np.cos(ang[1]), 0, np.sin(ang[1])], [0, 1, 0], [-np.sin(ang[1]), 0, np.cos(ang[1])]])
        Rz = np.array([[np.cos(ang[2]), -np.sin(ang[2]), 0], [np.sin(ang[2]), np.cos(ang[2]), 0], [0, 0, 1]])
        R = Rz @ Ry @ Rx
        t = rs.uniform(-0.5, 0.5, size=3)
        n0 = np.array([0.15, -0.1, 1.0]); n0 /= np.linalg.norm(n0)
        dpl = 5.0  # plane n0 . X = dpl in camera 0
        Kinv = np.linalg.inv(K)
        ys, xs = np.meshgrid(np.arange(H) + 0.5, np.arange(W) + 0.5, indexing="ij")
        rays = np.stack([xs, ys, np.ones_like(xs)], -1) @ Kinv.T
        depth0 = dpl / (rays @ n0)
        n1 = R @ n0
        d1 = dpl + n1 @ t
        depth1 = d1 / (rays @ n1)
        depth0[:, 200:230] = 0.0  # a band without depth in each view (invalid keypoints)
        depth1[100:130, :] = 0.0
        kp0 = np.stack([rs.uniform(2, W - 2, M), rs.uniform(2, H - 2, M)], -1)
        kp1 = np.stack([rs.uniform(2, W - 2, N), rs.uniform(2, H - 2, N)], -1)
        Kn = int(0.45 * min(M, N))
        r0 = np.concatenate([kp0[:Kn], np.ones((Kn, 1))], 1) @ Kinv.T
        X0 = r0 * (dpl / (r0 @ n0))[:, None]
        X1 = X0 @ R.T + t
        proj = (X1 / X1[:, 2:]) @ K.T
        cand = proj[:, :2] + 0.7 * rs.standard_normal((Kn, 2))
        ok = (cand[:, 0] > 2) & (cand[:, 0] < W - 2) & (cand[:, 1] > 2) & (cand[:, 1] < H - 2)
        kp1[:Kn][ok] = cand[ok]
        kp1 = kp1[rs.permutation(N)]
        for k, v in (("K0", K), ("K1", K), ("R", R), ("t", t), ("depth0", depth0), ("depth1", depth1), ("kp0", kp0), ("kp1", kp1)):
            out[k].append(v)
    return {k: torch.from_numpy(np.stack(v)).float() for k, v in out.items()}


class PinholeCamera:
    """Duck-typed stand-in for gluefactory.geometry.wrappers.Camera (PINHOLE, no distortion) with exactly the methods
    the depth ground truth calls (wrappers.py:271-398): data = [w, h, fx, fy, cx, cy] per batch element."""

    eps = 1e-4

    def __init__(self, K):
        self.f = torch.stack([K[..., 0, 0], K[..., 1, 1]], -1)
        self.c = torch.stack([K[..., 0, 2], K[..., 1, 2]], -1)
        self.size = 2 * self.c
        self._K = K

    def to(self, device):
        return PinholeCamera(self._K.to(device))

    def calibration_matrix(self):
        return self._K

    def image2cam(self, p2d):
        p = (p2d - self.c.unsqueeze(-2)) / self.f.unsqueeze(-2)
        return torch.cat([p, torch.ones_like(p[..., :1])], -1)

    def cam2image(self, p3d):
        z = p3d[..., -1]
        visible = z > self.eps
        p2d = p3d[..., :-1] / z.clamp(min=self.eps).unsqueeze(-1)
        p2d = p2d * self.f.unsqueeze(-2) + self.c.unsqueeze(-2)
        inside = torch.all((p2d >= 0) & (p2d <= (self.size.unsqueeze(-2) - 1)), -1)
        return p2d, visible & inside


class RigidPose:
    """Duck-typed stand-in for gluefactory.geometry.wrappers.Pose: p -> R p + t."""

    def __init__(self, R, t):
        self.R, self.t = R, t

    def to(self, device):
        return RigidPose(self.R.to(device), self.t.to(device))

    def transform(self, p3d):
        return p3d @ self.R.transpose(-1, -2) + self.t.unsqueeze(-2)

    def inv(self):
        Rt = self.R.transpose(-1, -2)
        return RigidPose(Rt, -(Rt @ self.t.unsqueeze(-1)).squeeze(-1))


# ----------------------------------------------------------------------------
# line ground truth (use_lines of matchers/homography_matcher.py and matchers/depth_matcher.py)
# ----------------------------------------------------------------------------
def _line_pairs(rs, to1, L0, L1, W, H):
    """View-0 segments and view-1 segments built from them: `to1` maps [n,2] view-0 points into view 1.  View 1 holds
    the mapped segments with 0.6 px endpoint noise (some shortened, so that they overlap partly), exact and near
    duplicates (tied costs), distractors, all permuted; 10 % of the segments of each view are flagged invalid.  Some
    view-0 segments start near the border and run out of the image (clamped), some map outside image 1."""
    ang = rs.uniform(0, np.pi, L0)
    length = rs.uniform(15, 160, L0)
    start = np.stack([rs.uniform(-20, W + 20, L0), rs.uniform(-20, H + 20, L0)], -1)
    end = start + length[:, None] * np.stack([np.cos(ang), np.sin(ang)], -1)
    l0 = np.stack([start, end], 1)                                   # [L0, 2, 2]
    K = min(int(0.6 * L0), L1 - 4)
    src = l0[:K].copy()
    cut = rs.uniform(size=K) < 0.3                                   # shortened copies: partial overlap
    f = rs.uniform(0.5, 0.9, size=(K, 1))
    src[cut, 1] = src[cut, 0] + f[cut] * (src[cut, 1] - src[cut, 0])
    m = to1(src.reshape(-1, 2)).reshape(K, 2, 2) + 0.6 * rs.standard_normal((K, 2, 2))
    nd = min(4, K)
    dups = m[:nd].copy()
    dups[nd // 2:] += 0.3 * rs.standard_normal((nd - nd // 2, 2, 2))  # near duplicates; the first half exact
    nrand = L1 - K - nd
    a1 = rs.uniform(0, np.pi, nrand)
    s1 = np.stack([rs.uniform(0, W, nrand), rs.uniform(0, H, nrand)], -1)
    r1 = np.stack([s1, s1 + rs.uniform(15, 160, (nrand, 1)) * np.stack([np.cos(a1), np.sin(a1)], -1)], 1)
    l1 = np.concatenate([m, dups, r1])[rs.permutation(L1)]
    v0, v1 = rs.uniform(size=L0) > 0.1, rs.uniform(size=L1) > 0.1
    return l0, l1, v0, v1


def line_gt_scene(kind, B, L0, L1, seed, W=640, H=480):
    """Seeded two-view line scene for the line ground truth.  kind "homography": lines0/1 [B,L,2,2], valid_lines0/1,
    H_0to1 [B,3,3], image_size (H, W).  kind "pose_depth": the camera / plane scene of `pose_depth_scene` (K0, K1, R,
    t, depth0, depth1) with view-1 segments reprojected through the plane."""
    rs = np.random.RandomState(seed)
    out = {k: [] for k in ("lines0", "lines1", "valid_lines0", "valid_lines1")}
    if kind == "homography":
        Hs = []
        for _ in range(B):
            Hm = _random_homography(rs, 512.0, difficulty=0.5)
            Hs.append(Hm)
            to1 = lambda p, Hm=Hm: (lambda q: q[:, :2] / q[:, 2:])(np.concatenate([p, np.ones((len(p), 1))], 1) @ Hm.T)  # noqa: E731
            for k, v in zip(out, _line_pairs(rs, to1, L0, L1, W, H)):
                out[k].append(v)
        extra = {"H_0to1": torch.from_numpy(np.stack(Hs)).float()}
    elif kind == "pose_depth":
        extra = pose_depth_scene(B, 1, 1, seed, W=W, H=H)
        del extra["kp0"], extra["kp1"]
        n0 = np.array([0.15, -0.1, 1.0]); n0 /= np.linalg.norm(n0)  # the plane of pose_depth_scene
        for b in range(B):
            Km, R, t = (extra[k][b].double().numpy() for k in ("K0", "R", "t"))
            Kinv = np.linalg.inv(Km)

            def to1(p, Kinv=Kinv, Km=Km, R=R, t=t):
                r0 = np.concatenate([p, np.ones((len(p), 1))], 1) @ Kinv.T
                X1 = (r0 * (5.0 / (r0 @ n0))[:, None]) @ R.T + t
                return ((X1 / X1[:, 2:]) @ Km.T)[:, :2]
            for k, v in zip(out, _line_pairs(rs, to1, L0, L1, W, H)):
                out[k].append(v)
    else:
        raise ValueError(kind)
    res = {k: torch.from_numpy(np.stack(v)) for k, v in out.items()}
    for k in ("lines0", "lines1"):
        res[k] = res[k].float()
    res.update(extra)
    res["image_size"] = (H, W)
    return res


def make_superpoint_weights(state_dict_like, seed=0, dtype=torch.float32):
    """Deterministic SuperPoint weights (names / shapes from `state_dict_like`): He-uniform conv weights
    U(-sqrt(6 / fan_in), ..), so activations keep their scale through the ReLU stack, biases U(-0.05, 0.05), and
    convPb's weights 4x larger, so the 65-way softmax gives peaked score maps with keypoints above the threshold."""
    rs = np.random.RandomState(seed)
    out = {}
    for k, v in state_dict_like.items():
        shp = tuple(v.shape)
        if k.endswith("weight"):
            bound = math.sqrt(6.0 / (shp[1] * shp[2] * shp[3])) * (4.0 if k.startswith("convPb") else 1.0)
        else:
            bound = 0.05
        out[k] = torch.from_numpy(rs.uniform(-bound, bound, size=shp)).to(dtype)
    return out


def make_superpoint_images(B, C, H, W, seed=0):
    """[B, C, H, W] float32 images in [0, 1]: a few Gaussian blobs and edges over low-amplitude noise."""
    rs = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:H, 0:W].astype(np.float64)
    out = np.empty((B, C, H, W), np.float32)
    for b in range(B):
        for c in range(C):
            img = 0.1 * rs.standard_normal((H, W))
            for _ in range(12):
                cy, cx, s, a = rs.uniform(0, H), rs.uniform(0, W), rs.uniform(1.5, 6.0), rs.uniform(-1, 1)
                img += a * np.exp(-((yy - cy) ** 2 + (xx - cx) ** 2) / (2 * s * s))
            img += 0.5 * (xx > rs.uniform(0, W)) * (yy > rs.uniform(0, H))
            out[b, c] = (img - img.min()) / (img.max() - img.min())
    return torch.from_numpy(out)


def make_superpoint_open_weights(state_dict_like, seed=0, dtype=torch.float32):
    """Deterministic SuperPoint-open weights (names / shapes from `state_dict_like`).  Convs as
    make_superpoint_weights (He-uniform, biases U(-0.05, 0.05)), detector.1's weights 4x larger so that keypoints
    clear the detection threshold.  BatchNorms: gamma of either sign with |gamma| in [0.5, 1.5] (a 2x2 max-pool placed
    before the affine gives a different map), beta U(-0.1, 0.1), running_mean U(0, 0.5), running_var U(0.5, 2),
    num_batches_tracked 0."""
    rs = np.random.RandomState(seed)
    out = {}
    for k, v in state_dict_like.items():
        shp = tuple(v.shape)
        if k.endswith("num_batches_tracked"):
            out[k] = torch.zeros((), dtype=torch.long)
            continue
        if k.endswith("conv.weight"):
            bound = math.sqrt(6.0 / (shp[1] * shp[2] * shp[3])) * (4.0 if k.startswith("detector.1") else 1.0)
            w = rs.uniform(-bound, bound, size=shp)
        elif k.endswith("conv.bias"):
            w = rs.uniform(-0.05, 0.05, size=shp)
        elif k.endswith("bn.weight"):
            w = rs.uniform(0.5, 1.5, size=shp) * rs.choice([-1.0, 1.0], size=shp)
        elif k.endswith("bn.bias"):
            w = rs.uniform(-0.1, 0.1, size=shp)
        elif k.endswith("running_mean"):
            w = rs.uniform(0.0, 0.5, size=shp)
        elif k.endswith("running_var"):
            w = rs.uniform(0.5, 2.0, size=shp)
        else:
            raise KeyError(k)
        out[k] = torch.from_numpy(w).to(dtype)
    return out
