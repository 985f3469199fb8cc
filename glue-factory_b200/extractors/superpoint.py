"""H100-native SuperPoint keypoint extractor, inference only -- drop-in for glue-factory's `gluefactory_nonfree.superpoint`
(the frozen extractor of `superpoint+lightglue_homography.yaml`, where every sample is a freshly warped image and the
features cannot be cached).

Select it with `model.extractor.name: gluefactory_b200.extractors.superpoint`.  Same `default_conf`,
`required_data_keys` and module tree (`conv1a` ... `convDb`) as the reference, so its `state_dict` and
`superpoint_v1.pth` load as they are.  Two plugin-only keys:
  * `weights`: "default" reads `superpoint_v1.pth` from torch-hub's checkpoint cache (never downloaded: a missing file
    raises FileNotFoundError naming the path), None keeps the random initialisation, any other string is a path.
  * `precision`: "bf16" (default) runs the encoder and heads as wgmma implicit-GEMM convolutions (bf16 activations,
    fp32 accumulation, csrc/superpoint.cu); "fp32" is the parity path: fp32 cuDNN convolutions with TF32 off.
Both feed the same CUDA kernels for NMS, border removal, thresholding, per-image top-k and descriptor sampling.

Keypoint order: when an image has no more than k candidates (or k <= 0) they come in row-major order, as the
reference's torch.where gives them; otherwise the k best in descending score order, exact score ties going to the
lower row-major index.  With `force_num_keypoints` the padding (score 0, coordinates drawn uniformly in the range of
the kept keypoints, or in (0, min(image_size)) when none is kept) is drawn on the device and the forward reads nothing
back to the host, so it can be captured in a CUDA graph.  Without it, B > 1 images with different keypoint counts
fail as the reference's torch.stack does.

Refused with NotImplementedError: `trainable: True` and any backward (the extractor is frozen in every config),
`refinement_radius > 0`, `randomize_keypoints_training` in training mode, `descriptor_dim` other than 256, and a
detector or descriptor head turned off.  No CPU fallback.
"""
import os

import torch
import torch.nn.functional as F
from torch import nn

from .. import _lib
from ..matchers import _weights
from ..matchers.lightglue import _Conf, _merge, _to_plain

EP_RELU, EP_POOL, EP_SOFTMAX, EP_L2N = 0, 1, 2, 3
MAX_K = 16384  # LGB200_SP_MAX_K
MAX_NMS_RADIUS = 9


def _p(t):
    return _lib.ptr(t)


def conv1a(image, weight, bias):
    """ReLU(conv3x3(gray(image))) as NHWC bf16 [B, H, W, 64]; image [B, 1 | 3, H, W] fp32, weight [64, 9] fp32."""
    B, C, H, W = image.shape
    out = torch.empty(B, H, W, 64, device=image.device, dtype=torch.bfloat16)
    _lib.call("lgb200_sp_conv1a", _p(image), C, _p(weight), _p(bias), _p(out), B, H, W, _lib.stream_ptr())
    return out


def conv(x, weight, bias, cout, ksize, epilogue, cin=None, c0=0):
    """Implicit-GEMM conv of NHWC bf16 x [B, H, W, ldx] (its channels [c0, c0 + cin)) with weight [Npad, k*k*cin]."""
    B, H, W, ldx = x.shape
    cin = ldx - c0 if cin is None else cin
    if epilogue == EP_POOL:
        out = torch.empty(B, H // 2, W // 2, cout, device=x.device, dtype=torch.bfloat16)
    elif epilogue == EP_RELU:
        out = torch.empty(B, H, W, cout, device=x.device, dtype=torch.bfloat16)
    elif epilogue == EP_SOFTMAX:
        out = torch.empty(B, 8 * H, 8 * W, device=x.device, dtype=torch.float32)
    else:
        out = torch.empty(B, H, W, cout, device=x.device, dtype=torch.float32)
    _lib.call("lgb200_sp_conv", x.data_ptr() + 2 * c0, ldx, _p(weight), _p(bias), _p(out), B, H, W, cin, cout, ksize,
              epilogue, _lib.stream_ptr())
    return out


def nms(scores, radius, remove_borders, image_size=None):
    """simple_nms + border removal of scores [B, H, W] fp32; image_size [B, 2] (w, h) or None."""
    B, H, W = scores.shape
    out = torch.empty_like(scores)
    _lib.call("lgb200_sp_nms", _p(scores), _p(image_size), _p(out), B, H, W, int(radius), int(remove_borders),
              _lib.stream_ptr())
    return out


def count(nms_scores, threshold):
    B, H, W = nms_scores.shape
    counts = torch.empty(B, device=nms_scores.device, dtype=torch.int32)
    _lib.call("lgb200_sp_count", _p(nms_scores), float(threshold), _p(counts), B, H, W, _lib.stream_ptr())
    return counts


def select(nms_scores, threshold, k, cap, uniform=None, pad_hi=None):
    """Keypoints [B, cap, 2] (x, y), scores [B, cap] and kept counts [B] (int32); see lgb200_sp_select."""
    B, H, W = nms_scores.shape
    dev = nms_scores.device
    kpts = torch.empty(B, cap, 2, device=dev, dtype=torch.float32)
    scores = torch.empty(B, cap, device=dev, dtype=torch.float32)
    counts = torch.empty(B, device=dev, dtype=torch.int32)
    if cap > 0:
        _lib.call("lgb200_sp_select", _p(nms_scores), float(threshold), int(k), int(cap), _p(uniform), _p(pad_hi),
                  _p(kpts), _p(scores), _p(counts), B, H, W, _lib.stream_ptr())
    else:
        counts.zero_()
    return kpts, scores, counts


def select_keypoints(s, threshold, max_kps, force, image_size, image_hw):
    """Keypoints [B, n, 2] (x, y) and scores [B, n] from the NMS'd score map s [B, H, W].  With `force` (max_kps > 0):
    n = max_kps, padded on the device inside the kept keypoints' range, or (0, min(image_size)) when none is kept
    (image_size [B, 2] on the device, or None for the image's own (H, W) = image_hw); nothing is read back to the host.
    Without it: every image's count is read back and must agree, as torch.stack requires."""
    B = s.shape[0]
    dev = s.device
    if force:
        if max_kps <= 0:
            raise AssertionError("force_num_keypoints needs max_num_keypoints > 0")
        uniform = torch.rand(B, max_kps, 2, device=dev)
        if image_size is not None:
            pad_hi = image_size.min().reshape(1)
        else:
            pad_hi = torch.full((1,), float(min(image_hw)), device=dev)
        kpts, kscores, _ = select(s, threshold, max_kps, max_kps, uniform, pad_hi)
    else:
        counts = count(s, threshold).tolist()
        kept = [min(c, max_kps) if max_kps > 0 else c for c in counts]
        if any(c != kept[0] for c in kept):
            raise RuntimeError(f"stack expects each tensor to be equal size, but got keypoint counts {kept}: pass "
                               "force_num_keypoints with B > 1")
        kpts, kscores, _ = select(s, threshold, max_kps, kept[0])
    return kpts, kscores


def sample(desc_nhwc, kpts, legacy):
    """L2-normalised bilinear samples [B, K, C] of desc [B, h, w, C] fp32 at kpts [B, K, 2] (score-map pixels)."""
    B, h, w, C = desc_nhwc.shape
    K = kpts.shape[1]
    out = torch.empty(B, K, C, device=desc_nhwc.device, dtype=torch.float32)
    _lib.call("lgb200_sp_sample", _p(desc_nhwc), _p(kpts), _p(out), B, K, h, w, C, int(bool(legacy)),
              _lib.stream_ptr())
    return out


class SuperPoint(nn.Module):
    default_conf = {
        "has_detector": True,
        "has_descriptor": True,
        "descriptor_dim": 256,
        "sparse_outputs": True,
        "dense_outputs": False,
        "nms_radius": 4,
        "refinement_radius": 0,
        "detection_threshold": 0.005,
        "max_num_keypoints": -1,
        "max_num_keypoints_val": None,
        "force_num_keypoints": False,
        "randomize_keypoints_training": False,
        "remove_borders": 4,
        "legacy_sampling": True,
        # glue-factory's BaseModel keys; the extractor is frozen, so trainable defaults to False here
        "name": None,
        "trainable": False,
        "freeze_batch_normalization": False,
        "timeit": False,
        # plugin-only
        "weights": "default",
        "precision": "bf16",
    }
    required_data_keys = ["image"]
    checkpoint_name = "superpoint_v1.pth"

    def __init__(self, conf=None):
        super().__init__()
        self.conf = conf = _Conf(_merge(self.default_conf, _to_plain(conf)))
        assert conf.precision in ("bf16", "fp32"), conf.precision
        if conf.trainable:
            raise NotImplementedError("gluefactory_b200 superpoint is inference only: trainable must be False")
        if conf.refinement_radius > 0:
            raise NotImplementedError("gluefactory_b200 superpoint: refinement_radius > 0 is not implemented")
        if not (conf.has_detector and conf.has_descriptor):
            raise NotImplementedError("gluefactory_b200 superpoint: the detector and descriptor heads are both required")
        if conf.descriptor_dim != 256:
            raise NotImplementedError(f"gluefactory_b200 superpoint: descriptor_dim {conf.descriptor_dim} (256 only)")
        if not 0 <= conf.nms_radius <= MAX_NMS_RADIUS:
            raise NotImplementedError(f"gluefactory_b200 superpoint: nms_radius {conf.nms_radius} (0 to {MAX_NMS_RADIUS})")
        for k in (conf.max_num_keypoints, conf.max_num_keypoints_val):
            if k is not None and k > MAX_K:
                raise NotImplementedError(f"gluefactory_b200 superpoint: at most {MAX_K} keypoints per image (got {k})")
        c1, c2, c3, c4, c5 = 64, 64, 128, 128, 256
        self.conv1a = nn.Conv2d(1, c1, kernel_size=3, stride=1, padding=1)
        self.conv1b = nn.Conv2d(c1, c1, kernel_size=3, stride=1, padding=1)
        self.conv2a = nn.Conv2d(c1, c2, kernel_size=3, stride=1, padding=1)
        self.conv2b = nn.Conv2d(c2, c2, kernel_size=3, stride=1, padding=1)
        self.conv3a = nn.Conv2d(c2, c3, kernel_size=3, stride=1, padding=1)
        self.conv3b = nn.Conv2d(c3, c3, kernel_size=3, stride=1, padding=1)
        self.conv4a = nn.Conv2d(c3, c4, kernel_size=3, stride=1, padding=1)
        self.conv4b = nn.Conv2d(c4, c4, kernel_size=3, stride=1, padding=1)
        self.convPa = nn.Conv2d(c4, c5, kernel_size=3, stride=1, padding=1)
        self.convPb = nn.Conv2d(c5, 65, kernel_size=1, stride=1, padding=0)
        self.convDa = nn.Conv2d(c4, c5, kernel_size=3, stride=1, padding=1)
        self.convDb = nn.Conv2d(c5, conf.descriptor_dim, kernel_size=1, stride=1, padding=0)
        if conf.weights is not None:
            self.load_state_dict(torch.load(self.weights_path(conf.weights), map_location="cpu"), strict=False)
        for p in self.parameters():
            p.requires_grad_(False)
        self._packed = None

    @classmethod
    def weights_path(cls, weights):
        """"default": torch-hub's cache file of the reference's checkpoint download (never downloaded); else a path."""
        path = str(_weights.hub_checkpoint(cls.checkpoint_name)) if weights == "default" else str(weights)
        if not os.path.isfile(path):
            raise FileNotFoundError(f"gluefactory_b200 superpoint: weights {weights!r} not found at {path} (this plugin "
                                    "never downloads; place the file there or pass weights=None)")
        return path

    # -- weights in the kernels' layouts, rebuilt when a parameter changes ------------------------------------------
    def _kernel_weights(self):
        key = tuple((p.data_ptr(), p._version, p.device) for p in self.parameters())
        if self._packed is not None and self._packed[0] == key:
            return self._packed[1]

        def k3(*convs):  # [Cout, Cin, 3, 3] -> [Cout, 9 Cin] bf16, K ordered (tap, channel)
            w = torch.cat([c.weight for c in convs])
            return w.permute(0, 2, 3, 1).reshape(w.shape[0], -1).to(torch.bfloat16).contiguous()

        def bias(*convs, n=None):
            b = torch.cat([c.bias for c in convs]).float()
            return F.pad(b, (0, (n or b.numel()) - b.numel())).contiguous()

        pb = self.convPb.weight.reshape(65, -1)
        pk = {
            "1a": (self.conv1a.weight.reshape(64, 9).float().contiguous(), bias(self.conv1a)),
            "1b": (k3(self.conv1b), bias(self.conv1b)),
            "2a": (k3(self.conv2a), bias(self.conv2a)),
            "2b": (k3(self.conv2b), bias(self.conv2b)),
            "3a": (k3(self.conv3a), bias(self.conv3a)),
            "3b": (k3(self.conv3b), bias(self.conv3b)),
            "4a": (k3(self.conv4a), bias(self.conv4a)),
            "4b": (k3(self.conv4b), bias(self.conv4b)),
            "PaDa": (k3(self.convPa, self.convDa), bias(self.convPa, self.convDa)),
            "Pb": (F.pad(pb, (0, 0, 0, 128 - 65)).to(torch.bfloat16).contiguous(), bias(self.convPb, n=128)),
            "Db": (self.convDb.weight.reshape(256, -1).to(torch.bfloat16).contiguous(), bias(self.convDb)),
        }
        self._packed = (key, pk)
        return pk

    def dense_bf16(self, image):
        """Dense scores [B, 8h, 8w] and L2-normalised descriptors [B, h, w, 256] (NHWC) from the wgmma kernels."""
        pk = self._kernel_weights()
        x = conv1a(image, *pk["1a"])
        x = conv(x, *pk["1b"], 64, 3, EP_POOL)
        x = conv(x, *pk["2a"], 64, 3, EP_RELU)
        x = conv(x, *pk["2b"], 64, 3, EP_POOL)
        x = conv(x, *pk["3a"], 128, 3, EP_RELU)
        x = conv(x, *pk["3b"], 128, 3, EP_POOL)
        x = conv(x, *pk["4a"], 128, 3, EP_RELU)
        x = conv(x, *pk["4b"], 128, 3, EP_RELU)
        pd = conv(x, *pk["PaDa"], 512, 3, EP_RELU)  # channels [0, 256): convPa, [256, 512): convDa
        scores = conv(pd, *pk["Pb"], 65, 1, EP_SOFTMAX, cin=256)
        desc = conv(pd, *pk["Db"], 256, 1, EP_L2N, cin=256, c0=256)
        return scores, desc

    def dense_fp32(self, image):
        """The parity path: fp32 cuDNN convolutions with TF32 off, the reference's dense formulas."""
        if image.shape[1] == 3:
            image = (image * image.new_tensor([0.299, 0.587, 0.114]).view(1, 3, 1, 1)).sum(1, keepdim=True)
        with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=True, allow_tf32=False):
            x = image
            for name in ("1a", "1b", "2a", "2b", "3a", "3b", "4a", "4b"):
                x = F.relu(getattr(self, "conv" + name)(x))
                if name in ("1b", "2b", "3b"):
                    x = F.max_pool2d(x, 2, 2)
            scores = self.convPb(F.relu(self.convPa(x)))
            desc = self.convDb(F.relu(self.convDa(x)))
        scores = F.softmax(scores, 1)[:, :-1]
        b, _, h, w = scores.shape
        scores = scores.permute(0, 2, 3, 1).reshape(b, h, w, 8, 8).permute(0, 1, 3, 2, 4).reshape(b, h * 8, w * 8)
        desc = F.normalize(desc, p=2, dim=1)
        return scores.contiguous(), desc.permute(0, 2, 3, 1).contiguous()

    def forward(self, data):
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        conf = self.conf
        image = data["image"]
        if any(p.requires_grad for p in self.parameters()) or (torch.is_grad_enabled() and image.requires_grad):
            raise NotImplementedError("gluefactory_b200 superpoint is inference only: no backward")
        if self.training and conf.randomize_keypoints_training:
            raise NotImplementedError("gluefactory_b200 superpoint: randomize_keypoints_training is not implemented")
        if not image.is_cuda:
            raise _lib.Lgb200Error("gluefactory_b200 superpoint runs on CUDA tensors only: there is no CPU fallback")
        image = image.float().contiguous()
        B, _, H, W = image.shape
        if H < 8 or W < 8:
            raise ValueError(f"gluefactory_b200 superpoint: image {H}x{W} is smaller than one 8x8 cell")
        with torch.no_grad():
            if conf.precision == "fp32":
                scores, desc = self.dense_fp32(image)
            else:
                scores, desc = self.dense_bf16(image)
            if not conf.sparse_outputs:
                return {"keypoint_scores": scores, "descriptors": desc.permute(0, 3, 1, 2)}
            return self._sparse(data, image, scores, desc)

    def _sparse(self, data, image, scores, desc):
        conf = self.conf
        dev = image.device
        image_size = data.get("image_size")
        if image_size is not None:
            image_size = image_size.to(device=dev, dtype=torch.float32).contiguous()
        s = nms(scores, conf.nms_radius, conf.remove_borders or 0, image_size)
        max_kps = conf.max_num_keypoints
        if not self.training and conf.max_num_keypoints_val is not None:
            max_kps = conf.max_num_keypoints_val
        kpts, kscores = select_keypoints(s, conf.detection_threshold, max_kps, conf.force_num_keypoints, image_size,
                                         image.shape[-2:])
        pred = {
            "keypoints": kpts + 0.5,
            "keypoint_scores": kscores,
            "descriptors": sample(desc, kpts, conf.legacy_sampling),
        }
        if conf.dense_outputs:
            pred["dense_descriptors"] = desc.permute(0, 3, 1, 2)
        return pred

    def loss(self, pred, data):
        raise NotImplementedError

    def metrics(self, pred, data):
        raise NotImplementedError


__main_model__ = SuperPoint
