"""H100-native SuperPoint-open keypoint extractor, inference only -- drop-in for glue-factory's MIT-licensed
`extractors.superpoint_open` (the frozen extractor of `superpoint-open+lightglue_homography.yaml`, where every sample
is a freshly warped image and the features cannot be cached).

Select it with `model.extractor.name: gluefactory_b200.extractors.superpoint_open`.  Same `default_conf`,
`required_data_keys` and module tree (`backbone.i.j.{conv,bn}`, `detector.j.*`, `descriptor.j.*`, each a VGGBlock
conv -> ReLU -> BatchNorm2d(eps=1e-3)) as the reference, so `superpoint_v6_from_tf.pth` and the reference's state_dict
load strictly in both directions.  `weights` keeps the reference's meaning: an existing path is loaded, otherwise the
default checkpoint is read from torch-hub's cache; this plugin never downloads (a missing file raises
FileNotFoundError naming the paths tried).  One plugin-only key, `precision`: "bf16" (default) runs the wgmma kernels of
csrc/superpoint.cu; "fp32" is the parity path, the module's own torch layers under fp32 cuDNN with TF32 off.

BatchNorm follows each BatchNorm module, as torch does: with running statistics (eval mode, or
`freeze_batch_normalization`) its affine is folded into the conv epilogues; with batch statistics (training mode, as
glue-factory's `model.train()` leaves it in every SuperPoint-open config) each BatchNorm normalises with the
statistics of this call's batch, summed across the ranks of an nn.SyncBatchNorm, and updates running_mean,
running_var and num_batches_tracked on the device.  With `force_num_keypoints` neither mode reads anything back to the
host, so the extractor can be captured in a CUDA graph together with the matcher step.

Keypoints come from the same NMS (fixed border frame of the score map), selection and sampling kernels as the
`superpoint` plugin: the k best in descending score order, exact ties to the lower row-major index, or every
candidate in row-major order when there are no more than k; descriptors sampled at kp + 0.5 (align_corners=False).

Refused with NotImplementedError: `trainable: True` and any backward, `channels` other than [64, 64, 128, 128, 256],
`descriptor_dim` other than 256, `nms_radius` > 9, more than 16384 keypoints, and (bf16) a BatchNorm with
momentum=None or affine=False.  B > 1 without `force_num_keypoints` raises ValueError: the reference fails there too.
No CPU fallback.
"""
from collections import OrderedDict

import torch
import torch.nn.functional as F
from torch import nn

from .. import _lib, ops
from ..matchers import _weights
from ..matchers.lightglue import _Conf, _merge, _to_plain
from . import superpoint as sp

EP_RELU, EP_POOL, EP_SOFTMAX, EP_L2N, EP_RAW = 0, 1, 2, 3, 4  # LGB200_SP_* and LGB200_SPO_RAW
BN_PLAIN, BN_POOL, BN_SOFTMAX, BN_L2N = 0, 1, 2, 3  # LGB200_SPO_BN_*
CHANNELS = [64, 64, 128, 128, 256]
_p = _lib.ptr


def conv1a(image, weight, bias, scale, shift):
    """ReLU(conv3x3(gray(image))) * scale + shift as NHWC bf16 [B, H, W, 64]."""
    B, C, H, W = image.shape
    out = torch.empty(B, H, W, 64, device=image.device, dtype=torch.bfloat16)
    _lib.call("lgb200_spo_conv1a", _p(image), C, _p(weight), _p(bias), _p(scale), _p(shift), _p(out), B, H, W,
              _lib.stream_ptr())
    return out


def conv(x, weight, bias, scale, shift, cout, ksize, epilogue, cin=None, c0=0):
    """sp.conv with the eval-mode BatchNorm affine in the epilogue, or EP_RAW: conv + bias as fp32 [B, H, W, Npad]."""
    B, H, W, ldx = x.shape
    cin = ldx - c0 if cin is None else cin
    dev = x.device
    if epilogue == EP_POOL:
        out = torch.empty(B, H // 2, W // 2, cout, device=dev, dtype=torch.bfloat16)
    elif epilogue == EP_RELU:
        out = torch.empty(B, H, W, cout, device=dev, dtype=torch.bfloat16)
    elif epilogue == EP_SOFTMAX:
        out = torch.empty(B, 8 * H, 8 * W, device=dev, dtype=torch.float32)
    elif epilogue == EP_RAW:
        out = torch.empty(B, H, W, -(-cout // 128) * 128, device=dev, dtype=torch.float32)
    else:
        out = torch.empty(B, H, W, cout, device=dev, dtype=torch.float32)
    _lib.call("lgb200_spo_conv", x.data_ptr() + 2 * c0, ldx, _p(weight), _p(bias), _p(scale), _p(shift), _p(out),
              B, H, W, cin, cout, ksize, epilogue, _lib.stream_ptr())
    return out


def bn_apply(x, sums, weight, bias, eps, op):
    """Training-mode BatchNorm of NHWC x from the batch statistics `sums` (ops.bn_stats layout over C = len(weight)),
    then nothing (BN_PLAIN), a 2x2 max-pool, the 65-way softmax with depth-to-space, or the L2 normalisation."""
    B, H, W, _ = x.shape
    C = weight.numel()
    dev = x.device
    if op == BN_PLAIN:
        out = torch.empty_like(x)
    elif op == BN_POOL:
        out = torch.empty(B, H // 2, W // 2, C, device=dev, dtype=x.dtype)
    elif op == BN_SOFTMAX:
        out = torch.empty(B, 8 * H, 8 * W, device=dev, dtype=torch.float32)
    else:
        out = torch.empty_like(x)
    _lib.call("lgb200_spo_bn_apply", _p(x), _p(sums), _p(weight), _p(bias), float(eps), _p(out), B, H, W, C, int(op),
              _lib.stream_ptr())
    return out


def batch_statistics(bn):
    """True when BatchNorm `bn` normalises with the statistics of the batch (torch: training, or no running stats)."""
    return bn.training or not bn.track_running_stats


def bn_affine(bn):
    """(scale, shift) [C] fp32 of BatchNorm `bn` with its running statistics, for the eval-mode epilogues.  Computed on
    the device at every call: the running statistics change without a version bump (lgb200_bn_running_update writes
    them in place, also from a replayed CUDA graph), so no cache could tell when they moved."""
    scale = (bn.weight.float() / torch.sqrt(bn.running_var.float() + bn.eps)).contiguous()
    return scale, (bn.bias.float() - bn.running_mean.float() * scale).contiguous()


class VGGBlock(nn.Sequential):
    """conv (padding k // 2) -> ReLU (or identity) -> BatchNorm2d(eps=1e-3), under the reference's module names."""

    def __init__(self, c_in, c_out, kernel_size, relu=True):
        super().__init__(OrderedDict(conv=nn.Conv2d(c_in, c_out, kernel_size, stride=1, padding=kernel_size // 2),
                                     activation=nn.ReLU(inplace=True) if relu else nn.Identity(),
                                     bn=nn.BatchNorm2d(c_out, eps=0.001)))


def _module_tree():
    """backbone (four stages of two VGGBlocks, the first three closed by a 2x2 max-pool), detector and descriptor."""
    c = [1] + CHANNELS[:-1]
    backbone = nn.Sequential(*[
        nn.Sequential(VGGBlock(c[i - 1], c[i], 3), VGGBlock(c[i], c[i], 3), *([nn.MaxPool2d(2, 2)] if i < 4 else []))
        for i in range(1, 5)])
    detector = nn.Sequential(VGGBlock(128, 256, 3), VGGBlock(256, 65, 1, relu=False))
    descriptor = nn.Sequential(VGGBlock(128, 256, 3), VGGBlock(256, 256, 1, relu=False))
    return backbone, detector, descriptor


class SuperPointOpen(nn.Module):
    default_conf = {
        "descriptor_dim": 256,
        "nms_radius": 4,
        "max_num_keypoints": None,
        "force_num_keypoints": False,
        "detection_threshold": 0.005,
        "remove_borders": 4,
        "channels": list(CHANNELS),
        "dense_outputs": None,
        "weights": None,
        # glue-factory's BaseModel keys; the extractor is frozen, so trainable defaults to False here
        "name": None,
        "trainable": False,
        "freeze_batch_normalization": False,
        "timeit": False,
        # plugin-only
        "precision": "bf16",
    }
    required_data_keys = ["image"]
    checkpoint_name = "superpoint_v6_from_tf.pth"

    def __init__(self, conf=None):
        super().__init__()
        self.conf = conf = _Conf(_merge(self.default_conf, _to_plain(conf)))
        assert conf.precision in ("bf16", "fp32"), conf.precision
        if conf.trainable:
            raise NotImplementedError("gluefactory_b200 superpoint_open is inference only: trainable must be False")
        if list(conf.channels) != CHANNELS:
            raise NotImplementedError(f"gluefactory_b200 superpoint_open: channels {list(conf.channels)} "
                                      f"({CHANNELS} only)")
        if conf.descriptor_dim != 256:
            raise NotImplementedError(f"gluefactory_b200 superpoint_open: descriptor_dim {conf.descriptor_dim} "
                                      "(256 only)")
        if not 0 <= conf.nms_radius <= sp.MAX_NMS_RADIUS:
            raise NotImplementedError(f"gluefactory_b200 superpoint_open: nms_radius {conf.nms_radius} "
                                      f"(0 to {sp.MAX_NMS_RADIUS})")
        if conf.max_num_keypoints is not None and conf.max_num_keypoints > sp.MAX_K:
            raise NotImplementedError(f"gluefactory_b200 superpoint_open: at most {sp.MAX_K} keypoints per image "
                                      f"(got {conf.max_num_keypoints})")
        self.backbone, self.detector, self.descriptor = _module_tree()
        self.load_state_dict(self.load_weights(conf.weights))
        for p in self.parameters():
            p.requires_grad_(False)
        self._packed = None

    @staticmethod
    def state_dict_template():
        """The module tree's state_dict at torch's initialisation: names and shapes, without reading any weights."""
        m = nn.Module()
        m.backbone, m.detector, m.descriptor = _module_tree()
        return m.state_dict()

    @classmethod
    def load_weights(cls, weights):
        """The reference's lookup without its download: `weights` when that file exists, else torch-hub's cache file
        of the default checkpoint; FileNotFoundError listing both when neither exists."""
        default = _weights.hub_checkpoint(cls.checkpoint_name)
        if weights is None:
            return _weights.load_weights(default, [], "superpoint_open")
        return _weights.load_weights(weights, [default], "superpoint_open")

    def train(self, mode=True):
        """nn.Module.train, then BaseModel's freeze_batch_normalization: every BatchNorm back to eval mode."""
        super().train(mode)
        if self.conf.freeze_batch_normalization:
            for m in self.modules():
                if isinstance(m, nn.modules.batchnorm._BatchNorm):
                    m.eval()
        return self

    def _blocks(self):
        return [self.backbone[i][j] for i in range(4) for j in range(2)]

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

        blocks = self._blocks()
        c1a = blocks[0].conv
        pk = {"enc": [(c1a.weight.reshape(64, 9).float().contiguous(), bias(c1a))] +
                     [(k3(b.conv), bias(b.conv)) for b in blocks[1:]]}
        pa, da, pb, db = self.detector[0].conv, self.descriptor[0].conv, self.detector[1].conv, self.descriptor[1].conv
        w, b = k3(pa, da), bias(pa, da)  # rows [0, 256): Pa, [256, 512): Da; the halves are contiguous views
        pk["PaDa"], pk["Pa"], pk["Da"] = (w, b), (w[:256], b[:256]), (w[256:], b[256:])
        pk["Pb"] = (F.pad(pb.weight.reshape(65, -1), (0, 0, 0, 128 - 65)).to(torch.bfloat16).contiguous(),
                    bias(pb, n=128))
        pk["Db"] = (db.weight.reshape(256, -1).to(torch.bfloat16).contiguous(), bias(db))
        self._packed = (key, pk)
        return pk

    def _batchnorms(self):
        """Every BatchNorm of the tree: BatchNorm2d, or nn.SyncBatchNorm after convert_sync_batchnorm (--distributed)."""
        return [m for m in self.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)]

    def _normalise(self, y, bn, op):
        """Training-mode BatchNorm of the pre-BatchNorm activation y [B, H, W, ld] (ld >= bn.num_features): batch
        statistics summed across the module's ranks, the running-statistics update, then `op`."""
        C = bn.num_features
        ld = y.shape[-1]
        exchange = ops.bn_exchange(bn)
        if exchange is None and y.numel() // ld < 2:
            raise ValueError(f"Expected more than 1 value per channel when training, got input size "
                             f"{(y.shape[0], C, *y.shape[1:3])}")
        sums = ops.bn_stats(y.view(-1, ld))
        if ld != C:
            sums = torch.cat([sums[:C], sums[ld:ld + C], sums[2 * ld:]])
        if exchange is not None:
            exchange(sums)
        if bn.training and bn.track_running_stats:
            ops.bn_running_update(sums, bn)
        return bn_apply(y, sums, bn.weight.float().contiguous(), bn.bias.float().contiguous(), bn.eps, op)

    def dense_bf16(self, image):
        """Dense scores [B, 8h, 8w] and L2-normalised descriptors [B, h, w, 256] (NHWC) from the wgmma kernels."""
        pk = self._kernel_weights()
        x = image
        for i, (blk, (w, b)) in enumerate(zip(self._blocks(), pk["enc"])):
            pool = i in (1, 3, 5)  # the MaxPool2d closing backbone.0 .. backbone.2
            cout = blk.conv.out_channels
            if not batch_statistics(blk.bn):
                x = conv1a(x, w, b, *bn_affine(blk.bn)) if i == 0 else \
                    conv(x, w, b, *bn_affine(blk.bn), cout, 3, EP_POOL if pool else EP_RELU)
            else:
                y = sp.conv1a(x, w, b) if i == 0 else sp.conv(x, w, b, cout, 3, EP_RELU)
                x = self._normalise(y, blk.bn, BN_POOL if pool else BN_PLAIN)
        (pa, pb), (da, db) = self.detector, self.descriptor
        if not (batch_statistics(pa.bn) or batch_statistics(da.bn)):
            scale, shift = (torch.cat([a, d]) for a, d in zip(bn_affine(pa.bn), bn_affine(da.bn)))
            xp = xd = conv(x, *pk["PaDa"], scale, shift, 512, 3, EP_RELU)
            cp, cd = 0, 256
        else:
            xp, xd = (conv(x, *pk[n], *bn_affine(m.bn), 256, 3, EP_RELU) if not batch_statistics(m.bn) else
                      self._normalise(sp.conv(x, *pk[n], 256, 3, EP_RELU), m.bn, BN_PLAIN)
                      for n, m in (("Pa", pa), ("Da", da)))
            cp = cd = 0
        if not batch_statistics(pb.bn):
            scale, shift = (F.pad(t, (0, 128 - 65)) for t in bn_affine(pb.bn))
            scores = conv(xp, *pk["Pb"], scale, shift, 65, 1, EP_SOFTMAX, cin=256, c0=cp)
        else:
            scores = self._normalise(conv(xp, *pk["Pb"], None, None, 65, 1, EP_RAW, cin=256, c0=cp), pb.bn,
                                     BN_SOFTMAX)
        if not batch_statistics(db.bn):
            desc = conv(xd, *pk["Db"], *bn_affine(db.bn), 256, 1, EP_L2N, cin=256, c0=cd)
        else:
            desc = self._normalise(conv(xd, *pk["Db"], None, None, 256, 1, EP_RAW, cin=256, c0=cd), db.bn, BN_L2N)
        return scores, desc

    def dense_fp32(self, image):
        """The parity path: the module's own layers (torch's BatchNorm in either mode) under fp32 cuDNN, TF32 off."""
        if image.shape[1] == 3:
            image = (image * image.new_tensor([0.299, 0.587, 0.114]).view(1, 3, 1, 1)).sum(1, keepdim=True)
        with torch.backends.cudnn.flags(enabled=True, benchmark=False, deterministic=True, allow_tf32=False):
            features = self.backbone(image)
            desc = F.normalize(self.descriptor(features), p=2, dim=1)
            scores = self.detector(features)
        scores = F.softmax(scores, 1)[:, :-1]
        b, _, h, w = scores.shape
        scores = scores.permute(0, 2, 3, 1).reshape(b, h, w, 8, 8).permute(0, 1, 3, 2, 4).reshape(b, h * 8, w * 8)
        return scores.contiguous(), desc.permute(0, 2, 3, 1).contiguous()

    def forward(self, data):
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        conf = self.conf
        image = data["image"]
        if any(p.requires_grad for p in self.parameters()) or (torch.is_grad_enabled() and image.requires_grad):
            raise NotImplementedError("gluefactory_b200 superpoint_open is inference only: no backward")
        B, _, H, W = image.shape
        if H < 8 or W < 8:
            raise ValueError(f"gluefactory_b200 superpoint_open: image {H}x{W} is smaller than one 8x8 cell")
        if B > 1 and not conf.force_num_keypoints:
            raise ValueError("gluefactory_b200 superpoint_open: B > 1 needs force_num_keypoints (the reference fails "
                             "there too: its per-image descriptors come back as a list)")
        if conf.precision == "bf16" and any(m.momentum is None or not m.affine for m in self._batchnorms()):
            raise NotImplementedError("gluefactory_b200 superpoint_open: BatchNorm with momentum=None or affine=False "
                                      "is not built")
        if not image.is_cuda:
            raise _lib.Lgb200Error("gluefactory_b200 superpoint_open runs on CUDA tensors only: there is no CPU "
                                   "fallback")
        image = image.float().contiguous()
        with torch.no_grad():
            scores, desc = self.dense_fp32(image) if conf.precision == "fp32" else self.dense_bf16(image)
            s = sp.nms(scores, conf.nms_radius, conf.remove_borders or 0)
            max_kps = -1 if conf.max_num_keypoints is None else conf.max_num_keypoints
            image_size = data.get("image_size")
            if image_size is not None:
                image_size = image_size.to(device=image.device, dtype=torch.float32).contiguous()
            kpts, kscores = sp.select_keypoints(s, conf.detection_threshold, max_kps, conf.force_num_keypoints,
                                                image_size, (H, W))
            kpts = kpts + 0.5
            # sample_descriptors' (kp + 0.5) / (wh s) is the fixed-mode formula at the shifted keypoints
            pred = {"keypoints": kpts, "keypoint_scores": kscores, "descriptors": sp.sample(desc, kpts, False)}
            if conf.dense_outputs:
                pred["dense_descriptors"] = desc.permute(0, 3, 1, 2)
        return pred

    def loss(self, pred, data):
        raise NotImplementedError

    def metrics(self, pred, data):
        raise NotImplementedError


__main_model__ = SuperPointOpen
