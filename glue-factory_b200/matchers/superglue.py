"""H100-native SuperGlue matcher -- drop-in for glue-factory's `gluefactory_nonfree.superglue` (BASELINE.json: the
SuperPoint + SuperGlue configuration, `configs/superpoint+superglue-official.yaml`).

Select it with `model.matcher.name: gluefactory_b200.matchers.superglue`.  Same constructor, `forward(data) -> pred`,
`required_data_keys` and module tree as the reference (superglue.py:70-355), so parameter / buffer names and shapes
equal the reference's state_dict and its checkpoints load as they are.

Kernels.  The point-side GNN is GlueStick's (matchers/_point_gnn.py: wgmma GEMMs and attention, fused BatchNorm +
ReLU); the assignment is log-domain Sinkhorn with a learnt dustbin score (superglue.py:186-214) as two persistent
kernels that read the bin score on the device (`ops.log_optimal_transport`); the NLL over its dense output is one
pass over the byte ground-truth mask (`ops.ot_nll`), and the match filter (superglue.py:301-311) runs on the row /
column argmax of that output (`ops.ot_filter_stats` + `ops.filter_matches`).  The Sinkhorn head is fp32 in both
precisions; in bf16 mode its cost comes from the fp32-output wgmma GEMM.  No CPU fallback.

Deliberate differences from the reference:
  * `loss` returns `(losses, metrics)` like every other matcher (TwoViewPipeline.loss unpacks two values,
    two_view_pipeline.py:107; the reference returns the losses alone, so it cannot train through the pipeline).
    `metrics` is matcher_metrics in eval mode and empty in training.
  * `weights: "indoor" | "outdoor"` never downloads: `superglue_{name}.pth` is read from torch-hub's checkpoint cache
    (`torch.hub.get_dir()/checkpoints`) and a missing file raises FileNotFoundError; any other string is a local file.
  * The keypoint range assertion (superglue.py:285-286) reads back to the host, so it runs only outside CUDA-graph
    capture.  `view["image"]` is read only when `image_size` is absent.
Training reproduces the reference's BatchNorm bookkeeping: its GNN layers run under torch.utils.checkpoint, whose
backward recomputes each layer in training mode and so updates the layer's BatchNorm running statistics a second
time (image 0, then image 1).  Here a backward hook per layer applies that second update from the batch statistics
the forward used.
"""
import os
from copy import deepcopy

import torch
from torch import nn

from .. import _lib, ops
from ._point_gnn import PointGNN
from .gluestick import MLP
from .lightglue import _Conf, _merge, _to_plain, matcher_metrics


class KeypointEncoder(nn.Module):
    def __init__(self, feature_dim, layers, use_scores=True):
        super().__init__()
        self.use_scores = use_scores
        self.encoder = MLP([3 if use_scores else 2] + list(layers) + [feature_dim])
        nn.init.constant_(self.encoder[-1].bias, 0.0)


class MultiHeadedAttention(nn.Module):
    def __init__(self, h, d_model):
        super().__init__()
        self.dim, self.h = d_model // h, h
        self.merge = nn.Conv1d(d_model, d_model, kernel_size=1)
        self.proj = nn.ModuleList([deepcopy(self.merge) for _ in range(3)])  # all four start equal, as the reference's


class AttentionalPropagation(nn.Module):
    def __init__(self, num_dim, num_heads):
        super().__init__()
        self.attn = MultiHeadedAttention(num_heads, num_dim)
        self.mlp = MLP([num_dim * 2, num_dim * 2, num_dim])
        nn.init.constant_(self.mlp[-1].bias, 0.0)


class AttentionalGNN(nn.Module):
    def __init__(self, feature_dim, layer_names):
        super().__init__()
        self.layers = nn.ModuleList([AttentionalPropagation(feature_dim, 4) for _ in range(len(layer_names))])
        self.names = list(layer_names)


class SuperGlue(PointGNN):
    default_conf = {
        "descriptor_dim": 256,
        "weights": "outdoor",
        "keypoint_encoder": [32, 64, 128, 256],
        "GNN_layers": ["self", "cross"] * 9,
        "num_sinkhorn_iterations": 50,
        "filter_threshold": 0.2,
        "use_scores": True,
        "loss": {"nll_balancing": 0.5},
        "precision": "bf16",
    }
    required_data_keys = ["view0", "view1", "keypoints0", "keypoints1", "descriptors0", "descriptors1",
                          "keypoint_scores0", "keypoint_scores1"]

    def __init__(self, conf=None):
        super().__init__()
        self.conf = conf = _Conf(_merge(self.default_conf, _to_plain(conf)))
        assert conf.precision in ("bf16", "fp32"), conf.precision
        D = conf.descriptor_dim
        if D != 256:
            raise NotImplementedError("gluefactory_b200 superglue: the attention kernels are built for 4 heads of 64 "
                                      f"channels (descriptor_dim 256), got {D}")
        for name in conf.GNN_layers:
            if name not in ("self", "cross"):
                raise ValueError(name)
        # registration order = the reference's (superglue.py:247-258): state_dict keys come out identical
        self.kenc = KeypointEncoder(D, conf.keypoint_encoder, conf.use_scores)
        self.gnn = AttentionalGNN(D, list(conf.GNN_layers))
        self.final_proj = nn.Conv1d(D, D, kernel_size=1, bias=True)
        self.register_parameter("bin_score", nn.Parameter(torch.tensor(1.0)))
        if conf.weights:
            self.load_state_dict(torch.load(self._weights_path(conf.weights), map_location="cpu"))
        self._register_head_perm(D)

    @staticmethod
    def _weights_path(weights):
        """"indoor" / "outdoor": the pretrained file in torch-hub's checkpoint cache (never downloaded); else a path."""
        if weights in ("indoor", "outdoor"):
            path = os.path.join(torch.hub.get_dir(), "checkpoints", f"superglue_{weights}.pth")
        else:
            path = weights
        if not os.path.isfile(path):
            raise FileNotFoundError(f"gluefactory_b200 superglue: weights {weights!r} not found at {path} (this "
                                    "plugin never downloads; place the file there or pass weights=None)")
        return path

    @staticmethod
    def _image_size(view, kpts):
        size = view.get("image_size")
        if size is not None:
            return size
        h, w = view["image"].shape[-2:]
        return kpts.new_tensor([[float(w), float(h)]])

    # ------------------------------------------------------------------------------------------ forward / loss
    def forward(self, data):
        with torch.autocast(device_type="cuda", enabled=False):
            return self._forward(data)

    def _forward(self, data):
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        kp0, kp1 = data["keypoints0"], data["keypoints1"]
        if kp0.shape[1] == 0 or kp1.shape[1] == 0:  # no keypoints (superglue.py:270-277)
            shape0, shape1 = kp0.shape[:-1], kp1.shape[:-1]
            return {"matches0": kp0.new_full(shape0, -1, dtype=torch.int),
                    "matches1": kp1.new_full(shape1, -1, dtype=torch.int),
                    "matching_scores0": kp0.new_zeros(shape0), "matching_scores1": kp1.new_zeros(shape1)}
        _lib.load()  # raises unless the CUDA library is built and the device is an H100 (no CPU fallback)
        kp0, kp1 = kp0.float(), kp1.float()
        B, n0 = kp0.shape[:2]
        n1 = kp1.shape[1]
        k0 = self._norm_kpts(kp0, self._image_size(data["view0"], kp0))
        k1 = self._norm_kpts(kp1, self._image_size(data["view1"], kp1))
        if not torch.cuda.is_current_stream_capturing():  # a host read-back: eager mode only
            assert torch.all(k0 >= -1) and torch.all(k0 <= 1)
            assert torch.all(k1 >= -1) and torch.all(k1 <= 1)
        D = self.conf.descriptor_dim

        def enc_in(k, s):
            return (torch.cat([k, s.float()[..., None]], -1) if self.conf.use_scores else k).reshape(B * k.shape[1], -1)

        d0 = data["descriptors0"].float().reshape(B * n0, D) + self._mlp(enc_in(k0, data["keypoint_scores0"]),
                                                                           self.kenc.encoder)
        d1 = data["descriptors1"].float().reshape(B * n1, D) + self._mlp(enc_in(k1, data["keypoint_scores1"]),
                                                                           self.kenc.encoder)
        recompute_bn = self.training and torch.is_grad_enabled()
        for layer, name in zip(self.gnn.layers, self.gnn.names):
            stats = [] if recompute_bn else None
            d0, d1 = self._gnn_layer(d0, d1, layer, name == "cross", B, stats)
            if stats and (d0.requires_grad or d1.requires_grad):
                self._bn_update_on_backward(d0, d1, stats)
        cost = self._similarity(self._conv(d0, self.final_proj), self._conv(d1, self.final_proj), B)
        scores = ops.log_optimal_transport(cost, self.bin_score, self.conf.num_sinkhorn_iterations)
        m0, m1, ms0, ms1 = ops.filter_matches(*ops.ot_filter_stats(scores.detach()), self.conf.filter_threshold)
        return {"sinkhorn_cost": cost, "log_assignment": scores, "matches0": m0, "matches1": m1,
                "matching_scores0": ms0, "matching_scores1": ms1}

    @staticmethod
    def _bn_update_on_backward(d0, d1, stats):
        """The reference's checkpointed layer is recomputed in training mode when the backward first reaches it; that
        recomputation updates the layer's BatchNorm running statistics again, image 0 then image 1.  The hook fires at
        the same point and applies the same updates from the statistics this forward saved (exchanged ones under
        SyncBatchNorm)."""
        def second_update(_):
            for bn, sums in stats:
                ops.bn_running_update(sums, bn)

        outs = tuple(t for t in (d0, d1) if t.requires_grad)
        torch.autograd.graph.register_multi_grad_hook(outs, second_update, mode="any")

    def loss(self, pred, data):
        """superglue.py:322-352, returned as (losses, metrics) like the other matchers."""
        with torch.autocast(device_type="cuda", enabled=False):
            nll_pos, nll_neg, num_pos, num_neg = ops.ot_nll(pred["log_assignment"], data["gt_assignment"],
                                                            data["gt_matches0"], data["gt_matches1"])
            bal = self.conf.loss.nll_balancing
            nll = bal * nll_pos + (1 - bal) * nll_neg
            losses = {"total": nll, "assignment_nll": nll, "nll_pos": nll_pos, "nll_neg": nll_neg,
                      "num_matchable": num_pos, "num_unmatchable": num_neg, "bin_score": self.bin_score[None]}
            metrics = {} if self.training else matcher_metrics(pred, data)
            return losses, metrics


__main_model__ = SuperGlue
