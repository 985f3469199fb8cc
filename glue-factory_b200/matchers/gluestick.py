"""H100-native GlueStick matcher (points + lines) -- drop-in for gluefactory's in-tree `matchers.gluestick`
(BASELINE.json configs[4]: SP + LSD + GlueStick; SURVEY.md section 8a row a15).

Select it with `model.matcher.name: gluefactory_b200.matchers.gluestick`.  Same constructor, `forward(data) -> pred`,
`loss(pred, data) -> (losses, metrics)`, `required_data_keys`, and the same module tree, so parameter / buffer names
and shapes equal the reference's state_dict (Conv1d weights [out, in, 1], BatchNorm running statistics) and
checkpoints are interchangeable (gluestick.py:68-141).

Layout and kernels.  The reference keeps channels first ([B, D, N], Conv1d with kernel 1, gluestick.py:158); here the
node features are token-major [B*N, D] like in the LightGlue plugin, so
  * every Conv1d(k=1) with a tensor-core-sized input is the library's wgmma GEMM (`ops.LinearFn`: bias in the
    epilogue, split-K weight gradient); the tiny encoder layers (3 / 5 / 32 input channels) are plain fp32 linears;
  * the attention core (gluestick.py:524-529) is the same wgmma flash-attention pair as LightGlue's, at head dim 64
    (descriptor_dim 256) or 32 (descriptor_dim 128, the configs' DISK variant).  GlueStick splits heads as
    channel = d * H + h; instead of permuting activations, the rows of the q / k / v projection weights and the
    columns of the merge weight are permuted once per call so the projections emit head-major [B, N, H, D / 4] directly;
  * the assignment is `log_double_softmax` with a learnt bin (gluestick.py:772-783) on the similarity produced by the
    batched wgmma GEMM: forward kernels + closed-form backward (`ops.log_double_softmax`, heads_grad.py);
  * match filtering (`_get_matches`, gluestick.py:318-331) is `filter_matches_kernel`;
  * every BatchNorm1d and the ReLU behind it are one fused pair of kernels (`ops.batchnorm_relu`): a deterministic fp64
    statistics pass, then normalisation + ReLU + the running-stat update on the device; the backward likewise.  Under
    glue-factory's distributed trainer the BatchNorms are `nn.SyncBatchNorm` (train.py:337-339, convert_sync_batchnorm
    before the DDP wrap): their statistics and backward sums are then all-reduced over the module's process group
    between the two passes, so every rank normalises with the global batch's statistics like the reference;
  * the LineLayer's gather and mean over junctions, and the line scores from the junction similarity, are kernels that
    sum in a fixed order in both directions (`ops.JunctionGather`, `ops.JunctionMean`, `ops.LineScores`): the endpoints
    are sorted stably by junction once per forward (`junction_layout`), so a wireframe with shared junctions trains to
    the same bits on every run.
Batches of pairs of different sizes (eval, `num_keypoints0/1`, `num_lines0/1`) run `_forward_packed`: packed tokens,
length-aware attention, the same LineLayer on a packed JunctionLayout and the varlen heads
(`ops.log_double_softmax_varlen`, `ops.line_scores_varlen`); see INTEGRATION.md for its outputs and refusals.
`precision: "bf16"` (default) rounds GEMM / attention operands to bf16 (the reference forces its attention to fp32,
gluestick.py:17-22; the fp32 mode reproduces that); `precision: "fp32"` is the parity path (fp32 cuBLAS linears,
CUDA-core attention).  No CPU fallback.

Intermediate line supervision (`inter_supervision`, gluestick.py:96-107, 272-292, 378-460): for each listed GNN block
the node features after its cross layer go through the same line head as the final ones (`_line_head`) with that
block's `inter_line_proj`, and their NLL is added to the total with the block's `loss.inter_supervision` weight.

Views without keypoints or lines follow the reference: no keypoints in a view returns its early-exit pred
(`_empty_pred`); no lines in a view skips every LineLayer and line head and returns zero / -1 line outputs, and `loss`
then raises ValueError (no loss is defined here for such views: the reference drops the line term without
inter_supervision and fails with it).  A view without `image_size` is normalised with
`view["image"].shape[-2:]`.  `weights` is a path or a name resolved to DATA_PATH/weights/{weights}_{version}.tar from
the local disk only (matchers/_weights.py).

Not built (raise NotImplementedError): `line_attention`, `skip_init`.
"""
from typing import NamedTuple, Optional

import torch
from torch import nn

from .. import _lib, ops
from . import _weights
from ._point_gnn import PointGNN, _norm_kpts_packed, _padded_outputs
from .lightglue import _Conf, _merge, _to_plain, keypoint_counts, matcher_metrics, ragged_layout, segment_rows


def MLP(channels, do_bn=True):
    """gluestick.py:465-475 (same module indices: conv, BN, ReLU, conv, ...)."""
    layers = []
    n = len(channels)
    for i in range(1, n):
        layers.append(nn.Conv1d(channels[i - 1], channels[i], kernel_size=1, bias=True))
        if i < n - 1:
            if do_bn:
                layers.append(nn.BatchNorm1d(channels[i]))
            layers.append(nn.ReLU())
    return nn.Sequential(*layers)


class KeypointEncoder(nn.Module):
    def __init__(self, feature_dim, layers):
        super().__init__()
        self.encoder = MLP([3] + list(layers) + [feature_dim])
        nn.init.constant_(self.encoder[-1].bias, 0.0)


class EndPtEncoder(nn.Module):
    def __init__(self, feature_dim, layers):
        super().__init__()
        self.encoder = MLP([5] + list(layers) + [feature_dim])
        nn.init.constant_(self.encoder[-1].bias, 0.0)


class MultiHeadedAttention(nn.Module):
    def __init__(self, h, d_model):
        super().__init__()
        self.dim, self.h = d_model // h, h
        self.merge = nn.Conv1d(d_model, d_model, kernel_size=1)
        self.proj = nn.ModuleList([nn.Conv1d(d_model, d_model, kernel_size=1) for _ in range(3)])


class AttentionalPropagation(nn.Module):
    def __init__(self, num_dim, num_heads):
        super().__init__()
        self.attn = MultiHeadedAttention(num_heads, num_dim)
        self.mlp = MLP([num_dim * 2, num_dim * 2, num_dim])
        nn.init.constant_(self.mlp[-1].bias, 0.0)


class GNNLayer(nn.Module):
    def __init__(self, feature_dim, layer_type):
        super().__init__()
        assert layer_type in ("cross", "self")
        self.type = layer_type
        self.update = AttentionalPropagation(feature_dim, 4)


class LineLayer(nn.Module):
    def __init__(self, feature_dim):
        super().__init__()
        self.mlp = MLP([feature_dim * 3, feature_dim * 2, feature_dim])


class AttentionalGNN(nn.Module):
    def __init__(self, feature_dim, layer_types):
        super().__init__()
        self.layers = nn.ModuleList([GNNLayer(feature_dim, t) for t in layer_types])
        self.line_layers = nn.ModuleList([LineLayer(feature_dim) for _ in range(len(layer_types) // 2)])


class GlueStick(PointGNN):
    default_conf = {
        "name": "gluestick",
        "input_dim": 256,
        "descriptor_dim": 256,
        "weights": None,
        "version": "v0.1_arxiv",
        "keypoint_encoder": [32, 64, 128, 256],
        "GNN_layers": ["self", "cross"] * 9,
        "num_line_iterations": 1,
        "line_attention": False,
        "filter_threshold": 0.2,
        "checkpointed": False,  # accepted; the fused attention keeps no N x N activations to checkpoint
        "skip_init": False,
        "inter_supervision": None,
        "loss": {"nll_weight": 1.0, "nll_balancing": 0.5, "inter_supervision": [0.3, 0.6]},
        "precision": "bf16",
    }
    required_data_keys = ["view0", "view1", "keypoints0", "keypoints1", "descriptors0", "descriptors1",
                          "keypoint_scores0", "keypoint_scores1", "lines0", "lines1", "lines_junc_idx0",
                          "lines_junc_idx1", "line_scores0", "line_scores1"]

    def __init__(self, conf=None):
        super().__init__()
        self.conf = conf = _Conf(_merge(self.default_conf, _to_plain(conf)))
        assert conf.precision in ("bf16", "fp32"), conf.precision
        if conf.line_attention or conf.skip_init:
            raise NotImplementedError("gluefactory_b200 gluestick: line_attention / skip_init are not built")
        if conf.inter_supervision is not None:
            self._check_inter_supervision(conf)
        D = conf.descriptor_dim
        if D not in (128, 256):  # 4 heads of 32 or 64 channels: the head dims the attention kernels are built for
            raise NotImplementedError(f"gluefactory_b200 gluestick: descriptor_dim {D} is not supported (128 or 256)")
        if conf.input_dim != D:
            self.input_proj = nn.Conv1d(conf.input_dim, D, kernel_size=1)
            nn.init.constant_(self.input_proj.bias, 0.0)
        # registration order = the reference's (gluestick.py:69-113): state_dict keys come out identical
        bin_score = nn.Parameter(torch.tensor(1.0))
        line_bin_score = nn.Parameter(torch.tensor(1.0))
        self.kenc = KeypointEncoder(D, conf.keypoint_encoder)
        self.lenc = EndPtEncoder(D, conf.keypoint_encoder)
        self.gnn = AttentionalGNN(D, list(conf.GNN_layers))
        self.final_proj = nn.Conv1d(D, D, kernel_size=1)
        nn.init.constant_(self.final_proj.bias, 0.0)
        nn.init.orthogonal_(self.final_proj.weight, gain=1)
        self.final_line_proj = nn.Conv1d(D, D, kernel_size=1)
        nn.init.constant_(self.final_line_proj.bias, 0.0)
        nn.init.orthogonal_(self.final_line_proj.weight, gain=1)
        if conf.inter_supervision is not None:
            self.inter_line_proj = nn.ModuleList([nn.Conv1d(D, D, kernel_size=1) for _ in conf.inter_supervision])
            self.layer2idx = {}
            for i, block in enumerate(conf.inter_supervision):
                nn.init.constant_(self.inter_line_proj[i].bias, 0.0)
                nn.init.orthogonal_(self.inter_line_proj[i].weight, gain=1)
                self.layer2idx[block] = i
        self.register_parameter("bin_score", bin_score)
        self.register_parameter("line_bin_score", line_bin_score)
        if conf.weights:
            # a path, else the file the reference's download writes to (gluestick.py:114-130); never downloaded here
            root = _weights.data_path()
            cand = [root / "weights" / f"{conf.weights}_{conf.version}.tar"] if root is not None else []
            sd = _weights.load_weights(conf.weights, cand, "gluestick")
            if "model" in sd:  # full glue-factory checkpoint (gluestick.py:131-139)
                sd = {k.replace("matcher.", "").replace("module.", ""): v for k, v in sd["model"].items() if "matcher." in k}
            self.load_state_dict(sd, strict=False)
        self._register_head_perm(D)

    @staticmethod
    def _check_inter_supervision(conf):
        """The reference takes the features of block l after the cross layer i with i // 2 == l, and weighs that head
        with loss.inter_supervision[position of l]; anything else would fail mid-forward there (KeyError / IndexError)."""
        blocks = {i // 2 for i, t in enumerate(conf.GNN_layers) if t == "cross"}
        for block in conf.inter_supervision:
            if isinstance(block, bool) or block not in blocks:
                raise ValueError(f"gluefactory_b200 gluestick: inter_supervision entry {block!r} is not the block index "
                                 f"(i // 2) of a cross layer i in GNN_layers; valid: {sorted(blocks)}")
        weights = conf.loss.get("inter_supervision") or []
        if len(weights) < len(conf.inter_supervision):
            raise ValueError(f"gluefactory_b200 gluestick: loss.inter_supervision {list(weights)} has fewer weights than "
                             f"inter_supervision {list(conf.inter_supervision)} has entries")

    def _line_layer(self, x, enc, lay, layer):
        """LineLayer (gluestick.py:589-691, line_attention = False) over the endpoints of a JunctionLayout `lay` into the
        token rows x [T, D]: each endpoint's update from [its junction ; the other end's junction ; its encoding enc],
        then every junction's row gets the mean of its endpoints' updates, summed in the layout's fixed order."""
        upd = self._mlp(torch.cat([ops.JunctionGather.apply(x, lay.tgt, lay.order, lay.tgt_sorted), enc], 1), layer.mlp)
        return ops.JunctionMean.apply(x, upd, lay.tgt, lay.order, lay.tgt_sorted)

    def _matches(self, scores):
        """_get_matches (gluestick.py:318-331) on the filter kernel."""
        inner = scores[:, :-1, :-1]
        mx0, mx1 = inner.max(2), inner.max(1)
        return ops.filter_matches(mx0.values.contiguous(), mx0.indices.to(torch.int32).contiguous(),
                                  mx1.indices.to(torch.int32).contiguous(), self.conf.filter_threshold)

    # ------------------------------------------------------------------------------------------ forward / loss
    def forward(self, data):
        with torch.autocast(device_type="cuda", enabled=False):
            return self._forward(data)

    def _forward(self, data):
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        kp0, kp1 = data["keypoints0"], data["keypoints1"]
        B, n0 = kp0.shape[:2]
        n1 = kp1.shape[1]
        L0, L1 = data["lines0"].shape[1], data["lines1"].shape[1]
        counts = self._counts(data, B, n0, n1, L0, L1)
        if counts is not None:
            return self._forward_packed(data, *counts)
        if n0 == 0 or n1 == 0:  # nothing to match: no computation
            return _empty_pred(B, n0, n1, L0, L1, kp0.device)
        _lib.load()  # raises unless the CUDA library is built and the device is an H100 (no CPU fallback)
        kp0, kp1 = kp0.float(), kp1.float()
        size0, size1 = _image_size(data["view0"], kp0), _image_size(data["view1"], kp1)
        D = self.conf.descriptor_dim
        d0 = data["descriptors0"].float().reshape(B * n0, -1)
        d1 = data["descriptors1"].float().reshape(B * n1, -1)
        if self.conf.input_dim != D:
            d0, d1 = self._conv(d0, self.input_proj), self._conv(d1, self.input_proj)
        enc_in = lambda k, s: torch.cat([k, s.float()[..., None]], -1).reshape(-1, 3)  # noqa: E731
        d0 = d0 + self._mlp(enc_in(self._norm_kpts(kp0, size0), data["keypoint_scores0"]), self.kenc.encoder)
        d1 = d1 + self._mlp(enc_in(self._norm_kpts(kp1, size1), data["keypoint_scores1"]), self.kenc.encoder)

        def line_enc(lines, scores, size):
            Ln = lines.shape[1]
            ln = self._norm_kpts(lines.float().reshape(B, 2 * Ln, 2), size).reshape(B, Ln, 2, 2)
            off = ln[:, :, 1] - ln[:, :, 0]
            off = torch.stack([off, -off], 2).reshape(B, 2 * Ln, 2)
            # the reference tiles the line scores over the interleaved endpoints (`scores.repeat(1, 2)`, gluestick.py:520)
            inp = torch.cat([ln.reshape(B, 2 * Ln, 2), off, scores.float().repeat(1, 2)[..., None]], -1)
            return self._mlp(inp.reshape(-1, 5), self.lenc.encoder)

        # a view without lines: no line encoding, LineLayer or line head runs, intermediate ones included
        # (gluestick.py:213-240, 257-312, 734-740)
        lines = L0 > 0 and L1 > 0
        if lines:
            enc0 = line_enc(data["lines0"], data["line_scores0"], size0)
            enc1 = line_enc(data["lines1"], data["line_scores1"], size1)
            idx0, idx1 = data["lines_junc_idx0"].reshape(B, -1), data["lines_junc_idx1"].reshape(B, -1)
            lay0 = junction_layout(idx0, n0, min(n0, 2 * L0))
            lay1 = junction_layout(idx1, n1, min(n1, 2 * L1))
        inter = {}  # block -> both images' features after its cross layer (gluestick.py:762-768)
        for i, layer in enumerate(self.gnn.layers):
            d0, d1 = self._gnn_layer(d0, d1, layer.update, layer.type == "cross", B)
            if layer.type == "self" and lines:
                for _ in range(self.conf.num_line_iterations):
                    line_layer = self.gnn.line_layers[i // 2]
                    d0, d1 = self._line_layer(d0, enc0, lay0, line_layer), self._line_layer(d1, enc1, lay1, line_layer)
            if (lines and self.conf.inter_supervision and layer.type == "cross"
                    and i // 2 in self.conf.inter_supervision):
                inter[i // 2] = (d0, d1)
        # points (keypoints and line junctions together)
        scores = ops.log_double_softmax(self._similarity(self._conv(d0, self.final_proj), self._conv(d1, self.final_proj), B),
                                        self.bin_score)
        m0, m1, ms0, ms1 = self._matches(scores.detach())
        pred = {"log_assignment": scores, "matches0": m0, "matches1": m1, "matching_scores0": ms0, "matching_scores1": ms1}
        if not lines:
            pred.update(_no_line_outputs(B, L0, L1, kp0.device), raw_line_scores=kp0.new_zeros(B, L0, L1))
            return pred
        lscores, lm0, lm1, lms0, lms1, raw = self._line_head(d0, d1, lay0, lay1, L0, L1, self.final_line_proj, B)
        pred.update({"line_log_assignment": lscores, "line_matches0": lm0, "line_matches1": lm1,
                     "line_matching_scores0": lms0, "line_matching_scores1": lms1, "raw_line_scores": raw})
        for block in self.conf.inter_supervision or []:
            proj = self.inter_line_proj[self.layer2idx[block]]
            la, lm0, lm1, lms0, lms1, _ = self._line_head(*inter[block], lay0, lay1, L0, L1, proj, B)
            pred.update({f"line_{block}_log_assignment": la, f"line_{block}_matches0": lm0,
                         f"line_{block}_matches1": lm1, f"line_{block}_matching_scores0": lms0,
                         f"line_{block}_matching_scores1": lms1})
        return pred

    def _line_head(self, d0, d1, lay0, lay1, L0, L1, proj, B):
        """_get_line_matches (gluestick.py:336-376) with the projection `proj`: junction similarity, best of the two
        endpoint orderings per line pair (ops.LineScores, from the JunctionLayouts lay0 / lay1), log_double_softmax with
        the line bin score, match filtering.
        Returns (log-assignment, matches0, matches1, matching_scores0, matching_scores1, raw line scores)."""
        D = d0.shape[1]
        ld0 = d0.view(B, -1, D)[:, :2 * L0].reshape(-1, D)
        ld1 = d1.view(B, -1, D)[:, :2 * L1].reshape(-1, D)
        s = self._similarity(self._conv(ld0, proj), self._conv(ld1, proj), B)
        full = lambda n: torch.full((B,), n, dtype=torch.int32, device=s.device)  # noqa: E731
        raw = ops.LineScores.apply(s.contiguous(), lay0.junc, lay1.junc, torch.stack([full(L0), full(L1)]), lay0.order,
                                   lay0.ptr, lay1.order, lay1.ptr)
        lscores = ops.log_double_softmax(raw, self.line_bin_score)
        return (lscores, *self._matches(lscores.detach()), raw)

    # ------------------------------------------------------------------------------------------ packed batches
    def _counts(self, data, B, M, N, L0, L1):
        """The optional per-pair counts num_keypoints0/1 (1 .. padded length) and num_lines0/1 (0 .. padded length) as
        int64 CPU tensors (n0, n1, l0, l1), a missing key meaning every row of that view; None without any of them."""
        kc = keypoint_counts(data, B, M, N, owner="GlueStick")
        lc = keypoint_counts(data, B, L0, L1, keys=("num_lines0", "num_lines1"), low=0, owner="GlueStick")
        if kc is None and lc is None:
            return None
        if self.training:
            raise ValueError("GlueStick: num_keypoints0/1 and num_lines0/1 are taken in eval mode only (BatchNorm "
                             "normalises training batches with their own statistics, padding included)")
        full = lambda n: torch.full((B,), n, dtype=torch.int64)  # noqa: E731
        kc = kc if kc is not None else (full(M), full(N))
        lc = lc if lc is not None else (full(L0), full(L1))
        return (*kc, *lc)

    @torch.no_grad()
    def _forward_packed(self, data, n0, n1, l0, l1):
        """Eval forward over B pairs with their own counts: pair b uses the first n0_b / n1_b keypoints and l0_b / l1_b
        lines of the padded views, and gets what a one-pair call on those truncated inputs returns, in the padded
        original indexing (see README, "Batches of pairs of different sizes").  The valid rows are gathered once into
        the packed token layout [view 0 of every pair; view 1 of every pair] (lightglue.ragged_layout); the encoders,
        GEMMs and BatchNorms run token-wise over it, attention is length-aware (_attention_packed), the LineLayer runs
        once over the endpoints of every lined pair and both views (eval-mode BatchNorm), and the heads run once over
        per-pair zero-padded operands on the varlen kernels.  The padding is never read."""
        _lib.load()  # raises unless the CUDA library is built and the device is an H100 (no CPU fallback)
        kp0, kp1 = data["keypoints0"], data["keypoints1"]
        (B, M), N = kp0.shape[:2], kp1.shape[1]
        Lp0, Lp1 = data["lines0"].shape[1], data["lines1"].shape[1]
        dev, D = kp0.device, self.conf.descriptor_dim
        layout = ragged_layout(n0, n1, M, N)
        src0, src1, pid0, pid1 = (t.to(dev) for t in (layout.src0, layout.src1, layout.pid0, layout.pid1))
        pick = lambda t, n, src: t.reshape(B * n, *t.shape[2:]).index_select(0, src)  # noqa: E731
        size0 = _image_size(data["view0"], kp0).to(dev).expand(B, 2)
        size1 = _image_size(data["view1"], kp1).to(dev).expand(B, 2)
        x = torch.cat([pick(data["descriptors0"], M, src0), pick(data["descriptors1"], N, src1)], 0).float()
        if self.conf.input_dim != D:
            x = self._conv(x, self.input_proj)
        k = torch.cat([_norm_kpts_packed(pick(kp0.float(), M, src0), size0, pid0),
                       _norm_kpts_packed(pick(kp1.float(), N, src1), size1, pid1)], 0)
        s = torch.cat([pick(data["keypoint_scores0"], M, src0), pick(data["keypoint_scores1"], N, src1)], 0).float()
        x = x + self._mlp(torch.cat([k, s[:, None]], -1), self.kenc.encoder, rowwise=True)

        # a pair with no lines in either view runs no LineLayer and no line head (gluestick.py:213-240, 257-317)
        lined = (l0 > 0) & (l1 > 0)
        tok_off = layout.seg[0].long().view(B, 2)
        views = [endpoint_layout(l, n, Lp, lined) for l, n, Lp in ((l0, n0, Lp0), (l1, n1, Lp1))]
        lines = bool(lined.any())
        if lines:
            enc, tgt, bad = [], [], []
            for v, (lay, size) in enumerate(zip(views, (size0, size1))):
                lsrc, lpid, esrc, epid, ssrc, bound = (t.to(dev) for t in lay)
                enc.append(_endpoint_inputs(data[f"lines{v}"], data[f"line_scores{v}"], size, lsrc, lpid, ssrc))
                junc = data[f"lines_junc_idx{v}"].reshape(-1).index_select(0, esrc).long()
                bad.append(((junc < 0) | (junc >= bound)).any())
                tgt.append(tok_off[:, v].to(dev)[epid] + junc)
            if bool(torch.stack(bad).any()):  # the junction check's one host read
                raise ValueError("GlueStick: lines_junc_idx0/1 of pair b's first num_lines lines must lie in "
                                 "0 .. min(num_keypoints, 2 * num_lines) - 1")
            enc = self._mlp(torch.cat(enc, 0), self.lenc.encoder, rowwise=True)
            tgt = torch.cat(tgt).int()
            lay = JunctionLayout(tgt, *junction_order(tgt), None, None)
        seg, max_len = layout.seg.to(dev), int(max(n0.max(), n1.max()))
        inter = {}
        for i, layer in enumerate(self.gnn.layers):
            x = self._gnn_layer_packed(x, layer.update, layer.type == "cross", seg, max_len)
            if layer.type == "self" and lines:
                for _ in range(self.conf.num_line_iterations):
                    x = self._line_layer(x, enc, lay, self.gnn.line_layers[i // 2])
            if (lines and self.conf.inter_supervision and layer.type == "cross"
                    and i // 2 in self.conf.inter_supervision):
                inter[i // 2] = x
        # points (keypoints and line junctions together)
        out = _padded_outputs(B, M, N, dev)
        md = self._conv(x, self.final_proj)
        T0 = src0.numel()
        sim = self._padded_similarity(md[:T0], md[T0:], pid0, layout.src0 % M, pid1, layout.src1 % N, B,
                                      int(n0.max()), int(n1.max()))
        pairs = torch.stack([n0, n1, torch.arange(B)]).to(dev, torch.int32)
        ops.log_double_softmax_varlen(sim, self.bin_score, pairs, self.conf.filter_threshold, out)
        pred = {"log_assignment": out["scores"], "matches0": out["m0"], "matches1": out["m1"],
                "matching_scores0": out["ms0"], "matching_scores1": out["ms1"], "_b200_packed": True}
        lh = _line_head_layout(data, lined, n0, n1, l0, l1, layout, dev) if lines else None
        heads = [("line_", self.final_line_proj, x)]
        heads += [(f"line_{blk}_", self.inter_line_proj[self.layer2idx[blk]], inter.get(blk))
                  for blk in self.conf.inter_supervision or []]
        for prefix, proj, xf in heads:
            lo = _padded_outputs(B, Lp0, Lp1, dev)
            raw = kp0.new_zeros(B, Lp0, Lp1, dtype=torch.float32)
            if lines:
                raw_g = self._line_head_packed(xf, proj, lh, lo)
                raw[lh["bs"], :raw_g.shape[1], :raw_g.shape[2]] = raw_g
            pred.update({prefix + "log_assignment": lo["scores"], prefix + "matches0": lo["m0"],
                         prefix + "matches1": lo["m1"], prefix + "matching_scores0": lo["ms0"],
                         prefix + "matching_scores1": lo["ms1"]})
            if prefix == "line_":
                pred["raw_line_scores"] = raw
        return pred

    def _line_head_packed(self, x, proj, lh, out):
        """_line_head of every lined pair at once: projection of each pair's first min(n, 2 L) tokens, one padded
        similarity, the raw line scores straight from it (ops.line_scores_varlen) and the varlen log_double_softmax +
        match filter into `out`.  Returns the raw scores [G, Lg0, Lg1] of the lined pairs."""
        md = self._conv(x.index_select(0, lh["rows"]), proj)
        T0 = lh["k0"].numel()
        s = self._padded_similarity(md[:T0], md[T0:], lh["k0"], lh["i0"], lh["k1"], lh["i1"], lh["G"], lh["P0"],
                                    lh["P1"])
        raw = ops.line_scores_varlen(s, lh["junc0"], lh["junc1"], lh["pairs"], lh["Lg0"], lh["Lg1"])
        ops.log_double_softmax_varlen(raw, self.line_bin_score, lh["pairs"], self.conf.filter_threshold, out)
        return raw

    def _sub_loss(self, pred, data, losses, bin_score, prefix, block=None):
        """gluestick.py:379-415; `block`: an intermediate line head (pred keys line_{block}_*, ground truth gt_line_*),
        weighted by its loss.inter_supervision entry and without the statistics entries."""
        suffix = "" if block is None else f"{block}_"
        la = pred[prefix + suffix + "log_assignment"]
        positive = data.get("gt_" + prefix + "assignment")
        if positive is None:  # labels as one-to-one match lists: one gathered entry per row
            pos_sum, num_pos = _list_positive_sum(la, data["gt_" + prefix + "matches0"],
                                                  data["gt_" + prefix + "matches1"])
        else:
            positive = positive.float()
            num_pos = positive.sum((1, 2)).clamp(min=1.0)
            pos_sum = (la[:, :-1, :-1] * positive).sum((1, 2))
        neg0 = (data["gt_" + prefix + "matches0"] == -1).float()
        neg1 = (data["gt_" + prefix + "matches1"] == -1).float()
        num_neg = (neg0.sum(1) + neg1.sum(1)).clamp(min=1.0)
        nll_pos = -pos_sum / num_pos
        nll_neg = (-(la[:, :-1, -1] * neg0).sum(1) - (la[:, -1, :-1] * neg1).sum(1)) / num_neg
        bal = self.conf.loss.nll_balancing
        nll = bal * nll_pos + (1 - bal) * nll_neg
        losses[prefix + suffix + "assignment_nll"] = nll
        if self.conf.loss.nll_weight > 0:
            term = nll * self.conf.loss.nll_weight
            if block is not None:
                term = term * self.conf.loss.inter_supervision[self.layer2idx[block]]
            losses["total"] = losses["total"] + term
        if block is None:
            losses[prefix + "num_matchable"] = num_pos
            losses[prefix + "num_unmatchable"] = num_neg
            losses[prefix + "sinkhorn_norm"] = la.exp()[:, :-1].sum(2).mean(1)
            losses[prefix + "bin_score"] = bin_score[None]
        return losses

    def loss(self, pred, data):
        """gluestick.py:417-462."""
        if pred.get("_b200_packed"):
            raise ValueError("GlueStick.loss cannot be taken on the pred of a forward with num_keypoints0/1 or "
                             "num_lines0/1: each pair was truncated on its own")
        if data["lines0"].shape[1] == 0 or data["lines1"].shape[1] == 0:
            raise ValueError("gluefactory_b200 gluestick: the line loss needs lines in both views (lines0 has "
                             f"{data['lines0'].shape[1]}, lines1 {data['lines1'].shape[1]})")
        with torch.autocast(device_type="cuda", enabled=False):
            losses = {"total": 0}
            losses = self._sub_loss(pred, data, losses, self.bin_score, "")
            losses = self._sub_loss(pred, data, losses, self.line_bin_score, "line_")
            for block in self.conf.inter_supervision or []:
                losses = self._sub_loss(pred, data, losses, self.line_bin_score, "line_", block)
            metrics = {}
            if not self.training:
                metrics = {**matcher_metrics(pred, data), **_line_metrics(pred, data, "line_")}
                for block in self.conf.inter_supervision or []:
                    metrics.update(_line_metrics(pred, data, f"line_{block}_"))
            return losses, metrics


def _list_positive_sum(la, gt0, gt1):
    """(sum_i la[b, i, gt0[b, i]] over the rows with gt0 >= 0, num_pos) for one-to-one match lists gt0 [B, M] /
    gt1 [B, N]: the positive part of gluestick.py:389-393 without the [B, M, N] mask, by torch gathers (the gather's
    backward writes one entry per row: no index repeats).  NaN for a pair whose lists disagree."""
    gt0, gt1 = gt0.long(), gt1.long()
    M, N = gt0.shape[1], gt1.shape[1]
    _, _, num_pos = ops.match_list_counts(gt0, gt1)
    pos = gt0 >= 0
    j = gt0.clamp(0, N - 1)
    bad = pos & ((gt0 >= N) | (gt1.gather(1, j) != torch.arange(M, device=gt0.device)))
    v = la[:, :-1, :-1].gather(2, j[..., None])[..., 0]
    s = torch.where(pos, v, torch.zeros_like(v)).sum(1)
    return torch.where(bad.any(1), torch.full_like(s, float("nan")), s), num_pos


def _image_size(view, kpts):
    """view["image_size"] as given, or (w, h) from view["image"].shape[-2:] when a view has none
    (gluestick.py:146-156, normalize_keypoints :477-482)."""
    if "image_size" in view:
        return view["image_size"]
    h, w = view["image"].shape[-2:]
    return kpts.new_tensor([[w, h]])


def endpoint_layout(nl, nk, Lp, lined):
    """The line endpoints of one view over B pairs (CPU int64 tensors; nl / nk: each pair's line / keypoint counts, Lp
    the padded line count, lined: the pairs whose line layers run).  Lines of lined pairs in pair order, endpoints
    2 l, 2 l + 1 of line l in line order.  Returns
      lsrc, lpid: each line's row of the flattened [B * Lp] lines and its pair;
      esrc, epid: each endpoint's entry of the flattened [B * 2 Lp] junction indices and its pair;
      ssrc: the row of the flattened [B * Lp] line scores each endpoint takes: line e % nl of its pair for endpoint e,
            as the reference tiles the scores over the interleaved endpoints (`scores.repeat(1, 2)`, gluestick.py:520);
      bound: each endpoint's junction-index bound min(nk, 2 nl) (the rows the line head's gathers see)."""
    B = nl.numel()
    n = torch.where(lined, nl, torch.zeros_like(nl))
    lsrc, lpid, li = segment_rows(torch.arange(B) * Lp, n)
    e = (2 * li[:, None] + torch.arange(2)).reshape(-1)
    epid = lpid.repeat_interleave(2)
    esrc = epid * 2 * Lp + e
    ssrc = epid * Lp + e % n[epid].clamp(min=1)
    bound = torch.minimum(nk, 2 * nl)[epid]
    return lsrc, lpid, esrc, epid, ssrc, bound


def junction_order(tgt):
    """The endpoints sorted stably by their target token rows tgt [E] int32: (order, tgt_sorted), both int32.  Built once
    per forward; every LineLayer sums each junction's endpoints in this order."""
    tgt_sorted, order = torch.sort(tgt, stable=True)
    return order.int(), tgt_sorted.int()


class JunctionLayout(NamedTuple):
    """The line endpoints of one forward and the junction rows they read and update, built once per forward.
    tgt [E] int32: each endpoint's token row (endpoints 2 l, 2 l + 1 of line l); order / tgt_sorted: junction_order(tgt).
    Uniform batches (junction_layout) also carry the line heads' operands: junc [B, 2 L] int32 the junction indices,
    ptr [B, P + 1] int32 the endpoints at junction r < P of pair b, order[ptr[b, r] .. ptr[b, r + 1])."""
    tgt: torch.Tensor
    order: torch.Tensor
    tgt_sorted: torch.Tensor
    junc: Optional[torch.Tensor]
    ptr: Optional[torch.Tensor]


def junction_layout(idx, n, P):
    """JunctionLayout of one view of a uniform batch: idx [B, 2 L] the junction indices (lines_junc_idx), n the nodes
    per pair (token row of pair b's junction j: b * n + j), P the rows of the line heads' similarity (min(n, 2 L)).
    No host read: it is built inside a captured training step."""
    B = idx.shape[0]
    junc = idx.int().contiguous()
    base = torch.arange(B, device=idx.device, dtype=torch.int32)[:, None] * n
    tgt = (junc + base).reshape(-1)
    order, tgt_sorted = junction_order(tgt)
    rows = (base + torch.arange(P + 1, device=idx.device, dtype=torch.int32)).reshape(-1)
    ptr = torch.searchsorted(tgt_sorted, rows, out_int32=True).view(B, P + 1)
    return JunctionLayout(tgt, order, tgt_sorted, junc, ptr)


def _endpoint_inputs(lines, scores, size, lsrc, lpid, ssrc):
    """The endpoint encoder's input [2 nl, 5] of the packed lines (gluestick.py:512-521, as GlueStick._forward's
    line_enc): normalised endpoint, offset to the other end (negated for the second), tiled line score."""
    ln = lines.float().reshape(-1, 2, 2).index_select(0, lsrc)
    ln = _norm_kpts_packed(ln.reshape(-1, 2), size, lpid.repeat_interleave(2)).reshape(-1, 2, 2)
    off = ln[:, 1] - ln[:, 0]
    off = torch.stack([off, -off], 1).reshape(-1, 2)
    sc = scores.reshape(-1).index_select(0, ssrc).float()
    return torch.cat([ln.reshape(-1, 2), off, sc[:, None]], -1)


def _line_head_layout(data, lined, n0, n1, l0, l1, layout, dev):
    """The packed line heads' operands, shared by the final and the intermediate heads: the lined pairs bs, the token
    rows of each one's first min(n, 2 L) tokens per view (with their pair k and index i in the group), the junction
    indices [G, 2 Lg] and pairs [3, G] = (l0, l1, batch row)."""
    bs = lined.nonzero()[:, 0]
    tok_off = layout.seg[0].long().view(-1, 2)[bs]
    lh = {"bs": bs.to(dev), "G": bs.numel()}
    rows = []
    for v, (nk, nl) in enumerate(((n0, l0), (n1, l1))):
        p = torch.minimum(nk, 2 * nl)[bs]
        r, k, i = segment_rows(tok_off[:, v], p)
        rows.append(r)
        Lg = int(nl[bs].max())
        lh.update({f"k{v}": k.to(dev), f"i{v}": i.to(dev), f"P{v}": int(p.max()), f"Lg{v}": Lg,
                   f"junc{v}": data[f"lines_junc_idx{v}"].reshape(len(nk), -1)[bs.to(dev), :2 * Lg].int().contiguous()})
    lh["rows"] = torch.cat(rows).to(dev)
    lh["pairs"] = torch.stack([l0[bs], l1[bs], bs]).to(dev, torch.int32)
    return lh


def _no_line_outputs(B, L0, L1, device):
    """The line head's outputs for a view without lines (gluestick.py:293-308)."""
    return {"line_log_assignment": torch.zeros(B, L0, L1, dtype=torch.float, device=device),
            "line_matches0": torch.full((B, L0), -1, device=device, dtype=torch.int64),
            "line_matches1": torch.full((B, L1), -1, device=device, dtype=torch.int64),
            "line_matching_scores0": torch.zeros((B, L0), device=device, dtype=torch.float32),
            "line_matching_scores1": torch.zeros((B, L1), device=device, dtype=torch.float32)}


def _empty_pred(B, n0, n1, L0, L1, device):
    """The reference's pred for a view without keypoints (gluestick.py:163-195), key for key.  As there,
    log_assignment is [B, M, N] (no bin row / column) and line_matching_scores1 is [B, N]."""
    pred = {"log_assignment": torch.zeros(B, n0, n1, dtype=torch.float, device=device),
            "matches0": torch.full((B, n0), -1, device=device, dtype=torch.int64),
            "matches1": torch.full((B, n1), -1, device=device, dtype=torch.int64),
            "matching_scores0": torch.zeros((B, n0), device=device, dtype=torch.float32),
            "matching_scores1": torch.zeros((B, n1), device=device, dtype=torch.float32)}
    pred.update(_no_line_outputs(B, L0, L1, device))
    pred["line_matching_scores1"] = torch.zeros((B, n1), device=device, dtype=torch.float32)
    return pred


def _line_metrics(pred, data, prefix):
    """matcher_metrics(pred, data, prefix, prefix_gt="line_") (models/utils/metrics.py:4-50) of a line head."""
    m = matcher_metrics({"matches0": pred[prefix + "matches0"], "matching_scores0": pred[prefix + "matching_scores0"]},
                        {"gt_matches0": data["gt_line_matches0"]})
    return {prefix + k: v for k, v in m.items()}


__main_model__ = GlueStick
