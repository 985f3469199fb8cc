"""H100-native LightGlue matcher -- drop-in for gluefactory's in-tree matcher.

Select it from a glue-factory config with

    model:
      matcher:
        name: gluefactory_b200.matchers.lightglue     # instead of matchers.lightglue

`get_model` (reference gluefactory/models/__init__.py:7-30) imports this module,
finds no BaseModel subclass and returns `__main_model__`, exactly as it does for
the reference matcher (gluefactory/models/matchers/lightglue.py:312, 630).

Same constructor (`cls(conf_dict)`), same `forward(data) -> pred`, same
`loss(pred, data) -> (losses, metrics)`, same parameter names (state_dict /
checkpoints are interchangeable, SURVEY.md Appendix B.2).  Each transformer
layer is one hand-scheduled autograd node (engine.LayerFn) and each
deep-supervision head of the loss another (engine.HeadFn).  The arithmetic of
the N x N path -- rotary split, self / cross attention, LayerNorm+GELU, the
assignment head, its NLL terms, argmax and match filtering, and all of their
backward passes -- runs in the hand-written sm_90a kernels behind the C ABI
of include/lgb200.h.  There is no CPU path: without the built library and an
H100 `forward` raises.  `loss` takes only the pred of this module's own
`forward`, which carries the per-layer states it needs.  `weights` is a path
or a pretrained name (superpoint, disk, ...) looked up where the reference
looks, DATA_PATH then torch-hub's cache, and never downloaded
(matchers/_weights.py).

conf additions over the reference's default_conf:
    precision: "bf16" -> bf16 operands / fp32 accumulation on the Hopper tensor cores (default)
               "fp32" -> full-precision parity path (CUDA cores + fp32 cuBLAS)
"""
import copy
import math

import torch
import torch.nn.functional as F
from torch import nn

from .. import _lib, engine, ops
from . import _weights


class _Conf(dict):
    """Attribute-access view of a (nested) plain dict (stands in for OmegaConf's DictConfig)."""

    def __getattr__(self, k):
        try:
            v = self[k]
        except KeyError as e:
            raise AttributeError(k) from e
        return _Conf(v) if isinstance(v, dict) and not isinstance(v, _Conf) else v


def _to_plain(conf):
    if conf is None:
        return {}
    try:  # OmegaConf DictConfig, when the host framework passes one
        from omegaconf import OmegaConf  # type: ignore

        if OmegaConf.is_config(conf):
            return OmegaConf.to_container(conf, resolve=True)
    except Exception:
        pass
    return {k: (_to_plain(v) if isinstance(v, dict) else v) for k, v in dict(conf).items()}


def _merge(base, new):
    out = copy.deepcopy(base)
    for k, v in new.items():
        if isinstance(v, dict) and isinstance(out.get(k), dict):
            out[k] = _merge(out[k], v)
        else:
            out[k] = copy.deepcopy(v)
    return out


def normalize_keypoints(kpts, size):
    """lightglue.py:27-39 (always fp32, like the reference's custom_fwd cast)."""
    kpts = kpts.float()
    if size is None:
        size = 1 + kpts.max(-2).values - kpts.min(-2).values
    elif not isinstance(size, torch.Tensor):
        size = torch.tensor(size, device=kpts.device, dtype=kpts.dtype)
    size = size.to(kpts)
    shift = size / 2
    scale = size.max(-1).values / 2
    return (kpts - shift[..., None, :]) / scale[..., None, None]


# ---- parameter containers: same module tree / names as the reference (lightglue.py:52-65, 131-148,
# ---- 166-183, 271-276, 68-72).  They only hold parameters; the math lives in LightGlue below.
class LearnableFourierPositionalEncoding(nn.Module):
    def __init__(self, M, dim, F_dim=None, gamma=1.0):
        super().__init__()
        F_dim = F_dim if F_dim is not None else dim
        self.Wr = nn.Linear(M, F_dim // 2, bias=False)
        nn.init.normal_(self.Wr.weight.data, mean=0, std=gamma**-2)


def _ffn(d):
    return nn.Sequential(nn.Linear(2 * d, 2 * d), nn.LayerNorm(2 * d, elementwise_affine=True), nn.GELU(),
                         nn.Linear(2 * d, d))


class SelfBlock(nn.Module):
    def __init__(self, d, h):
        super().__init__()
        self.Wqkv = nn.Linear(d, 3 * d)
        self.out_proj = nn.Linear(d, d)
        self.ffn = _ffn(d)


class CrossBlock(nn.Module):
    def __init__(self, d, h):
        super().__init__()
        self.to_qk = nn.Linear(d, d)
        self.to_v = nn.Linear(d, d)
        self.to_out = nn.Linear(d, d)
        self.ffn = _ffn(d)


class TransformerLayer(nn.Module):
    def __init__(self, d, h):
        super().__init__()
        self.self_attn = SelfBlock(d, h)
        self.cross_attn = CrossBlock(d, h)


class MatchAssignment(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.matchability = nn.Linear(d, 1)
        self.final_proj = nn.Linear(d, d)


class TokenConfidence(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.token = nn.Sequential(nn.Linear(d, 1), nn.Sigmoid())


class LightGlue(nn.Module):
    default_conf = {
        "name": "lightglue",
        "input_dim": 256,
        "add_scale_ori": False,
        "descriptor_dim": 256,
        "n_layers": 9,
        "num_heads": 4,
        "flash": False,  # accepted for config compatibility; attention is always the fused kernel
        "mp": False,
        "depth_confidence": -1,  # > 0: early stopping at inference (eval mode, one pair; _forward_adaptive)
        "width_confidence": -1,  # > 0: point pruning at inference
        "filter_threshold": 0.0,
        "checkpointed": False,  # accepted; the fused attention keeps no N x N activations to checkpoint
        "weights": None,
        "weights_from_version": "v0.1_arxiv",
        "loss": {"gamma": 1.0, "fn": "nll", "nll_balancing": 0.5},
        "precision": "bf16",
        # pred["ref_descriptors{0,1}"] = per-layer states stacked [B, L, N, D] (lightglue.py:540-541).  The matcher's
        # own loss reads the un-stacked layer outputs instead, so "auto" skips the two 0.6 GB stacks while training.
        # True: always stack.
        "stack_ref_descriptors": "auto",
    }
    required_data_keys = ["keypoints0", "keypoints1", "descriptors0", "descriptors1"]

    def __init__(self, conf=None):
        super().__init__()
        self.conf = conf = _Conf(_merge(self.default_conf, _to_plain(conf)))
        assert conf.precision in ("bf16", "fp32"), conf.precision
        d, h, n = conf.descriptor_dim, conf.num_heads, conf.n_layers
        # head_dim = descriptor_dim // num_heads (lightglue.py:347): 64 (256 / 4, the default) or 32 (128 / 4, 256 / 8)
        if d % h or d // h not in (32, 64):
            raise NotImplementedError(f"gluefactory_b200 lightglue: head_dim = descriptor_dim // num_heads must be 32 or "
                                      f"64, the head dims the kernels are built for (descriptor_dim {d}, num_heads {h})")
        hd = d // h
        self.input_proj = nn.Linear(conf.input_dim, d) if conf.input_dim != d else nn.Identity()
        # add_scale_ori (SIFT-style features, lightglue.py:347-349, 426-443): scale and orientation join (x, y) as inputs
        # of the learnt Fourier encoding, Wr becomes [hd/2, 4]; only the rotary ANGLES change, not the kernels
        self.posenc = LearnableFourierPositionalEncoding(2 + 2 * bool(conf.add_scale_ori), hd, hd)
        self.transformers = nn.ModuleList([TransformerLayer(d, h) for _ in range(n)])
        self.log_assignment = nn.ModuleList([MatchAssignment(d) for _ in range(n)])
        self.token_confidence = nn.ModuleList([TokenConfidence(d) for _ in range(n - 1)])
        self.register_buffer(
            "confidence_thresholds",
            torch.tensor([min(max(0.8 + 0.1 * math.exp(-4.0 * i / n), 0.0), 1.0) for i in range(n)]))
        if conf.weights is not None:
            state_dict = _weights.load_weights(conf.weights, self._weights_candidates(conf), "lightglue")
            for i in range(n):  # legacy names, lightglue.py:384-391
                state_dict = {k.replace(f"self_attn.{i}", f"transformers.{i}.self_attn"): v for k, v in state_dict.items()}
                state_dict = {k.replace(f"cross_attn.{i}", f"transformers.{i}.cross_attn"): v for k, v in state_dict.items()}
            self.load_state_dict(state_dict, strict=False)

    @staticmethod
    def _weights_candidates(conf):
        """Where the reference looks for `weights` when it is not a path (lightglue.py:365-382): DATA_PATH / weights
        (skipped without glue-factory), then torch-hub's cache file of the pretrained download."""
        root = _weights.data_path()
        hub = _weights.hub_checkpoint(f"{conf.weights}_{conf.weights_from_version}".replace(".", "-") + ".pth")
        return ([root / str(conf.weights)] if root is not None else []) + [hub]

    # ------------------------------------------------------------------------------------------
    @property
    def _bf16(self):
        return self.conf.precision == "bf16"

    @property
    def _cdt(self):
        return torch.bfloat16 if self._bf16 else torch.float32

    def _refresh_shadow(self):
        """Compute-dtype copies of the weights, refreshed once per forward.  With a flat parameter buffer
        (trainer.FlatParams) this is ONE cast kernel over the whole buffer; otherwise one cast per tensor."""
        if not self._bf16:
            self._shadow = {n: p.detach() for n, p in self.named_parameters()}
            return
        fp = getattr(self, "_b200_flat", None)
        if fp is not None:
            self._shadow = fp.shadow_bf16()
        else:
            self._shadow = {n: p.detach().to(torch.bfloat16) for n, p in self.named_parameters()}

    def _layer_weights(self, i):
        pre = f"transformers.{i}."
        w, params = [], []
        named = dict(self.transformers[i].named_parameters())
        for slot, name in enumerate(engine.LAYER_PARAMS):
            p = named[name]
            params.append(p)
            w.append(p.detach() if slot in engine._LN_SLOTS else self._shadow[pre + name])
        return w, params

    def _lin(self, x, layer):
        """nn.Linear: bf16 mode -> the library's wgmma GEMM (bf16 operands, fp32 accumulate, fp32 bias epilogue);
        fp32 parity mode -> fp32 cuBLAS."""
        if self._bf16:
            shp = x.shape
            y = ops.LinearFn.apply(x.reshape(-1, shp[-1]).to(torch.bfloat16).contiguous(), layer.weight, layer.bias)
            return y.view(*shp[:-1], y.shape[-1])
        return F.linear(x, layer.weight, layer.bias)

    def _head_inputs(self, d0, d1, i):
        """final_proj / matchability of layer i (lightglue.py:280-285)."""
        la = self.log_assignment[i]
        D = d0.shape[-1]
        md0 = self._lin(d0, la.final_proj).float() / D**0.25
        md1 = self._lin(d1, la.final_proj).float() / D**0.25
        z0 = F.linear(d0, la.matchability.weight, la.matchability.bias).squeeze(-1)
        z1 = F.linear(d1, la.matchability.weight, la.matchability.bias).squeeze(-1)
        return md0.contiguous(), md1.contiguous(), z0, z1

    # ------------------------------------------------------------------------------------------
    def forward(self, data):
        """lightglue.py:412-543.  The caller may be inside torch.autocast (train.py:468-472 `--mp bfloat16|float16`):
        the numeric mode here is chosen by conf.precision, not by the ambient autocast state, so the body runs with
        autocast disabled (fp32 keypoint normalisation / rotary angles / residual stream as in the reference's
        custom_fwd(cast_inputs=float32) regions, bf16 tensor-core operands inside the kernels) and every input is
        converted explicitly -- descriptors may arrive in fp16, cf. the `.half()` quirk of lightglue.py:451-453."""
        with torch.autocast(device_type="cuda", enabled=False):
            return self._forward(data)

    def _forward(self, data):
        for key in self.required_data_keys:
            assert key in data, f"Missing key {key} in data"
        _lib.load()  # raises unless the CUDA library is built and the device is an H100 (no CPU fallback)
        conf = self.conf
        adaptive = not self.training and (conf.depth_confidence > 0 or conf.width_confidence > 0)
        kpts0, kpts1 = data["keypoints0"], data["keypoints1"]
        B, M, _ = kpts0.shape
        N = kpts1.shape[1]
        assert M > 0 and N > 0, "empty keypoint sets are not supported"
        size0 = data["view0"].get("image_size") if "view0" in data else None
        size1 = data["view1"].get("image_size") if "view1" in data else None
        kpts0, kpts1 = normalize_keypoints(kpts0, size0), normalize_keypoints(kpts1, size1)
        desc0, desc1 = data["descriptors0"].contiguous(), data["descriptors1"].contiguous()
        assert desc0.shape[-1] == conf.input_dim and desc1.shape[-1] == conf.input_dim
        D = conf.descriptor_dim
        x = torch.cat([desc0.reshape(B * M, -1), desc1.reshape(B * N, -1)], 0).float()
        if not isinstance(self.input_proj, nn.Identity):
            x = self._lin(x, self.input_proj).float()
        # rotary angles, cached for all layers (lightglue.py:456-458); cos/sin are taken in-kernel
        if conf.add_scale_ori:
            ext = lambda k, sc, o: torch.cat([k, (sc if sc.dim() == 3 else sc[..., None]).float(),  # noqa: E731
                                              (o if o.dim() == 3 else o[..., None]).float()], -1)
            kpts0, kpts1 = ext(kpts0, data["scales0"], data["oris0"]), ext(kpts1, data["scales1"], data["oris1"])
        kd = kpts0.shape[-1]
        kp = torch.cat([kpts0.reshape(B * M, kd), kpts1.reshape(B * N, kd)], 0)
        theta = ops.PosencTheta.apply(kp.float().contiguous(), self.posenc.Wr.weight.float()).contiguous()
        sizes = (B, M, N)
        all0, all1, layers_x = [], [], []
        L = conf.n_layers
        self._refresh_shadow()
        if adaptive:
            return self._forward_adaptive(x, theta, sizes)
        # head -> layer gradient hand-over of the training step (engine.LayerFn / HeadFn docstrings)
        stash = {} if (self.training and torch.is_grad_enabled()) else None
        for i in range(L):
            w, params = self._layer_weights(i)
            fp = getattr(self, "_b200_flat", None)
            fp = fp if (fp is not None and fp.direct_groups) else None
            sink = (fp, i, stash) if torch.is_grad_enabled() else None
            x = engine.LayerFn.apply(x, theta, sizes, conf.num_heads, self._cdt, self.transformers[i].self_attn.ffn[1].eps,
                                     w, sink, *params)
            if self.training or i == L - 1:
                layers_x.append(x)
                all0.append(x[: B * M].view(B, M, D))
                all1.append(x[B * M:].view(B, N, D))
        d0, d1 = all0[-1], all1[-1]
        with torch.no_grad():
            md0, md1, z0, z1 = self._head_inputs(d0, d1, L - 1)
            sim = engine.similarity(md0, md1, self._cdt)
            st = ops.assign_stats(sim, F.logsigmoid(z0), F.logsigmoid(z1), F.logsigmoid(-z0), F.logsigmoid(-z1),
                                  dense=True)
            m0, m1, ms0, ms1 = ops.filter_matches(st["rowmax"], st["rowarg"], st["colarg"], conf.filter_threshold)
        pred = {
            "matches0": m0,
            "matches1": m1,
            "matching_scores0": ms0,
            "matching_scores1": ms1,
            "log_assignment": st["scores"],
            "prune0": torch.ones_like(ms0) * L,
            "prune1": torch.ones_like(ms1) * L,
        }
        if conf.stack_ref_descriptors is True or not self.training:
            pred["ref_descriptors0"] = torch.stack(all0, 1)
            pred["ref_descriptors1"] = torch.stack(all1, 1)
        # private side channel for loss(): the per-layer token tensors (both images, [T, D]); avoids
        # slicing the stacked ref_descriptors (whose backward would scatter into 9 zero-filled stacks).
        # Also the final layer's argmax including the dustbin (labels of TokenConfidence.loss) and the
        # row_norm monitor, both by-products of the dense pass.
        pred["_b200_layers"] = layers_x
        pred["_b200_sizes"] = sizes
        pred["_b200_stash"] = stash
        du0, du1 = F.logsigmoid(-z0), F.logsigmoid(-z1)
        pred["_b200_final_arg"] = (
            self._argmax_with_dustbin(st["rowmax"], st["rowarg"], du0, N).contiguous(),
            self._argmax_with_dustbin(st["colmax"], st["colarg"], du1, M).contiguous())
        pred["_b200_row_expsum"] = st["row_expsum"]
        return pred

    # ------------------------------------------------------------------------------------------
    @torch.no_grad()
    def _forward_adaptive(self, x, theta, sizes):
        """Inference-time adaptive depth / width (lightglue.py:461-526, 545-576; eval only, one pair): after every
        layer but the last, (a) stop when the fraction of confident points exceeds depth_confidence, (b) drop the points
        predicted unmatchable (matchability <= 1 - width_confidence) unless their confidence is still low, compacting the
        token matrix and the rotary angles with index_select.  The layers run on the same kernels (M != N after the
        first pruning); the two per-token logits come from one head_token pass.  On an early stop the assignment head of
        the stopping layer is used (upstream LightGlue's behaviour; the in-tree reference cannot take that branch: it
        stacks an empty list after the break, lightglue.py:485-492, 533)."""
        conf = self.conf
        B, M, N = sizes
        assert B == 1, "adaptive depth / width runs one pair at a time (lightglue.py:487, 492)"
        dev, D, L = x.device, conf.descriptor_dim, conf.n_layers
        do_stop, do_prune = conf.depth_confidence > 0, conf.width_confidence > 0
        ind0, ind1 = torch.arange(M, device=dev), torch.arange(N, device=dev)
        prune0 = torch.ones(1, M, device=dev, dtype=torch.int64)
        prune1 = torch.ones(1, N, device=dev, dtype=torch.int64)
        m, n = M, N
        last = L - 1
        for i in range(L):
            w, params = self._layer_weights(i)
            x = engine.LayerFn.apply(x, theta, (1, m, n), conf.num_heads, self._cdt, self.transformers[i].self_attn.ffn[1].eps,
                                     w, None, *params)
            if i == L - 1:
                break
            la, tk = self.log_assignment[i], self.token_confidence[i].token[0]
            _, zt, _, _ = ops.head_token_fwd(x, la.matchability.weight.view(-1), la.matchability.bias, tk.weight.view(-1),
                                             tk.bias, self._cdt)
            token = torch.sigmoid(zt[:, 1]) if do_stop else None  # token confidences only exist with early stopping on
            if do_stop:
                thr = self.confidence_thresholds[i]
                ratio = 1.0 - (token < thr).float().sum() / (M + N)  # relative to the ORIGINAL point count (lightglue.py:489)
                if bool(ratio > conf.depth_confidence):
                    last = i
                    break
            if do_prune:
                keep = torch.sigmoid(zt[:, 0]) > (1 - conf.width_confidence)
                if token is not None:  # low-confidence points are never pruned (lightglue.py:556-557)
                    keep = keep | (token <= self.confidence_thresholds[i])
                k0, k1 = torch.where(keep[:m])[0], torch.where(keep[m:])[0]
                ind0, ind1 = ind0.index_select(0, k0), ind1.index_select(0, k1)
                sel = torch.cat([k0, k1 + m])
                x, theta = x.index_select(0, sel).contiguous(), theta.index_select(0, sel).contiguous()
                m, n = int(k0.numel()), int(k1.numel())
                assert m > 0 and n > 0, "point pruning removed every keypoint of a view"
                prune0[:, ind0] += 1
                prune1[:, ind1] += 1
        d0, d1 = x[:m].view(1, m, D), x[m:].view(1, n, D)
        md0, md1, z0, z1 = self._head_inputs(d0, d1, last)
        sim = engine.similarity(md0, md1, self._cdt)
        st = ops.assign_stats(sim, F.logsigmoid(z0), F.logsigmoid(z1), F.logsigmoid(-z0), F.logsigmoid(-z1), dense=True)
        m0, m1, ms0, ms1 = ops.filter_matches(st["rowmax"], st["rowarg"], st["colarg"], conf.filter_threshold)
        if do_prune:  # scatter back to the full keypoint sets (lightglue.py:517-526)
            m0_ = torch.full((1, M), -1, device=dev, dtype=m0.dtype)
            m1_ = torch.full((1, N), -1, device=dev, dtype=m1.dtype)
            m0_[:, ind0] = torch.where(m0 == -1, -1, ind1[None].gather(1, m0.clamp(min=0)))
            m1_[:, ind1] = torch.where(m1 == -1, -1, ind0[None].gather(1, m1.clamp(min=0)))
            ms0_, ms1_ = torch.zeros(1, M, device=dev), torch.zeros(1, N, device=dev)
            ms0_[:, ind0] = ms0
            ms1_[:, ind1] = ms1
            m0, m1, ms0, ms1 = m0_, m1_, ms0_, ms1_
        else:
            prune0, prune1 = torch.ones_like(ms0) * L, torch.ones_like(ms1) * L
        # for loss(): one state, which gets head n_layers - 1 as in eval mode; a pruned pred (m, n < M, N) is rejected there
        return {"matches0": m0, "matches1": m1, "matching_scores0": ms0, "matching_scores1": ms1,
                "ref_descriptors0": d0[:, None], "ref_descriptors1": d1[:, None], "log_assignment": st["scores"],
                "prune0": prune0, "prune1": prune1, "stop_layer": last,
                "_b200_layers": [x], "_b200_sizes": (1, m, n), "_b200_row_expsum": st["row_expsum"]}

    # ------------------------------------------------------------------------------------------
    def _loss(self, pred, data):
        """lightglue.py:578-627 on the hand-scheduled heads (engine.HeadFn): per layer one autograd node that
        yields the NLL and the token-confidence BCE; the O(M+N) terms are two small fused kernels."""
        conf = self.conf
        layers_x = pred.get("_b200_layers")
        if layers_x is None:
            raise ValueError("LightGlue.loss needs the pred of this module's own forward: pred['_b200_layers'] is missing")
        (B, M, N), L = pred["_b200_sizes"], len(layers_x)
        gt = data["gt_assignment"]
        if tuple(gt.shape) != (B, M, N):
            raise ValueError(f"gt_assignment has shape {tuple(gt.shape)} but the forward ran on (B, M, N) = {(B, M, N)}; "
                             "the loss cannot be taken after point pruning (width_confidence)")
        gt_u8 = gt.contiguous().view(torch.uint8) if gt.dtype == torch.bool else gt.to(torch.uint8).contiguous()
        # both counts in one pass over the 4.2 MB/pair mask (`gt.sum(2)` / `gt.sum(1)` each widen it first: int64 by
        # default, fp32 with dtype=)
        rowcnt, colcnt = ops.mask_counts(gt_u8)
        neg0 = (data["gt_matches0"] == -1).float()
        neg1 = (data["gt_matches1"] == -1).float()
        num_pos = rowcnt.sum(1).clamp(min=1.0)
        num_neg0, num_neg1 = neg0.sum(1).clamp(min=1.0), neg1.sum(1).clamp(min=1.0)
        gtd = {"u8": gt_u8, "rowcnt": rowcnt.contiguous(), "colcnt": colcnt.contiguous(), "neg0": neg0.contiguous(),
               "neg1": neg1.contiguous(), "num_pos": num_pos.contiguous(), "num_neg": (num_neg0 + num_neg1).contiguous()}
        if self._bf16 and torch.is_grad_enabled():
            # the fused backward walks the mask by columns as well: one transposed copy per step, shared by all layers
            gt_t = data.get("gt_assignment_t")  # written by the plugin's ground-truth components when asked to
            gtd["u8_t"] = (gt_t.contiguous().view(torch.uint8) if gt_t is not None and gt_t.dtype == torch.bool
                           else gt_u8.transpose(1, 2).contiguous())
        fin = pred.get("_b200_final_arg")  # read only for L > 1, i.e. a training-mode forward, which always sets it

        def head(i):
            # the last stacked state always belongs to the LAST layer's head (lightglue.py:588 `loss_params(pred, -1)`):
            # in eval mode only that state is stacked (lightglue.py:485), so L == 1 while the head index is n_layers - 1
            hi = conf.n_layers - 1 if i == L - 1 else i
            la_i = self.log_assignment[hi]
            pre = f"log_assignment.{hi}.final_proj."
            tok = self.token_confidence[i].token[0] if (i < L - 1 and self.training) else None
            stash = pred.get("_b200_stash")
            # layers_x[i] is the output of transformer layer i only when every layer's state was kept (training)
            slot = (stash, i) if (stash is not None and L == conf.n_layers) else None
            return engine.HeadFn.apply(layers_x[i], (B, M, N), self._cdt, gtd, conf.loss.nll_balancing, fin, slot,
                                       self._shadow[pre + "weight"], self._shadow[pre + "bias"],
                                       la_i.final_proj.weight, la_i.final_proj.bias, la_i.matchability.weight,
                                       la_i.matchability.bias, tok.weight if tok is not None else None,
                                       tok.bias if tok is not None else None)

        nll, _, nll_pos, nll_neg = head(L - 1)
        losses = {
            "total": nll,
            "last": nll.clone().detach(),
            "assignment_nll": nll,
            "nll_pos": nll_pos,
            "nll_neg": nll_neg,
            "num_matchable": num_pos,
            "num_unmatchable": (num_neg0 + num_neg1) / 2.0,
        }
        if self.training:
            losses["confidence"] = 0.0
        losses["row_norm"] = pred["_b200_row_expsum"].mean(1)
        sum_weights = 1.0
        for i in range(L - 1):
            nll_i, conf_i, _, _ = head(i)
            weight = conf.loss.gamma ** (L - i - 1) if conf.loss.gamma > 0.0 else i + 1
            sum_weights += weight
            losses["total"] = losses["total"] + nll_i * weight
            if self.training:
                losses["confidence"] = losses["confidence"] + conf_i / (L - 1)
        losses["total"] = losses["total"] / sum_weights
        if self.training:
            losses["total"] = losses["total"] + losses["confidence"]
        metrics = {} if self.training else matcher_metrics(pred, data)
        return losses, metrics

    @staticmethod
    def _argmax_with_dustbin(val, arg, dust, width):
        """argmax over [inner scores | dustbin]: the dustbin (highest index) wins only when strictly larger."""
        return torch.where(dust > val, torch.full_like(arg, width), arg)

    def loss(self, pred, data):
        """lightglue.py:578-627 without materialising any of the per-layer log-assignment matrices.  Like forward, runs
        with the ambient autocast disabled; its backward is linear in the incoming gradient (GradScaler, train.py:490)."""
        with torch.autocast(device_type="cuda", enabled=False):
            return self._loss(pred, data)


@torch.no_grad()
def matcher_metrics(pred, data):
    """models/utils/metrics.py:4-50 restated (recall / precision / accuracy / ranking AP of matches0)."""
    m, gt_m, scores = pred["matches0"], data["gt_matches0"], pred["matching_scores0"]
    hit = (m == gt_m).float()
    r_mask = (gt_m > -1).float()
    a_mask = (gt_m >= -1).float()
    p_mask = ((m > -1) & (gt_m >= -1)).float()
    rec = (hit * r_mask).sum(1) / (1e-8 + r_mask.sum(1))
    acc = (hit * a_mask).sum(1) / (1e-8 + a_mask.sum(1))
    prec = (hit * p_mask).sum(1) / (1e-8 + p_mask.sum(1))
    order = torch.argsort(-scores)
    sp, sr, st = (torch.gather(t, -1, order) for t in (p_mask, r_mask, hit))
    p_pts = torch.cumsum(st * sp, -1) / (1e-8 + torch.cumsum(sp, -1))
    r_pts = torch.cumsum(st * sr, -1) / (1e-8 + sr.sum(-1)[:, None])
    ap = torch.sum((r_pts[..., 1:] - r_pts[..., :-1]) * p_pts[:, None, -1], dim=-1)
    return {"match_recall": rec, "match_precision": prec, "accuracy": acc, "average_precision": ap}


__main_model__ = LightGlue
