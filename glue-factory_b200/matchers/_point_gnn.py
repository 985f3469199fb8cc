"""Point-side building blocks shared by the GlueStick and SuperGlue plugins: both reference models use the same
MultiHeadedAttention (channel = d * H + h), the same MLP of Conv1d + BatchNorm1d + ReLU, the same keypoint
normalisation and the same similarity (gluestick.py:465-551, superglue.py:70-147, 294-295).

Node features are token-major [B*N, D].  A Conv1d(k=1) with a tensor-core-sized input is the library's wgmma GEMM
(`ops.LinearFn`) in bf16 mode and an fp32 linear otherwise; the attention core is the wgmma / CUDA-core attention
pair with the projection weights permuted to head-major once per layer; BatchNorm + ReLU is `ops.batchnorm_relu`.
"""
import torch
import torch.nn.functional as F
from torch import nn
from torch.nn.modules.batchnorm import _BatchNorm

from .. import ops


class _BmmNT(torch.autograd.Function):
    """sim [B,M,N] fp32 = alpha * a [B,M,D] . b [B,N,D]^T on the batched wgmma GEMM, with its two backward
    contractions (gluestick.py:248-249 `einsum("bdn,bdm->bnm")`)."""

    @staticmethod
    def forward(ctx, a, b, alpha):
        ctx.save_for_backward(a, b)
        ctx.alpha = alpha
        return ops.gemm_bf16(a, b, alpha=alpha)

    @staticmethod
    def backward(ctx, g):
        a, b = ctx.saved_tensors
        g16 = g.to(torch.bfloat16).contiguous()
        da = ops.gemm_bf16(g16, b, a_mn_major=False, b_mn_major=True, out_dtype=torch.bfloat16, alpha=ctx.alpha)
        db = ops.gemm_bf16(g16, a, a_mn_major=True, b_mn_major=True, out_dtype=torch.bfloat16, alpha=ctx.alpha)
        return da, db, None


class PointGNN(nn.Module):
    """Base of the point matchers: needs `self.conf.precision` and `_register_head_perm(D)` called in __init__."""

    def _register_head_perm(self, D, H=4):
        # head permutation: reference channel c = d * H + h  <->  head-major channel h * 64 + d
        dh = D // H
        c = torch.arange(D)
        self.register_buffer("_perm", ((c % dh) * H + c // dh), persistent=False)

    @property
    def _bf16(self):
        return self.conf.precision == "bf16"

    def _conv(self, x, conv, w=None, b=None, keep_bf16=False):
        """Conv1d(kernel 1) on token-major x [T, C_in]; w / b override the module's parameters (permuted views).
        bf16 mode: x may already be bf16 (no second cast), and keep_bf16 leaves the GEMM's bf16 output as it is for a
        consumer that rounds to bf16 anyway (the next GEMM, BatchNorm + ReLU in front of one, the attention kernels)."""
        w = conv.weight[:, :, 0] if w is None else w
        b = conv.bias if b is None else b
        if self._bf16 and w.shape[1] % 64 == 0 and w.shape[0] % 8 == 0:
            y = ops.LinearFn.apply(x.to(torch.bfloat16).contiguous(), w, b)
            return y if keep_bf16 else y.float()
        return F.linear(x.float(), w, b)

    def _mlp(self, x, seq, stats=None):
        """`stats`: None or a list that receives (BatchNorm module, batch statistics) of every training-mode BatchNorm."""
        mods = list(seq)
        for i, m in enumerate(mods):
            if isinstance(m, nn.Conv1d):
                # an inner layer's output only feeds BatchNorm / ReLU and the next GEMM, which rounds it to bf16 at the
                # same point either way: keep it bf16 (BatchNorm still accumulates its statistics in fp64)
                x = self._conv(x, m, keep_bf16=self._bf16 and i < len(mods) - 1)
            elif isinstance(m, _BatchNorm):
                # BatchNorm1d, or SyncBatchNorm after convert_sync_batchnorm (statistics summed over its process
                # group), fused with the ReLU that MLP() puts behind it; [T, C]: statistics over all tokens of this call
                assert isinstance(mods[i + 1], nn.ReLU), mods[i + 1]
                saved = [] if stats is not None else None
                x = ops.batchnorm_relu(x if x.dtype == torch.bfloat16 else x.float(), m, ops.bn_exchange(m), saved)
                if saved:
                    stats.append((m, saved[0]))
            elif not isinstance(mods[i - 1], _BatchNorm):
                x = torch.relu(x)
        return x

    def _attn_weights(self, attn):
        """The projection / merge weights of one MultiHeadedAttention with the head permutation applied (rows of q, k, v,
        columns of merge); computed once per layer and shared by both images."""
        perm = self._perm
        return ([(p.weight[:, :, 0][perm], p.bias[perm]) for p in attn.proj], attn.merge.weight[:, :, 0][:, perm])

    def _attention(self, x, src, attn, B, wts=None):
        """MultiHeadedAttention (gluestick.py:532-551): x [B*N, D] attends to src [B*M, D]."""
        D = x.shape[1]
        proj_w, merge_w = wts if wts is not None else self._attn_weights(attn)
        if self._bf16:  # one cast per input, projections stay bf16 into the attention kernels and out of them
            x, src = x.to(torch.bfloat16), (src.to(torch.bfloat16) if src is not x else None)
            src = x if src is None else src
        q, k, v = (self._conv(t, p, w, b, keep_bf16=True) for p, (w, b), t in zip(attn.proj, proj_w, (x, src, src)))
        cdt = torch.bfloat16 if self._bf16 else torch.float32
        shp = lambda t: t.to(cdt).view(B, -1, 4, D // 4)  # noqa: E731  head-major thanks to the permuted rows
        o = ops.Attention.apply(shp(q), shp(k), shp(v), 0, (D // 4) ** -0.5)
        return self._conv(o.reshape(-1, D), attn.merge, merge_w, attn.merge.bias)

    def _gnn_layer(self, d0, d1, prop, cross, B, stats=None):
        """One AttentionalPropagation `prop` applied to both images: x + MLP([x ; MHA(x, src)]), src the other image's
        features when `cross`.  `stats` as in _mlp."""
        s0, s1 = (d1, d0) if cross else (d0, d1)
        wts = self._attn_weights(prop.attn)
        out = []
        for x, src in ((d0, s0), (d1, s1)):
            msg = self._attention(x, src, prop.attn, B, wts)
            out.append(x + self._mlp(torch.cat([x, msg], 1), prop.mlp, stats))
        return out[0], out[1]

    @staticmethod
    def _norm_kpts(kpts, size):
        """gluestick.py:478-490 (superglue.py:83-93): centre, divide by 0.7 * the longer side."""
        size = size.to(kpts)
        return (kpts - (size / 2)[:, None, :]) / (size.max(1, keepdim=True).values * 0.7)[:, None, :]

    def _similarity(self, m0, m1, B):
        """[B,M,N] fp32 = m0 . m1^T / sqrt(D): the wgmma GEMM with fp32 output in bf16 mode, fp32 bmm otherwise."""
        D = m0.shape[1]
        a, b = m0.view(B, -1, D), m1.view(B, -1, D)
        if self._bf16 and a.shape[1] % 8 == 0 and b.shape[1] % 8 == 0:
            return _BmmNT.apply(a.to(torch.bfloat16).contiguous(), b.to(torch.bfloat16).contiguous(), D ** -0.5)
        return torch.bmm(a, b.transpose(1, 2)) / D ** 0.5
