"""Hand-scheduled forward/backward of the matcher's two repeating units.

`LayerFn`  : one LightGlue transformer layer (self block on both images + bidirectional cross block,
             lightglue.py:224-245) as ONE autograd node.
`HeadFn`   : one deep-supervision head (MatchAssignment + NLL terms + argmax, lightglue.py:271-290,
             losses.py:6-73) as ONE autograd node.

Each node schedules its kernels explicitly instead of leaving the composition to torch autograd: weights
are read from a compute-dtype shadow refreshed once per step, weight gradients are produced in fp32
directly by the GEMM (`out_dtype`), the residual update emits the next GEMM's operand in the same
pass, there are no per-op dtype casts or cat/slice copies, and nothing N x N is ever kept besides
`sim`.

In `precision: bf16` every GEMM of the layer and of the head -- the nine nn.Linear projections, their input-gradient
and weight-gradient contractions -- runs on the library's own persistent wgmma GEMM (`ops.linear`: bias and
fp32 accumulate-into-dx epilogues; `ops.wgrad_bf16`: split-K, fp32 out); no cuBLAS kernel is launched.  The fp32
parity mode (`precision: fp32`) keeps fp32 cuBLAS (`torch.addmm/mm`) for the projections.
"""
from typing import NamedTuple

import torch
import torch.nn.functional as F

from . import ops

_head_counters = {}


def _lin(x, W, b, out=None):
    """y = x W^T + b.  bf16: own wgmma GEMM with the fp32 bias added in the epilogue (W = bf16 shadow, b = the fp32
    parameter); fp32 parity mode: cuBLAS."""
    if x.dtype == torch.bfloat16:
        return ops.linear(x, W, b, out=out)
    return torch.addmm(b, x, W.t()) if out is None else torch.addmm(b, x, W.t(), out=out)


def _dgrad(dy, W):
    """dx = dy W (compute dtype)."""
    if dy.dtype == torch.bfloat16:
        return ops.linear(dy, W, w_is_kn=True)
    return torch.mm(dy, W)


def _wgrad(dy, a, out=None):
    """dW [out, in] fp32 = dy^T a for compute-dtype dy [T, out], a [T, in] (row-strided views allowed); `out`: write
    straight into this fp32 view (a parameter's slot of the trainer's flat gradient buffer)."""
    if dy.dtype == torch.float32:
        return torch.mm(dy.t(), a) if out is None else torch.mm(dy.t(), a, out=out)
    return ops.wgrad_bf16(dy, a, out=out)


def _bgrad(dy):
    return ops.colsum(dy)


def similarity(md0, md1, cdt, alpha=1.0):
    """sim [B, M, N] fp32 = alpha md0 md1^T: bf16 operands on the wgmma GEMM when cdt is bf16; in the fp32 parity mode
    cuBLAS."""
    if cdt == torch.bfloat16:
        return ops.gemm_bf16(md0.to(torch.bfloat16).contiguous(), md1.to(torch.bfloat16).contiguous(), alpha=alpha)
    sim = torch.bmm(md0, md1.transpose(1, 2))
    return sim.mul_(alpha) if alpha != 1 else sim


def assign_unfused_bwd(md0, md1, sim, lse_row, lse_col, gt_u8, gcoef, rowcnt, colcnt, gt0=None):
    """d(mdesc0) [B, M, D], d(mdesc1) [B, N, D] (md0's dtype) of the NLL through a stored sim: dsim = gcoef (2 gt -
    softmax_row rowcnt - softmax_col colcnt) from lgb200_assign_bwd, then dsim md1 and dsim^T md0.  The unfused
    counterpart of ops.assign_fused_bwd, for fp32 and for operands assign_fused_ok rejects.  gt_u8 None: gt is the
    match list gt0 [B, M] int64 (lgb200_assign_bwd_sparse, the same dsim)."""
    B, M, N = sim.shape
    cdt = md0.dtype
    tc = cdt == torch.bfloat16 and N % 8 == 0 and M % 8 == 0
    dsim = torch.empty(B, M, N, device=sim.device, dtype=torch.bfloat16 if tc else torch.float32)
    ops.call("lgb200_assign_bwd" if gt_u8 is not None else "lgb200_assign_bwd_sparse", ops.ptr(sim), ops.ptr(lse_row),
             ops.ptr(lse_col), ops.ptr(gt_u8 if gt_u8 is not None else gt0), ops.ptr(gcoef), ops.ptr(rowcnt),
             ops.ptr(colcnt), ops.ptr(dsim), ops._code(dsim.dtype), B, M, N, ops.stream_ptr())
    if tc:
        dmd0 = ops.gemm_bf16(dsim, md1, a_mn_major=False, b_mn_major=True, out_dtype=cdt)  # dsim   md1
        dmd1 = ops.gemm_bf16(dsim, md0, a_mn_major=True, b_mn_major=True, out_dtype=cdt)   # dsim^T md0
    else:
        dmd0 = torch.bmm(dsim, md1.float()).to(cdt)
        dmd1 = torch.bmm(dsim.transpose(1, 2), md0.float()).to(cdt)
    return dmd0, dmd1


def _dgrad_acc(acc, dy, w):
    """acc (fp32 [T, in]) += dy (compute dtype [T, out]) @ w ([out, in]), IN PLACE: the GEMM's epilogue stages its
    tile in shared memory and adds it into acc with a TMA reduce-add (bf16 operands), so the residual-stream gradient
    is accumulated in fp32 and never re-read by an SM (an acc that is not 16-byte aligned is read-modify-written from
    registers instead).  Every `acc` handed in is a gradient buffer this engine owns."""
    if dy.dtype == torch.float32:
        return acc.addmm_(dy, w)
    return ops.linear(dy, w, out=acc, w_is_kn=True, accumulate=True)


class Ragged(NamedTuple):
    """`sizes` of a forward-only layer over pairs of different lengths (adaptive depth / width): seg [4, 2B] int32 on
    the device = (offset, length, partner's offset, partner's length) of segment 2b (image 0 of pair b) and 2b + 1
    (image 1); max_len bounds every length."""
    seg: torch.Tensor
    max_len: int


def _attend_fwd(q, k, v, sizes, H, cross):
    """q,k,v [T, H*hd] over tokens [image0 (B*M); image1 (B*N)] -> (out [T, H*hd], lse tuple).  The head dim hd = 64 or
    32 is read from the shapes; the scale is hd^-1/2 (lightglue.py:139, 173).  Ragged sizes: one launch over the
    packed segments, each attending to itself (self) or to its partner (cross)."""
    hd = q.shape[1] // H
    scale = hd ** -0.5
    if isinstance(sizes, Ragged):
        off, ln, poff, pln = sizes.seg
        shp = (q.shape[0], H, hd)
        out, lse = ops.attn_fwd_varlen(q.view(shp), k.view(shp), v.view(shp), off, ln, poff if cross else off,
                                       pln if cross else ln, sizes.max_len, scale)
        return out.view(q.shape), (lse,)
    B, M, N = sizes
    if M == N:
        shp = (2 * B, M, H, hd)
        out, lse = ops.attn_fwd(q.view(shp), k.view(shp), v.view(shp), B if cross else 0, scale)
        return out.view(q.shape), (lse,)
    t0 = B * M
    q0, q1 = q[:t0].view(B, M, H, hd), q[t0:].view(B, N, H, hd)
    k0, k1 = k[:t0].view(B, M, H, hd), k[t0:].view(B, N, H, hd)
    v0, v1 = v[:t0].view(B, M, H, hd), v[t0:].view(B, N, H, hd)
    if cross:
        o0, l0 = ops.attn_fwd(q0, k1, v1, 0, scale)
        o1, l1 = ops.attn_fwd(q1, k0, v0, 0, scale)
    else:
        o0, l0 = ops.attn_fwd(q0, k0, v0, 0, scale)
        o1, l1 = ops.attn_fwd(q1, k1, v1, 0, scale)
    return torch.cat([o0.reshape(t0, -1), o1.reshape(B * N, -1)], 0), (l0, l1)


def _attend_bwd(q, k, v, out, lses, dout, sizes, H, cross):
    B, M, N = sizes
    hd = q.shape[1] // H
    scale = hd ** -0.5
    if M == N:
        shp = (2 * B, M, H, hd)
        dq, dk, dv = ops.attn_bwd(q.view(shp), k.view(shp), v.view(shp), out.view(shp), lses[0], dout.view(shp),
                                  B if cross else 0, scale)
        return dq.view(q.shape), dk.view(q.shape), dv.view(q.shape)
    t0 = B * M
    sp = lambda t: (t[:t0].view(B, M, H, hd), t[t0:].view(B, N, H, hd))  # noqa: E731
    (q0, q1), (k0, k1), (v0, v1), (o0, o1), (g0, g1) = sp(q), sp(k), sp(v), sp(out), sp(dout.contiguous())
    if cross:
        dq0, dk1, dv1 = ops.attn_bwd(q0, k1, v1, o0, lses[0], g0, 0, scale)
        dq1, dk0, dv0 = ops.attn_bwd(q1, k0, v0, o1, lses[1], g1, 0, scale)
    else:
        dq0, dk0, dv0 = ops.attn_bwd(q0, k0, v0, o0, lses[0], g0, 0, scale)
        dq1, dk1, dv1 = ops.attn_bwd(q1, k1, v1, o1, lses[1], g1, 0, scale)
    cat = lambda a, b: torch.cat([a.reshape(t0, -1), b.reshape(B * N, -1)], 0)  # noqa: E731
    return cat(dq0, dq1), cat(dk0, dk1), cat(dv0, dv1)


def _attend_bwd_shared_qk(qk, v, out, lses, dout, sizes, H):
    """Cross-attention backward with one to_qk projection as query in one direction and key in the other
    (lightglue.py:207-216) -> (dqk = dq + dk, dv).  The one-sweep shared-qk kernel is built for head dim 64; at
    head dim 32, and whenever M != N, both directions write separate dq / dk buffers that are then added."""
    B, M, N = sizes
    hd = qk.shape[1] // H
    if M != N or hd != 64:
        dq, dk, dv = _attend_bwd(qk, qk, v, out, lses, dout, sizes, H, cross=True)
        return dq.add_(dk), dv
    shp = (2 * B, M, H, hd)
    dqk, dv = ops.attn_bwd_shared_qk(qk.view(shp), v.view(shp), out.view(shp), lses[0], dout.view(shp), 0.125)
    return dqk.view(qk.shape), dv.view(qk.shape)


# order of the per-layer tensors (reference names, lightglue.py:139-148, 174-183)
LAYER_PARAMS = [
    "self_attn.Wqkv.weight", "self_attn.Wqkv.bias", "self_attn.out_proj.weight", "self_attn.out_proj.bias",
    "self_attn.ffn.0.weight", "self_attn.ffn.0.bias", "self_attn.ffn.1.weight", "self_attn.ffn.1.bias",
    "self_attn.ffn.3.weight", "self_attn.ffn.3.bias",
    "cross_attn.to_qk.weight", "cross_attn.to_qk.bias", "cross_attn.to_v.weight", "cross_attn.to_v.bias",
    "cross_attn.to_out.weight", "cross_attn.to_out.bias", "cross_attn.ffn.0.weight", "cross_attn.ffn.0.bias",
    "cross_attn.ffn.1.weight", "cross_attn.ffn.1.bias", "cross_attn.ffn.3.weight", "cross_attn.ffn.3.bias",
]
_LN_SLOTS = (6, 7, 18, 19)  # LayerNorm affine stays fp32


class LayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, theta, sizes, H, cdt, eps, w, sink, *params):
        """sink: None, or (flat-parameter object or None, layer index, stash or None).
        flat-parameter object (a trainer that owns a flat gradient buffer): the backward writes this layer's 22
        parameter gradients straight into their slots of that buffer (weight gradients as the GEMM output, no
        per-parameter copy) and tells the trainer the slice is final.
        stash (dict): the supervision head that reads this layer's output leaves its gradient w.r.t. that output in
        stash[layer index] instead of returning it to autograd (HeadFn); this backward merges it with the gradient
        coming from the next layer in the same pass that produces the bf16 copy the first GEMMs need (autograd would
        run a separate accumulation kernel over the [T, D] fp32 tensor, and the cast after it).  Autograd's dependency
        rule -- a node runs after every consumer of its outputs has run -- guarantees the head has filled the stash."""
        (Wqkv, bqkv, Wo, bo, W0, b0, g1, be1, W3, b3,
         Wqk, bqk, Wv, bv, Wout, bout, W0c, b0c, g2, be2, W3c, b3c) = w
        if cdt == torch.bfloat16:  # biases are added in fp32 in the GEMM epilogue: take the master parameters
            bqkv, bo, b0, b3, bqk, bv, bout, b0c, b3c = (params[i].detach() for i in (1, 3, 5, 9, 11, 13, 15, 17, 21))
        D = x.shape[1]
        x = x.contiguous()
        # The FFN input cat([x, msg], -1) (lightglue.py:162, 219) is never concatenated: the compute-dtype copy of x
        # and the out-projection's result are written straight into the two halves of one [T, 2D] buffer, which
        # then feeds ffn.0 as ONE K=2D GEMM (and, in backward, one [2D x 2D] weight-gradient GEMM).
        T = x.shape[0]
        # ---- self block (lightglue.py:150-163)
        cat1 = torch.empty(T, 2 * D, device=x.device, dtype=cdt)
        x16, msg = cat1[:, :D], cat1[:, D:]
        ops.residual_add_cast(x, None, cdt, out_cast=x16)
        qkv = _lin(x16, Wqkv, bqkv)
        q, k, v = ops.rope_fwd(qkv, theta, H)
        del qkv
        att, lse1 = _attend_fwd(q, k, v, sizes, H, cross=False)
        _lin(att, Wo, bo, out=msg)
        h = _lin(cat1, W0, b0)
        g, mean1, rstd1 = ops.ln_gelu_fwd(h, g1, be1, eps)
        y = _lin(g, W3, b3)
        cat2 = torch.empty(T, 2 * D, device=x.device, dtype=cdt)
        x1_16, msg2 = cat2[:, :D], cat2[:, D:]
        x1, _ = ops.residual_add_cast(x, y, cdt, out_cast=x1_16)
        del y
        # ---- cross block (lightglue.py:195-221)
        qk = _lin(x1_16, Wqk, bqk)
        vv = _lin(x1_16, Wv, bv)
        m, lse2 = _attend_fwd(qk, qk, vv, sizes, H, cross=True)
        _lin(m, Wout, bout, out=msg2)
        h2 = _lin(cat2, W0c, b0c)
        gg, mean2, rstd2 = ops.ln_gelu_fwd(h2, g2, be2, eps)
        y2 = _lin(gg, W3c, b3c)
        x2, _ = ops.residual_add_cast(x1, y2, None)
        ctx.save_for_backward(theta, cat1, q, k, v, att, h, mean1, rstd1, g, cat2, qk, vv, m, h2, mean2,
                              rstd2, gg, *lse1, *lse2, *w)
        ctx.meta = (sizes, H, cdt, len(lse1), len(lse2), D)
        ctx.sink = sink
        ctx.set_materialize_grads(False)  # the output's gradient may arrive through the stash only
        return x2

    @staticmethod
    def backward(ctx, dx):
        sizes, H, cdt, n1, n2, D = ctx.meta
        sv = ctx.saved_tensors
        (theta, cat1, q, k, v, att, h, mean1, rstd1, g, cat2, qk, vv, m, h2, mean2, rstd2, gg) = sv[:18]
        x16, x1_16 = cat1[:, :D], cat2[:, :D]
        lse1, lse2 = sv[18:18 + n1], sv[18 + n1:18 + n1 + n2]
        (Wqkv, bqkv, Wo, bo, W0, b0, g1, be1, W3, b3,
         Wqk, bqk, Wv, bv, Wout, bout, W0c, b0c, g2, be2, W3c, b3c) = sv[18 + n1 + n2:]
        fp, slot, stash = ctx.sink if ctx.sink is not None else (None, None, None)
        extra = stash.pop(slot, None) if stash is not None else None  # the supervision head's share (see forward)
        if dx is None and extra is None:
            return (None,) * (8 + 22)
        if dx is None:
            dx, dy2 = extra, extra.to(cdt)
        elif extra is None:
            dx = dx.contiguous()
            dy2 = dx.to(cdt)
        else:
            dx = dx.contiguous()
            if dx.dtype == torch.float32 and extra.dtype == torch.float32 and dx.is_cuda:
                dx, dy2 = ops.add_f32_cast_(dx, extra.contiguous(), cdt)  # dx is this node's own incoming buffer
            else:
                dx = dx + extra
                dy2 = dx.to(cdt)
        gv = fp.direct_views(slot) if fp is not None else [None] * 22  # LAYER_PARAMS order; None for a frozen slot
        need = ctx.needs_input_grad[8:]  # per LAYER_PARAMS slot: a frozen parameter's GEMM / column sum is skipped
        wg = lambda i, d, a: _wgrad(d, a, gv[i]) if need[i] else None  # noqa: E731
        bg = lambda i, d: _bgrad(d) if need[i] else None  # noqa: E731
        # ---- cross block
        dW3c, db3c = wg(20, dy2, gg), bg(21, dy2)
        dgg = _dgrad(dy2, W3c)
        dh2, dg2, dbe2, db0c = ops.ln_gelu_bwd(dgg, h2, g2, be2, mean2, rstd2, want_dxsum=True)
        del dgg
        dW0c = wg(16, dh2, cat2)
        dmsg2 = _dgrad(dh2, W0c[:, D:])
        dx1 = _dgrad_acc(dx, dh2, W0c[:, :D])  # fp32 accumulation of the residual-stream gradient
        del dh2
        dWout, dbout = wg(14, dmsg2, m), bg(15, dmsg2)
        dm = _dgrad(dmsg2, Wout)
        dqk, dvv = _attend_bwd_shared_qk(qk, vv, m, lse2, dm, sizes, H)
        dWqk, dbqk = wg(10, dqk, x1_16), bg(11, dqk)
        dWv, dbv = wg(12, dvv, x1_16), bg(13, dvv)
        dx1 = _dgrad_acc(dx1, dqk, Wqk)
        dx1 = _dgrad_acc(dx1, dvv, Wv)
        # ---- self block
        dy = dx1.to(cdt)
        dW3, db3 = wg(8, dy, g), bg(9, dy)
        dg = _dgrad(dy, W3)
        dh, dg1, dbe1, db0 = ops.ln_gelu_bwd(dg, h, g1, be1, mean1, rstd1, want_dxsum=True)
        del dg
        dW0 = wg(4, dh, cat1)
        dmsg = _dgrad(dh, W0[:, D:])
        dx0 = _dgrad_acc(dx1, dh, W0[:, :D]) if ctx.needs_input_grad[0] else None
        del dh
        dWo, dbo = wg(2, dmsg, att), bg(3, dmsg)
        datt = _dgrad(dmsg, Wo)
        dq, dk, dv = _attend_bwd(q, k, v, att, lse1, datt, sizes, H, cross=False)
        dqkv, dtheta = ops.rope_bwd(dq, dk, dv, q, k, theta, H, need_dtheta=ctx.needs_input_grad[1])
        dWqkv, dbqkv = wg(0, dqkv, x16), bg(1, dqkv)
        if dx0 is not None:
            dx0 = _dgrad_acc(dx0, dqkv, Wqkv)
        grads = (dWqkv, dbqkv, dWo, dbo, dW0, db0, dg1, dbe1, dW3, db3,
                 dWqk, dbqk, dWv, dbv, dWout, dbout, dW0c, db0c, dg2, dbe2, dW3c, db3c)
        grads = tuple(gr if need[i] else None for i, gr in enumerate(grads))  # the LayerNorm kernel's by-products
        if fp is not None:
            # the trainable weight gradients are already in place; the vectors go in with one multi-tensor copy
            small = [i for i in range(22) if grads[i] is not None and grads[i].data_ptr() != gv[i].data_ptr()]
            torch._foreach_copy_([gv[i] for i in small], [grads[i].view_as(gv[i]) for i in small])
            grads = (None,) * 22
        return (dx0, dtheta, None, None, None, None, None, None) + grads


class HeadFn(torch.autograd.Function):
    """x [T, D] fp32 (tokens of both images) -> (nll [B], conf [B]) of this layer: the NLL of its assignment
    and the token-confidence BCE against the final layer's argmax (`fin`; None for the last layer),
    plus the detached nll_pos / nll_neg for logging."""

    @staticmethod
    def forward(ctx, x, sizes, cdt, gt, bal, fin, stash, wfp, bfp, Wfp_p, bfp_p, wm, bm, wt, bt):
        """stash: None, or (dict, key): the backward then leaves the gradient w.r.t. x in dict[key] for the LayerFn that
        produced x (which merges it with the next layer's gradient in one fused pass) instead of returning it.
        gt["u8"] None: the labels are the match lists gt["m0"] / gt["m1"] (int64), and the positive term is one entry per
        row (ops.assign_pos_fwd / assign_pos_bwd, lgb200_assign_bwd_sparse) instead of a pass over the mask."""
        B, M, N = sizes
        D = x.shape[1]
        t0 = B * M
        dev = x.device
        x = x.contiguous()
        has_tok = wt is not None
        # compute-dtype x for final_proj + [matchability logit, token-confidence logit] per token, one pass over x
        x16, zt, ls, du = ops.head_token_fwd(x, wm.view(-1), bm, wt.view(-1) if has_tok else None,
                                             bt if has_tok else None, cdt)
        md = _lin(x16, wfp, bfp_p.detach() if cdt == torch.bfloat16 else bfp)  # final_proj, un-scaled; d^-1/2 is folded into sim
        md0, md1 = md[:t0].view(B, M, D), md[t0:].view(B, N, D)
        alpha = float(D) ** -0.5
        ls0, ls1, du0, du1 = ls[:t0].view(B, M), ls[t0:].view(B, N), du[:t0].view(B, M), du[t0:].view(B, N)
        sparse = gt["u8"] is None
        fused = ops.assign_fused_ok(md, D) and (sparse or gt.get("u8_t") is not None)
        if fused:
            # GEMM + LSE, then GEMM + scores / argmax / positives: the similarity matrix stays in tensor memory
            sim = None
            st = ops.assign_fused_stats(md0, md1, alpha, ls0, ls1, gt_u8=gt["u8"])
        else:
            sim = similarity(md0, md1, cdt, alpha)
            st = ops.assign_stats(sim, ls0, ls1, du0, du1, gt_u8=gt["u8"], dense=False)
        if sparse:
            st["pos_row_sum"] = (ops.assign_pos_fwd(gt["m0"], gt["m1"], st["lse_row"], st["lse_col"], alpha, md0, md1)
                                 if fused else
                                 ops.assign_pos_fwd(gt["m0"], gt["m1"], st["lse_row"], st["lse_col"], alpha, sim=sim))
        out = torch.empty(4, B, device=dev, dtype=torch.float32)
        f0, f1 = (fin if (fin is not None and has_tok) else (None, None))
        hws = torch.empty(4 * B * ((M + N + 255) // 256), device=dev, dtype=torch.float32)
        cnt = _head_counters.get(dev)
        if cnt is None:
            cnt = _head_counters[dev] = torch.zeros(4096, device=dev, dtype=torch.int32)
        assert B <= 4096
        ops.call("lgb200_head_terms_fwd", ops.ptr(zt), ops.ptr(st["pos_row_sum"]), ops.ptr(gt["rowcnt"]),
                 ops.ptr(gt["colcnt"]), ops.ptr(gt["neg0"]), ops.ptr(gt["neg1"]), ops.ptr(st["rowmax"]),
                 ops.ptr(st["rowarg"]), ops.ptr(st["colmax"]), ops.ptr(st["colarg"]), ops.ptr(f0), ops.ptr(f1),
                 ops.ptr(gt["num_pos"]), ops.ptr(gt["num_neg"]), float(bal), ops.ptr(out[0]), ops.ptr(out[1]),
                 ops.ptr(out[2]), ops.ptr(out[3]), ops.ptr(hws), ops.ptr(cnt), B, M, N, ops.stream_ptr())
        nll, nll_pos, nll_neg, conf = out[0], out[1], out[2], out[3]
        saved = [x, x16, md, sim if sim is not None else gt.get("u8_t"), st["lse_row"], st["lse_col"], zt, st["rowmax"],
                 st["rowarg"], st["colmax"], st["colarg"], wfp, wm, gt["u8"], gt["rowcnt"], gt["colcnt"], gt["neg0"],
                 gt["neg1"], gt["num_pos"], gt["num_neg"], gt.get("m0"), gt.get("m1")]
        if f0 is not None:
            saved += [f0, f1]
        ctx.save_for_backward(*saved)
        ctx.meta = (sizes, cdt, bal, alpha, has_tok, f0 is not None, fused)
        ctx.stash = stash
        ctx.mark_non_differentiable(nll_pos, nll_neg)
        return nll, conf, nll_pos, nll_neg

    @staticmethod
    def backward(ctx, g_nll, g_conf, *_):
        sv = ctx.saved_tensors
        (x, x16, md, sim, lse_row, lse_col, zt, rowmax, rowarg, colmax, colarg, wfp, wm, gt_u8, rowcnt, colcnt, neg0,
         neg1, num_pos, num_neg, gt0, gt1) = sv[:22]
        (B, M, N), cdt, bal, alpha, has_tok, has_fin, fused = ctx.meta
        f0, f1 = (sv[22], sv[23]) if has_fin else (None, None)
        D = x.shape[1]
        t0 = B * M
        g_nll = g_nll.float().contiguous()
        g_conf = g_conf.float().contiguous() if g_conf is not None else torch.zeros_like(g_nll)
        dzt = torch.empty_like(zt)
        ops.call("lgb200_head_terms_bwd", ops.ptr(zt), ops.ptr(rowcnt), ops.ptr(colcnt), ops.ptr(neg0), ops.ptr(neg1),
                 ops.ptr(rowmax), ops.ptr(rowarg), ops.ptr(colmax), ops.ptr(colarg), ops.ptr(f0), ops.ptr(f1),
                 ops.ptr(num_pos), ops.ptr(num_neg), float(bal), ops.ptr(g_nll), ops.ptr(g_conf), ops.ptr(dzt), B, M, N,
                 ops.stream_ptr())
        # similarity: dsim = gc (2 gt - softmax_row * rowcnt - softmax_col * colcnt), gc includes d^-1/2
        # frozen parameters (and an x that needs no gradient, when every layer up to this head is frozen) are skipped
        need_x, need_wfp, need_bfp, need_wm, need_bm, need_wt, need_bt = (ctx.needs_input_grad[i]
                                                                           for i in (0, 9, 10, 11, 12, 13, 14))
        dmd = None
        if need_x or need_wfp or need_bfp:
            gc = (g_nll * (-bal * alpha) / num_pos).contiguous()
            md0, md1 = md[:t0].view(B, M, D), md[t0:].view(B, N, D)
            if fused:
                # dsim is recomputed tile by tile and contracted with the other image's descriptors in the same kernel
                dmd = torch.empty(t0 + B * N, D, device=x.device, dtype=cdt)
                ops.assign_fused_bwd(md0, md1, alpha, lse_row, lse_col, gt_u8, sim, gc, rowcnt, colcnt, dmd[:t0],
                                     dmd[t0:])
                if gt_u8 is None:
                    ops.assign_pos_bwd(md0, md1, gc, gt0, gt1, dmd[:t0], dmd[t0:])
            else:
                dmd0, dmd1 = assign_unfused_bwd(md0, md1, sim, lse_row, lse_col, gt_u8, gc, rowcnt, colcnt, gt0)
                dmd = torch.cat([dmd0.reshape(t0, D), dmd1.reshape(B * N, D)], 0)
        dWfp = _wgrad(dmd, x16) if need_wfp else None
        dbfp = _bgrad(dmd) if need_bfp else None
        dx = dW2 = db2 = None
        if need_x or need_wm or need_bm or need_wt or need_bt:
            # dx = dmd W_fp + dzt[:,0] wm (the token-confidence head reads a detached x, lightglue.py:82-83), dW2, db2
            dx, dW2, db2 = ops.head_token_bwd(x, _dgrad(dmd, wfp) if need_x else None, dzt, wm.view(-1))
        pick = lambda t, row, want: t[row:row + 1] if want else None  # noqa: E731
        dwm, dbm = pick(dW2, 0, need_wm), pick(db2, 0, need_bm)
        dwt, dbt = (pick(dW2, 1, need_wt), pick(db2, 1, need_bt)) if has_tok else (None, None)
        if ctx.stash is not None and dx is not None:
            d, key = ctx.stash
            d[key] = dx if key not in d else d[key] + dx
            dx = None
        return dx, None, None, None, None, None, None, None, None, dWfp, dbfp, dwm, dbm, dwt, dbt
