"""torch.autograd bindings of the lgb200 kernels.

PyTorch is used here only as plumbing: it owns the device buffers, the stream
and the autograd tape; every numerical step of the N x N path is one of the
C-ABI entry points of include/lgb200.h.  Nothing in this file has a CPU
branch: on a machine without the built library or without an H100 the first
call raises `Lgb200Error`.
"""
import torch

from . import _lib
from ._lib import BF16, F32, call, ptr, stream_ptr


def _code(dtype):
    if dtype == torch.float32:
        return F32
    if dtype == torch.bfloat16:
        return BF16
    raise TypeError(f"lgb200 kernels take float32 or bfloat16 tensors, got {dtype}")


def _chk(t, dtype=None, strided_rows=False):
    if not t.is_cuda:
        raise _lib.Lgb200Error("lgb200 ops take CUDA tensors only: there is no CPU fallback")
    if strided_rows:  # 2-D view with unit inner stride (a column slice of a wider matrix)
        assert t.dim() == 2 and t.stride(1) == 1, "lgb200 op needs rows with unit inner stride"
    else:
        assert t.is_contiguous(), "lgb200 ops need contiguous tensors"
    if dtype is not None:
        assert t.dtype == dtype, (t.dtype, dtype)
    return t


# ------------------------------------------------------------------------------------------------
# rotary split (lightglue.py:157-160)
# ------------------------------------------------------------------------------------------------
def rope_fwd(qkv, theta, H):
    """qkv [T, H*3*hd] (feature = h*3*hd + d*3 + {q,k,v}), theta [T, hd/2] -> rotated q, k and v [T, H*hd]; the head
    dim hd = 64 or 32 is read from the shapes."""
    _chk(qkv)
    _chk(theta, torch.float32)
    T = qkv.shape[0]
    hd = qkv.shape[1] // (3 * H)
    assert qkv.shape[1] == 3 * H * hd and theta.shape == (T, hd // 2), (tuple(qkv.shape), tuple(theta.shape), H)
    q = torch.empty(T, H * hd, device=qkv.device, dtype=qkv.dtype)
    k, v = torch.empty_like(q), torch.empty_like(q)
    args = (ptr(qkv), ptr(theta), ptr(q), ptr(k), ptr(v), T, H, _code(qkv.dtype))
    if hd == 64:
        call("lgb200_rope_split_fwd", *args, stream_ptr())
    else:
        call("lgb200_rope_split_fwd_hd", *args, hd, stream_ptr())
    return q, k, v


def rope_bwd(dq, dk, dv, q, k, theta, H, dtheta=None, need_dtheta=True):
    """Returns (dqkv, dtheta); ACCUMULATES into dtheta (allocated zeroed when None).  need_dtheta=False: the angles
    need no gradient (frozen position encoder), none is computed and dtheta is returned as None."""
    T = q.shape[0]
    hd = q.shape[1] // H
    assert q.shape[1] == H * hd and theta.shape == (T, hd // 2), (tuple(q.shape), tuple(theta.shape), H)
    dq, dk, dv = (g.contiguous() for g in (dq, dk, dv))
    dqkv = torch.empty(T, H * 3 * hd, device=q.device, dtype=q.dtype)
    if dtheta is None and need_dtheta:
        dtheta = torch.zeros_like(theta)
    args = (ptr(dq), ptr(dk), ptr(dv), ptr(q), ptr(k), ptr(theta), ptr(dqkv), ptr(dtheta), T, H, _code(q.dtype))
    if hd == 64:
        call("lgb200_rope_split_bwd", *args, stream_ptr())
    else:
        call("lgb200_rope_split_bwd_hd", *args, hd, stream_ptr())
    return dqkv, dtheta


# ------------------------------------------------------------------------------------------------
# attention (lightglue.py:118-121, 207-216)
# ------------------------------------------------------------------------------------------------
def _head_dim(q):
    D = q.shape[3]
    assert D in (32, 64), "head_dim must be 32 or 64"
    return D


def attn_fwd(q, k, v, kv_shift, scale):
    _chk(q), _chk(k), _chk(v)
    B, Nq, H, _ = q.shape
    D = _head_dim(q)
    Nk = k.shape[1]
    out = torch.empty_like(q)
    lse = torch.empty(B, H, Nq, device=q.device, dtype=torch.float32)
    args = (ptr(q), ptr(k), ptr(v), ptr(out), ptr(lse), B, Nq, Nk, H, kv_shift, float(scale), _code(q.dtype))
    if D == 64:
        call("lgb200_attn_fwd", *args, stream_ptr())
    else:
        call("lgb200_attn_fwd_hd", *args, D, stream_ptr())
    return out, lse


def attn_fwd_varlen(q, k, v, q_off, q_len, k_off, k_len, max_q_len, scale, out=None):
    """Forward over packed sequences: q [Tq, H, D], k / v [Tk, H, D] token-major; sequence s has the queries
    q_off[s] .. q_off[s] + q_len[s] - 1 and the keys k_off[s] .. k_off[s] + k_len[s] - 1 (int32 CUDA tensors of S
    entries, never read on the host); max_q_len bounds every q_len.  Returns (out [Tq, H, D], lse [H, Tq]); only the
    query rows of the sequences are written, so `out` (allocated when None) keeps its other rows."""
    _chk(q), _chk(k), _chk(v)
    Tq, H, D = q.shape
    assert D in (32, 64), "head_dim must be 32 or 64"
    assert k.shape[1:] == q.shape[1:] and v.shape == k.shape and k.dtype == q.dtype == v.dtype
    seqs = [_chk(t, torch.int32) for t in (q_off, q_len, k_off, k_len)]
    S = q_off.numel()
    assert all(t.numel() == S for t in seqs)
    out = torch.empty_like(q) if out is None else _chk(out, q.dtype)
    assert out.shape == q.shape
    lse = torch.empty(H, Tq, device=q.device, dtype=torch.float32)
    call("lgb200_attn_fwd_varlen", ptr(q), ptr(k), ptr(v), ptr(out), ptr(lse), *(ptr(t) for t in seqs), S,
         int(max_q_len), Tq, k.shape[0], H, float(scale), _code(q.dtype), D, stream_ptr())
    return out, lse


def attn_bwd(q, k, v, out, lse, dout, kv_shift, scale):
    B, Nq, H, _ = q.shape
    D = _head_dim(q)
    Nk = k.shape[1]
    dout = dout.contiguous()
    dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    delta = torch.empty(_lib.load().lgb200_attn_bwd_ws_floats(B, Nq, Nk, H), device=q.device, dtype=torch.float32)
    args = (ptr(q), ptr(k), ptr(v), ptr(out), ptr(lse), ptr(dout), ptr(dq), ptr(dk), ptr(dv), ptr(delta), B, Nq, Nk,
            H, kv_shift, float(scale), _code(q.dtype))
    if D == 64:
        call("lgb200_attn_bwd", *args, stream_ptr())
    else:
        call("lgb200_attn_bwd_hd", *args, D, stream_ptr())
    return dq, dk, dv


def attn_bwd_shared_qk(qk, v, out, lse, dout, scale):
    """Backward of the cross-attention whose query and key are the same tensor qk [2B,N,H,64] (batch b attends to
    batch (b + B) % 2B, lightglue.py:207-216).  Returns (dqk, dv) with dqk the total gradient dq + dk of qk.
    bf16: one pass over the shared similarity (lgb200_attn_bwd with q == k and dq == dk)."""
    B2 = qk.shape[0]
    if qk.dtype != torch.bfloat16:
        dq, dk, dv = attn_bwd(qk, qk, v, out, lse, dout, B2 // 2, scale)
        return dq.add_(dk), dv
    _, N, H, _ = qk.shape
    dout = dout.contiguous()
    dqk, dv = torch.empty_like(qk), torch.empty_like(v)
    delta = torch.empty(_lib.load().lgb200_attn_bwd_ws_floats(B2, N, N, H), device=qk.device, dtype=torch.float32)
    call("lgb200_attn_bwd", ptr(qk), ptr(qk), ptr(v), ptr(out), ptr(lse), ptr(dout), ptr(dqk), ptr(dqk), ptr(dv),
         ptr(delta), B2, N, N, H, B2 // 2, float(scale), _code(qk.dtype), stream_ptr(), launches=2)  # prep + sweep
    return dqk, dv


class Attention(torch.autograd.Function):
    """q [B,Nq,H,D], k,v [B,Nk,H,D] -> softmax(scale q k^T) v, keys of batch b taken from batch
    (b + kv_shift) % B.  Head dim D = 64 or 32, read from the shape."""

    @staticmethod
    def forward(ctx, q, k, v, kv_shift, scale):
        out, lse = attn_fwd(q, k, v, kv_shift, scale)
        ctx.save_for_backward(q, k, v, out, lse)
        ctx.meta = (kv_shift, float(scale))
        return out

    @staticmethod
    def backward(ctx, dout):
        q, k, v, out, lse = ctx.saved_tensors
        kv_shift, scale = ctx.meta
        dq, dk, dv = attn_bwd(q, k, v, out, lse, dout, kv_shift, scale)
        return dq, dk, dv, None, None


# ------------------------------------------------------------------------------------------------
# LayerNorm + GELU (lightglue.py:143-148)
# ------------------------------------------------------------------------------------------------
def ln_gelu_fwd(x, g, b, eps):
    """g, b fp32 contiguous. Returns y, mean, rstd."""
    _chk(x)
    T, W = x.shape
    y = torch.empty_like(x)
    mean = torch.empty(T, device=x.device, dtype=torch.float32)
    rstd = torch.empty_like(mean)
    call("lgb200_ln_gelu_fwd", ptr(x), ptr(g), ptr(b), ptr(y), ptr(mean), ptr(rstd), T, W, float(eps),
         _code(x.dtype), stream_ptr())
    return y, mean, rstd


def ln_gelu_bwd(dy, x, g, b, mean, rstd, want_dxsum=False):
    """Returns dx, dgamma, dbeta (and, on request, the column sums of dx = bias gradient of the Linear before)."""
    T, W = x.shape
    dy = dy.contiguous()
    dx = torch.empty_like(x)
    parts = _lib.load().lgb200_ln_gelu_bwd_parts(T)
    red = torch.empty(3, parts, W, device=x.device, dtype=torch.float32)
    call("lgb200_ln_gelu_bwd", ptr(dy), ptr(x), ptr(g), ptr(b), ptr(mean), ptr(rstd), ptr(dx), ptr(red[0]), ptr(red[1]),
         ptr(red[2]), T, W, _code(x.dtype), stream_ptr())
    sums = red.sum(1)  # one reduction for the three partial sets
    if want_dxsum:
        return dx, sums[0], sums[1], sums[2]
    return dx, sums[0], sums[1]


_colsum_counters = {}


class PosencTheta(torch.autograd.Function):
    """theta = kp Wr^T (lightglue.py:37-44; kp [T, 2|4] fp32, Wr [C, kd], C = head_dim / 2 = 32 or 16); the weight
    gradient -- a [C,T] x [T,kd] contraction over all tokens -- runs as one streaming kernel + a 296-row sum instead of
    a split-K sgemm."""

    @staticmethod
    def forward(ctx, kp, weight):
        ctx.save_for_backward(kp)
        return kp @ weight.t()

    @staticmethod
    def backward(ctx, g):
        (kp,) = ctx.saved_tensors
        T, C = g.shape
        kd = kp.shape[1]
        if C not in (16, 32) or kd > 4 or not g.is_cuda:
            return None, g.t() @ kp
        g = g.contiguous()
        nb = _lib.load().lgb200_posenc_wgrad_blocks()
        part = torch.empty(nb, C, kd, device=g.device, dtype=torch.float32)
        call("lgb200_posenc_wgrad", ptr(g), ptr(kp), ptr(part), T, C, kd, stream_ptr())
        return None, part.sum(0)


def mask_counts(mask_u8):
    """0/1 byte mask [B,M,N] -> (rowcnt [B,M], colcnt [B,N]) fp32, one pass (lgb200_mask_counts); shapes the kernel does
    not take (N not a multiple of 16, N > 4096) use the two torch reductions."""
    B, M, N = mask_u8.shape
    if N % 16 or N > 4096 or not mask_u8.is_contiguous() or mask_u8.data_ptr() % 16 or not mask_u8.is_cuda:
        return mask_u8.sum(2, dtype=torch.float32), mask_u8.sum(1, dtype=torch.float32)
    rowcnt = torch.empty(B, M, device=mask_u8.device, dtype=torch.float32)
    colcnt = torch.empty(B, N, device=mask_u8.device, dtype=torch.float32)
    call("lgb200_mask_counts", ptr(mask_u8), ptr(rowcnt), ptr(colcnt), B, M, N, stream_ptr())
    return rowcnt, colcnt


def _colsum_counter(dev, cols):
    """Self-resetting arrival counters of the column-sum kernels, zeroed once per device."""
    cnt = _colsum_counters.get(dev)
    if cnt is None:
        cnt = _colsum_counters[dev] = torch.zeros(64, device=dev, dtype=torch.int32)
    assert cols <= 64 * 64
    return cnt


def colsum(a):
    """[rows, cols] (fp32 / bf16) -> fp32 [cols] column sums (bias gradients); one launch."""
    _chk(a)
    rows, cols = a.shape
    if cols % 8:
        return a.sum(0, dtype=torch.float32)
    dev = a.device
    cnt = _colsum_counter(dev, cols)
    out = torch.empty(cols, device=dev, dtype=torch.float32)
    ws = torch.empty(_lib.load().lgb200_colsum_slabs(rows, cols) * cols, device=dev, dtype=torch.float32)
    call("lgb200_colsum", ptr(a), ptr(out), ptr(ws), ptr(cnt), rows, cols, _code(a.dtype), stream_ptr())
    return out


# ------------------------------------------------------------------------------------------------
# BatchNorm1d + ReLU (GlueStick MLPs, gluestick.py:465-475), statistics optionally summed across ranks
# ------------------------------------------------------------------------------------------------
def _bn_ws(T, C, dev):
    return torch.empty(_lib.load().lgb200_colsum_slabs(T, C) * 2 * C, device=dev, dtype=torch.float64)


def bn_stats(x):
    """x [T, C] -> fp64 [2C+1] = [sum x | sum x^2 | T] per channel (lgb200_bn_stats)."""
    _chk(x)
    T, C = x.shape
    sums = torch.empty(2 * C + 1, device=x.device, dtype=torch.float64)
    # both held until the launch: a temporary freed inside the argument list could be handed to the other
    cnt, ws = _colsum_counter(x.device, C), _bn_ws(T, C, x.device)
    call("lgb200_bn_stats", ptr(x), ptr(sums), ptr(ws), ptr(cnt), T, C, _code(x.dtype), stream_ptr())
    return sums


def bn_relu_fwd(x, sums, weight, bias, running_mean, running_var, momentum, eps):
    """y = relu(batch_norm(x)) with the statistics in `sums` (bn_stats, possibly summed across ranks; the running
    statistics are updated in place) or, when sums is None, the running statistics.  Returns y, mean, rstd [C]."""
    _chk(x), _chk(weight, torch.float32), _chk(bias, torch.float32)
    for t in (running_mean, running_var):
        if t is not None:
            _chk(t, torch.float32)
    T, C = x.shape
    y = torch.empty_like(x)
    mean = torch.empty(C, device=x.device, dtype=torch.float32)
    rstd = torch.empty_like(mean)
    call("lgb200_bn_relu_fwd", ptr(x), ptr(sums), ptr(weight), ptr(bias), ptr(running_mean), ptr(running_var),
         float(momentum), float(eps), ptr(y), ptr(mean), ptr(rstd), T, C, _code(x.dtype), stream_ptr())
    return y, mean, rstd


def bn_relu_bwd_reduce(dy, x, weight, bias, mean, rstd):
    """fp64 [2C] = [sum dy' | sum dy' xhat] with dy' = dy [relu output > 0]: dbeta and dgamma of these rows."""
    _chk(dy, x.dtype), _chk(x)
    T, C = x.shape
    sums = torch.empty(2 * C, device=x.device, dtype=torch.float64)
    cnt, ws = _colsum_counter(x.device, C), _bn_ws(T, C, x.device)
    call("lgb200_bn_relu_bwd_reduce", ptr(dy), ptr(x), ptr(weight), ptr(bias), ptr(mean), ptr(rstd), ptr(sums), ptr(ws),
         ptr(cnt), T, C, _code(x.dtype), stream_ptr())
    return sums


def bn_relu_bwd(dy, x, weight, bias, mean, rstd, sums, count):
    """dx from the (possibly summed across ranks) backward sums and the count behind the forward statistics (a 1-element
    fp64 view); sums = count = None: eval mode."""
    _chk(dy, x.dtype), _chk(x)
    T, C = x.shape
    dx = torch.empty_like(x)
    call("lgb200_bn_relu_bwd", ptr(dy), ptr(x), ptr(weight), ptr(bias), ptr(mean), ptr(rstd), ptr(sums), ptr(count),
         ptr(dx), T, C, _code(x.dtype), stream_ptr())
    return dx


class BnRelu(torch.autograd.Function):
    """relu(batch_norm(x)) on token-major x [T, C] (fp32 or bf16, C a power of two <= 512), statistics over all T rows.
    `exchange`: None, or a callable that sums an fp64 vector in place over the ranks that share the statistics; it is
    called once in forward on [sum x | sum x^2 | count] and once in backward on [sum dy' | sum dy' xhat].  dgamma and
    dbeta come from this rank's sums (the gradient all-reduce adds the other ranks'), dx from the exchanged ones."""

    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, training, momentum, eps, exchange, saved=None):
        x = x.contiguous()
        w, b = weight.detach().float().contiguous(), bias.detach().float().contiguous()
        sums = None
        if training:
            if exchange is None and x.shape[0] < 2:
                raise ValueError(f"Expected more than 1 value per channel when training, got input size {tuple(x.shape)}")
            sums = bn_stats(x)
            if exchange is not None:
                exchange(sums)
            if saved is not None:
                saved.append(sums)
        y, mean, rstd = bn_relu_fwd(x, sums, w, b, running_mean, running_var, momentum, eps)
        ctx.save_for_backward(x, w, b, mean, rstd, sums)
        ctx.exchange = exchange
        return y

    @staticmethod
    def backward(ctx, dy):
        x, w, b, mean, rstd, sums = ctx.saved_tensors
        dy = dy.to(x.dtype).contiguous()
        C = x.shape[1]
        red = bn_relu_bwd_reduce(dy, x, w, b, mean, rstd)
        dbeta, dgamma = red[:C].float(), red[C:].float()  # copies: taken before the exchange
        count = None
        if sums is not None:
            if ctx.exchange is not None:
                ctx.exchange(red)
            count = sums[2 * C:]
        dx = bn_relu_bwd(dy, x, w, b, mean, rstd, red if sums is not None else None, count)
        return dx, dgamma, dbeta, None, None, None, None, None, None, None


def bn_running_update(sums, bn):
    """One more training-mode running-statistics step of BatchNorm `bn` from the batch statistics `sums` of an earlier
    call (bn_stats layout, after any exchange), the same formula as bn_relu_fwd's; num_batches_tracked += 1."""
    C = bn.running_mean.numel()
    _chk(sums, torch.float64), _chk(bn.running_mean, torch.float32), _chk(bn.running_var, torch.float32)
    assert sums.numel() == 2 * C + 1
    call("lgb200_bn_running_update", ptr(sums), ptr(bn.running_mean), ptr(bn.running_var), float(bn.momentum), C,
         stream_ptr())
    bn.num_batches_tracked.add_(1)


def bn_exchange(bn):
    """The cross-rank sum for the statistics of BatchNorm module `bn`: an in-place all_reduce over its process group
    (WORLD when unset) when it is a training nn.SyncBatchNorm and that group has more than one rank, else None."""
    import torch.distributed as dist

    if not (isinstance(bn, torch.nn.SyncBatchNorm) and bn.training and dist.is_available() and dist.is_initialized()):
        return None
    group = bn.process_group if bn.process_group is not None else dist.group.WORLD
    if dist.get_world_size(group) < 2:
        return None
    return lambda t: dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group)


def batchnorm_relu(x, bn, exchange=None, saved=None):
    """relu(bn(x)) for an nn.BatchNorm1d / nn.SyncBatchNorm `bn` on token-major x [T, C], with the module's semantics:
    batch statistics in training mode (or without running statistics), running statistics in eval mode; a training call
    updates running_mean / running_var and num_batches_tracked.  `exchange` as in BnRelu (see bn_exchange).
    `saved`: None or a list that receives the batch statistics a training call used (see bn_running_update)."""
    if bn.momentum is None or not bn.affine:
        raise NotImplementedError("gluefactory_b200 batchnorm_relu: momentum=None and affine=False are not built")
    rm, rv = (bn.running_mean, bn.running_var) if bn.track_running_stats else (None, None)
    if bn.training and bn.track_running_stats:
        bn.num_batches_tracked.add_(1)
    return BnRelu.apply(x, bn.weight, bn.bias, rm, rv, bn.training or rm is None, bn.momentum, bn.eps, exchange, saved)


def residual_add_cast(x, y, cdt, want_sum=True, out_cast=None):
    """x fp32 [.., D] + y (compute dtype or None) -> (x_new fp32 or None, cast(x_new) in cdt).
    cdt None: only the fp32 sum is produced (y gives the kernel's element type).
    out_cast: optional destination for the cast copy, a [rows, D] column block (unit inner stride) of a wider matrix."""
    _chk(x, torch.float32)
    xo = torch.empty_like(x) if (want_sum and y is not None) else None
    if out_cast is not None:
        _chk(out_cast, cdt, strided_rows=True)
        rows, cols = out_cast.shape
        assert x.numel() == rows * cols
        call("lgb200_residual_add_cast_pitched", ptr(x), ptr(y), ptr(xo), ptr(out_cast), rows, cols, out_cast.stride(0),
             _code(cdt), stream_ptr())
        return (xo if xo is not None else x), out_cast
    xc = torch.empty(x.shape, device=x.device, dtype=cdt) if cdt is not None else None
    call("lgb200_residual_add_cast", ptr(x), ptr(y), ptr(xo), ptr(xc), x.numel(),
         _code(cdt if cdt is not None else y.dtype), stream_ptr())
    return (xo if xo is not None else x), xc


def add_f32_cast_(x, y, cdt):
    """x += y (both fp32, in place) and the compute-dtype copy of the sum, one pass (lgb200_add_f32_cast)."""
    _chk(x, torch.float32), _chk(y, torch.float32)
    assert x.shape == y.shape
    xc = torch.empty(x.shape, device=x.device, dtype=cdt)
    call("lgb200_add_f32_cast", ptr(x), ptr(y), ptr(x), ptr(xc), x.numel(), _code(cdt), stream_ptr())
    return x, xc


def gluestick_attention(query, key, value):
    """GlueStick's attention core (models/matchers/gluestick.py:524-529) on the same kernels: query [B, dh, H, N],
    key/value [B, dh, H, M] (channels first, channel = d * H + h) -> [B, dh, H, N], head dim dh = 64 or 32.  The
    reference forces fp32 here (AMP_CUSTOM_FWD_F32): fp32 inputs run the full-precision kernels, bf16 inputs the
    wgmma ones."""
    dh = query.shape[1]
    assert dh in (32, 64), "head dimension 32 or 64 only"
    tm = lambda t: t.permute(0, 3, 2, 1).contiguous()  # noqa: E731  -> token-major [B, N, H, dh]
    out = Attention.apply(tm(query), tm(key), tm(value), 0, dh ** -0.5)
    return out.permute(0, 3, 2, 1)


# ------------------------------------------------------------------------------------------------
# batched GEMM on wgmma (lightglue.py:283)
# ------------------------------------------------------------------------------------------------
def gemm_bf16(a, b, a_mn_major=False, b_mn_major=False, out_dtype=torch.float32, alpha=1.0):
    """C[i] = opA(a[i]) @ opB(b[i])^T-style contraction on the tensor cores (see lgb200.h).
    a: [batch, M, K] (or [batch, K, M] when a_mn_major); b: [batch, N, K] (or [batch, K, N])."""
    _chk(a, torch.bfloat16), _chk(b, torch.bfloat16)
    batch = a.shape[0]
    M, K = (a.shape[2], a.shape[1]) if a_mn_major else (a.shape[1], a.shape[2])
    N, Kb = (b.shape[2], b.shape[1]) if b_mn_major else (b.shape[1], b.shape[2])
    assert K == Kb and b.shape[0] == batch
    c = torch.empty(batch, M, N, device=a.device, dtype=out_dtype)
    call("lgb200_gemm_bf16", ptr(a), ptr(b), ptr(c), batch, M, N, K, int(a_mn_major), int(b_mn_major),
         a.shape[2], b.shape[2], N, a.shape[1] * a.shape[2], b.shape[1] * b.shape[2], M * N, _code(out_dtype),
         float(alpha), stream_ptr())
    return c


def linear(a, w, bias=None, out=None, out_dtype=torch.bfloat16, w_is_kn=False, accumulate=False, alpha=1.0):
    """The nn.Linear-shaped GEMMs of the layer on the persistent wgmma kernel (lgb200_linear, include/lgb200.h):
        out[M, N] (=|+=) alpha * a[M, K] @ W^T + bias,   W = w[N, K]  (forward: y = x W^T + b)
                                                     or  W^T = w[K, N] when w_is_kn (dgrad: dx = dy W, w = the [out, in] weight)
    a, w bf16 2-D with unit inner stride (row-strided views are fine: column blocks of wider matrices);
    bias fp32 [N]; out may be a row-strided view; accumulate=True adds into an fp32 `out` (TMA reduce-add)."""
    _chk(a, torch.bfloat16, strided_rows=True), _chk(w, torch.bfloat16, strided_rows=True)
    M, K = a.shape
    N = w.shape[1] if w_is_kn else w.shape[0]
    assert (w.shape[0] if w_is_kn else w.shape[1]) == K, (a.shape, w.shape, w_is_kn)
    if out is None:
        assert not accumulate
        out = torch.empty(M, N, device=a.device, dtype=out_dtype)
    else:
        assert out.shape == (M, N) and out.stride(1) == 1
    if accumulate:
        assert out.dtype == torch.float32
    if bias is not None:
        _chk(bias, torch.float32)
        assert bias.numel() == N
    call("lgb200_linear", ptr(a), ptr(w), ptr(out), ptr(bias), M, N, K, 0, int(w_is_kn), a.stride(0), w.stride(0),
         out.stride(0), _code(out.dtype), float(alpha), int(accumulate), stream_ptr())
    return out


class LinearFn(torch.autograd.Function):
    """nn.Linear on the library's GEMMs with autograd: x [T, in] bf16, weight [out, in] / bias [out] fp32 parameters.
    forward y = x W^T + b (bf16 out, fp32 bias in the epilogue); backward dgrad (bf16), split-K wgrad (fp32), bias
    gradient by the column-sum kernel; the weight and bias gradients of a frozen (requires_grad=False) weight or bias
    are not computed.  Used for LightGlue's input_proj and dense final head in bf16, and for GlueStick's and
    SuperGlue's 1x1 convolutions."""

    @staticmethod
    def forward(ctx, x, weight, bias):
        w16 = weight.detach().to(torch.bfloat16)
        ctx.save_for_backward(x, w16)
        return linear(x, w16, bias.detach().float().contiguous())

    @staticmethod
    def backward(ctx, dy):
        x, w16 = ctx.saved_tensors
        dy = dy.contiguous()
        need = ctx.needs_input_grad
        dx = linear(dy, w16, w_is_kn=True) if need[0] else None
        return dx, wgrad_bf16(dy, x) if need[1] else None, colsum(dy) if need[2] else None


# ------------------------------------------------------------------------------------------------
# assignment head (lightglue.py:256-290, losses.py)
# ------------------------------------------------------------------------------------------------
def assign_stats(sim, ls0, ls1, dust0, dust1, gt_u8=None, dense=False):
    """Runs the two assignment passes on sim [B,M,N].  Returns a dict with lse_row/lse_col,
    rowmax/rowarg/colmax/colarg (int32, dustbin excluded), optional pos_row_sum, and when
    `dense` the full scores [B,M+1,N+1] and row_expsum."""
    _chk(sim, torch.float32)
    B, M, N = sim.shape
    dev = sim.device
    f = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)  # noqa: E731
    lse_row, lse_col = f(B, M), f(B, N)
    ws = torch.empty(_lib.load().lgb200_assign_ws_bytes(B, M, N), device=dev, dtype=torch.uint8)
    call("lgb200_assign_lse", ptr(sim), ptr(lse_row), ptr(lse_col), ptr(ws), B, M, N, stream_ptr())
    out = {"lse_row": lse_row, "lse_col": lse_col, "rowmax": f(B, M), "colmax": f(B, N),
           "rowarg": torch.empty(B, M, device=dev, dtype=torch.int32),
           "colarg": torch.empty(B, N, device=dev, dtype=torch.int32)}
    scores = f(B, M + 1, N + 1) if dense else None
    row_expsum = f(B, M) if dense else None
    pos_row_sum = f(B, M) if gt_u8 is not None else None
    ls0, ls1, dust0, dust1 = (t.detach().float().contiguous() for t in (ls0, ls1, dust0, dust1))
    call("lgb200_assign_scores", ptr(sim), ptr(lse_row), ptr(lse_col), ptr(ls0), ptr(ls1), ptr(dust0), ptr(dust1),
         ptr(gt_u8), ptr(scores), ptr(out["rowmax"]), ptr(out["rowarg"]), ptr(out["colmax"]), ptr(out["colarg"]),
         ptr(pos_row_sum), ptr(row_expsum), ptr(ws), B, M, N, stream_ptr())
    out.update(scores=scores, row_expsum=row_expsum, pos_row_sum=pos_row_sum)
    return out


def assign_fused_ok(md, D):
    """The fused GEMM + assignment kernels take bf16 descriptors of width 64..256 (multiple of 64)."""
    return md.dtype == torch.bfloat16 and D % 64 == 0 and 64 <= D <= 256


def assign_fused_stats(md0, md1, alpha, ls0, ls1, gt_u8=None):
    """md0 [B,M,D], md1 [B,N,D] bf16 -> the same dict as assign_stats(dense=False) (lse_row/lse_col, rowmax/rowarg,
    colmax/colarg, pos_row_sum) without ever writing sim = alpha md0 md1^T (csrc/assign_tc.cu: two passes, each a
    wgmma GEMM whose accumulator tiles are reduced in the epilogue)."""
    _chk(md0, torch.bfloat16), _chk(md1, torch.bfloat16)
    B, M, D = md0.shape
    N = md1.shape[1]
    dev = md0.device
    f = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)  # noqa: E731
    out = {"lse_row": f(B, M), "lse_col": f(B, N), "rowmax": f(B, M), "colmax": f(B, N),
           "rowarg": torch.empty(B, M, device=dev, dtype=torch.int32),
           "colarg": torch.empty(B, N, device=dev, dtype=torch.int32),
           "pos_row_sum": f(B, M) if gt_u8 is not None else None, "scores": None, "row_expsum": None}
    call("lgb200_assign_fused_lse", ptr(md0), ptr(md1), float(alpha), ptr(out["lse_row"]), ptr(out["lse_col"]), B, M, N, D,
         stream_ptr())
    ls0, ls1 = (t.detach().float().contiguous() for t in (ls0, ls1))
    call("lgb200_assign_fused_stats", ptr(md0), ptr(md1), float(alpha), ptr(out["lse_row"]), ptr(out["lse_col"]), ptr(ls0),
         ptr(ls1), ptr(gt_u8), ptr(out["rowmax"]), ptr(out["rowarg"]), ptr(out["colmax"]), ptr(out["colarg"]),
         ptr(out["pos_row_sum"]), B, M, N, D, stream_ptr())
    return out


def assign_fused_bwd(md0, md1, alpha, lse_row, lse_col, gt_u8, gt_t_u8, gcoef, rowcnt, colcnt, dmd0, dmd1):
    """d(mdesc0), d(mdesc1) (bf16, written into dmd0 [B*M, D] / dmd1 [B*N, D]) of the NLL through sim: dsim is
    recomputed per tile from the two LSE vectors and contracted with the other image's descriptors in the same kernel.
    gt_u8 = gt_t_u8 = None (labels as match lists): without the positive term, which assign_pos_bwd then adds."""
    B, M, D = md0.shape
    N = md1.shape[1]
    for t in (lse_row, lse_col, gcoef, rowcnt, colcnt):
        _chk(t, torch.float32)
    if gt_u8 is not None or gt_t_u8 is not None:
        _chk(gt_u8), _chk(gt_t_u8)
    _chk(dmd0, torch.bfloat16), _chk(dmd1, torch.bfloat16)
    call("lgb200_assign_fused_bwd", ptr(md0), ptr(md1), float(alpha), ptr(lse_row), ptr(lse_col), ptr(gt_u8), ptr(gt_t_u8),
         ptr(gcoef), ptr(rowcnt), ptr(colcnt), ptr(dmd0), ptr(dmd1), B, M, N, D, stream_ptr())


def match_list_counts(gt0, gt1):
    """Labels as match lists gt0 [B,M] / gt1 [B,N] (one-to-one; -1 unmatched, -2 ignored) -> (rowcnt [B,M] = (gt0 >= 0),
    colcnt [B,N] = (gt1 >= 0) as fp32, num_pos [B] = the positives clamped at 1).  num_pos is NaN for a pair whose two
    lists hold different numbers of positives; with the per-row check gt1[gt0[i]] == i that the loss kernels make, equal
    counts mean the lists agree (gt1[j] = i <=> gt0[i] = j).  Device ops only: no host read."""
    rowcnt, colcnt = (gt0 >= 0).float(), (gt1 >= 0).float()
    n0, n1 = rowcnt.sum(1), colcnt.sum(1)
    num_pos = torch.where(n0 == n1, n0, torch.full_like(n0, float("nan"))).clamp(min=1.0)
    return rowcnt.contiguous(), colcnt.contiguous(), num_pos.contiguous()


def assign_pos_fwd(gt0, gt1, lse_row, lse_col, alpha, md0=None, md1=None, sim=None):
    """pos_row_sum [B,M] of match-list labels (lgb200_assign_pos_fwd): the positive entry of row i, j = gt0[i],
    from sim [B,M,N] fp32 ((sim - lse_row) + (sim - lse_col), as assign_stats computes it from the mask) or from the
    bf16 descriptors md0 [B,M,D] / md1 [B,N,D] (2 alpha md0_i . md1_j - lse_row_i - lse_col_j); 0 without a positive,
    NaN where the lists disagree."""
    _chk(gt0, torch.int64), _chk(gt1, torch.int64), _chk(lse_row, torch.float32), _chk(lse_col, torch.float32)
    B, M = gt0.shape
    N = gt1.shape[1]
    D = 0
    if sim is not None:
        _chk(sim, torch.float32)
        assert sim.shape == (B, M, N)
    else:
        _chk(md0, torch.bfloat16), _chk(md1, torch.bfloat16)
        D = md0.shape[2]
        assert md0.shape == (B, M, D) and md1.shape == (B, N, D)
    out = torch.empty(B, M, device=gt0.device, dtype=torch.float32)
    call("lgb200_assign_pos_fwd", ptr(md0), ptr(md1), ptr(sim), float(alpha), ptr(lse_row), ptr(lse_col), ptr(gt0),
         ptr(gt1), ptr(out), B, M, N, D, stream_ptr())
    return out


def assign_pos_bwd(md0, md1, gcoef, gt0, gt1, dmd0, dmd1):
    """dmd0 [B*M, D] += 2 gcoef_b md1[gt0[i]], dmd1 [B*N, D] += 2 gcoef_b md0[gt1[j]] in place (bf16;
    lgb200_assign_pos_bwd): the positive term that assign_fused_bwd leaves out without masks."""
    _chk(md0, torch.bfloat16), _chk(md1, torch.bfloat16), _chk(gcoef, torch.float32)
    _chk(gt0, torch.int64), _chk(gt1, torch.int64), _chk(dmd0, torch.bfloat16), _chk(dmd1, torch.bfloat16)
    B, M, D = md0.shape
    N = md1.shape[1]
    assert gt0.shape == (B, M) and gt1.shape == (B, N) and dmd0.numel() == B * M * D and dmd1.numel() == B * N * D
    call("lgb200_assign_pos_bwd", ptr(md0), ptr(md1), ptr(gcoef), ptr(gt0), ptr(gt1), ptr(dmd0), ptr(dmd1), B, M, N, D,
         stream_ptr())


def head_logsig(zt):
    T = zt.shape[0]
    ls = torch.empty(T, device=zt.device, dtype=torch.float32)
    du = torch.empty_like(ls)
    call("lgb200_head_logsig", ptr(zt), ptr(ls), ptr(du), T, stream_ptr())
    return ls, du


def wgrad_bf16(dy, a, out=None):
    """dW [out, in] fp32 = dy^T a for bf16 dy [T, out], a [T, in] (rows may be strided views with unit inner stride):
    split-K wgmma GEMM with both operands consumed MN-major, i.e. exactly as they lie in memory."""
    _chk(dy, torch.bfloat16, strided_rows=True), _chk(a, torch.bfloat16, strided_rows=True)
    T, M = dy.shape
    N = a.shape[1]
    assert a.shape[0] == T
    if out is None:
        out = torch.empty(M, N, device=dy.device, dtype=torch.float32)
    assert out.stride(1) == 1
    ws = torch.empty(_lib.load().lgb200_gemm_splitk_ws_floats(M, N, T), device=dy.device, dtype=torch.float32)
    call("lgb200_gemm_bf16_splitk", ptr(dy), ptr(a), ptr(out), M, N, T, 1, 1, dy.stride(0), a.stride(0), out.stride(0),
         ptr(ws), stream_ptr())
    return out


def gt_matches_from_homography(kp0, kp1, H, pos_th=3.0, neg_th=6.0, dense=True, dense_t=False):
    """Device-side gt_matches_from_homography (geometry/gt_generation.py:109-161; defaults as the reference's).
    kp0 [B,M,2], kp1 [B,N,2] pixel coordinates, H [B,3,3] -> dict with `assignment` (bool [B,M,N], omitted when
    dense=False), `matches0/1` (int64: index, -1 unmatched, -2 ignored), `matching_scores0/1`, `proj_0to1/1to0`.
    The dense `reward` map of the reference is not produced (no consumer on the matcher's path)."""
    from .geometry import inv3x3, warp_points

    kp0, kp1 = kp0.float().contiguous(), kp1.float().contiguous()
    _chk(kp0, torch.float32), _chk(kp1, torch.float32)
    B = kp0.shape[0]
    Hm = H.float().expand(B, 3, 3) if H.dim() == 2 else H.float()
    kp0_1 = warp_points(kp0, Hm).contiguous()  # O(M+N): homography.py:161-180
    kp1_0 = warp_points(kp1, inv3x3(Hm)).contiguous()
    out = gt_matches_from_reprojection(kp0, kp1, kp0_1, kp1_0, pos_th=pos_th, neg_th=neg_th, dense=dense, dense_t=dense_t)
    m0, m1 = out["matches0"], out["matches1"]
    out.update({"matching_scores0": (m0 > -1).float(), "matching_scores1": (m1 > -1).float(), "proj_0to1": kp0_1,
                "proj_1to0": kp1_0})
    return out


def gt_matches_from_reprojection(kp0, kp1, kp0_1, kp1_0, visible0=None, visible1=None, valid0=None, valid1=None,
                                 pos_th=3.0, neg_th=5.0, dense=True, dense_t=False):
    """The O(M N) label pass of gt_matches_from_pose_depth (geometry/gt_generation.py:47-74) for given reprojections:
    kp0_1 = view-0 keypoints projected into view 1, kp1_0 the converse, visibility / depth-validity masks [B,M] /
    [B,N] (bool; None = all true).  Returns assignment (bool [B,M,N] when dense), matches0/1 (int64: index, -1, -2)."""
    kp0, kp1, kp0_1, kp1_0 = (t.float().contiguous() for t in (kp0, kp1, kp0_1, kp1_0))
    B, M = kp0.shape[:2]
    N = kp1.shape[1]
    dev = kp0.device
    u8 = lambda t: None if t is None else t.to(torch.uint8).contiguous()  # noqa: E731
    vis0, vis1, val0, val1 = u8(visible0), u8(visible1), u8(valid0), u8(valid1)
    m0 = torch.empty(B, M, device=dev, dtype=torch.int64)
    m1 = torch.empty(B, N, device=dev, dtype=torch.int64)
    asg = torch.empty(B, M, N, device=dev, dtype=torch.bool) if dense else None
    asg_t = torch.empty(B, N, M, device=dev, dtype=torch.bool) if dense_t else None
    ws = torch.empty(_lib.load().lgb200_gt_homography_ws_bytes(B, M, N), device=dev, dtype=torch.uint8)
    call("lgb200_gt_from_reprojection", ptr(kp0), ptr(kp1), ptr(kp0_1), ptr(kp1_0), ptr(vis0), ptr(vis1), ptr(val0),
         ptr(val1), float(pos_th), float(neg_th), ptr(m0), ptr(m1), ptr(asg), ptr(asg_t), ptr(ws), B, M, N, stream_ptr())
    out = {"matches0": m0, "matches1": m1}
    if dense:
        out["assignment"] = asg
    if dense_t:
        out["assignment_t"] = asg_t  # [B,N,M]: the same mask transposed (read by the fused assignment backward)
    return out


def gt_epipolar_unmatched_(kp0, kp1, F, valid0, valid1, m0, m1, th):
    """In-place epipolar exclusion of gt_matches_from_pose_depth (gt_generation.py:82-90) on matches0 / matches1."""
    kp0, kp1, F = kp0.float().contiguous(), kp1.float().contiguous(), F.float().contiguous()
    B, M = kp0.shape[:2]
    N = kp1.shape[1]
    v0, v1 = valid0.to(torch.uint8).contiguous(), valid1.to(torch.uint8).contiguous()
    _chk(m0, torch.int64), _chk(m1, torch.int64)
    ws = torch.empty(B * (M + N), device=kp0.device, dtype=torch.uint8)
    call("lgb200_gt_epipolar_unmatched", ptr(kp0), ptr(kp1), ptr(F), ptr(v0), ptr(v1), float(th), ptr(m0), ptr(m1), ptr(ws),
         B, M, N, stream_ptr())


def line_segments(lines, h, w):
    """Lines [B,L,2,2], [B,L,4] or [B,L,K,2] (first and last point) -> [B,L,4] fp32 segments clamped to [0, w-1] x
    [0, h-1] (geometry/gt_generation.py:430-448)."""
    if lines.shape[-2:] == (2, 2):
        lines = lines.flatten(-2)
    elif lines.dim() == 4:
        lines = torch.cat([lines[:, :, 0], lines[:, :, -1]], dim=2)
    if lines.shape[1] == 0:
        raise ValueError("line ground truth needs at least one line per view")
    x, y = lines.float()[..., 0::2].clamp(0, w - 1), lines.float()[..., 1::2].clamp(0, h - 1)  # no host tensor: capturable
    return torch.stack([x[..., 0], y[..., 0], x[..., 1], y[..., 1]], -1).contiguous()


def sample_line_points(segs, npts):
    """segs [B,L,4] -> [B, L*npts, 2]: npts points evenly spaced from start to end (sample_pts, :164-170)."""
    _chk(segs, torch.float32)
    B, L = segs.shape[:2]
    pts = torch.empty(B, L * npts, 2, device=segs.device, dtype=torch.float32)
    call("lgb200_gt_line_sample", ptr(segs), ptr(pts), B, L, int(npts), stream_ptr())
    return pts


def linear_sum_assignment(cost):
    """cost [B,rows,cols] float64 (finite) -> (row2col [B,rows], col2row [B,cols]) int32, -1 where unassigned: the
    minimum-cost assignment scipy.optimize.linear_sum_assignment returns for each matrix, ties included."""
    cost = _chk(cost.contiguous(), torch.float64)
    B, R, C = cost.shape
    row2col = torch.empty(B, R, device=cost.device, dtype=torch.int32)
    col2row = torch.empty(B, C, device=cost.device, dtype=torch.int32)
    call("lgb200_lsap", ptr(cost), ptr(row2col), ptr(col2row), B, R, C, stream_ptr())
    return row2col, col2row


def gt_line_matches_from_projection(segs0, segs1, pts0_1, pts1_0, size0, size1, valid_lines0, valid_lines1,
                                    visible0=None, visible1=None, valid_pts0=None, valid_pts1=None, npts=50, dist_th=5,
                                    overlap_th=0.2, min_visibility_th=0.5, return_cost=False):
    """The O(L0 L1 npts) label pass and the assignment of the line ground truth (gt_generation.py:173-204, 290-406,
    460-558) for given projections.  segs0/1 [B,L,4]: clamped segments (line_segments); pts0_1 [B,L0*npts,2]: the
    sampled points of segs0 projected into view 1, whose image is size1 = (h1, w1) (pts1_0, size0 likewise).
    visible0/1, valid_pts0/1 [B,L*npts] bool: visibility in the other view and valid depth of each point, all None in
    the homography variant.  Returns {line_assignment bool [B,L0,L1], line_matches0/1 int64 (partner, -1 unmatched, -2
    ignored)}, plus `cost` (the float64 matrix given to the assignment) when return_cost."""
    segs0, segs1 = _chk(segs0.contiguous(), torch.float32), _chk(segs1.contiguous(), torch.float32)
    pts0_1, pts1_0 = pts0_1.float().contiguous(), pts1_0.float().contiguous()
    B, L0, L1 = segs0.shape[0], segs0.shape[1], segs1.shape[1]
    if L0 == 0 or L1 == 0:
        raise ValueError("line ground truth needs at least one line per view")
    assert pts0_1.numel() == B * L0 * npts * 2 and pts1_0.numel() == B * L1 * npts * 2, "points: [B, L*npts, 2]"
    dev = segs0.device
    u8 = lambda t: None if t is None else t.to(torch.uint8).contiguous()  # noqa: E731
    m0 = torch.empty(B, L0, device=dev, dtype=torch.int64)
    m1 = torch.empty(B, L1, device=dev, dtype=torch.int64)
    asg = torch.empty(B, L0, L1, device=dev, dtype=torch.bool)
    ws = torch.empty(_lib.load().lgb200_gt_lines_ws_bytes(B, L0, L1), device=dev, dtype=torch.uint8)
    (h0, w0), (h1, w1) = (int(s) for s in size0), (int(s) for s in size1)
    # byte copies held until the launch is queued (a temporary would go back to the allocator before it)
    vis0, vis1, vp0, vp1, vl0, vl1 = (u8(t) for t in (visible0, visible1, valid_pts0, valid_pts1, valid_lines0,
                                                      valid_lines1))
    call("lgb200_gt_line_matches", ptr(segs0), ptr(segs1), ptr(pts0_1), ptr(pts1_0), ptr(vis0), ptr(vis1), ptr(vp0),
         ptr(vp1), ptr(vl0), ptr(vl1), w0, h0, w1, h1, int(npts),
         float(dist_th), float(overlap_th), float(min_visibility_th), ptr(m0), ptr(m1), ptr(asg), ptr(ws), B, L0, L1,
         stream_ptr())
    out = {"line_assignment": asg, "line_matches0": m0, "line_matches1": m1}
    if return_cost:
        out["cost"] = ws[:B * L0 * L1 * 8].view(torch.float64).view(B, L0, L1)
    return out


def gt_line_matches_from_homography(lines0, lines1, valid_lines0, valid_lines1, shape0, shape1, H, npts=50, dist_th=5,
                                    overlap_th=0.2, min_visibility_th=0.2):
    """Device-side gt_line_matches_from_homography (geometry/gt_generation.py:409-558; defaults as the reference's).
    lines [B,L,2,2] / [B,L,4] / [B,L,K,2] in pixels, valid_lines [B,L] bool, shape0/1 (..., h, w) of the images, H
    [B,3,3] -> {line_assignment, line_matches0, line_matches1}, with no host synchronisation."""
    from .geometry import inv3x3, warp_points

    (h0, w0), (h1, w1) = tuple(shape0[-2:]), tuple(shape1[-2:])
    segs0, segs1 = line_segments(lines0, h0, w0), line_segments(lines1, h1, w1)
    B = segs0.shape[0]
    Hm = H.float().expand(B, 3, 3) if H.dim() == 2 else H.float()
    pts0_1 = warp_points(sample_line_points(segs0, npts), Hm)  # O(L npts): homography.py:161-180
    pts1_0 = warp_points(sample_line_points(segs1, npts), inv3x3(Hm))
    return gt_line_matches_from_projection(segs0, segs1, pts0_1, pts1_0, (h0, w0), (h1, w1), valid_lines0,
                                           valid_lines1, npts=npts, dist_th=dist_th, overlap_th=overlap_th,
                                           min_visibility_th=min_visibility_th)


_head_token_counters = {}


def head_token_fwd(x, wm, bm, wt, bt, cdt):
    """x [T,D] fp32 -> (x in cdt, zt [T,2] = (matchability, token-confidence) logits, ls, du); see lgb200.h."""
    _chk(x, torch.float32)
    T, D = x.shape
    dev = x.device
    xc = torch.empty(T, D, device=dev, dtype=cdt)
    zt = torch.empty(T, 2, device=dev, dtype=torch.float32)
    ls = torch.empty(T, device=dev, dtype=torch.float32)
    du = torch.empty_like(ls)
    f = lambda t: None if t is None else t.detach().float().contiguous()  # noqa: E731
    wm, bm, wt, bt = f(wm), f(bm), f(wt), f(bt)
    call("lgb200_head_token_fwd", ptr(x), ptr(wm), ptr(bm), ptr(wt), ptr(bt), ptr(xc), ptr(zt), ptr(ls), ptr(du), T, D,
         _code(cdt), stream_ptr())
    return xc, zt, ls, du


def adaptive_compact(x, theta, ind, zt, seg, fin, layer, sizes, conf_thr=None, depth_conf=-1.0, width_conf=-1.0,
                     finish=False, pair_pts=None):
    """One layer's stop / prune step of adaptive depth / width on a batch of pairs (lgb200_adaptive_compact,
    include/lgb200.h).  x [T, D], theta [T, R] fp32, ind [T] int32, zt [T, 2] (None when finish), seg [4, 2B] int32.
    fin: dict of the per-batch outputs updated in place -- x [B (M + N), D], ind [B (M + N)], len [2B], stop [B]
    (int32) and prune0 [B, M] / prune1 [B, N] (int64).  pair_pts: None, or [B] int32 = each pair's original point count
    when the pairs have different sizes (M, N are then the padded sizes; lgb200_adaptive_compact_varlen).  Returns
    (x, theta, ind, seg, status): the packed state of the next layer with T rows of capacity, and status [2] int32 =
    (kept tokens, emptied-view flag), still on the device."""
    B, M, N = sizes
    T, D = x.shape
    R = theta.shape[1]
    _chk(x, torch.float32), _chk(theta, torch.float32), _chk(ind, torch.int32), _chk(seg, torch.int32)
    if zt is not None:
        _chk(zt, torch.float32)
    if conf_thr is not None:  # read as one fp32 on the device
        _chk(conf_thr, torch.float32)
        assert conf_thr.numel() >= 1 and conf_thr.device == x.device
    dev = x.device
    x_out, theta_out, ind_out = torch.empty_like(x), torch.empty_like(theta), torch.empty_like(ind)
    seg_out = torch.empty_like(seg)
    status = torch.empty(2, device=dev, dtype=torch.int32)
    ws = torch.empty(_lib.load().lgb200_adaptive_compact_ws_ints(T, B), device=dev, dtype=torch.int32)
    do_stop, do_prune = depth_conf > 0, width_conf > 0
    args = (ptr(x), ptr(theta), ptr(ind), ptr(zt), ptr(seg), ptr(x_out), ptr(theta_out), ptr(ind_out), ptr(seg_out),
            ptr(fin["x"]), ptr(fin["ind"]), ptr(fin["len"]), ptr(fin["stop"]), ptr(fin["prune0"]), ptr(fin["prune1"]),
            ptr(status), ptr(ws), ptr(conf_thr))
    rest = (float(depth_conf), float(1 - width_conf), int(do_stop), int(do_prune), int(layer), int(finish), B, M, N, T,
            D, R, stream_ptr())
    if pair_pts is None:
        call("lgb200_adaptive_compact", *args, *rest)
    else:
        _chk(pair_pts, torch.int32)
        assert pair_pts.shape == (B,) and pair_pts.device == x.device
        call("lgb200_adaptive_compact_varlen", *args, ptr(pair_pts), *rest)
    return x_out, theta_out, ind_out, seg_out, status


def head_token_bwd(x, dmdw, dzt, wm):
    """-> (dx [T,D] fp32 = float(dmdw) + dzt[:,0] wm, dW2 [2,D] = dzt^T x, db2 [2]); dmdw None: dx is None."""
    _chk(x, torch.float32), _chk(dzt, torch.float32)
    if dmdw is not None:
        _chk(dmdw)
    T, D = x.shape
    dev = x.device
    cnt = _head_token_counters.get(dev)
    if cnt is None:
        cnt = _head_token_counters[dev] = torch.zeros(1, device=dev, dtype=torch.int32)
    dx = torch.empty_like(x) if dmdw is not None else None
    dW2 = torch.empty(2, D, device=dev, dtype=torch.float32)
    db2 = torch.empty(2, device=dev, dtype=torch.float32)
    ws = torch.empty(_lib.load().lgb200_head_token_bwd_ws_floats(D), device=dev, dtype=torch.float32)
    wmf = wm.detach().float().contiguous()
    call("lgb200_head_token_bwd", ptr(x), ptr(dmdw), ptr(dzt), ptr(wmf), ptr(dx), ptr(dW2), ptr(db2), ptr(ws), ptr(cnt),
         T, D, _code(dmdw.dtype if dmdw is not None else x.dtype), stream_ptr())
    return dx, dW2, db2


def filter_matches(rowmax, rowarg, colarg, th):
    """lightglue.py:293-309 from the pass-2 argmax."""
    B, M = rowmax.shape
    N = colarg.shape[1]
    dev = rowmax.device
    m0 = torch.empty(B, M, device=dev, dtype=torch.int64)
    m1 = torch.empty(B, N, device=dev, dtype=torch.int64)
    ms0 = torch.empty(B, M, device=dev, dtype=torch.float32)
    ms1 = torch.empty(B, N, device=dev, dtype=torch.float32)
    call("lgb200_filter_matches", ptr(rowmax), ptr(rowarg), ptr(colarg), float(th), ptr(m0), ptr(m1), ptr(ms0),
         ptr(ms1), B, M, N, stream_ptr())
    return m0, m1, ms0, ms1


def assign_varlen(sim, ls0, ls1, dust0, dust1, pairs, ind0, ind1, th, out):
    """The evaluation head (assign_stats(dense=True) + filter_matches) over G pairs of different sizes in one pass each
    (lgb200_assign_{lse,scores}_varlen + lgb200_filter_matches_varlen, include/lgb200.h).  sim [G, M, N] fp32 padded;
    ls0 / dust0 [G, M], ls1 / dust1 [G, N]; pairs [3, G] int32 = (m, n, output batch row); ind0 [G, M] / ind1 [G, N]
    int32 original keypoint indices; nothing past a pair's (m, n) is read.  `out` holds the batch outputs, written in
    place at the original indices: scores [Bo, Mo + 1, No + 1], m0 / ms0 [Bo, Mo] (int64 / fp32), m1 / ms1 [Bo, No].
    Returns the padded per-row statistics (rowmax, rowarg, row_expsum [G, M]; colmax, colarg [G, N])."""
    _chk(sim, torch.float32)
    for t in (pairs, ind0, ind1):
        _chk(t, torch.int32)
    G, M, N = sim.shape
    assert pairs.shape == (3, G) and ind0.shape == (G, M) and ind1.shape == (G, N), (pairs.shape, ind0.shape, ind1.shape)
    scores, m0, m1, ms0, ms1 = (out[k] for k in ("scores", "m0", "m1", "ms0", "ms1"))
    _chk(scores, torch.float32), _chk(m0, torch.int64), _chk(m1, torch.int64), _chk(ms0, torch.float32)
    _chk(ms1, torch.float32)
    Mo, No = m0.shape[1], m1.shape[1]
    assert scores.shape[1:] == (Mo + 1, No + 1) and ms0.shape == m0.shape and ms1.shape == m1.shape
    dev = sim.device
    f = lambda *s: torch.empty(*s, device=dev, dtype=torch.float32)  # noqa: E731
    st = {"lse_row": f(G, M), "lse_col": f(G, N), "rowmax": f(G, M), "colmax": f(G, N), "row_expsum": f(G, M),
          "rowarg": torch.empty(G, M, device=dev, dtype=torch.int32),
          "colarg": torch.empty(G, N, device=dev, dtype=torch.int32)}
    ws = torch.empty(_lib.load().lgb200_assign_ws_bytes(G, M, N), device=dev, dtype=torch.uint8)
    call("lgb200_assign_lse_varlen", ptr(sim), ptr(st["lse_row"]), ptr(st["lse_col"]), ptr(ws), ptr(pairs), G, M, N,
         stream_ptr())
    ls0, ls1, dust0, dust1 = (t.detach().float().contiguous() for t in (ls0, ls1, dust0, dust1))
    assert ls0.shape == dust0.shape == (G, M) and ls1.shape == dust1.shape == (G, N)
    call("lgb200_assign_scores_varlen", ptr(sim), ptr(st["lse_row"]), ptr(st["lse_col"]), ptr(ls0), ptr(ls1), ptr(dust0),
         ptr(dust1), ptr(scores), ptr(st["rowmax"]), ptr(st["rowarg"]), ptr(st["colmax"]), ptr(st["colarg"]),
         ptr(st["row_expsum"]), ptr(ws), ptr(pairs), ptr(ind0), ptr(ind1), G, M, N, Mo, No, stream_ptr())
    call("lgb200_filter_matches_varlen", ptr(st["rowmax"]), ptr(st["rowarg"]), ptr(st["colarg"]), float(th), ptr(m0),
         ptr(m1), ptr(ms0), ptr(ms1), ptr(pairs), ptr(ind0), ptr(ind1), G, M, N, Mo, No, stream_ptr())
    return st


def _log_double_softmax_fwd(sim, bin_score):
    _chk(sim, torch.float32)
    B, M, N = sim.shape
    out = torch.empty(B, M + 1, N + 1, device=sim.device, dtype=torch.float32)
    ws = torch.empty(_lib.load().lgb200_heads_ws_bytes(B, M, N), device=sim.device, dtype=torch.uint8)
    if torch.is_tensor(bin_score) and bin_score.is_cuda:  # learnt bin: read on the device (no .item(), graph-capturable)
        bs = bin_score.detach().reshape(-1)[:1].float().contiguous()
        call("lgb200_log_double_softmax_dev", ptr(sim), ptr(bs), ptr(out), ptr(ws), B, M, N, stream_ptr())
    else:
        call("lgb200_log_double_softmax", ptr(sim), float(bin_score), ptr(out), ptr(ws), B, M, N, stream_ptr())
    return out


def log_double_softmax(sim, bin_score):
    """gluestick.py:772-783.  Differentiable w.r.t. sim and a tensor bin_score (heads_grad.LogDoubleSoftmaxFn)."""
    if torch.is_tensor(bin_score) and (sim.requires_grad or bin_score.requires_grad):
        from .heads_grad import LogDoubleSoftmaxFn

        return LogDoubleSoftmaxFn.apply(sim, bin_score)
    return _log_double_softmax_fwd(sim, bin_score)


def log_double_softmax_varlen(sim, bin_score, pairs, th, out):
    """GlueStick's evaluation head (log_double_softmax + _get_matches, gluestick.py:318-331, 772-783) over G pairs of
    different sizes (lgb200_log_double_softmax_varlen + lgb200_filter_matches_varlen, include/lgb200.h).  sim [G, M, N]
    fp32 padded; bin_score a CUDA tensor (read on the device); pairs [3, G] int32 = (m, n, output batch row); nothing
    past a pair's (m, n) is read.  `out` holds the batch outputs, written in place: scores [Bo, Mo + 1, No + 1] (pair
    block top-left, dustbins at Mo / No), m0 / ms0 [Bo, Mo] (int64 / fp32), m1 / ms1 [Bo, No]; other entries are kept."""
    _chk(sim, torch.float32), _chk(pairs, torch.int32)
    G, M, N = sim.shape
    assert pairs.shape == (3, G), pairs.shape
    scores, m0, m1, ms0, ms1 = (out[k] for k in ("scores", "m0", "m1", "ms0", "ms1"))
    _chk(scores, torch.float32), _chk(m0, torch.int64), _chk(m1, torch.int64), _chk(ms0, torch.float32)
    _chk(ms1, torch.float32)
    Mo, No = m0.shape[1], m1.shape[1]
    assert scores.shape[1:] == (Mo + 1, No + 1) and ms0.shape == m0.shape and ms1.shape == m1.shape
    bs = _bin_dev(bin_score)
    assert bs is not None, "log_double_softmax_varlen: the bin score must be a CUDA tensor"
    dev = sim.device
    rowmax = torch.empty(G, M, device=dev, dtype=torch.float32)
    rowarg = torch.empty(G, M, device=dev, dtype=torch.int32)
    colarg = torch.empty(G, N, device=dev, dtype=torch.int32)
    ws = torch.empty(_lib.load().lgb200_heads_ws_bytes(G, M, N), device=dev, dtype=torch.uint8)
    call("lgb200_log_double_softmax_varlen", ptr(sim), ptr(bs), ptr(scores), ptr(rowmax), ptr(rowarg), ptr(colarg),
         ptr(ws), ptr(pairs), G, M, N, Mo, No, stream_ptr())
    ind0 = torch.arange(M, device=dev, dtype=torch.int32).expand(G, M).contiguous()
    ind1 = torch.arange(N, device=dev, dtype=torch.int32).expand(G, N).contiguous()
    call("lgb200_filter_matches_varlen", ptr(rowmax), ptr(rowarg), ptr(colarg), float(th), ptr(m0), ptr(m1), ptr(ms0),
         ptr(ms1), ptr(pairs), ptr(ind0), ptr(ind1), G, M, N, Mo, No, stream_ptr())


def line_scores_varlen(sim, junc0, junc1, pairs, L0, L1):
    """raw line scores [G, L0, L1] fp32 (gluestick.py:348-361) of G pairs from their endpoint similarity blocks sim
    [G, P0, P1] fp32 and junction indices junc0 [G, 2 L0] / junc1 [G, 2 L1] int32; pairs [2+, G] int32 = each pair's
    line counts (m, n).  Entries past (m, n) are zero."""
    _chk(sim, torch.float32), _chk(junc0, torch.int32), _chk(junc1, torch.int32), _chk(pairs, torch.int32)
    G, P0, P1 = sim.shape
    assert junc0.shape == (G, 2 * L0) and junc1.shape == (G, 2 * L1) and pairs.shape[1] == G
    raw = torch.zeros(G, L0, L1, device=sim.device, dtype=torch.float32)
    call("lgb200_line_scores_varlen", ptr(sim), ptr(junc0), ptr(junc1), ptr(raw), ptr(pairs), G, P0, P1, L0, L1,
         stream_ptr())
    return raw


def junction_mean_(x, upd, order, tgt_sorted):
    """x [T, D] fp32 += (in place) the mean of the endpoint updates upd [E, D] fp32 per target row, summed in the order
    `order` [E] int32 (the endpoints sorted stably by target row; tgt_sorted [E] int32 their rows).  Returns x."""
    _chk(x, torch.float32), _chk(upd, torch.float32), _chk(order, torch.int32), _chk(tgt_sorted, torch.int32)
    E, D = upd.shape
    assert x.shape[1] == D and order.shape == tgt_sorted.shape == (E,)
    if E:
        call("lgb200_junction_mean_varlen", ptr(x), ptr(upd), ptr(order), ptr(tgt_sorted), E, D, stream_ptr())
    return x


def _junction_sum_(x, src, order, tgt_sorted):
    """x [T, D] fp32 += (in place) per target row, the sum over the endpoints e aimed at it of src[e, :D] +
    src[e ^ 1, D:2D] (src [E, >= 2D] fp32 with unit inner stride), in the order `order` (lgb200_junction_sum)."""
    _chk(x, torch.float32), _chk(order, torch.int32), _chk(tgt_sorted, torch.int32)
    E, D = src.shape[0], x.shape[1]
    if src.dtype != torch.float32 or src.stride(1) != 1 or src.stride(0) % 4 or src.data_ptr() % 16:
        src = src.float().contiguous()
    _chk(src, strided_rows=True)
    assert src.shape[1] >= 2 * D and order.shape == tgt_sorted.shape == (E,)
    if E:
        call("lgb200_junction_sum", ptr(x), ptr(src), ptr(order), ptr(tgt_sorted), E, D, src.stride(0), stream_ptr())
    return x


class JunctionGather(torch.autograd.Function):
    """The LineLayer's endpoint gather (gluestick.py:664-675): x [T, D] fp32 -> [E, 2D] = [x[tgt[e]] ; x[tgt[e ^ 1]]]
    (endpoint e's junction, then its line's other end's).  tgt [E] int32; order / tgt_sorted [E] int32: the endpoints
    sorted stably by tgt (gluestick.junction_order).  Backward: per junction row, the sum of its endpoints' two column
    blocks in that order (lgb200_junction_sum), so it has no atomics and gives the same bits on every run."""

    @staticmethod
    def forward(ctx, x, tgt, order, tgt_sorted):
        E, D = tgt.numel(), x.shape[1]
        both = torch.stack([tgt, tgt.view(-1, 2).flip(1).reshape(-1)], 1).reshape(-1)
        ctx.save_for_backward(order, tgt_sorted)
        ctx.T = x.shape[0]
        return x.index_select(0, both).view(E, 2 * D)

    @staticmethod
    def backward(ctx, g):
        order, tgt_sorted = ctx.saved_tensors
        dx = torch.zeros(ctx.T, g.shape[1] // 2, device=g.device, dtype=torch.float32)
        return _junction_sum_(dx, g, order, tgt_sorted), None, None, None


class JunctionMean(torch.autograd.Function):
    """x [T, D] fp32 + per target row, the mean of the endpoint updates upd [E, D] aimed at it (the LineLayer's
    scatter-mean, gluestick.py:682-690), summed in the order `order` (lgb200_junction_mean_varlen on a copy of x).
    tgt [E] int32 each endpoint's row; order / tgt_sorted as for JunctionGather.  Backward: dx = g, d upd[e] =
    g[tgt[e]] / (number of endpoints at tgt[e]), the same division as the forward's."""

    @staticmethod
    def forward(ctx, x, upd, tgt, order, tgt_sorted):
        out = junction_mean_(x.float().clone(), upd.float().contiguous(), order, tgt_sorted)
        ctx.save_for_backward(tgt, tgt_sorted)
        return out

    @staticmethod
    def backward(ctx, g):
        tgt, tgt_sorted = ctx.saved_tensors
        cnt = torch.searchsorted(tgt_sorted, tgt, right=True) - torch.searchsorted(tgt_sorted, tgt)
        return g, g.index_select(0, tgt) / cnt[:, None].float(), None, None, None


def _line_scores_train(sim, junc0, junc1, pairs):
    _chk(sim, torch.float32), _chk(junc0, torch.int32), _chk(junc1, torch.int32), _chk(pairs, torch.int32)
    G, P0, P1 = sim.shape
    L0, L1 = junc0.shape[1] // 2, junc1.shape[1] // 2
    assert junc0.shape == (G, 2 * L0) and junc1.shape == (G, 2 * L1) and pairs.shape[1] == G
    raw = torch.zeros(G, L0, L1, device=sim.device, dtype=torch.float32)
    call("lgb200_line_scores_train", ptr(sim), ptr(junc0), ptr(junc1), ptr(raw), ptr(pairs), G, P0, P1, L0, L1,
         stream_ptr())
    return raw


def line_scores_bwd(graw, sim, junc0, junc1, order0, ptr0, order1, ptr1, pairs):
    """d sim [G, P0, P1] of LineScores (lgb200_line_scores_bwd): every entry written, 0 where no line reads it."""
    graw = graw.float().contiguous()
    for t in (order0, ptr0, order1, ptr1):
        _chk(t, torch.int32)
    G, P0, P1 = sim.shape
    L0, L1 = junc0.shape[1] // 2, junc1.shape[1] // 2
    assert graw.shape == (G, L0, L1) and ptr0.shape == (G, P0 + 1) and ptr1.shape == (G, P1 + 1)
    assert order0.shape == (G * 2 * L0,) and order1.shape == (G * 2 * L1,)
    dsim = torch.empty_like(sim)
    call("lgb200_line_scores_bwd", ptr(graw), ptr(sim), ptr(junc0), ptr(junc1), ptr(order0), ptr(ptr0), ptr(order1),
         ptr(ptr1), ptr(pairs), ptr(dsim), G, P0, P1, L0, L1, stream_ptr())
    return dsim


class LineScores(torch.autograd.Function):
    """raw line scores [G, L0, L1] = 0.5 * maximum(s[a0,c0] + s[a1,c1], s[a0,c1] + s[a1,c0]) (gluestick.py:348-361) from
    sim [G, P0, P1] fp32 and the junction indices junc0 [G, 2 L0] / junc1 [G, 2 L1] int32; pairs [2+, G] int32: each
    pair's line counts (m, n), raw is 0 past them.  Forward: lgb200_line_scores_train, bit-identical to the torch formula
    (NaN included).  order0 / ptr0, order1 / ptr1: each view's endpoints per junction (gluestick.junction_layout), for the
    backward, lgb200_line_scores_bwd: torch's gradient summed in a fixed order."""

    @staticmethod
    def forward(ctx, sim, junc0, junc1, pairs, order0, ptr0, order1, ptr1):
        ctx.save_for_backward(sim, junc0, junc1, pairs, order0, ptr0, order1, ptr1)
        return _line_scores_train(sim, junc0, junc1, pairs)

    @staticmethod
    def backward(ctx, graw):
        sim, junc0, junc1, pairs, *csr = ctx.saved_tensors
        return (line_scores_bwd(graw, sim, junc0, junc1, *csr, pairs), *([None] * 7))


def _bin_dev(alpha):
    """A CUDA tensor bin score as a 1-element fp32 device vector (read by the kernels: no host read-back), else None."""
    if torch.is_tensor(alpha) and alpha.is_cuda:
        return alpha.detach().reshape(-1)[:1].float().contiguous()
    return None


def _log_optimal_transport_fwd(sim, alpha, iters, keep_potentials=False):
    """One persistent cooperative kernel for all iterations.  keep_potentials: also return the per-iteration
    potentials (uh [iters,B,M+1], vh [iters,B,N+1]) the backward sweep consumes.  alpha: a CUDA tensor is read on the
    device (lgb200_sinkhorn_fwd_dev), anything else is a host scalar."""
    _chk(sim, torch.float32)
    B, M, N = sim.shape
    out = torch.empty(B, M + 1, N + 1, device=sim.device, dtype=torch.float32)
    ws = torch.empty(_lib.load().lgb200_heads_ws_bytes(B, M, N), device=sim.device, dtype=torch.uint8)
    a_dev = _bin_dev(alpha)
    uh = vh = None
    if keep_potentials:
        uh = torch.empty(max(iters, 1), B, M + 1, device=sim.device, dtype=torch.float32)
        vh = torch.empty(max(iters, 1), B, N + 1, device=sim.device, dtype=torch.float32)
    if a_dev is not None:
        call("lgb200_sinkhorn_fwd_dev", ptr(sim), ptr(a_dev), int(iters), ptr(out), ptr(uh), ptr(vh), ptr(ws), B, M, N,
             stream_ptr())
    elif keep_potentials:
        call("lgb200_sinkhorn_fwd", ptr(sim), float(alpha), int(iters), ptr(out), ptr(uh), ptr(vh), ptr(ws), B, M, N,
             stream_ptr())
    else:
        call("lgb200_sinkhorn", ptr(sim), float(alpha), int(iters), ptr(out), ptr(ws), B, M, N, stream_ptr())
    return (out, uh, vh) if keep_potentials else out


def _log_optimal_transport_bwd(sim, alpha, iters, grad, uh, vh):
    """Reverse sweep of the iterations (lgb200_sinkhorn_bwd, or _dev for a CUDA tensor alpha): returns dsim [B,M,N]
    and d alpha (0-dim, on the device)."""
    _chk(sim, torch.float32)
    _chk(grad, torch.float32)
    B, M, N = sim.shape
    assert grad.shape == (B, M + 1, N + 1) and iters > 0
    dsim = torch.empty_like(sim)
    dzr = torch.empty(B, N + 1, device=sim.device, dtype=torch.float32)
    dzc = torch.empty(B, M, device=sim.device, dtype=torch.float32)
    ws = torch.empty(_lib.load().lgb200_heads_ws_bytes(B, M, N), device=sim.device, dtype=torch.uint8)
    a_dev = _bin_dev(alpha)
    if a_dev is not None:
        call("lgb200_sinkhorn_bwd_dev", ptr(sim), ptr(a_dev), int(iters), ptr(grad), ptr(uh), ptr(vh), ptr(dsim),
             ptr(dzr), ptr(dzc), ptr(ws), B, M, N, stream_ptr())
    else:
        call("lgb200_sinkhorn_bwd", ptr(sim), float(alpha), int(iters), ptr(grad), ptr(uh), ptr(vh), ptr(dsim),
             ptr(dzr), ptr(dzc), ptr(ws), B, M, N, stream_ptr())
    return dsim, dzr.sum() + dzc.sum()


def log_optimal_transport(sim, alpha, iters):
    """gluefactory_nonfree/superglue.py:198-214.  Differentiable w.r.t. sim and a tensor alpha
    (heads_grad.LogOptimalTransportFn: reverse Sinkhorn iterations, no dense autograd tape)."""
    if torch.is_tensor(alpha) and (sim.requires_grad or alpha.requires_grad):
        from .heads_grad import LogOptimalTransportFn

        return LogOptimalTransportFn.apply(sim, alpha, int(iters))
    return _log_optimal_transport_fwd(sim, alpha if _bin_dev(alpha) is not None else float(alpha), iters)


def log_optimal_transport_varlen(sim, alpha, iters, pairs, out):
    """SuperGlue's evaluation head (superglue.py:186-214) over G pairs of different sizes in one persistent launch
    (lgb200_sinkhorn_varlen, include/lgb200.h).  sim [G, M, N] fp32 padded; alpha a CUDA tensor (read on the device);
    pairs [3, G] int32 = (m, n, output batch row); nothing past a pair's (m, n) is read.  Pair g's result is written in
    place into out [Bo, Mo + 1, No + 1] fp32: its block top-left of row pairs[2, g], its dustbins at Mo / No; every other
    entry is kept.  Forward only."""
    _chk(sim, torch.float32), _chk(pairs, torch.int32), _chk(out, torch.float32)
    G, M, N = sim.shape
    assert pairs.shape == (3, G) and out.dim() == 3, (pairs.shape, out.shape)
    a_dev = _bin_dev(alpha)
    assert a_dev is not None, "log_optimal_transport_varlen: the bin score must be a CUDA tensor"
    Mo, No = out.shape[1] - 1, out.shape[2] - 1
    ws = torch.empty(_lib.load().lgb200_sinkhorn_varlen_ws_bytes(G, M, N), device=sim.device, dtype=torch.uint8)
    call("lgb200_sinkhorn_varlen", ptr(sim), ptr(a_dev), int(iters), ptr(out), ptr(ws), ptr(pairs), G, M, N, Mo, No,
         stream_ptr())
    return out


# ------------------------------------------------------------------------------------------------
# SuperGlue's NLL head and match filter on the dense Sinkhorn output (superglue.py:301-311, 322-352)
# ------------------------------------------------------------------------------------------------
def ot_nll_sums(Z, mask_u8, neg0, neg1, gt0=None, gt1=None):
    """Z [B,M+1,N+1] fp32, mask u8 [B,M,N], neg0 [B,M] / neg1 [B,N] fp32 0/1 -> (pos, neg) [B]:
    pos = sum mask * Z[:, :M, :N], neg = sum neg0 * Z[:, :M, N] + sum neg1 * Z[:, M, :N] (lgb200_ot_nll_fwd).
    mask_u8 None: the positives are the match lists gt0 [B,M] / gt1 [B,N] int64 (lgb200_ot_nll_fwd_sparse, the same
    bits; NaN pos for a pair whose lists disagree)."""
    _chk(Z, torch.float32), _chk(neg0, torch.float32), _chk(neg1, torch.float32)
    B, M1, N1 = Z.shape
    M, N = M1 - 1, N1 - 1
    assert neg0.shape == (B, M) and neg1.shape == (B, N)
    pos = torch.empty(B, device=Z.device, dtype=torch.float32)
    neg = torch.empty_like(pos)
    ws = torch.empty(_lib.load().lgb200_heads_ws_bytes(B, M, N), device=Z.device, dtype=torch.uint8)
    if mask_u8 is None:
        _chk(gt0, torch.int64), _chk(gt1, torch.int64)
        assert gt0.shape == (B, M) and gt1.shape == (B, N)
        call("lgb200_ot_nll_fwd_sparse", ptr(Z), ptr(gt0), ptr(gt1), ptr(neg0), ptr(neg1), ptr(pos), ptr(neg), ptr(ws),
             B, M, N, stream_ptr())
        return pos, neg
    _chk(mask_u8, torch.uint8)
    assert mask_u8.shape == (B, M, N)
    call("lgb200_ot_nll_fwd", ptr(Z), ptr(mask_u8), ptr(neg0), ptr(neg1), ptr(pos), ptr(neg), ptr(ws), B, M, N,
         stream_ptr())
    return pos, neg


def ot_nll_bwd(mask_u8, neg0, neg1, num_pos, num_neg, gpos, gneg, gt0=None):
    """dZ [B,M+1,N+1] of nll_pos = -pos / num_pos and nll_neg = -neg / num_neg for incoming gradients gpos, gneg [B]
    (lgb200_ot_nll_bwd: everything read on the device, linear in the incoming gradients).  mask_u8 None: the positives
    are the match list gt0 [B,M] int64 (lgb200_ot_nll_bwd_sparse, the same bits)."""
    B, M = neg0.shape
    N = neg1.shape[1]
    for t in (neg0, neg1, num_pos, num_neg, gpos, gneg):
        _chk(t, torch.float32)
    dZ = torch.empty(B, M + 1, N + 1, device=neg0.device, dtype=torch.float32)
    if mask_u8 is None:
        _chk(gt0, torch.int64)
        assert gt0.shape == (B, M)
        call("lgb200_ot_nll_bwd_sparse", ptr(gt0), ptr(neg0), ptr(neg1), ptr(num_pos), ptr(num_neg), ptr(gpos),
             ptr(gneg), ptr(dZ), B, M, N, stream_ptr())
        return dZ
    assert mask_u8.shape == (B, M, N)
    call("lgb200_ot_nll_bwd", ptr(mask_u8), ptr(neg0), ptr(neg1), ptr(num_pos), ptr(num_neg), ptr(gpos), ptr(gneg),
         ptr(dZ), B, M, N, stream_ptr())
    return dZ


class OtNllFn(torch.autograd.Function):
    """(nll_pos, nll_neg) [B] of superglue.py:325-336 from the dense log assignment Z, differentiable w.r.t. Z; the
    reference's dense fp32 copies of the mask and of mask * Z are never formed.  mask_u8 None: the positives are the
    match lists gt0 / gt1."""

    @staticmethod
    def forward(ctx, Z, mask_u8, neg0, neg1, num_pos, num_neg, gt0=None, gt1=None):
        pos, neg = ot_nll_sums(Z, mask_u8, neg0, neg1, gt0, gt1)
        ctx.save_for_backward(mask_u8, neg0, neg1, num_pos, num_neg, gt0)
        return -pos / num_pos, -neg / num_neg

    @staticmethod
    def backward(ctx, gpos, gneg):
        mask_u8, neg0, neg1, num_pos, num_neg, gt0 = ctx.saved_tensors
        z = torch.zeros_like(num_pos)
        gpos = z if gpos is None else gpos.float().contiguous()
        gneg = z if gneg is None else gneg.float().contiguous()
        return ot_nll_bwd(mask_u8, neg0, neg1, num_pos, num_neg, gpos, gneg, gt0), None, None, None, None, None, None, None


def ot_nll(Z, gt_assignment, gt_matches0, gt_matches1):
    """superglue.py:325-336 -> (nll_pos, nll_neg, num_pos, num_neg) [B]; counts from lgb200_mask_counts.
    gt_assignment None: the positives come from the one-to-one match lists gt_matches0/1 (match_list_counts); the
    losses and dZ are then bit-identical to the mask's, and NaN for a pair whose lists disagree."""
    neg0 = (gt_matches0 == -1).float().contiguous()
    neg1 = (gt_matches1 == -1).float().contiguous()
    num_neg = (neg0.sum(1) + neg1.sum(1)).clamp(min=1.0)
    if gt_assignment is None:
        gt0, gt1 = gt_matches0.long().contiguous(), gt_matches1.long().contiguous()
        _, _, num_pos = match_list_counts(gt0, gt1)
        nll_pos, nll_neg = OtNllFn.apply(Z.contiguous(), None, neg0, neg1, num_pos, num_neg, gt0, gt1)
        return nll_pos, nll_neg, num_pos, num_neg
    mask = gt_assignment.to(torch.uint8).contiguous()
    rowcnt, _ = mask_counts(mask)
    num_pos = rowcnt.sum(1).clamp(min=1.0)
    nll_pos, nll_neg = OtNllFn.apply(Z.contiguous(), mask, neg0, neg1, num_pos, num_neg)
    return nll_pos, nll_neg, num_pos, num_neg


def ot_filter_stats(Z):
    """Row max / argmax and column argmax (int32, first index on ties) of Z[:, :-1, :-1] (lgb200_ot_filter_stats)."""
    _chk(Z, torch.float32)
    B, M1, N1 = Z.shape
    M, N = M1 - 1, N1 - 1
    rowmax = torch.empty(B, M, device=Z.device, dtype=torch.float32)
    rowarg = torch.empty(B, M, device=Z.device, dtype=torch.int32)
    colarg = torch.empty(B, N, device=Z.device, dtype=torch.int32)
    call("lgb200_ot_filter_stats", ptr(Z), ptr(rowmax), ptr(rowarg), ptr(colarg), B, M, N, stream_ptr())
    return rowmax, rowarg, colarg


def adam_flat_(p, g, m, v, step, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.0, grad_scale=1.0, lr_scale_per_elem=None,
               step_dev=None, lr_dev=None, loss_scale_dev=None, found_inf_dev=None):
    """In-place Adam on flat fp32 buffers (train.py:358-361, 513).  The *_dev device scalars replace the host values
    when the call is captured in a CUDA graph: step count, learning rate, GradScaler scale, skip flag (lgb200.h)."""
    for t in (p, g, m, v):
        _chk(t, torch.float32)
    call("lgb200_adam_flat", ptr(p), ptr(g), ptr(m), ptr(v), p.numel(), ptr(lr_scale_per_elem), float(lr),
         float(betas[0]), float(betas[1]), float(eps), float(weight_decay), int(step), ptr(step_dev), float(grad_scale),
         ptr(lr_dev), ptr(loss_scale_dev), ptr(found_inf_dev), stream_ptr())


def adamw_flat_(p, g, m, v, step, lr, betas=(0.9, 0.999), eps=1e-8, weight_decay=0.01, grad_scale=1.0,
                lr_scale_per_elem=None, step_dev=None, lr_dev=None, loss_scale_dev=None, found_inf_dev=None):
    """In-place torch.optim.AdamW on flat fp32 buffers; arguments as adam_flat_ (lgb200_adamw_flat)."""
    for t in (p, g, m, v):
        _chk(t, torch.float32)
    call("lgb200_adamw_flat", ptr(p), ptr(g), ptr(m), ptr(v), p.numel(), ptr(lr_scale_per_elem), float(lr),
         float(betas[0]), float(betas[1]), float(eps), float(weight_decay), int(step), ptr(step_dev), float(grad_scale),
         ptr(lr_dev), ptr(loss_scale_dev), ptr(found_inf_dev), stream_ptr())


def sgd_flat_(p, g, momentum_buffer, step, lr, momentum=0.0, dampening=0.0, nesterov=False, weight_decay=0.0,
              grad_scale=1.0, lr_scale_per_elem=None, step_dev=None, lr_dev=None, loss_scale_dev=None,
              found_inf_dev=None):
    """In-place torch.optim.SGD on flat fp32 buffers (lgb200_sgd_flat): momentum_buffer is None exactly when
    momentum == 0; at step count 1 the buffer is set to the gradient."""
    for t in (p, g) + ((momentum_buffer,) if momentum_buffer is not None else ()):
        _chk(t, torch.float32)
    call("lgb200_sgd_flat", ptr(p), ptr(g), ptr(momentum_buffer), p.numel(), ptr(lr_scale_per_elem), float(lr),
         float(momentum), float(dampening), int(bool(nesterov)), float(weight_decay), int(step), ptr(step_dev),
         float(grad_scale), ptr(lr_dev), ptr(loss_scale_dev), ptr(found_inf_dev), stream_ptr())


def rmsprop_flat_(p, g, square_avg, momentum_buffer, grad_avg, lr, alpha=0.99, eps=1e-8, weight_decay=0.0,
                  momentum=0.0, grad_scale=1.0, lr_scale_per_elem=None, lr_dev=None, loss_scale_dev=None,
                  found_inf_dev=None):
    """In-place torch.optim.RMSprop on flat fp32 buffers (lgb200_rmsprop_flat): momentum_buffer is None exactly when
    momentum == 0, grad_avg is given for `centered`."""
    for t in (p, g, square_avg) + tuple(t for t in (momentum_buffer, grad_avg) if t is not None):
        _chk(t, torch.float32)
    call("lgb200_rmsprop_flat", ptr(p), ptr(g), ptr(square_avg), ptr(momentum_buffer), ptr(grad_avg), p.numel(),
         ptr(lr_scale_per_elem), float(lr), float(alpha), float(eps), float(weight_decay), float(momentum),
         float(grad_scale), ptr(lr_dev), ptr(loss_scale_dev), ptr(found_inf_dev), stream_ptr())


def flat_grad_check(g, found_inf):
    """found_inf[0] <- 1.0 if any element of the flat fp32 buffer g is non-finite else 0.0 (no host sync)."""
    _chk(g, torch.float32), _chk(found_inf, torch.float32)
    call("lgb200_flat_grad_check", ptr(g), g.numel(), ptr(found_inf), stream_ptr())


def flat_grad_norm_ws(n_norm, device):
    """Scratch for flat_grad_norm over n_norm elements (allocate once: a captured step keeps using it)."""
    return torch.empty(_lib.load().lgb200_flat_grad_norm_ws_bytes(int(n_norm)), device=device, dtype=torch.uint8)


def flat_grad_norm(g, n_norm, grad_scale, loss_scale, max_norm, found_inf, norm_out, adam_div_out, ws):
    """clip_grad_norm_ on the device (no host sync): norm_out <- ||g[:n_norm] * grad_scale / loss_scale|| (fp64 sum in
    a fixed order), found_inf <- any non-finite element of g or a non-finite norm, adam_div_out <- the loss_scale_dev
    that makes adam_flat_ apply the clip coefficient.  loss_scale: device scalar or None (lgb200.h)."""
    for t in (g, found_inf, norm_out, adam_div_out):
        _chk(t, torch.float32)
    if loss_scale is not None:
        _chk(loss_scale, torch.float32)
    call("lgb200_flat_grad_norm", ptr(g), int(n_norm), g.numel(), float(grad_scale), ptr(loss_scale), float(max_norm),
         ptr(found_inf), ptr(norm_out), ptr(adam_div_out), ptr(ws), stream_ptr())


def amp_update(found_inf, step_dev=None, loss_scale=None, growth_tracker=None, growth_factor=2.0, backoff_factor=0.5,
               growth_interval=2000):
    """Device-side bookkeeping of one optimiser step: step count (unless skipped) + GradScaler.update rule."""
    call("lgb200_amp_update", ptr(found_inf), ptr(step_dev), ptr(loss_scale), ptr(growth_tracker), float(growth_factor),
         float(backoff_factor), int(growth_interval), stream_ptr())
