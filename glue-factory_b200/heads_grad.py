"""Backward of the two other assignment heads on the path (SURVEY 8a rows a15 / a16), as closed-form tensor math.

The forward of both heads is a hand-written kernel (csrc/heads.cu: `lgb200_log_double_softmax`, `lgb200_sinkhorn`).
No N x N autograd tape (the reference keeps ~100 dense tensors alive for Sinkhorn, superglue.py:186-214): only the
two LSE vectors / the per-iteration potentials u_k, v_k are kept and the softmax matrices are recomputed on the fly.
The Sinkhorn gradient runs as a kernel (csrc/heads.cu `sk_bwd_persistent_kernel`); the tensor-math functions below are
device-agnostic statements of the same formulas, pinned on the CPU against gradients produced by the reference's
autograd (tests/golden/heads_grad.npz) and used on the GPU as the checker of the kernel.
"""
import math

import torch


def log_double_softmax_backward(sim, bin_score, scores, grad):
    """d/d(sim, bin) of gluestick.py:772-783.  sim [B,M,N], bin_score scalar tensor, scores = forward output
    [B,M+1,N+1], grad = dL/dscores.  The two LSE vectors are read back from the output's bin column / row:
    scores[i,N] = bin - lse_row[i], scores[M,j] = bin - lse_col[j]."""
    B, M, N = sim.shape
    lse_row = bin_score - scores[:, :M, N]
    lse_col = bin_score - scores[:, M, :N]
    gi = grad[:, :M, :N] * 0.5                       # scores[:M,:N] = (s0 + s1) / 2
    r0 = gi.sum(2) + grad[:, :M, N]                  # total gradient entering row i of s0 (N + 1 entries)
    c1 = gi.sum(1) + grad[:, M, :N]                  # total gradient entering column j of s1 (M + 1 entries)
    dsim = 2.0 * gi
    dsim = dsim - torch.exp(sim - lse_row[:, :, None]) * r0[:, :, None]
    dsim = dsim - torch.exp(sim - lse_col[:, None, :]) * c1[:, None, :]
    dbin = (grad[:, :M, N] - torch.exp(scores[:, :M, N]) * r0).sum() + \
           (grad[:, M, :N] - torch.exp(scores[:, M, :N]) * c1).sum()
    return dsim, dbin


def sinkhorn_potentials(sim, alpha, iters):
    """The potentials (u_k, v_k), k = 1..iters, of log_optimal_transport (superglue.py:186-214) and the bordered
    coupling Z; O(iters (M+N)) memory besides Z."""
    B, M, N = sim.shape
    Z = sim.new_empty(B, M + 1, N + 1)
    Z[:, :M, :N] = sim
    Z[:, :M, N] = alpha
    Z[:, M, :] = alpha
    norm = -math.log(M + N)
    log_mu = sim.new_full((B, M + 1), norm)
    log_mu[:, M] = math.log(N) + norm
    log_nu = sim.new_full((B, N + 1), norm)
    log_nu[:, N] = math.log(M) + norm
    us, vs = [], []
    u, v = torch.zeros_like(log_mu), torch.zeros_like(log_nu)
    for _ in range(iters):
        u = log_mu - torch.logsumexp(Z + v[:, None, :], 2)
        v = log_nu - torch.logsumexp(Z + u[:, :, None], 1)
        us.append(u)
        vs.append(v)
    return Z, log_mu, log_nu, us, vs


def log_optimal_transport_backward(sim, alpha, iters, grad):
    """d/d(sim, alpha) of log_optimal_transport by reverse iteration: with P_k = softmax_j(Z + v_{k-1}) and
    Q_k = softmax_i(Z + u_k) recomputed from the potentials,
        dZ -= Q_k dv_k ;  du_k -= Q_k dv_k ;  dZ -= P_k du_k ;  dv_{k-1} = -P_k^T du_k   for k = iters .. 1."""
    B, M, N = sim.shape
    with torch.no_grad():
        Z, log_mu, log_nu, us, vs = sinkhorn_potentials(sim, alpha, iters)
        dZ = grad.clone()
        du = grad.sum(2)
        dv = grad.sum(1)
        for k in range(iters - 1, -1, -1):
            u_k, v_k = us[k], vs[k]
            v_prev = vs[k - 1] if k > 0 else torch.zeros_like(v_k)
            Q = torch.exp(Z + u_k[:, :, None] + (v_k - log_nu)[:, None, :])     # columns sum to 1
            dZ -= Q * dv[:, None, :]
            du = du - (Q * dv[:, None, :]).sum(2)
            P = torch.exp(Z + v_prev[:, None, :] + (u_k - log_mu)[:, :, None])  # rows sum to 1
            dZ -= P * du[:, :, None]
            dv = -(P * du[:, :, None]).sum(1)
            du = torch.zeros_like(du)
        dsim = dZ[:, :M, :N]
        dalpha = dZ[:, :M, N].sum() + dZ[:, M, :].sum()
    return dsim, dalpha


class LogDoubleSoftmaxFn(torch.autograd.Function):
    """forward: lgb200_log_double_softmax; backward: log_double_softmax_backward."""

    @staticmethod
    def forward(ctx, sim, bin_score):
        from . import ops

        scores = ops._log_double_softmax_fwd(sim, bin_score)
        ctx.save_for_backward(sim, bin_score, scores)
        return scores

    @staticmethod
    def backward(ctx, grad):
        sim, bin_score, scores = ctx.saved_tensors
        dsim, dbin = log_double_softmax_backward(sim, bin_score.to(sim.dtype), scores, grad.contiguous())
        return dsim, dbin.to(bin_score.dtype).reshape(bin_score.shape)


class LogOptimalTransportFn(torch.autograd.Function):
    """forward: lgb200_sinkhorn_fwd (keeps the O(iters (M+N)) potentials); backward: lgb200_sinkhorn_bwd, the reverse
    sweep as one persistent kernel (`log_optimal_transport_backward` above is its tensor-math statement, used by the
    CPU tests to pin the formulas against the reference's autograd)."""

    @staticmethod
    def forward(ctx, sim, alpha, iters):
        from . import ops

        sim = sim.contiguous()
        # a CUDA alpha is read by the kernels on the device: no host read-back on a training step
        a = alpha if ops._bin_dev(alpha) is not None else float(alpha)
        out, uh, vh = ops._log_optimal_transport_fwd(sim, a, iters, keep_potentials=True)
        ctx.save_for_backward(sim, alpha, uh, vh)
        ctx.iters = iters
        return out

    @staticmethod
    def backward(ctx, grad):
        from . import ops

        sim, alpha, uh, vh = ctx.saved_tensors
        if ctx.iters == 0:      # out = Z - norm
            M, N = sim.shape[1:]
            dsim, dalpha = grad[:, :M, :N].contiguous(), grad[:, :M, N].sum() + grad[:, M, :].sum()
        else:
            a = alpha if ops._bin_dev(alpha) is not None else float(alpha)
            dsim, dalpha = ops._log_optimal_transport_bwd(sim, a, ctx.iters, grad.contiguous().float(), uh, vh)
        return dsim, dalpha.to(alpha.dtype).reshape(alpha.shape), None
