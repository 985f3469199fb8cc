"""CPU oracle for the LightGlue matcher hot path (TEST INFRASTRUCTURE ONLY).

A plain-PyTorch-on-CPU restatement of the reference algorithm, written from the
math (SURVEY.md Appendix A), NOT a copy of the reference modules.  It is pinned
against the UNMODIFIED reference (imported from /root/reference in the build
container by `oracle/make_golden.py`) through the fixtures under
`tests/golden/` -- see `tests/test_oracle_golden.py`.  The reference's own test
suite holds no numeric vectors for this path (SURVEY.md section 8c), so the
pin is "outputs of the reference itself run here".

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` leg may import this file.  The product path
(`gluefactory_b200`) never does.

Every function cites the reference lines it restates
(paths relative to /root/reference/gluefactory/).

All functions take a flat weight dict `w` whose keys are the reference
state_dict names (models/matchers/lightglue.py:359-372), so the same dict can
be loaded into the reference module and into the CUDA plugin.

`rnd` is an optional operand-rounding hook (e.g. bf16 round trip) applied to
every tensor-core GEMM operand at the same places the CUDA path rounds, so that
kernel-level parity of the bf16 path can be asserted tightly against an fp64
evaluation of the *same rounded operands*.
"""
import math

import torch
import torch.nn.functional as F


def _id(x):
    return x


def bf16_round(x):
    return x.to(torch.bfloat16).to(x.dtype)


class _RoundBoth(torch.autograd.Function):
    """bf16 round trip in forward AND of the incoming gradient in backward: models a tensor that the CUDA path
    stores in bf16 and whose gradient it also produces in bf16."""

    @staticmethod
    def forward(ctx, x):
        return bf16_round(x)

    @staticmethod
    def backward(ctx, g):
        return bf16_round(g)


class _RoundGrad(torch.autograd.Function):
    """identity in forward, bf16 round trip of the gradient in backward."""

    @staticmethod
    def forward(ctx, x):
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        return bf16_round(g)


class Bf16Mirror:
    """Rounding model of the CUDA `precision: bf16` path (glue-factory_b200/engine.py), for tight parity tests of
    the tensor-core kernels at sizes where comparing with fp64 only measures bf16 noise.  Passed as `rnd=`:

      operand(x): GEMM / attention operand taken from an fp32 tensor (the residual stream, weights) -- rounded in
                  forward, gradient left in fp32 (the CUDA path accumulates the residual-stream gradient in fp32);
      store(x):   a tensor the CUDA path keeps in bf16 (every Linear output, rotated q / k, attention output,
                  LayerNorm+GELU output) -- rounded in forward and its gradient rounded in backward;
      bias(b):    Linear biases stay fp32 (added to the fp32 accumulator in the GEMM epilogue);
      grad(x):    fp32 in forward, gradient produced in bf16 (the similarity matrix: dsim is bf16).

    Not mirrored (second-order): P is rounded after normalisation here and before it in the kernels; the shared
    to_qk gradient is rounded per direction before the sum in the CUDA path; final_proj's input gradient."""

    def __call__(self, x):  # plain operand rounding, so the object can be passed wherever `rnd` is a callable
        return bf16_round(x)

    operand = staticmethod(bf16_round)
    bias = staticmethod(_id)
    store = staticmethod(_RoundBoth.apply)
    grad = staticmethod(_RoundGrad.apply)


def _hook(rnd, name):
    """`rnd` is either a plain callable (operand rounding only; the round-1 hook) or a Bf16Mirror-like object."""
    f = getattr(rnd, name, None)
    if f is not None:
        return f
    return rnd if name == "operand" else _id


# ----------------------------------------------------------------------------
# positional encoding / rotary
# ----------------------------------------------------------------------------
def normalize_keypoints(kpts, size):
    """models/matchers/lightglue.py:27-39 (size given as [B,2] (w,h))."""
    if size is None:
        size = 1 + kpts.max(-2).values - kpts.min(-2).values
    size = torch.as_tensor(size).to(kpts)
    shift = size / 2
    scale = size.max(-1).values / 2
    return (kpts - shift[..., None, :]) / scale[..., None, None]


def posenc_angles(w, kpts_n):
    """theta = Wr . kpt  [B,N,32]   (lightglue.py:60-62); cos/sin taken later."""
    return kpts_n @ w["posenc.Wr.weight"].t()


def rope(t, theta):
    """Rotate adjacent channel pairs of t [B,H,N,64] by theta [B,N,32]
    (lightglue.py:42-49: t*cos + rotate_half(t)*sin with freqs repeated x2)."""
    c = torch.cos(theta)[:, None]  # [B,1,N,32]
    s = torch.sin(theta)[:, None]
    te, to = t[..., 0::2], t[..., 1::2]
    out = torch.empty_like(t)
    out[..., 0::2] = te * c - to * s
    out[..., 1::2] = to * c + te * s
    return out


# ----------------------------------------------------------------------------
# transformer blocks
# ----------------------------------------------------------------------------
def _linear(x, w, name, rnd=_id):
    op = _hook(rnd, "operand")
    return _hook(rnd, "store")(op(x) @ op(w[name + ".weight"]).t() + _hook(rnd, "bias")(w[name + ".bias"]))


def _ffn(x, msg, w, pre, rnd=_id):
    """ffn = Linear(2D,2D) -> LayerNorm(2D) -> GELU(erf) -> Linear(2D,D)
    (lightglue.py:143-148, 178-183)."""
    h = _linear(torch.cat([x, msg], -1), w, pre + ".ffn.0", rnd)
    h = F.layer_norm(h, h.shape[-1:], w[pre + ".ffn.1.weight"], w[pre + ".ffn.1.bias"], 1e-5)
    h = _hook(rnd, "store")(F.gelu(h))
    return _linear(h, w, pre + ".ffn.3", rnd)


def _attend(q, k, v, scale, rnd=_id):
    """softmax(q k^T * scale) v  over [B,H,N,dh]  (lightglue.py:118-121, 207-216)."""
    op = _hook(rnd, "operand")
    s = (op(q) @ op(k).transpose(-1, -2)) * scale
    p = torch.softmax(s, -1)
    return _hook(rnd, "store")(op(p) @ op(v))


def self_block(x, theta, w, pre, H, rnd=_id):
    """lightglue.py:150-163.  Wqkv output feature = h*3dh + d*3 + {q,k,v}."""
    B, N, D = x.shape
    dh = D // H
    qkv = _linear(x, w, pre + ".Wqkv", rnd).view(B, N, H, dh, 3).permute(0, 2, 1, 3, 4)
    q, k, v = qkv[..., 0], qkv[..., 1], qkv[..., 2]
    st = _hook(rnd, "store")
    q, k = st(rope(q, theta)), st(rope(k, theta))
    ctx = _attend(q, k, v, dh**-0.5, rnd)
    msg = _linear(ctx.transpose(1, 2).reshape(B, N, D), w, pre + ".out_proj", rnd)
    return x + _ffn(x, msg, w, pre, rnd)


def cross_block(x0, x1, w, pre, H, rnd=_id):
    """lightglue.py:195-221 (non-flash branch: one shared similarity, row and
    column softmax)."""
    B, M, D = x0.shape
    dh = D // H

    def heads(t):
        return t.view(t.shape[0], t.shape[1], H, dh).transpose(1, 2)

    qk0, qk1 = heads(_linear(x0, w, pre + ".to_qk", rnd)), heads(_linear(x1, w, pre + ".to_qk", rnd))
    v0, v1 = heads(_linear(x0, w, pre + ".to_v", rnd)), heads(_linear(x1, w, pre + ".to_v", rnd))
    m0 = _attend(qk0, qk1, v1, dh**-0.5, rnd)
    m1 = _attend(qk1, qk0, v0, dh**-0.5, rnd)
    m0 = _linear(m0.transpose(1, 2).reshape(B, -1, D), w, pre + ".to_out", rnd)
    m1 = _linear(m1.transpose(1, 2).reshape(B, -1, D), w, pre + ".to_out", rnd)
    return x0 + _ffn(x0, m0, w, pre, rnd), x1 + _ffn(x1, m1, w, pre, rnd)


def transformer_layer(d0, d1, th0, th1, w, i, H, rnd=_id):
    """lightglue.py:241-245."""
    d0 = self_block(d0, th0, w, f"transformers.{i}.self_attn", H, rnd)
    d1 = self_block(d1, th1, w, f"transformers.{i}.self_attn", H, rnd)
    return cross_block(d0, d1, w, f"transformers.{i}.cross_attn", H, rnd)


# ----------------------------------------------------------------------------
# assignment head
# ----------------------------------------------------------------------------
def sigmoid_log_double_softmax(sim, z0, z1):
    """lightglue.py:256-268.  z0 [B,M], z1 [B,N]."""
    B, M, N = sim.shape
    lse_r = torch.logsumexp(sim, 2, keepdim=True)
    lse_c = torch.logsumexp(sim, 1, keepdim=True)
    scores = sim.new_zeros(B, M + 1, N + 1)
    scores[:, :M, :N] = (sim - lse_r) + (sim - lse_c) + (F.logsigmoid(z0)[:, :, None] + F.logsigmoid(z1)[:, None, :])
    scores[:, :M, N] = F.logsigmoid(-z0)
    scores[:, M, :N] = F.logsigmoid(-z1)
    return scores


def match_assignment(d0, d1, w, i, rnd=_id):
    """lightglue.py:278-287. Returns (scores [B,M+1,N+1], sim [B,M,N])."""
    pre = f"log_assignment.{i}"
    D = d0.shape[-1]
    md0 = _linear(d0, w, pre + ".final_proj", rnd) / D**0.25
    md1 = _linear(d1, w, pre + ".final_proj", rnd) / D**0.25
    op = _hook(rnd, "operand")
    sim = _hook(rnd, "grad")(op(md0) @ op(md1).transpose(1, 2))
    z0 = (d0 @ w[pre + ".matchability.weight"].t() + w[pre + ".matchability.bias"]).squeeze(-1)
    z1 = (d1 @ w[pre + ".matchability.weight"].t() + w[pre + ".matchability.bias"]).squeeze(-1)
    return sigmoid_log_double_softmax(sim, z0, z1), sim


def filter_matches(scores, th):
    """lightglue.py:293-309 (ties -> lowest index, like torch.max on CPU)."""
    inner = scores[:, :-1, :-1]
    max0, max1 = inner.max(2), inner.max(1)
    m0, m1 = max0.indices, max1.indices
    i0 = torch.arange(m0.shape[1], device=m0.device)[None]
    i1 = torch.arange(m1.shape[1], device=m1.device)[None]
    mutual0 = i0 == m1.gather(1, m0)
    mutual1 = i1 == m0.gather(1, m1)
    ms0 = torch.where(mutual0, max0.values.exp(), max0.values.new_zeros(()))
    ms1 = torch.where(mutual1, ms0.gather(1, m1), ms0.new_zeros(()))
    valid0 = mutual0 & (ms0 > th)
    valid1 = mutual1 & valid0.gather(1, m1)
    return torch.where(valid0, m0, -1), torch.where(valid1, m1, -1), ms0, ms1


# ----------------------------------------------------------------------------
# forward
# ----------------------------------------------------------------------------
def lightglue_forward(w, data, conf, rnd=_id, layer=None):
    """lightglue.py:412-543, training-mode path (no early stop / pruning).

    conf: dict with n_layers, num_heads, filter_threshold.
    layer: stands in for transformer_layer (same signature), e.g. the same layer under activation checkpointing.
    Returns the reference's pred dict.
    """
    layer = transformer_layer if layer is None else layer
    L, H = conf["n_layers"], conf["num_heads"]
    k0 = normalize_keypoints(data["keypoints0"], data["view0"]["image_size"])
    k1 = normalize_keypoints(data["keypoints1"], data["view1"]["image_size"])
    d0, d1 = data["descriptors0"], data["descriptors1"]
    if "input_proj.weight" in w:
        d0, d1 = _linear(d0, w, "input_proj", rnd), _linear(d1, w, "input_proj", rnd)
    if conf.get("add_scale_ori"):  # lightglue.py:426-443
        k0 = torch.cat([k0, data["scales0"][..., None], data["oris0"][..., None]], -1)
        k1 = torch.cat([k1, data["scales1"][..., None], data["oris1"][..., None]], -1)
    th0, th1 = posenc_angles(w, k0), posenc_angles(w, k1)
    all0, all1 = [], []
    for i in range(L):
        d0, d1 = layer(d0, d1, th0, th1, w, i, H, rnd)
        all0.append(d0)
        all1.append(d1)
    scores, _ = match_assignment(d0, d1, w, L - 1, rnd)
    m0, m1, ms0, ms1 = filter_matches(scores, conf.get("filter_threshold", 0.0))
    return {
        "matches0": m0,
        "matches1": m1,
        "matching_scores0": ms0,
        "matching_scores1": ms1,
        "ref_descriptors0": torch.stack(all0, 1),
        "ref_descriptors1": torch.stack(all1, 1),
        "log_assignment": scores,
        "prune0": torch.ones_like(ms0) * L,
        "prune1": torch.ones_like(ms1) * L,
    }


# ----------------------------------------------------------------------------
# loss
# ----------------------------------------------------------------------------
def nll_terms(scores, gt_assignment, gt_m0, gt_m1, balancing=0.5):
    """models/utils/losses.py:6-25, 39-73.  Sparse restatement: no dense
    weight matrix, only the entries that carry non-zero weight."""
    B, M1, N1 = scores.shape
    M, N = M1 - 1, N1 - 1
    pos = gt_assignment.to(scores.dtype)
    neg0 = (gt_m0 == -1).to(scores.dtype)
    neg1 = (gt_m1 == -1).to(scores.dtype)
    num_pos = pos.sum((-1, -2)).clamp(min=1.0)
    num_neg0 = neg0.sum(-1).clamp(min=1.0)
    num_neg1 = neg1.sum(-1).clamp(min=1.0)
    nll_pos = -(scores[:, :M, :N] * pos).sum((-1, -2)) / num_pos
    nll_neg = -((scores[:, :M, N] * neg0).sum(-1) + (scores[:, M, :N] * neg1).sum(-1)) / (num_neg0 + num_neg1)
    nll = balancing * nll_pos + (1 - balancing) * nll_neg
    return nll, nll_pos, nll_neg, num_pos, (num_neg0 + num_neg1) / 2.0


def token_confidence_loss(w, i, d0, d1, la_now, la_final):
    """lightglue.py:81-94."""
    pre = f"token_confidence.{i}.token.0"
    logit0 = (d0.detach() @ w[pre + ".weight"].t() + w[pre + ".bias"]).squeeze(-1)
    logit1 = (d1.detach() @ w[pre + ".weight"].t() + w[pre + ".bias"]).squeeze(-1)
    la_now, la_final = la_now.detach(), la_final.detach()
    c0 = la_final[:, :-1, :].max(-1).indices == la_now[:, :-1, :].max(-1).indices
    c1 = la_final[:, :, :-1].max(-2).indices == la_now[:, :, :-1].max(-2).indices
    bce = F.binary_cross_entropy_with_logits
    return (
        bce(logit0, c0.to(logit0.dtype), reduction="none").mean(-1)
        + bce(logit1, c1.to(logit1.dtype), reduction="none").mean(-1)
    ) / 2.0


def lightglue_loss(w, pred, data, conf, training=True, rnd=_id):
    """lightglue.py:578-627 (training branch; metrics omitted)."""
    L = pred["ref_descriptors0"].shape[1]
    gamma = conf.get("loss", {}).get("gamma", 1.0)
    bal = conf.get("loss", {}).get("nll_balancing", 0.5)
    gt = (data["gt_assignment"], data["gt_matches0"], data["gt_matches1"])

    def head(i):
        return match_assignment(pred["ref_descriptors0"][:, i], pred["ref_descriptors1"][:, i], w, i, rnd)[0]

    nll, nll_pos, nll_neg, num_pos, num_neg = nll_terms(head(L - 1), *gt, balancing=bal)
    losses = {
        "total": nll,
        "last": nll.clone().detach(),
        "assignment_nll": nll,
        "nll_pos": nll_pos,
        "nll_neg": nll_neg,
        "num_matchable": num_pos,
        "num_unmatchable": num_neg,
    }
    if training:
        losses["confidence"] = 0.0
    losses["row_norm"] = pred["log_assignment"].exp()[:, :-1].sum(2).mean(1)
    sum_weights = 1.0
    for i in range(L - 1):
        la = head(i)
        nll_i = nll_terms(la, *gt, balancing=bal)[0]
        weight = gamma ** (L - i - 1) if gamma > 0.0 else i + 1
        sum_weights += weight
        losses["total"] = losses["total"] + nll_i * weight
        losses["confidence"] = losses["confidence"] + token_confidence_loss(
            w, i, pred["ref_descriptors0"][:, i], pred["ref_descriptors1"][:, i], la, pred["log_assignment"]
        ) / (L - 1)
    losses["total"] = losses["total"] / sum_weights
    if training:
        losses["total"] = losses["total"] + losses["confidence"]
    return losses


# ----------------------------------------------------------------------------
# other assignment heads on the path (BASELINE.json config 5 / SURVEY 8a a15, a16)
# ----------------------------------------------------------------------------
def log_double_softmax(sim, bin_score):
    """models/matchers/gluestick.py:772-783. sim [B,M,N], bin_score scalar."""
    B, M, N = sim.shape
    beta = torch.as_tensor(bin_score, dtype=sim.dtype)
    s0 = torch.log_softmax(torch.cat([sim, beta.expand(B, M, 1)], 2), 2)
    s1 = torch.log_softmax(torch.cat([sim, beta.expand(B, 1, N)], 1), 1)
    scores = sim.new_zeros(B, M + 1, N + 1)
    scores[:, :M, :N] = (s0[:, :, :N] + s1[:, :M, :]) / 2
    scores[:, :M, N] = s0[:, :, N]
    scores[:, M, :N] = s1[:, M, :]
    return scores


def gluestick_attention(query, key, value):
    """models/matchers/gluestick.py:524-529. query [B, dh, H, N], key/value [B, dh, H, M] (GlueStick keeps channels
    first and splits heads as channel = d * H + h, gluestick.py:544-547) -> [B, dh, H, N]; fp32-forced in the reference."""
    dh = query.shape[1]
    scores = torch.einsum("bdhn,bdhm->bhnm", query, key) / dh**0.5
    return torch.einsum("bhnm,bdhm->bdhn", torch.softmax(scores, -1), value)


def gluestick_mha(x, source, params, num_heads=4):
    """MultiHeadedAttention.forward (gluestick.py:532-551) with query = x, key = value = source ([B, D, N] / [B, D, M]);
    params: merge.{weight,bias}, proj.{0,1,2}.{weight,bias} (Conv1d k=1 == Linear over channels)."""
    lin = lambda t, i: torch.einsum("oc,bcn->bon", params[f"proj.{i}.weight"][:, :, 0], t) + \
        params[f"proj.{i}.bias"][None, :, None]  # noqa: E731
    B, D = x.shape[:2]
    dh = D // num_heads
    q, k, v = lin(x, 0), lin(source, 1), lin(source, 2)
    o = gluestick_attention(q.view(B, dh, num_heads, -1), k.view(B, dh, num_heads, -1), v.view(B, dh, num_heads, -1))
    o = o.contiguous().view(B, D, -1)
    return torch.einsum("oc,bcn->bon", params["merge.weight"][:, :, 0], o) + params["merge.bias"][None, :, None]


def log_optimal_transport(scores, alpha, iters):
    """gluefactory_nonfree/superglue.py:186-214, restated from the algorithm:
    log-domain Sinkhorn on the (M+1)x(N+1) coupling with dustbin score alpha,
    marginals mu = [1..1, N]/(M+N), nu = [1..1, M]/(M+N); result multiplied by
    (M+N)."""
    B, M, N = scores.shape
    alpha = torch.as_tensor(alpha, dtype=scores.dtype)
    Z = scores.new_empty(B, M + 1, N + 1)
    Z[:, :M, :N] = scores
    Z[:, :M, N] = alpha
    Z[:, M, :] = alpha
    norm = -math.log(M + N)
    log_mu = scores.new_full((B, M + 1), norm)
    log_mu[:, M] = math.log(N) + norm
    log_nu = scores.new_full((B, N + 1), norm)
    log_nu[:, N] = math.log(M) + norm
    u, v = torch.zeros_like(log_mu), torch.zeros_like(log_nu)
    for _ in range(iters):
        u = log_mu - torch.logsumexp(Z + v[:, None, :], 2)
        v = log_nu - torch.logsumexp(Z + u[:, :, None], 1)
    return Z + u[:, :, None] + v[:, None, :] - norm


# ----------------------------------------------------------------------------
# full training step on the CPU (the cpu_baseline / --impl reference leg)
# ----------------------------------------------------------------------------
def train_step_cpu(w, data, conf, lr=1e-4, adam_state=None):
    """One optimiser step = forward + loss + backward + Adam, restating
    train.py:466-517 around the matcher.  `w` holds leaf tensors with
    requires_grad; they are updated in place."""
    for p in w.values():
        p.grad = None
    pred = lightglue_forward(w, data, conf)
    losses = lightglue_loss(w, pred, data, conf, training=True)
    loss = losses["total"].mean()
    loss.backward()
    if adam_state is None:
        adam_state = {"opt": torch.optim.Adam([p for p in w.values() if p.requires_grad], lr=lr)}
    adam_state["opt"].step()
    return loss.detach(), adam_state
