"""GPU: the fp32 parity path's attention (csrc/attn_simt.cu: the CUDA-core forward, the packed forward, attn_delta and
the dQ / dK-dV backward kernels) at head dim 64, and the rotary split forward at head dim 64
(lgb200_rope_split_fwd), element by element against fp64, at the launches the matchers make in `precision: "fp32"`, at
the benchmark's shapes and at tile edges.

Units and scale: U32 = 2^-24 (one fp32 rounding); scale = hd^-1/2 (1/8 at head dim 64, 32^-1/2 at 32).

Reference (attn_ref_f32, per sequence, fp64 on the operands the kernel read).  What the kernel does, row by row:
  qr = fl(q * scale)        ONE rounding before the dot product.  Exact at head dim 64 (scale = 2^-3); at head dim 32
                            it moves each term by U32 |q_d k_d| scale, and the fp32 value of scale itself by U32 more.
  s  = qr . k               two chains of hd/2 fmas (one per thread of the row's pair), then one shuffle add:
                            off by (hd/2 + 1) U32 scale |q||k| at most.  With the two roundings above the S error is at
                            most (hd/2 + 3) U32 scale |q||k| <= hd U32 scale |q||k| for hd >= 6.
  p  = expf(s - m)          expf is within 2 ulp (4 U32); the fp32 difference adds U32 |s - m| <= U32 (|S| + |m|):
       eps = hd U32 scale (|q| |k|) + 4 U32 + 3 U32 (|S| + |max S|)   (relative error of each p; the factor 3 leaves
                                                                      room for the second-order terms)
  running maximum           at each new maximum (R per row: the keys, after the first, that exceed every key before
                            them, counted on the fp64 logits in key order) o and l are both multiplied by
                            a = expf(m_old - s).  The error of a cancels in o / l; the two fp32 multiplies do not.
  o, l                      Nk fmas / adds each, plus R rescales: (Nk + R) U32 of P|V| and of l.
  out = o * (1 / l)         two roundings: 2 U32 |O|.
  underflow                 a p below fp32's normal range (|S| ~ 80: expf(-160) is 0) is off by up to itself, which is
                            below TINY = 2^-126 (l >= 1, the maximum's p being 1): an absolute TINY per key.
    O     2 (P eps)|V| + 2 (P eps)1 |O| + (2 Nk + 2 R + 64) U32 P|V| + U32 |O| + TINY sum_j |v_j|
    lse = m + logf(l)       l is off by its chain, by the errors of the R factors a (each expf: 4 U32, its argument
                            U32 |m_old - s|, the multiply U32; the arguments sum to at most |m| + max|S|), and logf and
                            the add round:
          (P eps)1 + (2 Nk + 6 R + 64) U32 + 4 U32 (|max S| + |lse|) + U32 max|S|     (absolute)
Backward (the dQ kernel over keys, the dK / dV kernel over queries, both recompute s):
  p  = expf(s - L)          L is the STORED lse, off by blse: p is off by eps_b = eps + blse + U32 |lse| relative.
  dp = dO . v               (hd/2 + 1) U32 |dO||v|;  delta = rowsum(dO o O) of the stored O (attn_delta: 8 lanes of hd/8
                            channels, then 3 shuffle adds): (hd/8 + 3) U32 rowsum(|dO||O|); dp - delta and the two
                            multiplies of ds = p (dp - delta) scale: 3 U32 more.
       Bd = |dO| |V|^T + rowsum(|dO| o |O|),  A = P o Bd   A bounds P |dp - delta| and every rounding above
       ds is off by A (eps_b + (hd + 5) U32) scale, plus TINY Bd scale where p underflows
    dQ    scale (A (2 (eps_b + (hd + 5) U32) + (2 Nk + 64) U32) + TINY Bd) |K| + U32 |dQ|     (the Nk-fma chain of dq)
    dK    scale (A (2 (eps_b + (hd + 5) U32) + (2 Nq + 64) U32) + TINY Bd)^T |Q| + U32 |dK|  (the Nq-fma chain of dk)
    dV    (2 P eps_b + (2 Nq + 64) U32 P + TINY)^T |dO| + U32 |dV|
  Shared query / key (LightGlue's cross-attention, fp32: two directions into separate dq / dk, then dq.add_(dk)):
    |dqk - (dQ + dK)| <= bdQ + bdK + U32 |dQ + dK|, dQ of the tensor's own direction and dK of the other's.
The bounds are worst-case sums of every rounding.  Measured errors sit one to four orders of magnitude below them, and
a kernel that drops or misroutes a tile, a batch or a channel block is off by far more than they allow.

Rotary split (lightglue.py:42-49, 156-160; Wqkv feature h*192 + d*3 + {q,k,v}, theta [T, 32], pairs (2i, 2i+1)):
  |got - ref| <= u_out |ref| + 1e-5 (|a| + |b|) for each rotated pair (a, b); v copied, u_out |ref| (u_out = 2^-8 bf16,
  2^-23 fp32).  Controls that must fail: the pairing by halves (i, i + 32), and the angles the head-dim-32 kernel would
  apply to this buffer (theta read with a row stride of 16, pair p of a 64-channel head given angle p mod 16).

A. Launch census: ops.attn_fwd, attn_bwd, attn_bwd_shared_qk, attn_fwd_varlen and rope_fwd are wrapped by recording
   shims while one fp32 training step (forward, loss, backward) runs per configuration (LightGlue 256/4, 128/4 and 512/8
   channels / heads with M == N and M != N, GlueStick at 256 and 128 channels, SuperGlue), and one fp32 packed eval call
   of each matcher.  Each call is reduced to (entry, dtype, head dim, H, kv_shift: 0 / half of B / other, Nq == Nk);
   every signature seen must be a row of FP32_ROWS, and every row is seen or marked contract-only.
B. Uniform forward + backward (fp32, head dim 64) into guarded buffers, per sequence against fp64: the benchmark's
   launch (64 sequences x 2048, 4 heads, self and cross, a fixed subset of sequences checked, the guards over all),
   GlueStick's (3072 nodes self; cross 3072 x 2600 at kv_shift 0, one launch per direction), every pair of tile edges
   Nq, Nk in EDGES, 8 heads at three edge pairs, B = 3 with kv_shift 1 (the dK / dV kernel's batch map
   qb = (kb - kv_shift) mod B, which the matchers' symmetric shifts cannot tell from +kv_shift), and the logit regimes
   spike / rising / zero_q / large (|S| ~ 80: expf(m - s) underflows to 0 at the running-maximum rescale and for the low
   keys; outputs must stay finite).  Large launches run twice and must agree bit for bit.
C. The fp32 shared query / key backward against the fp64 total gradient.
D. The packed forward (lengths 1, 63, 64, 65, 127, 2048, 0 with guard rows, self and cross) at head dims 64 and 32.
E. Rotary split forward at head dim 64: T in {131072, 1003, 7, 1}, H in {4, 8}, bf16 and fp32, deterministic.
F. CPU negative controls: each check rejects a wrong answer built from its own reference.

Budget: recorded by the module fixture (wall time and peak device memory); see profiles/attention_fp32_tests_h100.md.
"""
import time

import pytest
import torch

from gluefactory_b200 import _lib, ops, synthetic
from gluefactory_b200._lib import call, ptr, stream_ptr
from tests.test_gpu_attention_varlen import LENS, LSE_GUARD, OUT_GUARD, PARTNER, _layout
from tests.test_gpu_attention_varlen import _inputs as _varlen_inputs
from tests.test_gpu_tensor_core_kernels import (DEV, U32, _guarded, _guards_intact, _within, _Worst, check_attn_bwd,
                                                check_attn_fwd)
from tests.util import report

GPU = pytest.mark.gpu
HD = 64
SCALE = HD ** -0.5
BENCH_T = 2 * 32 * 2048  # both images of the benchmark's 32 pairs at 2048 keypoints
TINY = 2.0 ** -126  # smallest normal fp32: a p that underflows in expf (to a subnormal or 0) is off by less than this


@pytest.fixture(scope="module", autouse=True)
def _file_budget():
    """Wall time and peak device memory of this file (the machines running it are shared)."""
    if not torch.cuda.is_available():
        yield
        return
    torch.cuda.reset_peak_memory_stats()
    t = time.time()
    yield
    torch.cuda.synchronize()
    report("test_gpu_attention_fp32", seconds=time.time() - t, peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)


# ================================================================================================
# reference and checks (device-agnostic: the negative controls run them on the CPU)
# ================================================================================================
def attn_ref_f32(q, k, v, hd, out=None, do=None):
    """fp64 attention of one sequence, q [Nq,H,hd], k / v [Nk,H,hd] (the kernel's fp32 values), with the fp32 CUDA-core
    bounds of the module docstring.  With out (the kernel's stored O) and do: the backward too, delta taken from out."""
    scale = hd ** -0.5
    Q, K, V = (t.double().permute(1, 0, 2) for t in (q, k, v))  # [H, N, hd]
    Nq, Nk = Q.shape[1], K.shape[1]
    S = scale * (Q @ K.transpose(1, 2))
    m = S.amax(-1, keepdim=True)
    P = torch.softmax(S, -1)
    lse = torch.logsumexp(S, -1, keepdim=True)
    R = (S[..., 1:] > S.cummax(-1).values[..., :-1]).sum(-1, keepdim=True).double()  # new running maxima
    Smax = S.abs().amax(-1, keepdim=True)
    eps = (hd * U32 * scale) * (Q.abs() @ K.abs().transpose(1, 2)) + 4 * U32 + 3 * U32 * (S.abs() + m.abs())
    del S
    Pe = P * eps
    aV = V.abs()
    O = P @ V
    Pe1 = Pe.sum(-1, keepdim=True)
    blse = Pe1 + (2 * Nk + 6 * R + 64) * U32 + 4 * U32 * (m.abs() + lse.abs()) + U32 * Smax
    r = dict(O=O, lse=lse.squeeze(-1),
             bO=2 * (Pe @ aV) + 2 * Pe1 * O.abs() + (2 * Nk + 2 * R + 64) * U32 * (P @ aV) + U32 * O.abs()
             + TINY * aV.sum(-2, keepdim=True),
             blse=blse.squeeze(-1))
    del Pe
    if do is not None:
        dO, Os = do.double().permute(1, 0, 2), out.double().permute(1, 0, 2)
        adO = dO.abs()
        delta = (dO * Os).sum(-1, keepdim=True)
        dS = P * (dO @ V.transpose(1, 2) - delta)
        r["dV"], r["dQ"], r["dK"] = P.transpose(1, 2) @ dO, scale * (dS @ K), scale * (dS.transpose(1, 2) @ Q)
        del dS
        eps_b = eps + blse + U32 * lse.abs()
        del eps
        r["bdV"] = (2 * P * eps_b + (2 * Nq + 64) * U32 * P + TINY).transpose(1, 2) @ adO + U32 * r["dV"].abs()
        Bd = adO @ aV.transpose(1, 2) + (adO * Os.abs()).sum(-1, keepdim=True)
        A = P * Bd
        E = 2 * (eps_b + (hd + 5) * U32)
        del eps_b
        r["bdQ"] = scale * ((A * (E + (2 * Nk + 64) * U32) + TINY * Bd) @ K.abs()) + U32 * r["dQ"].abs()
        r["bdK"] = scale * ((A * (E + (2 * Nq + 64) * U32) + TINY * Bd).transpose(1, 2) @ Q.abs()) + U32 * r["dK"].abs()
    # back to the kernel's layouts: O / dQ [Nq,H,hd], dK / dV [Nk,H,hd], lse [H,Nq]
    return {key: (t if key in ("lse", "blse") else t.permute(1, 0, 2)) for key, t in r.items()}


def check_batches(q, k, v, do, out, lse, dq, dk, dv, shift, w, seqs=None):
    """Query batch b attends to key batch (b + shift) % B; the dK / dV of key batch kb come from query batch
    (kb - shift) % B.  Checks the query batches `seqs` (all when None) and the key batches they read."""
    B, hd = q.shape[0], q.shape[3]
    for b in (range(B) if seqs is None else seqs):
        kb = (b + shift) % B
        r = attn_ref_f32(q[b], k[kb], v[kb], hd, out[b], do[b])
        check_attn_fwd(out[b], lse[b], r, w)
        check_attn_bwd(dq[b], dk[kb], dv[kb], r, w)
        del r


def shared_qk_ref(r_own, r_other):
    """fp64 total gradient of a shared query / key tensor (dQ of its own direction plus dK of the other) and its bound:
    the two gradients' bounds and the fp32 rounding of their sum."""
    ref = r_own["dQ"] + r_other["dK"]
    return ref, r_own["bdQ"] + r_other["bdK"] + U32 * ref.abs()


# ================================================================================================
# inputs and launches
# ================================================================================================
def _gen(seed, dev):
    return torch.Generator(device=dev).manual_seed(seed)


def _inputs(B, Nq, Nk, H, regime, seed, hd=HD, dev=DEV):
    """fp32 q, k, v, dout [B, N, H, hd].  Regimes: randn (logits ~ randn * 1.5); spike (the last key, in a partial tile
    when Nk % 64 != 0, ~40 above every other logit); rising (logits climb ~60 over the keys: the running maximum grows
    in every key tile); zero_q (q = 0: every p is 1, out = mean of V); large (logits ~ +-80, the first key at -80: at
    the first +80 key the rescale expf(-160) underflows to 0, and so does every p of a -80 key)."""
    scale = hd ** -0.5
    g = _gen(seed, dev)
    q = torch.randn(B, Nq, H, hd, device=dev, generator=g) * 1.5
    k = torch.randn(B, Nk, H, hd, device=dev, generator=g)
    v = torch.randn(B, Nk, H, hd, device=dev, generator=g)
    do = torch.randn(B, Nq, H, hd, device=dev, generator=g)
    if regime == "spike":
        q[..., 0] = 8.0
        k[..., 0] = 0.0
        k[:, Nk - 1, :, 0] = 40.0 / (8.0 * scale)
    elif regime == "rising":
        q[..., 0] = 8.0
        k[..., 0] = torch.linspace(0.0, 60.0 / (8.0 * scale), Nk, device=dev)[None, :, None]
    elif regime == "zero_q":
        q.zero_()
        v = 1.25 + 0.1 * v
    elif regime == "large":
        q[..., 0] = 8.0
        sign = torch.where(torch.rand(Nk, device=dev, generator=g) < 0.5, -1.0, 1.0)
        sign[0] = -1.0
        k[..., 0] = (80.0 / (8.0 * scale)) * sign[None, :, None]
    return tuple(t.contiguous() for t in (q, k, v, do))


def _fwd_guarded(q, k, v, shift):
    B, Nq, H, hd = q.shape
    go = _guarded((B, Nq, H, hd), torch.float32, 2 * H * hd)
    gl = _guarded((B, H, Nq), torch.float32, 64)
    call("lgb200_attn_fwd_hd", ptr(q), ptr(k), ptr(v), ptr(go[1]), ptr(gl[1]), B, Nq, k.shape[1], H, shift,
         float(hd ** -0.5), _lib.F32, hd, stream_ptr())
    return go, gl


def _bwd_guarded(q, k, v, out, lse, do, shift):
    B, Nq, H, hd = q.shape
    Nk = k.shape[1]
    gq = _guarded((B, Nq, H, hd), torch.float32, 2 * H * hd)
    gk = _guarded((B, Nk, H, hd), torch.float32, 2 * H * hd)
    gv = _guarded((B, Nk, H, hd), torch.float32, 2 * H * hd)
    ws = torch.empty(_lib.load().lgb200_attn_bwd_ws_floats(B, Nq, Nk, H), device=DEV)
    call("lgb200_attn_bwd_hd", ptr(q), ptr(k), ptr(v), ptr(out), ptr(lse), ptr(do), ptr(gq[1]), ptr(gk[1]),
         ptr(gv[1]), ptr(ws), B, Nq, Nk, H, shift, float(hd ** -0.5), _lib.F32, hd, stream_ptr())
    return gq, gk, gv


def _run(B, Nq, Nk, H, shift, regime, seed, again=False, seqs=None, tag=""):
    q, k, v, do = _inputs(B, Nq, Nk, H, regime, seed)
    go, gl = _fwd_guarded(q, k, v, shift)
    out, lse = go[1], gl[1]
    gq, gk, gv = _bwd_guarded(q, k, v, out, lse, do, shift)
    if again:
        out2, lse2 = ops.attn_fwd(q, k, v, shift, SCALE)
        assert torch.equal(out, out2) and torch.equal(lse, lse2), (tag, "forward not bit-identical")
        del out2, lse2
        again_ = ops.attn_bwd(q, k, v, out, lse, do, shift, SCALE)
        assert all(torch.equal(a, b[1]) for a, b in zip(again_, (gq, gk, gv))), (tag, "backward not bit-identical")
        del again_
    for gb in (go, gl, gq, gk, gv):
        _guards_intact(gb, tag)
        assert torch.isfinite(gb[1]).all(), (tag, "non-finite output")
    w = _Worst(tag)
    check_batches(q, k, v, do, out, lse, gq[1], gk[1], gv[1], shift, w, seqs)
    w.report()


# ================================================================================================
# A. launch census
# ================================================================================================
F32 = "f32"
# (entry, dtype, head dim, H, kv_shift kind, Nq == Nk) -> where it is tested.  kv_shift kind: "0", "half" (B / 2: both
# directions of cross-attention in one launch) or "other"; attn_fwd_varlen: "self" (each segment on its own keys) or
# "partner"; rope_fwd has neither.
HERE = "this file"
HD32 = "test_gpu_attention_hd32.py::test_hd32_fp32_cuda_core_path"
CONTRACT = "contract-only"
FP32_ROWS = {}
for _H in (4, 8):
    FP32_ROWS.update({
        ("attn_fwd", F32, 64, _H, "0", True): HERE, ("attn_fwd", F32, 64, _H, "half", True): HERE,
        ("attn_fwd", F32, 64, _H, "0", False): HERE,
        ("attn_bwd", F32, 64, _H, "0", True): HERE, ("attn_bwd", F32, 64, _H, "half", True): HERE,
        ("attn_bwd", F32, 64, _H, "0", False): HERE,
        ("attn_bwd_shared_qk", F32, 64, _H, "half", True): HERE,
        ("attn_fwd_varlen", F32, 64, _H, "self", "-"): HERE, ("attn_fwd_varlen", F32, 64, _H, "partner", "-"): HERE,
        ("rope_fwd", F32, 64, _H, "-", "-"): HERE,
    })
FP32_ROWS.update({
    ("attn_fwd", F32, 32, 4, "0", True): HD32, ("attn_fwd", F32, 32, 4, "half", True): HD32,
    ("attn_fwd", F32, 32, 4, "0", False): HD32,
    ("attn_bwd", F32, 32, 4, "0", True): HD32, ("attn_bwd", F32, 32, 4, "half", True): HD32,
    ("attn_bwd", F32, 32, 4, "0", False): HD32,
    ("attn_fwd_varlen", F32, 32, 4, "self", "-"): HERE, ("attn_fwd_varlen", F32, 32, 4, "partner", "-"): HERE,
    ("rope_fwd", F32, 32, 4, "-", "-"): "test_gpu_rope_hd32.py::test_rope_fwd_hd32_against_fp64",
    # B = 3, kv_shift 1 (test_b3_shift_one_batch_map): the documented batch map, which no matcher launches
    ("attn_fwd", F32, 64, 4, "other", False): CONTRACT, ("attn_bwd", F32, 64, 4, "other", False): CONTRACT,
})
_DT = {torch.float32: F32, torch.bfloat16: "bf16"}


def _signature(name, args):
    if name == "rope_fwd":
        qkv, _, H = args[:3]
        return (name, _DT[qkv.dtype], qkv.shape[1] // (3 * H), H, "-", "-")
    q = args[0]
    if name == "attn_fwd_varlen":
        return (name, _DT[q.dtype], q.shape[2], q.shape[1], "self" if torch.equal(args[3], args[5]) else "partner", "-")
    if name == "attn_bwd_shared_qk":
        return (name, _DT[q.dtype], q.shape[3], q.shape[2], "half", True)
    k = args[1]
    shift = args[3] if name == "attn_fwd" else args[6]
    kind = "0" if shift == 0 else ("half" if 2 * shift == q.shape[0] else "other")
    return (name, _DT[q.dtype], q.shape[3], q.shape[2], kind, q.shape[1] == k.shape[1])


SHIMMED = ("attn_fwd", "attn_bwd", "attn_bwd_shared_qk", "attn_fwd_varlen", "rope_fwd")


def _record(monkeypatch, sigs):
    for name in SHIMMED:
        orig = getattr(ops, name)

        def shim(*args, _orig=orig, _name=name, **kw):
            assert not kw, (_name, sorted(kw))  # the signatures read positional arguments
            sigs.add(_signature(_name, args))
            return _orig(*args, **kw)

        monkeypatch.setattr(ops, name, shim)


def check_census(seen):
    """seen: {configuration: set of signatures}.  Every signature is a row of FP32_ROWS; every row is seen by some
    configuration or is contract-only."""
    missing = sorted({(cfg, s) for cfg, sigs in seen.items() for s in sigs if s not in FP32_ROWS}, key=repr)
    assert not missing, "fp32 launch signatures outside the table:\n" + "\n".join(f"  {c}: {s!r}" for c, s in missing)
    everything = set().union(*seen.values()) if seen else set()
    unseen = sorted((s for s, where in FP32_ROWS.items() if s not in everything and where != CONTRACT), key=repr)
    assert not unseen, f"table rows no configuration launches: {unseen}"


def _lightglue(D, H, M, N, train):
    from gluefactory_b200.matchers.lightglue import LightGlue

    conf = dict(synthetic.DEFAULT_CONF, descriptor_dim=D, input_dim=D, num_heads=H, n_layers=2, precision="fp32")
    model = LightGlue(conf)
    model.load_state_dict(synthetic.make_weights(conf, seed=D + H), strict=False)
    data = synthetic.to_device(synthetic.make_pairs(2, N, seed=M + N, D=D, M=M), DEV)
    if train:
        model = model.to(DEV).train()
        pred = model(data)
        losses, _ = model.loss(pred, data)
        losses["total"].mean().backward()
    else:
        model = model.to(DEV).eval()
        data.update(num_keypoints0=torch.tensor([M, M - 5]), num_keypoints1=torch.tensor([N - 3, N]))
        with torch.no_grad():
            model(data)


def _gluestick(D, M, N, train):
    from gluefactory_b200.matchers.gluestick import GlueStick

    conf = {"GNN_layers": ["self", "cross"], "descriptor_dim": D, "input_dim": D, "filter_threshold": 0.2}
    model = GlueStick(dict(conf, precision="fp32"))
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=D), strict=True)
    d = synthetic.make_gluestick_batch(2, max(M, N), 40, seed=D + M, D=D)
    if M != N:  # view 1 cut to N points (its lines are made of its first 80), labels cut the same way
        for key in ("keypoints1", "descriptors1", "keypoint_scores1"):
            d[key] = d[key][:, :N].contiguous()
        d["gt_matches0"] = torch.where(d["gt_matches0"] >= N, torch.full_like(d["gt_matches0"], -1), d["gt_matches0"])
        d["gt_matches1"] = d["gt_matches1"][:, :N].contiguous()
        d["gt_assignment"] = d["gt_assignment"][:, :, :N].contiguous()
    data = synthetic.to_device(d, DEV)
    if train:
        model = model.to(DEV).train()
        pred = model(data)
        losses, _ = model.loss(pred, data)
        losses["total"].mean().backward()
    else:
        model = model.to(DEV).eval()
        data["num_lines0"] = torch.tensor([40, 37])
        with torch.no_grad():
            model(data)


def _superglue(M, N, train):
    from gluefactory_b200.matchers.superglue import SuperGlue

    conf = {"GNN_layers": ["self", "cross"], "filter_threshold": 0.2}
    model = SuperGlue(dict(conf, weights=None, precision="fp32"))
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=M + N), strict=True)
    data = synthetic.to_device(synthetic.make_superglue_batch(2, M, N, seed=M + 3 * N), DEV)
    if train:
        model = model.to(DEV).train()
        pred = model(data)
        losses, _ = model.loss(pred, data)
        losses["total"].mean().backward()
    else:
        model = model.to(DEV).eval()
        data.update(num_keypoints0=torch.tensor([M - 7, M]), num_keypoints1=torch.tensor([N, N - 1]))
        with torch.no_grad():
            model(data)


CENSUS = {  # keypoint counts off the tile edges; M != N configurations for the two-launch cross-attention
    "lightglue d256 h4": lambda: _lightglue(256, 4, 200, 200, True),
    "lightglue d256 h4 M!=N": lambda: _lightglue(256, 4, 168, 200, True),
    "lightglue d128 h4": lambda: _lightglue(128, 4, 200, 200, True),
    "lightglue d128 h4 M!=N": lambda: _lightglue(128, 4, 168, 200, True),
    "lightglue d512 h8": lambda: _lightglue(512, 8, 200, 200, True),
    "lightglue d512 h8 M!=N": lambda: _lightglue(512, 8, 168, 200, True),
    "gluestick d256 M!=N": lambda: _gluestick(256, 200, 168, True),
    "gluestick d128": lambda: _gluestick(128, 200, 200, True),
    "superglue M!=N": lambda: _superglue(150, 200, True),
    "lightglue d256 h4 packed eval": lambda: _lightglue(256, 4, 168, 200, False),
    "lightglue d128 h4 packed eval": lambda: _lightglue(128, 4, 168, 200, False),
    "lightglue d512 h8 packed eval": lambda: _lightglue(512, 8, 168, 200, False),
    "gluestick d256 packed eval": lambda: _gluestick(256, 200, 200, False),
    "gluestick d128 packed eval": lambda: _gluestick(128, 200, 200, False),
    "superglue packed eval": lambda: _superglue(150, 200, False),
}


@GPU
def test_fp32_launch_census(monkeypatch):
    """Every fp32 attention and rotary-split launch of the matchers' training steps and packed eval calls is a row of
    FP32_ROWS, and every row is launched (or is contract-only)."""
    seen = {}
    for cfg, step in CENSUS.items():
        sigs = set()
        with monkeypatch.context() as m:
            _record(m, sigs)
            step()
        torch.cuda.synchronize()
        seen[cfg] = sigs
        report(f"census fp32 {cfg}",
               **{f"s{i}": repr(s).replace(" ", "") for i, s in enumerate(sorted(sigs, key=repr))})
    assert all(all(s[1] == F32 for s in sigs) for sigs in seen.values()), "a bf16 launch in precision fp32"
    check_census(seen)


# ================================================================================================
# B. uniform forward + backward at head dim 64
# ================================================================================================
BENCH_SEQS = (0, 1, 31, 32, 63)


@GPU
@pytest.mark.parametrize("shift", [0, 32], ids=["self", "cross"])
def test_fp32_bench_shape(shift):
    """The step's launch in fp32: 64 sequences (32 pairs x 2 images) x 2048 tokens x 4 heads, forward and backward twice
    (bit-identical), guarded; sequences BENCH_SEQS (and the key batches they read) against fp64."""
    _run(64, 2048, 2048, 4, shift, "randn", seed=17 + shift, again=True, seqs=BENCH_SEQS,
         tag=f"fp32 bench shift={shift}")


@GPU
def test_fp32_gluestick_self_shape():
    """GlueStick's self-attention launch: 3072 nodes (2048 points + 1024 line endpoints) per image, 4 heads."""
    _run(2, 3072, 3072, 4, 0, "randn", seed=31, again=True, tag="fp32 gluestick self 3072")


@GPU
def test_fp32_gluestick_cross_shape():
    """GlueStick's cross-attention between views of different sizes: one launch per direction, kv_shift 0, Nq != Nk."""
    _run(2, 3072, 2600, 4, 0, "randn", seed=32, again=True, tag="fp32 gluestick cross 3072x2600")


EDGES = (1, 2, 63, 64, 65, 127, 128, 129, 1000, 2049)


@GPU
@pytest.mark.parametrize("Nk", EDGES)
@pytest.mark.parametrize("Nq", EDGES)
def test_fp32_tile_edges(Nq, Nk):
    _run(2, Nq, Nk, 4, (Nq + Nk) % 2, "randn", seed=Nq * 13 + Nk, tag=f"fp32 Nq={Nq} Nk={Nk}")


@GPU
@pytest.mark.parametrize("Nq,Nk", [(65, 129), (2049, 63), (129, 1000)])
def test_fp32_eight_heads_tile_edges(Nq, Nk):
    """LightGlue at 512 channels / 8 heads runs head dim 64 with H = 8 (census)."""
    _run(2, Nq, Nk, 8, (Nq + Nk) % 2, "randn", seed=Nq + 5 * Nk, tag=f"fp32 H=8 Nq={Nq} Nk={Nk}")


@GPU
@pytest.mark.parametrize("Nq,Nk", [(65, 129), (1000, 63)])
def test_fp32_b3_shift_one_batch_map(Nq, Nk):
    """B = 3, kv_shift 1: query batch b reads key batch b + 1; the dK / dV of key batch kb come from query batch
    kb - 1 (mod 3), which +kv_shift would get wrong."""
    _run(3, Nq, Nk, 4, 1, "randn", seed=Nq + Nk + 3, tag=f"fp32 B=3 shift=1 Nq={Nq} Nk={Nk}")


@GPU
@pytest.mark.parametrize("regime", ["spike", "rising", "zero_q", "large"])
@pytest.mark.parametrize("Nq,Nk", [(129, 65), (300, 1000)])
def test_fp32_logit_regimes(regime, Nq, Nk):
    _run(2, Nq, Nk, 2, 1, regime, seed=Nq + Nk, tag=f"fp32 {regime} Nq={Nq} Nk={Nk}")


# ================================================================================================
# C. shared query / key backward
# ================================================================================================
@GPU
@pytest.mark.parametrize("pairs,N,seqs", [(32, 2048, BENCH_SEQS), (2, 65, None), (3, 1000, None)])
def test_fp32_shared_qk_backward(pairs, N, seqs):
    """ops.attn_bwd_shared_qk in fp32 (LightGlue's cross block at M == N): dqk against dQ + dK of the shared tensor, dv
    against dV, per sequence; the benchmark shape twice (bit-identical)."""
    B2, H = 2 * pairs, 4
    qk, _, v, do = _inputs(B2, N, N, H, "randn", seed=pairs * 7 + N)
    out, lse = ops.attn_fwd(qk, qk, v, pairs, SCALE)
    dqk, dv = ops.attn_bwd_shared_qk(qk, v, out, lse, do, SCALE)
    if N == 2048:
        again, dv2 = ops.attn_bwd_shared_qk(qk, v, out, lse, do, SCALE)
        assert torch.equal(again, dqk) and torch.equal(dv2, dv)
        del again, dv2
    assert torch.isfinite(dqk).all() and torch.isfinite(dv).all()
    w = _Worst(f"fp32 shared_qk {pairs}x{N}")
    for b in (range(B2) if seqs is None else seqs):
        p = (b + pairs) % B2
        r_own = attn_ref_f32(qk[b], qk[p], v[p], HD, out[b], do[b])  # b's queries on p's keys: dQ_b
        r_other = attn_ref_f32(qk[p], qk[b], v[b], HD, out[p], do[p])  # p's queries on b's keys: dK_b, dV_b
        check_attn_fwd(out[b], lse[b], r_own, w)
        ref, bound = shared_qk_ref(r_own, r_other)
        w("dqk", (dqk[b].double() - ref).abs(), bound)
        w("dv", (dv[b].double() - r_other["dV"]).abs(), r_other["bdV"])
        del r_own, r_other, ref, bound
    w.report()


# ================================================================================================
# D. packed forward
# ================================================================================================
@GPU
@pytest.mark.parametrize("cross", [False, True], ids=["self", "cross"])
@pytest.mark.parametrize("hd,H", [(64, 4), (32, 4)])
def test_fp32_packed_forward_bounds(hd, H, cross):
    """lgb200_attn_fwd_varlen in fp32 on the layout of test_gpu_attention_varlen.py (sequences of 1, 63, 64, 65, 127,
    2048 and 0 tokens between guard rows), every sequence held to attn_ref_f32's bounds; no out row or lse entry outside
    the computed sequences is written."""
    offs, T = _layout()
    q, k, v = _varlen_inputs(T, H, hd, torch.float32, seed=hd + 11 * H + int(cross))
    partner = PARTNER if cross else list(range(len(LENS)))
    i32 = dict(device=DEV, dtype=torch.int32)
    q_off, q_len = torch.tensor(offs, **i32), torch.tensor(LENS, **i32)
    k_off, k_len = q_off[partner].contiguous(), q_len[partner].contiguous()
    out = torch.full_like(q, OUT_GUARD)
    lse = torch.full((H, T), LSE_GUARD, device=DEV)
    call("lgb200_attn_fwd_varlen", ptr(q), ptr(k), ptr(v), ptr(out), ptr(lse), ptr(q_off), ptr(q_len), ptr(k_off),
         ptr(k_len), len(LENS), max(LENS), T, T, H, float(hd ** -0.5), _lib.F32, hd, stream_ptr())
    torch.cuda.synchronize()
    written = torch.zeros(T, dtype=torch.bool)
    w = _Worst(f"fp32 packed hd{hd} H{H} {'cross' if cross else 'self'}")
    for s, (o, n) in enumerate(zip(offs, LENS)):
        ko, kn = offs[partner[s]], LENS[partner[s]]
        if n == 0 or kn == 0:
            continue
        written[o:o + n] = True
        r = attn_ref_f32(q[o:o + n], k[ko:ko + kn], v[ko:ko + kn], hd)
        check_attn_fwd(out[o:o + n], lse[:, o:o + n], r, w)
    w.report()
    assert written.any()
    wd = written.to(DEV)
    assert torch.equal(out[~wd], torch.full_like(out[~wd], OUT_GUARD)), "out rows outside the sequences were written"
    assert torch.equal(lse[:, ~wd], torch.full_like(lse[:, ~wd], LSE_GUARD)), "lse outside the sequences was written"


# ================================================================================================
# E. rotary split forward at head dim 64
# ================================================================================================
def _u(dtype):
    return 2.0 ** -8 if dtype == torch.bfloat16 else 2.0 ** -23


def _rope_inputs(T, H, dtype, seed, dev=DEV):
    g = _gen(seed, dev)
    qkv = torch.randn(T, H * 3 * HD, device=dev, generator=g).to(dtype)
    theta = (torch.rand(T, HD // 2, device=dev, generator=g) * 8 - 4).contiguous()  # |kp Wr^T| of a few radians
    return qkv, theta


def _rot(t, th, pairs):
    """t [T, H, 64] fp64 rotated by th [T, 1 or H, 32]: pairs "adjacent" (2i, 2i+1) (lightglue.py:42-49) or "halves"
    (i, i + 32), the convention the kernel must NOT implement."""
    c, s = torch.cos(th), torch.sin(th)
    out = torch.empty_like(t)
    if pairs == "adjacent":
        a, b = t[..., 0::2], t[..., 1::2]
        out[..., 0::2], out[..., 1::2] = a * c - b * s, b * c + a * s
    else:
        a, b = t[..., :HD // 2], t[..., HD // 2:]
        out[..., :HD // 2], out[..., HD // 2:] = a * c - b * s, b * c + a * s
    return out


def _pair_sum(t, pairs):
    """|a| + |b| of the rotation pair each element belongs to."""
    a = t.abs()
    if pairs == "adjacent":
        return a[..., 0::2].repeat_interleave(2, -1) + a[..., 1::2].repeat_interleave(2, -1)
    return torch.cat([a[..., :HD // 2] + a[..., HD // 2:]] * 2, -1)


def rope_angles(theta, control=None):
    """[T, 1, 32] fp64 angle of each rotation pair; control "hd32": the angles the head-dim-32 kernel applies to this
    buffer (its Wqkv layout h*96 + d*3 of 2H heads is this memory order; it reads theta with a row stride of 16 and
    gives pair p of a 64-channel head -- pair p mod 16 of 32-channel head 2h + p // 16 -- angle
    theta_flat[16 t + p mod 16])."""
    th = theta.double()
    if control == "hd32":
        T = th.shape[0]
        idx = 16 * torch.arange(T, device=th.device)[:, None] + torch.arange(HD // 2, device=th.device) % 16
        th = th.reshape(-1)[idx]
    return th[:, None, :]


def check_rope(q, k, v, qkv, theta, H, dtype, control=None, chunk=16384):
    """(all within the bound, worst err / bound) of the rotated q, k and copied v [T, H*64] against the fp64 rotation;
    control None (the kernel's contract), "halves" or "hd32" (module docstring).  In token chunks (bounded memory)."""
    pairs = "halves" if control == "halves" else "adjacent"
    ok, worst = True, 0.0
    for t0 in range(0, qkv.shape[0], chunk):
        x = qkv[t0:t0 + chunk].double()
        T = x.shape[0]
        x = x.view(T, H, HD, 3)
        th = rope_angles(theta[t0:t0 + chunk], control)
        for got, src, rot in ((q, x[..., 0], True), (k, x[..., 1], True), (v, x[..., 2], False)):
            ref = _rot(src, th, pairs) if rot else src
            bound = _u(dtype) * ref.abs() + (1e-5 * _pair_sum(src, pairs) if rot else 0.0)
            err = (got[t0:t0 + chunk].double().view(T, H, HD) - ref).abs()
            ok = ok and bool((err <= bound).all())
            worst = max(worst, float((err / bound.clamp(min=1e-30)).max()))
    return ok, worst


@GPU
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
@pytest.mark.parametrize("H", [4, 8])
@pytest.mark.parametrize("T", [BENCH_T, 1003, 7, 1])
def test_rope_fwd_hd64_against_fp64(T, H, dtype):
    qkv, theta = _rope_inputs(T, H, dtype, seed=3 * T + H)
    q, k, v = ops.rope_fwd(qkv, theta, H)
    assert q.shape == (T, H * HD) and q.dtype == dtype
    ok, worst = check_rope(q, k, v, qkv, theta, H, dtype)
    report(f"rope hd64 T={T} H={H} {_DT[dtype]}", max_err_over_bound=worst)
    assert ok, worst
    # controls: the pairing by halves, and the head-dim-32 kernel's angles
    assert not check_rope(q, k, v, qkv, theta, H, dtype, control="halves")[0]
    assert not check_rope(q, k, v, qkv, theta, H, dtype, control="hd32")[0]
    q2, k2, v2 = ops.rope_fwd(qkv, theta, H)
    assert torch.equal(q, q2) and torch.equal(k, k2) and torch.equal(v, v2)


# ================================================================================================
# F. CPU negative controls
# ================================================================================================
def test_fp32_checks_reject_wrong_answers():
    """Each check rejects a wrong answer built from its own reference: a dropped partial last key tile (out, lse, dQ),
    a dropped query tile (dK, dV), bf16-rounded outputs, dQ + dK with dK missing."""
    w = lambda name, e, b: _within(e, b, name, log=False)  # noqa: E731
    q, k, v, do = (t[0] for t in _inputs(1, 70, 150, 2, "randn", 6, dev="cpu"))
    out = attn_ref_f32(q, k, v, HD)["O"].float()
    r = attn_ref_f32(q, k, v, HD, out, do)
    f = lambda t: t.float()  # noqa: E731
    check_attn_fwd(f(r["O"]), f(r["lse"]), r, w)
    check_attn_bwd(f(r["dQ"]), f(r["dK"]), f(r["dV"]), r, w)
    # the partial last key tile (keys 128..149) left out: out, lse, dQ
    r_k = attn_ref_f32(q, k[:128], v[:128], HD, out, do)
    with pytest.raises(AssertionError):
        check_attn_fwd(f(r_k["O"]), f(r["lse"]), r, w)
    with pytest.raises(AssertionError):
        check_attn_fwd(f(r["O"]), f(r_k["lse"]), r, w)
    with pytest.raises(AssertionError):
        check_attn_bwd(f(r_k["dQ"]), f(r["dK"]), f(r["dV"]), r, w)
    # the partial last query tile (queries 64..69) left out: dK, dV
    r_q = attn_ref_f32(q[:64], k, v, HD, out[:64], do[:64])
    with pytest.raises(AssertionError):
        check_attn_bwd(f(r["dQ"]), f(r_q["dK"]), f(r["dV"]), r, w)
    with pytest.raises(AssertionError):
        check_attn_bwd(f(r["dQ"]), f(r["dK"]), f(r_q["dV"]), r, w)
    # bf16-rounded outputs and gradients (what the tensor-core path would store)
    bf = lambda t: t.to(torch.bfloat16).float()  # noqa: E731
    with pytest.raises(AssertionError):
        check_attn_fwd(bf(r["O"]), f(r["lse"]), r, w)
    for i in range(3):
        grads = [f(r[n]) for n in ("dQ", "dK", "dV")]
        grads[i] = bf(grads[i])
        with pytest.raises(AssertionError):
            check_attn_bwd(*grads, r, w)
    # shared query / key: dQ + dK passes, dQ alone (dK missing) does not
    qk, _, v2, do2 = _inputs(2, 90, 90, 2, "randn", 8, dev="cpu")
    o2 = torch.stack([attn_ref_f32(qk[b], qk[1 - b], v2[1 - b], HD)["O"].float() for b in range(2)])
    r_own = attn_ref_f32(qk[0], qk[1], v2[1], HD, o2[0], do2[0])
    r_other = attn_ref_f32(qk[1], qk[0], v2[0], HD, o2[1], do2[1])
    ref, bound = shared_qk_ref(r_own, r_other)
    w("dqk", ((r_own["dQ"] + r_other["dK"]).float().double() - ref).abs(), bound)
    with pytest.raises(AssertionError):
        w("dqk", (r_own["dQ"].float().double() - ref).abs(), bound)


def test_fp32_check_rejects_the_plus_shift_batch_map():
    """B = 3, kv_shift 1: dK / dV of key batch kb from query batch kb - 1 pass; from kb + 1 (the +kv_shift map) fail."""
    w = lambda name, e, b: _within(e, b, name, log=False)  # noqa: E731
    B, shift = 3, 1
    q, k, v, do = _inputs(B, 70, 90, 1, "randn", 9, dev="cpu")
    out = torch.stack([attn_ref_f32(q[b], k[(b + shift) % B], v[(b + shift) % B], HD)["O"].float() for b in range(B)])
    lse = torch.stack([attn_ref_f32(q[b], k[(b + shift) % B], v[(b + shift) % B], HD)["lse"].float()
                       for b in range(B)])

    def grads(qb_of):
        dq, dk, dv = torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
        for b in range(B):
            dq[b] = attn_ref_f32(q[b], k[(b + shift) % B], v[(b + shift) % B], HD, out[b], do[b])["dQ"].float()
        for kb in range(B):
            qb = qb_of(kb)
            r = attn_ref_f32(q[qb], k[kb], v[kb], HD, out[qb], do[qb])
            dk[kb], dv[kb] = r["dK"].float(), r["dV"].float()
        return dq, dk, dv

    check_batches(q, k, v, do, out, lse, *grads(lambda kb: ((kb - shift) % B + B) % B), shift, w)
    with pytest.raises(AssertionError):
        check_batches(q, k, v, do, out, lse, *grads(lambda kb: (kb + shift) % B), shift, w)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float32], ids=["bf16", "fp32"])
def test_rope_check_rejects_the_halves_pairing_and_hd32_angles(dtype):
    """The fp64 rotation rounded once to the dtype passes; the same built with the pairing by halves, or with the angles
    the head-dim-32 kernel would read, fails."""
    T, H = 20, 4
    qkv, theta = _rope_inputs(T, H, dtype, seed=2, dev="cpu")

    def rotated(control=None):
        pairs = "halves" if control == "halves" else "adjacent"
        x = qkv.double().view(T, H, HD, 3)
        th = rope_angles(theta, control)
        return tuple(t.reshape(T, H * HD).to(dtype) for t in (_rot(x[..., 0], th, pairs), _rot(x[..., 1], th, pairs),
                                                               x[..., 2]))

    assert check_rope(*rotated(), qkv, theta, H, dtype)[0]
    for control in ("halves", "hd32"):
        assert not check_rope(*rotated(control), qkv, theta, H, dtype)[0], control
        assert not check_rope(*rotated(), qkv, theta, H, dtype, control=control)[0], control
