"""GPU: the shared-qk cross-attention backward (lgb200_attn_bwd with q == k and dq == dk, one pass over the similarity
both directions share) against fp64 autograd of the reference's cross-attention (lightglue.py:207-216: one `sim`, a
softmax over each of its two axes), against the generic backward's dq + dk, and in a training step that must replay
bit for bit as a CUDA graph.  bf16 tolerances as in test_gpu_kernels.test_attention_forward_backward."""
import pytest
import torch

from gluefactory_b200 import _lib, ops, synthetic
from gluefactory_b200.matchers.lightglue import LightGlue
from gluefactory_b200.trainer import MatcherTrainer
from tests.util import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"
SHAPES = [(2, 128, 4), (2, 200, 2), (3, 512, 4), (2, 2048, 2)]  # (pairs, N, heads)


def _rand(*shape, seed, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(torch.bfloat16).to(DEV)


def _cross_ref(qk, v, B):
    """fp64 restatement of lightglue.py:207-216 on [2B, N, H, 64] tensors (image0 = batches :B, image1 = B:)."""
    qk0, qk1 = qk[:B].permute(0, 2, 1, 3), qk[B:].permute(0, 2, 1, 3)
    v0, v1 = v[:B].permute(0, 2, 1, 3), v[B:].permute(0, 2, 1, 3)
    sim = torch.einsum("bhid,bhjd->bhij", qk0, qk1) * 0.125
    m0 = torch.softmax(sim, -1) @ v1
    m1 = torch.softmax(sim.transpose(-2, -1), -1) @ v0
    return torch.cat([m0, m1], 0).permute(0, 2, 1, 3)


def _inputs(B, N, H):
    qk = _rand(2 * B, N, H, 64, seed=1, scale=1.5)
    v = _rand(2 * B, N, H, 64, seed=2)
    go = _rand(2 * B, N, H, 64, seed=3)
    out, lse = ops.attn_fwd(qk, qk, v, B, 0.125)
    return qk, v, go, out, lse


@pytest.mark.parametrize("B,N,H", SHAPES)
def test_shared_qk_backward_matches_fp64_reference(B, N, H):
    qk, v, go, out, lse = _inputs(B, N, H)
    dqk, dv = ops.attn_bwd_shared_qk(qk, v, out, lse, go, 0.125)
    qr, vr = (t.detach().double().requires_grad_(True) for t in (qk, v))
    ref = _cross_ref(qr, vr, B)
    ref.backward(go.double())
    assert rel_err(out, ref) < 1e-2
    assert rel_err(dqk, qr.grad) < 1e-2
    assert rel_err(dv, vr.grad) < 1e-2


@pytest.mark.parametrize("B,N,H", SHAPES)
def test_shared_qk_backward_matches_generic_dq_plus_dk(B, N, H):
    qk, v, go, out, lse = _inputs(B, N, H)
    l0 = _lib.launch_count
    dqk, dv = ops.attn_bwd_shared_qk(qk, v, out, lse, go, 0.125)
    assert _lib.launch_count - l0 == 2  # prep + the shared sweep
    dq, dk, dv_ref = ops.attn_bwd(qk, qk, v, out, lse, go, B, 0.125)  # separate outputs: the generic kernels
    assert rel_err(dqk, dq.double() + dk.double()) < 1e-2
    assert rel_err(dv, dv_ref) < 1e-2
    again, dv2 = ops.attn_bwd_shared_qk(qk, v, out, lse, go, 0.125)  # fixed summation order
    assert torch.equal(again, dqk) and torch.equal(dv2, dv)


def test_training_step_replays_bit_for_bit():
    """Eager steps and CUDA-graph replays of a bf16 training step (M == N: the shared-qk backward runs in every
    layer) leave bit-identical parameters and losses."""
    conf = dict(synthetic.DEFAULT_CONF, n_layers=2)
    batches = [synthetic.to_device(synthetic.make_pairs(2, 256, seed=70 + i), DEV) for i in range(3)]

    def run(graphed):
        model = LightGlue(dict(conf, precision="bf16"))
        model.load_state_dict(synthetic.make_weights(conf, seed=71), strict=False)
        tr = MatcherTrainer(model.to(DEV).train(), lr=1e-3)
        tr.step(batches[0])
        if graphed:
            tr.capture(batches[0], DEV, warmup=0)
        losses = [(tr.step_graphed(b) if graphed else tr.step(b))[0].clone() for b in batches]
        torch.cuda.synchronize()
        return tr.fp.flat.clone(), torch.stack(losses)

    p_eager, l_eager = run(False)
    p_graph, l_graph = run(True)
    assert torch.equal(l_graph, l_eager)
    assert torch.equal(p_graph, p_eager)
