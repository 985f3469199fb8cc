"""GPU: the GEMMs' staged epilogue (shared-memory staging + TMA store / TMA reduce-add) against the register epilogue
that serves a C TMA cannot address.  Both apply the same per-element arithmetic and write or add every element once,
so a product written into a 16-byte-aligned C and into a C offset by one element must be bit-identical."""
import pytest
import torch

from gluefactory_b200 import _lib, ops
from gluefactory_b200._lib import BF16, F32, call, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _rand(*shape, seed=0, dtype=torch.float32, scale=1.0):
    g = torch.Generator().manual_seed(seed)
    return (torch.randn(*shape, generator=g) * scale).to(dtype).to(DEV)


def _pair(M, N, dtype, init=None):
    """Two [M, N] views of the same shape: one at a 16-byte-aligned base (TMA epilogue), one a single element past it
    (register epilogue).  Both start from `init` when given."""
    buf_a = torch.zeros(M * N + 16, device=DEV, dtype=dtype)
    buf_u = torch.zeros(M * N + 16, device=DEV, dtype=dtype)
    a, u = buf_a[:M * N].view(M, N), buf_u[1:1 + M * N].view(M, N)
    assert a.data_ptr() % 16 == 0 and u.data_ptr() % 16 != 0
    if init is not None:
        a.copy_(init)
        u.copy_(init)
    return a, u


# (T, K, N): K = 256 runs the A-panel-resident kernel, K = 512 / 768 the generic one; ragged T and N included
SHAPES = [(4096, 256, 768), (777, 512, 256), (130, 256, 72), (1000, 768, 256), (300, 512, 136)]


@pytest.mark.parametrize("T,K,N", SHAPES)
def test_linear_tma_epilogue_matches_register_epilogue(T, K, N):
    x = _rand(T, K, seed=1, dtype=torch.bfloat16)
    w = _rand(N, K, seed=2, dtype=torch.bfloat16, scale=K ** -0.5)
    b = _rand(N, seed=3)
    # bf16 out with bias
    ya, yu = _pair(T, N, torch.bfloat16)
    ops.linear(x, w, b, out=ya)
    ops.linear(x, w, b, out=yu)
    assert torch.equal(ya, yu)
    # fp32 out with bias
    ya, yu = _pair(T, N, torch.float32)
    ops.linear(x, w, b, out=ya)
    ops.linear(x, w, b, out=yu)
    assert torch.equal(ya, yu)
    # fp32 accumulate (dgrad into the residual-stream gradient): dy [T, N] @ w [N, K]
    dy = _rand(T, N, seed=4, dtype=torch.bfloat16)
    acc0 = _rand(T, K, seed=5)
    aa, au = _pair(T, K, torch.float32, init=acc0)
    ops.linear(dy, w, out=aa, w_is_kn=True, accumulate=True)
    ops.linear(dy, w, out=au, w_is_kn=True, accumulate=True)
    assert torch.equal(aa, au)
    assert not torch.equal(aa, acc0)


def _gemm_mn_mn(dy, a, off):
    """dy^T a (both operands MN-major, as stored) into an fp32 C `off` elements past a 16-byte-aligned base"""
    K, M = dy.shape
    N = a.shape[1]
    c = torch.zeros(M * N + 16, device=DEV)[off:off + M * N]
    call("lgb200_gemm_bf16", ptr(dy), ptr(a), ptr(c), 1, M, N, K, 1, 1, M, N, N, K * M, K * N, M * N, F32, 1.0,
         stream_ptr())
    return c.view(M, N)


@pytest.mark.parametrize("T,M,N", [(4096, 256, 256), (10000, 256, 256), (777, 768, 256)])
def test_splitk_tma_epilogue_matches_register_epilogue(T, M, N):
    """The split-K weight gradient writes its partial tiles into the workspace through the staged epilogue.  Each
    partial is the plain GEMM over that split's rows (same 64-row k blocks in the same order), here written through the
    register epilogue; summed in split order they give the same weight gradient, bit for bit."""
    dy = _rand(T, M, seed=1, dtype=torch.bfloat16)
    a = _rand(T, N, seed=2, dtype=torch.bfloat16)
    splits = _lib.load().lgb200_gemm_splitk_ws_floats(M, N, T) // (M * N)
    nk = (T + 63) // 64
    kps = (nk + splits - 1) // splits
    assert (nk + kps - 1) // kps == splits
    ref = torch.zeros(M, N, device=DEV)
    for s in range(splits):
        rows = slice(64 * kps * s, min(T, 64 * kps * (s + 1)))
        ref += _gemm_mn_mn(dy[rows], a[rows], off=1)
    assert torch.equal(ops.wgrad_bf16(dy, a), ref)
    # the plain GEMM's two epilogues agree as well
    assert torch.equal(_gemm_mn_mn(dy, a, off=0), _gemm_mn_mn(dy, a, off=1))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_batched_gemm_tma_epilogue_matches_register_epilogue(dtype):
    batch, M, N, K = 3, 200, 136, 72
    a = _rand(batch, M, K, seed=1, dtype=torch.bfloat16)
    b = _rand(batch, N, K, seed=2, dtype=torch.bfloat16)
    outs = []
    for off in (0, 1):
        c = torch.zeros(batch * M * N + 16, device=DEV, dtype=dtype)[off:off + batch * M * N]
        call("lgb200_gemm_bf16", ptr(a), ptr(b), ptr(c), batch, M, N, K, 0, 0, K, K, N, M * K, N * K, M * N,
             F32 if dtype == torch.float32 else BF16, 0.5, stream_ptr())
        outs.append(c.view(batch, M, N))
    assert torch.equal(outs[0], outs[1])
    assert torch.equal(outs[0], ops.gemm_bf16(a, b, out_dtype=dtype, alpha=0.5))


@pytest.mark.parametrize("dtype,accumulate", [(torch.bfloat16, False), (torch.float32, False), (torch.float32, True)])
@pytest.mark.parametrize("T,K,N", [(777, 256, 72), (130, 512, 136), (300, 768, 256)])
def test_tma_epilogue_leaves_neighbours_untouched(dtype, accumulate, T, K, N):
    """C is a column block of a wider matrix with rows after it: the sentinel columns either side of it and the rows
    past M keep their values, and the block itself matches a contiguous C."""
    pad = 16 // torch.empty((), dtype=dtype).element_size() * 2  # two 16-byte units each side
    sentinel = -3.0
    big = torch.full((T + 5, pad + N + pad), sentinel, device=DEV, dtype=dtype)
    c = big[:T, pad:pad + N]
    assert c.data_ptr() % 16 == 0 and (c.stride(0) * c.element_size()) % 16 == 0
    if accumulate:  # dx [T, N] += dy [T, K] @ wk [K, N]
        dy = _rand(T, K, seed=1, dtype=torch.bfloat16)
        wk = _rand(K, N, seed=6, dtype=torch.bfloat16, scale=K ** -0.5)
        ref = torch.full((T, N), sentinel, device=DEV, dtype=dtype)
        ops.linear(dy, wk, out=c, w_is_kn=True, accumulate=True)
        ops.linear(dy, wk, out=ref, w_is_kn=True, accumulate=True)
    else:
        x = _rand(T, K, seed=1, dtype=torch.bfloat16)
        w = _rand(N, K, seed=2, dtype=torch.bfloat16, scale=K ** -0.5)
        b = _rand(N, seed=3)
        ops.linear(x, w, b, out=c)
        ref = ops.linear(x, w, b, out_dtype=dtype)
    assert torch.equal(c, ref)
    assert bool((big[:, :pad] == sentinel).all()) and bool((big[:, pad + N:] == sentinel).all())
    assert bool((big[T:] == sentinel).all())


@pytest.mark.parametrize("T,K,N", [(4096, 256, 256), (1000, 512, 512)])
def test_tma_epilogue_repeatable(T, K, N):
    x = _rand(T, K, seed=1, dtype=torch.bfloat16)
    w = _rand(N, K, seed=2, dtype=torch.bfloat16, scale=K ** -0.5)
    b = _rand(N, seed=3)
    assert torch.equal(ops.linear(x, w, b), ops.linear(x, w, b))
    dy = _rand(T, N, seed=4, dtype=torch.bfloat16)
    acc0 = _rand(T, K, seed=5)
    a1, a2 = acc0.clone(), acc0.clone()
    ops.linear(dy, w, out=a1, w_is_kn=True, accumulate=True)
    ops.linear(dy, w, out=a2, w_is_kn=True, accumulate=True)
    assert torch.equal(a1, a2)
