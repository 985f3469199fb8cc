"""GPU: the fused assignment kernels (csrc/assign_tc.cu) with the mask tile and the per-column vectors staged in shared
memory by the producer warpgroup: dense masks (many positives per row), ragged widths that take the byte-wise copy,
last tiles of 1 and 63 columns with positives in them, three K blocks, and run-to-run bit equality."""
import pytest
import torch

from gluefactory_b200 import ops
from tests.util import rel_err

pytestmark = pytest.mark.gpu
DEV = "cuda"


def _case(B, M, N, D, seed, p_pos=None, last_tile_pos=False):
    g = torch.Generator().manual_seed(seed)
    md0 = (torch.randn(B, M, D, generator=g) * 2).to(torch.bfloat16).to(DEV)
    md1 = (torch.randn(B, N, D, generator=g) * 2).to(torch.bfloat16).to(DEV)
    z0, z1 = torch.randn(B, M, generator=g), torch.randn(B, N, generator=g)
    ls0, ls1 = (torch.nn.functional.logsigmoid(z).to(DEV) for z in (z0, z1))
    if p_pos is not None:
        gt = torch.rand(B, M, N, generator=g) < p_pos
    else:
        gt = torch.zeros(B, M, N, dtype=torch.bool)
        K = min(M, N) // 3
        for b in range(B):
            gt[b, torch.randperm(M, generator=g)[:K], torch.randperm(N, generator=g)[:K]] = True
    if last_tile_pos:  # positives in the last column tile of each direction (and in the last rows)
        gt[:, torch.arange(0, M, 7), N - 1] = True
        gt[:, M - 1, torch.arange(0, N, 5)] = True
        gt[:, 3, (N // 64) * 64:] = True
    gt_u8 = gt.to(DEV).view(torch.uint8)
    gc = (torch.rand(B, generator=g) + 0.1).to(DEV) * D ** -0.5
    return md0, md1, D ** -0.5, ls0, ls1, gt_u8, gc


def _run(md0, md1, alpha, ls0, ls1, gt_u8, gc):
    B, M, D = md0.shape
    N = md1.shape[1]
    f = ops.assign_fused_stats(md0, md1, alpha, ls0, ls1, gt_u8=gt_u8)
    rowcnt, colcnt = gt_u8.sum(2, dtype=torch.float32), gt_u8.sum(1, dtype=torch.float32)
    dmd = torch.empty(B * M + B * N, D, device=DEV, dtype=torch.bfloat16)
    ops.assign_fused_bwd(md0, md1, alpha, f["lse_row"], f["lse_col"], gt_u8, gt_u8.transpose(1, 2).contiguous(), gc,
                         rowcnt, colcnt, dmd[:B * M], dmd[B * M:])
    f["dmd0"], f["dmd1"] = dmd[:B * M], dmd[B * M:]
    return f, rowcnt, colcnt


def _check_fp64(md0, md1, alpha, ls0, ls1, gt_u8, gc, f, rowcnt, colcnt):
    B, M, D = md0.shape
    N = md1.shape[1]
    s64 = (md0.double() @ md1.double().transpose(1, 2)) * alpha
    lr, lc = torch.logsumexp(s64, 2), torch.logsumexp(s64, 1)
    assert (f["lse_row"].double() - lr).abs().max().item() < 1e-4
    assert (f["lse_col"].double() - lc).abs().max().item() < 1e-4
    sc = (s64 - lr[:, :, None]) + (s64 - lc[:, None, :]) + (ls0.double()[:, :, None] + ls1.double()[:, None, :])
    assert (f["rowmax"].double() - sc.max(2).values).abs().max().item() < 1e-3
    assert (f["colmax"].double() - sc.max(1).values).abs().max().item() < 1e-3
    gt = gt_u8.bool()
    pos = torch.where(gt, 2 * s64 - lr[:, :, None] - lc[:, None, :], torch.zeros_like(s64)).sum(2)
    assert rel_err(f["pos_row_sum"], pos) < 1e-4
    p_r = torch.exp(s64 - lr[:, :, None])
    p_c = torch.exp(s64 - lc[:, None, :])
    dsim = gc.double()[:, None, None] * (2 * gt.double() - p_r * rowcnt.double()[:, :, None]
                                         - p_c * colcnt.double()[:, None, :])
    assert rel_err(f["dmd0"], (dsim @ md1.double()).reshape(B * M, D)) < 8e-3
    assert rel_err(f["dmd1"], (dsim.transpose(1, 2) @ md0.double()).reshape(B * N, D)) < 8e-3


def test_dense_mask_against_fp64():
    """About a quarter of all pairs positive: every row and column holds many positives."""
    x = _case(2, 2048, 2048, 256, seed=11, p_pos=0.25)
    f, rc, cc = _run(*x)
    _check_fp64(*x, f, rc, cc)
    torch.cuda.synchronize()


@pytest.mark.parametrize("M,N", [(200, 129), (129, 200), (191, 321), (300, 127), (96, 208)])
def test_ragged_last_tile_against_fp64(M, N):
    """N % 16 != 0 (byte-wise copy of the mask) and N % 16 == 0 but not % 64; last tiles of 1 and 63 columns, with
    positives in them."""
    x = _case(2, M, N, 128, seed=12, last_tile_pos=True)
    f, rc, cc = _run(*x)
    _check_fp64(*x, f, rc, cc)
    torch.cuda.synchronize()


@pytest.mark.parametrize("p_pos", [None, 0.25])
def test_three_k_blocks_against_fp64(p_pos):
    x = _case(2, 200, 321, 192, seed=13, p_pos=p_pos)
    f, rc, cc = _run(*x)
    _check_fp64(*x, f, rc, cc)
    torch.cuda.synchronize()


def test_two_calls_bit_identical():
    x = _case(3, 1000, 777, 256, seed=14, last_tile_pos=True)
    f1, _, _ = _run(*x)
    f2, _, _ = _run(*x)
    for k in ("lse_row", "lse_col", "rowmax", "rowarg", "colmax", "colarg", "pos_row_sum", "dmd0", "dmd1"):
        assert torch.equal(f1[k], f2[k]), k
