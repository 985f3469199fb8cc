"""Time the three fused assignment-head kernels (csrc/assign_tc.cu) at the training shape, and optionally save their
outputs on seeded inputs so that two builds can be compared bit for bit.

    python scripts/bench_assign.py [--tree DIR] [--iters 20] [--dump OUT_DIR]

--tree imports the package from another checkout (for before/after runs in one session).  The timed shape is the
flagship step's: B=32 pairs, M=N=2048 keypoints, D=256, with a ground truth of at most one positive per row and
column (a random partial permutation, as homography or depth supervision gives).  STATS is timed with and without the
mask (gt=None skips the positives sum)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ap = argparse.ArgumentParser()
ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--B", type=int, default=32)
ap.add_argument("--N", type=int, default=2048)
ap.add_argument("--D", type=int, default=256)
ap.add_argument("--dump", default=None, help="save every output of the seeded cases here as .npy")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.tree))
from gluefactory_b200 import ops  # noqa: E402

DEV = "cuda"


def inputs(B, M, N, D, seed, dense=False):
    g = torch.Generator().manual_seed(seed)
    md0 = (torch.randn(B, M, D, generator=g) * 2).to(torch.bfloat16).to(DEV)
    md1 = (torch.randn(B, N, D, generator=g) * 2).to(torch.bfloat16).to(DEV)
    z0, z1 = torch.randn(B, M, generator=g), torch.randn(B, N, generator=g)
    ls0 = torch.nn.functional.logsigmoid(z0).to(DEV)
    ls1 = torch.nn.functional.logsigmoid(z1).to(DEV)
    if dense:
        gt = torch.rand(B, M, N, generator=g) < 0.25
    else:
        gt = torch.zeros(B, M, N, dtype=torch.bool)
        K = min(M, N) // 2
        for b in range(B):
            gt[b, torch.randperm(M, generator=g)[:K], torch.randperm(N, generator=g)[:K]] = True
    gt_u8 = gt.to(DEV).view(torch.uint8)
    gt_t = gt_u8.transpose(1, 2).contiguous()
    gc = (torch.rand(B, generator=g) + 0.1).to(DEV) * D ** -0.5
    return dict(md0=md0, md1=md1, alpha=D ** -0.5, ls0=ls0, ls1=ls1, gt=gt_u8, gt_t=gt_t, gc=gc,
                rowcnt=gt_u8.sum(2, dtype=torch.float32), colcnt=gt_u8.sum(1, dtype=torch.float32))


def run_all(x):
    B, M, D = x["md0"].shape
    N = x["md1"].shape[1]
    st = ops.assign_fused_stats(x["md0"], x["md1"], x["alpha"], x["ls0"], x["ls1"], gt_u8=x["gt"])
    dmd = torch.empty(B * M + B * N, D, device=DEV, dtype=torch.bfloat16)
    ops.assign_fused_bwd(x["md0"], x["md1"], x["alpha"], st["lse_row"], st["lse_col"], x["gt"], x["gt_t"], x["gc"],
                         x["rowcnt"], x["colcnt"], dmd[:B * M], dmd[B * M:])
    out = {k: v for k, v in st.items() if v is not None}
    out["dmd0"], out["dmd1"] = dmd[:B * M], dmd[B * M:]
    return out


def timed(fn, iters):
    for _ in range(3):
        fn()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters  # us per call


def bench():
    B, M, N, D = args.B, args.N, args.N, args.D
    x = inputs(B, M, N, D, seed=0)
    md0, md1, alpha = x["md0"], x["md1"], x["alpha"]
    f = lambda *s: torch.empty(*s, device=DEV, dtype=torch.float32)  # noqa: E731
    lse_r, lse_c = f(B, M), f(B, N)
    rmax, cmax, prs = f(B, M), f(B, N), f(B, M)
    rarg = torch.empty(B, M, device=DEV, dtype=torch.int32)
    carg = torch.empty(B, N, device=DEV, dtype=torch.int32)
    dmd = torch.empty(B * M + B * N, D, device=DEV, dtype=torch.bfloat16)
    s = ops.stream_ptr()
    P = ops.ptr

    def lse():
        ops.call("lgb200_assign_fused_lse", P(md0), P(md1), alpha, P(lse_r), P(lse_c), B, M, N, D, s)

    def stats(mask):
        ops.call("lgb200_assign_fused_stats", P(md0), P(md1), alpha, P(lse_r), P(lse_c), P(x["ls0"]), P(x["ls1"]),
                 P(x["gt"]) if mask else None, P(rmax), P(rarg), P(cmax), P(carg), P(prs) if mask else None,
                 B, M, N, D, s)

    def bwd():
        ops.call("lgb200_assign_fused_bwd", P(md0), P(md1), alpha, P(lse_r), P(lse_c), P(x["gt"]), P(x["gt_t"]),
                 P(x["gc"]), P(x["rowcnt"]), P(x["colcnt"]), P(dmd[:B * M]), P(dmd[B * M:]), B, M, N, D, s)

    lse()
    torch.cuda.synchronize()
    res = {"shape": [B, M, N, D], "lse_us": timed(lse, args.iters),
           "stats_mask_us": timed(lambda: stats(True), args.iters),
           "stats_nomask_us": timed(lambda: stats(False), args.iters),
           "bwd_us": timed(bwd, args.iters)}
    print(json.dumps({k: (round(v, 1) if isinstance(v, float) else v) for k, v in res.items()}))


def dump(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    cases = [(32, 2048, 2048, 256, False), (2, 2048, 2048, 256, True), (2, 256, 256, 256, False),
             (3, 150, 203, 256, False), (1, 72, 300, 128, False), (1, 130, 64, 64, False), (2, 200, 321, 192, True)]
    for i, (B, M, N, D, dense) in enumerate(cases):
        out = run_all(inputs(B, M, N, D, seed=100 + i, dense=dense))
        for k, v in out.items():
            np.save(os.path.join(out_dir, f"c{i}_{k}.npy"), v.detach().view(torch.int16).cpu().numpy()
                    if v.dtype == torch.bfloat16 else v.detach().cpu().numpy())
    torch.cuda.synchronize()


if __name__ == "__main__":
    if args.dump:
        dump(args.dump)
    bench()
