"""Event timing of the layer's dense GEMMs (lgb200_linear, and the split-K weight gradient) at the bench token count
(T = 131072 = 32 pairs x 2 images x 2048), called exactly as engine.LayerFn calls them: row-strided A and C views,
fp32 bias, fp32 accumulation into the residual-stream gradient.

    python scripts/prof_linear.py [--tree DIR] [--iters 20] [--dump OUT_DIR]

For each call it prints the time, the least HBM traffic the call needs (each operand read once, each output written
once, an accumulated fp32 C read and written once), the achieved TB/s, and the larger of the two hardware bounds
(bytes / 3.35 TB/s, FLOPs / 989 TFLOP/s: H100 SXM data-sheet figures).  --tree imports the package from another
checkout (before/after runs in one session); --dump saves every call's output on seeded inputs as .npy for a bitwise
comparison between builds."""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

ap = argparse.ArgumentParser()
ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--T", type=int, default=131072)
ap.add_argument("--D", type=int, default=256)
ap.add_argument("--dump", default=None, help="save every call's output here as .npy")
args = ap.parse_args()
sys.path.insert(0, os.path.abspath(args.tree))
from gluefactory_b200 import ops  # noqa: E402

DEV = "cuda"
HBM_TBS, BF16_TFLOPS = 3.35, 989.0
T, D = args.T, args.D


def rnd(g, *s, scale=1.0, dtype=torch.bfloat16):
    return (torch.randn(*s, device=DEV, generator=g) * scale).to(dtype)


def calls():
    """(name, kernel group, fn -> output, bytes, flops) for each distinct GEMM of a layer step (engine.LayerFn)."""
    g = torch.Generator(device=DEV).manual_seed(0)
    cat = rnd(g, T, 2 * D)                      # [x16 | msg] halves: row-strided A and C
    att = rnd(g, T, D)
    ffn_h = rnd(g, T, 2 * D)                    # ffn.0 input / ffn.3 input (g = LN-GELU output)
    dy_d, dy_2d, dy_3d = rnd(g, T, D), rnd(g, T, 2 * D), rnd(g, T, 3 * D)
    Wqkv, Wd, W0 = rnd(g, 3 * D, D, scale=D ** -0.5), rnd(g, D, D, scale=D ** -0.5), rnd(g, 2 * D, 2 * D, scale=0.04)
    W3 = rnd(g, D, 2 * D, scale=0.04)
    b3d, bd, b2d = (torch.randn(n, device=DEV, generator=g) for n in (3 * D, D, 2 * D))
    acc0 = torch.randn(T, D, device=DEV, generator=g)
    acc = acc0.clone()
    dW0 = torch.empty(2 * D, 2 * D, device=DEV)
    outs = {}

    def new(name, n, dt=torch.bfloat16):
        if name not in outs:
            outs[name] = torch.empty(T, n, device=DEV, dtype=dt)
        return outs[name]

    def accumulate(dy, w):
        return lambda: ops.linear(dy, w, out=acc, w_is_kn=True, accumulate=True)

    x16, msg = cat[:, :D], cat[:, D:]
    bf, f4 = 2, 4
    res = [
        ("fwd qkv      K=256 N=768 (A row-strided, bias)", "apanel<false,bf16>",
         lambda: ops.linear(x16, Wqkv, b3d, out=new("qkv", 3 * D)), T * D * bf + T * 3 * D * bf, 2 * T * D * 3 * D),
        ("fwd out_proj K=256 N=256 (C row-strided, bias)", "apanel<false,bf16>",
         lambda: ops.linear(att, Wd, bd, out=msg), T * D * bf + T * D * bf, 2 * T * D * D),
        ("fwd to_qk    K=256 N=256 (A row-strided, bias)", "apanel<false,bf16>",
         lambda: ops.linear(x16, Wd, bd, out=new("qk", D)), T * D * bf + T * D * bf, 2 * T * D * D),
        ("fwd ffn.0    K=512 N=512 (bias)", "bf16<false,false,bf16>",
         lambda: ops.linear(cat, W0, b2d, out=new("h", 2 * D)), T * 2 * D * bf + T * 2 * D * bf, 2 * T * 4 * D * D),
        ("fwd ffn.3    K=512 N=256 (bias)", "bf16<false,false,bf16>",
         lambda: ops.linear(ffn_h, W3, bd, out=new("y", D)), T * 2 * D * bf + T * D * bf, 2 * T * 2 * D * D),
        ("dgrad ffn.3  K=256 N=512", "apanel<true,bf16>",
         lambda: ops.linear(dy_d, W3, w_is_kn=True, out=new("dg", 2 * D)), T * D * bf + T * 2 * D * bf,
         2 * T * 2 * D * D),
        ("dgrad proj   K=256 N=256", "apanel<true,bf16>",
         lambda: ops.linear(dy_d, Wd, w_is_kn=True, out=new("dm", D)), T * D * bf + T * D * bf, 2 * T * D * D),
        ("dmsg         K=512 N=256 (B = W0[:, D:])", "bf16<false,true,bf16>",
         lambda: ops.linear(dy_2d, W0[:, D:], w_is_kn=True, out=new("dmsg", D)), T * 2 * D * bf + T * D * bf,
         2 * T * 2 * D * D),
        ("dx += K=256 N=256 (fp32 accumulate)", "apanel<true,float>",
         accumulate(dy_d, Wd), T * D * bf + 2 * T * D * f4, 2 * T * D * D),
        ("dx += K=512 N=256 (fp32 accumulate, B = W0[:, :D])", "bf16<false,true,float>",
         accumulate(dy_2d, W0[:, :D]), T * 2 * D * bf + 2 * T * D * f4, 2 * T * 2 * D * D),
        ("dx += K=768 N=256 (fp32 accumulate, B = Wqkv)", "bf16<false,true,float>",
         accumulate(dy_3d, Wqkv), T * 3 * D * bf + 2 * T * D * f4, 2 * T * 3 * D * D),
        ("wgrad ffn.0  [512 x 512] over T (split-K)", "bf16<true,true,float> + reduce",
         lambda: ops.wgrad_bf16(dy_2d, cat, out=dW0),
         2 * T * 2 * D * bf + 4 * D * D * f4, 2 * T * 4 * D * D),
    ]
    return res, acc, acc0


def timed(fn, iters):
    """us per call, back-to-back calls (the accumulating ones keep adding into the same C)"""
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) * 1e3 / iters


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as ex:
        q = f"nvidia-smi unavailable ({ex})"
    return f"{torch.cuda.get_device_name()} | name, power limit, SM clock, max SM clock: {q}"


def main():
    res, acc, acc0 = calls()
    print(f"tree={os.path.abspath(args.tree)} T={T} D={D}")
    print(card())
    if args.dump:
        os.makedirs(args.dump, exist_ok=True)
        for i, (name, _, fn, _, _) in enumerate(res):
            if "accumulate" in name:
                acc.copy_(acc0)
            out = fn().detach()
            np.save(os.path.join(args.dump, f"call{i:02d}.npy"),
                    out.view(torch.int16).cpu().numpy() if out.dtype == torch.bfloat16 else out.cpu().numpy())
        torch.cuda.synchronize()
    print("| call | kernel | us | MB | TB/s | bound us | bound | share of bound |")
    print("|---|---|---:|---:|---:|---:|---|---:|")
    for name, kern, fn, nbytes, flops in res:
        us = timed(fn, args.iters)
        t_mem, t_math = nbytes / (HBM_TBS * 1e6), flops / (BF16_TFLOPS * 1e6)
        bound, which = (t_mem, "HBM") if t_mem >= t_math else (t_math, "BF16")
        print(f"| {name} | `{kern}` | {us:.1f} | {nbytes / 1e6:.0f} | {nbytes / us / 1e6:.2f} | {bound:.1f} | {which} "
              f"| {bound / us:.2f} |")
    print(card())


if __name__ == "__main__":
    main()
