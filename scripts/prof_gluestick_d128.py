"""GlueStick with 128-channel descriptors (attention at head dim 32) against 256 channels (head dim 64) on one GPU.

    python scripts/prof_gluestick_d128.py [--out FILE]     # prints the results; --out also writes them to FILE

1. The bf16 training step (forward + loss + backward + Adam) of the plugin at D = 128 and D = 256, alternating, eager
   (MatcherTrainer.step) and as a CUDA-graph replay, at the C5 shape: PB pairs (default 8) of 2048 points + 512 lines
   per image, 18 GNN layers.
2. The unmodified reference module (staged under oracle/_ref) at D = 128 under bf16 autocast and in fp32, same batch.
3. The attention kernels alone, with CUDA events: forward and backward (prep + dQ + dK/dV) of a self-attention over
   3072 nodes (2048 points + 2 x 512 line endpoints) x 4 heads for 2 PB sequences, at head dim 32 and 64; then the
   three kernels separately from a torch.profiler pass.  Rates against the data sheet (989 TFLOP/s dense bf16) and the
   exponential unit (16 ex2 per clock per SM at the card's maximum SM clock).
The card's name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gluefactory_b200 import ops, synthetic  # noqa: E402
from gluefactory_b200.matchers.gluestick import GlueStick  # noqa: E402
from gluefactory_b200.trainer import MatcherTrainer  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--out", help="also write the results to this file")
args = ap.parse_args()
B, N, L = int(os.environ.get("PB", "8")), 2048, 512
ROUNDS = int(os.environ.get("ROUNDS", "3"))
dev = torch.device("cuda", 0)
lines = []


def out(s=""):
    print(s, flush=True)
    lines.append(s)


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    r = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, clk = (x.strip() for x in r.stdout.splitlines()[0].split(","))
    return name, power, float(clk.split()[0])


def timed(step, reps=5, warm=2):
    for _ in range(warm):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        step()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3


def step_times(D):
    conf = dict(GlueStick.default_conf, input_dim=D, descriptor_dim=D)
    data = synthetic.to_device(synthetic.make_gluestick_batch(B, N, L, 5, D=D), dev)
    m = GlueStick(dict(conf))
    m.load_state_dict(synthetic.make_gluestick_weights(m.state_dict(), seed=3), strict=True)
    tr = MatcherTrainer(m.to(dev).train(), lr=1e-5)
    eager = timed(lambda: tr.step(data))
    tr.capture(data, dev)
    graph = timed(lambda: tr.step_graphed(data), reps=10)
    del tr, m, data
    torch.cuda.empty_cache()
    return eager, graph


def reference_time(D, autocast):
    from oracle.stage_reference import import_reference

    get_model = import_reference()
    if get_model is None:
        return float("nan")
    conf = {k: v for k, v in GlueStick.default_conf.items() if k != "precision"}
    conf.update(input_dim=D, descriptor_dim=D, name="matchers.gluestick")
    ref = get_model("matchers.gluestick")(conf)
    ref.load_state_dict(synthetic.make_gluestick_weights(GlueStick(dict(conf)).state_dict(), seed=3), strict=True)
    ref = ref.to(dev).train()
    data = synthetic.to_device(synthetic.make_gluestick_batch(B, N, L, 5, D=D), dev)
    opt = torch.optim.Adam(ref.parameters(), lr=1e-5)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=autocast, enabled=autocast is not None):
            pred = ref(data)
            losses, _ = ref.loss(pred, data)
            loss = losses["total"].mean()
        loss.backward()
        opt.step()

    ms = timed(step, reps=3, warm=1)
    del ref, data, opt
    torch.cuda.empty_cache()
    return ms


def attention_times(hd, S=3072, H=4, reps=20):
    Bs = 2 * B
    g = torch.Generator(device=dev).manual_seed(hd)
    q, k, v, do = (torch.randn(Bs, S, H, hd, device=dev, generator=g).to(torch.bfloat16) for _ in range(4))
    scale = hd ** -0.5
    o, lse = ops.attn_fwd(q, k, v, 0, scale)
    ops.attn_bwd(q, k, v, o, lse, do, 0, scale)
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    for _ in range(reps):
        ops.attn_fwd(q, k, v, 0, scale)
    ev[1].record()
    for _ in range(reps):
        ops.attn_bwd(q, k, v, o, lse, do, 0, scale)
    ev[2].record()
    torch.cuda.synchronize()
    fwd, bwd = ev[0].elapsed_time(ev[1]) / reps, ev[1].elapsed_time(ev[2]) / reps
    from torch.profiler import ProfilerActivity, profile

    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(5):
            ops.attn_fwd(q, k, v, 0, scale)
            ops.attn_bwd(q, k, v, o, lse, do, 0, scale)
        torch.cuda.synchronize()
    per = {}
    for e in prof.key_averages():
        for tag in ("attn_fwd_tc_kernel", "attn_bwd_dq_kernel", "attn_bwd_dkv_kernel", "attn_bwd_prep_fused_kernel"):
            if tag in e.key:
                per[tag] = e.device_time_total / e.count / 1e3
    return Bs, S, H, fwd, bwd, per


name, power, clk = gpu_info()
out(f"GPU: {name}, power limit {power}, max SM clock {clk:.0f} MHz")
out(f"GlueStick bf16 training step, {B} pairs, {N} points + {L} lines per image, 18 GNN layers")
res = {128: [], 256: []}
for r in range(ROUNDS):
    for D in (128, 256):
        res[D].append(step_times(D))
        out(f"  round {r} D={D}: eager {res[D][-1][0]:.1f} ms, graph replay {res[D][-1][1]:.1f} ms")
for D in (128, 256):
    e = sorted(x[0] for x in res[D])
    gr = sorted(x[1] for x in res[D])
    out(f"D={D}: eager median {e[len(e) // 2]:.1f} ms (range {e[0]:.1f}-{e[-1]:.1f}) = {B / e[len(e) // 2] * 1e3:.1f} pairs/s; "
        f"graph replay median {gr[len(gr) // 2]:.1f} ms (range {gr[0]:.1f}-{gr[-1]:.1f}) = {B / gr[len(gr) // 2] * 1e3:.1f} pairs/s")
for ac, tag in ((torch.bfloat16, "bf16 autocast"), (None, "fp32")):
    try:
        ms = reference_time(128, ac)
        out(f"reference D=128, {tag}: {ms:.1f} ms/step = {B / ms * 1e3:.1f} pairs/s")
    except Exception as ex:  # noqa: BLE001
        out(f"reference D=128, {tag}: not measured ({type(ex).__name__}: {str(ex)[:160]})")

n_sm = torch.cuda.get_device_properties(dev).multi_processor_count
out(f"Attention kernels, self-attention, {2 * B} sequences x 3072 nodes x 4 heads ({n_sm} SMs)")
for hd in (32, 64):
    Bs, S, H, fwd, bwd, per = attention_times(hd)
    flop_f = 4.0 * Bs * H * S * S * hd            # Q K^T and P V
    exps_f = float(Bs * H * S * S)
    flop_b = 14.0 * Bs * H * S * S * hd           # S, dP, dQ (dQ kernel) and S^T, dP^T, dV, dK (dK/dV kernel)
    t_mma = flop_f / 989e12 * 1e3
    t_exp = exps_f / (16 * n_sm * clk * 1e6) * 1e3
    out(f"  hd={hd}: fwd {fwd:.3f} ms ({flop_f / fwd / 1e9:.0f} TFLOP/s, {exps_f / fwd / 1e9:.2f} T ex2/s); "
        f"bound: tensor pipe {t_mma:.3f} ms, exponentials {t_exp:.3f} ms -> fwd at "
        f"{100 * max(t_mma, t_exp) / fwd:.0f}% of the larger ({'exp' if t_exp > t_mma else 'tensor'}); "
        f"tensor-pipe share {100 * t_mma / fwd:.0f}%; time per N^2 {fwd / (Bs * H * S * S) * 1e9:.3f} ps")
    out(f"  hd={hd}: bwd call {bwd:.3f} ms ({flop_b / bwd / 1e9:.0f} TFLOP/s over its 7 products); per kernel (profiler): "
        + ", ".join(f"{k} {v:.3f} ms" for k, v in sorted(per.items())))

if args.out:
    with open(args.out, "w") as f:
        f.write("\n".join(lines) + "\n")
