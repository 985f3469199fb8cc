"""SuperGlue inference over a batch of pairs of different sizes: one call per pair against one packed call.

Workload: 32 pairs, 1024-2048 keypoints per view (padded to 2048), the default configuration (18 GNN layers, 50
Sinkhorn iterations, 256 channels), bf16, eval mode, synthetic weights.  Arms, timed in alternating rounds (medians
and spread reported):
  a  one uniform call per pair on its truncated inputs (the only way before num_keypoints0/1);
  b  one packed call per pair (counts given, B = 1);
  c  one packed call of all 32 pairs.
Then, in a torch.profiler run of its own after the timed rounds: the device time of the packed Sinkhorn launch over
arm c's costs against a per-pair loop of the uniform Sinkhorn kernel over the same costs.
The card's name and power limit are read in the same process.  Usage (on an H100):
  python scripts/prof_superglue_packed.py [--rounds 5] [--out result.json] [--md profile.md]
The result is printed as one JSON line, also written to --out, and summarised as markdown in --md when given."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from gluefactory_b200 import ops, synthetic  # noqa: E402
from gluefactory_b200.matchers.superglue import SuperGlue  # noqa: E402

B, P, DEV = 32, 2048, "cuda"
KEYS = ("keypoints", "descriptors", "keypoint_scores")


def make_pairs(seed=0):
    g = torch.Generator().manual_seed(seed)
    pairs = []
    for b in range(B):
        n0, n1 = (int(x) for x in torch.randint(1024, P + 1, (2,), generator=g))
        d = synthetic.make_superglue_batch(1, n0, n1, seed + b)
        pairs.append(synthetic.to_device({k: d[k] for k in ("view0", "view1") + tuple(f"{k}{v}" for k in KEYS
                                                                                     for v in (0, 1))}, DEV))
    return pairs


def pad_batch(pairs):
    data = {f"view{v}": {"image_size": torch.cat([p[f"view{v}"]["image_size"] for p in pairs])} for v in (0, 1)}
    for v in (0, 1):
        for k in KEYS:
            data[f"{k}{v}"] = torch.cat([torch.cat([p[f"{k}{v}"], torch.full(
                (1, P - p[f"{k}{v}"].shape[1], *p[f"{k}{v}"].shape[2:]), float("nan"), dtype=p[f"{k}{v}"].dtype,
                device=DEV)], 1) for p in pairs])
        data[f"num_keypoints{v}"] = torch.tensor([p[f"keypoints{v}"].shape[1] for p in pairs])
    return data


def counted(p):
    return {**p, **{f"num_keypoints{v}": torch.tensor([p[f"keypoints{v}"].shape[1]]) for v in (0, 1)}}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def sinkhorn_profile(model, batch, pred):
    """Device time (us) of the packed Sinkhorn over the packed call's costs and of a per-pair loop of the uniform
    kernel over the same costs (torch.profiler, kernels picked by name)."""
    n0, n1 = batch["num_keypoints0"], batch["num_keypoints1"]
    cost = pred["sinkhorn_cost"].contiguous()
    per_pair = [cost[b:b + 1, :int(n0[b]), :int(n1[b])].contiguous() for b in range(B)]
    pairs = torch.stack([n0, n1, torch.arange(B)]).to(DEV, torch.int32)
    out = torch.full((B, P + 1, P + 1), float("-inf"), device=DEV)
    iters = model.conf.num_sinkhorn_iterations
    packed = lambda: ops.log_optimal_transport_varlen(cost, model.bin_score, iters, pairs, out)  # noqa: E731
    loop = lambda: [ops.log_optimal_transport(c, model.bin_score, iters) for c in per_pair]  # noqa: E731
    packed(), loop()
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile

    names = {"packed": ("sk_varlen_items_kernel", "sk_fwd_varlen_kernel"), "uniform_loop": ("sk_fwd_persistent_kernel",)}
    res = {}
    for arm, f in (("packed", packed), ("uniform_loop", loop)):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            f()
            torch.cuda.synchronize()
        us, calls = 0.0, 0
        for e in prof.key_averages():
            if any(k in e.key for k in names[arm]):
                us += e.device_time_total
                calls += e.count
        res[arm] = {"us": us, "kernel_launches": calls}
    res["speedup"] = res["uniform_loop"]["us"] / max(res["packed"]["us"], 1e-9)
    return res


def write_md(path, res):
    s, k = res["seconds_median"], res["sinkhorn_device"]
    lines = [
        "# SuperGlue over a batch of pairs of different sizes (`scripts/prof_superglue_packed.py`)", "",
        f"Card: {res['gpu']} (name, power limit; read in the measuring process).  Workload: {B} pairs of 1024-{P} "
        f"keypoints per view, padded to {P}; 18 GNN layers, 50 Sinkhorn iterations, bf16, eval, synthetic weights.  "
        f"{res['rounds']} alternating rounds; medians, with the min-max spread.", "",
        "| arm | s per 32 pairs (median) | spread (min-max) | pairs/s |", "|---|---|---|---|"]
    for a in s:
        lines.append(f"| {a} | {s[a]:.4f} | {min(res['seconds_all'][a]):.4f}-{max(res['seconds_all'][a]):.4f} | "
                     f"{res['pairs_per_s'][a]:.1f} |")
    lines += ["", f"Arm c against arm a: {s['a_uniform_per_pair'] / s['c_packed_batch']:.1f}x; against arm b: "
                  f"{s['b_packed_per_pair'] / s['c_packed_batch']:.1f}x.", "",
              "Sinkhorn head alone (torch.profiler device time over the packed call's costs, 32-row strips):", "",
              "| | device time (us) | kernel launches |", "|---|---|---|",
              f"| packed (`sk_varlen_items_kernel` + `sk_fwd_varlen_kernel`) | {k['packed']['us']:.0f} | "
              f"{k['packed']['kernel_launches']} |",
              f"| uniform kernel, one launch per pair (`sk_fwd_persistent_kernel`) | {k['uniform_loop']['us']:.0f} | "
              f"{k['uniform_loop']['kernel_launches']} |", "",
              f"Packed against the per-pair loop: {k['speedup']:.2f}x.", ""]
    with open(path, "w") as f:
        f.write("\n".join(lines))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    ap.add_argument("--md", default=None, help="also write a markdown summary to this file")
    args = ap.parse_args()
    model = SuperGlue({"precision": "bf16", "weights": None})
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=1))
    model = model.to(DEV).eval()
    pairs = make_pairs()
    batch = pad_batch(pairs)
    single = [counted(p) for p in pairs]
    arms = {"a_uniform_per_pair": lambda: [model(p) for p in pairs],
            "b_packed_per_pair": lambda: [model(p) for p in single],
            "c_packed_batch": lambda: model(batch)}
    res = {"gpu": gpu_info(), "pairs": B, "layers": 18, "iterations": 50, "channels": 256, "precision": "bf16",
           "rounds": args.rounds}
    with torch.no_grad():
        for f in arms.values():  # warm every shape
            f()
        torch.cuda.synchronize()
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, f in arms.items():
                torch.cuda.synchronize()
                t = time.perf_counter()
                f()
                torch.cuda.synchronize()
                times[k].append(time.perf_counter() - t)
        res["seconds_median"] = {k: statistics.median(v) for k, v in times.items()}
        res["pairs_per_s"] = {k: B / v for k, v in res["seconds_median"].items()}
        res["seconds_all"] = times
        res["sinkhorn_device"] = sinkhorn_profile(model, batch, model(batch))
    res["gpu_after"] = gpu_info()
    for path in (args.out, args.md):
        if path:
            os.makedirs(os.path.dirname(os.path.abspath(path)), exist_ok=True)
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    if args.md:
        write_md(args.md, res)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
