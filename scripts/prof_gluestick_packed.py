"""GlueStick inference over a batch of pairs of different sizes: one call per pair against one packed call.

Workload: 32 pairs, 1024-2048 keypoints and 256-512 lines per view (padded to the batch maximum), shared junctions,
18 GNN layers, 256 channels, bf16, eval mode.  Arms, timed in alternating rounds (medians reported):
  a  one uniform call per pair on its truncated inputs (the only way before num_keypoints / num_lines);
  b  one packed call per pair (counts given, B = 1);
  c  one packed call of all 32 pairs.
--profile: instead, one torch.profiler run of arm c, with the device time of the three packed kernels.
The card's name and power limit are read in the same process.  Usage (on an H100):
  python scripts/prof_gluestick_packed.py [--rounds 5] [--profile] [--out result.json]
The result is printed as one JSON line, and also written to --out when given."""
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

from gluefactory_b200 import synthetic  # noqa: E402
from gluefactory_b200.matchers.gluestick import GlueStick  # noqa: E402

B, DEV = 32, "cuda"


def make_pairs(seed=0):
    g = torch.Generator().manual_seed(seed)
    pairs = []
    for b in range(B):
        n0, n1 = (int(x) for x in torch.randint(1024, 2049, (2,), generator=g))
        L0, L1 = (int(x) for x in torch.randint(256, 513, (2,), generator=g))
        d = synthetic.make_gluestick_batch(1, max(n0, n1), max(L0, L1), seed + b)
        p = {"view0": d["view0"], "view1": d["view1"]}
        for v, (n, L) in enumerate(((n0, L0), (n1, L1))):
            for k in ("keypoints", "descriptors", "keypoint_scores"):
                p[f"{k}{v}"] = d[f"{k}{v}"][:, :n]
            # 2 L endpoints on 1.5 L junctions among the first 2 L keypoints: many junctions end several lines
            junc = torch.randint(0, (3 * L) // 2, (1, L, 2), generator=g)
            p[f"lines_junc_idx{v}"] = junc
            p[f"lines{v}"] = p[f"keypoints{v}"][0][junc.reshape(-1)].reshape(1, L, 2, 2)
            p[f"line_scores{v}"] = d[f"line_scores{v}"][:, :L]
        pairs.append(synthetic.to_device(p, DEV))
    return pairs


def pad_batch(pairs):
    data = {"view0": {"image_size": torch.cat([p["view0"]["image_size"] for p in pairs])},
            "view1": {"image_size": torch.cat([p["view1"]["image_size"] for p in pairs])}}
    for v in (0, 1):
        for k in ("keypoints", "descriptors", "keypoint_scores", "lines", "line_scores", "lines_junc_idx"):
            n = max(p[f"{k}{v}"].shape[1] for p in pairs)
            fill = 0 if k == "lines_junc_idx" else float("nan")
            data[f"{k}{v}"] = torch.cat([torch.cat([p[f"{k}{v}"], torch.full(
                (1, n - p[f"{k}{v}"].shape[1], *p[f"{k}{v}"].shape[2:]), fill, dtype=p[f"{k}{v}"].dtype,
                device=DEV)], 1) for p in pairs])
        data[f"num_keypoints{v}"] = torch.tensor([p[f"keypoints{v}"].shape[1] for p in pairs])
        data[f"num_lines{v}"] = torch.tensor([p[f"lines{v}"].shape[1] for p in pairs])
    return data


def counted(p):
    return {**p, **{f"num_{k}{v}": torch.tensor([p[f"{k}{v}"].shape[1]]) for v in (0, 1)
                    for k in ("keypoints", "lines")}}


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--profile", action="store_true")
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    args = ap.parse_args()
    model = GlueStick({"precision": "bf16"})
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=1))
    model = model.to(DEV).eval()
    pairs = make_pairs()
    batch = pad_batch(pairs)
    single = [counted(p) for p in pairs]
    arms = {"a_uniform_per_pair": lambda: [model(p) for p in pairs],
            "b_packed_per_pair": lambda: [model(p) for p in single],
            "c_packed_batch": lambda: model(batch)}
    res = {"gpu": gpu_info(), "pairs": B, "layers": 18, "channels": 256, "precision": "bf16"}
    with torch.no_grad():
        for f in arms.values():  # warm every shape
            f()
        torch.cuda.synchronize()
        if args.profile:
            from torch.profiler import ProfilerActivity, profile

            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                arms["c_packed_batch"]()
                torch.cuda.synchronize()
            names = {"lds_scores_kernel<true>": "lds_scores_kernel<true>", "lds_colarg_varlen": "lds_colarg_varlen",
                     "line_scores_varlen": "line_scores_varlen", "junction_mean": "junction_mean",
                     "assign_lse_kernel<true>": "assign_lse_kernel<true>"}
            kt = {k: {"calls": 0, "us": 0.0} for k in names}
            for e in prof.key_averages():
                for k in names:
                    if k in e.key:
                        kt[k]["calls"] += e.count
                        kt[k]["us"] += e.device_time_total
            res["kernels_us_total_per_call"] = kt
        else:
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
    res["gpu_after"] = gpu_info()
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
