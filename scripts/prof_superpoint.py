"""SuperPoint forward on Hopper against the unmodified reference (oracle/_ref, staged by the build), in alternating
rounds, and the uncached homography pre-training step (extractor on both views + device ground truth + LightGlue).
Prints JSON lines: the card with its power limit and max SM clock, median times per arm, per-kernel times from CUDA
events with the convolutions' share of the dense BF16 rate and the selection kernels' bytes/s against HBM.

    python scripts/prof_superpoint.py [--shapes 256x480x640,64x1024x1024] [--rounds 3] [--no-ref]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gluefactory_b200 import _lib, synthetic  # noqa: E402
from gluefactory_b200.extractors.superpoint import SuperPoint  # noqa: E402

BF16_PEAK, HBM = 989e12, 3.35e12  # H100 SXM data sheet, dense BF16 and HBM3
SP_ENTRIES = {"lgb200_sp_conv1a", "lgb200_sp_conv", "lgb200_sp_nms", "lgb200_sp_count", "lgb200_sp_select",
              "lgb200_sp_sample"}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def conv_flops(H, W):
    """Multiply-adds x 2 of every conv of one image (floor sizes, as the network computes them)."""
    h2, w2 = H // 2, W // 2
    h4, w4 = h2 // 2, w2 // 2
    h8, w8 = h4 // 2, w4 // 2
    macs = H * W * 64 * 9 * (1 + 64) + h2 * w2 * 64 * 9 * 64 * 2 + h4 * w4 * 9 * (64 * 128 + 128 * 128) \
        + h8 * w8 * (9 * 128 * 128 * 2 + 9 * 128 * 512 + 256 * 65 + 256 * 256)
    return 2 * macs


def reference(sd):
    from oracle import stage_reference

    if stage_reference.import_reference() is None:
        return None
    from gluefactory_nonfree.superpoint import SuperPoint as Reference

    saved = torch.hub.load_state_dict_from_url
    torch.hub.load_state_dict_from_url = lambda *a, **k: sd
    try:
        return Reference({"max_num_keypoints": 512, "force_num_keypoints": True}).cuda().eval()
    finally:
        torch.hub.load_state_dict_from_url = saved


def timed(fn, reps=3):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="256x480x640,64x1024x1024")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-ref", action="store_true")
    ap.add_argument("--step-pairs", type=int, default=128)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    conf = {"max_num_keypoints": 512, "force_num_keypoints": True, "weights": None}
    mine = {p: SuperPoint({**conf, "precision": p}) for p in ("bf16", "fp32")}
    sd = synthetic.make_superpoint_weights(mine["bf16"].state_dict(), seed=7)
    for m in mine.values():
        m.load_state_dict(sd)
        m.cuda().eval()
    ref = None if args.no_ref else reference(sd)
    for shape in args.shapes.split(","):
        B, H, W = map(int, shape.split("x"))
        data = {"image": synthetic.make_superpoint_images(1, 1, H, W, seed=1).expand(B, 1, H, W).contiguous().cuda()}
        arms = {"b200_bf16": lambda: mine["bf16"](data), "b200_fp32": lambda: mine["fp32"](data)}
        if ref is not None:
            def ref_fp32():
                with torch.no_grad(), torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
                    ref(data)

            def ref_autocast():
                with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                    ref(data)
            arms.update({"reference_fp32": ref_fp32, "reference_bf16_autocast": ref_autocast})
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                try:
                    times[k].append(timed(fn))
                except torch.OutOfMemoryError:
                    times[k].append(float("nan"))
                torch.cuda.empty_cache()
        res = {"shape": shape, "ms": {k: statistics.median(v) for k, v in times.items()},
               "conv_gflop_per_image": conv_flops(H, W) / 1e9}
        # per-kernel times, a separate pass
        _lib.timed_entry, _lib.timed_events = SP_ENTRIES, []
        _lib.timed_tagger = lambda name, a: (a[11] if name == "lgb200_sp_conv" else None)
        mine["bf16"](data)
        torch.cuda.synchronize()
        per = {}
        for s, e, tag in _lib.timed_events:
            per[str(tag)] = per.get(str(tag), 0.0) + s.elapsed_time(e)
        _lib.timed_entry, _lib.timed_tagger, _lib.timed_events = None, None, []
        conv_ms = sum(v for k, v in per.items() if "sp_conv" in k)
        res["kernel_ms"] = per
        res["conv_share_of_bf16_peak"] = conv_flops(H, W) * B / (conv_ms * 1e-3) / BF16_PEAK
        nms_bytes = B * (H // 8 * 8) * (W // 8 * 8) * 4 * 2  # read scores, write suppressed map
        sel_bytes = B * (H // 8 * 8) * (W // 8 * 8) * 4 * 7  # count pass + 4 radix passes + 2 gather passes (upper bound)
        nms_ms = sum(v for k, v in per.items() if "sp_nms" in k)
        sel_ms = sum(v for k, v in per.items() if "sp_select" in k)
        res["nms_bytes_per_s_share_of_hbm"] = nms_bytes / (nms_ms * 1e-3) / HBM
        res["select_bytes_per_s_share_of_hbm"] = sel_bytes / (sel_ms * 1e-3) / HBM
        print(json.dumps(res), flush=True)
        del data
        torch.cuda.empty_cache()
    step(args, mine["bf16"], ref)


def step(args, ext, ref):
    """Uncached homography pre-training step at P pairs x 512 keypoints, 480 x 640 views."""
    from gluefactory_b200.matchers.homography_matcher import HomographyMatcher
    from gluefactory_b200.matchers.lightglue import LightGlue
    from gluefactory_b200.trainer import MatcherTrainer

    P, H, W = args.step_pairs, 480, 640
    img = synthetic.make_superpoint_images(1, 1, H, W, seed=2).cuda()
    v0, v1 = img.expand(P, 1, H, W).contiguous(), img.flip(-1).expand(P, 1, H, W).contiguous()
    size = torch.tensor([W, H], dtype=torch.float32, device="cuda").expand(P, 2).contiguous()
    Hs = torch.eye(3, device="cuda").expand(P, 3, 3).contiguous()
    lconf = dict(synthetic.DEFAULT_CONF, precision="bf16")
    lg = LightGlue(lconf)
    lg.load_state_dict(synthetic.make_weights(lconf, seed=5), strict=False)
    tr = MatcherTrainer(lg.cuda().train(), lr=1e-5, ground_truth=HomographyMatcher({}))

    def run(extract):
        f0, f1 = extract(v0), extract(v1)
        tr.step({"keypoints0": f0["keypoints"], "keypoints1": f1["keypoints"], "descriptors0": f0["descriptors"],
                 "descriptors1": f1["descriptors"], "view0": {"image_size": size}, "view1": {"image_size": size},
                 "H_0to1": Hs})

    arms = {"b200_extractor": lambda: run(lambda v: ext({"image": v, "image_size": size}))}
    if ref is not None:
        def ref_extract(v):
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
                p = ref({"image": v, "image_size": size})
            return {k: t.float() for k, t in p.items()}
        arms["reference_extractor_bf16_autocast"] = lambda: run(ref_extract)
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, fn in arms.items():
            times[k].append(timed(fn, reps=2))
    print(json.dumps({"step": f"{P} pairs x 512 keypoints, {H}x{W}, extractor + ground truth + LightGlue",
                      "ms": {k: statistics.median(v) for k, v in times.items()}}), flush=True)


if __name__ == "__main__":
    main()
