"""SuperPoint-open forward on Hopper, eval and training mode, against the non-free plugin on the same shapes and the
unmodified reference `superpoint_open` (oracle/_ref, staged by the build) under bf16 autocast and fp32, in alternating
rounds; then the uncached homography pre-training step (the extractor in training mode on both views + device ground
truth + LightGlue), eager and captured as one CUDA graph.  Prints JSON lines: the card with its power limit (same
call), then median times per arm.

    python scripts/prof_superpoint_open.py [--shapes 256x480x640x512,64x1024x1024x2048] [--rounds 3] [--no-ref]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gluefactory_b200 import synthetic  # noqa: E402
from gluefactory_b200.extractors.superpoint import SuperPoint  # noqa: E402
from gluefactory_b200.extractors.superpoint_open import SuperPointOpen  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else torch.cuda.get_device_name()


def timed(fn, reps=3):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn()
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / reps


def reference(path, K):
    from oracle import stage_reference

    if stage_reference.import_reference() is None:
        return None
    from gluefactory.models.extractors.superpoint_open import SuperPoint as Reference

    return Reference({"max_num_keypoints": K, "force_num_keypoints": True, "weights": path, "trainable": False}).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="256x480x640x512,64x1024x1024x2048")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-ref", action="store_true")
    ap.add_argument("--step-pairs", type=int, default=128)
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    tmp = tempfile.mkdtemp()
    path = os.path.join(tmp, "sp_open.pth")
    torch.save(synthetic.make_superpoint_open_weights(SuperPointOpen.state_dict_template(), seed=11), path)
    for shape in args.shapes.split(","):
        B, H, W, K = map(int, shape.split("x"))
        conf = {"max_num_keypoints": K, "force_num_keypoints": True, "weights": path}
        mine = SuperPointOpen(conf).cuda()
        nonfree = SuperPoint({"max_num_keypoints": K, "force_num_keypoints": True, "weights": None}).cuda().eval()
        nonfree.load_state_dict(synthetic.make_superpoint_weights(nonfree.state_dict(), seed=7))
        ref = None if args.no_ref else reference(path, K)
        data = {"image": synthetic.make_superpoint_images(1, 1, H, W, seed=1).expand(B, 1, H, W).contiguous().cuda()}
        arms = {"open_bf16_eval": lambda: mine.eval()(data), "open_bf16_train": lambda: mine.train()(data),
                "nonfree_plugin_bf16": lambda: nonfree(data)}
        if ref is not None:
            def ref_arm(train, autocast):
                def run():
                    ref.train(train)
                    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast), \
                            torch.backends.cudnn.flags(enabled=True, allow_tf32=False):
                        ref(data)
                return run
            arms.update({"reference_eval_bf16_autocast": ref_arm(False, True), "reference_eval_fp32": ref_arm(False, False),
                         "reference_train_bf16_autocast": ref_arm(True, True),
                         "reference_train_fp32": ref_arm(True, False)})
        times = {k: [] for k in arms}
        for _ in range(args.rounds):
            for k, fn in arms.items():
                try:
                    times[k].append(timed(fn))
                except torch.OutOfMemoryError:
                    times[k].append(float("nan"))
                torch.cuda.empty_cache()
        print(json.dumps({"shape": f"{B} x {H}x{W}, K {K}", "ms": {k: statistics.median(v) for k, v in times.items()},
                          "peak_gib": torch.cuda.max_memory_allocated() / 2 ** 30}), flush=True)
        del data, mine, nonfree, ref
        torch.cuda.empty_cache()
    step(args, path)


def step(args, path):
    """Uncached homography pre-training step at P pairs x 512 keypoints, 480 x 640 views, extractor in training mode."""
    from gluefactory_b200.matchers.homography_matcher import HomographyMatcher
    from gluefactory_b200.matchers.lightglue import LightGlue
    from gluefactory_b200.trainer import MatcherTrainer

    P, H, W = args.step_pairs, 480, 640
    ext = SuperPointOpen({"max_num_keypoints": 512, "force_num_keypoints": True, "detection_threshold": -1,
                          "nms_radius": 3, "weights": path}).cuda().train()
    img = synthetic.make_superpoint_images(1, 1, H, W, seed=2).cuda()
    v0, v1 = img.expand(P, 1, H, W).contiguous(), img.flip(-1).expand(P, 1, H, W).contiguous()
    size = torch.tensor([W, H], dtype=torch.float32, device="cuda").expand(P, 2).contiguous()
    Hs = torch.eye(3, device="cuda").expand(P, 3, 3).contiguous()
    lconf = dict(synthetic.DEFAULT_CONF, precision="bf16")
    lg = LightGlue(lconf)
    lg.load_state_dict(synthetic.make_weights(lconf, seed=5), strict=False)
    tr = MatcherTrainer(lg.cuda().train(), lr=1e-5, ground_truth=HomographyMatcher({}))

    def run():
        f0, f1 = ext({"image": v0, "image_size": size}), ext({"image": v1, "image_size": size})
        tr.step({"keypoints0": f0["keypoints"], "keypoints1": f1["keypoints"], "descriptors0": f0["descriptors"],
                 "descriptors1": f1["descriptors"], "view0": {"image_size": size}, "view1": {"image_size": size},
                 "H_0to1": Hs})

    def ext_only():
        ext({"image": v0, "image_size": size}), ext({"image": v1, "image_size": size})

    res = {"step": f"{P} pairs x 512 keypoints, {H}x{W}, extractor (training mode) x 2 + ground truth + LightGlue"}
    eager = [timed(run, reps=2) for _ in range(args.rounds)]
    res["eager_ms"] = statistics.median(eager)
    res["extractor_x2_ms"] = statistics.median([timed(ext_only, reps=2) for _ in range(args.rounds)])
    try:
        s = torch.cuda.Stream()
        s.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(s):
            run()
        torch.cuda.current_stream().wait_stream(s)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            run()
        res["graph_ms"] = statistics.median([timed(graph.replay, reps=3) for _ in range(args.rounds)])
    except Exception as ex:  # noqa: BLE001 -- report why the step could not be captured
        res["graph_error"] = f"{type(ex).__name__}: {ex}"[:300]
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
