"""Cost of the device line ground truth (csrc/gt_lines.cu): CUDA-event times of the label pass and of the assignment
solver at B in {8, 32} x L in {250, 512} lines per image (npts 50), and the GlueStick CUDA-graph training step at
prof_gluestick.py's shape (8 pairs, 2048 points + 512 lines) with the line labels produced on the device by the
ground-truth component against labels precomputed once.  Prints the card and its power limit first."""
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gluefactory_b200 import ops, synthetic  # noqa: E402
from gluefactory_b200.geometry import inv3x3, warp_points  # noqa: E402

dev = torch.device("cuda", 0)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip()
    return f"{torch.cuda.get_device_name(0)} | nvidia-smi: {q}"


def event_ms(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def kernels(B, L, npts=50, h=480, w=640):
    sc = synthetic.to_device(synthetic.line_gt_scene("homography", B, L, L, 400 + B + L), dev)
    segs = [ops.line_segments(sc[f"lines{i}"], h, w) for i in "01"]
    p01 = warp_points(ops.sample_line_points(segs[0], npts), sc["H_0to1"])
    p10 = warp_points(ops.sample_line_points(segs[1], npts), inv3x3(sc["H_0to1"]))
    args = (segs[0], segs[1], p01, p10, (h, w), (h, w), sc["valid_lines0"], sc["valid_lines1"])
    full = event_ms(lambda: ops.gt_line_matches_from_projection(*args, npts=npts))
    cost = ops.gt_line_matches_from_projection(*args, npts=npts, return_cost=True)["cost"].clone()
    solver = event_ms(lambda: ops.linear_sum_assignment(cost))
    whole = event_ms(lambda: ops.gt_line_matches_from_homography(sc["lines0"], sc["lines1"], sc["valid_lines0"],
                                                                  sc["valid_lines1"], (h, w), (h, w), sc["H_0to1"],
                                                                  npts=npts, min_visibility_th=0.5))
    pos = int(ops.gt_line_matches_from_projection(*args, npts=npts)["line_assignment"].sum())
    return full, solver, whole, pos


def gluestick_step(B=8, N=2048, L=512, reps=10):
    from gluefactory_b200.matchers.gluestick import GlueStick
    from gluefactory_b200.matchers.homography_matcher import HomographyMatcher
    from gluefactory_b200.trainer import MatcherTrainer

    d = synthetic.make_gluestick_batch(B, N, L, 5)
    for i in "01":
        d[f"valid_lines{i}"] = torch.ones(B, L, dtype=torch.bool)
        d[f"view{i}"]["image"] = torch.zeros(B, 1, 1024, 1024)
    data = synthetic.to_device(d, dev)
    gt = HomographyMatcher({"use_lines": True, "th_positive": 3.0, "th_negative": 3.0})
    pre = dict(data, **{f"gt_{k}": v for k, v in gt(data).items()})  # the same labels, computed once
    w = None
    rows = []
    for tag, batch, g in (("device labels in the step", data, gt), ("precomputed labels", pre, None)):
        m = GlueStick(dict(GlueStick.default_conf, precision="bf16"))
        w = synthetic.make_gluestick_weights(m.state_dict(), seed=3) if w is None else w
        m.load_state_dict(w, strict=True)
        tr = MatcherTrainer(m.to(dev).train(), lr=1e-5, ground_truth=g)
        tr.capture(batch, dev)
        rows.append((tag, event_ms(lambda: tr.step_graphed(batch), reps=reps, warm=2)))
        del tr, m
    t_gt = event_ms(lambda: gt(data), reps=reps)
    return rows, t_gt


if __name__ == "__main__":
    print(card())
    print("line ground truth, homography variant, npts 50, L0 = L1 = L (times per call, all B pairs)")
    print(f"{'B':>4} {'L':>5} {'label pass+solver ms':>21} {'solver alone ms':>16} {'whole op ms':>12} {'positives':>10}")
    for B in (8, 32):
        for L in (250, 512):
            full, solver, whole, pos = kernels(B, L)
            print(f"{B:4d} {L:5d} {full:21.3f} {solver:16.3f} {whole:12.3f} {pos:10d}")
    rows, t_gt = gluestick_step()
    print("GlueStick bf16 training step, CUDA-graph replay, B=8, N=2048, L=512")
    for tag, ms in rows:
        print(f"  {tag:28s} {ms:8.2f} ms/step")
    print(f"  ground-truth component alone (points + lines, eager) {t_gt:8.2f} ms")
