"""SuperGlue training step on one GPU: the plugin (bf16 and fp32, eager and as one CUDA-graph replay through
trainer.MatcherTrainer) against the unmodified reference module from oracle/_ref in PyTorch eager on the same GPU (fp32
and bf16 autocast), plus the time of the Sinkhorn forward and backward entry points inside the plugin's step.

    PB=8,32 PN=2048 python scripts/prof_superglue.py

Forward + loss + backward + Adam on a synthetic batch of PB pairs (comma list) with PN keypoints per image, the
default configuration (9 self + 9 cross layers, 50 Sinkhorn iterations).  Achieved bandwidth of the Sinkhorn kernels is
from algorithmic bytes: the forward streams the [B,M,N] fp32 cost twice per iteration (row and column phase),
2 iters B M N 4 bytes; the backward reads the cost twice and reads + writes the gradient once per iteration,
4 iters B M N 4 bytes.  With the strip cache on (B * strips <= SMs and the strip fits in shared memory) the cost is
read from shared memory after the first pass, so these figures then exceed HBM bandwidth.
"""
import os
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gluefactory_b200 import _lib, synthetic  # noqa: E402
from gluefactory_b200.matchers.superglue import SuperGlue  # noqa: E402

BS = [int(b) for b in os.environ.get("PB", "8,32").split(",")]
N = int(os.environ.get("PN", "2048"))
dev = torch.device("cuda", 0)
SK = ("lgb200_sinkhorn_fwd_dev", "lgb200_sinkhorn_bwd_dev")


def timed(step, reps=5, warm=2):
    for _ in range(warm):
        step()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        step()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / reps * 1e3


def make_step(model, data, autocast=None, reference=False):
    opt = torch.optim.Adam(model.parameters(), lr=1e-5)

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=autocast, enabled=autocast is not None):
            pred = model(data)
            out = model.loss(pred, data)
            losses = out if reference else out[0]  # the reference's loss returns the losses alone
            loss = losses["total"].mean()
        loss.backward()
        opt.step()
        return loss

    return step


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as e:  # noqa: BLE001
        return f"nvidia-smi unavailable: {e}"


print("card (name, power limit, max SM clock):", card())
conf = {k: v for k, v in SuperGlue.default_conf.items()}
conf["weights"] = None
iters = conf["num_sinkhorn_iterations"]
for B in BS:
    data = synthetic.to_device(synthetic.make_superglue_batch(B, N, N, 5), dev)
    rows = []
    w = None
    for prec in ("bf16", "fp32"):
        m = SuperGlue(dict(conf, precision=prec))
        w = synthetic.make_gluestick_weights(m.state_dict(), seed=3) if w is None else w
        m.load_state_dict(w, strict=True)
        m = m.to(dev).train()
        ms = timed(make_step(m, data))
        rows.append((f"plugin {prec}, eager", ms))
        # per-entry-point time of the Sinkhorn kernels inside one more eager step
        _lib.timed_entry, _lib.timed_events[:] = set(SK), []
        make_step(m, data)()
        torch.cuda.synchronize()
        _lib.timed_entry = None
        ev = _lib.timed_events  # one forward call, then one backward call
        assert len(ev) == 2, len(ev)
        t = {SK[0]: ev[0][0].elapsed_time(ev[0][1]), SK[1]: ev[1][0].elapsed_time(ev[1][1])}
        fwd_b, bwd_b = 2 * iters * B * N * N * 4, 4 * iters * B * N * N * 4
        rows.append((f"  sinkhorn fwd ({prec} step)", t[SK[0]], fwd_b / (t[SK[0]] * 1e-3) / 1e9))
        rows.append((f"  sinkhorn bwd ({prec} step)", t[SK[1]], bwd_b / (t[SK[1]] * 1e-3) / 1e9))
        rows.append((f"  sinkhorn share of the {prec} eager step", 100 * (t[SK[0]] + t[SK[1]]) / ms, None))
        del m
        torch.cuda.empty_cache()
    for prec in ("bf16", "fp32"):
        try:
            from gluefactory_b200.trainer import MatcherTrainer

            m = SuperGlue(dict(conf, precision=prec))
            m.load_state_dict(w, strict=True)
            tr = MatcherTrainer(m.to(dev).train(), lr=1e-5)
            rows.append((f"plugin {prec}, MatcherTrainer eager", timed(lambda: tr.step(data))))
            tr.capture(data, dev)
            rows.append((f"plugin {prec}, CUDA-graph replay", timed(lambda: tr.step_graphed(data))))
            del m, tr
        except Exception as e:  # noqa: BLE001
            rows.append((f"plugin {prec} graph: {type(e).__name__}: {str(e)[:120]}", float("nan")))
        torch.cuda.empty_cache()
    try:
        from oracle.stage_reference import import_reference

        if import_reference() is None:
            raise RuntimeError("oracle/_ref not staged")
        from gluefactory_nonfree.superglue import SuperGlue as Reference

        ref_data = dict(data)
        for i in "01":  # the reference reads view["image"].shape even when image_size is given
            ref_data["view" + i] = dict(data["view" + i], image=torch.zeros((), device=dev).expand(B, 1, 1024, 1024))
        ref_conf = {k: v for k, v in conf.items() if k != "precision"}
        for ac, tag in ((None, "fp32"), (torch.bfloat16, "bf16 autocast")):
            try:
                ref = Reference(dict(ref_conf))
                ref.load_state_dict(w, strict=True)
                ms = timed(make_step(ref.to(dev).train(), ref_data, ac, reference=True), reps=3, warm=1)
                rows.append((f"reference eager {tag}", ms))
            except torch.OutOfMemoryError:
                rows.append((f"reference eager {tag}: out of memory (80 GB)", float("nan")))
            ref = None
            torch.cuda.empty_cache()
    except Exception as e:  # noqa: BLE001
        rows.append((f"reference unavailable: {type(e).__name__}: {str(e)[:120]}", float("nan")))
    print(f"SuperGlue training step, B={B} pairs, N={N} keypoints per image, {iters} Sinkhorn iterations")
    for r in rows:
        if len(r) == 3 and r[2] is None:
            print(f"  {r[0]:44s} {r[1]:9.1f} %")
        elif len(r) == 3:
            print(f"  {r[0]:44s} {r[1]:9.2f} ms       {r[2]:8.0f} GB/s (algorithmic)")
        else:
            print(f"  {r[0]:44s} {r[1]:9.1f} ms/step  {B / r[1] * 1e3:8.1f} pairs/s")
    sys.stdout.flush()
