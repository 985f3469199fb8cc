"""Generate the head-dimension-32 LightGlue fixtures under tests/golden/ by running the UNMODIFIED reference LightGlue
(gluefactory/models/matchers/lightglue.py) on the CPU: `descriptor_dim 128` with the default 4 heads (the compact model
for 128-channel DISK / ALIKED features) and `descriptor_dim 256` with 8 heads, both of which the reference builds with
head_dim = descriptor_dim // num_heads = 32 (lightglue.py:347), a [16, 2 (+2)] Fourier encoding and the scale
32^-1/2 in both attention blocks.  Test infrastructure only; it needs the reference tree ($GLUEFACTORY_REFERENCE) and
the omegaconf stand-in of oracle/_shim, like oracle/make_golden.py, whose helpers it uses.  It writes no other fixture.

    python scripts/make_lightglue_hd32_golden.py

Training mode, forward + loss + backward in fp64 (oracle/make_golden.py `run_case`, same keys as the head-dim-64
fixtures), plus one eval-mode point-pruning case in fp32 (the reference's pruning branch mixes default-dtype buffers
with the model dtype, so fp64 fails there) whose seed is chosen for margin, as `run_adaptive` does.
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import make_golden  # noqa: E402  (puts the reference and oracle/_shim on sys.path)
from gluefactory_b200 import synthetic  # noqa: E402

D128_H4 = dict(synthetic.DEFAULT_CONF, descriptor_dim=128, input_dim=128, num_heads=4)
D256_H8 = dict(synthetic.DEFAULT_CONF, num_heads=8)

# name -> (conf, B, N, M, seed)
CASES = {
    "lg_hd32_d128_h4_l3_n128": (dict(D128_H4, n_layers=3), 2, 128, 128, 211),
    "lg_hd32_d128_h4_l3_m80_n112": (dict(D128_H4, n_layers=3), 2, 112, 80, 213),
    "lg_hd32_d256_h8_l2_n128": (dict(D256_H8, n_layers=2), 2, 128, 128, 215),
    "lg_hd32_sift_d128_h4_l2_n96": (dict(D128_H4, n_layers=2, add_scale_ori=True), 1, 96, 80, 217),
}
ADAPTIVE = "lg_hd32_d128_h4_adaptive_prune"


def run_adaptive_hd32(name=ADAPTIVE, N=224, M=200, seeds=range(220, 260)):
    """Eval-mode point pruning (width_confidence 0.6, lightglue.py:461-526, 545-558) at 128 channels / 4 heads.  The
    seed is the first one whose every pruning decision clears its threshold by more than 2e-4 and that keeps between
    20 and M - 20 points of view 0, so the fixture does not hinge on fp32 rounding."""
    from gluefactory.models import get_model

    conf = dict(D128_H4, n_layers=5, width_confidence=0.6, depth_confidence=-1, filter_threshold=0.0)
    for seed in seeds:
        w = synthetic.make_weights(conf, seed=seed)
        model = get_model("matchers.lightglue")(dict(conf, name="matchers.lightglue"))
        missing, unexpected = model.load_state_dict(w, strict=False)
        assert not unexpected and missing in ([], ["confidence_thresholds"]), (missing, unexpected)
        model = model.eval()
        data = synthetic.make_pairs(1, N, seed=seed + 1, D=conf["input_dim"], M=M)
        margins = []
        orig = model.get_pruning_mask

        def spy(confidences, scores, layer_index, _orig=orig):
            margins.append((scores - (1 - conf["width_confidence"])).abs().min().item())
            return _orig(confidences, scores, layer_index)
        model.get_pruning_mask = spy
        with torch.no_grad():
            pred = model(data)
        kept = pred["log_assignment"].shape[1] - 1
        if min(margins) > 2e-4 and 20 < kept < M - 20:
            break
    else:
        raise RuntimeError("no seed with comfortable pruning margins")
    out = {"meta|conf": np.array(repr(conf)), "meta|seed": np.array(seed), "meta|M": np.array(M), "meta|N": np.array(N),
           "meta|min_margin": np.array(min(margins))}
    for k in ["matches0", "matches1", "matching_scores0", "matching_scores1", "prune0", "prune1", "log_assignment"]:
        out["pred|" + k] = pred[k].numpy()
    path = os.path.join(make_golden.OUT, name + ".npz")
    np.savez_compressed(path, **out)
    print(f"{name}: seed={seed} kept0={kept} kept1={pred['log_assignment'].shape[2] - 1} min margin={min(margins):.2e} "
          f"matches={int((pred['matches0'] > -1).sum())} -> {path} ({os.path.getsize(path) / 1e6:.2f} MB)")


if __name__ == "__main__":
    torch.manual_seed(0)
    torch.set_num_threads(8)
    for name, (conf, B, N, M, seed) in CASES.items():
        make_golden.run_case(name, conf, B=B, N=N, M=M, seed=seed)
    run_adaptive_hd32()
