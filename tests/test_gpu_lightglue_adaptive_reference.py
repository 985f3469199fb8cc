"""GPU: LightGlue's adaptive depth / width (eval mode, fp32) against the early-stopping fixtures recorded from the
unmodified reference (scripts/make_lightglue_adaptive_golden.py, tests/golden/lg_adaptive_*.npz).

Each fixture holds one weight set and 2-4 pairs that stop at different layers (`depth_confidence`) and, in cases
b-d, keep different numbers of points (`width_confidence`); case d has views of 1100 / 1300 tokens.  Every recorded
decision clears its threshold by at least 3 tokens (stop ratio) or 2e-4 (sigmoids), so the fixtures do not hinge on
fp32 rounding.  Each fixture is run three ways -- every pair alone, all pairs as one batch, the batch in reversed
order -- and held to the bars of the one-pair pruning tests: stop layer, prune0/1 and matches0/1 exactly, matching
scores within 1e-3 relative / 1e-6 absolute, log_assignment within 1e-3 / 1e-3 on the survivors' rows and columns plus
the dustbins, and -inf at the pruned rows and columns of the batched [B, M+1, N+1] matrix.  bf16 stays out: its
decisions may legitimately flip near a threshold (its self-consistency is in test_gpu_lightglue_adaptive_batch.py).

Budget: well under a minute and under 2 GiB of device memory on one H100, recorded by the module fixture."""
import ast
import os
import time

import numpy as np
import pytest
import torch

from gluefactory_b200 import synthetic
from gluefactory_b200.matchers.lightglue import LightGlue
from tests.util import GOLDEN, report

pytestmark = pytest.mark.gpu
DEV = "cuda"
CASES = ["lg_adaptive_a_depth", "lg_adaptive_b_both", "lg_adaptive_c_d128_both", "lg_adaptive_d_long"]


@pytest.fixture(scope="module", autouse=True)
def _file_budget():
    """Wall time and peak device memory of this file (the machines running it are shared)."""
    torch.cuda.reset_peak_memory_stats()
    t = time.time()
    yield
    torch.cuda.synchronize()
    report("test_gpu_lightglue_adaptive_reference", seconds=time.time() - t,
           peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)


def load_fixture(name):
    """(golden dict, conf, weights, [one-pair input dicts on the CPU]) rebuilt from the stored seeds: make_weights with
    the matchability and token-confidence weights scaled by meta|head_scale and the calibrated token biases."""
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    conf = ast.literal_eval(str(g["meta|conf"]))
    M, N, D = int(g["meta|M"]), int(g["meta|N"]), conf["input_dim"]
    w = dict(synthetic.make_weights(conf, seed=int(g["meta|seed"])))
    scale = float(g["meta|head_scale"])
    for i in range(conf["n_layers"]):
        for k in (f"log_assignment.{i}.matchability.weight", f"log_assignment.{i}.matchability.bias",
                  f"token_confidence.{i}.token.0.weight"):
            if k in w:
                w[k] = w[k] * scale
    for i, b in enumerate(g["meta|token_bias"]):
        w[f"token_confidence.{i}.token.0.bias"] = torch.tensor([float(b)], dtype=torch.float32)
    pairs = [synthetic.make_pairs(1, N, seed=int(s), D=D, M=M, frac=float(f))
             for s, f in zip(g["meta|pair_seeds"], g["meta|fracs"])]
    pairs = [{k: p[k] for k in ("keypoints0", "keypoints1", "descriptors0", "descriptors1")} |
             {"view0": {"image_size": p["view0"]["image_size"]}, "view1": {"image_size": p["view1"]["image_size"]}}
             for p in pairs]
    return g, conf, w, pairs


def _cat(pairs):
    c = lambda key: torch.cat([p[key] for p in pairs])  # noqa: E731
    return synthetic.to_device({"keypoints0": c("keypoints0"), "keypoints1": c("keypoints1"),
                                "descriptors0": c("descriptors0"), "descriptors1": c("descriptors1"),
                                "view0": {"image_size": torch.cat([p["view0"]["image_size"] for p in pairs])},
                                "view1": {"image_size": torch.cat([p["view1"]["image_size"] for p in pairs])}}, DEV)


def _check_la(la, g, p, tag):
    """la [m+1, n+1] in the survivors' indexing against pair p's fixture (full, or case d's subset)."""
    if p + "log_assignment" in g:
        ref = g[p + "log_assignment"][0]
        assert la.shape == ref.shape, (tag, la.shape, ref.shape)
        np.testing.assert_allclose(la, ref, rtol=1e-3, atol=1e-3, err_msg=tag)
        return float(np.abs(la - ref).max())
    m, n = int(g[p + "la_shape"][1]) - 1, int(g[p + "la_shape"][2]) - 1
    assert la.shape == (m + 1, n + 1), (tag, la.shape)
    worst = 0.0
    for got, ref in ((la[np.ix_(g[p + "la_rows"], g[p + "la_cols"])], g[p + "la_sub"]),
                     (la[m], g[p + "la_dust_row"]), (la[:, n], g[p + "la_dust_col"])):
        np.testing.assert_allclose(got, ref, rtol=1e-3, atol=1e-3, err_msg=tag)
        worst = max(worst, float(np.abs(got - ref).max()))
    lse = torch.logsumexp(torch.from_numpy(la[:m]).double(), -1).numpy()
    np.testing.assert_allclose(lse, g[p + "la_row_lse"], rtol=1e-3, atol=1e-3, err_msg=tag)
    return worst


def _check_pair(pred, b, g, j, M, N, batched, tag):
    """Pair b of pred against fixture pair j."""
    p = f"p{j}|"
    stop = pred["stop_layer"][b] if batched else pred["stop_layer"]
    assert int(stop) == int(g[p + "stop_layer"]), (tag, int(stop), int(g[p + "stop_layer"]))
    for k in ("prune0", "prune1", "matches0", "matches1"):
        got = pred[k][b].cpu().numpy()
        assert np.array_equal(got, g[p + k][0].astype(got.dtype)), (tag, k, np.flatnonzero(got != g[p + k][0])[:8])
    for k in ("matching_scores0", "matching_scores1"):
        np.testing.assert_allclose(pred[k][b].cpu().numpy(), g[p + k][0], rtol=1e-3, atol=1e-6, err_msg=f"{tag} {k}")
    la = pred["log_assignment"][b].cpu().numpy()
    if batched:  # original indexing: survivors' rows / columns + dustbins, -inf elsewhere
        p0, p1 = g[p + "prune0"][0], g[p + "prune1"][0]
        rows = np.concatenate([np.flatnonzero(p0 == p0.max()), [M]])
        cols = np.concatenate([np.flatnonzero(p1 == p1.max()), [N]])
        pruned_r = np.setdiff1d(np.arange(M + 1), rows)
        pruned_c = np.setdiff1d(np.arange(N + 1), cols)
        assert np.isneginf(la[pruned_r]).all() and np.isneginf(la[:, pruned_c]).all(), tag
        la = la[np.ix_(rows, cols)]
    return _check_la(la, g, p, tag)


@pytest.mark.parametrize("name", CASES)
def test_adaptive_against_reference_fixture(name):
    g, conf, w, pairs = load_fixture(name)
    M, N, P = int(g["meta|M"]), int(g["meta|N"]), int(g["meta|pairs"])
    model = LightGlue(dict(conf, precision="fp32"))
    missing, unexpected = model.load_state_dict(w, strict=False)
    assert not unexpected and missing in ([], ["confidence_thresholds"])
    model = model.to(DEV).eval()
    worst = 0.0
    with torch.no_grad():
        for j, pair in enumerate(pairs):
            worst = max(worst, _check_pair(model(synthetic.to_device(pair, DEV)), 0, g, j, M, N, False,
                                           f"{name} pair {j} alone"))
        for order in (list(range(P)), list(range(P))[::-1]):
            pred = model(_cat([pairs[j] for j in order]))
            assert pred["log_assignment"].shape == (P, M + 1, N + 1)
            for b, j in enumerate(order):
                worst = max(worst, _check_pair(pred, b, g, j, M, N, True, f"{name} batch {order} pair {j}"))
    stops = [int(g[f"p{j}|stop_layer"]) for j in range(P)]
    report(f"adaptive reference {name}", la_max_abs=worst, stops=str(stops))
