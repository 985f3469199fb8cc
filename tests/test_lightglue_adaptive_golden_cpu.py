"""CPU: the early-stopping fixtures (tests/golden/lg_adaptive_*.npz, recorded from the unmodified reference by
scripts/make_lightglue_adaptive_golden.py) are consistent on their own, without the reference: each pair's stop layer
follows from its recorded low-confidence counts and depth_confidence (lightglue.py:559-570, in fp32), every stop test
clears depth_confidence by at least 3 tokens, the survivors implied by prune0/1 are the rows and columns of the
stored log_assignment, and the cases cover what the GPU test relies on (distinct and shared stop layers, views longer
than one 1024-token scan chunk)."""
import ast
import os

import numpy as np
import pytest

from tests.util import GOLDEN

CASES = ["lg_adaptive_a_depth", "lg_adaptive_b_both", "lg_adaptive_c_d128_both", "lg_adaptive_d_long"]


def _load(name):
    g = dict(np.load(os.path.join(GOLDEN, name + ".npz")))
    return g, ast.literal_eval(str(g["meta|conf"]))


@pytest.mark.parametrize("name", CASES)
def test_fixture_stop_layers_and_survivors(name):
    g, conf = _load(name)
    M, N, P, L = int(g["meta|M"]), int(g["meta|N"]), int(g["meta|pairs"]), conf["n_layers"]
    dc, wc = conf["depth_confidence"], conf["width_confidence"]
    assert dc > 0 and float(g["meta|min_ratio_margin_tokens"]) >= 3
    if wc > 0:
        assert float(g["meta|min_sig_margin"]) > 2e-4
    assert os.path.getsize(os.path.join(GOLDEN, name + ".npz")) < 2e6
    for j in range(P):
        p = f"p{j}|"
        low, stop = g[p + "low"], int(g[p + "stop_layer"])
        assert low.shape == (L - 1,)
        ratios = np.float32(1) - low.astype(np.float32) / np.float32(M + N)
        stops = [i for i in range(L - 1) if low[i] >= 0 and ratios[i] > np.float32(dc)]
        assert stops == ([stop] if stop < L - 1 else []), (j, low, stop)
        assert (low[:stop + 1 if stop < L - 1 else L - 1] >= 0).all() and (low[stop + 1:] == -1).all()
        checked = low[low >= 0]
        assert (np.abs((1 - dc) * (M + N) - checked) >= 3).all(), (j, checked)
        p0, p1 = g[p + "prune0"][0], g[p + "prune1"][0]
        if wc > 0:  # int64 layer counts: survivors were kept at every pruning step before the stop layer
            assert p0.dtype == p1.dtype == np.int64
            assert p0.max() == p1.max() == 1 + stop and p0.min() >= 1 and p1.min() >= 1
        else:
            assert (p0 == L).all() and (p1 == L).all()
        m, n = int((p0 == p0.max()).sum()), int((p1 == p1.max()).sum())
        shape = tuple(g[p + "la_shape"]) if p + "la_shape" in g else g[p + "log_assignment"].shape
        assert shape == (1, m + 1, n + 1), (j, shape, m, n)
        if p + "la_shape" in g:
            assert g[p + "la_rows"].max() < m and g[p + "la_cols"].max() < n
            assert g[p + "la_dust_row"].shape == (n + 1,) and g[p + "la_dust_col"].shape == (m + 1,)
            assert g[p + "la_row_lse"].shape == (m,)
        m0, m1 = g[p + "matches0"][0], g[p + "matches1"][0]
        assert (p0[m0 >= 0] == p0.max()).all() and (p1[m1 >= 0] == p1.max()).all()  # only survivors match
        assert all(m1[m0[i]] == i for i in np.flatnonzero(m0 >= 0))


def test_fixture_cases_cover_the_branches():
    stops = lambda g: [int(g[f"p{j}|stop_layer"]) for j in range(int(g["meta|pairs"]))]  # noqa: E731
    a, conf = _load("lg_adaptive_a_depth")
    s = stops(a)
    assert len(set(s)) >= 2 and min(s) < conf["n_layers"] - 1 and len(set(s)) < len(s)  # shared: one batched head
    for name in ("lg_adaptive_b_both", "lg_adaptive_c_d128_both"):
        g, _ = _load(name)
        kept = [int((g[f"p{j}|prune0"] == g[f"p{j}|prune0"].max()).sum()) for j in range(int(g["meta|pairs"]))]
        assert len(set(stops(g))) >= 2 and len(set(kept)) >= 2, (name, stops(g), kept)
    d, _ = _load("lg_adaptive_d_long")
    assert int(d["meta|M"]) > 1024 and int(d["meta|N"]) > 1024
    assert max(stops(d)) > 0  # a pair that goes on: its views are scanned in two chunks
    total = sum(os.path.getsize(os.path.join(GOLDEN, n + ".npz")) for n in
                ("lg_adaptive_a_depth", "lg_adaptive_b_both", "lg_adaptive_c_d128_both", "lg_adaptive_d_long"))
    assert total < 6e6
