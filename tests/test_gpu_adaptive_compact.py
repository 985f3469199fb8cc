"""GPU: LightGlue's adaptive stop / prune / gather step (lgb200_adaptive_compact: adaptive_decide_kernel and
adaptive_gather_kernel) against a plain per-token restatement of the reference's rules (lightglue.py:485-511,
550-570), at evaluation sizes, at the ABI's limits and at exact decision ties.

The restatement (`ref_step`) computes every sigmoid with torch.sigmoid on the GPU in fp32 and compares it with the
thresholds as the reference does: a pair stops when 1 - #(confidence < thr) / (M + N) > depth_confidence (the
ORIGINAL M + N, strict, fp32), and a token of a pair that goes on stays when its matchability > 1 - width_confidence
or, with early stopping, its confidence <= thr.  No logit is moved away from a threshold, so every decision, keep
and stop, must equal torch's element for element; the packed x / theta / ind, the new segments, the prune counters,
the final buffer and the status are compared exactly.

Sizes: views of 2048 tokens and segments of 1023, 1024, 1025, 2047 and 2048 tokens (one, two and exactly full
1024-thread scan chunks of the decide kernel); 300 pairs with stopped ones interleaved (more than 256 segments per
gather thread block, so each thread scans several); a token count from the SM count at which the gather's grid-stride
loop wraps; 4096 pairs, the ABI's limit; D / R = 256 / 32 and 128 / 16.  Ties: logits whose sigmoid lands exactly on,
and within 64 fp32 ulps of, each confidence threshold of a 9-layer model and 1 - width_confidence at 0.99 and 0.6;
low counts that put the stop ratio exactly on depth_confidence and one count either side.  Chained: L - 1 steps in a
row, each on the previous one's output, then the finishing step without logits.

Budget: a few seconds and well under 1 GiB of device memory on one H100, recorded by the module fixture."""
import math
import time

import pytest
import torch

from gluefactory_b200 import ops
from tests.util import report

pytestmark = pytest.mark.gpu
DEV = "cuda"
I32 = dict(device=DEV, dtype=torch.int32)
STOP_SENTINEL, IND_SENTINEL, X_SENTINEL = 77, -7, -3.5


@pytest.fixture(scope="module", autouse=True)
def _file_budget():
    """Wall time and peak device memory of this file (the machines running it are shared)."""
    torch.cuda.reset_peak_memory_stats()
    t = time.time()
    yield
    torch.cuda.synchronize()
    report("test_gpu_adaptive_compact", seconds=time.time() - t, peak_gib=torch.cuda.max_memory_allocated() / 2 ** 30)


def thresholds(n_layers):
    """LightGlue's per-layer confidence thresholds as the module registers them (fp32)."""
    return torch.tensor([min(max(0.8 + 0.1 * math.exp(-4.0 * i / n_layers), 0.0), 1.0) for i in range(n_layers)])


def new_fin(B, M, N, D):
    return {"x": torch.full((B * (M + N), D), X_SENTINEL, device=DEV),
            "ind": torch.full((B * (M + N),), IND_SENTINEL, **I32), "len": torch.zeros(2 * B, **I32),
            "stop": torch.full((B,), STOP_SENTINEL, **I32),
            "prune0": torch.ones(B, M, device=DEV, dtype=torch.int64),
            "prune1": torch.ones(B, N, device=DEV, dtype=torch.int64)}


def _clone(fin):
    return {k: v.clone() for k, v in fin.items()}


def ref_step(x, theta, ind, zt, off, ln, fin, thr, dc, wc, layer, finish, B, M, N):
    """One step of the reference's rules on the packed state.  off / ln: the 2B segment offsets and lengths (lists);
    fin is updated in place.  Returns (x, theta, ind, new offsets, new lengths, status, keep) with the packed rows in
    pair-major segment order."""
    S = 2 * B
    lens = torch.tensor(ln, device=DEV, dtype=torch.int64)
    starts = torch.tensor(off, device=DEV, dtype=torch.int64)
    excl = torch.cumsum(lens, 0) - lens
    tot = int(lens.sum())
    sid = torch.arange(S, device=DEV).repeat_interleave(lens)
    pos = torch.arange(tot, device=DEV) - excl.repeat_interleave(lens)
    order = starts.repeat_interleave(lens) + pos          # tokens segment by segment, in their order
    b, img = sid // 2, sid % 2
    active = (lens.view(B, 2).sum(1) > 0)
    if finish:
        stop_b = active
    elif dc > 0:
        tok = torch.sigmoid(zt[order, 1])
        low = torch.zeros(B, device=DEV, dtype=torch.int64).index_add_(0, b, (tok < thr).long())
        ratio = 1.0 - low.float() / (M + N)                  # lightglue.py:569-570 (fp32, original M + N)
        stop_b = active & (ratio > dc)
    else:
        stop_b = torch.zeros(B, device=DEV, dtype=torch.bool)
    stop_t = stop_b[b]
    keep = ~stop_t
    if wc > 0 and not finish:
        k = torch.sigmoid(zt[order, 0]) > (1 - wc)           # lightglue.py:554
        if dc > 0:
            k = k | (tok <= thr)                              # lightglue.py:556 (low confidence is never pruned)
        keep = keep & k
    cnt = torch.zeros(S, device=DEV, dtype=torch.int64).index_add_(0, sid, keep.long())
    new_len = cnt.tolist()
    new_off = (torch.cumsum(cnt, 0) - cnt).tolist()
    src = order[keep]
    if wc > 0 and not finish:
        for j, (p, n) in enumerate(((fin["prune0"], M), (fin["prune1"], N))):
            sel = keep & (img == j)
            p.view(-1).index_put_((b[sel] * n + ind[order[sel]].long(),), torch.ones_like(b[sel]), accumulate=True)
    fsrc = order[stop_t]
    frow = b[stop_t] * (M + N) + torch.where(img[stop_t] == 0, pos[stop_t], M + pos[stop_t])
    fin["x"][frow] = x[fsrc]
    fin["ind"][frow] = ind[fsrc]
    sb = torch.where(stop_b)[0]
    fin["stop"][sb] = layer
    fin["len"].view(B, 2)[sb] = lens.view(B, 2)[sb].int()
    emptied = bool((active & ~stop_b & (cnt.view(B, 2) == 0).any(1)).any())
    return x[src], theta[src], ind[src], new_off, new_len, [len(src), int(emptied)], keep


def run_both(x, theta, ind, zt, off, ln, fin, fin_ref, thr, dc, wc, layer, B, M, N, finish=False, tag=""):
    """The kernel and the restatement on the same state; every output compared exactly.  Returns the next state."""
    S = 2 * B
    seg = torch.tensor([off, ln, [off[s ^ 1] for s in range(S)], [ln[s ^ 1] for s in range(S)]], **I32)
    thr_t = thr.reshape(1).to(DEV, torch.float32)
    xo, to, io, so, status = ops.adaptive_compact(x, theta, ind, None if finish else zt, seg, fin, layer, (B, M, N),
                                                  conf_thr=None if finish else thr_t, depth_conf=dc, width_conf=wc,
                                                  finish=finish)
    rx, rt, ri, roff, rlen, rstatus, _ = ref_step(x, theta, ind, zt, off, ln, fin_ref, thr_t[0], dc, wc, layer, finish,
                                                  B, M, N)
    kept = rstatus[0]
    assert status.tolist() == rstatus, (tag, status.tolist(), rstatus)
    assert so.tolist() == [roff, rlen, [roff[s ^ 1] for s in range(S)], [rlen[s ^ 1] for s in range(S)]], tag
    assert torch.equal(xo[:kept], rx) and torch.equal(to[:kept], rt) and torch.equal(io[:kept], ri), tag
    for k in ("x", "ind", "len", "stop", "prune0", "prune1"):  # rows of pairs that have not stopped keep the sentinels
        assert torch.equal(fin[k], fin_ref[k]), (tag, k)
    return xo[:kept], to[:kept], io[:kept], roff, rlen


def make_state(lens, M, N, D, R, seed, layout="pair-major"):
    """Packed state with segment lengths `lens` (2B entries); each token's keypoint index is distinct within its view.
    layout "pair-major": segments back to back in segment order; "first": [image 0 of every pair; image 1 of every
    pair], as the adaptive forward packs the first layer."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    B = len(lens) // 2
    order = list(range(0, 2 * B, 2)) + list(range(1, 2 * B, 2)) if layout == "first" else list(range(2 * B))
    off, r = [0] * (2 * B), 0
    for s in order:
        off[s] = r
        r += lens[s]
    T = r
    x = torch.randn(T, D, generator=g).to(DEV)
    theta = torch.randn(T, R, generator=g).to(DEV)
    ind = torch.empty(T, dtype=torch.int32)
    for s in range(2 * B):
        n = M if s % 2 == 0 else N
        c = int(torch.randint(0, n, (1,), generator=g))
        a = next(a for a in (7, 11, 13) if math.gcd(a, n) == 1)  # coprime to n: distinct indices within the view
        ind[off[s]:off[s] + lens[s]] = (torch.arange(lens[s]) * a + c) % n
    return x, theta, ind.to(DEV), off, T


def random_zt(T, seed, conf_shift=None, sid=None):
    g = torch.Generator(device="cpu").manual_seed(seed)
    zt = (torch.randn(T, 2, generator=g) * 3).to(DEV)
    if conf_shift is not None:  # per-pair shift of the confidence logits: some pairs stop, others go on
        zt[:, 1] += conf_shift[sid // 2]
    return zt


def _sid(off, ln, T):
    sid = torch.empty(T, dtype=torch.int64)
    for s, (o, n) in enumerate(zip(off, ln)):
        sid[o:o + n] = s
    return sid.to(DEV)


def _size_case(name, sm):
    g = torch.Generator(device="cpu").manual_seed(len(name))
    if name == "eval_2048":    # two pairs at 2048 / 2048 and segments around the 1024-thread scan chunk
        M = N = 2048
        lens = [2048, 2048, 2048, 2048, 1023, 1024, 1025, 2047, 2048, 1023, 1024, 1025]
    elif name == "b300":       # 600 segments: several per gather thread; every fifth pair stopped earlier
        M, N = 24, 20
        lens = []
        for b in range(300):
            lens += [0, 0] if b % 5 == 2 else [int(torch.randint(1, M + 1, (1,), generator=g)),
                                               int(torch.randint(1, N + 1, (1,), generator=g))]
    elif name == "wrap":       # more token rows than 8 x 4 x SM count: the gather's grid-stride loop wraps
        M = N = 1024
        T = 3 * 32 * sm + 37
        full = T // (M + N)
        lens = [M, N] * full
        rest = T - sum(lens)
        lens += [rest // 2, rest - rest // 2]
        assert sum(lens) == T and T > 32 * sm
    else:                      # "b4096": the ABI's limit on pairs
        M, N = 8, 8
        lens = []
        for b in range(4096):
            lens += [0, 0] if b % 7 == 3 else [int(torch.randint(1, M + 1, (1,), generator=g)),
                                               int(torch.randint(1, N + 1, (1,), generator=g))]
    return M, N, lens


@pytest.mark.parametrize("D,R", [(256, 32), (128, 16)])
@pytest.mark.parametrize("case", ["eval_2048", "b300", "wrap", "b4096"])
def test_compact_at_evaluation_sizes(case, D, R):
    """A pruning step on the given segments (every pair scanned at its full length), then a step with early stopping
    and pruning on the packed result, on random logits (no clearing)."""
    sm = torch.cuda.get_device_properties(0).multi_processor_count
    M, N, lens = _size_case(case, sm)
    B = len(lens) // 2
    layout = "first" if case == "eval_2048" else "pair-major"
    x, theta, ind, off, T = make_state(lens, M, N, D, R, seed=B + D, layout=layout)
    fin = new_fin(B, M, N, D)
    fin_ref = _clone(fin)
    thr = thresholds(9)
    nx, nt, ni, noff, nlen = run_both(x, theta, ind, random_zt(T, B + 1), off, lens, fin, fin_ref, thr[1], -1, 0.5, 1,
                                      B, M, N, tag=f"{case} width")
    # the next layer: early stopping and pruning; a per-pair shift of the confidence logits makes some pairs stop
    g = torch.Generator(device="cpu").manual_seed(B)
    shift = (torch.randint(-4, 7, (B,), generator=g).float()).to(DEV)
    Tn = nx.shape[0]
    zt = random_zt(Tn, B + 2, shift, _sid(noff, nlen, Tn))
    run_both(nx.contiguous(), nt.contiguous(), ni.contiguous(), zt, noff, nlen, fin, fin_ref, thr[2], 0.6, 0.5, 2, B, M,
             N, tag=f"{case} depth+width")
    stopped = int((fin["stop"] == 2).sum())
    assert 0 < stopped < sum(1 for b in range(B) if lens[2 * b] + lens[2 * b + 1] > 0), (case, stopped)
    report(f"adaptive compact {case} D{D}", T=T, B=B, stopped=stopped, kept=sum(nlen))


def _probe_logits(thr, band=64, span=512):
    """fp32 logits around logit(thr) whose CUDA torch.sigmoid lies within `band` fp32 ulps of thr (ties included);
    returns (logits, number of exact ties)."""
    z0 = torch.tensor([math.log(thr / (1 - thr))], dtype=torch.float32)
    zs = (z0.view(torch.int32) + torch.arange(-span, span + 1, dtype=torch.int32)).view(torch.float32)
    zs = zs.to(DEV)
    s = torch.sigmoid(zs)
    t = torch.tensor(thr, dtype=torch.float32, device=DEV)
    ulp = torch.nextafter(t, torch.tensor(2.0, device=DEV)) - t
    sel = (s - t).abs() <= band * ulp
    assert sel.any() and not sel[0] and not sel[-1], "the scanned span does not cover the band"
    return zs[sel], int((s == t).sum())


def _tie_run(z, zother, col, thr, dc, wc, tag):
    """B = len(z) pairs of one token per view (M = N = 1): the probe logit in column `col` of image 0's token, image 1's
    token fixed by zother; returns (kernel fin, kernel kept count per segment) after checking them against the
    restatement."""
    B = z.numel()
    x, theta, ind, off, T = make_state([1, 1] * B, 1, 1, 8, 2, seed=B)
    zt = torch.empty(T, 2, device=DEV)
    zt[0::2] = torch.tensor(zother[0], device=DEV)
    zt[1::2] = torch.tensor(zother[1], device=DEV)
    zt[0::2, col] = z
    fin = new_fin(B, 1, 1, 8)
    fin_ref = _clone(fin)
    run_both(x, theta, ind, zt, off, [1, 1] * B, fin, fin_ref, thr, dc, wc, 4, B, 1, 1, tag=tag)
    return fin


def test_compact_decisions_at_threshold_ties():
    """Every keep / stop decision on logits at and around each threshold equals torch.sigmoid's comparison, element
    for element; the exact ties exist for at least some thresholds, so `>` / `>=` and `<` / `<=` are told apart."""
    ties = {"stop": 0, "exempt": 0, "width": 0}
    n = 0
    for thr in thresholds(9).tolist():
        z, nt = _probe_logits(thr)
        n += z.numel()
        # stop test (lightglue.py:569): image 1's token confident, the probe decides low count 0 or 1 -> ratio 1 or
        # 0.5 against depth_confidence 0.75
        fin = _tie_run(z, [(0.0, 0.0), (20.0, 20.0)], 1, torch.tensor(thr), 0.75, -1, f"stop thr={thr}")
        want = torch.sigmoid(z) >= torch.tensor(thr, device=DEV)
        assert torch.equal(fin["stop"] == 4, want), thr
        # exemption (lightglue.py:556): both tokens unmatchable, image 1's low-confidence, so no pair stops (ratio
        # <= 0.5 < 0.75); the probe's token stays exactly when its confidence <= thr
        fin = _tie_run(z, [(-20.0, 0.0), (-20.0, -20.0)], 1, torch.tensor(thr), 0.75, 0.5, f"exempt thr={thr}")
        assert (fin["stop"] == STOP_SENTINEL).all()
        assert torch.equal(fin["prune0"][:, 0] == 2, torch.sigmoid(z) <= torch.tensor(thr, device=DEV)), thr
        ties["stop"] += nt
        ties["exempt"] += nt
    for wc in (0.99, 0.6):
        wthr = float(torch.tensor(1 - wc, dtype=torch.float32))
        z, nt = _probe_logits(wthr)
        n += z.numel()
        fin = _tie_run(z, [(0.0, 0.0), (20.0, 0.0)], 0, torch.tensor(0.9), -1, wc, f"width wc={wc}")
        assert torch.equal(fin["prune0"][:, 0] == 2, torch.sigmoid(z) > (1 - wc)), wc
        ties["width"] += nt
    report("adaptive compact ties", probes=n, **{f"exact_ties_{k}": v for k, v in ties.items()})
    assert ties["stop"] > 0 and ties["width"] > 0, ties


@pytest.mark.parametrize("c", [1, 7, 8, 333, 1000, 1398])
def test_compact_stop_ratio_ties(c):
    """Low counts c - 1, c, c + 1 against depth_confidence = float32(1 - c / (M + N)): the ratio equals it exactly at
    c, so only c - 1 stops (strict `>`).  The views hold fewer tokens than M / N (pruned earlier), so a ratio taken
    against the current token count would stop other pairs."""
    M, N, n0, n1 = 700, 900, 600, 800
    dc = float(1.0 - torch.tensor(float(c)) / (M + N))
    lows = [c - 1, c, c + 1]
    B = len(lows)
    lens = [n0, n1] * B
    x, theta, ind, off, T = make_state(lens, M, N, 128, 16, seed=c)
    zt = torch.full((T, 2), 20.0, device=DEV)
    for b, lo in enumerate(lows):
        o = off[2 * b]  # the pair's first `lo` tokens (image 0, then image 1) have low confidence
        zt[o:o + min(lo, n0), 1] = -20.0
        zt[off[2 * b + 1]:off[2 * b + 1] + max(0, lo - n0), 1] = -20.0
    fin = new_fin(B, M, N, 128)
    fin_ref = _clone(fin)
    run_both(x, theta, ind, zt, off, lens, fin, fin_ref, thresholds(9)[1], dc, 0.5, 1, B, M, N, tag=f"ratio c={c}")
    assert fin["stop"].tolist() == [1, STOP_SENTINEL, STOP_SENTINEL], (c, dc, fin["stop"].tolist())


@pytest.mark.parametrize("D,R", [(256, 32), (128, 16)])
def test_compact_chained_layers(D, R):
    """L - 1 steps of a 9-layer model in a row, each on the previous step's packed output, then the finishing step
    (zt None): prune counters accumulated over the layers, the final buffer's x / ind / len / stop, the segments
    after every step and the status all equal the chained restatement."""
    L = 9
    B, M, N = 6, 1100, 1040
    lens = [M, N] * B
    x, theta, ind, off, T = make_state(lens, M, N, D, R, seed=D, layout="first")
    ln = list(lens)
    thr = thresholds(L)
    fin = new_fin(B, M, N, D)
    fin_ref = _clone(fin)
    g = torch.Generator(device="cpu").manual_seed(D + 1)
    shift = torch.linspace(-4.0, 2.0, B).to(DEV)   # the pairs' confidence rises layer by layer, at different rates
    rate = torch.linspace(0.2, 1.2, B).to(DEV)
    stops_seen = []
    for i in range(L - 1):
        Tn = x.shape[0]
        sid = _sid(off, ln, Tn)
        zt = (torch.randn(Tn, 2, generator=g) * 3).to(DEV)
        zt[:, 1] += (shift + rate * i)[sid // 2]
        zt[:, 0] += 1.0
        x, theta, ind, off, ln = run_both(x.contiguous(), theta.contiguous(), ind.contiguous(), zt, off, ln, fin,
                                          fin_ref, thr[i], 0.7, 0.6, i, B, M, N, tag=f"layer {i}")
        stops_seen.append(int((fin["stop"] != STOP_SENTINEL).sum()))
        if x.shape[0] == 0:
            break
    if x.shape[0]:
        run_both(x.contiguous(), theta.contiguous(), ind.contiguous(), None, off, ln, fin, fin_ref, thr[L - 1], 0.7,
                 0.6, L - 1, B, M, N, finish=True, tag="finish")
    stops = fin["stop"].tolist()
    assert STOP_SENTINEL not in stops and len(set(stops)) >= 3, stops
    report(f"adaptive compact chained D{D}", stops=str(stops), stopped_by_layer=str(stops_seen))
