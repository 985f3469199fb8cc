"""GPU: GlueStick's BatchNorm + ReLU kernels (ops.batchnorm_relu) and their cross-rank statistics (nn.SyncBatchNorm,
as glue-factory's distributed trainer converts every BatchNorm: train.py:337-339).

  1. the kernels against fp64 torch (F.batch_norm + relu, autograd) per element, bf16 and fp32, at the channel counts of
     the GlueStick MLPs and token counts up to the reference's per-GPU batch (20 pairs x 3,072 nodes);
  2. data-parallel ranks emulated in one process through the substitutable exchange: every block of rows gets the rows
     of the whole-batch call, and bitwise-identical statistics;
  3. GlueStick at world size 2 (the reference's convert_sync_batchnorm + DDP route, and MatcherTrainer(sync_batchnorm))
     against one process on the whole batch;
  4. eval mode: running statistics, no collective.
"""
import copy
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp
import torch.nn.functional as F
from torch import nn

from gluefactory_b200 import ops, synthetic
from tests.util import rel_err, report

pytestmark = pytest.mark.gpu
DEV = "cuda"
EPS_F32 = 2.0 ** -24  # unit round-off of the fp32 arithmetic inside the kernels
ULP_BF16 = 2.0 ** -8  # relative spacing of bf16 outputs (one rounding: at most half of it)


def _inputs(T, C, dtype, seed):
    """x with a channel offset by 100x its std (1) and a constant channel (2); gamma with both signs."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(T, C, generator=g, device=DEV) * 1.5 + 0.3
    x[:, 1] = torch.randn(T, generator=g, device=DEV) * 0.5 + 50.0
    x[:, 2] = 0.37
    w = 1.0 + 0.5 * torch.randn(C, generator=g, device=DEV)
    b = 0.3 * torch.randn(C, generator=g, device=DEV)
    dy = torch.randn(T, C, generator=g, device=DEV)
    return x.to(dtype), w, b, dy.to(dtype)


def _bn(C, w, b):
    bn = nn.BatchNorm1d(C).to(DEV)
    with torch.no_grad():
        bn.weight.copy_(w)
        bn.bias.copy_(b)
    return bn


def _ours(x, bn, dy, exchange=None):
    xg = x.clone().requires_grad_(True)
    y = ops.batchnorm_relu(xg, bn, exchange)
    y.backward(dy)
    return y.detach(), xg.grad, bn.weight.grad.clone(), bn.bias.grad.clone()


def _reference(x, w, b, dy, rm, rv, training=True):
    """fp64 autograd of relu(F.batch_norm); rm / rv fp64 running buffers, updated in place like the module's."""
    xr = x.double().requires_grad_(True)
    wr = w.double().requires_grad_(True)
    br = b.double().requires_grad_(True)
    z = F.batch_norm(xr, rm, rv, wr, br, training=training, momentum=0.1, eps=1e-5)
    z.retain_grad()
    y = torch.relu(z)
    y.backward(dy.double())
    if training:
        mu, var = xr.detach().mean(0), xr.detach().var(0, unbiased=False)
    else:
        mu, var = rm, rv
    rs = (var + 1e-5).rsqrt()
    return dict(y=y.detach(), z=z.detach(), dx=xr.grad, dw=wr.grad, db=br.grad, mu=mu, rs=rs,
                xh=(xr.detach() - mu) * rs)


def _check_against_reference(x, w, b, dy, y, dx, dw, db, r, training=True):
    """Per-element bounds, each the error the kernels' arithmetic allows for (NaN fails every comparison):
      * y: the normalised input costs a few fp32 roundings of |xhat| and of |mean| rstd (the mean is kept in fp32), times
        |gamma|, plus |beta|: 64 EPS_F32 of that scale; a bf16 output adds one rounding (ULP_BF16 |y|).
      * dx: the same 64 EPS_F32 of gamma rstd (|dy| + |mean dy'| + |xhat| |mean dy' xhat|) (plus the xhat error carried
        by the last term), plus one bf16 rounding.  Elements whose pre-activation lies within the y bound of 0 may take
        the other side of the ReLU: their dx is not checked, and what they can move in the channel means is added.
      * dgamma / dbeta: 64 EPS_F32 of the sum of the terms' magnitudes, plus those elements' terms."""
    T = x.shape[0]
    bf16 = x.dtype == torch.bfloat16
    wd, bd = w.double(), b.double()
    xh, z, rs, mu = r["xh"], r["z"], r["rs"], r["mu"]
    xh_scale = xh.abs() + mu.abs() * rs + 1.0
    y_bound = 64 * EPS_F32 * (wd.abs() * xh_scale + bd.abs()) + (ULP_BF16 * r["y"].abs() if bf16 else 0.0)
    yd = y.double()
    assert torch.isfinite(yd).all()
    assert bool(((yd - r["y"]).abs() <= y_bound).all()), ((yd - r["y"]).abs() - y_bound).max().item()

    amb = z.abs() <= y_bound
    assert amb.double().mean().item() < 1e-3
    dyd = dy.double()
    dyp = dyd * (z > 0)
    m1 = dyp.mean(0).abs() if training else torch.zeros_like(mu)
    m2 = (dyp * xh).mean(0).abs() if training else torch.zeros_like(mu)
    a1 = (dyd.abs() * amb).sum(0) / T
    a2 = (dyd.abs() * xh.abs() * amb).sum(0) / T
    gr = wd.abs() * rs
    # the last two terms: the xhat error inside xhat mean(dy' xhat) and inside the kernel's own sum of dy' xhat
    dx_scale = gr * (dyd.abs() + m1 + xh.abs() * m2 + xh_scale * m2 +
                     (xh.abs() * (dyp.abs() * xh_scale).mean(0) if training else 0.0))
    dx_bound = 64 * EPS_F32 * dx_scale + (gr * (a1 + xh.abs() * a2) if training else 0.0) + \
        (ULP_BF16 * r["dx"].abs() if bf16 else 0.0)
    dxd = dx.double()
    assert torch.isfinite(dxd).all()
    ok = ((dxd - r["dx"]).abs() <= dx_bound) | amb
    assert bool(ok.all()), ((dxd - r["dx"]).abs() - dx_bound)[~amb].max().item()

    dw_bound = 64 * EPS_F32 * (dyp.abs() * xh_scale).sum(0) + (dyd.abs() * xh.abs() * amb).sum(0)
    db_bound = 64 * EPS_F32 * dyp.abs().sum(0) + (dyd.abs() * amb).sum(0)
    assert bool(((dw.double() - r["dw"]).abs() <= dw_bound).all())
    assert bool(((db.double() - r["db"]).abs() <= db_bound).all())
    report(f"bn_relu {x.dtype} T={T} C={x.shape[1]} training={training}",
           y=((yd - r["y"]).abs() / y_bound).max().item(), dx=((dxd - r["dx"]).abs() / dx_bound)[~amb].max().item(),
           ambiguous=int(amb.sum()))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("C", [32, 64, 128, 256, 512])
@pytest.mark.parametrize("T", [2, 7, 333, 8192, 61440])
def test_bn_relu_kernels_against_fp64(T, C, dtype):
    x, w, b, dy = _inputs(T, C, dtype, seed=T * 1000 + C)
    x2, _, _, _ = _inputs(T, C, dtype, seed=T * 1000 + C + 1)
    bn = _bn(C, w, b)
    rm = torch.zeros(C, device=DEV, dtype=torch.float64)
    rv = torch.ones(C, device=DEV, dtype=torch.float64)
    y, dx, dw, db = _ours(x, bn, dy)
    r = _reference(x, w, b, dy, rm, rv)
    _check_against_reference(x, w, b, dy, y, dx, dw, db, r)
    # running statistics after a second call: momentum 0.1, variance unbiased by the count
    bn.weight.grad = bn.bias.grad = None
    _ours(x2, bn, dy)
    _reference(x2, w, b, dy, rm, rv)
    assert int(bn.num_batches_tracked) == 2
    scale = r["mu"].abs() + 1.0
    assert bool(((bn.running_mean.double() - rm).abs() <= 64 * EPS_F32 * scale).all())
    assert bool(((bn.running_var.double() - rv).abs() <= 64 * EPS_F32 * (rv.abs() + 1.0)).all())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
def test_bn_relu_eval_mode_uses_running_statistics(dtype):
    T, C = 333, 256
    x, w, b, dy = _inputs(T, C, dtype, seed=7)
    bn = _bn(C, w, b)
    g = torch.Generator(device=DEV).manual_seed(8)
    with torch.no_grad():
        bn.running_mean.copy_(torch.randn(C, generator=g, device=DEV))
        bn.running_var.copy_(torch.rand(C, generator=g, device=DEV) + 0.5)
    rm, rv = bn.running_mean.double().clone(), bn.running_var.double().clone()
    bn.eval()
    calls = []
    y, dx, dw, db = _ours(x, bn, dy, exchange=calls.append)
    assert not calls  # eval mode never exchanges
    assert torch.equal(bn.running_mean.double(), rm) and torch.equal(bn.running_var.double(), rv)
    assert int(bn.num_batches_tracked) == 0
    r = _reference(x, w, b, dy, rm.clone(), rv.clone(), training=False)
    _check_against_reference(x, w, b, dy, y, dx, dw, db, r, training=False)


class _EmulatedRanks:
    """n data-parallel ranks in one process.  Rank r's exchange records its local fp64 vector and replaces it by the sum
    over all ranks in rank order, known from the previous round: the caller replays the same calls in rounds (forward
    totals after round 1, backward totals after round 2), so round 3 computes what n real ranks would."""

    def __init__(self, n):
        self.n, self.local, self.total = n, {}, {}

    def exchange(self, rank):
        def ex(t):
            key = t.numel()  # forward [2C + 1] or backward [2C]
            prev = self.local.get((key, rank))
            if prev is not None and key in self.total:  # the same inputs as last round: bitwise the same local sums
                assert torch.equal(prev, t), (key, rank)
            self.local[(key, rank)] = t.clone()
            if key in self.total:
                t.copy_(self.total[key])

        return ex

    def close_round(self):
        for key in {k for k, _ in self.local}:
            tot = self.local[(key, 0)].clone()
            for r in range(1, self.n):
                tot += self.local[(key, r)]
            self.total[key] = tot


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["fp32", "bf16"])
@pytest.mark.parametrize("sizes", [(3000, 5192), (1000, 4000, 3192)], ids=["2ranks", "3ranks"])
def test_bn_relu_emulated_ranks_equal_whole_batch(sizes, dtype):
    T, C = sum(sizes), 128
    x, w, b, dy = _inputs(T, C, dtype, seed=11)
    bounds = [0]
    for s in sizes:
        bounds.append(bounds[-1] + s)
    rows = [slice(lo, hi) for lo, hi in zip(bounds[:-1], bounds[1:])]
    base = _bn(C, w, b)

    bns = [copy.deepcopy(base) for _ in range(2)]
    whole = [_ours(x, bn, dy) for bn in bns]
    for a, c in zip(*whole):  # two identical calls are bit-equal
        assert torch.equal(a, c)
    assert torch.equal(bns[0].running_mean, bns[1].running_mean) and torch.equal(bns[0].running_var, bns[1].running_var)
    bn_whole, whole_out = bns[0], whole[0]

    ranks = _EmulatedRanks(len(sizes))
    for rnd in range(3):
        mods = [copy.deepcopy(base) for _ in sizes]
        outs = []
        for r, (sl, bn) in enumerate(zip(rows, mods)):
            if rnd == 0:  # forward statistics only
                ops.batchnorm_relu(x[sl].contiguous(), bn, ranks.exchange(r))
            else:
                outs.append(_ours(x[sl].contiguous(), bn, dy[sl].contiguous(), ranks.exchange(r)))
        ranks.close_round()

    y_w, dx_w, dw_w, db_w = whole_out
    tol = ULP_BF16 if dtype == torch.bfloat16 else 1e-5
    dy_max, dx_max = y_w.abs().max().item(), dx_w.abs().max().item()
    for (y, dx, _, _), sl, bn in zip(outs, rows, mods):
        dyv, dxv = (y.double() - y_w[sl].double()).abs().max().item(), (dx.double() - dx_w[sl].double()).abs().max().item()
        report(f"bn_relu emulated {len(sizes)} ranks {dtype}", y=dyv, dx=dxv)
        assert dyv <= tol * dy_max and dxv <= tol * dx_max, (dyv, dxv)
        # every rank holds bitwise the same statistics, equal to the whole batch's up to the fp64 summation order
        assert torch.equal(bn.running_mean, mods[0].running_mean) and torch.equal(bn.running_var, mods[0].running_var)
        torch.testing.assert_close(bn.running_mean, bn_whole.running_mean, rtol=1e-6, atol=1e-7)
        torch.testing.assert_close(bn.running_var, bn_whole.running_var, rtol=1e-6, atol=1e-7)
    # the gradient all-reduce of the affine parameters: the sum of the ranks' local dgamma / dbeta
    dw_sum = sum(o[2].double() for o in outs)
    db_sum = sum(o[3].double() for o in outs)
    assert rel_err(dw_sum, dw_w) < 1e-5 and rel_err(db_sum, db_w) < 1e-5


# --------------------------------------------------------------------------------------------------- world size 2
GS_CONF = {"GNN_layers": ["self", "cross"]}
N_BN_CALLS = 22  # per forward of GS_CONF: 4 + 4 encoder BatchNorms, 2 GNN layers, 1 line layer; each once per image


def _gs_model(dev):
    from gluefactory_b200.matchers.gluestick import GlueStick

    model = GlueStick(dict(GS_CONF, precision="bf16"))
    model.load_state_dict(synthetic.make_gluestick_weights(model.state_dict(), seed=62), strict=True)
    return model.to(dev).train()


def _rows(tree, sl):
    return {k: (_rows(v, sl) if isinstance(v, dict) else v[sl] if torch.is_tensor(v) else v) for k, v in tree.items()}


def _bn_state(model):
    return {k: v.clone() for k, v in model.state_dict().items() if "running_" in k or "num_batches_tracked" in k}


def _same_across_ranks(t):
    m = t.double().clone()
    dist.all_reduce(m, op=dist.ReduceOp.MAX)
    return bool(torch.equal(m, t.double()))


def _compare(tag, pred, grads, state, ref, sl):
    """-> list of (what, ok, value) for one route against the single-process run `ref` on the whole batch."""
    res = []
    la = rel_err(pred["log_assignment"], ref["pred"]["log_assignment"][sl])
    res.append((f"{tag} log_assignment rel_err", la < 1e-3, la))
    for k in ("matches0", "matches1", "line_matches0", "line_matches1"):
        diff = (pred[k] != ref["pred"][k][sl]).double().mean().item()
        res.append((f"{tag} {k} disagreement", diff <= 0.01, diff))
    g_all = torch.cat([g.reshape(-1) for g in ref["grads"].values()]).norm().item()
    worst = max((grads[n] - g).norm().item() / (5e-3 * g.norm().item() + 1e-5 * g_all) for n, g in ref["grads"].items())
    res.append((f"{tag} averaged gradients (error / bound)", worst <= 1.0, worst))
    for k, v in ref["state"].items():
        if "num_batches_tracked" in k:
            res.append((f"{tag} {k}", int(state[k]) == int(v), int(state[k])))
        else:
            err = ((state[k] - v).abs() / (1e-3 * v.abs() + 1e-5)).max().item()
            res.append((f"{tag} {k} (error / bound)", err <= 1.0, err))
        res.append((f"{tag} {k} identical across ranks", _same_across_ranks(state[k]), 0))
    return res


def _gs_worker(rank, world, port, backend, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dev = torch.device("cuda", rank if torch.cuda.device_count() >= world else 0)
    torch.cuda.set_device(dev)
    dist.init_process_group(backend, rank=rank, world_size=world)
    calls = [0]
    all_reduce = dist.all_reduce

    def counting_all_reduce(*a, **k):
        calls[0] += 1
        return all_reduce(*a, **k)

    dist.all_reduce = counting_all_reduce
    res = []
    try:
        from gluefactory_b200.trainer import MatcherTrainer

        B = 4
        full = synthetic.to_device(synthetic.make_gluestick_batch(B, 192, 24, 61), dev)
        sl = slice(rank * B // world, (rank + 1) * B // world)
        mine = _rows(full, sl)
        # one process, the whole batch, plain BatchNorm1d
        m_ref = _gs_model(dev)
        p = m_ref(full)
        losses, _ = m_ref.loss(p, full)
        losses["total"].mean().backward()
        ref = {"pred": p, "grads": {n: q.grad.clone() for n, q in m_ref.named_parameters()}, "state": _bn_state(m_ref)}

        # (a) the reference's route: convert_sync_batchnorm, then DDP, loss_fn bound before the wrap
        m_a = nn.SyncBatchNorm.convert_sync_batchnorm(_gs_model(dev))
        loss_fn = m_a.loss
        ddp = torch.nn.parallel.DistributedDataParallel(m_a, device_ids=[dev.index] if backend == "nccl" else None)
        calls[0] = 0
        pred = ddp(mine)
        res.append(("(a) collectives in forward", calls[0] == N_BN_CALLS, calls[0]))
        losses, _ = loss_fn(pred, mine)
        calls[0] = 0
        losses["total"].mean().backward()
        res.append(("(a) collectives in backward", calls[0] == N_BN_CALLS, calls[0]))
        res += _compare("(a)", pred, {n: q.grad for n, q in m_a.named_parameters()}, _bn_state(m_a), ref, sl)

        # (b) the flat-buffer trainer with sync_batchnorm (lr = 0: the parameters stay put)
        tr = MatcherTrainer(_gs_model(dev), lr=0.0, sync_batchnorm=True)
        n_sync = sum(isinstance(m, nn.SyncBatchNorm) for m in tr.model.modules())
        res.append(("(b) SyncBatchNorm modules", n_sync == 11, n_sync))
        captured = {}
        fwd = tr.model.forward

        def keep_pred(data):
            captured["pred"] = fwd(data)
            return captured["pred"]

        tr.model.forward = keep_pred
        calls[0] = 0
        tr.step(mine)
        res.append(("(b) collectives per step (BatchNorm forward + backward + the gradient exchange)",
                    calls[0] == 2 * N_BN_CALLS + 1, calls[0]))
        del tr.model.forward
        res += _compare("(b)", captured["pred"], {n: q.grad / world for n, q in tr.model.named_parameters()},
                        _bn_state(tr.model), ref, sl)

        # eval mode: the running statistics, no collective
        tr.model.eval()
        m_ref.eval()
        with torch.no_grad():
            calls[0] = 0
            pe = tr.model(mine)
            res.append(("eval collectives", calls[0] == 0, calls[0]))
            pr = m_ref(mine)
        e = rel_err(pe["log_assignment"], pr["log_assignment"])
        res.append(("eval log_assignment vs the single-process model in eval mode", e < 1e-3, e))
        out.put((rank, res, None))
    except Exception as ex:  # noqa: BLE001 -- reported to the parent process
        import traceback

        out.put((rank, res, traceback.format_exc()))
    finally:
        dist.all_reduce = all_reduce
        dist.destroy_process_group()


def test_gluestick_sync_batchnorm_world2_matches_whole_batch():
    """world size 2: NCCL when the box has two GPUs, else both ranks share cuda:0 over gloo (the wiring is the same)."""
    world = 2
    backend = "nccl" if torch.cuda.device_count() >= world else "gloo"
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        port = s.getsockname()[1]
    ctx = mp.get_context("spawn")
    out = ctx.Queue()
    procs = [ctx.Process(target=_gs_worker, args=(r, world, port, backend, out)) for r in range(world)]
    for p in procs:
        p.start()
    got = [out.get(timeout=600) for _ in range(world)]
    for p in procs:
        p.join(60)
        assert p.exitcode == 0
    for rank, res, tb in got:
        assert tb is None, f"rank {rank}:\n{tb}"
        for what, ok, val in res:
            report(f"sync_bn world2 {backend} rank {rank} {what}", value=float(val))
        bad = [(what, val) for what, ok, val in res if not ok]
        assert not bad, (rank, bad)
