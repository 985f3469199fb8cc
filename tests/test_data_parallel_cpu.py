"""CPU, world_size 2 over gloo: the flat-buffer gradient exchange (the path's one collective).
The optimiser kernel itself is CUDA-only; here we check the host logic: parameters are views of the flat
buffer, the gradients autograd hands over are packed into the flat gradient buffer, and one all_reduce
leaves every rank with the sum of the per-rank gradients."""
import os

import torch
import torch.distributed as dist
import torch.multiprocessing as mp


def _worker(rank, world, port, out):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gluefactory_b200.trainer import FlatParams, MatcherTrainer

    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.LayerNorm(16), torch.nn.Linear(16, 3))
    net.loss = None
    tr = MatcherTrainer.__new__(MatcherTrainer)
    tr.fp = FlatParams(net)
    tr.world, tr.group = world, None
    x = torch.full((4, 8), float(rank + 1))
    tr.fp.zero_grad()
    net(x).sum().backward()
    assert all(p.grad is not None and p.grad.data_ptr() != tr.fp.grad.data_ptr() + off * 4
               for p, off in zip(tr.fp.params, tr.fp.offsets))  # handed over by reference, not accumulated
    tr.fp.gather_grads()
    local = tr.fp.grad.clone()
    # gradients were packed into the flat buffer and the .grad views re-attached
    for p, off in zip(tr.fp.params, tr.fp.offsets):
        assert p.grad.data_ptr() == tr.fp.grad.data_ptr() + off * 4
        assert torch.equal(p.grad.reshape(-1), tr.fp.grad[off:off + p.numel()])
    tr.exchange_gradients()
    gathered = [torch.zeros_like(local) for _ in range(world)]
    dist.all_gather(gathered, local)
    assert torch.allclose(tr.fp.grad, sum(gathered))
    # parameter writes through the flat buffer are visible in the module
    tr.fp.flat.add_(1.0)
    assert torch.equal(net[0].weight.reshape(-1), tr.fp.flat[: net[0].weight.numel()])
    out.put((rank, float(tr.fp.grad.abs().sum())))
    dist.destroy_process_group()


def test_flat_gradient_allreduce_world2():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    os.environ["PYTHONPATH"] = root + os.pathsep + os.environ.get("PYTHONPATH", "")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29500 + os.getpid() % 2000
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    res = dict(q.get() for _ in range(2))
    assert abs(res[0] - res[1]) < 1e-6 and res[0] > 0


def _direct_worker(rank, world, port, out):
    """Direct parameter groups (their backward writes the flat gradient buffer in place) keep their .grad views through
    zero_grad, and MatcherTrainer.exchange_gradients is ONE sum-all-reduce of the whole buffer, loss slot included
    (host logic over gloo)."""
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    from gluefactory_b200.trainer import FlatParams, MatcherTrainer

    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.Linear(16, 16), torch.nn.Linear(16, 16), torch.nn.Linear(16, 3))
    tr = MatcherTrainer.__new__(MatcherTrainer)
    tr.fp = fp = FlatParams(net)
    tr.world, tr.group = world, None
    fp.enable_direct([list(net[1].parameters()), list(net[2].parameters())])
    assert net[1].weight.grad.data_ptr() == fp.direct_views(0)[0].data_ptr()
    fp.zero_grad()
    assert all(p.grad is not None for i in (1, 2) for p in net[i].parameters())  # direct slots stay attached
    assert all(p.grad is None for i in (0, 3) for p in net[i].parameters())
    g = torch.Generator().manual_seed(100 + rank)
    fp.grad_ext.copy_(torch.randn(fp.grad_ext.shape, generator=g))
    want = fp.grad_ext.clone()
    dist.all_reduce(want)
    tr.exchange_gradients()
    assert torch.equal(fp.grad_ext, want)
    out.put((rank, float(want.abs().sum())))
    dist.destroy_process_group()


def test_direct_groups_and_gradient_exchange_world2():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    os.environ["PYTHONPATH"] = root + os.pathsep + os.environ.get("PYTHONPATH", "")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31500 + os.getpid() % 2000
    procs = [ctx.Process(target=_direct_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    for p in procs:
        p.join(120)
        assert p.exitcode == 0
    res = dict(q.get() for _ in range(2))
    assert abs(res[0] - res[1]) < 1e-6 and res[0] > 0
