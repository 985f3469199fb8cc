"""Race hunt: repeated launches of the attention kernels on the same inputs must give bit-identical out / lse / dQ / dK /
dV, for self (shift 0) and cross (shift 2) launches."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gluefactory_b200 import ops
B, N, H = 4, 2048, 4
for shift in (0, 2):
    g = torch.Generator().manual_seed(5 + shift)
    mk = lambda s: (torch.randn(B, N, H, 64, generator=g) * s).to(torch.bfloat16).cuda()
    q, k, v, go = mk(1.5), mk(1.5), mk(1.0), mk(1.0)
    q0, k0, v0, go0 = q.clone(), k.clone(), v.clone(), go.clone()
    out0, lse0 = ops.attn_fwd(q, k, v, shift, 0.125)
    dq0, dk0, dv0 = ops.attn_bwd(q, k, v, out0, lse0, go, shift, 0.125)
    torch.cuda.synchronize()
    bad = {"out": 0, "lse": 0, "dq": 0, "dk": 0, "dv": 0, "inputs": 0}
    for it in range(40):
        out, lse = ops.attn_fwd(q, k, v, shift, 0.125)
        dq, dk, dv = ops.attn_bwd(q, k, v, out0, lse0, go, shift, 0.125)
        torch.cuda.synchronize()
        bad["out"] += int(not torch.equal(out, out0)); bad["lse"] += int(not torch.equal(lse, lse0))
        bad["dq"] += int(not torch.equal(dq, dq0))
        bad["dk"] += int(not torch.equal(dk, dk0)); bad["dv"] += int(not torch.equal(dv, dv0))
        bad["inputs"] += int(not (torch.equal(q, q0) and torch.equal(k, k0) and torch.equal(v, v0) and torch.equal(go, go0)))
    # reference check of the first result
    qr, kr, vr = (t.double().permute(0, 2, 1, 3) for t in (q, k, v))
    idx = (torch.arange(B, device="cuda") + shift) % B
    s = qr @ kr[idx].transpose(-1, -2) / 8.0
    ref = (torch.softmax(s, -1) @ vr[idx]).permute(0, 2, 1, 3)
    err = ((out0.double() - ref).norm() / ref.norm()).item()
    blk = ((out0.double() - ref).reshape(B, N // 128, 128, -1).norm(dim=(2, 3)) / ref.reshape(B, N // 128, 128, -1).norm(dim=(2, 3)))
    print(f"shift {shift}: mismatching repeats {bad}; out rel err {err:.4e}; worst blocks {blk.flatten().topk(3).values.tolist()} at {blk.flatten().topk(3).indices.tolist()}")
