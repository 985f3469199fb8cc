"""Event timing of the wgmma GEMM at the assignment-head shapes (32 pairs, N=M=2048, d=256)."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gluefactory_b200 import ops
B, N, D = int(os.environ.get("PB", "32")), 2048, 256
g = torch.Generator(device="cuda").manual_seed(0)
md0 = torch.randn(B, N, D, device="cuda", generator=g).to(torch.bfloat16)
md1 = torch.randn(B, N, D, device="cuda", generator=g).to(torch.bfloat16)
dsim = torch.randn(B, N, N, device="cuda", generator=g).to(torch.bfloat16)
def t(fn, n=10):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    fn(); torch.cuda.synchronize(); s.record()
    for _ in range(n): fn()
    e.record(); torch.cuda.synchronize(); return s.elapsed_time(e) / n * 1e3
t1 = t(lambda: ops.gemm_bf16(md0, md1, alpha=0.0625))
t2 = t(lambda: ops.gemm_bf16(dsim, md1, a_mn_major=False, b_mn_major=True, out_dtype=torch.bfloat16))
t3 = t(lambda: ops.gemm_bf16(dsim, md0, a_mn_major=True, b_mn_major=True, out_dtype=torch.bfloat16))
fl = 2 * B * N * N * D
print(f"sim {t1:.1f} us ({fl/t1/1e6:.0f} TF/s, {B*N*N*4/t1/1e6:.2f} TB/s out) | dmd0 {t2:.1f} us ({fl/t2/1e6:.0f} TF/s) | dmd1 {t3:.1f} us ({fl/t3/1e6:.0f} TF/s)")
ref = torch.bmm(md0[:2].float(), md1[:2].float().transpose(1, 2)) * 0.0625
print("max err", (ops.gemm_bf16(md0[:2].contiguous(), md1[:2].contiguous(), alpha=0.0625) - ref).abs().max().item())
T = B * 2 * N
dy = torch.randn(T, 512, device="cuda", generator=g).to(torch.bfloat16)
a = torch.randn(T, 512, device="cuda", generator=g).to(torch.bfloat16)
for (M_, N_) in ((256, 256), (512, 256), (256, 512), (768, 256)):
    d_, a_ = dy[:, :M_].contiguous(), a[:, :N_].contiguous()
    tw = t(lambda: ops.wgrad_bf16(d_, a_))
    tt = t(lambda: torch.mm(d_.t(), a_, out_dtype=torch.float32))
    print(f"wgrad [{M_}x{N_}] over T={T}: split-K {tw:.1f} us ({T*(M_+N_)*2/tw/1e6:.2f} TB/s) | cuBLAS {tt:.1f} us")
