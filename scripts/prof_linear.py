"""Event timing of the layer's GEMM shapes on the library's persistent wgmma kernel (lgb200_linear / split-K wgrad)
at the bench token count (T = 131072 = 32 pairs x 2 images x 2048), with the HBM bytes each one has to move."""
import os, sys, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from gluefactory_b200 import ops
T = int(os.environ.get("PT", "131072"))
dev = "cuda"
def t(fn, n=20):
    for _ in range(3): fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(n): fn()
    e.record(); torch.cuda.synchronize(); return s.elapsed_time(e) / n * 1e3
g = torch.Generator(device=dev).manual_seed(0)
rnd = lambda *s: torch.randn(*s, device=dev, generator=g).to(torch.bfloat16)
print(f"T={T}")
tot = 0.0
for name, K, N in [("qkv", 256, 768), ("proj 256", 256, 256), ("ffn.0", 512, 512), ("ffn.3", 512, 256)]:
    x, w, b = rnd(T, K), rnd(N, K), torch.randn(N, device=dev)
    dy = rnd(T, N)
    acc = torch.zeros(T, K, device=dev)
    us_f = t(lambda: ops.linear(x, w, b))
    us_d = t(lambda: ops.linear(dy, w, w_is_kn=True))
    us_a = t(lambda: ops.linear(dy, w, out=acc, w_is_kn=True, accumulate=True))
    us_w = t(lambda: ops.wgrad_bf16(dy, x))
    mb_f = (T * K + T * N) * 2 / 1e6
    mb_a = (T * N * 2 + T * K * 8) / 1e6
    print(f"{name:9s} fwd {us_f:6.1f} us ({mb_f/us_f*1e-0:5.2f} TB/s... {mb_f:.0f} MB) | dgrad {us_d:6.1f} us | dgrad+acc {us_a:6.1f} us ({mb_a/us_a:5.2f} TB/s) | wgrad {us_w:6.1f} us ({mb_f/us_w:5.2f} TB/s)")
    tot += us_f + us_d + us_w
print(f"sum fwd+dgrad+wgrad over the four shapes: {tot:.0f} us")
