"""Micro-benchmark of the LayerNorm kernels at the ImageGPT C5 geometry (P = 65536 rows x 512 channels)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pytorch_generative_b200 import _lib as L

dev = torch.device("cuda:0")
P, C = 65536, 512
x = torch.randn(P, C, device=dev)
gamma, beta = torch.randn(C, device=dev), torch.randn(C, device=dev)
y = torch.empty(P, C, device=dev, dtype=torch.bfloat16)
mean, rstd = torch.empty(P, device=dev), torch.empty(P, device=dev)
dy = torch.randn(P, C, device=dev).bfloat16()
r0, r1 = torch.randn(P, C, device=dev), torch.randn(P, C, device=dev)
dx, dxb = torch.empty(P, C, device=dev), torch.empty(P, C, device=dev, dtype=torch.bfloat16)
dg, db, cs = torch.zeros(C, device=dev), torch.zeros(C, device=dev), torch.zeros(C, device=dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

def timeit(fn, reps=10):
    for _ in range(3): fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]

L.layernorm_fwd(x, gamma, beta, 1e-5, y_bf16=y, mean=mean, rstd=rstd)
n = P * C
t = timeit(lambda: L.layernorm_fwd(x, gamma, beta, 1e-5, y_bf16=y, mean=mean, rstd=rstd))
print(f"ln fwd            : {t*1e3:7.1f} us  {n*6/t/1e6:7.1f} GB/s")
t = timeit(lambda: L.layernorm_bwd(dy, x, gamma, mean, rstd, dres0=r0, dx_f32=dx, dx_bf16=dxb, dgamma=dg, dbeta=db, dx_colsum=cs))
print(f"ln bwd (1 res)    : {t*1e3:7.1f} us  {n*16/t/1e6:7.1f} GB/s")
t = timeit(lambda: L.layernorm_bwd(dy, x, gamma, mean, rstd, dres0=r0, dres1=r1, dx_f32=dx, dx_bf16=dxb, dgamma=dg, dbeta=db, dx_colsum=cs))
print(f"ln bwd (2 res)    : {t*1e3:7.1f} us  {n*20/t/1e6:7.1f} GB/s")
t = timeit(lambda: L.layernorm_bwd(dy, x, gamma, mean, rstd, dres0=r0, dres1=r1, dx_f32=dx, dx_bf16=dxb))
print(f"ln bwd (no colsum): {t*1e3:7.1f} us  {n*20/t/1e6:7.1f} GB/s")

# GatedActivation at the GatedPixelCNN C3 ([P, 256] -> [P, 128], tanh) and PixelSNAIL C4 ([P, 512] -> [P, 256], identity)
# shapes, batch 128: algorithmic bytes fwd = 3 * P * C * sizeof, bwd = 5 * P * C * sizeof
for name, Cg, act in (("gated tanh  C3", 128, L.ACT_TANH), ("gated ident C4", 256, L.ACT_NONE)):
    Pg = 128 * 32 * 32
    xg = torch.randn(Pg, 2 * Cg, device=dev).bfloat16()
    yg = torch.empty(Pg, Cg, device=dev, dtype=torch.bfloat16)
    dyg = torch.randn(Pg, Cg, device=dev).bfloat16()
    dxg = torch.empty_like(xg)
    t = timeit(lambda: L.gated_act_fwd(xg, yg, act))
    print(f"{name} fwd (bf16): {t*1e3:7.1f} us  {Pg*Cg*3*2/t/1e6:7.1f} GB/s")
    t = timeit(lambda: L.gated_act_bwd(xg, dyg, dxg, act))
    print(f"{name} bwd (bf16): {t*1e3:7.1f} us  {Pg*Cg*5*2/t/1e6:7.1f} GB/s")
