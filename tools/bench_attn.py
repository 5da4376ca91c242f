"""Micro-benchmark of the wgmma attention kernels, by default at the ImageGPT C5 geometry (N=64, S=1024, 8 heads x 64).

    python tools/bench_attn.py --heads 4 --dim 128     the same FLOPs in 128-wide heads
Heads narrower than a kernel slot are timed in their zero-padded slot; FLOPs count the slot width."""
import argparse, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pytorch_generative_b200 import _lib as L, ops

ap = argparse.ArgumentParser()
ap.add_argument("--heads", type=int, default=8)
ap.add_argument("--dim", type=int, default=64, help="channels per head (q/k and v)")
args = ap.parse_args()
dev = torch.device("cuda:0")
N, S, H = int(os.environ.get("PG_N", 64)), 1024, args.heads
D = ops.head_slots(args.dim, args.dim)[0]
print(f"{torch.cuda.get_device_name(dev)}; N={N} S={S} heads={H} x {args.dim} (slot {D})")
P = N * S
qkv = torch.randn(P, 3 * H * D, device=dev).bfloat16()
q, k, v = qkv[:, :H * D], qkv[:, H * D:2 * H * D], qkv[:, 2 * H * D:]
o = torch.empty(P, H * D, device=dev, dtype=torch.bfloat16)
lse = torch.empty(N, H, S, device=dev)
do = torch.randn(P, H * D, device=dev).bfloat16()
dqkv = torch.empty_like(qkv)
delta = torch.empty(N, H, S, device=dev)
flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

def timeit(fn, reps=8):
    for _ in range(3): fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]

pairs = N * H * (S // 128) * (S // 128 + 1) // 2 * 128 * 128
fwd = lambda: L.causal_attn_fwd(q, k, v, o, lse, N, S, H, D, D, False, dk_true=args.dim)
def bwd():
    L.causal_attn_bwd(q, k, v, o, do, lse, delta, None, dqkv[:, :H * D], dqkv[:, H * D:2 * H * D], dqkv[:, 2 * H * D:], N, S, H, D, D,
                      False, dk_true=args.dim)
t = timeit(fwd); print(f"attn fwd: {t*1e3:8.1f} us  {4*D*pairs/t/1e9:7.1f} TFLOP/s (tile-granular causal flops)")
t = timeit(bwd); print(f"attn bwd: {t*1e3:8.1f} us  {10*D*pairs/t/1e9:7.1f} TFLOP/s (incl. delta and the dQ kernel)")
