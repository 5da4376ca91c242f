"""Micro-benchmark of the wgmma attention kernels, by default at the ImageGPT C5 geometry (N=64, S=1024, 8 heads x 64).

    python tools/bench_attn.py --heads 4 --dim 128     the same FLOPs in 128-wide heads
Heads narrower than a kernel slot are timed in their zero-padded slot; FLOPs count the slot width.  After the forward
and the whole backward (CUDA events), the backward's delta, dK / dV and dQ kernels are listed one by one."""
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

# the backward's three kernels one by one: device durations from a torch.profiler pass of its own (tracing slows the
# host, not the kernels), median over the launches, L2 flushed before each
REPS = 8
with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
    for _ in range(REPS):
        flush.zero_()
        bwd()
    torch.cuda.synchronize()
durs = {}
for ev in prof.events():
    if ev.device_type == torch.autograd.DeviceType.CUDA:
        durs.setdefault(ev.name, []).append(ev.device_time)
# MMAs per (query tile, key tile) pair of 2 * 128 * 128 * D flops each: dK / dV runs S^T, dP^T, dV, dK; dQ runs S, dP, dQ
for part, key, mmas in (("delta", "attn_delta", 0), ("dK/dV", "attn_bwd_tc_kernel", 4), ("dQ", "attn_dq_tc_kernel", 3)):
    for kname, us in durs.items():
        if key in kname:
            t = sorted(us)[len(us) // 2]
            rate = f"  {2*mmas*D*pairs/t/1e6:7.1f} TFLOP/s" if mmas else ""
            print(f"  {part:6s} {t:8.1f} us{rate}")
