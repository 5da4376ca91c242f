"""Micro-benchmark of the linear-attention numerator, pg_linear_attn_fwd and pg_linear_attn_fwd + _bwd, timed with CUDA
events after a warm-up (median of --windows windows of --iters calls each).

Rates are algorithmic: per position the sequential form makes one d x dv state update and one d x dv product, so the
forward counts 4 B L d dv FLOPs and the backward (dq, dv, dk: three such scans) 12 B L d dv.  They are compared with
67 TFLOP/s, the dense FP32 figure of NVIDIA's H100 SXM data sheet (a 700 W card), not a rate measured here.  The shapes
(B, L, d, dv) cover the domain of the earlier one-CTA-per-head kernel (d <= 64, dv <= 128), wide heads, and one image
with a long sequence; a shape a build does not support is reported as such.

    python tools/bench_linear_attn.py [--iters 20] [--windows 5]"""
import argparse, os, subprocess, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pytorch_generative_b200 import _lib as L

SHAPES = [(8, 784, 16, 32), (16, 1024, 64, 128), (64, 1024, 64, 64),
          (16, 1024, 128, 128), (16, 4096, 256, 256), (2, 4096, 512, 512),
          (1, 16384, 64, 64)]
FP32_DATASHEET = 67e12

ap = argparse.ArgumentParser()
ap.add_argument("--iters", type=int, default=20)
ap.add_argument("--windows", type=int, default=5)
args = ap.parse_args()
dev = torch.device("cuda:0")
try:
    smi = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    smi = "nvidia-smi unavailable"
print(f"{torch.cuda.get_device_name(dev)}; nvidia-smi name, power limit: {smi}; {L.sm_count()} SMs")


def timeit(fn):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(args.windows):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) / args.iters)
    return sorted(ts)[len(ts) // 2]  # ms per call


print(f"{'B':>3} {'L':>6} {'d':>4} {'dv':>4} | {'fwd ms':>9} {'TFLOP/s':>8} {'%67':>5} | {'fwd+bwd ms':>10} {'TFLOP/s':>8} {'%67':>5}")
for B, S, d, dv in SHAPES:
    g = torch.Generator(device=dev).manual_seed(B + S + d + dv)
    q, k = (torch.randn(B, S, d, device=dev, generator=g) for _ in range(2))
    v, go = (torch.randn(B, S, dv, device=dev, generator=g) for _ in range(2))
    out, dq, dk, dvv = torch.empty_like(v), torch.empty_like(q), torch.empty_like(k), torch.empty_like(v)
    fwd = lambda: L.linear_attn_fwd(q, k, v, out)

    def fwd_bwd():
        L.linear_attn_fwd(q, k, v, out)
        L.linear_attn_bwd(q, k, v, go, dq, dk, dvv)

    try:
        fwd_bwd()
    except RuntimeError as e:
        print(f"{B:>3} {S:>6} {d:>4} {dv:>4} | not supported by this build: {str(e).splitlines()[0][:80]}")
        continue
    flops = 4.0 * B * S * d * dv
    tf, tfb = timeit(fwd), timeit(fwd_bwd)
    rf, rfb = flops / tf / 1e9, 4 * flops / tfb / 1e9
    print(f"{B:>3} {S:>6} {d:>4} {dv:>4} | {tf:9.4f} {rf:8.2f} {1e14 * rf / FP32_DATASHEET:5.1f} | {tfb:10.4f} "
          f"{rfb:8.2f} {1e14 * rfb / FP32_DATASHEET:5.1f}")
