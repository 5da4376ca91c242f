"""Launch cost of the GEMM kernel: back-to-back launches of the smallest pg_gemm_bf16 problem (one 128 x 64 tile,
K = 64), where the kernel's run time is a few microseconds and the launch itself is a large part of each step.
    python tools/bench_launch.py [path/to/libpg_b200.so]

The library is loaded directly with ctypes and only pg_gemm_bf16 is bound, so two builds of the library (for example
before and after a change to the kernel's parameter block) can be compared with the same script.  Two numbers per run:
  * host: wall time per launch of 5000 eager launches followed by one synchronise (the enqueue path: ctypes, argument
    checks, TMA descriptor encoding, cudaLaunchKernel);
  * graph: device time per kernel of a captured CUDA graph of 500 launches, replayed 20 times (CUDA events): kernel
    run time plus the gap between dependent kernels, which grows with the parameter block each node carries.
The card's name and power limit are printed with the numbers."""
import ctypes
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from pytorch_generative_b200._lib import GemmEpilogue

dev = torch.device("cuda:0")
lib_path = sys.argv[1] if len(sys.argv) > 1 else os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(
    __file__))), "pytorch_generative_b200", "libpg_b200.so")
lib = ctypes.CDLL(lib_path)
_vp, _i32, _i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
lib.pg_gemm_bf16.argtypes = [_vp, _i32, _i64, _vp, _i32, _i64, _i32, _i32, _i32, _i32, ctypes.POINTER(GemmEpilogue), _i32,
                             _vp]
lib.pg_gemm_bf16.restype = ctypes.c_int
lib.pg_last_error.restype = ctypes.c_char_p

M, N, K = 128, 64, 64
A = torch.randn(M, K, device=dev).to(torch.bfloat16)
B = torch.randn(N, K, device=dev).to(torch.bfloat16)
out = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
e = GemmEpilogue()
e.out_bf16, e.ld_out_bf16, e.alpha = out.data_ptr(), N, 1.0


def launch():
    rc = lib.pg_gemm_bf16(A.data_ptr(), 0, K, B.data_ptr(), 0, K, M, N, K, 1, ctypes.byref(e), 0,
                          torch.cuda.current_stream().cuda_stream)
    assert rc == 0, lib.pg_last_error()


for _ in range(100):
    launch()
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(5000):
    launch()
torch.cuda.synchronize()
host_us = (time.perf_counter() - t0) / 5000 * 1e6

g = torch.cuda.CUDAGraph()
with torch.cuda.graph(g):  # launch() passes the capture stream: torch makes it current inside this block
    for _ in range(500):
        launch()
g.replay()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(20):
    g.replay()
e1.record()
torch.cuda.synchronize()
graph_us = e0.elapsed_time(e1) / (20 * 500) * 1e3

card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                      text=True).stdout.strip()
print(f"{os.path.relpath(lib_path)}: host {host_us:.2f} us/launch, graph {graph_us:.3f} us/kernel  ({card})", flush=True)
