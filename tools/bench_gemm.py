"""Micro-benchmark of pg_gemm_bf16 on the ImageGPT C5 shapes (CUDA events, L2 flushed between reps).
    python tools/bench_gemm.py [rows.json]   (the per-shape rows are also written as JSON when a path is given)"""
import sys, os, json
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pytorch_generative_b200 import _lib as L

dev = torch.device("cuda:0")
P = int(os.environ.get("PG_P", 65536))
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)

def timeit(fn, reps=10):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(); fn(); e.record(); torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]

rows = []
ONLY = os.environ.get("PG_CASES")
def case(name, M, N, K, **kw):
    if ONLY and not any(t in name for t in ONLY.split(",")):
        return
    a_mn, b_mn = kw.get("a_mn", False), kw.get("b_mn", False)
    A = torch.randn((K, M) if a_mn else (M, K), device=dev).bfloat16()
    B = torch.randn((K, N) if b_mn else (N, K), device=dev).bfloat16()
    outs = {}
    if kw.get("f32"): outs["out_f32"] = torch.zeros(M, N, device=dev)
    if kw.get("bf16", True) and not kw.get("f32_only"): outs["out_bf16"] = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    if kw.get("pre"): outs["out_pre"] = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    extra = {}
    if kw.get("bias"): extra["bias"] = torch.randn(N, device=dev)
    if kw.get("res"): extra["res0"] = torch.randn(M, N, device=dev)
    if kw.get("res2"): extra["res1"] = torch.randn(M, N, device=dev)
    if kw.get("act"): extra["act"] = kw["act"]
    if kw.get("dact"):
        extra["dact"] = kw["dact"]; extra["aux"] = torch.randn(M, N, device=dev).bfloat16()
    if kw.get("split_k"): extra["split_k"] = kw["split_k"]; extra["accumulate"] = True
    fn = lambda: L.gemm(A, B, M, N, K, a_mn=a_mn, b_mn=b_mn, **outs, **extra)
    ms = timeit(fn)
    tf = 2.0 * M * N * K / ms / 1e9
    rows.append(dict(name=name, M=M, N=N, K=K, ms=round(ms, 4), tflops=round(tf, 1)))
    print(f"{name:28s} M={M:6d} N={N:5d} K={K:6d}  {ms:8.4f} ms  {tf:8.1f} TFLOP/s", flush=True)

# forward
case("qkv fwd (bias)", P, 1536, 512, bias=True)
case("proj fwd (bias,res->f32)", P, 512, 512, bias=True, res=True, f32=True, f32_only=True)
case("fc1 fwd (bias,gelu,pre)", P, 2048, 512, bias=True, act=L.ACT_GELU, pre=True)
case("fc1 fwd (bias,gelu,gelu')", P, 2048, 512, bias=True, act=L.ACT_GELU | L.ACT_STORE_DERIV, pre=True)
case("fc2 fwd (bias,2res->f32)", P, 512, 2048, bias=True, res=True, res2=True, f32=True, f32_only=True)
case("plain 512x512", P, 512, 512)
case("plain 2048x512", P, 2048, 512)
# dgrad (B MN-major)
case("fc2 dgrad (dgelu)", P, 2048, 512, b_mn=True, dact=L.ACT_GELU)
case("fc2 dgrad (given gelu')", P, 2048, 512, b_mn=True, dact=L.ACT_GIVEN)
case("fc1 dgrad", P, 512, 2048, b_mn=True)
case("qkv dgrad", P, 512, 1536, b_mn=True)
# wgrad (MN,MN), split-K over pixels
for sk in (1, 4, 8, 16):
    case(f"fc1 wgrad split{sk}", 2048, 512, P, a_mn=True, b_mn=True, f32=True, f32_only=True, split_k=sk)
case("proj wgrad split32", 512, 512, P, a_mn=True, b_mn=True, f32=True, f32_only=True, split_k=32)
case("qkv wgrad split8", 1536, 512, P, a_mn=True, b_mn=True, f32=True, f32_only=True, split_k=8)
# cuBLAS reference point
A = torch.randn(P, 512, device=dev).bfloat16(); W = torch.randn(2048, 512, device=dev).bfloat16()
ms = timeit(lambda: torch.matmul(A, W.t()))
print(f"cuBLAS bf16 {P}x2048x512: {ms:.4f} ms {2.0*P*2048*512/ms/1e9:.1f} TFLOP/s")
if len(sys.argv) > 1:
    json.dump(rows, open(sys.argv[1], "w"), indent=1)
