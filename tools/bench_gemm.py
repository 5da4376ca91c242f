"""Micro-benchmark of pg_gemm_bf16 on the ImageGPT C5 shapes (CUDA events, L2 flushed between reps).
    python tools/bench_gemm.py [rows.json]   (the per-shape rows are also written as JSON when a path is given)

Each row also gives the algorithmic HBM bytes (operands read once, every epilogue input read once, every output
written once; an accumulated output is read and written) and the row's floor: the larger of its FLOPs at the H100 SXM
data sheet's dense BF16 rate and its bytes at the data sheet's HBM3 bandwidth (700 W card).  `floor` is that time over
the measured time; the epilogue-heavy K = 512 rows are bandwidth-bound, where TFLOP/s alone cannot show the headroom.
A card with a lower power limit runs its SM clock below the data sheet's, so its floor fractions read low: the card's
name, power limit and SM clock before and after the rows are printed with the table and stored with the JSON rows."""
import sys, os, json, subprocess
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pytorch_generative_b200 import _lib as L

dev = torch.device("cuda:0")
P = int(os.environ.get("PG_P", 65536))
PEAK_TFLOPS, PEAK_HBM_GBS = 989.0, 3350.0
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def gpu_state():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader", "-i", str(dev.index or 0)],
                             capture_output=True, text=True, timeout=10).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or "nvidia-smi unavailable"


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
    if kw.get("bias_grad"): extra["bias_grad"] = torch.zeros(M, device=dev)
    fn = lambda: L.gemm(A, B, M, N, K, a_mn=a_mn, b_mn=b_mn, **outs, **extra)
    old = L.reserve_sms(0)
    if kw.get("grid"):  # persistent grid of this many CTAs (the other SMs reserved)
        L.reserve_sms(L.sm_count() - kw["grid"])
    try:
        ms = timeit(fn)
    finally:
        L.reserve_sms(old)
    flops = 2.0 * M * N * K
    nbytes = A.numel() * 2 + B.numel() * 2 + sum(t.numel() * t.element_size() for t in extra.values() if torch.is_tensor(t))
    nbytes += sum(t.numel() * t.element_size() * (2 if k == "out_f32" and "split_k" in extra else 1) for k, t in outs.items())
    floor_ms = max(flops / (PEAK_TFLOPS * 1e9), nbytes / (PEAK_HBM_GBS * 1e6))
    bound = "tensor" if flops / (PEAK_TFLOPS * 1e9) >= nbytes / (PEAK_HBM_GBS * 1e6) else "hbm"
    tf = flops / ms / 1e9
    rows.append(dict(name=name, M=M, N=N, K=K, ms=round(ms, 4), tflops=round(tf, 1), bytes=nbytes,
                     floor_ms=round(floor_ms, 4), floor_bound=bound, floor_frac=round(floor_ms / ms, 3)))
    print(f"{name:28s} M={M:6d} N={N:5d} K={K:6d}  {ms:8.4f} ms  {tf:6.1f} TFLOP/s  {nbytes / 2**20:7.1f} MiB  "
          f"floor {floor_ms:7.4f} ms ({bound:6s})  {floor_ms / ms:6.1%} of floor", flush=True)

gpu_before = gpu_state()
print(f"GPU (name, power limit, SM clock, max SM clock): {gpu_before}", flush=True)
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
# the training step's weight gradients: one wave of work items (ops._split_k_for on 132 SMs), bias gradient fused
for name, M, N, sk in (("fc1", 2048, 512, 2), ("fc2", 512, 2048, 2), ("proj", 512, 512, 8), ("qkv", 1536, 512, 2)):
    case(f"{name} wgrad split{sk} +bgrad", M, N, P, a_mn=True, b_mn=True, f32=True, f32_only=True, split_k=sk,
         bias_grad=True)
# The same launches without the bias gradient, which only the N block 0 CTAs sum, and on 66 CTAs, each running two of
# the full grid's items back to back.  Together they show whether the bias-gradient CTAs or the main loop's operand
# delivery set the pace (DESIGN.md section 4).
for name, M, N in (("fc1", 2048, 512), ("fc2", 512, 2048)):
    case(f"{name} wgrad split2", M, N, P, a_mn=True, b_mn=True, f32=True, f32_only=True, split_k=2)
    case(f"{name} wgrad split2 +bgrad 66 CTAs", M, N, P, a_mn=True, b_mn=True, f32=True, f32_only=True, split_k=2,
         bias_grad=True, grid=66)
    case(f"{name} wgrad split2 66 CTAs", M, N, P, a_mn=True, b_mn=True, f32=True, f32_only=True, split_k=2, grid=66)
# cuBLAS reference point
A = torch.randn(P, 512, device=dev).bfloat16(); W = torch.randn(2048, 512, device=dev).bfloat16()
ms = timeit(lambda: torch.matmul(A, W.t()))
print(f"cuBLAS bf16 {P}x2048x512: {ms:.4f} ms {2.0*P*2048*512/ms/1e9:.1f} TFLOP/s")
gpu_after = gpu_state()
print(f"GPU after the rows: {gpu_after}", flush=True)
if len(sys.argv) > 1:
    json.dump(dict(gpu_before=gpu_before, gpu_after=gpu_after, rows=rows), open(sys.argv[1], "w"), indent=1)
