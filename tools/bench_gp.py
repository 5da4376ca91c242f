"""GaussianProcess on the H100: the fp64 Cholesky alone, predict, predict + backward and sample(x, 16), each against a
plain-torch fp64 arm on the same GPU (torch.linalg.cholesky, solve_triangular and matmul, i.e. cuSOLVER / cuBLAS) run
alternately with it in the same call, plus a CPU arm running the reference's formula (torch.linalg.solve) at M = 1024.

    python tools/bench_gp.py [--sizes 1024,4096,16384] [--queries 4096] [--dim 8] [--reps 3] [--out r.json]

Times are CUDA events around each call, best of `--reps`, after a warm-up.  FLOP counts come from the shapes: M^3 / 3
for the factorisation, M^2 (N + k) for the solves and M N^2 for Q (k = 1 output).  One extra Cholesky per size runs
under torch.profiler to split its time between the diagonal-block factor (the serial critical path), the panel solves
and the trailing GEMM.  The card's name and power limit are printed with the numbers.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
from torch import nn

from pytorch_generative_b200 import _lib, models

F64 = torch.float64


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                        "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


class Mean(nn.Module):
    def __init__(self):
        super().__init__()
        self.c = nn.Parameter(torch.tensor(0.1, dtype=F64))

    def forward(self, x):
        return torch.ones(x.shape[0], 1, dtype=x.dtype, device=x.device) * self.c


class SqExp(nn.Module):
    """s^2 exp(-0.5 |a - b|^2 / l^2) through |a|^2 + |b|^2 - 2 a.b (no [M, N, D] intermediate at these sizes)."""

    def __init__(self):
        super().__init__()
        self.s = nn.Parameter(torch.tensor(1.0, dtype=F64))
        self.ell = nn.Parameter(torch.tensor(1.5, dtype=F64))

    def forward(self, a, b):
        sq = ((a * a).sum(1)[:, None] + (b * b).sum(1)[None, :] - 2 * a @ b.T).clamp_min(0)
        return self.s ** 2 * torch.exp(-0.5 * sq / self.ell ** 2)


def event_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return min(times)


def torch_predict(mean, kernel, noise, tx, ty, x):
    A = kernel(tx, tx) + noise * torch.eye(tx.shape[0], dtype=F64, device=tx.device)
    Lc = torch.linalg.cholesky(A)
    V = torch.linalg.solve_triangular(Lc, kernel(tx, x), upper=False)
    beta = torch.linalg.solve_triangular(Lc, ty - mean(tx), upper=False)
    return mean(x) + V.T @ beta, kernel(x, x) - V.T @ V


def phase_split(A, noise):
    """ms per kernel family of one pg_gp_potrf, from torch.profiler's CUDA activities."""
    from torch.profiler import ProfilerActivity, profile

    d = torch.zeros(1, dtype=torch.int32, device="cuda")
    Ac = A.clone()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        _lib.gp_potrf(Ac, noise, d)
        torch.cuda.synchronize()
    split = {}
    for ev in prof.events():
        if ev.device_type.name != "CUDA":
            continue
        for key in ("potrf_diag", "tri_solve", "gemm_f64", "potrf_prep"):
            if key in ev.name:
                split[key] = split.get(key, 0.0) + ev.device_time / 1e3
    return split


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1024,4096,16384")
    ap.add_argument("--queries", type=int, default=4096)
    ap.add_argument("--dim", type=int, default=8)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_gp: needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    res = dict(card=card(), queries=args.queries, dim=args.dim, sizes={})
    print(res["card"], flush=True)
    noise = 1e-2
    N, D = args.queries, args.dim
    for M in [int(s) for s in args.sizes.split(",")]:
        g = torch.Generator().manual_seed(M)
        tx = (torch.rand(M, D, generator=g, dtype=F64) * 6).cuda()
        ty = torch.sin(tx).sum(1, keepdim=True)
        x = (torch.rand(N, D, generator=g, dtype=F64) * 6).cuda()
        mean, kernel = Mean().cuda(), SqExp().cuda()
        gp = models.GaussianProcess(mean, kernel, noise)
        gp.fit(tx, ty)
        with torch.no_grad():
            K = kernel(tx, tx)
        nz = float(gp.noise_var)
        d = torch.zeros(1, dtype=torch.int32, device="cuda")
        eye = torch.eye(M, dtype=F64, device="cuda")
        xs = x.clone().requires_grad_(True)

        def ours_potrf():
            _lib.gp_potrf(K.clone(), nz, d)

        def torch_potrf():
            torch.linalg.cholesky(K + nz * eye)

        def ours_predict():
            with torch.no_grad():
                gp.predict(x)

        def torch_pred():
            with torch.no_grad():
                torch_predict(mean, kernel, nz, tx, ty, x)

        def ours_fb():
            mu, sig = gp.predict(xs)
            (mu.sum() + sig.sum()).backward()

        def torch_fb():
            mu, sig = torch_predict(mean, kernel, nz, tx, ty, xs)
            (mu.sum() + sig.sum()).backward()

        def ours_sample():
            gp.sample(x, 16)

        def torch_sample():
            with torch.no_grad():
                mu, sig = torch_predict(mean, kernel, nz, tx, ty, x)
                Ls = torch.linalg.cholesky(sig + 1e-10 * torch.eye(N, dtype=F64, device="cuda"))
                mu.T + torch.randn(16, N, dtype=F64, device="cuda") @ Ls.T

        row = {}
        for name, ours, theirs in (("potrf", ours_potrf, torch_potrf), ("predict", ours_predict, torch_pred),
                                   ("predict_backward", ours_fb, torch_fb), ("sample16", ours_sample, torch_sample)):
            a, b = [], []
            for _ in range(2):  # alternate the two arms
                a.append(event_ms(ours, args.reps))
                try:
                    b.append(event_ms(theirs, args.reps))
                except RuntimeError as e:  # e.g. cuSOLVER refusing the sample covariance
                    b.append(float("nan"))
                    row[f"{name}_torch_error"] = str(e)[:200]
            row[name] = dict(ours_ms=min(a), torch_ms=min(b))
        k = 1
        flops = dict(potrf=M ** 3 / 3, solves=M ** 2 * (N + k), q=M * N ** 2)
        row["flops"] = flops
        row["potrf"]["ours_tflops"] = flops["potrf"] / row["potrf"]["ours_ms"] / 1e9
        row["potrf"]["torch_tflops"] = flops["potrf"] / row["potrf"]["torch_ms"] / 1e9
        tot = sum(flops.values())
        row["predict"]["ours_tflops"] = tot / row["predict"]["ours_ms"] / 1e9
        row["predict"]["torch_tflops"] = tot / row["predict"]["torch_ms"] / 1e9
        row["potrf_phase_ms"] = phase_split(K, nz)
        row["dropped"] = int(gp.dropped)
        res["sizes"][M] = row
        print(M, json.dumps(row), flush=True)
        del K, gp, eye
        torch.cuda.empty_cache()
    # CPU arm: the reference's formula at M = 1024
    g = torch.Generator().manual_seed(1)
    tx = torch.rand(1024, D, generator=g, dtype=F64) * 6
    ty = torch.sin(tx).sum(1, keepdim=True)
    x = torch.rand(N, D, generator=g, dtype=F64) * 6
    mean, kernel = Mean(), SqExp()
    with torch.no_grad():
        best = float("inf")
        for _ in range(args.reps):
            t0 = time.perf_counter()
            A = kernel(tx, tx) + torch.tensor(noise) * torch.eye(1024)
            solved = torch.linalg.solve(A, kernel(tx, x)).T
            mean(x) + solved @ (ty - mean(tx)), kernel(x, x) - solved @ kernel(tx, x)
            best = min(best, (time.perf_counter() - t0) * 1e3)
    res["cpu_reference_predict_ms_m1024"] = best
    res["cpu_threads"] = torch.get_num_threads()
    print(json.dumps(res))
    if args.out:
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
