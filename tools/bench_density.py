"""KernelDensityEstimator and the mixture models at MNIST size, each against a plain-torch arm running the reference's
expressions in the same run (fp32, TF32 off).

    python tools/bench_density.py [--queries 10000] [--train 60000] [--torch-queries 1000] [--reps 3] [--out r.json]

KDE: `--queries` seeded synthetic MNIST-shaped queries (784 features in [0, 1]) against `--train` training points, for
the Gaussian kernel (forward, and forward plus the query gradient) and the Parzen window.  Each time is CUDA events
around the call, best of `--reps`, after a warm-up.  The reference broadcasts [N, M, D], so the torch arm is run chunked
over the queries (the chunk size is reported) on the first `--torch-queries` queries, and its time is reported for that
subset as measured.  Achieved FLOP/s counts 3 FLOP per (query, training point, feature) for the Gaussian pass (a
subtraction, a multiply and an add), set against the H100 SXM data sheet's 67 TFLOP/s FP32.

Mixture models: a training step (zero_grad, forward, -mean log-likelihood, backward, Adam) of GaussianMixtureModel and
BernoulliMixtureModel at batch 1024, K = 64, D = 784, eager and under `trainstep.GraphedTrainStep`, against the
reference's expressions under torch autograd with torch.optim.Adam.

It also reports whether torch on CUDA divides an fp32 tensor by a Python float exactly as IEEE division does (the
CPU reference's result), on 2^22 samples per bandwidth.  The card's name and power limit are printed with the numbers.
"""
import argparse
import copy
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

from pytorch_generative_b200 import _lib, models, trainstep

FP32_FLOPS = 67e12  # H100 SXM data sheet, dense FP32


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                        "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def event_ms(fn, reps, warmup=1):
    for _ in range(warmup):
        fn()
    best = float("inf")
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b))
    return best


def torch_gauss(x, t, h, chunk):
    """The reference's GaussianKernel.forward, chunked over the queries."""
    n, d = t.shape
    nt, ht, pi = torch.tensor(n, dtype=torch.float32), torch.tensor(h), torch.tensor(np.pi)
    Z = (0.5 * d * torch.log(2 * pi) + d * torch.log(ht) + torch.log(nt)).to(x.device)
    out = []
    for i in range(0, x.shape[0], chunk):
        diffs = (x[i:i + chunk, None, :] - t[None]) / h
        out.append(torch.logsumexp(-0.5 * torch.norm(diffs, p=2, dim=-1) ** 2 - Z, dim=-1))
    return torch.cat(out)


def torch_parzen(x, t, h, chunk):
    """The reference's ParzenWindowKernel.forward, chunked over the queries (its coefficient in fp32 as the product's
    log-density, so that the arm runs at D = 784 where 1 / h**D overflows)."""
    out = []
    d = t.shape[1]
    for i in range(0, x.shape[0], chunk):
        inside = (torch.abs(x[i:i + chunk, None, :] - t[None]) / h <= 0.5).sum(-1) == d
        out.append(torch.log(inside.float().mean(1)) - d * float(np.log(h)))
    return torch.cat(out)


def bench_kde(args, dev):
    g = torch.Generator(device=dev).manual_seed(0)
    D = 784
    t = (torch.rand((args.train, D), device=dev, generator=g) < 0.13).float() * torch.rand((args.train, D), device=dev,
                                                                                           generator=g)
    x = t[torch.randint(0, args.train, (args.queries,), device=dev, generator=g)] + \
        0.05 * torch.randn((args.queries, D), device=dev, generator=g)
    N, M = args.queries, args.train
    chunk = max(1, (1 << 31) // (M * D * 4))  # a [chunk, M, D] fp32 broadcast of at most 2 GiB
    res = {"queries": N, "train": M, "features": D, "torch_queries": args.torch_queries, "torch_chunk": chunk}
    flops = 3.0 * N * M * D
    gauss = models.KernelDensityEstimator(t, models.GaussianKernel(bandwidth=1.0))
    parzen = models.KernelDensityEstimator(t, models.ParzenWindowKernel(bandwidth=0.5))
    with torch.no_grad():
        res["gauss_fwd_ms"] = event_ms(lambda: gauss(x), args.reps)
        res["parzen_ms"] = event_ms(lambda: parzen(x), args.reps)
    xg = x.clone().requires_grad_(True)
    res["gauss_fwd_bwd_ms"] = event_ms(lambda: torch.autograd.grad(gauss(xg).sum(), xg), args.reps)
    res["gauss_fwd_tflops"] = flops / res["gauss_fwd_ms"] * 1e-9
    res["gauss_fwd_fp32_share"] = res["gauss_fwd_tflops"] * 1e12 / FP32_FLOPS
    res["gauss_fwd_floor_ms"] = flops / FP32_FLOPS * 1e3
    xs = x[: args.torch_queries]
    with torch.no_grad():
        res["torch_gauss_fwd_ms_subset"] = event_ms(lambda: torch_gauss(xs, t, 1.0, chunk), args.reps)
        res["torch_parzen_ms_subset"] = event_ms(lambda: torch_parzen(xs, t, 0.5, chunk), args.reps)
        ours = gauss(xs)
        ref = torch_gauss(xs.double(), t.double(), 1.0, max(1, chunk // 2)).float()
        res["gauss_max_abs_diff_vs_float64"] = (ours - ref).abs().max().item()
        res["parzen_equal_to_torch"] = bool(torch.equal(parzen(xs), torch_parzen(xs, t, 0.5, chunk)))
    return res


def _ref_mixture_loss(cls, p, x):
    from _density_reference import mixture_forward

    return -mixture_forward(cls, p, x).mean()


def bench_mixture(args, dev):
    res = {}
    for cls in ("GaussianMixtureModel", "BernoulliMixtureModel"):
        torch.manual_seed(0)
        m = getattr(models, cls)(64, 784).to(dev)
        g = torch.Generator(device=dev).manual_seed(1)
        x = torch.rand((1024, 1, 28, 28), device=dev, generator=g)
        if cls == "BernoulliMixtureModel":
            x = (x < 0.13).float()
        eager = copy.deepcopy(m)
        opt = torch.optim.Adam(eager.parameters(), lr=1e-3)

        def eager_step():
            opt.zero_grad(set_to_none=True)
            (-eager(x).mean()).backward()
            opt.step()

        graphed = copy.deepcopy(m)
        step = trainstep.GraphedTrainStep(graphed, graphed.parameters(), lambda p, xx: -p.mean(), x, lr=1e-3,
                                          lr_gamma=1.0)
        ref_p = {k: v.detach().clone().requires_grad_(True) for k, v in m.named_parameters()}
        ref_opt = torch.optim.Adam(list(ref_p.values()), lr=1e-3)

        def torch_step():
            ref_opt.zero_grad(set_to_none=True)
            _ref_mixture_loss(cls, ref_p, x).backward()
            ref_opt.step()

        steps = max(1, args.steps)
        before = _lib.launch_count()
        eager_step()
        torch.cuda.synchronize()
        launches = _lib.launch_count() - before
        res[cls] = {"batch": 1024, "components": 64, "features": 784, "launches_per_step": launches,
                    "eager_ms": event_ms(lambda: [eager_step() for _ in range(steps)], args.reps) / steps,
                    "graphed_ms": event_ms(lambda: [step(x) for _ in range(steps)], args.reps) / steps,
                    "torch_ms": event_ms(lambda: [torch_step() for _ in range(steps)], args.reps) / steps}
    return res


def division_check(dev):
    """Whether torch on CUDA computes fp32 `a / h` (h a Python float) as IEEE division, against torch on the CPU."""
    g = torch.Generator().manual_seed(0)
    a = torch.rand(1 << 22, generator=g) * 4
    out = {}
    for h in (0.1, 0.3, 0.5, 0.7, 2.0 / 3.0):
        cpu = a / h
        cuda = (a.to(dev) / h).cpu()
        recip = a * np.float32(1.0 / np.float32(h))
        out[str(h)] = {"mismatches_vs_cpu": int((cpu != cuda).sum()),
                       "cuda_equals_multiply_by_reciprocal": bool(torch.equal(cuda, recip)),
                       "boundary_flips": int(((cpu <= 0.5) != (cuda <= 0.5)).sum())}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=10000)
    ap.add_argument("--train", type=int, default=60000)
    ap.add_argument("--torch-queries", type=int, default=1000)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_density.py measures the CUDA path: no GPU found")
    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda")
    res = {"card": card(), "division": division_check(dev), "kde": bench_kde(args, dev),
           "mixture": bench_mixture(args, dev)}
    text = json.dumps(res, indent=1)
    print(text)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
