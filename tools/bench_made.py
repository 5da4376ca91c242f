"""MADE at its recipe size, MADE(784, [8000]) on binarized 28x28 images: the training step and sample().

    python tools/bench_made.py [--steps 50] [--warmup 5] [--reps 3] [--out results.json]

Training step: Trainer._train_one_batch's work (zero_grad, forward, recipe loss, backward, FusedAdam.clip_and_step) at
batch 64, timed with a device synchronise around `--steps` steps: ms per step, images/s and max_memory_allocated.  At
M = 64 rows the step is bound by HBM traffic, not by the tensor cores (2 * 3 * 64 * 12.5 M = 4.8 GFLOP per step), so the
bytes the step must move are counted from the shapes (`step_bytes`) and set against the H100 SXM's 3.35 TB/s.

Sampling: sample(16) and sample(64) on the incremental sampler against one full forward per dimension (the reference's
scheme), alternating in one run.  The card's name and power limit are printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from pytorch_generative_b200 import losses, models, optim

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
D, HIDDEN, BATCH = 784, 8000, 64


def step_bytes(d=D, hidden=HIDDEN):
    """HBM bytes one training step must move, per item (activations at batch 64 are under 1 MB and left out)."""
    w = 2 * d * hidden          # weights of the two masked layers
    b = hidden + d
    return {
        "mask_cast: fp32 weights read, bf16 operands written": 4 * w + 2 * w,
        "forward GEMMs: bf16 operands read": 2 * w,
        "dgrad of the output layer: its bf16 operand read": 2 * d * hidden,
        "wgrad: fp32 gradients zeroed and written": 2 * 4 * w + 2 * 4 * b,
        "gradient norm: fp32 gradients read": 4 * (w + b),
        "Adam: parameters, gradients and both moments read, parameters and moments written": 7 * 4 * (w + b),
    }


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def bench_train(steps, warmup):
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = models.MADE(D, [HIDDEN]).to(dev)
    opt = optim.FusedAdam(model.parameters())
    g = torch.Generator(device=dev).manual_seed(1)
    batches = [torch.bernoulli(torch.full((BATCH, 1, 28, 28), 0.5, device=dev), generator=g) for _ in range(8)]

    def step(x):
        opt.zero_grad()
        loss = losses.bce_with_logits_sum_mean(model(x), x)
        loss.backward()
        return opt.clip_and_step(1e50)

    for i in range(warmup):
        step(batches[i % 8])
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    for i in range(steps):
        step(batches[i % 8])
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3 / steps
    moved = sum(step_bytes().values())
    return dict(ms_per_step=ms, images_per_s=BATCH / ms * 1e3, max_memory_allocated_mb=torch.cuda.max_memory_allocated() / 2**20,
                step_bytes=moved, hbm_share=moved / (ms * 1e-3) / HBM_BYTES_PER_S), model


def bench_sample(model, reps):
    model._register_shape(1, 28, 28)
    model._sample_fn = lambda logits: torch.bernoulli(torch.sigmoid(logits))
    out = {}
    for n in (16, 64):
        times = {"incremental": [], "full_forward": []}
        for incremental in (True, False):  # warm-up: module loads, graph capture
            model._incremental_sampling = incremental
            model.sample(n)
        for _ in range(reps):
            for incremental in (True, False):
                model._incremental_sampling = incremental
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                model.sample(n)
                torch.cuda.synchronize()
                times["incremental" if incremental else "full_forward"].append((time.perf_counter() - t0) * 1e3)
        out[f"sample({n})"] = {k: dict(ms_min=min(v), ms_all=v) for k, v in times.items()}
    model._incremental_sampling = True
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_made.py measures on a CUDA device; none is available")
    gpu = card()
    print(f"GPU (name, power limit): {gpu}", flush=True)
    train, model = bench_train(args.steps, args.warmup)
    print(f"training step MADE({D}, [{HIDDEN}]) batch {BATCH}: {train['ms_per_step']:.3f} ms, "
          f"{train['images_per_s']:.0f} images/s, max_memory_allocated {train['max_memory_allocated_mb']:.0f} MB", flush=True)
    for what, nbytes in step_bytes().items():
        print(f"  {nbytes / 1e6:8.1f} MB  {what}")
    print(f"  {train['step_bytes'] / 1e6:8.1f} MB per step = {100 * train['hbm_share']:.1f}% of 3.35 TB/s over the step time")
    sampling = bench_sample(model, args.reps)
    for k, v in sampling.items():
        inc, full = v["incremental"]["ms_min"], v["full_forward"]["ms_min"]
        print(f"{k}: incremental {inc:.1f} ms, full forward per dimension {full:.1f} ms ({full / inc:.1f}x)")
    result = dict(gpu=gpu, train=train, sampling=sampling)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
