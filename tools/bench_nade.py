"""NADE at its recipe size, NADE(784, 500) on binarized 28x28 images: the training step and sample(), each against the
per-dimension torch loop of tests/_nade_reference.py (the reference's own scheme) on the same GPU, alternating in one
run.

    python tools/bench_nade.py [--steps 50] [--warmup 5] [--ref-steps 5] [--reps 3] [--out results.json]

Training step: Trainer._train_one_batch's work (zero_grad, forward, recipe loss, backward, FusedAdam.clip_and_step) at
batch 512, timed with a device synchronise around `--steps` steps: ms per step, images/s, the forward alone (so the
rest of the step is the backward and the optimizer), and the memory of the CUDA step: max_memory_allocated over its own
steps (torch's allocations), plus the library's scratch, which is cudaMalloc'ed outside torch and counted from the
shapes (`scratch_bytes`).  The FLOPs and the HBM bytes the step needs are counted from the shapes (`step_flops`,
`step_bytes`) and set against the H100 SXM's 67 TFLOP/s fp32 and 3.35 TB/s; the larger of the two times is the bound.  The comparison arm runs the same step
with the torch loop and torch.optim.Adam.

Sampling: sample(16) and sample(64), one scan launch each, against the torch loop.  The card's name and power limit are
printed with the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch

import _nade_reference as R
from pytorch_generative_b200 import _lib, losses, models, optim

FP32_FLOPS = 67e12         # H100 SXM data sheet, dense fp32
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
D, HIDDEN, BATCH = 784, 500, 512
BWD_TILES = 16             # image tiles of pg_nade_bwd at batch 512 (32 images each)


def step_flops(n=BATCH, d=D, h=HIDDEN):
    """fp32 operations per (image, dimension, hidden unit) of the algorithm, times n * d * h."""
    ndh = n * d * h
    return {
        "forward: the dot with relu (2) and the update of a (2)": 4 * ndh,
        "backward: a recomputed from its checkpoint (2)": 2 * ndh,
        "backward: _h_W gradient (2), _in_W gradient (2), ReLU' and da (2), the running sum s (1)": 7 * ndh,
    }


def step_bytes(n=BATCH, d=D, h=HIDDEN, tiles=BWD_TILES):
    """HBM bytes one training step must move (inputs, p and the loss are under 10 MB and left out)."""
    chunks = -(-d // _lib.NADE_CHUNK)
    params = 2 * d * h + d + h
    return {
        "checkpoints of a: written by the forward, read by the backward": 2 * 4 * n * chunks * h,
        "running sums s between chunks: written and read per chunk": 2 * 4 * n * h * chunks,
        "weight-gradient partials: written, then read by the fixed-order sum": 2 * 2 * 4 * tiles * d * h,
        "weights: read by the forward (with the transpose of _in_W) and the backward": 4 * 4 * d * h,
        "gradients: zeroed, then read and written by the sum": 3 * 4 * params,
        "gradient norm and Adam: parameters, gradients and both moments read, parameters and moments written": 8 * 4 * params,
    }


def scratch_bytes(n=BATCH, d=D, h=HIDDEN, tiles=BWD_TILES):
    """pg_scratch bytes the step needs (the larger of its two uses; pg_scratch allocates at least 16 MB and grows by
    doubling, so the buffer may be larger): the forward's transposed _in_W, the backward's running sums and partials."""
    forward = 4 * d * h
    backward = 4 * (n * h + 2 * tiles * d * h + tiles * (d + h))
    return max(forward, backward)


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=name,power.limit",
                        "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def timed(fn, count):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(count):
        fn(i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / count


def bench_train(steps, warmup, ref_steps, reps):
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = models.NADE(D, HIDDEN).to(dev)
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    ref = R.TrainState(state, device=dev)
    opt = optim.FusedAdam(model.parameters())
    g = torch.Generator(device=dev).manual_seed(1)
    batches = [torch.bernoulli(torch.full((BATCH, 1, 28, 28), 0.5, device=dev), generator=g) for _ in range(8)]
    u = torch.zeros(BATCH, D, device=dev)  # binarized images: nothing is drawn

    def step(i):
        x = batches[i % 8]
        opt.zero_grad()
        loss = losses.bce_with_logits_sum_mean(model(x), x)
        loss.backward()
        opt.clip_and_step(1e50)

    def ref_step(i):
        ref.step(batches[i % 8], u)

    def forward(i):
        model(batches[i % 8])  # with gradients: the checkpoints are kept, as in the step

    for i in range(warmup):
        step(i)
    ref_step(0)
    torch.cuda.synchronize()
    times = {"cuda": [], "forward": [], "torch_loop": []}
    peak = 0.0
    for _ in range(reps):
        torch.cuda.reset_peak_memory_stats()  # the CUDA arm alone
        times["cuda"].append(timed(step, steps))
        peak = max(peak, torch.cuda.max_memory_allocated() / 2**20)
        times["forward"].append(timed(forward, steps))
        times["torch_loop"].append(timed(ref_step, ref_steps))
    ms = min(times["cuda"])
    flops, moved = sum(step_flops().values()), sum(step_bytes().values())
    t_flops, t_bytes = flops / FP32_FLOPS * 1e3, moved / HBM_BYTES_PER_S * 1e3
    return dict(ms_per_step=ms, ms_all=times["cuda"], images_per_s=BATCH / ms * 1e3,
                forward_ms=min(times["forward"]), forward_ms_all=times["forward"],
                scratch_mb=scratch_bytes() / 2**20,
                torch_loop_ms_per_step=min(times["torch_loop"]), torch_loop_ms_all=times["torch_loop"],
                max_memory_allocated_mb=peak, step_flops=flops, step_bytes=moved, fp32_share=t_flops / ms,
                hbm_share=t_bytes / ms, bound="fp32" if t_flops > t_bytes else "HBM"), model


def bench_sample(model, reps):
    state = {k: v.detach().clone() for k, v in model.state_dict().items()}
    dev = next(model.parameters()).device
    out = {}
    for n in (16, 64):
        canvas = -torch.ones(n, D, device=dev)
        arms = {"cuda": lambda _: model.sample(conditioned_on=canvas),
                "torch_loop": lambda _: R.sample(state, canvas, torch.rand(n, D, device=dev))}
        for fn in arms.values():  # warm-up
            fn(0)
        times = {k: [] for k in arms}
        for _ in range(reps):
            for k, fn in arms.items():
                times[k].append(timed(fn, 1))
        out[f"sample({n})"] = {k: dict(ms_min=min(v), ms_all=v) for k, v in times.items()}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--ref-steps", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nade.py measures on a CUDA device; none is available")
    gpu = card()
    print(f"GPU (name, power limit): {gpu}", flush=True)
    train, model = bench_train(args.steps, args.warmup, args.ref_steps, args.reps)
    print(f"training step NADE({D}, {HIDDEN}) batch {BATCH}: {train['ms_per_step']:.3f} ms "
          f"(runs {', '.join(f'{t:.3f}' for t in train['ms_all'])}), {train['images_per_s']:.0f} images/s, "
          f"max_memory_allocated {train['max_memory_allocated_mb']:.0f} MB + library scratch {train['scratch_mb']:.0f} MB; "
          f"torch loop {train['torch_loop_ms_per_step']:.1f} ms ({train['torch_loop_ms_per_step'] / train['ms_per_step']:.0f}x)",
          flush=True)
    print(f"  forward {train['forward_ms']:.3f} ms, backward and optimizer {train['ms_per_step'] - train['forward_ms']:.3f} ms")
    for what, f in step_flops().items():
        print(f"  {f / 1e9:8.2f} GFLOP  {what}")
    print(f"  {train['step_flops'] / 1e9:8.2f} GFLOP per step = {100 * train['fp32_share']:.1f}% of 67 TFLOP/s over the step time")
    for what, nbytes in step_bytes().items():
        print(f"  {nbytes / 1e6:8.1f} MB  {what}")
    print(f"  {train['step_bytes'] / 1e6:8.1f} MB per step = {100 * train['hbm_share']:.1f}% of 3.35 TB/s over the step time")
    print(f"  bound: {train['bound']}")
    sampling = bench_sample(model, args.reps)
    for k, v in sampling.items():
        cuda, loop = v["cuda"]["ms_min"], v["torch_loop"]["ms_min"]
        print(f"{k}: one scan {cuda:.2f} ms, torch loop {loop:.1f} ms ({loop / cuda:.0f}x)")
    result = dict(gpu=gpu, train=train, sampling=sampling)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
