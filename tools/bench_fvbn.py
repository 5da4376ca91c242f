"""FVBN at its recipe size, FullyVisibleBeliefNetwork(784) on binarized 28x28 images: the training step and sample(),
each against a torch arm of 784 nn.Linear modules (the reference's own scheme, written out here) with torch.optim.Adam
on the same GPU, in the same run.

    python tools/bench_fvbn.py [--steps 50] [--warmup 5] [--ref-steps 5] [--reps 3] [--out results.json]

Training step: Trainer._train_one_batch's work (zero_grad, forward, recipe loss, backward, clip to 1e50 and Adam) at
batch 512, timed with a device synchronise around `--steps` steps (wall time per step).  A separate torch.profiler run
of the same steps gives the GPU time of the step's kernels and the kernels launched per step, so the host's share of
the step (autograd over 1568 parameter inputs, AccumulateGrad, FusedAdam's pointer refresh) is the difference.  The
FLOPs and the HBM bytes the step needs are counted from the shapes and set against the H100 SXM data sheet's 67 TFLOP/s
fp32 and 3.35 TB/s.

Sampling: sample(16) and sample(64), one captured logit step replayed per pixel, against the torch arm's full forward
per pixel.  The card's name and power limit are printed with the numbers."""
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
from torch.nn import functional as F

from pytorch_generative_b200 import _lib, losses, models, optim

FP32_FLOPS = 67e12         # H100 SXM data sheet, dense fp32
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
D, BATCH = 784, 512
SPLITS = 4                 # batch slices of pg_fvbn_bwd at batch 512 (128 images each)


def step_flops(n=BATCH, d=D):
    tri = d * (d - 1) // 2
    params = tri + 1 + d
    return {
        "forward: logits, one multiply-add per (image, j < i)": 2 * n * tri,
        "backward: weight gradient, one multiply-add per (image, j < i)": 2 * n * tri,
        "backward: input gradient, one multiply-add per (image, j < i)": 2 * n * tri,
        "gradient norm and Adam (about 12 per parameter)": 12 * params,
    }


def step_bytes(n=BATCH, d=D, splits=SPLITS):
    """HBM bytes one training step must move."""
    params = d * (d - 1) // 2 + 1 + d
    return {
        "weights: read by the forward and by the input gradient": 2 * 4 * params,
        "x: read by the forward and the backward; logits written, their gradient read, dx written": 5 * 4 * n * d,
        "weight-gradient slice partials: written, then read by the fixed-order sum": 2 * 4 * splits * params,
        "gradient buffer: zeroed, then read and written by the sum": 3 * 4 * params,
        "gradient norm and Adam: parameters, gradients and both moments read, parameters and moments written": 8 * 4 * params,
    }


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


class TorchFVBN(nn.Module):
    """The torch arm: D nn.Linear(max(1, i), 1), a loop of D small GEMMs and a stack (the reference's scheme)."""

    def __init__(self, d):
        super().__init__()
        self._net = nn.ModuleList(nn.Linear(max(1, i), 1) for i in range(d))

    def forward(self, x):
        shape = x.shape
        x = x.view(shape[0], -1)
        out = [self._net[0](torch.zeros(shape[0], 1, device=x.device))]
        for i in range(1, len(self._net)):
            out.append(self._net[i](x[:, :i]))
        return torch.stack(out, dim=1).view(shape)

    @torch.no_grad()
    def sample(self, n):
        canvas = torch.full((n, 1, 28, 28), -1.0, device=next(self.parameters()).device)
        for r in range(28):
            for c in range(28):
                logits = self.forward(canvas)[:, :, r, c]
                drawn = torch.bernoulli(torch.sigmoid(logits))
                canvas[:, :, r, c] = torch.where(canvas[:, :, r, c] < 0, drawn, canvas[:, :, r, c])
        return canvas


def kernel_profile(step, steps):
    """(GPU time of the kernels per step in ms, kernels per step) from a torch.profiler run of `steps` steps."""
    from torch.profiler import ProfilerActivity, profile

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        for i in range(steps):
            step(i)
        torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    busy = sum(e.time_range.elapsed_us() for e in kernels) / 1e3
    return busy / steps, len(kernels) / steps


def bench_train(steps, warmup, ref_steps, reps):
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = models.FullyVisibleBeliefNetwork(D).to(dev)
    torch.manual_seed(0)
    ref = TorchFVBN(D).to(dev)
    opt = optim.FusedAdam(model.parameters())
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-3)
    g = torch.Generator(device=dev).manual_seed(1)
    batches = [torch.bernoulli(torch.full((BATCH, 1, 28, 28), 0.5, device=dev), generator=g) for _ in range(8)]

    def step(i):
        x = batches[i % 8]
        opt.zero_grad()
        loss = losses.bce_with_logits_sum_mean(model(x), x)
        loss.backward()
        opt.clip_and_step(1e50)

    def ref_step(i):
        x = batches[i % 8]
        ref_opt.zero_grad()
        loss = F.binary_cross_entropy_with_logits(ref(x).view(BATCH, -1), x.view(BATCH, -1), reduction="none").sum(1).mean()
        loss.backward()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), 1e50)
        ref_opt.step()

    def forward(i):
        model(batches[i % 8])

    def forward_backward(i):
        x = batches[i % 8]
        opt.zero_grad()
        losses.bce_with_logits_sum_mean(model(x), x).backward()

    for i in range(warmup):
        step(i)
    ref_step(0)
    torch.cuda.synchronize()
    before = _lib.launch_count()
    step(0)
    torch.cuda.synchronize()
    lib_launches = _lib.launch_count() - before
    times = {"cuda": [], "forward": [], "forward_backward": [], "torch": []}
    for _ in range(reps):
        times["cuda"].append(timed(step, steps))
        times["forward"].append(timed(forward, steps))
        times["forward_backward"].append(timed(forward_backward, steps))
        times["torch"].append(timed(ref_step, ref_steps))
    kernel_ms, kernels = kernel_profile(step, steps)
    ref_kernel_ms, ref_kernels = kernel_profile(ref_step, ref_steps)
    ms = min(times["cuda"])
    flops, moved = sum(step_flops().values()), sum(step_bytes().values())
    t_flops, t_bytes = flops / FP32_FLOPS * 1e3, moved / HBM_BYTES_PER_S * 1e3
    return dict(ms_per_step=ms, ms_all=times["cuda"], images_per_s=BATCH / ms * 1e3,
                forward_ms=min(times["forward"]), forward_ms_all=times["forward"],
                forward_backward_ms=min(times["forward_backward"]), forward_backward_ms_all=times["forward_backward"],
                kernel_ms_per_step=kernel_ms, kernels_per_step=kernels, library_launches_per_step=lib_launches,
                torch_ms_per_step=min(times["torch"]), torch_ms_all=times["torch"],
                torch_kernel_ms_per_step=ref_kernel_ms, torch_kernels_per_step=ref_kernels,
                step_flops=flops, step_bytes=moved, bound_ms=max(t_flops, t_bytes),
                bound="fp32" if t_flops > t_bytes else "HBM"), model, ref


def bench_sample(model, ref, reps):
    dev = next(model.parameters()).device
    model(torch.zeros(1, 1, 28, 28, device=dev))  # registers the image shape sample(n) draws
    out = {}
    for n in (16, 64):
        model.sample(n)  # warm-up: captures the step for this n
        cuda = [timed(lambda _: model.sample(n), 1) for _ in range(reps)]
        torch_ms = timed(lambda _: ref.sample(n), 1)  # one run: 784 forwards of 784 modules
        out[f"sample({n})"] = dict(cuda_ms_min=min(cuda), cuda_ms_all=cuda, torch_ms=torch_ms)
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
        raise SystemExit("bench_fvbn.py measures on a CUDA device; none is available")
    gpu = card()
    print(f"GPU (name, power limit): {gpu}", flush=True)
    train, model, ref = bench_train(args.steps, args.warmup, args.ref_steps, args.reps)
    print(f"training step FullyVisibleBeliefNetwork({D}) batch {BATCH}: wall {train['ms_per_step']:.3f} ms "
          f"(runs {', '.join(f'{t:.3f}' for t in train['ms_all'])}), {train['images_per_s']:.0f} images/s; "
          f"kernels {train['kernel_ms_per_step']:.3f} ms of GPU time, {train['kernels_per_step']:.0f} kernels per step "
          f"({train['library_launches_per_step']} of them this library's); "
          f"host-bound by {train['ms_per_step'] / train['kernel_ms_per_step']:.1f}x", flush=True)
    print(f"  wall time: forward {train['forward_ms']:.3f} ms, forward + loss + backward (with zero_grad) "
          f"{train['forward_backward_ms']:.3f} ms, so clip and Adam "
          f"{train['ms_per_step'] - train['forward_backward_ms']:.3f} ms")
    print(f"  torch arm (784 nn.Linear, torch.optim.Adam): wall {train['torch_ms_per_step']:.1f} ms "
          f"({train['torch_ms_per_step'] / train['ms_per_step']:.0f}x), kernels {train['torch_kernel_ms_per_step']:.2f} ms, "
          f"{train['torch_kernels_per_step']:.0f} kernels per step")
    for what, f in step_flops().items():
        print(f"  {f / 1e9:8.3f} GFLOP  {what}")
    for what, nbytes in step_bytes().items():
        print(f"  {nbytes / 1e6:8.2f} MB  {what}")
    print(f"  {train['step_flops'] / 1e9:.3f} GFLOP and {train['step_bytes'] / 1e6:.1f} MB per step: at least "
          f"{1e3 * train['bound_ms']:.1f} us ({train['bound']}-bound at the data-sheet rates); the kernels took "
          f"{1e3 * train['kernel_ms_per_step']:.1f} us, the step {1e3 * train['ms_per_step']:.1f} us")
    sampling = bench_sample(model, ref, args.reps)
    for k, v in sampling.items():
        print(f"{k}: {v['cuda_ms_min']:.2f} ms (runs {', '.join(f'{t:.2f}' for t in v['cuda_ms_all'])}), torch arm "
              f"{v['torch_ms']:.0f} ms ({v['torch_ms'] / v['cuda_ms_min']:.0f}x)")
    result = dict(gpu=gpu, train=train, sampling=sampling)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
