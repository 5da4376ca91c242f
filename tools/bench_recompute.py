"""ImageGPT C5 training steps (24 blocks, 8 heads, 512 channels, batch 64) with every activation kept against the
recompute path, and at 64x64 under the model's own memory rule.

    python tools/bench_recompute.py [--steps 20] [--warmup 3] [--rounds 4] [--steps-64 10]

1. 32x32: the store path against forced recompute, alternating in --rounds segments, --steps timed steps per path.
2. 64x64: the automatic rule (models.image_gpt.recompute_activations); the run stops unless it picks recompute.
Each run prints ms per step (CUDA events), images/s and torch.cuda.max_memory_allocated.  The card's name and power
limit are printed first."""
import argparse
import gc
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from pytorch_generative_b200 import losses, models, optim
from pytorch_generative_b200.models import image_gpt

dev = torch.device("cuda:0")
C5 = dict(in_channels=3, out_channels=3, n_transformer_blocks=24, n_attention_heads=8, n_embedding_channels=512)
BATCH = 64
AUTOMATIC = image_gpt.recompute_activations


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(dev.index or 0)], capture_output=True, text=True, timeout=10).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or f"{torch.cuda.get_device_name(dev)}, power limit unknown (nvidia-smi unavailable)"


def force(recompute):
    """None: the model's own rule; True / False: that path for every training forward."""
    image_gpt.recompute_activations = AUTOMATIC if recompute is None else (lambda mem, available: recompute)


def make(side):
    torch.manual_seed(0)
    m = models.ImageGPT(in_size=side, **C5).to(dev).train()
    g = torch.Generator().manual_seed(0)
    x = (torch.randint(0, 256, (BATCH, 3, side, side), generator=g).float() / 255).to(dev)
    return m, optim.FusedAdam(m.parameters(), lr=5e-3), x


def step(m, opt, x):
    opt.zero_grad()
    losses.bce_with_logits_sum_mean(m(x), x).backward()
    opt.clip_and_step(1e50)


def timed(m, opt, x, steps):
    """(ms per step, max_memory_allocated in bytes) over `steps` steps."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step(m, opt, x)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, torch.cuda.max_memory_allocated(dev)


def report(label, ms, peak):
    print(f"{label}: {ms:.1f} ms/step, {BATCH / (ms / 1e3):.1f} images/s, max_memory_allocated {peak / 2**30:.2f} GiB",
          flush=True)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--steps", type=int, default=20, help="timed steps per path at 32x32 (at least --rounds)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps-64", type=int, default=10, help="timed steps at 64x64")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_recompute.py needs a CUDA device")
    capacity = torch.cuda.get_device_properties(dev).total_memory
    print(f"GPU (name, power limit): {card()}; {capacity / 2**30:.1f} GiB", flush=True)

    # ---- 32x32: store against forced recompute, alternating ----
    m, opt, x = make(32)
    paths = {"store": False, "recompute": True}
    per_round = max(1, args.steps // args.rounds)
    for recompute in paths.values():
        force(recompute)
        for _ in range(args.warmup):
            step(m, opt, x)
    times = {p: [] for p in paths}
    peaks = {p: 0 for p in paths}
    for _ in range(args.rounds):
        for p, recompute in paths.items():
            force(recompute)
            ms, peak = timed(m, opt, x, per_round)
            times[p].append(ms)
            peaks[p] = max(peaks[p], peak)
    for p in paths:
        ms = sum(times[p]) / len(times[p])
        report(f"C5 32x32 batch {BATCH} {p:9s} ({per_round * args.rounds} steps, per-round "
               f"{min(times[p]):.1f}-{max(times[p]):.1f} ms)", ms, peaks[p])
    store_ms, rec_ms = (sum(times[p]) / len(times[p]) for p in paths)
    print(f"recompute costs {100 * (rec_ms / store_ms - 1):.1f} % per step at 32x32", flush=True)
    force(None)
    print(f"automatic rule at 32x32 picks: {'recompute' if m._recompute_for(x) else 'store'}", flush=True)
    del m, opt, x
    gc.collect()
    torch.cuda.empty_cache()

    # ---- 64x64 under the automatic rule ----
    m, opt, x = make(64)
    est = image_gpt.activation_memory(BATCH * 64 * 64, 512, 8, 64, 64, C5["n_transformer_blocks"])
    free, _ = torch.cuda.mem_get_info(dev)
    print(f"C5 64x64 batch {BATCH}: the store path would keep {est.store / 1e9:.1f} GB (+ {est.backward / 1e9:.1f} GB "
          f"for one block's backward), recompute keeps {est.recompute / 1e9:.1f} GB; driver free memory "
          f"{free / 1e9:.1f} GB", flush=True)
    if not m._recompute_for(x):
        sys.exit("the automatic rule picked the store path at 64x64: not running it")
    print("automatic rule at 64x64 picks: recompute", flush=True)
    for _ in range(args.warmup):
        step(m, opt, x)
    ms, peak = timed(m, opt, x, args.steps_64)
    report(f"C5 64x64 batch {BATCH} automatic ({args.steps_64} steps)", ms, peak)
    print(f"peak {peak / 2**30:.2f} GiB of {capacity / 2**30:.1f} GiB", flush=True)


if __name__ == "__main__":
    main()
