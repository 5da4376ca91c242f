"""Times the 256-way categorical likelihood of 8-bit images.

1. `losses.categorical_nll` forward + backward (`pg_categorical_xent_fwd_bwd`, then a scale of the saved dlogits) on
   [64, 768, 32, 32] fp32 logits against `F.cross_entropy(reduction="sum") / N` + backward, and the loss kernel alone.
   Bytes are computed from the shapes, not measured: the kernel reads the logits twice and writes dlogits once
   (3 x 201 MB).
2. The ImageGPT C5 training step (24 blocks, 8 heads, 512 channels, batch 64, FusedAdam / the graphed step's Adam) with
   the 768-way head and `categorical_nll` against the 3-channel head and `bce_with_logits_sum_mean`, eager and as a
   `GraphedTrainStep`.  The two heads alternate within each phase.

The arms alternate in rounds after a warm-up and the medians over rounds are printed with the card's name and power
limit, one JSON line per number.

    python tools/bench_categorical.py [--steps 20] [--rounds 5] [--skip-step]
"""

import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.nn.functional as F

from pytorch_generative_b200 import _lib as L
from pytorch_generative_b200 import losses, models, optim, trainstep

C5 = dict(in_channels=3, in_size=32, n_transformer_blocks=24, n_attention_heads=8, n_embedding_channels=512)
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                        "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def timed_ms(fn, steps):
    """Milliseconds per call of `fn` over `steps` calls, between CUDA events."""
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def alternate(arms, steps, rounds):
    """{name: median ms per call} with the arms run in turn, `rounds` times, after one untimed call of each."""
    for fn in arms.values():
        fn()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(timed_ms(fn, steps))
    return {k: statistics.median(v) for k, v in times.items()}


def emit(gpu, **kw):
    print(json.dumps({"gpu": gpu, **kw}), flush=True)


def loss_arms(x, logits):
    n, c = x.shape[:2]
    K = logits.shape[1] // c
    target = losses.categorical_target(x, K)
    leaf = logits.detach().requires_grad_(True)
    nll, image_nll, dl = torch.empty(x.shape, device=x.device), torch.zeros(n, device=x.device), torch.empty_like(logits)

    def fused():
        leaf.grad = None
        losses.categorical_nll(x, None, leaf)["loss"].backward()

    def torch_ce():
        leaf.grad = None
        (F.cross_entropy(leaf.view(n, K, c, *x.shape[2:]), target, reduction="sum") / n).backward()

    def kernel():
        L.categorical_xent(logits, x, 1.0 / n, image_nll=image_nll, dlogits=dl)

    return dict(fused=fused, torch_cross_entropy=torch_ce, kernel_only=kernel)


def step_arms(x, graphed):
    """{head: one training step} for the 768-way categorical head and the 3-channel BCE head."""
    arms = {}
    for head, out_channels, loss_fn in (("categorical_768", 768, lambda p, xx: losses.categorical_nll(xx, None, p)["loss"]),
                                        ("bce_3", 3, lambda p, xx: losses.bce_with_logits_sum_mean(p, xx))):
        torch.manual_seed(0)
        m = models.ImageGPT(out_channels=out_channels, **C5).to(x.device).train()
        params = list(m.parameters())
        if graphed:
            g = trainstep.GraphedTrainStep(m, params, loss_fn, x, lr=5e-3, lr_gamma=0.999977)
            arms[head] = lambda g=g: g.graph.replay()
        else:
            opt = optim.FusedAdam(params, lr=5e-3)

            def step(m=m, opt=opt, loss_fn=loss_fn):
                opt.zero_grad()
                loss_fn(m(x), x).backward()
                opt.clip_and_step(1e50)

            arms[head] = step
    return arms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--skip-step", action="store_true", help="time the loss only")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_categorical.py needs a CUDA device")
    L.load()
    gpu = card()
    dev = torch.device("cuda", torch.cuda.current_device())
    g = torch.Generator().manual_seed(0)
    n = args.batch
    x = (torch.randint(0, 256, (n, 3, 32, 32), generator=g).float() / 255).to(dev)
    logits = torch.randn(n, 768, 32, 32, generator=g).to(dev)

    ms = alternate(loss_arms(x, logits), args.steps * 5, args.rounds)
    bytes_moved = 3 * logits.numel() * 4
    emit(gpu, what=f"loss + backward [{n}, 768, 32, 32]", ms=ms,
         kernel_hbm_bound_ms=bytes_moved / HBM_BYTES_PER_S * 1e3, kernel_bytes=bytes_moved,
         kernel_gbs=bytes_moved / (ms["kernel_only"] * 1e-3) / 1e9)
    del logits
    if args.skip_step:
        return
    for graphed in (False, True):
        arms = step_arms(x, graphed)
        ms = alternate(arms, args.steps, args.rounds)
        emit(gpu, what=f"ImageGPT C5 step, batch {n}, {'graphed' if graphed else 'eager'}", ms=ms,
             images_per_s={k: n / (v * 1e-3) for k, v in ms.items()},
             head_overhead=ms["categorical_768"] / ms["bce_3"] - 1)
        del arms
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
