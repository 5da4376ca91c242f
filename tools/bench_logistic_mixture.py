"""Times the discretised logistic mixture likelihood of 8-bit images.

1. `losses.logistic_mixture_nll` forward + backward (`pg_logistic_mixture_fwd_bwd`, then a scale of the saved dpreds)
   on [64, 100, 32, 32] fp32 parameters (10 components, RGB) against the same loss written in torch ops under autograd,
   and the loss kernel alone.  Bytes are computed from the shapes, not measured: the kernel reads the parameters twice,
   the input once and writes dpreds once.
2. A PixelSNAIL training step at `reproduce_pixel_snail`'s network (64 channels, 8 blocks) on 3 x 32 x 32 images,
   batch 64, with the 100-channel mixture head and `logistic_mixture_nll` against the 768-way categorical head and
   `categorical_nll`, eager (FusedAdam) and as a `GraphedTrainStep`.  The two heads alternate within each phase.
3. `sample()` of that PixelSNAIL with `logistic_mixture_sample_fn`, per pixel.

The arms alternate in rounds after a warm-up and the medians over rounds are printed with the card's name and power
limit, one JSON line per number.

    python tools/bench_logistic_mixture.py [--steps 10] [--rounds 5] [--skip-step] [--skip-sample]
"""

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import torch.nn.functional as F

from pytorch_generative_b200 import _lib as L
from pytorch_generative_b200 import losses, models, optim, trainstep

SNAIL = dict(in_channels=3, n_channels=64, n_pixel_snail_blocks=8, n_residual_blocks=2, attention_value_channels=32,
             attention_key_channels=4)
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


def torch_dmol(preds, x, M, K=256):
    """The same loss in torch ops (fp32, autograd): the layout and exact bin mass of `losses.logistic_mixture_nll`."""
    n, C = x.shape[:2]
    T = C * (C - 1) // 2
    pi = preds[:, :M]
    mu = preds[:, M:M + M * C].unflatten(1, (M, C))
    ls = preds[:, M + M * C:M + 2 * M * C].unflatten(1, (M, C)).clamp(min=-7.0)
    r = torch.tanh(preds[:, M + 2 * M * C:].unflatten(1, (M, T)))
    k = losses.categorical_target(x, K)
    xc = (2.0 * k.float() / (K - 1) - 1.0).unsqueeze(1)
    means = [mu[:, :, 0]]
    for c in range(1, C):
        means.append(mu[:, :, c] + sum(r[:, :, c * (c - 1) // 2 + j] * xc[:, :, j] for j in range(c)))
    mup = torch.stack(means, dim=2)
    inv = torch.exp(-ls)
    h = 1.0 / (K - 1)
    a, b = inv * (xc - mup + h), inv * (xc - mup - h)
    kk = k.unsqueeze(1)
    mid = -F.softplus(-a) - F.softplus(b) + torch.log(-torch.expm1(-2 * h * inv))
    lp = torch.where(kk == 0, -F.softplus(-a), torch.where(kk == K - 1, -F.softplus(b), mid))
    nll = torch.logsumexp(pi, dim=1) - torch.logsumexp(pi + lp.sum(dim=2), dim=1)
    return nll.sum() / n


def loss_arms(x, preds, M):
    n = x.shape[0]
    leaf = preds.detach().requires_grad_(True)
    image_nll, dp = torch.zeros(n, device=x.device), torch.empty_like(preds)

    def fused():
        leaf.grad = None
        losses.logistic_mixture_nll(x, None, leaf)["loss"].backward()

    def torch_ops():
        leaf.grad = None
        torch_dmol(leaf, x, M).backward()

    def kernel():
        L.logistic_mixture_nll_kernel(preds, x, M, 256, 1.0 / n, image_nll=image_nll, dpreds=dp)

    return dict(fused=fused, torch_ops=torch_ops, kernel_only=kernel)


def step_arms(x, graphed):
    """{head: one training step} for the 100-channel mixture head and the 768-way categorical head."""
    arms = {}
    for head, out_channels, loss_fn in (
            ("logistic_mixture_100", 100, lambda p, xx: losses.logistic_mixture_nll(xx, None, p)["loss"]),
            ("categorical_768", 768, lambda p, xx: losses.categorical_nll(xx, None, p)["loss"])):
        torch.manual_seed(0)
        m = models.PixelSNAIL(out_channels=out_channels, **SNAIL).to(x.device).train()
        params = list(m.parameters())
        if graphed:
            g = trainstep.GraphedTrainStep(m, params, loss_fn, x, lr=1e-3, lr_gamma=0.999977)
            arms[head] = lambda g=g: g.graph.replay()
        else:
            opt = optim.FusedAdam(params, lr=1e-3)

            def step(m=m, opt=opt, loss_fn=loss_fn):
                opt.zero_grad()
                loss_fn(m(x), x).backward()
                opt.clip_and_step(1e50)

            arms[head] = step
    return arms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--skip-step", action="store_true", help="do not time the training steps")
    ap.add_argument("--skip-sample", action="store_true", help="do not time sample()")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_logistic_mixture.py needs a CUDA device")
    L.load()
    gpu = card()
    dev = torch.device("cuda", torch.cuda.current_device())
    g = torch.Generator().manual_seed(0)
    n, M = args.batch, 10
    x = (torch.randint(0, 256, (n, 3, 32, 32), generator=g).float() / 255).to(dev)
    preds = torch.cat([torch.randn(n, M, 32, 32, generator=g), torch.randn(n, 3 * M, 32, 32, generator=g) * 0.5,
                       torch.rand(n, 3 * M, 32, 32, generator=g) * 4 - 5,
                       torch.randn(n, 3 * M, 32, 32, generator=g)], dim=1).to(dev)

    ms = alternate(loss_arms(x, preds, M), args.steps * 5, args.rounds)
    read = preds.numel() * 4
    bytes_one_read = read + x.numel() * 4 + read
    bytes_two_reads = bytes_one_read + read
    emit(gpu, what=f"loss + backward [{n}, 100, 32, 32]", ms=ms, kernel_bytes_two_reads=bytes_two_reads,
         kernel_hbm_bound_ms_one_read=bytes_one_read / HBM_BYTES_PER_S * 1e3,
         kernel_hbm_bound_ms_two_reads=bytes_two_reads / HBM_BYTES_PER_S * 1e3,
         kernel_gbs_two_reads=bytes_two_reads / (ms["kernel_only"] * 1e-3) / 1e9)
    del preds
    if not args.skip_step:
        for graphed in (False, True):
            try:
                arms = step_arms(x, graphed)
            except RuntimeError as exc:  # reported, not hidden: the eager numbers stand on their own
                emit(gpu, what=f"PixelSNAIL step, batch {n}, {'graphed' if graphed else 'eager'}", error=repr(exc))
                continue
            ms = alternate(arms, args.steps, args.rounds)
            emit(gpu, what=f"PixelSNAIL step, batch {n}, {'graphed' if graphed else 'eager'}", ms=ms,
                 images_per_s={k: n / (v * 1e-3) for k, v in ms.items()},
                 mixture_over_categorical=ms["logistic_mixture_100"] / ms["categorical_768"] - 1)
            del arms
            torch.cuda.empty_cache()
    if not args.skip_sample:
        torch.manual_seed(0)
        m = models.PixelSNAIL(out_channels=100, sample_fn=models.logistic_mixture_sample_fn(10, 256), **SNAIL)
        m = m.to(dev).eval()
        m(x[:1])
        times = []
        for _ in range(3):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            s = m.sample(n_samples=16)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        assert s.shape == (16, 3, 32, 32)
        emit(gpu, what="PixelSNAIL sample(n_samples=16), 32 x 32, logistic_mixture_sample_fn",
             s_per_call=statistics.median(times[1:]), us_per_pixel=statistics.median(times[1:]) / 1024 * 1e6)


if __name__ == "__main__":
    main()
