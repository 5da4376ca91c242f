"""VeryDeepVAE at its recipe size (stacks (3,5), (3,5), (2,4), (2,3), (2,2), (1,1); latent 16, hidden 64, bottleneck
32) on Bernoulli(0.5) 1x32x32 batches of 128: the training step, eager and under `trainstep.GraphedTrainStep`, against a
plain-torch fp32 arm of the same network in the same run (the reference's modules: nn.Conv2d on cuDNN with TF32 off,
nn.GELU, torch's BCE and torch.optim.Adam), and sample(64).

    python tools/bench_vd_vae.py [--steps 30] [--warmup 5] [--reps 3]

Training step: Trainer._train_one_batch's work (zero_grad, forward, recipe loss, backward, clip to 1e50 and Adam), timed
with a device synchronise around `--steps` steps (wall time per step), `--reps` times.  The kernels this library
launches per step are counted, and the step's FLOPs (forward and both backward contractions of every convolution) are
computed from the shapes.  The card's name, power limit and SM clock are read in the same run and printed with the
numbers."""
import argparse
import copy
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

from pytorch_generative_b200 import _lib, losses, models, optim, trainstep

from pytorch_generative_b200.models.vd_vae import StackConfig

STACKS = [(3, 5), (3, 5), (2, 4), (2, 3), (2, 2), (1, 1)]
CFG = dict(in_channels=1, out_channels=1, input_resolution=32, latent_channels=16, hidden_channels=64,
           bottleneck_channels=32)
BATCH, SIDE = 128, 32


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unavailable ({e})"


def step_flops(model, n=BATCH, side=SIDE):
    """2 * MACs of every convolution's forward, times 3 (forward, input gradient, weight gradient), from the shapes
    (the first layer's input gradient is not needed but counted: an upper bound by a fraction of a percent)."""
    macs = 0

    def hook(mod, inp, out):
        nonlocal macs
        w = mod.weight
        macs += out.numel() * w.shape[1] * w.shape[2] * w.shape[3]
    hs = [m.register_forward_hook(hook) for m in model.modules() if isinstance(m, nn.Conv2d)]
    with torch.no_grad():
        torch_forward(model, torch.zeros(n, 1, side, side))
    for h in hs:
        h.remove()
    return 3 * 2 * macs


def torch_forward(model, x):
    """The reference's forward on this package's module tree (the holders are plain nn modules)."""
    def block(b, x, residual):
        h = b._net(x)
        return x + h if residual else h

    n = x.shape[0]
    x = model._input(x)
    mixins = []
    for stack in model._encoder:
        for b in stack._residuals:
            x = block(b, x, True)
        mixins.append(x)
        if stack._pool is not None:
            x = stack._pool(x)
    x = torch.zeros_like(model._biases[-1]).repeat(n, 1, 1, 1)
    kl = torch.zeros(n, device=x.device)
    for stack, mixin, bias in zip(model._decoder, reversed(mixins), reversed(model._biases)):
        x = x + bias.repeat(n, 1, 1, 1)
        if stack._unpool is not None:
            x = stack._unpool(x)
        for td in stack._topdowns:
            L = td._latent_channels
            p_mean, p_log_std, p_h = torch.split(block(td._prior, x, False), [L, L, td._n_channels], dim=1)
            q_mean, q_log_std = torch.split(block(td._posterior, torch.cat((x, mixin), dim=1), False), L, dim=1)
            z = q_mean + q_log_std.exp() * torch.randn_like(q_log_std)
            div = -0.5 + (p_log_std - q_log_std) + (q_log_std.exp().pow(2) + (q_mean - p_mean) ** 2) / (
                2 * p_log_std.exp().pow(2))
            kl = kl + div.sum(dim=(1, 2, 3))
            x = block(td._out, x + p_h + td._latents(z), True)
    return model._output(x), kl


def torch_loss(x, preds):
    logits, kl = preds
    recon = F.binary_cross_entropy_with_logits(logits, x, reduction="none").sum(dim=(1, 2, 3))
    return (recon + kl).mean()


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(steps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) / steps * 1e3


class _Preds(tuple):
    def detach(self):
        return _Preds(t.detach() for t in self)


class _TupleModel(nn.Module):
    def __init__(self, vae):
        super().__init__()
        self.vae = vae

    def forward(self, x):
        return _Preds(self.vae(x))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vd_vae: needs a CUDA device")
    dev = torch.device("cuda")
    torch.manual_seed(0)
    model = models.VeryDeepVAE(stack_configs=[StackConfig(*s) for s in STACKS], **CFG).to(dev)
    ref_model = copy.deepcopy(model)
    x = torch.bernoulli(torch.full((BATCH, 1, SIDE, SIDE), 0.5, device=dev))
    opt = optim.FusedAdam(model.parameters(), lr=5e-4)

    def eager_step():
        opt.zero_grad()
        losses.vae_elbo(x, None, model(x))["loss"].backward()
        opt.clip_and_step(1e50)

    ref_params = list(ref_model.parameters())
    ref_opt = torch.optim.Adam(ref_params, lr=5e-4)

    def torch_step():
        ref_opt.zero_grad()
        torch_loss(x, torch_forward(ref_model, x)).backward()
        torch.nn.utils.clip_grad_norm_(ref_params, 1e50)
        ref_opt.step()

    graphed_model = _TupleModel(copy.deepcopy(model))
    graphed = trainstep.GraphedTrainStep(graphed_model, graphed_model.parameters(),
                                         lambda p, xx: losses.vae_elbo(xx, None, p)["loss"], x, lr=5e-4, lr_gamma=1.0)
    prev = torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32
    out = {"card": card(), "config": dict(CFG, stacks=STACKS), "batch": BATCH, "side": SIDE, "steps": args.steps}
    runs = {"eager_ms": [], "graphed_ms": [], "torch_ms": [], "sample64_ms": []}
    for _ in range(args.reps):
        runs["eager_ms"].append(timed(eager_step, args.steps, args.warmup))
        runs["graphed_ms"].append(timed(lambda: graphed(x), args.steps, args.warmup))
        torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
        try:
            runs["torch_ms"].append(timed(torch_step, args.steps, args.warmup))
        finally:
            torch.backends.cudnn.allow_tf32, torch.backends.cuda.matmul.allow_tf32 = prev
        runs["sample64_ms"].append(timed(lambda: model.sample(64), args.steps, args.warmup))
    out.update(runs)
    before = _lib.launch_count()
    eager_step()
    torch.cuda.synchronize()
    out["library_launches_per_step"] = _lib.launch_count() - before
    out["step_gflop"] = step_flops(copy.deepcopy(model).cpu()) / 1e9
    out["card_after"] = card()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
