"""Times `optim.AdaBelief.clip_and_step` over ImageGPT C5's parameter set (75,677,187 fp32 parameters, on the GPU)
against the corrected reference step restated with torch ops (per parameter, as the reference loops) and a
`torch._foreach_*` version of the same arithmetic.  The arms alternate in one run after a warm-up; each arm owns its
own copy of the parameters, gradients and moments.  `--rezero` also times forward + backward of
ReZeroWrapper(Identity) on a 64x512x32x32 fp32 tensor against torch's `x + alpha * f` under autograd.

Bytes are computed from the shapes, not measured: the norm pass reads g (4 B / parameter), the update reads p, g, m, v
and writes p, m, v (28 B / parameter, plus 4 B when clipping writes g back).  The card's name and power limit are
printed with the numbers.

    python tools/bench_adabelief.py [--steps 20] [--rounds 5] [--rezero]
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

from pytorch_generative_b200 import models, nn, optim

C5 = dict(in_channels=3, out_channels=3, in_size=32, n_transformer_blocks=24, n_attention_heads=8,
          n_embedding_channels=512)
HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                        "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def reference_step(params, states, lr, beta1, beta2):
    """The reference's AdaBelief.step with its unpack corrected, one parameter at a time."""
    for p, st in zip(params, states):
        st["step"] += 1
        m, v = st["ema_avg"], st["ema_var"]
        m.mul_(beta1).add_(p.grad, alpha=1 - beta1)
        e = p.grad - m
        v.mul_(beta2).addcmul_(e, e, value=1 - beta2).add_(1e-10)
        m_hat = m / (1 - beta1 ** st["step"])
        v_hat = v / (1 - beta2 ** st["step"])
        p.data.addcdiv_(-m_hat, v_hat.sqrt() + 1e-10, value=lr)


def foreach_step(params, states, lr, beta1, beta2):
    """The same arithmetic with torch._foreach_* over all parameters at once."""
    step = states[0]["step"] = states[0]["step"] + 1
    grads = [p.grad for p in params]
    ms, vs = [s["ema_avg"] for s in states], [s["ema_var"] for s in states]
    torch._foreach_mul_(ms, beta1)
    torch._foreach_add_(ms, grads, alpha=1 - beta1)
    es = torch._foreach_sub(grads, ms)
    torch._foreach_mul_(vs, beta2)
    torch._foreach_addcmul_(vs, es, es, value=1 - beta2)
    torch._foreach_add_(vs, 1e-10)
    m_hat = torch._foreach_div(ms, 1 - beta1 ** step)
    denom = torch._foreach_sqrt(torch._foreach_div(vs, 1 - beta2 ** step))
    torch._foreach_add_(denom, 1e-10)
    torch._foreach_neg_(m_hat)
    torch._foreach_addcdiv_([p.data for p in params], m_hat, denom, value=lr)


def time_ms(fn, steps):
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    end.record()
    torch.cuda.synchronize()
    return start.elapsed_time(end) / steps


def bench_optimizer(args):
    shapes = [p.shape for p in models.ImageGPT(**C5).parameters()]
    n_params = sum(s.numel() for s in shapes)
    g = torch.Generator(device="cuda").manual_seed(0)

    def fresh():
        ps = [torch.nn.Parameter(torch.randn(s, device="cuda", generator=g)) for s in shapes]
        for p in ps:
            p.grad = torch.randn(p.shape, device="cuda", generator=g) * 1e-3
        return ps

    ours_p = fresh()
    ours = optim.AdaBelief(ours_p, lr=1e-4)
    torch_states = {}
    arms = {"AdaBelief.clip_and_step": lambda: ours.clip_and_step()}
    for name, fn in (("reference per-parameter", reference_step), ("torch._foreach", foreach_step)):
        ps = fresh()
        sts = [{"step": 0, "ema_avg": torch.zeros_like(p), "ema_var": torch.zeros_like(p)} for p in ps]
        torch_states[name] = sts
        arms[name] = (lambda fn=fn, ps=ps, sts=sts: fn(ps, sts, 1e-4, 0.9, 0.999))
    for fn in arms.values():  # warm-up
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, fn in arms.items():
            times[k].append(time_ms(fn, args.steps))
    moved = n_params * (4 + 28)
    out = dict(card=card(), parameters=n_params, bytes_per_step=moved, hbm_bound_ms=moved / HBM_BYTES_PER_S * 1e3,
               steps_per_round=args.steps, rounds=args.rounds,
               ms_per_step={k: dict(median=statistics.median(v), min=min(v), max=max(v)) for k, v in times.items()})
    return out


def bench_rezero(args):
    x = torch.randn(64, 512, 32, 32, device="cuda", requires_grad=True)
    dy = torch.randn_like(x)
    w = nn.ReZeroWrapper(torch.nn.Identity()).cuda()
    with torch.no_grad():
        w._alpha.fill_(0.5)
    alpha = torch.nn.Parameter(torch.tensor([0.5], device="cuda"))

    def ours():
        torch.autograd.backward(w(x), dy)

    def plain():
        torch.autograd.backward(x + alpha * x, dy)

    arms = {"ReZeroWrapper": ours, "torch x + alpha * f": plain}
    for fn in arms.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, fn in arms.items():
            x.grad = None
            times[k].append(time_ms(fn, args.steps))
    return dict(card=card(), shape=list(x.shape),
                ms_per_fwd_bwd={k: dict(median=statistics.median(v), min=min(v), max=max(v)) for k, v in times.items()})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--rezero", action="store_true")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_adabelief.py measures on a GPU; none is available")
    result = dict(adabelief=bench_optimizer(args))
    if args.rezero:
        result["rezero"] = bench_rezero(args)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
