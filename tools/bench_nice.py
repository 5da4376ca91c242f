"""NICE at its recipe size, NICE(784, 4 coupling blocks, 5 hidden layers, 1000 units) on dequantised 28x28 images at
batch 1024: the training step, eager and under `trainstep.GraphedTrainStep`, and sample(16) / sample(1024), each
against a plain-torch arm in the same run (the reference's scheme written out here: nn.Linear / nn.ReLU coupling MLPs,
torch's softplus loss and torch.optim.Adam, all fp32 with torch's default matmul precision, i.e. TF32 off).

    python tools/bench_nice.py [--steps 30] [--warmup 5] [--reps 3] [--out results.json]

Training step: Trainer._train_one_batch's work (zero_grad, forward, recipe loss, backward, clip to 1e50 and Adam),
timed with a device synchronise around `--steps` steps (wall time per step), `--reps` times.  A separate pass brackets
every GEMM launch of one step with CUDA events and reports the GPU time per GEMM shape; the kernels launched by this
library per step and the step's peak torch allocation are counted too.  The GEMM FLOPs are counted from the shapes and
set against the H100 SXM data sheet's 989 TFLOP/s dense bf16.  The card's name, power limit and SM clock are printed
with the numbers."""
import argparse
import collections
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

BF16_FLOPS = 989e12  # H100 SXM data sheet, dense bf16
CFG = dict(n_features=784, n_coupling_blocks=4, n_hidden_layers=5, n_hidden_features=1000)
BATCH = 1024


def widths():
    return [CFG["n_features"] // 2] + [CFG["n_hidden_features"]] * CFG["n_hidden_layers"] + [CFG["n_features"] // 2]


def step_flops(n=BATCH):
    """GEMM FLOPs of one training step: forward, dgrad (block 0's first layer has no input gradient to give) and wgrad."""
    w = widths()
    per_block = sum(2 * n * a * b for a, b in zip(w[:-1], w[1:]))
    first = 2 * n * w[0] * w[1]
    return 3 * CFG["n_coupling_blocks"] * per_block - first


def card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()),
                        "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or torch.cuda.get_device_name()


def timed(fn, count):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(count):
        fn(i)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / count


class TorchNICE(nn.Module):
    """The torch arm: the reference's coupling MLPs and scaling, plain nn modules."""

    def __init__(self):
        super().__init__()
        d, h, layers = CFG["n_features"] // 2, CFG["n_hidden_features"], CFG["n_hidden_layers"]
        self.nets = nn.ModuleList()
        for _ in range(CFG["n_coupling_blocks"]):
            net = [nn.Linear(d, h), nn.ReLU()]
            for _ in range(layers - 1):
                net += [nn.Linear(h, h), nn.ReLU()]
            self.nets.append(nn.Sequential(*net, nn.Linear(h, d)))
        self.log_scale = nn.Parameter(torch.zeros(1, 2 * d))

    def _couple(self, x, sign):
        d = x.shape[1] // 2
        blocks = list(enumerate(self.nets))
        for b, net in (blocks if sign > 0 else reversed(blocks)):
            h1, h2 = x[:, :d], x[:, d:]
            if b % 2:
                h1 = h1 + sign * net(h2)
            else:
                h2 = h2 + sign * net(h1)
            x = torch.cat((h1, h2), 1)
        return x

    def forward(self, x):
        z = self._couple(x.view(x.shape[0], -1), 1) * torch.exp(self.log_scale)
        return z.view(x.shape), self.log_scale.sum()

    @torch.no_grad()
    def sample(self, n):
        z = torch.randn((n, 784)).to(self.log_scale.device) * torch.exp(-self.log_scale)
        return self._couple(z, -1).view(n, 1, 28, 28)


def torch_loss(preds):
    z, log_det = preds
    log_prob = -(F.softplus(z) + F.softplus(-z)).sum(dim=(1, 2, 3))
    return -(log_prob + log_det).mean()


class _Preds(tuple):
    """(z, log_det_J) with the .detach() GraphedTrainStep applies to a model's output."""

    def detach(self):
        return _Preds(t.detach() for t in self)


class _TupleModel(nn.Module):
    def __init__(self, nice):
        super().__init__()
        self.nice = nice

    def forward(self, x):
        return _Preds(self.nice(x))


def _graph_loss(preds, x):
    return losses.logistic_prior_nll(x, None, preds)["loss"]


def gemm_times(step):
    """GPU time per GEMM shape over one step: every _lib.gemm launch bracketed by CUDA events."""
    orig, events = _lib.gemm, []

    def gemm(A, B, M, N, K, **kw):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        orig(A, B, M, N, K, **kw)
        e1.record()
        kind = "wgrad" if kw.get("a_mn") else ("dgrad" if kw.get("b_mn") else "fwd")
        events.append(((kind, M, N, K, kw.get("split_k", 1)), e0, e1))

    _lib.gemm = gemm
    try:
        step(0)
        torch.cuda.synchronize()
    finally:
        _lib.gemm = orig
    per = collections.OrderedDict()
    for key, e0, e1 in events:
        t = per.setdefault(" ".join(map(str, key)), [0, 0.0])
        t[0] += 1
        t[1] += e0.elapsed_time(e1)
    return {k: {"launches": c, "ms": round(ms, 4)} for k, (c, ms) in per.items()}


def bench(steps, warmup, reps):
    dev = torch.device("cuda:0")
    torch.manual_seed(0)
    model = models.NICE(**CFG).to(dev)
    ref = TorchNICE().to(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    batches = [(torch.randint(0, 256, (BATCH, 1, 28, 28), device=dev, generator=g).float()
                + torch.rand((BATCH, 1, 28, 28), device=dev, generator=g)) / 256 for _ in range(4)]
    opt = optim.FusedAdam(model.parameters(), lr=1e-3)
    ref_opt = torch.optim.Adam(ref.parameters(), lr=1e-3)

    def step(i):
        x = batches[i % 4]
        opt.zero_grad()
        losses.logistic_prior_nll(x, None, model(x))["loss"].backward()
        opt.clip_and_step(1e50)

    def ref_step(i):
        x = batches[i % 4]
        ref_opt.zero_grad()
        torch_loss(ref(x)).backward()
        torch.nn.utils.clip_grad_norm_(ref.parameters(), 1e50)
        ref_opt.step()

    graphed_model = _TupleModel(copy.deepcopy(model))
    graphed = trainstep.GraphedTrainStep(graphed_model, graphed_model.parameters(), _graph_loss, batches[0], lr=1e-3,
                                         lr_gamma=1.0)

    out = {"card": card(), "batch": BATCH, "steps": steps, "reps": reps,
           "step_gemm_gflop": step_flops() / 1e9,
           "gemm_floor_ms_at_989_tflops": step_flops() / BF16_FLOPS * 1e3}
    for fn in (step, ref_step, lambda i: graphed(batches[i % 4])):
        timed(fn, warmup)
    for name, fn in (("step_eager_ms", step), ("step_graphed_ms", lambda i: graphed(batches[i % 4])),
                     ("torch_step_ms", ref_step)):
        out[name] = [round(timed(fn, steps), 3) for _ in range(reps)]
    torch.cuda.synchronize()
    before = _lib.launch_count()
    step(0)
    torch.cuda.synchronize()
    out["library_launches_per_step"] = _lib.launch_count() - before
    torch.cuda.reset_peak_memory_stats()
    for i in range(3):
        step(i)
    torch.cuda.synchronize()
    out["step_peak_allocated_mb"] = round(torch.cuda.max_memory_allocated() / 2 ** 20, 1)
    out["gemm_ms_per_shape"] = gemm_times(step)
    out["gemm_ms_total"] = round(sum(v["ms"] for v in out["gemm_ms_per_shape"].values()), 4)
    model.eval()
    for n in (16, 1024):
        timed(lambda i: model.sample(n), 2)
        timed(lambda i: ref.sample(n), 2)
        out[f"sample{n}_ms"] = [round(timed(lambda i: model.sample(n), 10), 3) for _ in range(reps)]
        out[f"torch_sample{n}_ms"] = [round(timed(lambda i: ref.sample(n), 10), 3) for _ in range(reps)]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_nice.py measures on a GPU; none is available")
    result = bench(args.steps, args.warmup, args.reps)
    print(json.dumps(result, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
