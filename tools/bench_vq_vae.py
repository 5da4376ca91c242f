"""VQ-VAE and VQ-VAE-2 at their recipe sizes on N(0, 1) 3x32x32 batches of 128 (CIFAR-10 after normalisation): the
training step, eager and under `trainstep.GraphedTrainStep`, against a plain-torch fp32 arm of the same network in the
same run (the reference's operations: nn.Conv2d / nn.ConvTranspose2d on cuDNN with TF32 off, the reference's quantizer
formula with its EMA update, F.mse_loss and torch.optim.Adam), and `pg_vq_assign` alone against the reference's torch
distances + argmin at each quantizer's shape.

    python tools/bench_vq_vae.py [--steps 30] [--warmup 5] [--reps 3]

Training step: zero_grad, forward, recipe loss, backward, clip to 1e50 and Adam, timed with a device synchronise around
`--steps` steps (wall time per step), `--reps` times.  The kernels this library launches per step are counted.  The
card's name, power limit and SM clock are read in the same run and printed with the numbers."""
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

from pytorch_generative_b200 import _lib, losses, models, trainstep
from pytorch_generative_b200.models import vae
from pytorch_generative_b200.nn import VectorQuantizer

BATCH, SIDE = 128, 32
RECIPES = {
    "vq_vae": (models.VectorQuantizedVAE, dict(in_channels=3, out_channels=3, hidden_channels=128, residual_channels=32,
                                               n_residual_blocks=2, n_embeddings=512, embedding_dim=64),
               losses.vq_vae_loss, 1.0),
    "vq_vae_2": (models.VectorQuantizedVAE2, dict(in_channels=3, out_channels=3, hidden_channels=128,
                                                  n_residual_blocks=2, residual_channels=64, n_embeddings=512,
                                                  embedding_dim=64), losses.vq_vae_2_loss, 0.25),
}


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                               "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return f"unavailable ({e})"


def torch_vq(vq, x):
    """reference nn/utils.py VectorQuantizer.forward on vq's tensors (EMA in training)."""
    n, c, h, w = x.shape
    flat_x = x.permute(0, 2, 3, 1).contiguous().view(-1, c)
    e = vq._embedding
    distances = torch.sum(flat_x**2, dim=1, keepdim=True) + torch.sum(e**2, dim=1) - 2 * flat_x @ e.t()
    idxs = torch.argmin(distances, dim=1, keepdim=True)
    one_hot = torch.zeros(idxs.shape[0], vq.n_embeddings, device=x.device)
    one_hot.scatter_(1, idxs, 1)
    quantized = (one_hot @ e).view(n, h, w, c).permute(0, 3, 1, 2).contiguous()
    loss = F.mse_loss(x, quantized.detach())
    with torch.no_grad():
        vq._cluster_size.mul_(vq._decay).add_(one_hot.sum(0), alpha=1 - vq._decay)
        vq._embedding_avg.mul_(vq._decay).add_((flat_x.t() @ one_hot).t(), alpha=1 - vq._decay)
        vq._embedding.copy_(vq._embedding_avg / (vq._cluster_size + 1e-5).unsqueeze(1))
    return x + (quantized - x).detach(), loss


def torch_run(mod, x):
    """The reference's forward of any module of the model tree, on torch ops."""
    if isinstance(mod, (nn.Conv2d, nn.ConvTranspose2d, nn.ReLU)):
        return mod(x)
    if isinstance(mod, VectorQuantizer):
        return torch_vq(mod, x)
    if isinstance(mod, vae.ResidualBlock):
        return x + torch_run(mod._net, x)
    if isinstance(mod, nn.Sequential):
        for m in mod:
            x = torch_run(m, x)
        return x
    return torch_run(mod._net, x)  # Encoder, Decoder, ResidualStack, Quantizer


def torch_forward(model, x):
    if isinstance(model, models.VectorQuantizedVAE):
        q, vq_loss = torch_run(model._quantizer, torch_run(model._encoder, x))
        return torch_run(model._decoder, q), vq_loss
    encoded_b = torch_run(model._encoder_b, x)
    encoded_t = torch_run(model._encoder_t, encoded_b)
    quantized_t, vq_loss_t = torch_run(model._quantizer_t, encoded_t)
    quantized_b, vq_loss_b = torch_run(model._quantizer_b, encoded_b)
    decoded_t = torch_run(model._decoder_t, quantized_t)
    xhat = torch_run(model._decoder_b, torch.cat((model._conv(decoded_t), quantized_b), dim=1))
    return xhat, 0.5 * (vq_loss_b + vq_loss_t) + F.mse_loss(decoded_t, encoded_b)


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
    def __init__(self, model):
        super().__init__()
        self.model = model

    def forward(self, x):
        return _Preds(self.model(x))


def bench_assign(P, K, d, steps):
    """pg_vq_assign (with the operand and the loss sum) against torch's distances + argmin at one quantizer's shape."""
    x = torch.randn(P, d, device="cuda")
    e = torch.randn(K, d, device="cuda")
    idx = torch.empty(P, dtype=torch.int32, device="cuda")
    out = torch.empty(P, d, dtype=torch.bfloat16, device="cuda")
    acc = torch.zeros(1, device="cuda")

    def ours():
        _lib.vq_assign(x, e, idx, out, 0, d, acc)

    def ref():
        dist = torch.sum(x**2, dim=1, keepdim=True) + torch.sum(e**2, dim=1) - 2 * x @ e.t()
        return torch.argmin(dist, dim=1)
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    res = {}
    for name, fn in (("pg_vq_assign", ours), ("torch", ref)):
        for _ in range(5):
            fn()
        start.record()
        for _ in range(steps):
            fn()
        end.record()
        torch.cuda.synchronize()
        res[name] = round(start.elapsed_time(end) / steps * 1e3, 1)  # microseconds
    same = torch.equal(idx.long(), ref())
    return res, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_vq_vae measures on a GPU only"
    torch.backends.cudnn.allow_tf32 = torch.backends.cuda.matmul.allow_tf32 = False
    result = {"card": card()}
    for name, (cls, kw, loss_fn, _) in RECIPES.items():
        torch.manual_seed(0)
        model = cls(**kw).cuda()
        x = torch.randn(BATCH, 3, SIDE, SIDE, device="cuda")
        opt = torch.optim.Adam(model.parameters(), lr=2e-4)

        def eager_step():
            opt.zero_grad(set_to_none=True)
            loss_fn(x, None, model(x))["loss"].backward()
            torch.nn.utils.clip_grad_norm_(model.parameters(), 1e50)
            opt.step()
        n0 = _lib.launch_count()
        eager_step()
        launches = _lib.launch_count() - n0
        tmodel = copy.deepcopy(model)
        topt = torch.optim.Adam(tmodel.parameters(), lr=2e-4)

        def torch_step():
            topt.zero_grad(set_to_none=True)
            xhat, vq_loss = torch_forward(tmodel, x)
            loss = F.mse_loss(xhat, x) + RECIPES[name][3] * vq_loss
            loss.backward()
            torch.nn.utils.clip_grad_norm_(tmodel.parameters(), 1e50)
            topt.step()
        gm = _TupleModel(copy.deepcopy(model))
        graphed = trainstep.GraphedTrainStep(gm, gm.parameters(), lambda p, xx: loss_fn(xx, None, p)["loss"], x,
                                             lr=2e-4, lr_gamma=1.0)
        res = {"launches_per_eager_step": launches}
        for key, fn in (("eager_ms", eager_step), ("graphed_ms", lambda: graphed.graph.replay()),
                        ("torch_fp32_ms", torch_step)):
            res[key] = [round(timed(fn, args.steps, args.warmup), 3) for _ in range(args.reps)]
        result[name] = res
    for shape in ((BATCH * 8 * 8, 512, 64), (BATCH * 16 * 16, 512, 64)):
        res, same = bench_assign(*shape, steps=100)
        result[f"assign_P{shape[0]}_K{shape[1]}_d{shape[2]}_us"] = res
        result[f"assign_P{shape[0]}_same_indices_as_torch"] = same
    result["card_after"] = card()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
