"""What a refactor of ImageGPT's training step must leave alone, written down so two trees can be compared.

    python tools/step_fingerprint.py OUT_DIR

1. Padded streams (bench.py has no such configuration): for 12 channels / 3 heads and 100 channels / 4 heads, 2 blocks,
   1x32x32 images, batch 4, one seeded forward + loss + backward; the logits and every parameter's gradient go to
   OUT_DIR/padded_<channels>.npz.  Every reduction on the path is fixed-order, so two trees that compute the same thing
   write the same bytes.
2. bench.py's c5 and c2: the kernels libpg_b200.so launches in one warm training step (forward, loss, backward,
   clip_and_step) and, for c5, torch.cuda.max_memory_allocated over that step.
The card's name and power limit are printed first."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
from pytorch_generative_b200 import _lib, losses, models, optim

dev = torch.device("cuda:0")


def padded(channels, heads, out_dir):
    cfg = dict(in_channels=1, out_channels=1, in_size=32, n_transformer_blocks=2, n_attention_heads=heads,
               n_embedding_channels=channels)
    torch.manual_seed(0)
    m = models.ImageGPT(**cfg).to(dev).train()
    x = bench.synthetic_batch(4, (1, 32, 32), seed=1).to(dev)
    logits = m(x)
    losses.bce_with_logits_sum_mean(logits, x).backward()
    arrays = {"logits": logits.detach().cpu().numpy()}
    arrays.update({name: p.grad.cpu().numpy() for name, p in m.named_parameters()})
    np.savez(os.path.join(out_dir, f"padded_{channels}.npz"), **arrays)
    print(f"padded stream, {channels} channels / {heads} heads: {len(arrays)} arrays written", flush=True)


def warm_step(name):
    spec = bench.CONFIGS[name]
    torch.manual_seed(0)
    m = getattr(models, spec["cls"])(**spec["cfg"]).to(dev).train()
    opt = optim.FusedAdam(m.parameters(), lr=spec["lr"])
    x = bench.synthetic_batch(spec["batch"], spec["shape"], seed=0).to(dev)

    def step():
        opt.zero_grad()
        losses.bce_with_logits_sum_mean(m(x), x).backward()
        opt.clip_and_step(1e50)

    for _ in range(3):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    before = _lib.launch_count()
    step()
    torch.cuda.synchronize()
    print(f"{name}: {_lib.launch_count() - before} kernel launches in one warm step, max_memory_allocated "
          f"{torch.cuda.max_memory_allocated(dev)} B", flush=True)


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    os.makedirs(sys.argv[1], exist_ok=True)
    print("GPU (name, power limit):", subprocess.run(
        ["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
        text=True).stdout.strip() or torch.cuda.get_device_name(dev), flush=True)
    for channels, heads in ((12, 3), (100, 4)):
        padded(channels, heads, sys.argv[1])
    for name in ("c5", "c2"):
        warm_step(name)
