"""sample() wall time: incremental (line buffers / KV caches, one graph replay per pixel) against the reference's scheme
(one full forward per pixel), both in the same run.

    python tools/bench_sample.py [c1 c3 c4 c5] [n]       the bench.py configurations at their own sizes
    python tools/bench_sample.py [c1w12 c3w100 c4w100] [n]
        c1, c3 and c4 at widths that are not multiples of 8 (PixelSNAIL at its recipe's key / value rule)
    python tools/bench_sample.py --size 64 [igpt snail] [n]
        an ImageGPT and a PixelSNAIL at size x size (above 32x32 the KV-cached decode runs one block per 1024 keys)

The card's name and power limit are printed with the times."""
import argparse, os, subprocess, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pytorch_generative_b200 import models

dev = torch.device("cuda:0")
CASES = {
    "c1": (lambda s: models.PixelCNN(1, 1, 15, 16, 32), (1, 28, 28)),
    "c3": (lambda s: models.GatedPixelCNN(3, 3, 15, 128, 32), (3, 32, 32)),
    "c4": (lambda s: models.PixelSNAIL(3, 3, 256, 8, 2, 16, 128), (3, 32, 32)),
    "c5": (lambda s: models.ImageGPT(3, 3, 32, 24, 8, 512), (3, 32, 32)),
    "c1w12": (lambda s: models.PixelCNN(1, 1, 15, 12, 30), (1, 28, 28)),
    "c3w100": (lambda s: models.GatedPixelCNN(3, 3, 15, 100, 30), (3, 32, 32)),
    "c4w100": (lambda s: models.PixelSNAIL(3, 3, 100, 8, 2, 6, 50), (3, 32, 32)),
    # --size: 4 blocks / 4 heads / 256 ch, and 4 blocks / 128 ch, key 16 / value 64
    "igpt": (lambda s: models.ImageGPT(1, 1, s, 4, 4, 256), (1, None, None)),
    "snail": (lambda s: models.PixelSNAIL(1, 1, 128, 4, 2, 16, 64), (1, None, None)),
}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i",
                              str(dev.index or 0)], capture_output=True, text=True, timeout=10).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or f"{torch.cuda.get_device_name(dev)}, power limit unknown (nvidia-smi unavailable)"


ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
ap.add_argument("cases", nargs="*", help="case names and optionally the number of images (default 16)")
ap.add_argument("--size", type=int, default=None, help="image height and width for the igpt / snail cases")
args = ap.parse_args()
names = [a for a in args.cases if a in CASES] or (["igpt", "snail"] if args.size else ["c1", "c3", "c4", "c5"])
n = next((int(a) for a in args.cases if a.isdigit()), 16)
print(f"GPU (name, power limit): {card()}", flush=True)
for name in names:
    torch.manual_seed(0)
    make, shape = CASES[name]
    if shape[1] is None:
        if not args.size:
            sys.exit(f"{name} needs --size")
        shape = (shape[0], args.size, args.size)
    m = make(shape[1]).to(dev).eval()
    with torch.no_grad():
        m(torch.rand(n, *shape, device=dev))
    tag = f"{name} {shape[0]}x{shape[1]}x{shape[2]} n={n}"

    def t(label):
        torch.cuda.synchronize(); t0 = time.perf_counter(); m.sample(n_samples=n); torch.cuda.synchronize()
        ms = (time.perf_counter() - t0) * 1e3
        print(f"{tag} {label} {ms:.0f} ms", flush=True)
        return ms

    t("incremental (capture)     ")
    inc = t("incremental (cached graph)")
    for k, v in m.__dict__.get("_pixel_states", {}).items():
        print("  sampler", k, "graph:", type(v["graph"]).__name__, str(v.get("graph_error", ""))[:300])
    m._incremental_sampling = False
    full = t("full forward per pixel, row-truncated where exact")
    print(f"{tag} incremental is {full / inc:.1f}x faster than one forward per pixel", flush=True)
    del m
