"""sample() wall time of the bench.py configurations: incremental (line buffers / KV caches, one graph replay per
pixel) against the reference's scheme (one full forward per pixel).  python tools/bench_sample.py [c1 c4 c5] [n]"""
import os, sys, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from pytorch_generative_b200 import models

dev = torch.device("cuda:0")
CASES = {
    "c1": (lambda: models.PixelCNN(1, 1, 15, 16, 32), (1, 28, 28)),
    "c3": (lambda: models.GatedPixelCNN(3, 3, 15, 128, 32), (3, 32, 32)),
    "c4": (lambda: models.PixelSNAIL(3, 3, 256, 8, 2, 16, 128), (3, 32, 32)),
    "c5": (lambda: models.ImageGPT(3, 3, 32, 24, 8, 512), (3, 32, 32)),
}
names = [a for a in sys.argv[1:] if a in CASES] or list(CASES)
n = next((int(a) for a in sys.argv[1:] if a.isdigit()), 16)
for name in names:
    torch.manual_seed(0)
    make, shape = CASES[name]
    m = make().to(dev).eval()
    with torch.no_grad():
        m(torch.rand(n, *shape, device=dev))

    def t(label):
        torch.cuda.synchronize(); t0 = time.perf_counter(); m.sample(n_samples=n); torch.cuda.synchronize()
        print(f"{name} n={n} {label} {(time.perf_counter() - t0) * 1e3:.0f} ms", flush=True)

    t("incremental (capture)     ")
    t("incremental (cached graph)")
    m._incremental_sampling = False
    m._sample_with_graphs = False
    t("full forward per pixel, row-truncated where exact")
    for k, v in {**m.__dict__.get("_samplers", {}), **m.__dict__.get("_pixel_states", {})}.items():
        print("  sampler", k, "graph:", type(v["graph"]).__name__, str(v.get("graph_error", ""))[:300])
    del m
