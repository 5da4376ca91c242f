"""Bit-for-bit comparison of what sample() computes in two builds of this package (for example a branch and its parent
commit, each built in its own tree).

    python tools/compare_samplers.py --against OTHER_TREE [--out DIR]
        runs the cases below once with this tree's package and once with OTHER_TREE's (each in a subprocess, both
        trees already built) and fails unless every tensor is bit-identical
    python tools/compare_samplers.py --dump DIR [--root TREE]
        only writes the tensors of one tree to DIR/<case>.pt

Cases:
  * teacher-forced sampling (every pixel given, per-pixel logits recorded through the sample_fn hook, two calls) for
    the sampler configurations of tests/test_parity_gpu.py and tests/test_wide_heads_gpu.py, and ImageGPT at 64x64;
  * sample() of 16 images with pre-drawn uniforms (seeded) for the bench.py configurations c1 to c5 at their own image
    sizes, seeded initial weights.
"""
import argparse
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

TEACHER_FORCED = [
    # tests/test_parity_gpu.py::test_incremental_sampler_logits_match_the_full_forward
    ("PixelCNN", dict(in_channels=1, out_channels=1, n_residual=3, residual_channels=16, head_channels=32), (3, 1, 28, 28)),
    ("PixelCNN", dict(in_channels=3, out_channels=3, n_residual=2, residual_channels=32, head_channels=16), (2, 3, 8, 16)),
    ("PixelSNAIL", dict(in_channels=3, out_channels=3, n_channels=64, n_pixel_snail_blocks=2, n_residual_blocks=2,
                        attention_key_channels=16, attention_value_channels=32), (2, 3, 16, 16)),
    ("GatedPixelCNN", dict(in_channels=1, out_channels=1, n_gated=3, gated_channels=32, head_channels=16), (3, 1, 28, 28)),
    ("GatedPixelCNN", dict(in_channels=3, out_channels=3, n_gated=2, gated_channels=64, head_channels=32), (2, 3, 8, 16)),
    ("GatedPixelCNN", dict(in_channels=1, out_channels=1, n_gated=0, gated_channels=16, head_channels=8), (2, 1, 6, 5)),
    ("PixelSNAIL", dict(in_channels=1, out_channels=1, n_channels=32, n_pixel_snail_blocks=1, n_residual_blocks=1,
                        attention_key_channels=4, attention_value_channels=128), (4, 1, 28, 28)),
    # tests/test_wide_heads_gpu.py::test_wide_head_incremental_sampler_matches_the_full_forward
    ("ImageGPT", dict(in_channels=3, out_channels=3, in_size=16, n_transformer_blocks=2, n_attention_heads=4,
                      n_embedding_channels=512), (2, 3, 16, 16)),
    ("PixelSNAIL", dict(in_channels=3, out_channels=3, n_channels=64, n_pixel_snail_blocks=2, n_residual_blocks=1,
                        attention_key_channels=128, attention_value_channels=32), (2, 3, 16, 16)),
    # tests/test_large_images_gpu.py::test_large_image_sampler_logits_match_the_full_forward: the split decode
    ("ImageGPT", dict(in_channels=1, out_channels=1, in_size=64, n_transformer_blocks=2, n_attention_heads=2,
                      n_embedding_channels=64), (2, 1, 64, 64)),
]
BENCH_SAMPLES = ["c1", "c2", "c3", "c4", "c5"]
N_SAMPLES = 16


def dump(root, out_dir):
    sys.path.insert(0, root)
    import torch

    from pytorch_generative_b200 import models   # the package of `root`, imported before anything else can add a path

    assert os.path.abspath(models.__file__).startswith(os.path.join(root, "")), models.__file__
    sys.path.append(HERE)
    from bench import CONFIGS
    dev = torch.device("cuda:0")
    os.makedirs(out_dir, exist_ok=True)
    for i, (cls, cfg, shape) in enumerate(TEACHER_FORCED):
        torch.manual_seed(7)
        m = getattr(models, cls)(**cfg).to(dev)
        with torch.no_grad():
            for p in m.parameters():
                p.mul_(1.5)
        x = torch.bernoulli(torch.full(shape, 0.5)).to(dev)
        calls = []
        for _ in range(2):
            seen = []
            m._sample_fn = lambda logits: (seen.append(logits.detach().clone()), torch.zeros_like(logits))[1]
            m.sample(conditioned_on=x)
            calls.append(torch.stack(seen).cpu())
        states = m.__dict__.get("_pixel_states")
        assert states and all(st["graph"] for st in states.values()), f"{cls}: not the graph-captured sampler"
        torch.save(dict(logits=calls), os.path.join(out_dir, f"teacher_{i}_{cls}.pt"))
        print(f"teacher-forced {i} {cls} {shape}: {calls[0].shape[0]} pixels", flush=True)
    for name in BENCH_SAMPLES:
        spec = CONFIGS[name]
        torch.manual_seed(0)
        m = getattr(models, spec["cls"])(**spec["cfg"]).to(dev)
        c, h, w = spec["shape"]
        g = torch.Generator().manual_seed(11)
        uniforms = [torch.rand(N_SAMPLES, c, generator=g) for _ in range(h * w)]
        it = iter(uniforms)
        logits_seen = []

        def draw(logits):
            logits_seen.append(logits.detach().clone())
            return (next(it).to(logits.device) < torch.sigmoid(logits)).float()

        m._sample_fn = draw
        out = m.sample(conditioned_on=torch.full((N_SAMPLES, c, h, w), -1.0, device=dev))
        torch.save(dict(sample=out.cpu(), logits=torch.stack(logits_seen).cpu()), os.path.join(out_dir, f"bench_{name}.pt"))
        print(f"bench {name}: {N_SAMPLES} samples of {spec['shape']}", flush=True)


def compare(dir_a, dir_b):
    import torch

    names = sorted(os.listdir(dir_a))
    assert names == sorted(os.listdir(dir_b)), "the two runs wrote different cases"
    bad = 0
    for fname in names:
        a = torch.load(os.path.join(dir_a, fname))
        b = torch.load(os.path.join(dir_b, fname))
        for key in a:
            ta, tb = a[key], b[key]
            pairs = zip(ta, tb) if isinstance(ta, list) else [(ta, tb)]
            same = all(x.shape == y.shape and torch.equal(x.view(torch.int32) if x.dtype == torch.float32 else x,
                                                          y.view(torch.int32) if y.dtype == torch.float32 else y)
                       for x, y in pairs)
            print(f"{fname:32s} {key:8s} {'bit-identical' if same else 'DIFFERENT'}")
            bad += not same
    return bad


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--dump", metavar="DIR")
    ap.add_argument("--root", default=HERE, help="tree whose pytorch_generative_b200 is imported (default: this one)")
    ap.add_argument("--against", metavar="OTHER_TREE")
    ap.add_argument("--out", default=None, help="where the two runs write their tensors (default: a temporary dir)")
    args = ap.parse_args()
    if args.dump:
        dump(os.path.abspath(args.root), args.dump)
        return
    if not args.against:
        ap.error("give --against OTHER_TREE or --dump DIR")
    import tempfile

    out = args.out or tempfile.mkdtemp(prefix="compare_samplers_")
    runs = {"this": HERE, "other": os.path.abspath(args.against)}
    for tag, root in runs.items():
        print(f"== {tag}: {root}", flush=True)
        subprocess.run([sys.executable, os.path.abspath(__file__), "--dump", os.path.join(out, tag), "--root", root],
                       check=True)
    bad = compare(os.path.join(out, "this"), os.path.join(out, "other"))
    print("all bit-identical" if bad == 0 else f"{bad} tensor(s) differ")
    sys.exit(1 if bad else 0)


if __name__ == "__main__":
    main()
