"""One training step of a bench.py configuration.

    python tools/one_step.py [config]                  step time (CUDA events, 5 steps); one step before them runs
                                                       between cudaProfilerStart/Stop for Nsight Compute:
        ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file out.csv \
            python tools/one_step.py c4
    python tools/one_step.py c5 --heads 4              an ImageGPT config with another head count (same channels)
    python tools/one_step.py c5 --profile OUT_DIR      also one warmed step under torch.profiler: a per-kernel table
                                                       (launches, total ms, mean us, share of kernel time) on stdout
                                                       and the Chrome trace in OUT_DIR
The profiled step runs on its own, before the timed steps: tracing slows the host, so its wall time is not the step
time."""
import argparse, collections, json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from pytorch_generative_b200 import losses, models, optim

ap = argparse.ArgumentParser()
ap.add_argument("config", nargs="?", default="c4", choices=sorted(bench.CONFIGS))
ap.add_argument("--profile", metavar="OUT_DIR", default=None)
ap.add_argument("--heads", type=int, default=0, help="n_attention_heads of an ImageGPT config (default: the config's)")
args = ap.parse_args()
name = args.config
spec = bench.CONFIGS[name]
cfg = dict(spec["cfg"])
if args.heads:
    if "n_attention_heads" not in cfg:
        ap.error(f"--heads applies to the ImageGPT configs, not {name}")
    cfg["n_attention_heads"] = args.heads
dev = torch.device("cuda:0")
torch.manual_seed(0)
model = getattr(models, spec["cls"])(**cfg).to(dev).train()
params = list(model.parameters())
opt = optim.FusedAdam(params, lr=spec["lr"])
x = bench.synthetic_batch(spec["batch"], spec["shape"], seed=0).to(dev)


def step():
    opt.zero_grad()
    loss = losses.bce_with_logits_sum_mean(model(x), x)
    loss.backward()
    return loss.item(), opt.clip_and_step(1e50).item()


def kernel_table(trace_path):
    """Per-kernel rows from the trace's device events: (name, launches, total us), longest first."""
    with open(trace_path) as f:
        events = json.load(f)["traceEvents"]
    agg = collections.defaultdict(lambda: [0, 0.0])
    for ev in events:
        if ev.get("ph") == "X" and ev.get("cat") == "kernel":
            a = agg[ev["name"]]
            a[0] += 1
            a[1] += float(ev["dur"])
    return sorted(((k, n, us) for k, (n, us) in agg.items()), key=lambda r: -r[2])


def profile(out_dir):
    os.makedirs(out_dir, exist_ok=True)
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=acts) as prof:
        step()
        torch.cuda.synchronize()
    trace = os.path.join(out_dir, f"one_step_{name}.pt.trace.json")
    prof.export_chrome_trace(trace)
    rows = kernel_table(trace)
    total = sum(us for _, _, us in rows)
    print(f"{name}: one step under torch.profiler, {sum(n for _, n, _ in rows)} kernel launches, "
          f"{total / 1e3:.3f} ms kernel time (trace: {trace})")
    print(f"{'kernel':90s} {'launches':>8s} {'total ms':>9s} {'mean us':>9s} {'share':>7s}")
    for k, n, us in rows:
        print(f"{k[:90]:90s} {n:8d} {us / 1e3:9.3f} {us / n:9.1f} {us / total:7.1%}")
    gemm_us = sum(us for k, _, us in rows if "gemm_wgmma_kernel" in k)
    print(f"gemm_wgmma_kernel: {gemm_us / 1e3:.3f} ms, {gemm_us / total:.1%} of kernel time", flush=True)


for _ in range(3):
    step()
torch.cuda.synchronize()
if args.profile:
    profile(args.profile)
else:  # one step between cudaProfilerStart/Stop, for `ncu --profile-from-start off`
    torch.cuda.profiler.start()
    step()
    torch.cuda.synchronize()
    torch.cuda.profiler.stop()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(5):
    step()
e1.record()
torch.cuda.synchronize()
print(f"{name}{f' --heads {args.heads}' if args.heads else ''}: {e0.elapsed_time(e1) / 5:.3f} ms/step", flush=True)
