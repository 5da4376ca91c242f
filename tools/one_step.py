"""One training step of a bench.py configuration between cudaProfilerStart/Stop, for launch lists:
  ncu --profile-from-start off --metrics gpu__time_duration.sum --clock-control none --csv --log-file out.csv \
      python tools/one_step.py c4
Without ncu it prints the step time (CUDA events, 5 steps)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench
from pytorch_generative_b200 import losses, models, optim

name = sys.argv[1] if len(sys.argv) > 1 else "c4"
spec = bench.CONFIGS[name]
dev = torch.device("cuda:0")
torch.manual_seed(0)
model = getattr(models, spec["cls"])(**spec["cfg"]).to(dev).train()
params = list(model.parameters())
opt = optim.FusedAdam(params, lr=spec["lr"])
x = bench.synthetic_batch(spec["batch"], spec["shape"], seed=0).to(dev)


def step():
    opt.zero_grad()
    loss = losses.bce_with_logits_sum_mean(model(x), x)
    loss.backward()
    return loss.item(), opt.clip_and_step(1e50).item()


for _ in range(3):
    step()
torch.cuda.synchronize()
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
print(f"{name}: {e0.elapsed_time(e1) / 5:.3f} ms/step", flush=True)
