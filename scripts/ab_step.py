"""Graph-replay time of one ShiftUNet decoder step at a given precision.
usage: python scripts/ab_step.py [workload] [batch] [reps] [precision]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

import pdae_b200
from bench import WORKLOADS
from pdae_b200.model.shift_unet import ShiftUNet
from pdae_b200.utils.synth import fill_module_, synth_normal

wl = sys.argv[1] if len(sys.argv) > 1 else "celeba64"
B = int(sys.argv[2]) if len(sys.argv) > 2 else 256
reps = int(sys.argv[3]) if len(sys.argv) > 3 else 30
prec = sys.argv[4] if len(sys.argv) > 4 else "bf16"
cfg, size = WORKLOADS[wl][0], WORKLOADS[wl][1]
pdae_b200.set_default_precision(prec)
dev = torch.device("cuda")
dec = fill_module_(ShiftUNet(latent_dim=512, **cfg), seed=0).eval().to(dev)
x = synth_normal((B, 3, size, size), 1).to(dev)
z = synth_normal((B, 512), 2).to(dev)
t = torch.full((B,), 500, device=dev, dtype=torch.long)
with torch.no_grad():
    dec(x, t, z)
plan, _ = dec.plan_for(B, size, size)
plan.capture_graph()
for _ in range(5):
    plan.run(prologue=False)
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
best = 1e9
tot = 0.0
for _ in range(3):
    e0.record()
    for _ in range(reps):
        plan.run(prologue=False)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    best = min(best, ms)
    tot += ms / 3
print(f"ab_step {wl} B={B} {prec}: {tot:.3f} ms/step avg, {best:.3f} best, {plan.n_launch} launches")
