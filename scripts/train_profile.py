"""Per-kernel device time of one PDAE training step's plans (frozen-half forward, trainable forward, backward, encoder fwd/bwd).
usage: python scripts/train_profile.py [batch] [--amp {off,bf16}]
--amp bf16: the step runs inside torch.autocast("cuda", dtype=torch.bfloat16), so the bf16 training plans are profiled."""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from bench import WORKLOADS
from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
from pdae_b200.model.representation_learning.encoder import CELEBA64Encoder
from pdae_b200.model.shift_unet import ShiftUNet
from pdae_b200.utils.synth import fill_module_, synth_images

ap = argparse.ArgumentParser()
ap.add_argument("batch", type=int, nargs="?", default=32)
ap.add_argument("--amp", choices=("off", "bf16"), default="off")
args = ap.parse_args()
B = args.batch


def train_loss():
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=args.amp == "bf16"):
        return gd.representation_learning_train_one_batch(enc, dec, x0)["prediction_loss"]



cfg, size = WORKLOADS["celeba64"][0], WORKLOADS["celeba64"][1]
dev = torch.device("cuda")
dec = fill_module_(ShiftUNet(latent_dim=512, **dict(cfg, dropout=0.1)), seed=0).to(dev)
enc = fill_module_(CELEBA64Encoder(latent_dim=512), seed=1).to(dev).train()
dec.freeze()
dec.set_train_mode()
dec.precision = enc.precision = "fp32"
gd = GaussianDiffusion({"timesteps": 1000, "betas_type": "linear"}, dev)
x0 = synth_images(B, 3, size, 3).to(dev)
print(f"{torch.cuda.get_device_properties(dev).name}, batch {B}, amp {args.amp}")
for _ in range(2):
    loss = train_loss()
    loss.backward()
tr = list(dec._train_cache.values())[0]
te = list(enc._train_cache.values())[0]
for name, plan in (("decoder frozen fwd", tr.frozen), ("decoder trainable fwd", tr.fwd), ("decoder bwd", tr.bwd), ("encoder fwd", te.fwd),
                   ("encoder bwd", te.bwd)):
    if plan is None:
        continue
    prof = plan.profile(reps=3)
    tot = sum(v["ms"] for v in prof.values())
    print(f"{name}: {tot:.2f} ms")
    for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])[:8]:
        print(f"    {k:22s} {v['ms']:8.3f} ms  n={v['launches']:4d}")

# ---- segment timeline of whole steps (CUDA events around the Python-level phases; host time of the same calls) ----
import copy
import time

from pdae_b200.optim import FusedAdamEMA

ema_dec, ema_enc = copy.deepcopy(dec).requires_grad_(False), copy.deepcopy(enc).requires_grad_(False)
groups = [list(enc.parameters()), list(dec.label_emb.parameters()), list(dec.shift_middle_block.parameters()),
          list(dec.shift_output_blocks.parameters()), list(dec.shift_out.parameters())]
opt = FusedAdamEMA([{"params": g} for g in groups], lr=1e-4, ema_decay=0.9999)
opt.attach_ema(enc, ema_enc)
opt.attach_ema(dec, ema_dec)
seg = {"forward+loss": [0.0, 0.0], "backward": [0.0, 0.0], "optimizer+EMA": [0.0, 0.0]}
N = 5
for it in range(N + 2):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
    torch.cuda.synchronize()
    h = [time.perf_counter()]
    ev[0].record()
    loss = train_loss()
    ev[1].record(); h.append(time.perf_counter())
    loss.backward()
    ev[2].record(); h.append(time.perf_counter())
    opt.step()
    opt.zero_grad(set_to_none=True)
    ev[3].record(); h.append(time.perf_counter())
    torch.cuda.synchronize()
    if it >= 2:
        for i, k in enumerate(seg):
            seg[k][0] += ev[i].elapsed_time(ev[i + 1]) / N
            seg[k][1] += (h[i + 1] - h[i]) * 1e3 / N
print("whole-step segments (device ms between events | host ms spent issuing):")
for k, (d, hh) in seg.items():
    print(f"    {k:16s} {d:7.2f} | {hh:7.2f}")
