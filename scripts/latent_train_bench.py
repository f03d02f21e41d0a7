"""Latent-DPM training step (trainer/train_latent_diffusion.py: the ffhq / celeba64 / horse / bedroom *_latent.yml configs,
128 latents per process) with and without autocast: the ffhq_latent MLPSkipNet (512 -> 2048 x 10 layers, time embedding 64),
the L1 latent loss, forward + loss.backward().

  python scripts/latent_train_bench.py [--batch 128] [--steps 50] [--warmup 10]

Prints one JSON line per result:
  * the card's name and power limit, read in this run;
  * ms per step of `--amp off` and `--amp bf16`, alternated twice (CUDA events over --steps steps after --warmup);
  * the device time of each plan of both trainers (Plan.profile, per kernel kind);
  * every split-K GEMM of the bf16 trainer: its shape and algorithmic TFLOP/s (2 B Cin Cout over its profiled time);
  * the frozen 128-px encoder's forward at the same batch (module.precision as the latent trainer uses it, forward only),
    timed on its own."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
from pdae_b200.engine import get_default_precision
from pdae_b200.model.mlp_skip_net import MLPSkipNet
from pdae_b200.model.representation_learning.encoder import FFHQEncoder
from pdae_b200.utils.synth import fill_module_, synth_images, synth_normal

FFHQ_LATENT = dict(input_channel=512, model_channel=2048, num_layers=10, time_emb_channel=64, use_norm=True, dropout=0.0)
DIFF = {"timesteps": 1000, "betas_type": "linear"}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit unknown"


def step(gd, mlp, z0, t, noise, amp):
    lc = gd.latent_diffusion_config
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
        z_t = gd.extract_coef_at_t(lc["sqrt_alphas_cumprod"], t, z0.shape) * z0 + \
            gd.extract_coef_at_t(lc["sqrt_one_minus_alphas_cumprod"], t, z0.shape) * noise
        loss = gd.p_loss(noise, mlp(z_t, t), loss_type=lc["loss_type"])      # the reference's L1 latent loss
    loss.backward()
    for p in mlp.parameters():
        p.grad = None


def time_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    st = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(st)
    for _ in range(steps):
        fn()
    e1.record(st)
    e1.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=128)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("latent_train_bench: needs a CUDA device")
    B = args.batch
    print(json.dumps({"card": card()}))
    dev = torch.device("cuda")
    gd = GaussianDiffusion(DIFF, dev)
    mlp = fill_module_(MLPSkipNet(**FFHQ_LATENT), seed=79).to(dev).train()
    z0, noise = synth_normal((B, 512), 81).to(dev), synth_normal((B, 512), 82).to(dev)
    t = torch.randint(0, 1000, (B,), generator=torch.Generator().manual_seed(83)).to(dev)
    res = {"B": B, "steps": args.steps}
    for rnd in range(2):
        for amp in (False, True):
            ms = time_ms(lambda: step(gd, mlp, z0, t, noise, amp), args.steps, args.warmup)
            res.setdefault("bf16" if amp else "off", []).append(round(ms, 3))
    print(json.dumps({"step_ms": res}))
    for tr in mlp._train_cache.values():
        mode = "bf16" if tr.amp else "off"
        for name, plan in (("fwd", tr.fwd), ("bwd", tr.bwd)):
            prof = plan.profile(reps=5)
            kinds = {k: {"ms": round(v["ms"], 4), "launches": v["launches"]} for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])}
            print(json.dumps({"plan": f"{mode}/{name}", "total_ms": round(sum(v["ms"] for v in prof.values()), 4), "kinds": kinds}))
            if tr.amp:
                for i, (fn, a) in enumerate(plan.ops):
                    if fn == "conv_tc2_splitk":
                        Bm, Cin, Cout = a[4], a[5], a[6]
                        us = plan.last_op_ms[i] * 1e3
                        print(json.dumps({"splitk": f"{mode}/{name}", "B": Bm, "Cin": Cin, "Cout": Cout, "us": round(us, 2),
                                          "tflops": round(plan.flops[i] / us / 1e6, 2)}))
    enc = fill_module_(FFHQEncoder(latent_dim=512), seed=7).to(dev).eval().requires_grad_(False)
    x = synth_images(B, 3, 128, 33).to(dev)
    with torch.no_grad():
        ms = time_ms(lambda: enc(x), args.steps, args.warmup)
    print(json.dumps({"frozen_encoder_fwd": {"B": B, "size": 128, "precision": enc.precision or get_default_precision(), "ms": round(ms, 3)}}))


if __name__ == "__main__":
    main()
