"""The DDPM ancestral loops and DDIM trajectory interpolation on the one-graph-per-step path, against the generic per-step loop
(the same network wrapped in a lambda, so every step replays its plan from Python and runs the update with torch ops).

  python scripts/sampler_bench.py [--ddpm-timesteps 100] [--ddim ddim100]

Workloads (each in "bf16x3" and "bf16"): representation-learning DDPM on the ffhq128-proxy ShiftUNet at B = 5
(sampler/autoencoding_example.py), regular DDPM on the MNIST UNet (config/mnist_regular.yml) at B = 36, and trajectory
interpolation on the ffhq128-proxy ShiftUNet at B = 1 with --ddim steps (sampler/interpolation.py).  Every DDPM step does the
same work, so a shortened schedule (--ddpm-timesteps) gives the per-step time of the 1000-step loop.
Prints one JSON line per result: the card's name and power limit, read in this run; then per workload and precision the
ms per step of the generic and the graphed loop in two alternating rounds (host clock around a whole loop that ends in a
device synchronise, after one untimed loop of each) and max |graphed - generic| over the same seeded draws."""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pdae_b200.configs import FFHQ128_PROXY, MNIST  # noqa: E402
from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion  # noqa: E402
from pdae_b200.model.shift_unet import ShiftUNet  # noqa: E402
from pdae_b200.model.unet import UNet  # noqa: E402
from pdae_b200.utils.synth import fill_module_, synth_normal  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit unknown"


def run_loop(kind, gd, net, x, z, z2, ddim):
    with torch.no_grad():
        if kind == "representation":
            return gd.representation_learning_ddpm_sample(None, net, x, x, z)
        if kind == "regular":
            return gd.regular_ddpm_sample(net, x)
        return gd.representation_learning_ddim_trajectory_interpolation(ddim, net, z, z2, x, 0.3)


def timed(fn, steps):
    torch.manual_seed(0)            # the same draws for both loops
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    y = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ddpm-timesteps", type=int, default=100)
    ap.add_argument("--ddim", default="ddim100")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("sampler_bench: needs a CUDA device")
    dev = torch.device("cuda")
    print(json.dumps({"card": card()}))
    gd = GaussianDiffusion({"timesteps": args.ddpm_timesteps, "betas_type": "linear"}, dev)
    gd1000 = GaussianDiffusion({"timesteps": 1000, "betas_type": "linear"}, dev)
    ffhq = fill_module_(ShiftUNet(**FFHQ128_PROXY, latent_dim=512), seed=1).to(dev).eval()
    mnist = fill_module_(UNet(**{k: v for k, v in MNIST.items() if k != "model"}), seed=2).to(dev).eval()
    workloads = [
        ("representation DDPM, ffhq128-proxy, B=5", "representation", gd, ffhq, 5, 3, 128, args.ddpm_timesteps),
        ("regular DDPM, MNIST UNet, B=36", "regular", gd, mnist, 36, 1, 32, args.ddpm_timesteps),
        (f"trajectory interpolation, ffhq128-proxy, B=1, {args.ddim}", "interpolation", gd1000, ffhq, 1, 3, 128,
         int(args.ddim[len("ddim"):])),
    ]
    for name, kind, d, net, B, C, size, steps in workloads:
        x = synth_normal((B, C, size, size), 3).to(dev)
        z, z2 = synth_normal((B, 512), 4).to(dev), synth_normal((B, 512), 5).to(dev)
        for precision in ("bf16x3", "bf16"):
            net.precision = precision
            loops = {"generic": lambda: run_loop(kind, d, lambda a, b, c: net(a, b, c), x, z, z2, args.ddim),
                     "graphed": lambda: run_loop(kind, d, net, x, z, z2, args.ddim)}
            for fn in loops.values():
                fn()                         # warm-up: plan recording, graph capture, lazy module loading
            ms, out = {k: [] for k in loops}, {}
            for _ in range(2):
                for k, fn in loops.items():
                    t, out[k] = timed(fn, steps)
                    ms[k].append(round(t, 3))
            print(json.dumps({"workload": name, "precision": precision, "steps": steps,
                              "generic_ms_per_step": ms["generic"], "graphed_ms_per_step": ms["graphed"],
                              "max_abs_diff": float((out["graphed"] - out["generic"]).abs().max())}))


if __name__ == "__main__":
    main()
