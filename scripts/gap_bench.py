"""The gap measure (GaussianDiffusion.representation_learning_gap_measure, sampler/gap_measure.py of the reference) on the
one-graph-per-step path, against the generic per-step loop (the same decoder wrapped in a lambda, so every step replays its
plan from Python, runs the posterior-mean arithmetic as torch ops and syncs the host twice for `.cpu().item()`).

  python scripts/gap_bench.py [--timesteps 50] [--precisions bf16,bf16x3]

Workloads: the celeba64-proxy ShiftUNet at B = 16 and B = 100, and the ffhq128-proxy ShiftUNet at B = 100 (the reference's
gap-measure configuration).  The semantic encoder runs once per call and is not part of the loop, so a fixed z stands in
for it.  Every step does the same work whatever its t, so a shortened schedule (--timesteps; the reference uses 1000) gives
the per-step time of the full loop; the JSON lines state the schedule length used.
Prints one JSON line per result: the card's name and power limit, read in this run; then per workload and precision the
ms per step of the generic and the graphed loop in two alternating rounds (host clock around a whole call that ends in a
device synchronise, after one untimed call of each), their ratio (generic / graphed, mean of the rounds), and the largest
absolute and relative difference between the two loops' gap lists on the same seeded draws and weights."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pdae_b200.configs import CELEBA64_PROXY, FFHQ128_PROXY  # noqa: E402
from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion  # noqa: E402
from pdae_b200.model.shift_unet import ShiftUNet  # noqa: E402
from pdae_b200.utils.synth import fill_module_, synth_images, synth_normal  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit unknown"


def timed(gd, net, x0, z, steps):
    torch.manual_seed(0)            # the same draws for both loops
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    with torch.no_grad():
        gp, ga = gd.representation_learning_gap_measure(lambda x: z, net, x0)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3 / steps, np.array([gp, ga], dtype=np.float64)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--timesteps", type=int, default=50)
    ap.add_argument("--precisions", default="bf16,bf16x3")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gap_bench: needs a CUDA device")
    dev = torch.device("cuda")
    print(json.dumps({"card": card(), "timesteps": args.timesteps,
                      "note": "shortened schedule: per-step work does not depend on t" if args.timesteps != 1000 else ""}))
    gd = GaussianDiffusion({"timesteps": args.timesteps, "betas_type": "linear"}, dev)
    celeba = fill_module_(ShiftUNet(**CELEBA64_PROXY, latent_dim=512), seed=1).to(dev).eval()
    ffhq = fill_module_(ShiftUNet(**FFHQ128_PROXY, latent_dim=512), seed=2).to(dev).eval()
    workloads = [("celeba64-proxy, B=16", celeba, 16, 64), ("celeba64-proxy, B=100", celeba, 100, 64),
                 ("ffhq128-proxy, B=100", ffhq, 100, 128)]
    for name, net, B, size in workloads:
        x0 = synth_images(B, 3, size, 3).to(dev)
        z = synth_normal((B, 512), 4).to(dev)
        for precision in args.precisions.split(","):
            net.precision = precision
            loops = {"generic": lambda a, b, c: net(a, b, c), "graphed": net}
            for fn in loops.values():
                timed(gd, fn, x0, z, args.timesteps)     # warm-up: plan recording, graph capture, lazy module loading
            ms, out = {k: [] for k in loops}, {}
            for _ in range(2):
                for k, fn in loops.items():
                    t, out[k] = timed(gd, fn, x0, z, args.timesteps)
                    ms[k].append(round(t, 3))
            diff = np.abs(out["graphed"] - out["generic"])
            print(json.dumps({"workload": name, "precision": precision, "timesteps": args.timesteps,
                              "generic_ms_per_step": ms["generic"], "graphed_ms_per_step": ms["graphed"],
                              "generic_over_graphed": round(float(np.mean(ms["generic"]) / np.mean(ms["graphed"])), 4),
                              "max_abs_diff": float(diff.max()),
                              "max_rel_diff": float((diff / np.abs(out["generic"])).max())}), flush=True)


if __name__ == "__main__":
    main()
