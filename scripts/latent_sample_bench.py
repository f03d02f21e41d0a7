"""The latent DPM's sampling side: the frozen ffhq_latent MLPSkipNet forward (512 -> 2048 x 10 layers, config/ffhq_latent.yml)
in every precision mode, and its DDIM latent loop on the one-graph-per-step path against the generic per-step loop (the same
network wrapped in a lambda, so every step replays its per-row plan from Python and runs the update as a separate call).

  python scripts/latent_sample_bench.py [--tree DIR] [--batches 8,128,256] [--ddim ddim100] [--reps 50]

--tree: import pdae_b200 from another checkout (e.g. the parent commit, built) to compare two versions in one session; the
script only uses the public surface (module call, DDIM.latent_ddim_sample_loop), so both versions run the same timing code.
Prints one JSON line per result: the card's name and power limit, read in this run; then per precision and batch size the ms
per forward (CUDA events around --reps calls, after warm-up), and per precision and batch size the ms per loop step of the
generic and the graphed loop in two alternating rounds (CUDA events around a whole loop, after one untimed loop of each) and
max |graphed - generic| over the same z_T."""
import argparse
import json
import os
import subprocess
import sys


def card(torch):
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit unknown"


def events_ms(torch, fn, reps):
    """Mean ms of fn() over `reps` calls, CUDA events on the current stream around all of them (fn enqueues device work)."""
    st = torch.cuda.current_stream()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record(st)
    for _ in range(reps):
        out = fn()
    b.record(st)
    b.synchronize()
    return a.elapsed_time(b) / reps, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tree", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    ap.add_argument("--batches", default="8,128,256")
    ap.add_argument("--ddim", default="ddim100")
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--precisions", default="bf16,bf16x3,fp32")
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.tree))
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("latent_sample_bench: needs a CUDA device")
    from pdae_b200.configs import FFHQ_LATENT
    from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
    from pdae_b200.model.mlp_skip_net import MLPSkipNet
    from pdae_b200.utils.synth import fill_module_, synth_normal
    dev = torch.device("cuda")
    print(json.dumps({"card": card(torch), "tree": os.path.abspath(args.tree)}))
    mlp = fill_module_(MLPSkipNet(**{k: v for k, v in FFHQ_LATENT.items() if k != "model"}), seed=5).eval().to(dev)
    gd = GaussianDiffusion({"timesteps": 1000, "betas_type": "linear"}, dev)
    ddim = gd._ddim(args.ddim, gd.latent_diffusion_config["alphas_cumprod"])
    steps = ddim.timesteps
    batches = [int(b) for b in args.batches.split(",")]
    precisions = args.precisions.split(",")
    for precision in precisions:
        mlp.precision = precision
        for B in batches:
            z = synth_normal((B, 512), 1).to(dev)
            t = torch.linspace(0, 999, B).round().long().to(dev)
            with torch.inference_mode():
                for _ in range(3):
                    mlp(z, t)
                ms, _ = events_ms(torch, lambda: mlp(z, t), args.reps)
            print(json.dumps({"workload": "ffhq_latent forward (per-row t)", "precision": precision, "B": B,
                              "ms_per_forward": round(ms, 4)}))
    for precision in precisions:
        mlp.precision = precision
        for B in batches:
            zT = synth_normal((B, 512), 2).clamp(-1, 1).to(dev)
            loops = {"generic": lambda: ddim.latent_ddim_sample_loop(lambda a, b, c=None: mlp(a, b), zT),
                     "graphed": lambda: ddim.latent_ddim_sample_loop(mlp, zT)}
            with torch.inference_mode():
                for fn in loops.values():
                    fn()                     # warm-up: plan recording, graph capture, lazy module loading
                ms, out = {k: [] for k in loops}, {}
                for _ in range(2):
                    for k, fn in loops.items():
                        t, out[k] = events_ms(torch, fn, 1)
                        ms[k].append(round(t / steps, 4))
            print(json.dumps({"workload": f"ffhq_latent latent loop {args.ddim}", "precision": precision, "B": B, "steps": steps,
                              "generic_ms_per_step": ms["generic"], "graphed_ms_per_step": ms["graphed"],
                              "max_abs_diff": float((out["graphed"] - out["generic"]).abs().max())}))


if __name__ == "__main__":
    main()
