"""Cost of torch.use_deterministic_algorithms: each workload timed with the switch off (default plans) and on (deterministic
plans), alternated twice in one process, with the largest |deterministic - default| of its output.
  * the ShiftUNet decoder step (one CUDA-graph replay) at celeba64-proxy B = 256 and ffhq128-proxy B = 64, "bf16x3" and "bf16";
  * the latent ddim100 loop of the ffhq_latent MLPSkipNet at B = 256 ("bf16");
  * the 128-px encoder's forward at B = 128 ("bf16").
usage: python scripts/deterministic_bench.py [--reps N] [--out FILE]   (card name and power limit are part of the output)"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from bench import WORKLOADS
from pdae_b200.utils.synth import fill_module_, synth_images, synth_normal

DEV = torch.device("cuda")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def events_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def decoder_step(wl, B, precision):
    from pdae_b200.model.shift_unet import ShiftUNet
    cfg, size = WORKLOADS[wl][0], WORKLOADS[wl][1]
    dec = fill_module_(ShiftUNet(latent_dim=512, **cfg), seed=0).eval().to(DEV)
    dec.precision = precision
    x, z = synth_normal((B, 3, size, size), 1).to(DEV), synth_normal((B, 512), 2).to(DEV)
    t = torch.full((B,), 500, device=DEV, dtype=torch.long)

    def setup():
        with torch.no_grad():
            out = torch.cat([o.flatten() for o in dec(x, t, z)])
        plan, _ = dec.plan_for(B, size, size)
        plan.capture_graph()
        return out, lambda: plan.run(prologue=False)
    return f"decoder step {wl}-proxy B={B} {precision}", setup


def latent_loop(B):
    from pdae_b200.diffusion.ddim import DDIM
    from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
    from pdae_b200.model.mlp_skip_net import MLPSkipNet
    from tests import cases
    from tests.configs import FFHQ_LATENT
    m = fill_module_(MLPSkipNet(**{k: v for k, v in FFHQ_LATENT.items() if k != "model"}), seed=3).eval().to(DEV)
    m.precision = "bf16"
    d = GaussianDiffusion(cases.DIFF, DEV)
    nb, tmap = d.get_ddim_betas_and_timestep_map("ddim100", d.latent_diffusion_config["alphas_cumprod"].cpu().numpy())
    dd = DDIM(nb, tmap, DEV)
    zT = synth_normal((B, 512), 4).to(DEV)

    def setup():
        def run():
            with torch.no_grad():
                return dd.latent_ddim_sample_loop(m, zT)
        return run(), run
    return f"latent ddim100 loop B={B} bf16", setup


def encoder_forward(B):
    from pdae_b200.model.representation_learning.encoder import FFHQEncoder
    enc = fill_module_(FFHQEncoder(latent_dim=512), seed=5).eval().to(DEV)
    enc.precision = "bf16"
    x = synth_images(B, 3, 128, 6).to(DEV)

    def setup():
        def run():
            with torch.no_grad():
                return enc(x)
        return run(), run
    return f"encoder 128px forward B={B} bf16", setup


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    gpu = card()
    print(f"[det-bench] card: {gpu}", flush=True)
    work = [decoder_step("celeba64", 256, "bf16x3"), decoder_step("celeba64", 256, "bf16"),
            decoder_step("ffhq128", 64, "bf16x3"), decoder_step("ffhq128", 64, "bf16"), latent_loop(256), encoder_forward(128)]
    rows = []
    for name, setup in work:
        ms = {False: [], True: []}
        outs = {}
        for rnd in range(2):
            for det in (False, True):
                torch.use_deterministic_algorithms(det, warn_only=True)
                out, fn = setup()
                outs[det] = out
                reps = args.reps if "loop" not in name else max(2, args.reps // 10)
                ms[det].append(events_ms(fn, reps))
        torch.use_deterministic_algorithms(False)
        off, on = min(ms[False]), min(ms[True])
        row = {"workload": name, "default_ms": [round(v, 4) for v in ms[False]], "det_ms": [round(v, 4) for v in ms[True]],
               "det_over_default": round(on / off, 4), "max_abs_det_minus_default": float((outs[True] - outs[False]).abs().max()),
               "card": gpu}
        rows.append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
