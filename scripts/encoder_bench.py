"""The frozen semantic encoder's forward (the hot path of trainer/train_latent_diffusion.py, trainer/train_manipulation.py and
sampler/infer_latents.py) in each precision mode, and the latent-DPM training step that runs it.

  python scripts/encoder_bench.py [--steps 50] [--warmup 10] [--root DIR]

--root DIR imports pdae_b200 from another checkout (built in place), so that two versions can be timed alternately on one card.
Prints one JSON line per result:
  * the card's name and power limit, read in this run;
  * ms per forward of the 128-px encoder at B = 128 and the 64-px encoder at B = 256, in "fp32", "bf16" and "bf16x3", two
    alternating rounds (CUDA events over --steps calls after --warmup);
  * the device time of each forward plan per kernel kind (Plan.profile), and every stride-2 conv of it (the stem included):
    kernel, shape, us and algorithmic TFLOP/s (2 B Ho Wo Cout Cin 9 over its profiled time);
  * ms per latent-DPM training step including the 128-px encoder (latent_diffusion_train_one_batch + backward, ffhq_latent
    MLPSkipNet, B = 128) with autocast off and on, for each encoder precision."""
import argparse
import json
import os
import subprocess
import sys


def _args():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    return ap.parse_args()


ARGS = _args()
sys.path.insert(0, os.path.abspath(ARGS.root))
import torch  # noqa: E402

import pdae_b200  # noqa: E402
from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion  # noqa: E402
from pdae_b200.model.mlp_skip_net import MLPSkipNet  # noqa: E402
from pdae_b200.model.representation_learning.encoder import CELEBA64Encoder, FFHQEncoder  # noqa: E402
from pdae_b200.utils.synth import fill_module_, synth_images, synth_normal  # noqa: E402

FFHQ_LATENT = dict(input_channel=512, model_channel=2048, num_layers=10, time_emb_channel=64, use_norm=True, dropout=0.0)
DIFF = {"timesteps": 1000, "betas_type": "linear"}
MODES = ("fp32", "bf16", "bf16x3")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit unknown"


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


def stride2_ops(plan):
    """(index, kernel, B, H, W, Cin, Cout) of every stride-2 conv of an encoder forward plan (H, W: its input size)."""
    out = []
    for i, (fn, a) in enumerate(plan.ops):
        if fn == "conv_tc2_s2":
            x3 = bool(a[0].split3)
            out.append((i, "conv_tc2_s2" + ("[x3]" if x3 else ""), a[6], a[7], a[8], a[9] // 3 if x3 else a[9], a[10]))
        elif fn == "conv2d_simt" and a[14] == 2:
            out.append((i, fn, a[8], a[9], a[10], a[11], a[12]))
        elif fn == "stem_conv_s2_bf16":
            out.append((i, fn, a[5], a[6], a[7], a[8], a[9]))
    return out


def main():
    if not torch.cuda.is_available():
        raise SystemExit("encoder_bench: needs a CUDA device")
    dev = torch.device("cuda")
    print(json.dumps({"card": card(), "package": os.path.dirname(os.path.abspath(pdae_b200.__file__))}))
    encs = {(128, 128): fill_module_(FFHQEncoder(latent_dim=512), seed=7), (64, 256): fill_module_(CELEBA64Encoder(latent_dim=512), seed=7)}
    res = {}
    for (size, B), enc in encs.items():
        enc = enc.to(dev).eval().requires_grad_(False)
        x = synth_images(B, 3, size, 33).to(dev)
        for rnd in range(2):
            for mode in MODES:
                enc.precision = mode
                with torch.no_grad():
                    ms = time_ms(lambda: enc(x), ARGS.steps, ARGS.warmup)
                res.setdefault(f"{size}px B={B}", {}).setdefault(mode, []).append(round(ms, 3))
        for mode in MODES:
            plan = [v for k, v in enc._plans().items() if k[1] == mode][0][0]
            prof = plan.profile(reps=5)
            kinds = {k: {"ms": round(v["ms"], 4), "launches": v["launches"]} for k, v in sorted(prof.items(), key=lambda kv: -kv[1]["ms"])}
            print(json.dumps({"plan": f"{size}px B={B} {mode}", "total_ms": round(sum(v["ms"] for v in prof.values()), 4),
                              "kinds": kinds}))
            for i, kern, Bm, H, W, Cin, Cout in stride2_ops(plan):
                us = plan.last_op_ms[i] * 1e3
                print(json.dumps({"stride2": f"{size}px {mode}", "kernel": kern, "B": Bm, "H": H, "Cin": Cin, "Cout": Cout,
                                  "us": round(us, 2), "tflops": round(plan.flops[i] / us / 1e6, 2)}))
    print(json.dumps({"encoder_fwd_ms": res}))

    gd = GaussianDiffusion(DIFF, dev)
    mlp = fill_module_(MLPSkipNet(**FFHQ_LATENT), seed=79).to(dev).train()
    enc = encs[(128, 128)]
    x = synth_images(128, 3, 128, 34).to(dev)
    mean, std = (synth_normal((1, 512), 34) * 0.1).to(dev), (synth_normal((1, 512), 35).abs() + 0.5).to(dev)

    def step(amp):
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=amp):
            loss = gd.latent_diffusion_train_one_batch(mlp, enc, x, mean, std)["prediction_loss"]
        loss.backward()
        for p in mlp.parameters():
            p.grad = None

    steps = {}
    for rnd in range(2):
        for mode in MODES:
            enc.precision = mode
            for amp in (False, True):
                ms = time_ms(lambda: step(amp), ARGS.steps, ARGS.warmup)
                steps.setdefault(f"encoder {mode}, amp {'bf16' if amp else 'off'}", []).append(round(ms, 3))
    print(json.dumps({"latent_step_with_encoder_ms": {"B": 128, **steps}}))


if __name__ == "__main__":
    main()
