"""Training-step throughput (SURVEY.md section 8(d) config 5): representation_learning_train_one_batch + backward + gradient
all-reduce + fused Adam/EMA step on the celeba64-proxy decoder + encoder.

  python scripts/train_bench.py [--batch 32] [--steps 5] [--amp {off,bf16}] [--deterministic {0,1}]   # 1 GPU
  python -m torch.distributed.run --nproc-per-node N ... scripts/train_bench.py --overlap 1   # N GPUs, batch per GPU fixed

Arithmetic: decoder forward, data gradients (conv_tc2) and weight gradients (wgrad_tc) on the tensor cores in the
split-operand fp32-grade mode; encoder and the stride-2 / 3-channel convs in fp32 on CUDA cores (DESIGN.md).  --amp bf16: the step
runs inside torch.autocast("cuda", dtype=torch.bfloat16) (the reference's enable_amp), so the decoder trains on the bf16
plans: frozen half in the "bf16" mode, single-pass bf16 forward convs, data and weight gradients; so does the encoder's
stride-2 and attention convs (its 3-channel stem and final Linear stay fp32 on CUDA cores).  --overlap 1: the decoder bucket's NCCL all-reduce is launched from a
post-accumulate-grad hook as soon as the ShiftUNet backward has delivered its gradients and runs while the encoder
backward computes (pdae_b200.utils.dist.OverlappedGradAllReduce); --overlap 0: all-reduce after backward.
--deterministic 1: the step runs under torch.use_deterministic_algorithms(True, warn_only=True), so the trainers record their
deterministic plans (no float atomics; bitwise-reproducible on one GPU).  Rank 0 prints one JSON line (with the card's name
and power limit)."""
import argparse
import copy
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import torch.distributed as dist

from bench import WORKLOADS
from pdae_b200.diffusion.gaussian_diffusion import GaussianDiffusion
from pdae_b200.model.representation_learning.encoder import CELEBA64Encoder
from pdae_b200.model.shift_unet import ShiftUNet
from pdae_b200.optim import FusedAdamEMA
from pdae_b200.utils.dist import OverlappedGradAllReduce, allreduce_grads_
from pdae_b200.utils.synth import fill_module_, synth_images

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=32)
ap.add_argument("--steps", type=int, default=5)
ap.add_argument("--overlap", type=int, default=1)
ap.add_argument("--amp", choices=("off", "bf16"), default="off")
ap.add_argument("--deterministic", type=int, choices=(0, 1), default=0)
args = ap.parse_args()
if args.deterministic:
    torch.use_deterministic_algorithms(True, warn_only=True)
world = int(os.environ.get("WORLD_SIZE", "1"))
rank = int(os.environ.get("RANK", "0"))
local = int(os.environ.get("LOCAL_RANK", "0"))
dev = torch.device("cuda", local)
torch.cuda.set_device(dev)
if os.environ.get("NCCL_DEBUG", "").upper() in ("", "VERSION"):
    os.environ["NCCL_DEBUG"] = "WARN"
if world > 1:
    dist.init_process_group("nccl", device_id=dev)
B = args.batch
cfg, size = WORKLOADS["celeba64"][0], WORKLOADS["celeba64"][1]
dec = fill_module_(ShiftUNet(latent_dim=512, **dict(cfg, dropout=0.1)), seed=0).to(dev)
enc = fill_module_(CELEBA64Encoder(latent_dim=512), seed=1).to(dev).train()
dec.freeze()
dec.set_train_mode()
dec.precision = enc.precision = "fp32"
ema_dec, ema_enc = copy.deepcopy(dec).requires_grad_(False), copy.deepcopy(enc).requires_grad_(False)
gd = GaussianDiffusion({"timesteps": 1000, "betas_type": "linear"}, dev)
groups = [list(enc.parameters()), list(dec.label_emb.parameters()), list(dec.shift_middle_block.parameters()),
          list(dec.shift_output_blocks.parameters()), list(dec.shift_out.parameters())]
opt = FusedAdamEMA([{"params": g} for g in groups], lr=1e-4, ema_decay=0.9999)
opt.attach_ema(enc, ema_enc)
opt.attach_ema(dec, ema_dec)
x0 = synth_images(B, 3, size, 3 + rank).to(dev)
dec_params = [p for g in groups[1:] for p in g]
red = OverlappedGradAllReduce([dec_params, groups[0]]) if (world > 1 and args.overlap) else None
all_params = [p for g in groups for p in g]


def step():
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=args.amp == "bf16"):
        loss = gd.representation_learning_train_one_batch(enc, dec, x0)["prediction_loss"]
    loss.backward()
    scale = red.finish() if red is not None else allreduce_grads_(all_params)
    opt.step(grad_scale=scale)
    opt.zero_grad(set_to_none=True)
    return loss


for _ in range(3):
    step()
if world > 1:
    dist.barrier()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(args.steps):
    loss = step()
e1.record()
torch.cuda.synchronize()
ms = torch.tensor([e0.elapsed_time(e1) / args.steps], device=dev)
if world > 1:
    dist.all_reduce(ms, op=dist.ReduceOp.MAX)
ms = float(ms)
n_train = sum(p.numel() for p in all_params)
if rank == 0:
    res = {"metric": "pdae_training_images_per_sec", "value": round(world * B / ms * 1e3, 2), "unit": "images/s",
           "n_gpus": world, "batch_per_gpu": B, "ms_per_step": round(ms, 2), "steps": args.steps, "warmup": 3,
           "scaling": "weak", "grad_allreduce": ("overlapped with the encoder backward" if red is not None else
                                                 ("after backward" if world > 1 else "none (1 GPU)")),
           "trainable_params": n_train, "allreduce_bytes_per_step": 4 * n_train if world > 1 else 0,
           "config": "celeba64-proxy encoder + ShiftUNet (shift half trainable), dropout 0.1, fused Adam+EMA; decoder "
                     "forward, data and weight gradients on the tensor cores (split-operand, fp32-grade); encoder "
                     "and stride-2 / 3-channel convs on CUDA cores (fp32)", "loss": float(loss.detach()),
           "deterministic": bool(args.deterministic), "gpu": torch.cuda.get_device_name(dev)}
    try:
        import subprocess
        res["power_limit_w"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader,nounits",
                                               "-i", str(dev.index)], capture_output=True, text=True).stdout.strip()
    except OSError:
        pass
    if args.amp != "off":
        res["amp"] = args.amp
        res["config"] = ("celeba64-proxy encoder + ShiftUNet (shift half trainable), dropout 0.1, fused Adam+EMA, bf16 autocast; "
                         "frozen decoder half in bf16, trainable decoder forward, data and weight gradients as single-pass "
                         "bf16 MMAs on the tensor cores, and so are the encoder's stride-2 and attention convs; fp32 "
                         "activations, GroupNorm and attention backward; 3-channel convs and the encoder's Linear on CUDA "
                         "cores (fp32)")
    print(json.dumps(res))
if world > 1:
    dist.destroy_process_group()
