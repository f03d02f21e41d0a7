"""One AttentionBlock's training step under bf16 autocast: the tensor-core attention (bf16 qkv, probabilities from the softmax
GEMM epilogue, softmax gradient in the dP GEMM's epilogue, transposed-operand GEMMs for dV / dQ / dK) against the CUDA-core
attention (attention_simt forward; gemm_batched_simt + softmax_bwd backward), both inside the same bf16 training plans.

  python scripts/attention_train_bench.py [--batch 32] [--reps 50] [--warmup 5]

Times the forward plan and the backward plan of one block with CUDA events over --reps replays after --warmup, and prints the
card's name and power limit, µs per pass, and algorithmic TFLOP/s of the attention core computed from shapes
(forward 4 B T^2 C, backward 8 B T^2 C; the block's 1x1 convs and GroupNorm are in the time but not in the FLOPs)."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch

from pdae_b200.engine import Plan
from pdae_b200.model.module import AttentionBlock, Src
from pdae_b200.train import Backward, GradSink, bwd_plan
from pdae_b200.utils.synth import fill_module_

SHAPES = [(256, 256, 1), (256, 384, 1), (256, 256, 4)]   # (T, C, heads) at 16 x 16


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        return out[torch.cuda.current_device()] if out else torch.cuda.get_device_name()
    except (OSError, subprocess.SubprocessError):
        return torch.cuda.get_device_name() + ", power limit unknown"


def build(blk, B, H, W, C, tensor_cores):
    """Forward and backward plans of one block in a bf16 training step; tensor_cores=False takes the CUDA-core attention."""
    dev = torch.device("cuda")
    elig = AttentionBlock.__dict__["amp_eligible"]      # (the staticmethod object itself, to put back)
    if not tensor_cores:
        AttentionBlock.amp_eligible = staticmethod(lambda T, ch: False)
    try:
        P = Plan(dev, "fp32")
        P.keep_all = True
        P.train_tc = "bf16"
        xin = P.new((B, H, W, C), torch.float32, "x")
        xin.keep = True
        tape = []
        y = blk.emit(P, Src(xin, C, B, H, W), tape=tape)
        y.b1.keep = True
        P.finalize()
    finally:
        AttentionBlock.amp_eligible = elig
    BP = bwd_plan(dev, True)
    bw = Backward(BP, GradSink())
    dy = BP.new((B, H, W, C), torch.float32, "dy")
    dy.keep = True
    (_, mod, sv), = tape
    bw.attention(mod, sv, dy).keep = True
    BP.finalize()
    g = torch.Generator(device="cpu").manual_seed(0)
    xin.tensor.copy_(torch.randn(B, H, W, C, generator=g))
    dy.tensor.copy_(torch.randn(B, H, W, C, generator=g) * 0.1)
    return P, BP


def time_plan(plan, reps, warmup):
    for _ in range(warmup):
        plan.run()
    st = torch.cuda.current_stream()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record(st)
    for _ in range(reps):
        plan.run()
    e1.record(st)
    e1.synchronize()
    return e0.elapsed_time(e1) * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=32)
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("attention_train_bench: needs a CUDA device")
    B = args.batch
    print(json.dumps({"card": card()}))
    for T, C, heads in SHAPES:
        H = W = int(round(T ** 0.5))
        blk = fill_module_(AttentionBlock(C, heads, -1, False), seed=3).cuda().train()
        fl_f, fl_b = 4.0 * B * T * T * C, 8.0 * B * T * T * C
        res = {"B": B, "T": T, "C": C, "heads": heads}
        for name, tc in (("tc", True), ("simt", False)):
            P, BP = build(blk, B, H, W, C, tc)
            P.run()
            tf, tb = time_plan(P, args.reps, args.warmup), time_plan(BP, args.reps, args.warmup)
            res[name] = {"fwd_us": round(tf, 1), "bwd_us": round(tb, 1), "fwd_tflops": round(fl_f / tf / 1e6, 2),
                         "bwd_tflops": round(fl_b / tb / 1e6, 2)}
            del P, BP
        print(json.dumps(res))


if __name__ == "__main__":
    main()
